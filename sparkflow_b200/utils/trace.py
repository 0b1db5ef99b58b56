"""Device-side timeline tracer (the framework's profiling subsystem; the reference has none).

Every kernel's CTA 0..n stamps ``%globaltimer`` at entry, after its programmatic-dependency wait and at
exit.  :class:`DeviceTrace` turns the raw records into one row per kernel launch with start / ready /
end times, so launch gaps, PDL overlap and branch concurrency of a CUDA-graph step are visible without
a profiler attached (ncu serialises kernels; this does not)."""
from __future__ import annotations

import os
from typing import Dict, List

import numpy as np
import torch

from ..ops import native

KERNEL_NAMES = {1: "gemm", 2: "cast_transpose", 3: "softmax_xent", 4: "mse", 5: "argmax", 6: "push", 7: "pull", 8: "im2col",
                9: "col2im", 10: "maxpool_fwd", 11: "maxpool_bwd", 12: "maxpool_gen_fwd", 13: "maxpool_gen_bwd", 14: "act_bwd_bias",
                15: "sigmoid_xent", 16: "sparse_softmax_xent"}


class DeviceTrace:
    def __init__(self, capacity: int = 1 << 16, device=None):
        self.C = native.cuda_ext()
        self.capacity = capacity
        self.buf = torch.zeros(capacity * 32, dtype=torch.uint8, device=device or "cuda")

    def __enter__(self):
        torch.cuda.current_stream().synchronize()      # stream-level: a persistent applier kernel may be resident
        self.C.trace_enable(native.ptr(self.buf), self.capacity)
        return self

    def __exit__(self, *exc):
        torch.cuda.current_stream().synchronize()
        self.n = min(self.C.trace_count(), self.capacity)
        self.C.trace_enable(0, 0)
        return False

    def records(self) -> np.ndarray:
        raw = self.buf[: self.n * 32].cpu().numpy()
        dt = np.dtype([("t0", "<u8"), ("t1", "<u8"), ("t2", "<u8"), ("kid", "<u4"), ("block", "<u4")])
        return raw.view(dt)

    def launches(self, gap_ns: int = 300) -> List[Dict[str, float]]:
        """Group CTA records into launches (same kernel id, entry times clustered) sorted by start."""
        rec = np.sort(self.records(), order="t0")
        out: List[Dict[str, float]] = []
        if len(rec) == 0:
            return out
        base = int(rec["t0"][0])
        groups: Dict[int, Dict[str, float]] = {}
        for r in rec:
            k = int(r["kid"])
            g = groups.get(k)
            if g is None or int(r["t0"]) - g["_last_t0"] > gap_ns and int(r["block"]) == 0 or int(r["t0"]) > g["end_abs"] + gap_ns:
                g = {"kernel": KERNEL_NAMES.get(k, str(k)), "start_abs": int(r["t0"]), "ready_abs": int(r["t1"]), "end_abs": int(r["t2"]),
                     "ctas": 0, "_last_t0": int(r["t0"])}
                groups[k] = g
                out.append(g)
            g["ctas"] += 1
            g["_last_t0"] = int(r["t0"])
            g["ready_abs"] = max(g["ready_abs"], int(r["t1"]))
            g["end_abs"] = max(g["end_abs"], int(r["t2"]))
        for g in out:
            g["start_us"] = (g.pop("start_abs") - base) / 1e3
            g["ready_us"] = (g.pop("ready_abs") - base) / 1e3
            g["end_us"] = (g.pop("end_abs") - base) / 1e3
            g.pop("_last_t0")
        return out


# ---------------------------------------------------------------------------------------------------------------------
# NVTX ranges (SPARKFLOW_NVTX=1): partition / iteration ranges of the worker loop for nsys / ncu range filters.  Off by
# default: the hot loop pays nothing.
# ---------------------------------------------------------------------------------------------------------------------
_NVTX = os.environ.get("SPARKFLOW_NVTX") == "1"


def nvtx_push(name: str) -> None:
    if _NVTX and torch.cuda.is_available():
        torch.cuda.nvtx.range_push(name)


def nvtx_pop() -> None:
    if _NVTX and torch.cuda.is_available():
        torch.cuda.nvtx.range_pop()
