"""Loader for the in-tree native extensions.

``_C``    – sm_90a kernels + C++ step-plan runtime (needs an H100 at run time, imports anywhere)
``_host`` – CPU-only native helpers (TF bundle codec, crc32c, carrier codec, CSV reader)

On a GPU box the CUDA path is THE path: if ``_C.so`` is missing we fail loudly instead of silently
falling back to eager PyTorch.
"""
from __future__ import annotations

import importlib.util
import os
import sys
from pathlib import Path
from types import ModuleType

_PKG_DIR = Path(__file__).resolve().parents[1]
_cache: dict[str, ModuleType] = {}


class NativeExtensionMissing(RuntimeError):
    pass


def _load(name: str) -> ModuleType:
    if name in _cache:
        return _cache[name]
    so = _PKG_DIR / f"{name}.so"
    if not so.exists():
        if os.environ.get("SPARKFLOW_NO_AUTOBUILD") != "1":
            try:
                sys.path.insert(0, str(_PKG_DIR.parent))
                from tools.build_ext import build  # type: ignore

                build(only="cuda" if name == "_C" else "host")
            except Exception as exc:  # pragma: no cover - build environment specific
                raise NativeExtensionMissing(
                    f"native extension {so} is missing and could not be built: {exc}. "
                    "Run `python tools/build_ext.py`."
                ) from exc
            finally:
                sys.path.pop(0)
        if not so.exists():
            raise NativeExtensionMissing(f"native extension {so} is missing; run `python tools/build_ext.py`")
    full = f"sparkflow_b200.{name}"
    spec = importlib.util.spec_from_file_location(full, so)
    assert spec and spec.loader
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules[full] = mod
    _cache[name] = mod
    return mod


_err_channel_devices = set()

WAIT_CODES = {0x100: "gemm: TMA producer waiting for a free smem stage", 0x200: "gemm: MMA issuer waiting for operands",
              0x300: "gemm: epilogue waiting for the accumulator", 0x401: "rw lock: write acquire", 0x402: "rw lock: read acquire",
              0x403: "push: CTA waiting for the lock grant", 0x404: "pull: CTA waiting for the lock grant",
              0x405: "pull / first GEMM: read-your-writes wait for the applier(s) to acknowledge my last post",
              0x406: "post: waiting for my mailbox to be consumed", 0x407: "applier: leader waiting for the other CTAs",
              0x408: "applier: follower CTA waiting for the leader's decision", 0x409: "applier: stale pull registrations (double-buffered publish)",
              0x40B: "sync_pull: CTAs of a shard waiting for each other's version",
              0x40C: "sync_pull: no consistent snapshot of a shard within the bound", 0x40D: "sync_pull: waiting for the shard leader's version pick"}


def cuda_ext() -> ModuleType:
    """The sm_90a kernel/runtime module (``sparkflow_b200._C``).  On a CUDA machine the first call per device
    also installs the host-visible error word that bounded device waits write before trapping."""
    mod = _load("_C")
    try:
        import torch

        if torch.cuda.is_available():
            dev = torch.cuda.current_device()
            if dev not in _err_channel_devices:
                mod.init_error_channel()
                _err_channel_devices.add(dev)
    except Exception:  # pragma: no cover
        pass
    return mod


def describe_device_error() -> str:
    """Human-readable form of the last bounded-wait failure (readable even after the CUDA context died)."""
    code = _load("_C").read_host_error_code()
    if not code:
        return "no device-side wait failure recorded"
    base = code & 0xFFF
    key = base if base in WAIT_CODES else (base & 0xF00)
    return f"device wait failure 0x{base:x} (block {code >> 12}): {WAIT_CODES.get(key, 'unknown')}"


def host_ext() -> ModuleType:
    """The CPU-only native helper module (``sparkflow_b200._host``)."""
    return _load("_host")


def num_sms() -> int:
    """SMs of the current CUDA device (132, an H100 SXM, when no device is visible)."""
    import torch

    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count if torch.cuda.is_available() else 132


def ptr(t) -> int:
    """Device address of a torch tensor (0 for ``None``)."""
    return 0 if t is None else int(t.data_ptr())


def current_stream() -> int:
    import torch

    return int(torch.cuda.current_stream().cuda_stream)
