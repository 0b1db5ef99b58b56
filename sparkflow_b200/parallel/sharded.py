"""Sharded parameter server: the master state is partitioned over ALL GPUs of the box.

The reference has ONE parameter server on the Spark driver: every ``GET /parameters`` and ``POST /update`` terminates
there (lifeomic/sparkflow/sparkflow/HogwildSparkModel.py:206-244).  On an H100 box that star topology wastes 7/8 of the
NVLink ports and serialises every optimizer step on one GPU.  Here (SURVEY.md section 5.1, "sharded master"):

* the flat state (one ``(p, slot0, slot1, slot2)`` tuple per parameter) is split by *push tile* (32 x 64 elements of one
  variable): shard ``r`` = tiles ``[T*r/S, T*(r+1)/S)`` lives on GPU ``r``;
* **push**: a worker's wgrad epilogues store every gradient tile straight into that worker's mailbox on the GPU that owns
  the tile (NVLink peer stores issued by the GEMM epilogue - no local gradient buffer, no copy kernel); one tiny kernel
  then posts a sequence number to every shard (``st.release.sys``);
* **apply**: every GPU runs an applier for its shard (``applier_kernel`` restricted to its tile range): all posted
  mailboxes are applied back to back in registers - each push still its own optimizer step, as in the reference - and the
  new bf16 ``W`` / ``W^T`` (+ the fp32 1-D tail) are **published into every GPU's replica with ``multimem.st``** (one
  store, replicated by the NVSwitch), bracketed by per-shard seqlock stamps; the applier then acknowledges each consumed
  push with a store into the *worker's own* memory;
* **pull**: nothing crosses NVLink.  The worker waits (local spin) until every shard acknowledged its last push
  (read-your-writes, like the blocking HTTP POST of the reference) and, with ``acquire_lock=True``, takes a seqlock
  snapshot of each shard's slice of the local inbox replica; Hogwild reads the inbox in place.

Consistency: with ``acquire_lock=True`` a pull never observes a partially applied update *of a shard* (the unit of
atomicity is the shard, as in any sharded parameter server, e.g. TF's own multi-``ps`` jobs); ``SPARKFLOW_PUSH_MODE=served``
keeps the single-master mode with whole-model atomicity.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from ..ops import native
from ..ops.layout import ParamLayout, round_up
from ..ops.optimizers import OptimizerSpec
from . import dist as D
from .device_engine import _sync_current, _view
from .symm import SymmetricHeap

_ALIGN = 256
VER_STRIDE = 32            # uint32 words between two shards' stamp pairs (begin at +0, end at +16: separate 64 B lines)
ACK_STRIDE = 16            # uint32 words between two shards' acknowledgement words inside a worker's segment


def shard_bounds(n_tiles: int, n_shards: int) -> List[int]:
    """Shard r owns push tiles [bounds[r], bounds[r + 1])."""
    return [(n_tiles * r) // n_shards for r in range(n_shards + 1)]


class ShardedMaster:
    """All shards as seen from one process (SPMD: the process owns shard ``rank``; single process: it owns all of them)."""

    sharded = True
    served = False
    dbuf_active = False

    def __init__(self, layout: ParamLayout, spec: OptimizerSpec, ctx: D.DistContext, devices: Sequence[torch.device],
                 mb_zero: bool = False):
        self.C = native.cuda_ext()
        self.layout, self.spec, self.ctx = layout, spec, ctx
        self.devices = list(devices)
        self.spmd = ctx.world > 1
        self.n = ctx.world if self.spmd else len(self.devices)
        if self.n > self.C.MAX_SHARDS:
            raise RuntimeError(f"at most {self.C.MAX_SHARDS} shards")
        self.my_shards = [ctx.rank] if self.spmd else list(range(self.n))
        self.device = self.devices[0]                  # "the" device of this process (SPMD) / of shard 0 (single process)
        self.mb_zero = bool(mb_zero)
        self.tiles = layout.tile_map()
        self.n_tiles = int(self.tiles.shape[0])
        self.bounds = shard_bounds(self.n_tiles, self.n)
        self.tile_prefix = layout.tile_prefix()
        C, lay = self.C, layout
        # ---- publish segment (multicast-bound): stamps | bf16 shadow | fp32 1-D tail ----
        off = 0

        def take(nbytes: int) -> int:
            nonlocal off
            start = off
            off = round_up(off + nbytes, _ALIGN)
            return start

        self.o_stamps = take(self.C.MAX_SHARDS * VER_STRIDE * 4)
        self.o_shadow = take(lay.shadow_total * 2)
        self.o_vec = take(max(lay.vec_count, 4) * 4)
        # second publish slot (lock mode: pass v lands in slot v & 1, a pull copies the newest complete pass and never
        # waits for one in flight); Hogwild uses slot 0 only
        self.o_shadow1 = take(lay.shadow_total * 2)
        self.o_vec1 = take(max(lay.vec_count, 4) * 4)
        self.slot_off_bf16 = (self.o_shadow1 - self.o_shadow) // 2
        self.slot_off_f32 = (self.o_vec1 - self.o_vec) // 4
        pub_bytes = off
        # ---- shard segment: ctrl | state | flags | applier sync | acks | mailboxes ----
        off = 0
        self.o_ctrl = take(C.CTRL_WORDS * 4)
        self.o_state = take(lay.total * 16)
        self.o_flags = take(self.n * C.MB_WORDS * 4)
        self.o_sync = take(64)
        self.o_ack = take(self.C.MAX_SHARDS * ACK_STRIDE * 4)
        self.o_heart = take(64)                         # worker heartbeat: (globaltimer ns of the last post, posts so far)
        self.mb_stride = round_up(lay.total, 64)
        self.o_mail = take(self.n * self.mb_stride * 4)
        seg_bytes = off
        idx = [d.index for d in self.devices]
        self.pub = SymmetricHeap(pub_bytes, ctx if self.spmd else None, idx, multicast=True, tag="pub")
        self.seg = SymmetricHeap(seg_bytes, ctx if self.spmd else None, idx, multicast=False, tag="seg")
        self.multicast = self.pub.multicast
        self.appliers: Dict[int, object] = {}
        self._stats: Dict[int, torch.Tensor] = {}
        self._keep: List[object] = []
        self._owner_index: Optional[List[torch.Tensor]] = None

    # ---- addressing ---------------------------------------------------------------------------------------
    def dev_of(self, shard: int) -> torch.device:
        return self.devices[0] if self.spmd else self.devices[shard]

    def seg_ptr(self, shard: int, off: int) -> int:
        return self.seg.base[shard] + off

    def pub_ptr(self, shard: int, off: int) -> int:
        return self.pub.base[shard] + off

    def mailbox_ptr(self, shard: int, worker: int) -> int:
        return self.seg.base[shard] + self.o_mail + worker * self.mb_stride * 4

    def posted_ptr(self, shard: int, worker: int) -> int:
        return self.seg.base[shard] + self.o_flags + worker * self.C.MB_WORDS * 4

    def ack_ptr(self, worker: int, shard: int) -> int:
        """Where shard ``shard`` acknowledges worker ``worker``: a word inside the WORKER's segment."""
        return self.seg.base[worker] + self.o_ack + shard * ACK_STRIDE * 4

    def heartbeat_ptr(self, worker: int) -> int:
        return self.seg.base[worker] + self.o_heart

    def worker_status(self, stale_after_s: float = 5.0) -> List[Dict[str, float]]:
        """Watchdog view (SURVEY.md section 5, failure detection): per worker the number of posts and the age of its last
        one.  ``stale`` marks workers that posted before but have been silent for ``stale_after_s`` - the sharded
        protocol needs no action for them (a dead worker simply stops posting; nothing waits on it), this is for
        operators / the session log."""
        dev = self.devices[0]
        out = []
        with torch.cuda.device(dev):
            now = None
            for w in range(self.n):
                hb = _view(self.heartbeat_ptr(w), 16, torch.int64, dev).cpu()
                t, n = int(hb[0]), int(hb[1])
                now = max(now or 0, t)
                out.append({"worker": w, "posts": n, "last_post_ns": t})
        for o in out:
            o["age_s"] = (now - o["last_post_ns"]) / 1e9 if o["posts"] else float("inf")
            o["stale"] = bool(o["posts"] and o["age_s"] > stale_after_s)
        return out

    def debug_state(self) -> Dict[str, object]:
        """Protocol words of every shard / worker, read on a private stream (safe while kernels spin): for debugging a
        stalled run before a bounded device wait traps."""
        dev = self.devices[0]
        C = self.C
        out: Dict[str, object] = {"bounds": self.bounds, "multicast": self.multicast}
        st = torch.cuda.Stream(device=dev)
        with torch.cuda.device(dev), torch.cuda.stream(st):
            for r in range(self.n):
                flags = _view(self.seg_ptr(r, self.o_flags), self.n * C.MB_WORDS * 4, torch.int32, dev).to("cpu", non_blocking=False).view(self.n, C.MB_WORDS)
                out[f"shard{r}.posted"] = flags[:, 0].tolist()
                out[f"shard{r}.applied"] = flags[:, C.MB_APPLIED].tolist()
                out[f"shard{r}.sync"] = _view(self.seg_ptr(r, self.o_sync), 64, torch.int32, dev).cpu().tolist()
                out[f"shard{r}.ctrl"] = self.view("ctrl", r, dev)[:8].cpu().tolist()
                out[f"worker{r}.acks"] = self.view("ack", r, dev).cpu().view(-1, ACK_STRIDE)[: self.n, 0].tolist()
                stamps = self.view("stamps", r, dev).cpu().view(-1, VER_STRIDE)
                out[f"replica{r}.stamps(begin,end)"] = [(int(stamps[q, 0]), int(stamps[q, 16])) for q in range(self.n)]
            st.synchronize()
        out["appliers_alive"] = {s: a.alive() for s, a in self.appliers.items()}
        out["applier_launches"] = {s: a.launches() for s, a in self.appliers.items()}
        return out

    def view(self, which: str, shard: int, device: Optional[torch.device] = None) -> torch.Tensor:
        lay, dev = self.layout, device or self.dev_of(shard)
        if which == "state":
            return _view(self.seg_ptr(shard, self.o_state), lay.total * 16, torch.float32, dev).view(lay.total, 4)
        if which == "ctrl":
            return _view(self.seg_ptr(shard, self.o_ctrl), self.C.CTRL_WORDS * 4, torch.int32, dev)
        if which == "ack":
            return _view(self.seg_ptr(shard, self.o_ack), self.C.MAX_SHARDS * ACK_STRIDE * 4, torch.int32, dev)
        if which == "shadow":
            return _view(self.pub_ptr(shard, self.o_shadow), lay.shadow_total * 2, torch.bfloat16, dev)
        if which == "vec":
            return _view(self.pub_ptr(shard, self.o_vec), max(lay.vec_count, 4) * 4, torch.float32, dev)
        if which == "shadow1":
            return _view(self.pub_ptr(shard, self.o_shadow1), lay.shadow_total * 2, torch.bfloat16, dev)
        if which == "vec1":
            return _view(self.pub_ptr(shard, self.o_vec1), max(lay.vec_count, 4) * 4, torch.float32, dev)
        if which == "stamps":
            return _view(self.pub_ptr(shard, self.o_stamps), self.C.MAX_SHARDS * VER_STRIDE * 4, torch.int32, dev)
        raise KeyError(which)

    # ---- state ------------------------------------------------------------------------------------------------
    def load_weights(self, weights: Optional[Sequence[np.ndarray]]) -> None:
        """Initialise every shard's state and every replica.  SPMD: collective; rank 0 provides ``weights`` and the other
        ranks copy the initial state / publish buffer from rank 0's segment over NVLink."""
        lay = self.layout
        if self.spmd and self.ctx.rank != 0:
            D.barrier(self.ctx)                                      # rank 0 has written its segments
            dev = self.devices[0]
            with torch.cuda.device(dev):
                me = self.ctx.rank
                self.view("state", me, dev).copy_(self.view("state", 0, dev))
                for nm in ("shadow", "vec", "shadow1", "vec1"):
                    self.view(nm, me, dev).copy_(self.view(nm, 0, dev))
                _sync_current(dev)
            D.barrier(self.ctx)
            return
        flat = lay.flatten(weights)
        host = torch.zeros(lay.total, 4)
        host[:, 0] = torch.from_numpy(flat)
        for i in range(self.spec.num_slots):
            host[:, 1 + i] = self.spec.slot_init(i)
        pub = torch.from_numpy(lay.publish_reference(flat)).to(torch.bfloat16)
        vec = torch.zeros(max(lay.vec_count, 4))
        vec[:lay.vec_count] = torch.from_numpy(flat[lay.vec_offset:lay.vec_offset + lay.vec_count])
        for s in self.my_shards:
            dev = self.dev_of(s)
            with torch.cuda.device(dev):
                self.view("state", s).copy_(host)
                self.view("shadow", s).copy_(pub)
                self.view("vec", s).copy_(vec)
                self.view("shadow1", s).copy_(pub)
                self.view("vec1", s).copy_(vec)
                self.view("ctrl", s).zero_()
                self.view("stamps", s).zero_()
                _sync_current(dev)
        if self.spmd:
            D.barrier(self.ctx)
            D.barrier(self.ctx)

    def _owners(self) -> List[torch.Tensor]:
        """Per shard: flat element indices it owns (host int64 tensors)."""
        if self._owner_index is None:
            lay = self.layout
            owner = np.zeros(lay.total, dtype=np.int8)
            for t in range(self.n_tiles):
                si, tr, tc = (int(v) for v in self.tiles[t])
                s = lay.segments[si]
                r = int(np.searchsorted(self.bounds, t, side="right") - 1)
                r = min(r, self.n - 1)
                rows = np.arange(tr * 32, min(tr * 32 + 32, s.rows))
                cols = np.arange(tc * 64, min(tc * 64 + 64, s.cols))
                idx = (s.offset + rows[:, None] * s.cols + cols[None, :]).reshape(-1)
                owner[idx] = r
            self._owner_index = [torch.from_numpy(np.nonzero(owner == r)[0].astype(np.int64)) for r in range(self.n)]
        return self._owner_index

    def _gather_column(self, col: int) -> np.ndarray:
        """Assemble one column of the state (0 = params, 1.. = slots) from the shards that own each element."""
        lay = self.layout
        dev = self.devices[0]
        out = torch.zeros(lay.total, dtype=torch.float32)
        with torch.cuda.device(dev):
            for r, idx in enumerate(self._owners()):
                if idx.numel() == 0:
                    continue
                st = self.view("state", r, dev)
                out[idx] = st[:, col].index_select(0, idx.to(dev)).cpu()
        return out.numpy()

    def weights(self) -> List[np.ndarray]:
        _sync_current(self.devices[0])
        return self.layout.unflatten(self._gather_column(0))

    def slot_arrays(self) -> List[List[np.ndarray]]:
        return [self.layout.unflatten(self._gather_column(1 + i)) for i in range(self.spec.num_slots)]

    def load_slots(self, slots: Sequence[Sequence[np.ndarray]], step: int) -> None:
        for s in self.my_shards:
            dev = self.dev_of(s)
            with torch.cuda.device(dev):
                st, ctrl = self.view("state", s), self.view("ctrl", s)
                for i, per_var in enumerate(slots[: self.spec.num_slots]):
                    st[:, 1 + i].copy_(torch.from_numpy(self.layout.flatten(per_var)))
                ctrl[2] = int(step)
                ctrl[3] = int(step)
                _sync_current(dev)

    def counters(self) -> Dict[str, int]:
        dev = self.devices[0]
        with torch.cuda.device(dev):
            cs = [self.view("ctrl", r, dev).cpu().numpy() for r in range(self.n)]
        # every push visits every shard once: a push counts as applied when the slowest shard has applied it
        return {"lock": 0, "version": int(min(c[1] for c in cs)), "step": int(min(c[2] for c in cs)), "pushes": int(min(c[3] for c in cs)),
                "errors": int(sum(c[4] for c in cs)), "dropped": int(cs[0][5]), "shards": self.n, "multicast": int(self.multicast)}

    # ---- appliers ---------------------------------------------------------------------------------------------
    def start_applier(self, acquire_lock: bool, scope_sys: bool = True, grid: int = 0, poll_window_s: float = 0.0, depth: int = 3,
                      max_batch: int = 0, dbuf: bool = False) -> None:
        """One applier per owned shard.  ``acquire_lock`` selects seqlock-stamped publishes (pulls snapshot a shard
        atomically); Hogwild publishes without stamps.  No RW lock anywhere: a shard has exactly one writer."""
        lay, C = self.layout, self.C
        self.lock_mode = bool(acquire_lock)
        # a launch lingers between passes (warm code / TLB) and exits after this long without a post
        poll_window_s = poll_window_s or float(os.environ.get("SPARKFLOW_APPLIER_IDLE_US", "300")) * 1e-6
        for s in self.my_shards:
            if s in self.appliers:
                continue
            dev = self.dev_of(s)
            with torch.cuda.device(dev):
                segs_dev = torch.frombuffer(bytearray(C.pack_segs(lay.seg_rows())), dtype=torch.uint8).to(dev)
                tile_map = torch.from_numpy(self.tiles).to(dev)
                self._keep += [segs_dev, tile_map]
                _sync_current(dev)
                if self.multicast:
                    shadow_dst = [self.pub.mc_base + self.o_shadow]
                    vec_dst = [self.pub.mc_base + self.o_vec]
                    stamps = [self.pub.mc_base + self.o_stamps]
                else:
                    # no NVLS on this box: one peer store per replica (own replica first)
                    order = [s] + [r for r in range(self.n) if r != s]
                    shadow_dst = [self.pub_ptr(r, self.o_shadow) for r in order]
                    vec_dst = [self.pub_ptr(r, self.o_vec) for r in order]
                    stamps = [self.pub_ptr(r, self.o_stamps) for r in order]
                push = dict(state=self.seg_ptr(s, self.o_state), ctrl=self.seg_ptr(s, self.o_ctrl), shadow_dst=shadow_dst,
                            shadow_is_mc=1 if self.multicast else 0, vec_dst=vec_dst if lay.vec_count else [], vec_offset=lay.vec_offset,
                            grad=0, applier=1, segs=native.ptr(segs_dev), tile_map=native.ptr(tile_map), num_tiles=self.n_tiles,
                            seg_rows=lay.seg_rows(), optimizer=self.spec.opt_id, lock_mode=0, drop=0, scope_sys=1 if scope_sys else 0,
                            grad_scale=1.0, hyper=self.spec.native_hyper(), mb_zero=1 if self.mb_zero else 0)
                if s not in self._stats:
                    self._stats[s] = torch.zeros(16, dtype=torch.int64, device=dev)
                shard = dict(tile_begin=self.bounds[s], tile_end=self.bounds[s + 1], ack=[self.ack_ptr(w, s) for w in range(self.n)],
                             stats=native.ptr(self._stats[s]), linger=int(os.environ.get("SPARKFLOW_APPLIER_LINGER", "1")))
                if self.lock_mode:
                    shard.update(ver_begin=[p + s * VER_STRIDE * 4 for p in stamps], ver_end=[p + (s * VER_STRIDE + 16) * 4 for p in stamps],
                                 ver_mc=1 if self.multicast else 0, ver_local=self.pub_ptr(s, self.o_stamps) + s * VER_STRIDE * 4,
                                 slot_off_bf16=self.slot_off_bf16, slot_off_f32=self.slot_off_f32)
                if grid and grid != self.applier_grid(s):
                    raise ValueError("the applier grid of a sharded master is fixed by applier_grid(): workers count its acknowledgements")
                g = self.applier_grid(s)
                self.appliers[s] = C.Applier(push, self.seg_ptr(s, self.o_mail), self.mb_stride, self.seg_ptr(s, self.o_flags), self.n,
                                             self.seg_ptr(s, self.o_sync), poll_window_s, g, depth,
                                             max_batch or int(os.environ.get("SPARKFLOW_APPLIER_BATCH", "8")), 0, 0, shard)

    def applier_grid(self, shard: int) -> int:
        """CTAs of shard ``shard``'s applier (the same number on every rank: workers wait for posts x grid acknowledgements)."""
        n_own = max(1, self.bounds[shard + 1] - self.bounds[shard])
        # An applier CTA (512 threads x ~96 registers) owns its SM while the launch lingers, and every CTA of the grid
        # must be resident at once: small shards get one CTA per tile (lowest pass latency), larger ones are capped so
        # the training kernels of the same GPU keep most of the SMs (big models: up to half of them).
        cap = 40 if n_own <= 160 else 74
        return int(os.environ.get("SPARKFLOW_APPLIER_CTAS", "0")) or min(cap, n_own)

    def applier_latency(self) -> Dict[str, float]:
        """Device-measured averages of the owned shards' appliers: decision -> all tiles applied + published (`apply_us`),
        decision -> every consumed push acknowledged (`ack_us`), pushes per pass."""
        out = {"apply_us": 0.0, "ack_us": 0.0, "passes": 0, "pushes_per_pass": 0.0}
        for s, t in self._stats.items():
            v = t.cpu().numpy()
            if v[2]:
                out["apply_us"] = max(out["apply_us"], v[0] / v[2] / 1e3)
                out["ack_us"] = max(out["ack_us"], v[1] / v[2] / 1e3)
                out["passes"] = max(out["passes"], int(v[2]))
                out["cta_saw_decision_us"] = v[4] / v[2] / 1e3
                out["cta_tiles_us"] = v[5] / v[2] / 1e3
                out["cta_flush_us"] = v[6] / v[2] / 1e3
                for i, nm in enumerate(["t_list", "t_issue", "t_loads_math", "t_stores", "t_transpose", "t_timer_read"]):
                    out["cta_" + nm + "_us"] = v[8 + i] / v[2] / 1e3
                out["pushes_per_pass"] = max(out["pushes_per_pass"], float(v[3]) / float(v[2]))
        return out

    @property
    def applier(self):
        """Truthy while this process's appliers run (``alive()`` like the single-master Applier)."""
        return _ApplierGroup(self.appliers) if self.appliers else None

    def stop_applier(self) -> None:
        for a in self.appliers.values():
            a.stop()
        self.appliers = {}

    @property
    def owner(self) -> bool:
        return True                      # every process owns (at least) one shard

    def close(self) -> None:
        self.stop_applier()
        self._keep = []
        self.pub.close()
        self.seg.close()


class _ApplierGroup:
    def __init__(self, appliers):
        self._a = appliers

    def alive(self) -> bool:
        return all(a.alive() for a in self._a.values())
