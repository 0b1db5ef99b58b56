"""H100 engine: master parameter state + per-GPU worker that executes compiled step plans.

Mapping of the reference's runtime (SURVEY.md sections 1, 3.1, 5.1) onto one H100 box:

* parameter-server process (Flask, HogwildSparkModel.py:175-244)  ->  :class:`MasterState`, one
  cudaMalloc'ed segment on the driver GPU holding the flat fp32 params, the optimizer slots, the bf16
  publish buffer and a 256-byte control block (RW lock word, version, step counters).  The segment
  is exported with CUDA IPC so every worker process addresses it over NVLink.
* Spark partition worker (``handle_model``, HogwildSparkModel.py:38-100)  ->  :class:`DeviceWorker`:
  one process per GPU.  A training step is a *compiled plan* – pull, input cast, wgmma GEMMs with
  fused epilogues, loss kernel, wgrad/dgrad GEMMs, fused push – captured once into a CUDA graph and
  replayed, so a step costs one graph launch on the host.
* ``GET /parameters`` -> ``pull`` kernel (or TMA reads of the master's publish buffer straight from
  the GEMMs in ``direct`` mode);  ``POST /update`` -> ``push`` kernel (optimizer applied on the master
  shard over NVLink, lock-free or under the device RW lock).
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ..graph.ir import GraphIR
from ..models.compiler import ACT_IDS, LayerPlan, compile_graph
from ..ops import native
from ..ops.layout import ParamLayout, round_up
from ..ops.optimizers import OptimizerSpec

_ALIGN = 256


class _RawCuda:
    """Expose a raw device allocation to torch through ``__cuda_array_interface__``."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


def _view(ptr: int, nbytes: int, dtype: torch.dtype, device: torch.device) -> torch.Tensor:
    return torch.as_tensor(_RawCuda(ptr, nbytes), device=device).view(dtype)


@dataclass
class MasterLayout:
    """Byte offsets of the fields inside the master segment."""
    ctrl: int
    state: int
    shadow: int
    nbytes: int
    mailboxes: int = 0
    mailbox_stride: int = 0        # floats
    flags: int = 0
    applier_sync: int = 0
    n_mailboxes: int = 0
    shadow_alt: int = 0            # second publish buffer + fp32 copies of the 1-D tail (double-buffered publish)
    vec_pub0: int = 0
    vec_pub1: int = 0

    @classmethod
    def build(cls, layout: ParamLayout, ctrl_words: int, n_mailboxes: int = 0, mb_words: int = 32) -> "MasterLayout":
        off = 0

        def take(n):
            nonlocal off
            start = off
            off = round_up(off + n, _ALIGN)
            return start

        ctrl = take(ctrl_words * 4)
        state = take(layout.total * 16)           # float4 (p, slot0, slot1, slot2) per element
        shadow = take(layout.shadow_total * 2)
        if n_mailboxes <= 0:
            return cls(ctrl, state, shadow, off)
        stride = round_up(layout.total, 64)
        flags = take(n_mailboxes * mb_words * 4)
        sync = take(64)
        boxes = take(n_mailboxes * stride * 4)
        shadow_alt = take(layout.shadow_total * 2)
        vp0 = take(max(layout.vec_count, 4) * 4)
        vp1 = take(max(layout.vec_count, 4) * 4)
        return cls(ctrl, state, shadow, off, boxes, stride, flags, sync, n_mailboxes, shadow_alt, vp0, vp1)


def _sync_current(device: torch.device) -> None:
    """Stream-level synchronisation.  NEVER a device-wide cudaDeviceSynchronize: in served push mode a persistent
    applier kernel lives on the master GPU and a device-wide sync would wait for it."""
    torch.cuda.current_stream(device).synchronize()


class MasterState:
    """The parameter server's state on the driver GPU (or a mapping of it in a worker process)."""

    def __init__(self, layout: ParamLayout, spec: OptimizerSpec, device: torch.device, base_ptr: Optional[int] = None,
                 n_mailboxes: int = 0):
        self.C = native.cuda_ext()
        self.layout, self.spec, self.device = layout, spec, device
        self.ml = MasterLayout.build(layout, self.C.CTRL_WORDS, n_mailboxes, self.C.MB_WORDS)
        self.applier = None
        self.owner = base_ptr is None
        with torch.cuda.device(device):
            self.base = self.C.ipc_alloc(self.ml.nbytes) if self.owner else int(base_ptr)
        nb = self.ml.nbytes
        self._bytes = _view(self.base, nb, torch.uint8, device)
        self.ctrl = self._bytes[self.ml.ctrl:self.ml.ctrl + self.C.CTRL_WORDS * 4].view(torch.int32)
        # element-interleaved state: one 16-byte (p, s0, s1, s2) tuple per parameter, so a push reads / writes a
        # parameter's tuple with single 16-byte accesses (no torn (m, v) pairs under Hogwild)
        self.state = self._bytes[self.ml.state:self.ml.state + layout.total * 16].view(torch.float32).view(layout.total, 4)
        self.p = self.state[:, 0]
        self.slots = [self.state[:, 1 + i] for i in range(3)]
        self.shadow = self._bytes[self.ml.shadow:self.ml.shadow + layout.shadow_total * 2].view(torch.bfloat16)
        # double-buffered publish (served push + lock mode + replica pulls): see SfPullArgs.dbuf in csrc/sf_api.h
        self.dbuf_capable = n_mailboxes > 0 and os.environ.get("SPARKFLOW_PUBLISH", "double") != "single"
        self.dbuf_active = False
        if n_mailboxes > 0:
            self.shadow_alt = self._bytes[self.ml.shadow_alt:self.ml.shadow_alt + layout.shadow_total * 2].view(torch.bfloat16)
            nv = max(layout.vec_count, 4)
            self.vec_pub = [self._bytes[o:o + nv * 4].view(torch.float32) for o in (self.ml.vec_pub0, self.ml.vec_pub1)]

    # -- owner-side API ---------------------------------------------------------------------------
    def ipc_handle(self) -> bytes:
        with torch.cuda.device(self.device):
            return bytes(self.C.ipc_get_handle(self.base))

    @classmethod
    def from_ipc(cls, layout: ParamLayout, spec: OptimizerSpec, device: torch.device, handle: bytes, n_mailboxes: int = 0) -> "MasterState":
        C = native.cuda_ext()
        with torch.cuda.device(device):
            base = C.ipc_open_handle(handle)
        return cls(layout, spec, device, base_ptr=base, n_mailboxes=n_mailboxes)

    # -- served push (mailboxes + master-resident applier) ------------------------------------------
    @property
    def served(self) -> bool:
        return self.ml.n_mailboxes > 0

    def mailbox_ptr(self, worker: int) -> int:
        return self.base + self.ml.mailboxes + worker * self.ml.mailbox_stride * 4

    def flags_ptr(self, worker: int) -> int:
        return self.base + self.ml.flags + worker * self.C.MB_WORDS * 4

    def start_applier(self, acquire_lock: bool, scope_sys: bool, grid: int = 0, poll_window_s: float = 30e-6, depth: int = 3,
                      max_batch: int = 0, dbuf: bool = False) -> None:
        """Start the applier (owner process only): a host thread that keeps `depth` finite poll-and-apply
        kernels queued on a dedicated high-priority stream of the master GPU.  `max_batch` pushes (default 8,
        env SPARKFLOW_APPLIER_BATCH) are applied per pass over the state - each still its own optimizer step."""
        assert self.owner and self.served
        lay = self.layout
        with torch.cuda.device(self.device):
            self._segs_dev = torch.frombuffer(bytearray(self.C.pack_segs(lay.seg_rows())), dtype=torch.uint8).to(self.device)
            self._tile_map = torch.from_numpy(lay.tile_map()).to(self.device)
            _sync_current(self.device)
            self.dbuf_active = bool(dbuf and acquire_lock and self.dbuf_capable)
            self.ctrl[self.C.CTRL_PUB + 1] = 1 if self.dbuf_active else 0        # workers read the publish protocol from here
            extra = {}
            if self.dbuf_active:
                self._sync_publish_buffers()
                extra = dict(vec_pub=[native.ptr(self.vec_pub[0])], vec_offset=lay.vec_offset)
            push = dict(state=native.ptr(self.state), ctrl=native.ptr(self.ctrl), shadow_dst=[native.ptr(self.shadow)], grad=0, applier=1, **extra,
                        segs=native.ptr(self._segs_dev), tile_map=native.ptr(self._tile_map), num_tiles=int(self._tile_map.shape[0]),
                        seg_rows=lay.seg_rows(), optimizer=self.spec.opt_id, lock_mode=1 if acquire_lock else 0, drop=0,
                        scope_sys=1 if scope_sys else 0, grad_scale=1.0, hyper=self.spec.native_hyper())
            # every CTA (512 threads, one per SM) must be resident at once, beside the training kernels of this GPU
            grid = grid or int(os.environ.get("SPARKFLOW_APPLIER_CTAS", "64"))
            self.applier = self.C.Applier(push, self.base + self.ml.mailboxes, self.ml.mailbox_stride, self.base + self.ml.flags,
                                          self.ml.n_mailboxes, self.base + self.ml.applier_sync, poll_window_s, grid, depth,
                                          max_batch or int(os.environ.get("SPARKFLOW_APPLIER_BATCH", "8")),
                                          native.ptr(self.shadow_alt) if self.dbuf_active else 0,
                                          native.ptr(self.vec_pub[1]) if self.dbuf_active else 0)

    def stop_applier(self) -> None:
        if self.applier is not None:
            self.applier.stop()
            self.applier = None
            if self.dbuf_active:
                self._settle_publish()

    def _sync_publish_buffers(self) -> None:
        """Both publish buffers (and the fp32 copies of the 1-D tail) = the current parameters; buffer 0 current."""
        lay = self.layout
        with torch.cuda.device(self.device):
            self.shadow_alt.copy_(self.shadow)
            if lay.vec_count:
                v = self.state[lay.vec_offset:lay.vec_offset + lay.vec_count, 0]
                self.vec_pub[0][:lay.vec_count].copy_(v)
                self.vec_pub[1][:lay.vec_count].copy_(v)
            self.ctrl[self.C.CTRL_PUB] = 0
            _sync_current(self.device)

    def _settle_publish(self) -> None:
        """The applier is stopped: make buffer 0 the current, complete one (readers that do not follow the double-buffer
        protocol - TMA-direct inference plans, worker-applied pushes - only know buffer 0)."""
        with torch.cuda.device(self.device):
            pub = int(self.ctrl[self.C.CTRL_PUB].item()) & 0xFFFFFFFF
            if pub >> 31:
                self.shadow.copy_(self.shadow_alt)
                self.vec_pub[0].copy_(self.vec_pub[1])
            self.ctrl[self.C.CTRL_PUB] = 0
            _sync_current(self.device)

    def load_weights(self, weights: Sequence[np.ndarray]) -> None:
        """Initialise params, slots, control block and the bf16 publish buffer (owner only)."""
        flat = self.layout.flatten(weights)
        host = torch.zeros(self.layout.total, 4)
        host[:, 0] = torch.from_numpy(flat)
        for i in range(self.spec.num_slots):
            host[:, 1 + i] = self.spec.slot_init(i)
        self.state.copy_(host)
        version = self.ctrl[1:2].clone()
        self.ctrl.zero_()
        self.ctrl[1:2] = version
        self._advance_version()
        pub = torch.from_numpy(self.layout.publish_reference(flat)).to(torch.bfloat16)
        self.shadow.copy_(pub)
        if self.ml.n_mailboxes > 0:
            self._sync_publish_buffers()
        _sync_current(self.device)

    def weights(self) -> List[np.ndarray]:
        _sync_current(self.device)
        return self.layout.unflatten(self.p.detach().contiguous().cpu().numpy())

    def slot_arrays(self) -> List[List[np.ndarray]]:
        return [self.layout.unflatten(s.detach().contiguous().cpu().numpy()) for s in self.slots[: self.spec.num_slots]]

    def load_slots(self, slots: Sequence[Sequence[np.ndarray]], step: int) -> None:
        """Restore optimizer slots + the global step (resume from a snapshot)."""
        for i, per_var in enumerate(slots[: self.spec.num_slots]):
            self.state[:, 1 + i].copy_(torch.from_numpy(self.layout.flatten(per_var)))
        self.ctrl[2] = int(step)
        self.ctrl[3] = int(step)
        self._advance_version()
        _sync_current(self.device)

    def _advance_version(self) -> None:
        """A host write of the master state moves SF_CTRL_VERSION on, and never back: a worker whose replica_version
        equals it trusts what it read at its own last push (the locked push's early tuple loads, the locked pull's
        skipped copy).  While it is 0 no push has been applied, so no worker holds a matching version and it stays 0."""
        v = self.ctrl[1:2]
        v.add_((v != 0).to(v.dtype))

    def counters(self) -> Dict[str, int]:
        c = self.ctrl.cpu().numpy()
        return {"lock": int(c[0]), "version": int(c[1]), "step": int(c[2]), "pushes": int(c[3]), "errors": int(c[4]),
                "dropped": int(c[5])}

    def close(self) -> None:
        self.stop_applier()
        if self.base:
            with torch.cuda.device(self.device):
                (self.C.ipc_free if self.owner else self.C.ipc_close_handle)(self.base)
            self.base = 0


@dataclass
class StepBuffers:
    x_stage: torch.Tensor          # fp32 [B, D]   H2D target
    y_stage: Optional[torch.Tensor]
    loss_out: torch.Tensor
    result: Optional[torch.Tensor] = None
    idx: Optional[torch.Tensor] = None     # resident mode: device int32 [B] row ids gathered by the prep plan
    prep: Any = None                       # staged plans: the plan that prepares the step's operands (run before the step)


class DeviceWorker:
    """One GPU's replica + compiled step plans."""

    def __init__(self, ir: GraphIR, tf_input: str, tf_label: Optional[str], spec: OptimizerSpec, master: MasterState,
                 acquire_lock: bool = False, pull_mode: Optional[str] = None, use_graphs: bool = True,
                 device: Optional[torch.device] = None, plan: Optional[LayerPlan] = None, shared: bool = True,
                 worker_index: int = 0, reads_between_pulls: bool = False):
        """``reads_between_pulls``: steps without a pull (several minibatches per pull) or a partition loss read this
        worker's replica, and must see the weights of its last pull."""
        self.C = native.cuda_ext()
        self.ir = ir
        self.plan: LayerPlan = plan if plan is not None else compile_graph(ir, tf_input, tf_label, None, need_loss=True)
        from .plan_builder import check_grammar

        check_grammar(self.plan)
        self.spec, self.master = spec, master
        self.layout = master.layout
        self.device = device or master.device
        self.lock_mode = 1 if acquire_lock else 0
        self.scope_sys = 1 if shared else 0        # more than one GPU touches the master -> system-scope lock
        self.worker_index = worker_index
        self.sharded = bool(getattr(master, "sharded", False))      # master state sharded over all GPUs (parallel/sharded.py)
        self.served = bool(master.served)          # push = post to my mailbox, the master-resident applier applies it
        self.pull_mode = pull_mode or os.environ.get("SPARKFLOW_PULL_MODE", "copy")
        # lock mode without a lock on the read side: pulls pick the complete one of two publish buffers (see start_applier)
        self.use_dbuf = False
        if self.served:
            applier_dbuf = int(master.ctrl[self.C.CTRL_PUB + 1].item()) == 1      # written by start_applier (before any worker exists)
            if applier_dbuf and (self.pull_mode != "copy" or not acquire_lock):
                raise RuntimeError("the applier publishes double-buffered (lock mode, replica pulls) but this worker was created with "
                                   f"pull_mode={self.pull_mode!r}, acquire_lock={acquire_lock}")
            self.use_dbuf = applier_dbuf
        if self.sharded:
            self.pull_mode = "copy" if self.lock_mode else "inbox"     # lock: seqlock snapshot; Hogwild: GEMMs read the inbox in place
        if self.pull_mode == "direct" and self.lock_mode:
            self.pull_mode = "copy"            # a locked pull must be a private snapshot
        # locked worker-applied push: it also publishes into this worker's replica, and the next pull skips its copy when
        # no other push came in between.  Not when something reads the replica without pulling first: those reads must
        # see the weights of the last pull, not of the last push.
        self.own_publish = bool(self.lock_mode and not self.served and not self.sharded and self.pull_mode == "copy"
                                and not reads_between_pulls)
        self.use_graphs = use_graphs and os.environ.get("SPARKFLOW_NO_GRAPHS") != "1"
        self.use_branches = os.environ.get("SPARKFLOW_NO_BRANCHES") != "1"
        self.fuse_loss = os.environ.get("SPARKFLOW_NO_FUSED_LOSS") != "1"
        self.C.set_pdl(0 if os.environ.get("SPARKFLOW_NO_PDL") == "1" else 1)
        self.stream = torch.cuda.Stream(device=self.device)
        self.copy_stream = torch.cuda.Stream(device=self.device)
        dev = self.device
        lay = self.layout
        # local replica of what a pull fetches
        if self.sharded:
            m = master
            inbox_shadow, inbox_vec = m.view("shadow", worker_index, dev), m.view("vec", worker_index, dev)
            if self.lock_mode:
                self.replica, self.vec_local = inbox_shadow.clone(), inbox_vec.clone()      # working copy (pads / initial weights included)
            else:
                self.replica, self.vec_local = inbox_shadow, inbox_vec                       # zero-copy pull
            self.inbox_shadow, self.inbox_vec = inbox_shadow, inbox_vec
            # the worker's words inside its own symmetric segment: my_posted lives right behind the acknowledgement words
            self.ack_words = m.view("ack", worker_index, dev)
            self.my_posted = torch.zeros(4, dtype=torch.int32, device=dev)
            self.shard_stats = torch.zeros(64, dtype=torch.int64, device=dev)      # device-side latency accounting (SfSyncPullArgs.stats)
            ryw = self.C.pack_ryw(m.n, [m.applier_grid(r) for r in range(m.n)], native.ptr(self.ack_words), native.ptr(self.my_posted),
                                  native.ptr(self.shard_stats))
            self.ryw_dev = torch.frombuffer(bytearray(ryw), dtype=torch.uint8).to(dev)
            # Hogwild: the read-your-writes wait is fused into the step's first GEMM (no pull kernel at all)
            self.fuse_ryw = (not self.lock_mode) and os.environ.get("SPARKFLOW_NO_FUSED_PULL") != "1"
            route = self.C.pack_route(m.n, m.bounds, [m.mailbox_ptr(r, worker_index) for r in range(m.n)])
            self.route_dev = torch.frombuffer(bytearray(route), dtype=torch.uint8).to(dev)
            vt = []
            for i, sgm in enumerate(lay.segments):
                if sgm.rows == 1:
                    for tc in range((sgm.cols + 63) // 64):
                        vt.append((m.tile_prefix[i] + tc, sgm.offset + tc * 64, min(64, sgm.cols - tc * 64)))
            # the fused first-conv weight gradient is accumulated locally too (direct CUDA-core kernel): forward its rows
            from .plan_builder import fused_first_conv

            fc = fused_first_conv(self.plan)
            if fc is not None:
                sgm = lay.by_name(self.plan.layers[fc].kernel)
                tiles_c = (sgm.cols + 63) // 64
                for r_ in range(sgm.rows):
                    for tc in range(tiles_c):
                        vt.append((m.tile_prefix[sgm.index] + (r_ // 32) * tiles_c + tc, sgm.offset + r_ * sgm.cols + tc * 64,
                                   min(64, sgm.cols - tc * 64)))
            self.vec_tiles = torch.tensor(vt if vt else [(0, 0, 0)], dtype=torch.int64, device=dev)
            self.n_vec_tiles = len(vt)
            # snapshot pull: the copy is latency bound, so give every shard as many CTAs as it has tiles (all CTAs of the
            # kernel must be co-resident for the per-shard version agreement: at most one CTA per SM in total)
            tiles_per_shard = max(1, -(-m.n_tiles // m.n))
            self.sync_cps = max(1, min(tiles_per_shard, native.num_sms() // m.n, int(os.environ.get("SPARKFLOW_PULL_CTAS_PER_SHARD", "16"))))
            init = torch.zeros(8, 8, dtype=torch.int64)
            init[:, 1] = 0xFFFFFFFF
            self.sync_sp = torch.from_numpy(init.numpy().astype("uint32").view("int32").copy()).to(dev)
        else:
            self.replica = torch.zeros(lay.shadow_total, dtype=torch.bfloat16, device=dev)
            self.vec_local = torch.zeros(max(lay.vec_count, 4), dtype=torch.float32, device=dev)
        self.grads = torch.zeros(lay.total, dtype=torch.float32, device=dev)
        self.loss_acc = torch.zeros(1, dtype=torch.float32, device=dev)
        self.sync_push = torch.zeros(8, dtype=torch.int32, device=dev)
        self.sync_pull = torch.zeros(8, dtype=torch.int32, device=dev)
        self.seen_version = torch.zeros(1, dtype=torch.int32, device=dev)
        # version of the master's publish the replica holds (own_publish); -1: none yet, the first pull copies
        self.replica_version = torch.full((1,), -1, dtype=torch.int32, device=dev)
        self.segs_dev = torch.frombuffer(bytearray(self.C.pack_segs(lay.seg_rows())), dtype=torch.uint8).to(dev)
        self.tile_map = torch.from_numpy(lay.tile_map()).to(dev)
        self._plans: Dict[Tuple[int, int], object] = {}
        self._ordered: set = set()
        self._input_sets: Dict[Tuple[int, int], Dict[str, Any]] = {}
        self._bufs: Dict[Tuple[int, int], StepBuffers] = {}
        self._keep: List[object] = []
        self.drop_next = 0
        self.launches_per_step = 0
        self._order_after_build()          # the tables uploaded above (torch current stream) precede any plan kernel

    @classmethod
    def for_inference(cls, ir: GraphIR, plan: LayerPlan, spec: OptimizerSpec, master: MasterState) -> "DeviceWorker":
        """Forward-only worker reading weights straight from ``master`` (no replica, no optimizer)."""
        return cls(ir, plan.input_name, None, spec, master, acquire_lock=False, pull_mode="direct", use_graphs=False, plan=plan,
                   shared=False)

    # ------------------------------------------------------------------------------------------
    def _weight_src(self) -> torch.Tensor:
        """Where the forward/backward GEMMs read bf16 weights from."""
        return self.master.shadow if self.pull_mode == "direct" else self.replica

    def _bias_ptr(self, seg) -> int:
        # biases are always read from the local fp32 copy (the master keeps them interleaved with their slots)
        return native.ptr(self.vec_local) + (seg.offset - self.layout.vec_offset) * 4

    def _push_args(self, loss_out: torch.Tensor, drop: int = 0) -> dict:
        m = self.master
        args = dict(state=native.ptr(m.state), ctrl=native.ptr(m.ctrl), shadow_dst=[native.ptr(m.shadow)], grad=native.ptr(self.grads),
                    loss_acc=native.ptr(self.loss_acc), loss_out=native.ptr(loss_out), segs=native.ptr(self.segs_dev),
                    tile_map=native.ptr(self.tile_map), num_tiles=int(self.tile_map.shape[0]), seg_rows=self.layout.seg_rows(),
                    optimizer=self.spec.opt_id, lock_mode=self.lock_mode, drop=drop, scope_sys=self.scope_sys, grad_scale=1.0, hyper=self.spec.native_hyper())
        if self.own_publish:
            # the replica has the publish buffer's flat layout, vec_local the 1-D tail's (indexed from vec_offset)
            args.update(shadow_dst=[native.ptr(m.shadow), native.ptr(self.replica)], replica_version=native.ptr(self.replica_version))
            if self.layout.vec_count:
                args.update(vec_pub=[native.ptr(self.vec_local)], vec_offset=self.layout.vec_offset)
        return args

    def _post_args(self, loss_out: torch.Tensor, drop: int = 0) -> dict:
        m = self.master
        return dict(grad=native.ptr(self.grads), mailbox=m.mailbox_ptr(self.worker_index), flags=m.flags_ptr(self.worker_index),
                    loss_acc=native.ptr(self.loss_acc), loss_out=native.ptr(loss_out), n=self.layout.total, drop=drop)

    # ---- sharded master ------------------------------------------------------------------------------------
    def _sync_pull_args(self, copy: bool) -> dict:
        m, lay = self.master, self.layout
        from .sharded import VER_STRIDE

        stamps = m.pub_ptr(self.worker_index, m.o_stamps)
        d = dict(n_shards=m.n, bounds=m.bounds, applied=native.ptr(self.ack_words), my_posted=native.ptr(self.my_posted),
                 copy=1 if (copy and self.lock_mode) else 0, stats=native.ptr(self.shard_stats),
                 ack_grid=[m.applier_grid(r) for r in range(m.n)])
        if d["copy"]:
            d.update(ver_begin=stamps, ver_end=stamps + 16 * 4, ver_stride=VER_STRIDE, slot_off_bf16=m.slot_off_bf16, slot_off_f32=m.slot_off_f32,
                     src=native.ptr(self.inbox_shadow), dst=native.ptr(self.replica),
                     src_vec=native.ptr(self.inbox_vec) if lay.vec_count else 0, dst_vec=native.ptr(self.vec_local) if lay.vec_count else 0,
                     vec_offset=lay.vec_offset, segs=native.ptr(self.segs_dev), tile_map=native.ptr(self.tile_map),
                     ctas_per_shard=self.sync_cps, sync=native.ptr(self.sync_sp))
        return d

    def _post_flags_args(self, loss_out: torch.Tensor, drop: int = 0, phase: int = 0) -> dict:
        m = self.master
        return dict(phase=phase, n_shards=m.n, bounds=m.bounds, posted=[m.posted_ptr(r, self.worker_index) for r in range(m.n)],
                    mailbox=[m.mailbox_ptr(r, self.worker_index) for r in range(m.n)], grad=native.ptr(self.grads),
                    vec_tiles=native.ptr(self.vec_tiles), n_vec_tiles=self.n_vec_tiles, loss_acc=native.ptr(self.loss_acc),
                    loss_out=native.ptr(loss_out), my_posted=native.ptr(self.my_posted), drop=drop, total=self.layout.total,
                    mb_zero=1 if m.mb_zero else 0, heartbeat=m.heartbeat_ptr(self.worker_index), stats=native.ptr(self.shard_stats))

    def exposed_latency(self, reset: bool = False) -> Dict[str, float]:
        """Sharded master: device-measured (%globaltimer) per-step latencies of this worker, averaged since the last reset
        and taken over the slowest shard: how long after its post the next step started waiting (`covered_us`: work that
        hid the push), how long it then stalled for the acknowledgement (`exposed_push_us`: the exposed part of
        push -> apply -> publish), and the snapshot copy of the pull (`exposed_pull_us`, lock mode only)."""
        if not self.sharded:
            return {}
        self.stream.synchronize()
        st = self.shard_stats.cpu().numpy()
        out = {"covered_us": 0.0, "exposed_push_us": 0.0, "exposed_pull_us": 0.0, "steps": 0}
        for sh in range(self.master.n):
            n = int(st[11 + 4 * sh])
            if n:
                out["steps"] = max(out["steps"], n)
                out["covered_us"] = max(out["covered_us"], st[8 + 4 * sh] / n / 1e3)
                out["exposed_push_us"] = max(out["exposed_push_us"], st[9 + 4 * sh] / n / 1e3)
                out["exposed_pull_us"] = max(out["exposed_pull_us"], st[10 + 4 * sh] / n / 1e3)
        if reset:
            with torch.cuda.stream(self.stream):
                self.shard_stats[8:].zero_()
            self.stream.synchronize()
        return out

    def route_args(self, seg) -> dict:
        """Epilogue fields that send a wgrad's fp32 tiles to the owning shards' mailboxes (GEMM dict entries)."""
        m = self.master
        return dict(route=native.ptr(self.route_dev), route_tile0=m.tile_prefix[seg.index], route_tiles_c=(seg.cols + 63) // 64,
                    route_off=seg.offset, ld_f32=seg.cols)

    def _pull_args(self) -> dict:
        lay, m = self.layout, self.master
        direct = self.pull_mode == "direct"       # weights are read in place by TMA; only the 1-D tail is copied
        return dict(src=native.ptr(m.shadow), dst=native.ptr(self.replica), n_bf16=0 if direct else lay.shadow_total,
                    src_state=native.ptr(m.state) + lay.vec_offset * 16 if lay.vec_count else 0,
                    dst_f32=native.ptr(self.vec_local) if lay.vec_count else 0, n_f32=lay.vec_count,
                    ctrl=native.ptr(m.ctrl), seen_version=native.ptr(self.seen_version), lock_mode=self.lock_mode,
                    scope_sys=self.scope_sys,
                    wait_applied=(m.flags_ptr(self.worker_index) + self.C.MB_APPLIED * 4) if self.served else 0,
                    my_posted=(native.ptr(self.sync_push) + 16) if self.served else 0,
                    replica_version=native.ptr(self.replica_version) if self.own_publish else 0,
                    **(dict(dbuf=1, src_alt=native.ptr(m.shadow_alt), vec_pub0=native.ptr(m.vec_pub[0]), vec_pub1=native.ptr(m.vec_pub[1]))
                       if self.use_dbuf else {}))

    # ------------------------------------------------------------------------------------------
    def input_set(self, B: int, slot: int) -> Dict[str, Any]:
        from .plan_builder import use_mn_possible

        key = (B, slot)
        if key not in self._input_sets:
            lp, D = self.plan, self.plan.input_dim
            ldB = round_up(B, 8)
            first = next(l for l in lp.layers if l.kind in ("dense", "conv"))
            dev = self.device
            need_t = first.kind == "dense" and not use_mn_possible(True)     # K-major first wgrad
            self._input_sets[key] = dict(
                x32=torch.zeros(B, D, dtype=torch.float32, device=dev),
                a0=torch.zeros(B, round_up(D, 8), dtype=torch.bfloat16, device=dev),
                a0T=torch.zeros(D, ldB, dtype=torch.bfloat16, device=dev) if need_t else None,
                y=None if lp.target_is_input or not lp.label_dim else torch.zeros(B, lp.label_dim, dtype=torch.float32, device=dev))
        return self._input_sets[key]

    def _order_after_build(self) -> None:
        """Plan building allocates (zero-fills) and uploads through torch's CURRENT stream; the worker's streams are
        non-blocking ones, so nothing orders those fills before the plan's first kernels unless we say so."""
        cur = torch.cuda.current_stream(self.device)
        self.stream.wait_stream(cur)
        self.copy_stream.wait_stream(cur)

    def build_plan(self, B: int, slot: int = 0, with_pull: bool = True, with_push: bool = True,
                   resident: Optional[Tuple[torch.Tensor, Optional[torch.Tensor]]] = None, staged: bool = False):
        """Compile the training step for batch size ``B`` reading from staging-buffer set ``slot``.

        ``staged`` (implied by ``resident``): the step consumes input set ``slot`` and ``bufs.prep`` is the plan that
        prepares it - cast of the rows copied into ``bufs.x_stage``, or, with ``resident`` = (X, Y) device tensors, the
        gather of the rows whose ids are in ``bufs.idx``.  Running it before the step (on the stream that stages the
        minibatch) takes the cast / gather off the step graph, which then starts with the pull.  Otherwise the step
        casts ``bufs.x_stage`` itself."""
        from . import plan_builder

        staged = staged or resident is not None
        key = (B, slot, with_pull, with_push, staged, None if resident is None else resident[0].data_ptr())
        if key not in self._plans and staged:
            ins = self.input_set(B, slot)
            built = plan_builder.build(self, B, train=True, with_pull=with_pull, with_push=with_push, inputs=ins)
            prep, idx = plan_builder.build_prep(self, B, ins, None if resident is None else dict(x=resident[0], y=resident[1]))
            self.last_debug = built.debug
            self._plans[key] = built.plan
            self._bufs[key] = StepBuffers(built.x_stage, built.y_stage, built.loss_out, built.result, idx, prep)
            self._keep.append(built.keep)
            self.launches_per_step = len(built.plan)
            self._last_names = list(built.plan.names())
        if key not in self._plans:
            built = plan_builder.build(self, B, train=True, with_pull=with_pull, with_push=with_push)
            self.last_debug = built.debug           # per-layer intermediate buffers of the newest plan (tests / tools)
            self._plans[key] = built.plan
            self._bufs[key] = StepBuffers(built.x_stage, built.y_stage, built.loss_out, built.result)
            self._keep.append(built.keep)
            self.launches_per_step = len(built.plan)
            self._last_names = list(built.plan.names())
        if key not in self._ordered:
            self._ordered.add(key)
            self._order_after_build()
        return self._plans[key], self._bufs[key]

    def build_forward_plan(self, B: int, upto: Optional[int] = None, post: Optional[str] = None, with_loss: bool = False,
                           with_pull: bool = False):
        """Forward-only plan: up to dense layer ``upto`` (inclusive, default last) producing an fp32
        output (+ArgMax), or the full forward + loss kernel (no gradients) when ``with_loss``."""
        from . import plan_builder

        key = ("fwd", B, upto, post, with_loss, with_pull)
        if key not in self._plans:
            built = plan_builder.build(self, B, train=False, with_pull=with_pull, upto=upto, post=post, with_loss=with_loss)
            self._plans[key] = built.plan
            self._bufs[key] = StepBuffers(built.x_stage, built.y_stage, built.loss_out, built.result)
            self._keep.append(built.keep)
            self._order_after_build()
        return self._plans[key], self._bufs[key]

    EVAL_CHUNK = 4096

    def partition_loss(self, X: torch.Tensor, Y: Optional[torch.Tensor]) -> float:
        """Full-partition loss with the worker's current weights (reference: HogwildSparkModel.py:94-96)."""
        n = X.shape[0]
        total = 0.0
        for r in range(0, n, self.EVAL_CHUNK):
            rows = min(self.EVAL_CHUNK, n - r)
            plan, bufs = self.build_forward_plan(rows, with_loss=True, with_pull=self.pull_mode == "direct")
            with torch.cuda.stream(self.stream):
                bufs.x_stage.copy_(X[r:r + rows], non_blocking=True)
                if bufs.y_stage is not None and Y is not None:
                    bufs.y_stage.copy_(Y[r:r + rows], non_blocking=True)
                bufs.loss_out.zero_()
                plan.run(self.stream.cuda_stream)
            self.stream.synchronize()
            total += float(bufs.loss_out[0]) * rows
        return total / max(n, 1) + self._penalty_value()

    def _penalty_value(self) -> float:
        """The loss's L2 weight penalties, sum of c * sum(v^2), over the bf16 kernel replica (its W^T copy, which is always
        published) and the fp32 biases the forward plans read"""
        lay, total = self.layout, 0.0
        with torch.cuda.stream(self.stream):
            wsrc = self._weight_src()
            for name, c in self.plan.penalty.items():
                seg = lay.by_name(name)
                if seg.wt_off >= 0:
                    v = wsrc[seg.wt_off:seg.wt_off + seg.cols * seg.wt_ld].view(seg.cols, seg.wt_ld)[:, :seg.rows]
                else:
                    v = self.vec_local[seg.offset - lay.vec_offset:seg.offset - lay.vec_offset + seg.rows * seg.cols]
                total += c * float(v.double().square().sum())
        return total

    def predict(self, X: np.ndarray, upto: int, post: Optional[str]) -> np.ndarray:
        n = X.shape[0]
        Xp = torch.as_tensor(np.ascontiguousarray(X, dtype=np.float32)).pin_memory()
        outs = []
        for r in range(0, n, self.EVAL_CHUNK):
            rows = min(self.EVAL_CHUNK, n - r)
            plan, bufs = self.build_forward_plan(rows, upto=upto, post=post, with_pull=True)     # predict with fresh master weights
            with torch.cuda.stream(self.stream):
                bufs.x_stage.copy_(Xp[r:r + rows], non_blocking=True)
                plan.run(self.stream.cuda_stream)
            self.stream.synchronize()
            outs.append(bufs.result.detach().cpu().numpy().copy())
        return np.concatenate(outs, axis=0) if outs else np.zeros((0,), np.float32)

    def drain(self, timeout_s: float = 30.0) -> None:
        """Served push: block until the applier has consumed every gradient this worker posted."""
        self.stream.synchronize()
        if self.sharded:
            import time

            posted = int(self.my_posted[0])
            t0 = time.time()
            while True:
                acks = self.ack_words.view(-1, 16)[: self.master.n, 0].cpu()
                # every CTA of a shard's applier acknowledges a consumed push: posts x grid acknowledgements per shard
                if all(((int(a) - posted * self.master.applier_grid(r)) & 0xFFFFFFFF) < 0x80000000 for r, a in enumerate(acks)):
                    return
                if time.time() - t0 > timeout_s:
                    raise TimeoutError(f"shard appliers did not consume post {posted} of worker {self.worker_index} (acks={acks.tolist()})")
                time.sleep(0.0005)
        if not self.served:
            return
        import time

        posted = int(self.sync_push[4])
        flags = _view(self.master.flags_ptr(self.worker_index), self.C.MB_WORDS * 4, torch.int32, self.device)
        t0 = time.time()
        while True:
            applied = int(flags[self.C.MB_APPLIED])
            if ((applied - posted) & 0xFFFFFFFF) < 0x80000000:
                return
            if time.time() - t0 > timeout_s:
                raise TimeoutError(f"applier did not consume post {posted} of worker {self.worker_index} (applied={applied})")
            time.sleep(0.0005)

    def last_plan_names(self) -> List[str]:
        """Kernel names (``name@branch``) of the most recently built training plan."""
        return list(getattr(self, "_last_names", []))

    def need_w_map(self) -> Tuple[Dict[str, bool], Dict[str, bool]]:
        return plan_publish_needs(self.plan)

    # ------------------------------------------------------------------------------------------
    def run_prep(self, bufs: StepBuffers, stream) -> None:
        """Prepare a staged step's operands on ``stream`` (a CUDA graph once captured)."""
        st = stream.cuda_stream
        if not self.use_graphs:
            bufs.prep.run(st)
            return
        if not bufs.prep.captured():
            bufs.prep.capture(st)
        bufs.prep.replay(st)

    def run_plan(self, plan) -> None:
        """Launch one step on the worker stream (CUDA graph after the first eager execution)."""
        st = self.stream.cuda_stream
        if not self.use_graphs:
            plan.run(st)
            return
        if not plan.captured():
            plan.run(st)                      # eager warm-up (sets func attributes, validates launches)
            self.stream.synchronize()
            # the eager step consumed the gradient; capture records a second, identical step
            plan.capture(st)
            return
        plan.replay(st)


def plan_publish_needs(lp: LayerPlan) -> Tuple[Dict[str, bool], Dict[str, bool]]:
    """Which bf16 layouts each kernel variable must be published in (W for dgrad, W^T for forward)."""
    need_w: Dict[str, bool] = {}
    need_wt: Dict[str, bool] = {}
    first = True
    for l in lp.layers:
        if l.kind in ("dense", "conv"):
            need_wt[l.kernel] = True
            need_w[l.kernel] = not first
            first = False
    return need_w, need_wt


def external_push(master: MasterState, layout: ParamLayout, spec: OptimizerSpec, grads: Sequence[np.ndarray], acquire_lock: bool) -> None:
    """Apply one host-provided gradient list through the fused push kernel."""
    C = native.cuda_ext()
    dev = master.device
    with torch.cuda.device(dev):
        g = torch.from_numpy(layout.flatten(grads)).to(dev)
        segs = torch.frombuffer(bytearray(C.pack_segs(layout.seg_rows())), dtype=torch.uint8).to(dev)
        tmap = torch.from_numpy(layout.tile_map()).to(dev)
        sync = torch.zeros(8, dtype=torch.int32, device=dev)
        loss = torch.zeros(2, dtype=torch.float32, device=dev)
        args = dict(state=native.ptr(master.state), ctrl=native.ptr(master.ctrl), shadow_dst=[native.ptr(master.shadow)],
                    grad=native.ptr(g), loss_acc=native.ptr(loss), loss_out=native.ptr(loss) + 4, segs=native.ptr(segs),
                    tile_map=native.ptr(tmap), num_tiles=int(tmap.shape[0]), optimizer=spec.opt_id,
                    lock_mode=1 if acquire_lock else 0, grad_scale=1.0, hyper=spec.native_hyper())
        C.push(args, native.ptr(sync), 0, native.current_stream())
        _sync_current(dev)
