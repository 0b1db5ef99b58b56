"""The per-partition training loop (engine-agnostic) and the two engines that execute its steps.

Loop semantics are the reference's ``handle_model`` (lifeomic/sparkflow/sparkflow/HogwildSparkModel.py:38-100):

* per outer iteration: pull, optional shuffle, then ONE of
  A. ``mini_stochastic_iters >= 1`` – that many random minibatches (without replacement inside a batch),
     all computed on the weights pulled at the start of the iteration (no re-pull), one push each;
  B. ``mini_batch_size >= 1`` – a full sweep in contiguous minibatches, re-pulling before each;
  C. otherwise – one gradient over the whole partition;
* a failed push is reported ("Timeout error from partition ...") and training continues;
* ``verbose`` / ``loss_callback``: full-partition loss after every outer iteration.

Engines:
* :class:`TorchEngine` – GraphProgram (autograd) + a host transport (threads or gloo). CPU path, and the
  generic path for graphs the compiled plan does not cover.
* :class:`B200Engine`  – DeviceWorker: compiled sm_90a step plans, pinned-host partitions fed through
  a side stream, fused NVLink push/pull.
"""
from __future__ import annotations

import uuid
from typing import Callable, List, Optional, Sequence, Union

import os

import numpy as np
import torch

from ..graph.executor import GraphProgram
from ..graph.ir import GraphIR

Rows = Union[slice, np.ndarray]


def check_class_labels(labels: np.ndarray, n_classes: int) -> None:
    """Class-index labels of a sparse softmax cross-entropy plan: each must be finite and truncate (toward zero, as TF's
    Cast does) into [0, n_classes).  TF rejects any other label too; the step kernels would silently give its row no
    target.  Raises ValueError naming the first bad row."""
    v = np.asarray(labels, dtype=np.float32)
    v = v[:, 0] if v.ndim == 2 else v.reshape(-1)
    with np.errstate(invalid="ignore"):
        bad = ~np.isfinite(v) | (np.trunc(v) < 0) | (np.trunc(v) >= n_classes)
    if bad.any():
        r = int(np.argmax(bad))
        raise ValueError(f"label {v[r]} of row {r} is not a class index in [0, {n_classes}) (the graph takes class labels "
                         f"through a sparse softmax cross-entropy over {n_classes} classes)")


def clamp_batch(n: int, mini_batch_size: int) -> int:
    """``mini_batch_size > n  ->  n - 1`` (reference quirk, ml_util.py:105-106)."""
    return n - 1 if mini_batch_size > n else mini_batch_size


class Engine:
    partition_rows = 0

    def load_partition(self, features: np.ndarray, labels: Optional[np.ndarray]) -> None:
        raise NotImplementedError

    def train(self, rows: Rows, pull: bool) -> None:
        raise NotImplementedError

    def partition_loss(self) -> float:
        raise NotImplementedError

    def finish(self) -> None:
        pass


def run_partition(engine: Engine, features: np.ndarray, labels: Optional[np.ndarray], iters: int = 1000,
                  mini_batch_size: int = -1, shuffle: bool = True, mini_stochastic_iters: int = -1, verbose: int = 0,
                  loss_callback: Optional[Callable[[float, int, str], None]] = None, partition_id: Optional[str] = None,
                  seed: Optional[int] = None, on_iteration: Optional[Callable[[int], None]] = None) -> str:
    from ..utils.metrics import MetricsLogger
    from ..utils.trace import nvtx_pop, nvtx_push

    metrics = MetricsLogger()
    partition_id = partition_id or uuid.uuid4().hex
    n = int(features.shape[0])
    if n == 0:
        return partition_id
    engine.load_partition(features, labels)
    rng = np.random.default_rng(seed)
    order: Optional[np.ndarray] = None
    fast = hasattr(engine, "train_contiguous")
    sweep = mini_stochastic_iters < 1 and mini_batch_size >= 1
    for i in range(iters):
        nvtx_push(f"sparkflow {partition_id} iteration {i}")
        if shuffle:
            order = rng.permutation(n)
            if fast and sweep:
                engine.permute(order)          # physical shuffle (what the reference does), then contiguous batches
                order = None

        def rows_of(sel: Rows) -> Rows:
            if order is None:
                return sel
            return order[sel]

        if mini_stochastic_iters >= 1:
            mbs = clamp_batch(n, mini_batch_size)
            for j in range(mini_stochastic_iters):
                if mbs <= 0:
                    sel: Rows = slice(0, n)
                else:
                    sel = rng.choice(n, mbs, replace=False)
                engine.train(rows_of(sel), pull=(j == 0))
        elif mini_batch_size >= 1:
            # the reference strides by the ORIGINAL mini_batch_size and only clamps the slice length
            # (HogwildSparkModel.py:73-74 + ml_util.py:105-106): mbs > n means ONE batch of n-1 rows per iteration
            mbs = max(clamp_batch(n, mini_batch_size), 1)
            stride = max(mini_batch_size, 1)
            if fast and order is None and stride == mbs:
                full = n // mbs
                engine.train_contiguous([k * mbs for k in range(full)], mbs, pull=True)
                if full * mbs < n:
                    engine.train(slice(full * mbs, n), pull=True)
            else:
                for r in range(0, n, stride):
                    engine.train(rows_of(slice(r, min(r + mbs, n))), pull=True)
        else:
            engine.train(rows_of(slice(0, n)), pull=True)

        if verbose or loss_callback:
            loss = engine.partition_loss()
            if verbose:
                print("Partition Id: %s, Iteration: %i, Loss: %f" % (partition_id, i, loss))
            if loss_callback:
                loss_callback(loss, i, partition_id)
            if metrics.enabled:
                metrics.log(event="iteration", partition=partition_id, iteration=i, loss=float(loss), rows=n)
        elif metrics.enabled:
            metrics.log(event="iteration", partition=partition_id, iteration=i, rows=n)
        if on_iteration is not None:
            on_iteration(i)
        nvtx_pop()
    engine.finish()
    return partition_id


# -------------------------------------------------------------------------------------------------
class TorchEngine(Engine):
    def __init__(self, ir: GraphIR, tf_input: str, tf_label: Optional[str], transport, device: str = "cpu",
                 partition_id: str = ""):
        self.prog = GraphProgram(ir, device)
        self.tf_input, self.tf_label, self.transport = tf_input, tf_label, transport
        self.weights: Optional[List[np.ndarray]] = None
        self.partition_id = partition_id
        self.failed_pushes = 0

    def load_partition(self, features, labels):
        self.X = torch.as_tensor(np.asarray(features, dtype=np.float32))
        self.Y = None if labels is None else torch.as_tensor(np.asarray(labels, dtype=np.float32))
        self.partition_rows = self.X.shape[0]

    def _feed(self, rows: Rows):
        idx = rows if isinstance(rows, slice) else torch.as_tensor(np.asarray(rows, dtype=np.int64))
        feed = {self.tf_input: self.X[idx]}
        if self.tf_label is not None and self.Y is not None:
            feed[self.tf_label] = self.Y[idx]
        return feed

    def train(self, rows, pull):
        if pull or self.weights is None:
            self.weights = self.transport.pull()
        _, grads = self.prog.loss_and_grads(self._feed(rows), self.weights)
        try:
            self.transport.push(grads)
        except Exception as exc:
            from .param_server import TooManyFailures

            if isinstance(exc, TooManyFailures):
                raise
            self.failed_pushes += 1
            print("Timeout error from partition %s" % self.partition_id)

    def partition_loss(self) -> float:
        return self.prog.loss(self._feed(slice(0, self.partition_rows)), self.weights or self.transport.pull())


# -------------------------------------------------------------------------------------------------
class B200Engine(Engine):
    """Pinned-host partition + DeviceWorker.  Every step copies its minibatch host->device on a side
    stream (double-buffered staging) and leaves the step's loss in a pinned host ring."""

    LOSS_RING = 64

    def __init__(self, worker):
        self.w = worker
        self.step_idx = 0
        self.loss_ring = torch.zeros(self.LOSS_RING, dtype=torch.float32).pin_memory()
        # staging slots: the host may run SLOTS-1 steps ahead of the GPU (H2D of step k+1.. overlaps step k)
        self.SLOTS = max(2, int(os.environ.get("SPARKFLOW_SLOTS", "4")))
        S = self.SLOTS
        self._slot_free = [torch.cuda.Event() for _ in range(S)]
        self._slot_ready = [torch.cuda.Event() for _ in range(S)]
        self._primed = [False] * S
        self._pending = [None] * S              # slot -> (ring index, pinned loss word) not yet harvested
        self.h2d_bytes = 0
        self.d2h_bytes = 0
        self._gather = [None] * S
        self._driver = None
        self._driver_plans = {}
        self._driver_last = None
        self.partition_mode = os.environ.get("SPARKFLOW_PARTITION", "pinned")
        self.resident = False
        self.Xd = self.Yd = self.perm_d = None
        self._resident_driver = {}
        self._idx_pinned = [None] * S
        self._X2 = self._Y2 = None

    def load_partition(self, features, labels):
        """``SPARKFLOW_PARTITION=pinned`` (default): the partition stays in pinned host memory and every step copies its
        minibatch host->device.  ``resident``: the partition is uploaded to HBM once (80 GB per H100 hold any Spark
        partition the reference could train on); shuffles are a device index permutation and every step gathers its rows
        on the device - no PCIe traffic in the training loop.  ``auto``: resident when it fits in a quarter of free HBM."""
        lp = self.w.plan
        if labels is not None and lp.loss == "sparse_softmax_xent":
            check_class_labels(labels, lp.layers[-1].out_features)        # before any device work
        self.X = torch.as_tensor(np.ascontiguousarray(features, dtype=np.float32)).pin_memory()
        self.Y = None
        if labels is not None and not self.w.plan.target_is_input:
            self.Y = torch.as_tensor(np.ascontiguousarray(labels, dtype=np.float32)).pin_memory()
        self.partition_rows = self.X.shape[0]
        mode = self.partition_mode
        if mode == "auto":
            need = self.X.numel() * 4 + (0 if self.Y is None else self.Y.numel() * 4)
            free, _ = torch.cuda.mem_get_info(self.w.device)
            mode = "resident" if need * 4 <= free else "pinned"
        self.resident = mode == "resident"
        self.Xd = self.Yd = self.perm_d = None
        if self.resident:
            with torch.cuda.stream(self.w.stream):
                self.Xd = self.X.to(self.w.device, non_blocking=True)
                self.Yd = None if self.Y is None else self.Y.to(self.w.device, non_blocking=True)
                self.perm_d = torch.arange(self.partition_rows, dtype=torch.int32, device=self.w.device)
            self.w.stream.synchronize()
            self._resident_driver = {}

    def _host_batch(self, rows: Rows, slot: int):
        if isinstance(rows, slice):
            return self.X[rows], (None if self.Y is None else self.Y[rows])
        idx = torch.as_tensor(np.asarray(rows, dtype=np.int64))
        B = idx.numel()
        g = self._gather[slot]
        if g is None or g[0].shape[0] != B:
            gx = torch.empty(B, self.X.shape[1], dtype=torch.float32).pin_memory()
            gy = None if self.Y is None else torch.empty(B, self.Y.shape[1], dtype=torch.float32).pin_memory()
            g = self._gather[slot] = (gx, gy)
        torch.index_select(self.X, 0, idx, out=g[0])
        if g[1] is not None:
            torch.index_select(self.Y, 0, idx, out=g[1])
        return g

    def _train_resident(self, rows, pull, slot):
        w = self.w
        B = (rows.stop - rows.start) if isinstance(rows, slice) else len(rows)
        plan, bufs = w.build_plan(B, slot, with_pull=pull, resident=(self.Xd, self.Yd))
        if self._primed[slot]:
            self._slot_free[slot].synchronize()
            self._harvest(slot)
        with torch.cuda.stream(w.stream):
            if isinstance(rows, slice):
                bufs.idx.copy_(self.perm_d[rows], non_blocking=True)
            else:
                # explicit row ids index the partition in its CURRENT (possibly permuted) order
                host = self._idx_pinned[slot]
                if host is None or host.numel() != B:
                    host = self._idx_pinned[slot] = torch.empty(B, dtype=torch.int64).pin_memory()
                host.copy_(torch.as_tensor(np.asarray(rows, dtype=np.int64)))
                self.h2d_bytes += B * 8
                bufs.idx.copy_(self.perm_d[host.to(w.device, non_blocking=True)], non_blocking=True)
        w.run_prep(bufs, w.stream)
        w.run_plan(plan)
        self._slot_free[slot].record(w.stream)
        self._pending[slot] = (self.step_idx % self.LOSS_RING, bufs.loss_out)
        self.d2h_bytes += 4
        self._primed[slot] = True
        self._driver_last = None
        self.step_idx += 1

    def train(self, rows, pull, slot=None):
        w = self.w
        slot = (self.step_idx % self.SLOTS) if slot is None else slot
        if self._driver_last is not None:
            # the native loop ran since the last Python-driven step: its steps share these staging buffers
            w.stream.synchronize()
            if self._driver is not None:
                self._driver.flush()
        if self.resident:
            return self._train_resident(rows, pull, slot)
        B = (rows.stop - rows.start) if isinstance(rows, slice) else len(rows)
        plan, bufs = w.build_plan(B, slot, with_pull=pull, staged=True)
        if self._primed[slot]:
            self._slot_free[slot].synchronize()            # host gather buffer + staging are reusable
            self._harvest(slot)
        hx, hy = self._host_batch(rows, slot)
        with torch.cuda.stream(w.copy_stream):
            bufs.x_stage.copy_(hx, non_blocking=True)
            self.h2d_bytes += hx.numel() * 4
            if bufs.y_stage is not None and hy is not None:
                bufs.y_stage.copy_(hy, non_blocking=True)
                self.h2d_bytes += hy.numel() * 4
            w.run_prep(bufs, w.copy_stream)
            self._slot_ready[slot].record(w.copy_stream)
        w.stream.wait_event(self._slot_ready[slot])
        w.run_plan(plan)
        # the step's last kernel (push / post) stores the loss into the plan's pinned host word: a 4-byte zero-copy
        # D2H per step, harvested into the ring when the slot is reused or the loss is asked for
        self._slot_free[slot].record(w.stream)
        self._pending[slot] = (self.step_idx % self.LOSS_RING, bufs.loss_out)
        self.d2h_bytes += 4
        self._primed[slot] = True
        self._driver_last = None
        self.step_idx += 1

    def _harvest(self, slot: int) -> None:
        pend = self._pending[slot]
        if pend is not None:
            self.loss_ring[pend[0]] = float(pend[1][0])
            self._pending[slot] = None

    def permute(self, order: np.ndarray) -> None:
        """Shuffle the partition: a device index permutation when it is HBM-resident, otherwise a physical shuffle of the
        pinned host copy (threaded native row gather into the spare buffers)."""
        if self.resident:
            with torch.cuda.stream(self.w.stream):
                order_d = torch.as_tensor(np.asarray(order, dtype=np.int64)).to(self.w.device)
                self.perm_d = self.perm_d[order_d].contiguous()
            return
        self.w.stream.synchronize()
        self.w.copy_stream.synchronize()
        from ..ops.native import host_ext

        H = host_ext()
        if self._X2 is None:
            self._X2 = torch.empty_like(self.X).pin_memory()
            self._Y2 = None if self.Y is None else torch.empty_like(self.Y).pin_memory()
        idx = np.ascontiguousarray(order, dtype=np.int64)
        H.gather_rows(self.X.data_ptr(), self._X2.data_ptr(), idx, self.X.shape[1] * 4, 8)
        self.X, self._X2 = self._X2, self.X
        if self.Y is not None:
            H.gather_rows(self.Y.data_ptr(), self._Y2.data_ptr(), idx, self.Y.shape[1] * 4, 4)
            self.Y, self._Y2 = self._Y2, self.Y
        self._driver = None                     # the DMA driver has the host base pointers baked into it
        self._driver_plans = {}

    # ---- native inner loop -------------------------------------------------------------------------
    def train_contiguous(self, starts: Sequence[int], batch: int, pull: bool = True) -> None:
        """Run ``len(starts)`` steps on contiguous row blocks ``[s, s + batch)`` through the C++ StepDriver - no Python
        in the loop.  A pinned partition is fed by a copy-engine H2D of every minibatch on the copy stream, SLOTS-deep,
        with an event hand-off to the step graph; an HBM-resident one by a device-side row-id copy and gather."""
        w = self.w
        if not w.use_graphs or len(starts) == 0:
            for s0 in starts:
                self.train(slice(int(s0), int(s0) + batch), pull)
            return
        starts = [int(v) for v in starts]
        if self.resident:
            self._train_contiguous_resident(starts, batch, pull)
            return
        key = (batch, pull)
        drv_ids = self._driver_plans.get(key)
        if drv_ids is None:
            if self._driver is None:
                self._driver = w.C.StepDriver(w.stream.cuda_stream, w.copy_stream.cuda_stream, self.X.data_ptr(),
                                              self.X.shape[1] * 4, 0 if self.Y is None else self.Y.data_ptr(),
                                              0 if self.Y is None else self.Y.shape[1] * 4, self.loss_ring.data_ptr(), self.LOSS_RING)
            drv_ids = []
            for slot in range(self.SLOTS):
                plan, bufs = w.build_plan(batch, slot, with_pull=pull, staged=True)
                if not plan.captured():
                    # the first use of a plan runs it eagerly (a REAL step on the next scheduled minibatch) and
                    # captures the graph; step counts therefore stay exactly iters x batches
                    if not starts:
                        self._driver_plans.pop(key, None)
                        return
                    self.train(slice(starts[0], starts[0] + batch), pull, slot=slot)
                    starts = starts[1:]
                drv_ids.append(self._driver.add_plan(plan, bufs.x_stage.data_ptr(), 0 if bufs.y_stage is None else bufs.y_stage.data_ptr(),
                                                     bufs.loss_out.data_ptr(), batch, self._captured_prep(bufs)))
            self._driver_plans[key] = drv_ids
        if not starts:
            return
        self.w.stream.synchronize()       # python-path steps (if any) are done before the driver takes over the ring
        for slot in range(self.SLOTS):
            self._harvest(slot)
        ids = np.asarray([drv_ids[(self._driver.steps() + k) % self.SLOTS] for k in range(len(starts))], dtype=np.int32)
        self._driver.run(ids, np.asarray(starts, dtype=np.int64))
        n = len(starts)
        self.h2d_bytes += n * batch * (self.X.shape[1] + (0 if self.Y is None else self.Y.shape[1])) * 4
        self.d2h_bytes += n * 4
        self._driver_last = (self._driver.steps() - 1) % self.LOSS_RING
        self.step_idx += n

    def _captured_prep(self, bufs):
        """The StepDriver replays a staged step's prep plan on the copy stream, after the minibatch copy."""
        if not bufs.prep.captured():
            bufs.prep.capture(self.w.copy_stream.cuda_stream)
        return bufs.prep

    def _train_contiguous_resident(self, starts: List[int], batch: int, pull: bool) -> None:
        w = self.w
        key = (batch, pull, self.Xd.data_ptr())
        drv = self._resident_driver.get(key)
        if drv is None:
            d = w.C.StepDriver(w.stream.cuda_stream, w.copy_stream.cuda_stream, 0, 0, 0, 0, self.loss_ring.data_ptr(), self.LOSS_RING)
            for slot in range(self.SLOTS):
                plan, bufs = w.build_plan(batch, slot, with_pull=pull, resident=(self.Xd, self.Yd))
                if not plan.captured():
                    plan.capture(w.stream.cuda_stream)
                d.add_plan(plan, bufs.idx.data_ptr(), 0, bufs.loss_out.data_ptr(), batch, self._captured_prep(bufs))
            drv = self._resident_driver[key] = d
        w.stream.synchronize()
        for slot in range(self.SLOTS):
            self._harvest(slot)
        n = len(starts)
        ids = np.asarray([(drv.steps() + k) % self.SLOTS for k in range(n)], dtype=np.int32)
        drv.run_resident(ids, np.asarray(starts, dtype=np.int64), self.perm_d.data_ptr())
        self.d2h_bytes += n * 8
        self._driver = drv
        self._driver_last = (drv.steps() - 1) % self.LOSS_RING
        self.step_idx += n

    def last_loss(self) -> float:
        self.w.stream.synchronize()
        for slot in range(self.SLOTS):
            self._harvest(slot)
        if self._driver is not None:
            self._driver.flush()
        if self._driver_last is not None:
            return float(self.loss_ring[self._driver_last])
        return float(self.loss_ring[(self.step_idx - 1) % self.LOSS_RING])

    def partition_loss(self) -> float:
        return self.w.partition_loss(self.X, self.Y)

    def finish(self):
        self.w.drain()
