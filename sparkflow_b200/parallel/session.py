"""TrainingSession: owns the master state and the workers for one ``HogwildSparkModel.train`` call.

Execution modes (chosen automatically):

=============================  =================================================================
SPMD + GPUs (torchrun)          one rank per GPU; the master is sharded over the GPUs' symmetric VMM segments
                                (parallel/sharded.py; NVSwitch multicast publish); B200Engine everywhere.
SPMD, CPU only (gloo)           rank 0 hosts the ParameterServer + GlooServer threads; every rank
                                (0 included) runs a TorchEngine  (BASELINE.json config 1).
single process + GPUs           one worker thread per GPU (peer access to the master on cuda:0).
single process, CPU             worker threads + in-process ParameterServer (Spark local[N] analogue).
=============================  =================================================================

The reference's fixed costs are gone: no server process spawn, no 8 s sleep
(lifeomic/sparkflow/sparkflow/HogwildSparkModel.py:118,135) – ``open`` returns once the master is ready.
"""
from __future__ import annotations

import os
import sys
import threading
import warnings
from collections import Counter
from concurrent.futures import ThreadPoolExecutor
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ..graph.executor import GraphProgram
from ..graph.ir import GraphIR
from ..models.compiler import UnsupportedGraph, compile_graph
from ..ops.layout import ParamLayout
from ..ops.optimizers import OptimizerSpec
from . import dist as D
from .param_server import GlooServer, GlooTransport, LocalTransport, ParameterServer
from .worker import B200Engine, Engine, TorchEngine, run_partition

Partition = Tuple[np.ndarray, Optional[np.ndarray]]


# how many sessions each engine kind served in this process (printed by the test-suite summary and by bench.py)
ENGINE_USES: Counter = Counter()


class TrainingSession:
    def __init__(self, graph_json: str, tf_input: str, tf_label: Optional[str], optimizer: OptimizerSpec,
                 acquire_lock: bool = False, iters: int = 1000, mini_batch: int = -1, mini_stochastic_iters: int = -1,
                 shuffle: bool = True, verbose: int = 0, loss_callback: Optional[Callable] = None, engine: str = "auto",
                 seed: Optional[int] = None, initial_weights: Optional[Sequence[np.ndarray]] = None,
                 pull_mode: Optional[str] = None, resume_from: Optional[str] = None, checkpoint_dir: Optional[str] = None,
                 checkpoint_every: int = 0, push_mode: Optional[str] = None, devices: Optional[Sequence[int]] = None):
        self.ir = GraphIR.from_metagraph(graph_json)
        self.tf_input, self.tf_label, self.spec = tf_input, tf_label, optimizer
        self.acquire_lock, self.iters = bool(acquire_lock), int(iters)
        self.mini_batch, self.msi, self.shuffle = int(mini_batch), int(mini_stochastic_iters), bool(shuffle)
        self.verbose, self.loss_callback, self.seed = verbose, loss_callback, seed
        self.initial_weights = initial_weights
        self.pull_mode = pull_mode
        self.resume_from, self.checkpoint_dir, self.checkpoint_every = resume_from, checkpoint_dir, int(checkpoint_every or 0)
        self._resume_state = None
        self.graph_json = graph_json
        # push_mode: 'direct' = the worker applies the optimizer on the master's memory over NVLink;
        #            'served' = the worker posts its gradient to a mailbox and a persistent applier kernel on the
        #                       master GPU applies it (4 B/param over NVLink instead of 36 B, no remote round trips)
        self.push_mode = push_mode or os.environ.get("SPARKFLOW_PUSH_MODE") or "auto"
        self.devices = None if devices is None else [int(d) for d in devices]     # single-process mode: GPUs to use
        self.ctx = D.get_context()
        self.use_cuda = torch.cuda.is_available() and engine != "torch" and os.environ.get("SPARKFLOW_ENGINE", "") != "torch"
        self.engine_kind = "torch"
        self.engine_reason = "no CUDA device" if not torch.cuda.is_available() else "engine='torch' requested"
        if self.use_cuda:
            try:
                from .plan_builder import check_grammar

                check_grammar(compile_graph(self.ir, tf_input, tf_label))
                self.engine_kind = "b200"
                self.engine_reason = "graph compiled to the native sm_90a plan"
            except UnsupportedGraph as exc:
                if engine == "b200":
                    raise
                self.engine_reason = f"graph outside the compiled plan family: {exc}"
                warnings.warn(f"sparkflow_b200: graph is outside the compiled sm_90a plan family ({exc}); "
                              "running the generic PyTorch interpreter engine on the GPU instead", RuntimeWarning)
        elif engine == "b200":
            raise RuntimeError("engine='b200' requested but no CUDA device is available")
        ENGINE_USES[self.engine_kind] += 1
        if torch.cuda.is_available() and (self.engine_kind != "b200" or self.verbose or os.environ.get("SPARKFLOW_LOG_ENGINE")):
            # never silent about which engine trains the model on a GPU box
            print(f"[sparkflow_b200] engine={self.engine_kind} ({self.engine_reason})", file=sys.stderr, flush=True)
        self.master = None           # MasterState (GPU) or ParameterServer (host)
        self.gloo_server: Optional[GlooServer] = None
        self._gloo_transport: Optional[GlooTransport] = None      # one per non-master rank, shared by its partitions
        self._workers: List[object] = []
        self._dev_workers: dict = {}
        self._opened = False

    # -------------------------------------------------------------------------------------------
    def _init_weights(self) -> List[np.ndarray]:
        if self.resume_from:
            from ..utils.checkpoint import load_master_state

            w, slots, step = load_master_state(self.resume_from, [v.name for v in self.ir.trainable], self.spec)
            self._resume_state = (slots, step)
            return [np.asarray(a, dtype=np.float32) for a in w]
        if self.initial_weights is not None:
            return [np.asarray(w, dtype=np.float32) for w in self.initial_weights]
        return GraphProgram(self.ir).init_weights(seed=self.seed)

    def local_devices(self) -> List[torch.device]:
        if not self.use_cuda:
            return [torch.device("cpu")]
        if self.ctx.world > 1:
            return [torch.device("cuda", self.ctx.local_rank % torch.cuda.device_count())]
        if self.devices is not None:
            return [torch.device("cuda", i) for i in self.devices]
        return [torch.device("cuda", i) for i in range(torch.cuda.device_count())]

    def open(self) -> "TrainingSession":
        if self._opened:
            return self
        ctx = self.ctx
        if self.engine_kind == "b200":
            from .device_engine import MasterState, plan_publish_needs

            lp = compile_graph(self.ir, self.tf_input, self.tf_label)
            need_w, need_wt = plan_publish_needs(lp)
            self.layout = ParamLayout.build(self.ir.param_shapes(), need_w, need_wt)
            dev0 = self.local_devices()[0]
            n_workers = ctx.world if ctx.world > 1 else len(self.local_devices())
            shared = n_workers > 1
            if self.push_mode == "auto":
                self.push_mode = "sharded" if shared else "direct"
            n_mb = n_workers if self.push_mode == "served" else 0
            if self.push_mode == "sharded":
                from .sharded import ShardedMaster

                # accumulating (split-K) conv wgrads add into the mailboxes: the appliers hand them back zeroed
                self.master = ShardedMaster(self.layout, self.spec, ctx, self.local_devices(), mb_zero=any(l.kind == "conv" for l in lp.layers))
                w0 = self._init_weights() if (ctx.is_master or ctx.world == 1 or self.resume_from) else None
                self.master.load_weights(w0 if (ctx.is_master or ctx.world == 1) else None)
            elif ctx.world > 1:
                if ctx.is_master:
                    self.master = MasterState(self.layout, self.spec, dev0, n_mailboxes=n_mb)
                    self.master.load_weights(self._init_weights())
                    handle = self.master.ipc_handle()
                else:
                    handle = None
                handle = D.broadcast_object(ctx, handle, src=0)
                if not ctx.is_master:
                    self.master = MasterState.from_ipc(self.layout, self.spec, dev0, handle, n_mailboxes=n_mb)
                D.barrier(ctx)
            else:
                self.master = MasterState(self.layout, self.spec, dev0, n_mailboxes=n_mb)
                self.master.load_weights(self._init_weights())
                from ..ops import native

                for d in self.local_devices()[1:]:
                    with torch.cuda.device(d):
                        if not native.cuda_ext().enable_peer_access(dev0.index):
                            raise RuntimeError(f"GPU {d.index} cannot access the master on GPU {dev0.index} (no P2P)")
        else:
            if ctx.world > 1:
                if ctx.is_master:
                    self.master = ParameterServer(self._init_weights(), self.spec, self.acquire_lock, max_errors=max(self.iters, 1))
                    self.gloo_server = GlooServer(self.master, ctx.world, ctx.control_group)
                else:
                    self._gloo_transport = GlooTransport(ctx.rank, [v.shape for v in self.ir.trainable], ctx.control_group)
                D.barrier(ctx)
            else:
                self.master = ParameterServer(self._init_weights(), self.spec, self.acquire_lock, max_errors=max(self.iters, 1))
        if self._resume_state is not None and self.master is not None and (self.ctx.is_master or self.ctx.world == 1 or self.push_mode == "sharded"):
            slots, step = self._resume_state
            self.master.load_slots(slots, step)
        if self.engine_kind == "b200" and self.push_mode in ("served", "sharded") and self.master.owner:
            n_workers = ctx.world if ctx.world > 1 else len(self.local_devices())
            self.master.start_applier(self.acquire_lock, scope_sys=n_workers > 1, dbuf=self._dbuf())
        D.barrier(ctx)
        self._opened = True
        return self

    def _dbuf(self) -> bool:
        """Double-buffered publish is usable when every worker pulls into a replica (not TMA-direct from buffer 0)."""
        import os

        return (self.pull_mode or os.environ.get("SPARKFLOW_PULL_MODE", "copy")) == "copy"

    def master_desc(self) -> str:
        """One-line description of where the master state lives (goes into benchmark / log records)."""
        if self.engine_kind != "b200":
            return "host parameter server"
        n = self.ctx.world if self.ctx.world > 1 else len(self.local_devices())
        if self.push_mode == "sharded":
            return f"master sharded over {n} gpus, one applier per shard, multicast publish"
        return "master on gpu0" + (", mailbox + applier" if self.push_mode == "served" else ", worker-applied push")

    def sync_all(self) -> None:
        """Collective: drain every worker (its last push is applied everywhere), barrier, device-wide
        ``torch.cuda.synchronize()``, barrier - WITHOUT stopping the appliers (they are finite, re-queued kernels: a
        device-wide synchronise only waits for the launches already enqueued).  Benchmarks bracket timed regions with it."""
        ctx = self.ctx
        for w in self._workers:
            if hasattr(w, "drain"):
                w.drain()
        D.barrier(ctx)
        if self.use_cuda:
            for d in self.local_devices():
                torch.cuda.synchronize(d)
        D.barrier(ctx)

    def quiesce(self) -> None:
        """Collective: drain every worker, stop the applier, do a genuine device-wide ``torch.cuda.synchronize()``
        and bring the applier back.  Benchmarks bracket their timed regions with this (a device-wide synchronise
        can never return while the persistent applier kernel is resident)."""
        ctx = self.ctx
        for w in self._workers:
            if hasattr(w, "drain"):
                w.drain()
        D.barrier(ctx)
        served = self.engine_kind == "b200" and self.push_mode in ("served", "sharded")
        if served and self.master.owner:
            self.master.stop_applier()
        if served:
            D.barrier(ctx)                  # sharded: no applier anywhere may still be publishing into a peer's replica
        if self.use_cuda:
            for d in self.local_devices():
                torch.cuda.synchronize(d)
        if served and self.master.owner:
            n_workers = ctx.world if ctx.world > 1 else len(self.local_devices())
            self.master.start_applier(self.acquire_lock, scope_sys=n_workers > 1, dbuf=self._dbuf())
        D.barrier(ctx)

    # -- snapshot / resume ------------------------------------------------------------------------------
    def snapshot(self, prefix: str) -> Optional[str]:
        """Write the master's parameters + optimizer slots as a TF-V2 checkpoint (rank 0 only)."""
        if not (self.ctx.is_master or self.ctx.world == 1) or self.master is None:
            return None
        from ..utils.checkpoint import save_master_state

        if self.engine_kind == "b200":
            for w in self._workers:
                w.stream.synchronize()
            step = self.master.counters()["step"]
        else:
            step = self.master.pushes
        return save_master_state(prefix, [v.name for v in self.ir.trainable], self.master.weights(), self.master.slot_arrays(),
                                 self.spec, step, self.graph_json)

    def maybe_snapshot(self, iteration: int) -> None:
        if self.checkpoint_dir and self.checkpoint_every > 0 and (iteration + 1) % self.checkpoint_every == 0:
            import os

            os.makedirs(self.checkpoint_dir, exist_ok=True)
            self.snapshot(os.path.join(self.checkpoint_dir, f"master-{iteration + 1}"))

    # -------------------------------------------------------------------------------------------
    def make_engine(self, device: torch.device, partition_id: str = "", lane: Optional[int] = None) -> Engine:
        if self.engine_kind == "b200":
            from .device_engine import DeviceWorker, MasterState

            # one DeviceWorker per device for the whole session: it owns the replica, gradient buffers, streams and
            # captured CUDA graphs, all of which are reusable across partitions and partition_shuffles rounds
            devs = self.local_devices()
            if lane is None:
                lane = devs.index(device) if device in devs else 0
            w = self._dev_workers.get(lane)
            if w is None:
                master = self.master
                if self.push_mode != "sharded" and master.device != device:        # single-process multi-GPU: alias of the master seen from `device`
                    master = MasterState(self.layout, self.spec, device, base_ptr=self.master.base, n_mailboxes=self.master.ml.n_mailboxes)
                shared = self.ctx.world > 1 or len(self.local_devices()) > 1
                # mailbox index = position of the device in the session's device list (NOT its CUDA ordinal)
                widx = self.ctx.rank if self.ctx.world > 1 else lane
                w = DeviceWorker(self.ir, self.tf_input, self.tf_label, self.spec, master, acquire_lock=self.acquire_lock,
                                 pull_mode=self.pull_mode, device=device, shared=shared, worker_index=widx,
                                 reads_between_pulls=self.msi > 1 or bool(self.verbose) or self.loss_callback is not None)
                self._dev_workers[lane] = w
                self._workers.append(w)
            return B200Engine(w)
        if self.ctx.world > 1 and not self.ctx.is_master:
            transport = self._gloo_transport
        else:
            transport = LocalTransport(self.master)
        eng = TorchEngine(self.ir, self.tf_input, self.tf_label, transport, device=str(device) if device.type == "cuda" else "cpu",
                          partition_id=partition_id)
        self._workers.append(eng)
        return eng

    def train_partitions(self, partitions: Sequence[Partition]) -> None:
        """Train over ``partitions`` (global list; under SPMD every rank passes the same list and
        takes the partitions ``i % world == rank``)."""
        self.open()
        ctx = self.ctx
        if self.engine_kind == "b200" and self.push_mode in ("served", "sharded") and self.master.owner:
            if self.master.applier is None or not self.master.applier.alive():      # idle timeout between rounds
                n_workers = ctx.world if ctx.world > 1 else len(self.local_devices())
                self.master.start_applier(self.acquire_lock, scope_sys=n_workers > 1, dbuf=self._dbuf())
        D.barrier(ctx)
        mine = [(i, p) for i, p in enumerate(partitions) if i % ctx.world == ctx.rank]
        devices = self.local_devices()
        lanes: List[List[Tuple[int, Partition]]] = [[] for _ in devices]
        n_lanes = len(devices) if self.use_cuda else max(1, len(mine))
        if not self.use_cuda:
            devices = [torch.device("cpu")] * n_lanes
            lanes = [[] for _ in range(n_lanes)]
        for j, item in enumerate(mine):
            lanes[j % len(lanes)].append(item)
        errors: List[BaseException] = []

        def run_lane(lane_idx: int) -> None:
            dev = devices[lane_idx]
            if dev.type == "cuda":
                torch.cuda.set_device(dev)
            for pid, (feat, lab) in lanes[lane_idx]:
                engine = self.make_engine(dev, partition_id=f"partition-{pid}", lane=lane_idx if self.use_cuda else None)
                run_partition(engine, feat, lab, iters=self.iters, mini_batch_size=self.mini_batch, shuffle=self.shuffle,
                              mini_stochastic_iters=self.msi, verbose=self.verbose, loss_callback=self.loss_callback,
                              partition_id=f"partition-{pid}", seed=None if self.seed is None else self.seed + pid,
                              on_iteration=self.maybe_snapshot if (pid == 0 and self.checkpoint_every) else None)

        active = [i for i, l in enumerate(lanes) if l]
        if len(active) <= 1:
            for i in active:
                run_lane(i)
        else:
            with ThreadPoolExecutor(max_workers=len(active)) as ex:
                futs = [ex.submit(run_lane, i) for i in active]
                for f in futs:
                    try:
                        f.result()
                    except BaseException as exc:  # noqa: BLE001
                        errors.append(exc)
        if errors:
            raise errors[0]
        D.barrier(ctx)

    # -------------------------------------------------------------------------------------------
    def weights(self) -> List[np.ndarray]:
        ctx = self.ctx
        if self.engine_kind == "b200":
            for w in self._workers:
                w.drain()
            D.barrier(ctx)
            return self.master.weights()
        if ctx.world > 1:
            w = self.master.weights() if ctx.is_master else None
            return D.broadcast_object(ctx, w, src=0)
        return self.master.weights()

    def push_external(self, grads) -> None:
        """One optimizer step on the master from an externally computed gradient list."""
        if self.engine_kind == "b200":
            if self.push_mode == "sharded":
                raise NotImplementedError("push_external on a sharded master: open the session with push_mode='served' or 'direct'")
            from .device_engine import external_push

            external_push(self.master, self.layout, self.spec, [np.asarray(g, dtype=np.float32) for g in grads], self.acquire_lock)
        else:
            LocalTransport(self.master).push(grads)

    def counters(self) -> dict:
        if self.engine_kind == "b200":
            return self.master.counters()
        m = self.master
        if m is None:
            return {}
        return {"pushes": m.pushes, "errors": m.errors, "dropped": m.dropped}

    def close(self) -> None:
        if not self._opened:
            return
        ctx = self.ctx
        if self._gloo_transport is not None:
            self._gloo_transport.close()       # _OP_DONE exactly once per rank, also when it had no partition
            self._gloo_transport = None
        D.barrier(ctx)
        if self.gloo_server is not None:
            self.gloo_server.join(timeout=10)
            if self.gloo_server.failure:
                raise self.gloo_server.failure
        if self.engine_kind == "b200" and self.master is not None:
            for w in self._workers:
                try:
                    w.drain()
                except TimeoutError:
                    pass
            D.barrier(ctx)
            if self.push_mode == "sharded":
                self.master.stop_applier()      # nobody publishes into a peer's replica any more ...
                D.barrier(ctx)                  # ... before any rank unmaps its segments
            self.master.close()
        self._workers.clear()
        self._dev_workers.clear()
        self.master = None
        self._opened = False
