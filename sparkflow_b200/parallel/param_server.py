"""Host parameter server: the CPU / gloo twin of the fused GPU push/pull path.

Reference behaviour that is preserved (lifeomic/sparkflow/sparkflow/HogwildSparkModel.py:175-244):
  * the master holds the weights AND all optimizer state; workers only ever send raw gradients;
  * ONE optimizer step per push, gradients are never summed across workers;
  * ``acquire_lock=False`` (Hogwild): pulls and updates race freely; ``True``: writer-priority RW lock;
  * a failing update is swallowed and counted, training aborts after ``max_errors`` (= iters) failures.
Reference behaviour that is fixed: no 8 s start-up sleep (readiness is explicit), no HTTP/pickle.

Two transports expose the same ``pull`` / ``push`` calls to the worker loop:
  * :class:`LocalTransport` – workers are threads of the driver process (Spark ``local[N]`` analogue);
  * :class:`GlooTransport`  – one process per worker, rank 0 hosts the server threads, messages are
    flat fp32 tensors over ``torch.distributed`` send/recv (BASELINE.json config 1: CPU / gloo).
"""
from __future__ import annotations

import itertools
import threading
import time
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from ..ops.optimizers import OptimizerSpec, apply_update
from .rwlock import RWLock


class TooManyFailures(RuntimeError):
    pass


class ParameterServer:
    """Master copy of the flat parameters + optimizer slots."""

    def __init__(self, weights: Sequence[np.ndarray], spec: OptimizerSpec, acquire_lock: bool = False, max_errors: int = 1000):
        self.shapes = [tuple(np.shape(w)) for w in weights]
        self.sizes = [int(np.prod(s)) if s else 1 for s in self.shapes]
        flat = np.concatenate([np.asarray(w, dtype=np.float32).reshape(-1) for w in weights]) if weights else np.zeros(0, np.float32)
        self.spec = spec
        # element-interleaved state [P, 1 + slots]: (p_i, slot0_i, slot1_i, ...) are adjacent, so a Hogwild
        # write-back (one memcpy) stores every element's tuple together, like TF's fused Apply* kernels
        ns = spec.num_slots
        self.state = torch.empty(flat.size, 1 + ns, dtype=torch.float32)
        self.state[:, 0] = torch.from_numpy(flat)
        for i in range(ns):
            self.state[:, 1 + i] = spec.slot_init(i)
        self.p = self.state[:, 0]
        self.slots = [self.state[:, 1 + i] for i in range(ns)]
        self.lock = RWLock() if acquire_lock else None
        self.max_errors = max_errors
        self.pushes = 0
        self.errors = 0
        self.dropped = 0
        self._counter = itertools.count(1)
        self._count_lock = threading.Lock()
        self.fault_hook: Optional[Callable[[int], Optional[str]]] = None     # push index -> None | 'drop' | 'raise' | 'delay:<s>'

    # -- the two "routes" ---------------------------------------------------------------------------
    def get_parameters(self) -> torch.Tensor:
        if self.lock:
            with self.lock.reading():
                return self.p.clone().contiguous()
        return self.p.clone().contiguous()

    def _bump(self, field: str) -> None:
        with self._count_lock:
            setattr(self, field, getattr(self, field) + 1)

    def update_parameters(self, grad_flat: torch.Tensor) -> str:
        with self._count_lock:
            idx = next(self._counter)
        action = self.fault_hook(idx) if self.fault_hook else None
        if action == "drop":
            self._bump("dropped")
            return "dropped"
        if action and action.startswith("delay:"):
            time.sleep(float(action.split(":", 1)[1]))
        try:
            if action == "raise":
                raise RuntimeError("injected update failure")
            if grad_flat.numel() != self.p.numel():
                raise ValueError("gradient size does not match the parameter vector")
            if self.lock:
                with self.lock.writing():
                    self._apply(grad_flat)
            else:
                self._apply(grad_flat)
        except Exception:
            self._bump("errors")
            if self.errors >= self.max_errors:
                raise TooManyFailures("Too many failures during training")
            return "failed"
        return "completed"

    HOGWILD_CHUNK = 8192      # elements per read-modify-write of a Hogwild push

    def _apply(self, g: torch.Tensor) -> None:
        # the optimizer step number comes from an atomic counter: two racing pushes never share a bias-correction step
        with self._count_lock:
            self.pushes += 1
            step = self.pushes
        if self.lock is not None:
            apply_update(self.spec, self.p, g, self.slots, step)
            return
        # Hogwild: like TF's in-place Apply* kernels (use_locking=False) and the GPU push kernel, pushes race PER ELEMENT.
        # The state is walked in small chunks; each chunk's (p, slots) tuples are read, updated together in private
        # storage and written back, so a concurrent push can only lose the updates of the chunk both are inside at the
        # same instant (not the whole push, which a clone-everything / copy-everything-back scheme would lose), and no
        # thread ever combines its momentum with another thread's half-written second moment.
        ns, n, ck = self.spec.num_slots, self.state.shape[0], self.HOGWILD_CHUNK
        for lo in range(0, n, ck):
            hi = min(lo + ck, n)
            local = self.state[lo:hi].clone()
            apply_update(self.spec, local[:, 0], g[lo:hi], [local[:, 1 + i] for i in range(ns)], step)
            self.state[lo:hi] = local

    def slot_arrays(self) -> List[List[np.ndarray]]:
        return [self.unflatten(s.clone().contiguous()) for s in self.slots]

    def load_slots(self, slots: Sequence[Sequence[np.ndarray]], step: int) -> None:
        for i, per_var in enumerate(slots[: self.spec.num_slots]):
            self.state[:, 1 + i] = torch.from_numpy(np.concatenate([np.asarray(a, np.float32).reshape(-1) for a in per_var]))
        self.pushes = int(step)

    # -- conversions ----------------------------------------------------------------------------------
    def unflatten(self, flat: torch.Tensor) -> List[np.ndarray]:
        out, off = [], 0
        arr = flat.detach().cpu().numpy()
        for shp, n in zip(self.shapes, self.sizes):
            out.append(arr[off:off + n].reshape(shp).copy())
            off += n
        return out

    def weights(self) -> List[np.ndarray]:
        return self.unflatten(self.get_parameters())


def flatten_grads(grads: Sequence) -> torch.Tensor:
    return torch.cat([(g if isinstance(g, torch.Tensor) else torch.as_tensor(np.asarray(g))).reshape(-1).to(torch.float32).cpu() for g in grads])


class LocalTransport:
    def __init__(self, server: ParameterServer):
        self.server = server

    def pull(self) -> List[np.ndarray]:
        return self.server.unflatten(self.server.get_parameters())

    def push(self, grads: Sequence) -> str:
        return self.server.update_parameters(flatten_grads(grads))

    def close(self) -> None:
        pass


# -------------------------------------------------------------------------------------------------
# gloo
# -------------------------------------------------------------------------------------------------
_OP_PULL, _OP_PUSH, _OP_DONE = 1, 2, 3


class GlooServer:
    """Rank-0 side: one service thread per remote worker (the reference's Flask is ``threaded=True``:
    one thread per request, so updates from different workers interleave exactly like here)."""

    def __init__(self, server: ParameterServer, world_size: int, group=None):
        import torch.distributed as dist

        self.server, self.world, self.group, self.dist = server, world_size, group, dist
        self.threads = [threading.Thread(target=self._serve, args=(r,), daemon=True, name=f"ps-serve-{r}") for r in range(1, world_size)]
        self.failure: Optional[BaseException] = None
        for t in self.threads:
            t.start()

    def _serve(self, src: int) -> None:
        dist = self.dist
        n = self.server.p.numel()
        try:
            while True:
                hdr = torch.zeros(2, dtype=torch.int64)
                dist.recv(hdr, src=src, group=self.group, tag=src)
                op = int(hdr[0])
                if op == _OP_DONE:
                    return
                if op == _OP_PULL:
                    dist.send(self.server.get_parameters(), dst=src, group=self.group, tag=1000 + src)
                elif op == _OP_PUSH:
                    g = torch.empty(n, dtype=torch.float32)
                    dist.recv(g, src=src, group=self.group, tag=src)
                    try:
                        status = self.server.update_parameters(g)
                    except TooManyFailures as exc:
                        self.failure = exc
                        status = "fatal"
                    code = {"completed": 0, "failed": 1, "dropped": 2, "fatal": 3}[status]
                    dist.send(torch.tensor([code], dtype=torch.int64), dst=src, group=self.group, tag=1000 + src)
        except Exception as exc:  # pragma: no cover - transport failure
            self.failure = exc

    def join(self, timeout: Optional[float] = None) -> None:
        for t in self.threads:
            t.join(timeout)


class GlooTransport:
    """Worker-side stub (ranks != 0).  Rank 0's own worker uses a :class:`LocalTransport`."""

    def __init__(self, rank: int, shapes: Sequence[tuple], group=None):
        import torch.distributed as dist

        self.rank, self.group, self.dist = rank, group, dist
        self.shapes = [tuple(s) for s in shapes]
        self.sizes = [int(np.prod(s)) if s else 1 for s in self.shapes]
        self.n = int(sum(self.sizes))
        # ONE transport per rank: the partitions of a rank run on threads, and the server has one service thread per
        # rank, so every pull / push exchange (header, payload, reply share the rank's tags) is done under this mutex
        self._mutex = threading.Lock()
        self._closed = False

    def _hdr(self, op: int) -> None:
        self.dist.send(torch.tensor([op, self.n], dtype=torch.int64), dst=0, group=self.group, tag=self.rank)

    def pull(self) -> List[np.ndarray]:
        with self._mutex:
            self._hdr(_OP_PULL)
            flat = torch.empty(self.n, dtype=torch.float32)
            self.dist.recv(flat, src=0, group=self.group, tag=1000 + self.rank)
        arr, out, off = flat.numpy(), [], 0
        for shp, n in zip(self.shapes, self.sizes):
            out.append(arr[off:off + n].reshape(shp).copy())
            off += n
        return out

    def push(self, grads: Sequence) -> str:
        flat = flatten_grads(grads)
        with self._mutex:
            self._hdr(_OP_PUSH)
            self.dist.send(flat, dst=0, group=self.group, tag=self.rank)
            code = torch.zeros(1, dtype=torch.int64)
            self.dist.recv(code, src=0, group=self.group, tag=1000 + self.rank)
        status = {0: "completed", 1: "failed", 2: "dropped", 3: "fatal"}[int(code)]
        if status == "fatal":
            raise TooManyFailures("Too many failures during training")
        return status

    def close(self) -> None:
        """Tell the rank's service thread to exit: exactly once per rank, whether or not it trained a partition."""
        with self._mutex:
            if not self._closed:
                self._closed = True
                self._hdr(_OP_DONE)
