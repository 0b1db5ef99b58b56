"""Symmetric GPU memory for the sharded parameter server.

Every GPU of the job allocates a segment with the SAME layout through the CUDA virtual-memory-management API
(``cuMemCreate``); every GPU maps every peer's segment (NVLink peer access), so kernels address "field f of GPU r" as
``base[r] + offset(f)``.  Optionally the segments are also bound to an NVSwitch **multicast object** (NVLS): a store to
the multicast alias (``multimem.st`` in the kernels) is replicated by the switch into every GPU's segment.

This replaces the reference's transport rendezvous (``master_url`` + Flask port + 8 s sleep,
lifeomic/sparkflow/sparkflow/HogwildSparkModel.py:118-135,145-166): there is no server address, only mapped memory.

Two process models:

* SPMD (one process per GPU, ``torchrun``): physical handles travel between the processes as POSIX file descriptors over
  abstract-namespace Unix sockets (``SCM_RIGHTS``); ``torch.distributed`` (gloo) is used only for the barrier / token.
* single process, several GPUs (one worker thread per GPU): one process creates and maps everything directly.
"""
from __future__ import annotations

import os
import socket
import threading
import uuid
from typing import Dict, List, Optional, Sequence

import torch

from ..ops import native
from . import dist as D


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class _FdServer:
    """Serves this rank's exported file descriptors to its peers (one request per connection: the key, answered with
    the descriptor as ancillary data)."""

    def __init__(self, name: str):
        self.fds: Dict[str, int] = {}
        self.sock = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        self.sock.bind("\0" + name)              # abstract namespace: no file to clean up
        self.sock.listen(64)
        self.sock.settimeout(0.2)
        self._stop = False
        self.thread = threading.Thread(target=self._loop, daemon=True, name="sparkflow-fd-server")
        self.thread.start()

    def offer(self, key: str, fd: int) -> None:
        self.fds[key] = fd

    def _loop(self) -> None:
        while not self._stop:
            try:
                conn, _ = self.sock.accept()
            except socket.timeout:
                continue
            except OSError:
                return
            with conn:
                try:
                    conn.settimeout(5.0)
                    key = conn.recv(256).decode()
                    fd = self.fds.get(key)
                    if fd is None:
                        conn.sendall(b"no")
                    else:
                        socket.send_fds(conn, [b"ok"], [fd])
                except OSError:
                    pass

    def close(self) -> None:
        self._stop = True
        try:
            self.sock.close()
        except OSError:
            pass
        self.thread.join(timeout=2)


def _fetch_fd(name: str, key: str, timeout: float = 30.0) -> int:
    import time

    t0 = time.time()
    while True:
        try:
            with socket.socket(socket.AF_UNIX, socket.SOCK_STREAM) as s:
                s.settimeout(5.0)
                s.connect("\0" + name)
                s.sendall(key.encode())
                msg, fds, _, _ = socket.recv_fds(s, 16, 1)
                if msg == b"ok" and fds:
                    return fds[0]
        except OSError:
            pass
        if time.time() - t0 > timeout:
            raise TimeoutError(f"could not fetch descriptor '{key}' from {name}")
        time.sleep(0.05)


class SymmetricHeap:
    """``n`` identically sized segments, one per GPU; ``base[r]`` is GPU r's segment as seen from the calling
    process / device, ``mc_base`` the multicast alias (0 when NVLS is not available or not requested)."""

    def __init__(self, nbytes: int, ctx: Optional[D.DistContext] = None, devices: Optional[Sequence[int]] = None,
                 multicast: bool = False, tag: str = "heap"):
        self.C = native.cuda_ext()
        self.ctx = ctx if ctx is not None else D.DistContext()
        self.spmd = self.ctx.world > 1
        self.devices = [int(d) for d in (devices if devices is not None else [torch.cuda.current_device()])]
        self.n = self.ctx.world if self.spmd else len(self.devices)
        self.rank = self.ctx.rank if self.spmd else 0
        self.tag = tag
        self.base: List[int] = [0] * self.n
        self.mc_base = 0
        self._handles: List[int] = []
        self._mc_handle = 0
        self._maps: List[int] = []
        C = self.C
        dev0 = self.devices[0]
        uniq = sorted(set(self.devices))            # a device may host several segments (two shards on one GPU in tests)
        self._uniq = uniq
        want_mc = bool(multicast) and os.environ.get("SPARKFLOW_MULTICAST", "1") != "0" and self.n > 1 and (self.spmd or len(uniq) == self.n)
        if want_mc:
            ok = all(C.vmm_multicast_supported(d) for d in self.devices)
            if self.spmd:
                ok = all(D.all_gather_object(self.ctx, ok))
            want_mc = ok
        for d in uniq:
            with torch.cuda.device(d):
                torch.zeros(1, device=f"cuda:{d}")               # make sure the primary context exists
        gran = C.vmm_granularity(dev0, want_mc, self.n)
        self.nbytes = round_up(max(int(nbytes), 1), gran)
        try:
            if self.spmd:
                self._init_spmd(want_mc)
            else:
                self._init_local(want_mc)
        except Exception:
            self.close()
            raise

    # -- single process: this process owns every device -----------------------------------------------------
    def _init_local(self, want_mc: bool) -> None:
        C = self.C
        for i, d in enumerate(self.devices):
            h = C.vmm_create(d, self.nbytes)
            self._handles.append(h)
            self.base[i] = C.vmm_map(h, self.nbytes, self._uniq)
            self._maps.append(self.base[i])
            with torch.cuda.device(d):
                C.memset_d8(self.base[i], 0, self.nbytes)
        if want_mc:
            try:
                mc = C.mc_create(self.n, self.nbytes)
                self._mc_handle = mc
                for d in self.devices:
                    C.mc_add_device(mc, d)
                for h in self._handles:
                    C.mc_bind(mc, 0, h, 0, self.nbytes)
                self.mc_base = C.vmm_map(mc, self.nbytes, self._uniq)
                self._maps.append(self.mc_base)
            except RuntimeError as exc:
                self._mc_error = str(exc)
                self.mc_base = 0

    # -- one process per GPU ------------------------------------------------------------------------------------
    def _init_spmd(self, want_mc: bool) -> None:
        C, ctx = self.C, self.ctx
        dev = self.devices[0]
        token = D.broadcast_object(ctx, uuid.uuid4().hex if ctx.rank == 0 else None, src=0)
        name = lambda r: f"sparkflow_b200-{token}-{self.tag}-{r}"       # noqa: E731
        server = _FdServer(name(ctx.rank))
        own_fds: List[int] = []
        try:
            h = C.vmm_create(dev, self.nbytes)
            self._handles.append(h)
            fd = C.vmm_export_fd(h)
            own_fds.append(fd)
            server.offer("seg", fd)
            mc_ok = want_mc
            if want_mc and ctx.rank == 0:
                try:
                    self._mc_handle = C.mc_create(self.n, self.nbytes)
                    mfd = C.vmm_export_fd(self._mc_handle)
                    own_fds.append(mfd)
                    server.offer("mc", mfd)
                except RuntimeError as exc:
                    self._mc_error = str(exc)
                    mc_ok = False
            if want_mc:
                mc_ok = D.broadcast_object(ctx, mc_ok, src=0)
            D.barrier(ctx)                                           # every server is listening, every fd is offered
            for r in range(self.n):
                if r == ctx.rank:
                    self.base[r] = C.vmm_map(h, self.nbytes, [dev])
                else:
                    pfd = _fetch_fd(name(r), "seg")
                    ph = C.vmm_import_fd(pfd)
                    os.close(pfd)
                    self._handles.append(ph)
                    self.base[r] = C.vmm_map(ph, self.nbytes, [dev])
                self._maps.append(self.base[r])
            C.memset_d8(self.base[ctx.rank], 0, self.nbytes)
            torch.cuda.synchronize(dev)
            if want_mc and mc_ok:
                if ctx.rank != 0:
                    mfd = _fetch_fd(name(0), "mc")
                    self._mc_handle = C.vmm_import_fd(mfd)
                    os.close(mfd)
                ok = True
                try:
                    C.mc_add_device(self._mc_handle, dev)
                except RuntimeError as exc:
                    self._mc_error = str(exc)
                    ok = False
                ok = all(D.all_gather_object(ctx, ok))                # also the barrier: every device is added before any bind
                if ok:
                    try:
                        C.mc_bind(self._mc_handle, 0, h, 0, self.nbytes)
                        self.mc_base = C.vmm_map(self._mc_handle, self.nbytes, [dev])
                        self._maps.append(self.mc_base)
                    except RuntimeError as exc:
                        self._mc_error = str(exc)
                        self.mc_base = 0
                ok = all(D.all_gather_object(ctx, self.mc_base != 0))
                if not ok:
                    self.mc_base = 0                                 # all or nothing: the kernels take one code path
            D.barrier(ctx)
        finally:
            server.close()
            for fd in own_fds:
                try:
                    os.close(fd)
                except OSError:
                    pass

    @property
    def multicast(self) -> bool:
        return self.mc_base != 0

    def close(self) -> None:
        C = self.C
        for va in self._maps:
            try:
                C.vmm_unmap(va, self.nbytes)
            except Exception:
                pass
        self._maps = []
        for h in self._handles:
            C.vmm_release(h)
        self._handles = []
        if self._mc_handle:
            C.vmm_release(self._mc_handle)
            self._mc_handle = 0
        self.base = [0] * self.n
        self.mc_base = 0
