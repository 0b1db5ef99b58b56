"""Writer-priority readers/writer lock (host side).

Same contract as the reference's lock (lifeomic/sparkflow/sparkflow/RWLock.py:10-65): many readers XOR
one writer; readers are held back while a writer holds the lock *or is waiting for it*, so updates
cannot starve.  Used by the host parameter server when ``acquire_lock=True``; the GPU path uses the
device-side twin in ``csrc/optim_push.cu`` (same state machine on one 32-bit word).
"""
from __future__ import annotations

import threading
from contextlib import contextmanager


class RWLock:
    def __init__(self) -> None:
        self._cond = threading.Condition(threading.Lock())
        self._active_readers = 0
        self._writer_active = False
        self._writers_waiting = 0

    # reference-compatible method names -----------------------------------------------------------
    def acquire_read(self) -> None:
        with self._cond:
            while self._writer_active or self._writers_waiting:
                self._cond.wait()
            self._active_readers += 1

    def acquire_write(self) -> None:
        with self._cond:
            self._writers_waiting += 1
            try:
                while self._writer_active or self._active_readers:
                    self._cond.wait()
            finally:
                self._writers_waiting -= 1
            self._writer_active = True

    def release(self) -> None:
        """Release whichever side the caller holds (the reference exposes a single ``release``)."""
        with self._cond:
            if self._writer_active:
                self._writer_active = False
            elif self._active_readers:
                self._active_readers -= 1
            else:
                raise RuntimeError("release() of an unlocked RWLock")
            self._cond.notify_all()

    # pythonic helpers -------------------------------------------------------------------------------
    @contextmanager
    def reading(self):
        self.acquire_read()
        try:
            yield
        finally:
            self.release()

    @contextmanager
    def writing(self):
        self.acquire_write()
        try:
            yield
        finally:
            self.release()

    @property
    def state(self) -> int:
        """>0: number of readers, -1: writer, 0: free (the reference's ``rwlock`` field)."""
        with self._cond:
            return -1 if self._writer_active else self._active_readers
