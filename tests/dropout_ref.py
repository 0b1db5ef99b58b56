"""Host reference of the fused dropout mask of the GEMM epilogue (csrc/gemm_sm90.cu, ``epi_chunk``).

Element (row, col) of a layer's output is kept when lane ``col & 3`` of Philox4x32-10 (Salmon et al., SC'11) over the
counter (row, col >> 2, step counter, stream) with key (seed, 0x5F3759DF) lies below ``keep * 2^32``; the product and
its clamp are float32 operations, as in the kernel.  ``dropout_seed`` is the seed ``plan_builder.build`` gives a plan.
"""
import os

import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK32 = np.uint64(0xFFFFFFFF)
KEY1 = 0x5F3759DF


def philox4x32_10(counter, key):
    """Philox4x32-10 of broadcastable uint32 arrays: ``counter`` = (c0, c1, c2, c3), ``key`` = (k0, k1).  Returns the
    four output words as uint32 arrays."""
    c = [np.asarray(v, dtype=np.uint64) & _MASK32 for v in counter]
    c = list(np.broadcast_arrays(*c))
    k0, k1 = (int(v) & 0xFFFFFFFF for v in key)
    for _ in range(10):
        p0, p1 = _M0 * c[0], _M1 * c[2]                # exact: both factors < 2^32
        hi0, lo0 = p0 >> np.uint64(32), p0 & _MASK32
        hi1, lo1 = p1 >> np.uint64(32), p1 & _MASK32
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return [v.astype(np.uint32) for v in c]


def keep_threshold(keep):
    """uint32(min(float32(keep) * 2^32, 4294967040)) in float32 arithmetic"""
    t = np.minimum(np.float32(keep) * np.float32(4294967296.0), np.float32(4294967040.0))
    return np.uint32(t)


def dropout_mask(B, N, keep, seed, stream, ctr):
    """bool [B, N]: the elements the epilogue keeps in a layer output of B rows and N columns"""
    row = np.arange(B, dtype=np.uint64)[:, None]
    col = np.arange(N, dtype=np.uint64)[None, :]
    words = philox4x32_10((row, col >> np.uint64(2), np.uint64(int(ctr) & 0xFFFFFFFF), np.uint64(int(stream) & 0xFFFFFFFF)),
                          (seed, KEY1))
    lane = (col & np.uint64(3)).astype(np.int64)
    rnd = np.choose(np.broadcast_to(lane, (B, N)), words)
    return rnd < keep_threshold(keep)


def dropout_seed(worker_index, ctr_ptr=None):
    """The seed of a plan's dropout layers: the base seed, the worker index and, for a training plan, the address of its
    step counter (a forward-only plan has no counter: its masks use counter 0 and the seed without that term)"""
    base = int(os.environ.get("SPARKFLOW_DROPOUT_SEED", "20260921"))
    return (base ^ (0x9E3779B9 * (worker_index + 1)) ^ ((ctr_ptr >> 4) if ctr_ptr is not None else 0)) & 0xFFFFFFFF
