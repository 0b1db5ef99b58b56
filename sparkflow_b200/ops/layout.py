"""Flat parameter layout shared by the master, the replicas and the push/pull kernels.

The reference ships parameters as a python list of per-variable numpy arrays in
``tf.trainable_variables()`` order (lifeomic/sparkflow/sparkflow/ml_util.py:9-28).  On the GPU all
variables live in ONE flat fp32 buffer (params, gradients and every optimizer slot use the same
offsets) so that a push is a single multi-tensor kernel launch, plus ONE bf16 "publish" buffer that
holds, for every matrix, the two K-major operand layouts the wgmma GEMMs consume:

* ``W``   [in, ld]  row-major  – B operand of dgrad  (dx = dy . W^T)
* ``W^T`` [out, ld] row-major  – B operand of forward (y = x . W)

Matrices come first and 1-D variables (biases) are packed into a contiguous tail so a pull can
fetch them with one 16-byte-granular fp32 copy.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

TILE_R = 32
TILE_C = 64


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


@dataclass
class Segment:
    name: str
    shape: Tuple[int, ...]          # original variable shape (e.g. [5,5,1,32] for a conv kernel)
    rows: int                       # matrix view [rows, cols]; 1-D variables: rows = 1
    cols: int
    offset: int                     # element offset in the flat fp32 buffers
    index: int                      # position in trainable-variable order
    w_off: int = -1                 # bf16 publish offsets (-1: not published)
    w_ld: int = 0
    wt_off: int = -1
    wt_ld: int = 0

    @property
    def size(self) -> int:
        return self.rows * self.cols


@dataclass
class ParamLayout:
    segments: List[Segment] = field(default_factory=list)   # in trainable-variable order
    total: int = 0                  # flat fp32 elements (padded to a multiple of 4)
    vec_offset: int = 0             # start of the 1-D tail
    vec_count: int = 0              # elements in the tail (multiple of 4)
    shadow_total: int = 0           # bf16 elements in the publish buffer (multiple of 64)

    @classmethod
    def build(cls, shapes: Sequence[Tuple[str, Tuple[int, ...]]], need_w: Optional[Dict[str, bool]] = None,
              need_wt: Optional[Dict[str, bool]] = None) -> "ParamLayout":
        """``shapes``: (name, shape) in trainable order. ``need_w`` / ``need_wt`` select which bf16
        layouts are published per matrix (default: both)."""
        segs: List[Segment] = []
        for i, (name, shape) in enumerate(shapes):
            shape = tuple(int(s) for s in shape)
            if len(shape) <= 1:
                rows, cols = 1, int(np.prod(shape)) if shape else 1
            else:
                rows, cols = int(np.prod(shape[:-1])), shape[-1]
            segs.append(Segment(name=name, shape=shape, rows=rows, cols=cols, offset=-1, index=i))
        off = 0
        for s in segs:                       # matrices first
            if s.rows > 1:
                s.offset = off
                off = round_up(off + s.size, 4)
        vec_offset = off
        for s in segs:                       # 1-D tail
            if s.rows == 1:
                s.offset = off
                off = round_up(off + s.size, 4)
        total = round_up(off, 4)
        sh = 0
        for s in segs:
            if s.rows == 1:
                continue
            if need_w is None or need_w.get(s.name, True):
                s.w_off, s.w_ld = sh, round_up(s.cols, 8)
                sh = round_up(sh + s.rows * s.w_ld, 64)
            if need_wt is None or need_wt.get(s.name, True):
                s.wt_off, s.wt_ld = sh, round_up(s.rows, 8)
                sh = round_up(sh + s.cols * s.wt_ld, 64)
        return cls(segments=segs, total=total, vec_offset=vec_offset, vec_count=total - vec_offset,
                   shadow_total=max(round_up(sh, 64), 64))

    # ---- host <-> flat conversions ------------------------------------------------------
    def by_name(self, name: str) -> Segment:
        for s in self.segments:
            if s.name == name:
                return s
        raise KeyError(name)

    def flatten(self, weights: Sequence[np.ndarray]) -> np.ndarray:
        flat = np.zeros(self.total, dtype=np.float32)
        assert len(weights) == len(self.segments), "weights list does not match the variable list"
        for s, w in zip(self.segments, weights):
            flat[s.offset:s.offset + s.size] = np.asarray(w, dtype=np.float32).reshape(-1)
        return flat

    def unflatten(self, flat: np.ndarray) -> List[np.ndarray]:
        return [np.array(flat[s.offset:s.offset + s.size], dtype=np.float32).reshape(s.shape) for s in self.segments]

    def valid_mask(self) -> np.ndarray:
        m = np.zeros(self.total, dtype=bool)
        for s in self.segments:
            m[s.offset:s.offset + s.size] = True
        return m

    # ---- tables for the push kernel -------------------------------------------------------
    def seg_rows(self) -> List[List[int]]:
        return [[s.offset, s.rows, s.cols, s.w_off, s.w_ld, s.wt_off, s.wt_ld] for s in self.segments]

    def tile_map(self) -> np.ndarray:
        tiles: List[Tuple[int, int, int]] = []
        for i, s in enumerate(self.segments):
            for tr in range((s.rows + TILE_R - 1) // TILE_R):
                for tc in range((s.cols + TILE_C - 1) // TILE_C):
                    tiles.append((i, tr, tc))
        return np.asarray(tiles, dtype=np.int32).reshape(-1, 3)

    def tile_prefix(self) -> List[int]:
        """Index of each segment's first push tile in :meth:`tile_map` order (one extra entry: the tile count)."""
        pre, acc = [], 0
        for s in self.segments:
            pre.append(acc)
            acc += ((s.rows + TILE_R - 1) // TILE_R) * ((s.cols + TILE_C - 1) // TILE_C)
        pre.append(acc)
        return pre

    def publish_reference(self, flat: np.ndarray) -> np.ndarray:
        """What the publish buffer must contain for the given fp32 params (fp32 values, to be
        compared after bf16 rounding)."""
        out = np.zeros(self.shadow_total, dtype=np.float32)
        for s in self.segments:
            w = flat[s.offset:s.offset + s.size].reshape(s.rows, s.cols)
            if s.w_off >= 0:
                blk = np.zeros((s.rows, s.w_ld), dtype=np.float32)
                blk[:, :s.cols] = w
                out[s.w_off:s.w_off + blk.size] = blk.reshape(-1)
            if s.wt_off >= 0:
                blk = np.zeros((s.cols, s.wt_ld), dtype=np.float32)
                blk[:, :s.rows] = w.T
                out[s.wt_off:s.wt_off + blk.size] = blk.reshape(-1)
        return out
