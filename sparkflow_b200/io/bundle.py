"""TensorFlow V2 checkpoint bundles (``<prefix>.index`` + ``<prefix>.data-00000-of-00001``) and the
``checkpoint`` state file – read AND write, without TensorFlow.

Layout (SURVEY.md section 2.5-5; decoded from lifeomic/sparkflow/tests/test_model): the index is a
leveldb-format SSTable whose first key ``""`` maps to a ``BundleHeaderProto`` and every other key
(a variable name, lexicographically sorted) to a ``BundleEntryProto{dtype, shape, shard_id, offset, size,
crc32c}``; the data file is the raw little-endian tensor bytes at those offsets; ``crc32c`` is the
*masked* CRC-32C of the tensor bytes.  The SSTable container and crc32c are native (csrc/hostlib.cpp);
the protos go through ``graph.pbwire``.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional

import numpy as np

from ..graph import pbwire
from ..ops.native import host_ext

_DT = {"DT_FLOAT": np.float32, "DT_DOUBLE": np.float64, "DT_INT32": np.int32, "DT_INT64": np.int64, "DT_BOOL": np.bool_,
       "DT_HALF": np.float16, "DT_UINT8": np.uint8, "DT_INT8": np.int8, "DT_INT16": np.int16}
_DT_REV = {np.dtype(v): k for k, v in _DT.items()}


def _shard_name(prefix: str, shard: int, num_shards: int) -> str:
    return "%s.data-%05d-of-%05d" % (prefix, shard, num_shards)


def read_bundle_entries(prefix: str) -> Dict[str, dict]:
    H = host_ext()
    with open(prefix + ".index", "rb") as fh:
        raw = fh.read()
    out: Dict[str, dict] = {}
    for key, value in H.sstable_read(raw, True):
        k = bytes(key).decode("utf-8")
        if k == "":
            out[""] = pbwire.decode("BundleHeaderProto", bytes(value))
        else:
            out[k] = pbwire.decode("BundleEntryProto", bytes(value))
    return out


def read_bundle(prefix: str, verify: bool = True) -> Dict[str, np.ndarray]:
    """All tensors of a V2 checkpoint, keyed by variable name."""
    H = host_ext()
    entries = read_bundle_entries(prefix)
    header = entries.pop("", {})
    num_shards = int(header.get("numShards", 1))
    if header.get("endianness", "LITTLE") != "LITTLE":
        raise NotImplementedError("big-endian bundles are not supported")
    shards: Dict[int, bytes] = {}
    tensors: Dict[str, np.ndarray] = {}
    for name, e in entries.items():
        if e.get("slices"):
            raise NotImplementedError(f"partitioned variable '{name}' is not supported")
        shard = int(e.get("shardId", 0))
        if shard not in shards:
            with open(_shard_name(prefix, shard, num_shards), "rb") as fh:
                shards[shard] = fh.read()
        off, size = int(e.get("offset", 0)), int(e.get("size", 0))
        blob = shards[shard][off:off + size]
        if verify and "crc32c" in e:
            if H.crc32c_mask(H.crc32c(blob)) != int(e["crc32c"]):
                raise IOError(f"checksum mismatch for tensor '{name}' in {prefix}")
        dt = _DT.get(e.get("dtype", "DT_FLOAT"))
        if dt is None:
            continue
        shape = [int(d.get("size", 0)) for d in e.get("shape", {}).get("dim", [])]
        tensors[name] = np.frombuffer(blob, dtype=np.dtype(dt).newbyteorder("<")).astype(dt).reshape(shape)
    return tensors


def write_bundle(prefix: str, tensors: Dict[str, np.ndarray]) -> None:
    """Write ``tensors`` as a single-shard V2 checkpoint."""
    H = host_ext()
    os.makedirs(os.path.dirname(os.path.abspath(prefix)), exist_ok=True)
    entries: List[tuple] = [(b"", pbwire.encode("BundleHeaderProto", {"numShards": 1, "endianness": "LITTLE",
                                                                      "version": {"producer": 1}}))]
    data = bytearray()
    for name in sorted(tensors, key=lambda s: s.encode("utf-8")):
        arr = np.asarray(tensors[name], order="C")          # (ascontiguousarray would promote 0-d to 1-d)
        dt = _DT_REV.get(arr.dtype)
        if dt is None:
            raise TypeError(f"unsupported dtype {arr.dtype} for tensor '{name}'")
        blob = arr.astype(arr.dtype.newbyteorder("<")).tobytes()
        entry = {"dtype": dt, "shape": {"dim": [{"size": str(d)} for d in arr.shape]} if arr.ndim else {},
                 "offset": str(len(data)), "size": str(len(blob)), "crc32c": H.crc32c_mask(H.crc32c(blob))}
        entries.append((name.encode("utf-8"), pbwire.encode("BundleEntryProto", entry)))
        data += blob
    index = H.sstable_write([(bytes(k), bytes(v)) for k, v in entries], 4096)
    with open(prefix + ".index", "wb") as fh:
        fh.write(bytes(index))
    with open(_shard_name(prefix, 0, 1), "wb") as fh:
        fh.write(bytes(data))


def read_checkpoint_state(checkpoint_dir: str, filename: str = "checkpoint") -> Optional[str]:
    """``tf.train.latest_checkpoint``: prefix named by the text-proto ``checkpoint`` file."""
    path = os.path.join(checkpoint_dir, filename)
    if not os.path.exists(path):
        return None
    with open(path) as fh:
        for line in fh:
            line = line.strip()
            if line.startswith("model_checkpoint_path:"):
                val = line.split(":", 1)[1].strip().strip('"')
                full = val if os.path.isabs(val) else os.path.join(checkpoint_dir, val)
                return full if os.path.exists(full + ".index") else None
    return None


def write_checkpoint_state(checkpoint_dir: str, basename: str, filename: str = "checkpoint") -> None:
    with open(os.path.join(checkpoint_dir, filename), "w") as fh:
        fh.write('model_checkpoint_path: "%s"\nall_model_checkpoint_paths: "%s"\n' % (basename, basename))
