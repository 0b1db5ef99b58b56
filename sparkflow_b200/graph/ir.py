"""MetaGraphDef (proto3-JSON or binary) -> GraphIR.

The reference moves models around as ``json_format.MessageToJson(MetaGraphDef)`` strings and parses
them back on the parameter server, on every worker and in ``predict_func``
(lifeomic/sparkflow/sparkflow/HogwildSparkModel.py:45-53,131-132,188-192; ml_util.py:57-69).  GraphIR is
our parsed form: nodes with decoded attrs, the trainable variables in collection order (this order
is the order of every weights list in the public API) and the ``losses`` collection.
"""
from __future__ import annotations

import base64
import json
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Tuple, Union

import numpy as np

from . import pbwire

_NP = {
    "DT_FLOAT": np.float32, "DT_DOUBLE": np.float64, "DT_INT32": np.int32, "DT_INT64": np.int64, "DT_BOOL": np.bool_,
    "DT_UINT8": np.uint8, "DT_HALF": np.float16, "DT_INT8": np.int8, "DT_INT16": np.int16,
}


def _dims(shape_obj: Optional[Dict[str, Any]]) -> Optional[List[int]]:
    if shape_obj is None or shape_obj.get("unknownRank"):
        return None
    return [int(d.get("size", 0)) for d in shape_obj.get("dim", [])]


def decode_tensor(t: Dict[str, Any]) -> np.ndarray:
    dt = t.get("dtype", "DT_FLOAT")
    if isinstance(dt, int):
        dt = pbwire.DATA_TYPE.get(dt, "DT_FLOAT")
    if dt == "DT_STRING":
        return np.asarray([base64.b64decode(v) for v in t.get("stringVal", [])], dtype=object)
    npd = _NP.get(dt)
    if npd is None:
        return np.zeros(0, dtype=np.float32)      # exotic dtypes only occur in saver / summary plumbing
    shape = _dims(t.get("tensorShape")) or []
    n = int(np.prod(shape)) if shape else 1
    if "tensorContent" in t and t["tensorContent"]:
        arr = np.frombuffer(base64.b64decode(t["tensorContent"]), dtype=np.dtype(npd).newbyteorder("<")).astype(npd)
        return arr.reshape(shape)
    for key in ("floatVal", "doubleVal", "intVal", "int64Val", "boolVal", "halfVal"):
        if key in t and len(t[key]):
            vals = np.asarray([float(v) if key in ("floatVal", "doubleVal") else int(v) if key != "boolVal" else bool(v) for v in t[key]])
            if key == "halfVal":
                vals = vals.astype(np.uint16).view(np.float16)
            vals = vals.astype(npd)
            if vals.size == n:
                return vals.reshape(shape)
            out = np.empty(n, dtype=npd)          # TF "splat": trailing values repeat the last one
            out[:vals.size] = vals[:n]
            out[vals.size:] = vals[-1]
            return out.reshape(shape)
    return np.zeros(shape, dtype=npd)


def decode_attr(a: Dict[str, Any]) -> Any:
    if "type" in a:
        v = a["type"]
        return pbwire.DATA_TYPE.get(v, v) if isinstance(v, int) else v
    if "shape" in a:
        return _dims(a["shape"])
    if "i" in a:
        return int(a["i"])
    if "f" in a:
        return float(a["f"])
    if "b" in a:
        return bool(a["b"])
    if "s" in a:
        return base64.b64decode(a["s"]).decode("utf-8", "replace")
    if "tensor" in a:
        return decode_tensor(a["tensor"])
    if "list" in a:
        lst = a["list"]
        if "i" in lst:
            return [int(v) for v in lst["i"]]
        if "f" in lst:
            return [float(v) for v in lst["f"]]
        if "s" in lst:
            return [base64.b64decode(v).decode("utf-8", "replace") for v in lst["s"]]
        if "shape" in lst:
            return [_dims(v) for v in lst["shape"]]
        if "type" in lst:
            return list(lst["type"])
        if "b" in lst:
            return [bool(v) for v in lst["b"]]
        return []
    return None


@dataclass
class Node:
    name: str
    op: str
    inputs: List[Tuple[str, int]]          # data inputs (node, output index)
    control: List[str]
    attrs: Dict[str, Any]


@dataclass
class VarInfo:
    name: str                              # node name, e.g. 'dense/kernel'
    shape: Tuple[int, ...]
    dtype: str
    initial_value: Optional[str] = None    # tensor name of the initial value
    snapshot: Optional[str] = None         # 'dense/kernel/read:0'


def split_ref(ref: str) -> Tuple[str, int]:
    if ":" in ref:
        n, i = ref.rsplit(":", 1)
        if i.isdigit():
            return n, int(i)
    return ref, 0


@dataclass
class GraphIR:
    nodes: Dict[str, Node] = field(default_factory=dict)
    order: List[str] = field(default_factory=list)
    trainable: List[VarInfo] = field(default_factory=list)
    variables: List[VarInfo] = field(default_factory=list)
    losses: List[str] = field(default_factory=list)
    meta: Dict[str, Any] = field(default_factory=dict)
    raw: Dict[str, Any] = field(default_factory=dict)

    # ------------------------------------------------------------------
    @classmethod
    def from_metagraph(cls, mg: Union[str, bytes, Dict[str, Any], Any]) -> "GraphIR":
        if hasattr(mg, "data") and isinstance(getattr(mg, "data"), dict):     # tfcompat.MetaGraphDef
            mg = mg.data
        if isinstance(mg, bytes):
            mg = pbwire.decode("MetaGraphDef", mg)
        elif isinstance(mg, str):
            mg = json.loads(mg)
        if not isinstance(mg, dict):
            raise TypeError(f"cannot parse a MetaGraphDef from {type(mg)!r}")
        ir = cls(raw=mg, meta=mg.get("metaInfoDef", {}))
        gd = mg.get("graphDef") or mg.get("graph_def") or {}
        for nd in gd.get("node", []):
            data_in, ctrl = [], []
            for ref in nd.get("input", []):
                if ref.startswith("^"):
                    ctrl.append(ref[1:])
                else:
                    data_in.append(split_ref(ref))
            attrs = {k: decode_attr(v) for k, v in (nd.get("attr") or {}).items()}
            node = Node(nd["name"], nd["op"], data_in, ctrl, attrs)
            ir.nodes[node.name] = node
            ir.order.append(node.name)
        coll = mg.get("collectionDef") or mg.get("collection_def") or {}
        ir.trainable = ir._vars_from_collection(coll.get("trainable_variables"))
        ir.variables = ir._vars_from_collection(coll.get("variables")) or list(ir.trainable)
        if not ir.trainable:
            # graphs without collections: every variable node, in creation order, is trainable
            ir.trainable = [ir._var_from_node(n) for n in ir.order if ir.nodes[n].op in ("VariableV2", "Variable", "VarHandleOp")]
            ir.variables = ir.variables or list(ir.trainable)
        losses = coll.get("losses") or {}
        ir.losses = list((losses.get("nodeList") or {}).get("value", []))
        return ir

    def _var_from_node(self, name: str, vd: Optional[Dict[str, Any]] = None) -> VarInfo:
        node = self.nodes[name]
        shape = node.attrs.get("shape")
        if shape is None:
            shapes = node.attrs.get("_output_shapes") or [None]
            shape = shapes[0]
        init = (vd or {}).get("initialValueName")
        if init is None and f"{name}/Assign" in self.nodes:
            a = self.nodes[f"{name}/Assign"]
            if len(a.inputs) >= 2:
                init = f"{a.inputs[1][0]}:{a.inputs[1][1]}"
        return VarInfo(name=name, shape=tuple(shape or ()), dtype=node.attrs.get("dtype", "DT_FLOAT"), initial_value=init,
                       snapshot=(vd or {}).get("snapshotName"))

    def _vars_from_collection(self, c: Optional[Dict[str, Any]]) -> List[VarInfo]:
        out: List[VarInfo] = []
        if not c:
            return out
        for b in (c.get("bytesList") or {}).get("value", []):
            vd = pbwire.decode("VariableDef", base64.b64decode(b))
            name = split_ref(vd.get("variableName", ""))[0]
            if name in self.nodes:
                out.append(self._var_from_node(name, vd))
        for ref in (c.get("nodeList") or {}).get("value", []):
            name = split_ref(ref)[0]
            if name in self.nodes and self.nodes[name].op in ("VariableV2", "Variable", "VarHandleOp"):
                out.append(self._var_from_node(name))
        return out

    # ------------------------------------------------------------------
    def node_of(self, tensor_name: str) -> Node:
        return self.nodes[split_ref(tensor_name)[0]]

    def has_tensor(self, tensor_name: str) -> bool:
        return split_ref(tensor_name)[0] in self.nodes

    def placeholder_shape(self, tensor_name: str) -> Optional[List[int]]:
        return self.node_of(tensor_name).attrs.get("shape")

    def to_json(self) -> str:
        return json.dumps(self.raw)

    def param_shapes(self) -> List[Tuple[str, Tuple[int, ...]]]:
        return [(v.name, v.shape) for v in self.trainable]

    def num_params(self) -> int:
        return int(sum(int(np.prod(v.shape)) if v.shape else 1 for v in self.trainable))
