"""Graph / Tensor / Variable primitives of the TensorFlow-1.x compatible graph builder.

The reference serialises user models with ``tf.train.export_meta_graph`` inside ``build_graph``
(lifeomic/sparkflow/sparkflow/graph_utils.py:6-15).  TensorFlow cannot be installed here, so this
package provides the slice of the TF-1.x graph-construction API that the reference, its examples
and its tests use, emitting *TensorFlow-compatible* NodeDefs (same op names, attrs, variable /
initializer / read-node naming, collections) so that the MetaGraphDef JSON we produce has the layout
real TF produces and real TF graphs parse with the same IR.
"""
from __future__ import annotations

import base64
import contextlib
import threading
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np

from .. import pbwire

# ---------------------------------------------------------------------------
# dtypes
# ---------------------------------------------------------------------------


class DType:
    def __init__(self, name: str, enum: str, np_dtype):
        self.name, self.enum, self.np = name, enum, np.dtype(np_dtype)

    def __repr__(self):
        return f"tf.{self.name}"

    @property
    def as_numpy_dtype(self):
        return self.np.type

    def __eq__(self, other):
        return isinstance(other, DType) and other.enum == self.enum or (isinstance(other, str) and as_dtype(other).enum == self.enum)

    def __hash__(self):
        return hash(self.enum)


float32 = DType("float32", "DT_FLOAT", np.float32)
float64 = DType("float64", "DT_DOUBLE", np.float64)
float16 = DType("float16", "DT_HALF", np.float16)
int32 = DType("int32", "DT_INT32", np.int32)
int64 = DType("int64", "DT_INT64", np.int64)
uint8 = DType("uint8", "DT_UINT8", np.uint8)
bool_ = DType("bool", "DT_BOOL", np.bool_)
_ALL = [float32, float64, float16, int32, int64, uint8, bool_]
_BY_NAME = {d.name: d for d in _ALL}
_BY_NAME.update({"float": float32, "double": float64, "half": float16, "int": int32})
_BY_ENUM = {d.enum: d for d in _ALL}


def as_dtype(x) -> DType:
    if isinstance(x, DType):
        return x
    if isinstance(x, str):
        if x in _BY_NAME:
            return _BY_NAME[x]
        if x in _BY_ENUM:
            return _BY_ENUM[x]
    try:
        npd = np.dtype(x)
        for d in _ALL:
            if d.np == npd:
                return d
    except TypeError:
        pass
    raise TypeError(f"cannot convert {x!r} to a dtype")


# ---------------------------------------------------------------------------
# attr helpers (proto3-JSON shaped)
# ---------------------------------------------------------------------------
def attr_type(dt) -> Dict[str, Any]:
    return {"type": as_dtype(dt).enum}


def attr_shape(shape: Optional[Sequence[Optional[int]]]) -> Dict[str, Any]:
    if shape is None:
        return {"shape": {"unknownRank": True}}
    return {"shape": {"dim": [{"size": str(-1 if d is None else int(d))} for d in shape]}} if len(shape) else {"shape": {}}


def attr_s(s: Union[str, bytes]) -> Dict[str, Any]:
    raw = s.encode() if isinstance(s, str) else s
    return {"s": base64.b64encode(raw).decode("ascii")}


def attr_i(i: int) -> Dict[str, Any]:
    return {"i": str(int(i))}


def attr_f(f: float) -> Dict[str, Any]:
    return {"f": float(f)}


def attr_b(b: bool) -> Dict[str, Any]:
    return {"b": bool(b)}


def attr_ilist(v: Sequence[int]) -> Dict[str, Any]:
    return {"list": {"i": [str(int(x)) for x in v]}}


def attr_class(var_name: str) -> Dict[str, Any]:
    return {"list": {"s": [base64.b64encode(f"loc:@{var_name}".encode()).decode("ascii")]}}


def attr_tensor(value: np.ndarray, dt: DType) -> Dict[str, Any]:
    arr = np.asarray(value, dtype=dt.np)
    t: Dict[str, Any] = {"dtype": dt.enum, "tensorShape": ({"dim": [{"size": str(d)} for d in arr.shape]} if arr.ndim else {})}
    if arr.size == 1 and dt.enum in ("DT_FLOAT", "DT_INT32", "DT_INT64", "DT_DOUBLE", "DT_BOOL"):
        key = {"DT_FLOAT": "floatVal", "DT_DOUBLE": "doubleVal", "DT_INT32": "intVal", "DT_INT64": "int64Val",
               "DT_BOOL": "boolVal"}[dt.enum]
        v = arr.reshape(-1)[0].item()
        t[key] = [str(v) if key == "int64Val" else v]
    else:
        t["tensorContent"] = base64.b64encode(arr.astype(dt.np.newbyteorder("<")).tobytes()).decode("ascii")
    return {"tensor": t}


# ---------------------------------------------------------------------------
# Graph
# ---------------------------------------------------------------------------
class GraphKeys:
    GLOBAL_VARIABLES = "variables"
    TRAINABLE_VARIABLES = "trainable_variables"
    LOSSES = "losses"
    TRAIN_OP = "train_op"
    UPDATE_OPS = "update_ops"
    REGULARIZATION_LOSSES = "regularization_losses"


class Operation:
    def __init__(self, graph: "Graph", node: Dict[str, Any], outputs: List["Tensor"]):
        self.graph, self.node_def, self.outputs = graph, node, outputs

    @property
    def name(self) -> str:
        return self.node_def["name"]

    @property
    def type(self) -> str:
        return self.node_def["op"]

    def run(self, feed_dict=None, session=None):
        from .session import get_default_session

        (session or get_default_session()).run(self, feed_dict=feed_dict)


class Tensor:
    """Symbolic handle on ``<node>:<index>`` with static dtype / shape."""

    def __init__(self, graph: "Graph", node_name: str, index: int, dtype: DType, shape: Optional[Tuple[Optional[int], ...]]):
        self.graph, self._node, self._index, self.dtype = graph, node_name, index, dtype
        self._shape = None if shape is None else tuple(None if d is None or (isinstance(d, int) and d < 0) else int(d) for d in shape)
        self.op: Optional[Operation] = None

    @property
    def name(self) -> str:
        return f"{self._node}:{self._index}"

    @property
    def ref(self) -> str:
        """How a consumer NodeDef references this tensor."""
        return self._node if self._index == 0 else f"{self._node}:{self._index}"

    @property
    def shape(self):
        return TensorShape(self._shape)

    def get_shape(self):
        return self.shape

    def __repr__(self):
        return f"<tf.Tensor '{self.name}' shape={self._shape} dtype={self.dtype.name}>"

    def eval(self, feed_dict=None, session=None):
        from .session import get_default_session

        return (session or get_default_session()).run(self, feed_dict=feed_dict)

    # arithmetic sugar -> graph ops
    def _bin(self, other, op, reverse=False):
        from . import ops

        a, b = (other, self) if reverse else (self, other)
        return ops.binary(op, a, b)

    def __add__(self, o): return self._bin(o, "Add")
    def __radd__(self, o): return self._bin(o, "Add", True)
    def __sub__(self, o): return self._bin(o, "Sub")
    def __rsub__(self, o): return self._bin(o, "Sub", True)
    def __mul__(self, o): return self._bin(o, "Mul")
    def __rmul__(self, o): return self._bin(o, "Mul", True)
    def __truediv__(self, o): return self._bin(o, "RealDiv")
    def __rtruediv__(self, o): return self._bin(o, "RealDiv", True)
    def __neg__(self):
        from . import ops

        return ops.unary("Neg", self)
    def __matmul__(self, o):
        from . import ops

        return ops.matmul(self, o)

    def __getitem__(self, key):
        from . import ops

        return ops.strided_slice_from_key(self, key)

    def __pow__(self, o): return self._bin(o, "Pow")
    def __gt__(self, o):
        from . import ops

        return ops.greater(self, o)

    def __ge__(self, o):
        from . import ops

        return ops.greater_equal(self, o)

    def __lt__(self, o):
        from . import ops

        return ops.less(self, o)

    def __le__(self, o):
        from . import ops

        return ops.less_equal(self, o)
    __hash__ = object.__hash__


class TensorShape:
    def __init__(self, dims):
        self._dims = dims

    @property
    def dims(self):
        return None if self._dims is None else list(self._dims)

    @property
    def ndims(self):
        return None if self._dims is None else len(self._dims)

    def as_list(self):
        if self._dims is None:
            raise ValueError("as_list() is not defined on an unknown TensorShape.")
        return list(self._dims)

    def __getitem__(self, i):
        return self._dims[i]

    def __len__(self):
        return len(self._dims)

    def __iter__(self):
        return iter(self._dims)

    def __repr__(self):
        return f"TensorShape({self._dims})"


class Variable:
    def __init__(self, graph: "Graph", name: str, dtype: DType, shape: Tuple[int, ...], handle: Tensor, read: Tensor,
                 initial_value: Tensor, initializer: Operation, trainable: bool):
        self.graph, self._name, self.dtype, self._shape = graph, name, dtype, tuple(shape)
        self._handle, self._read, self.initial_value, self.initializer, self.trainable = handle, read, initial_value, initializer, trainable

    @property
    def name(self) -> str:
        return f"{self._name}:0"

    @property
    def op(self):
        return self._handle.op

    @property
    def shape(self):
        return TensorShape(self._shape)

    def get_shape(self):
        return self.shape

    def value(self) -> Tensor:
        return self._read

    def read_value(self) -> Tensor:
        return self._read

    def to_proto(self) -> Dict[str, Any]:
        return {"variableName": self.name, "initializerName": self.initializer.name, "snapshotName": self._read.name,
                "initialValueName": self.initial_value.name}

    def eval(self, session=None):
        return self._read.eval(session=session)

    def __repr__(self):
        return f"<tf.Variable '{self.name}' shape={self._shape} dtype={self.dtype.name}>"


class Graph:
    def __init__(self):
        self.nodes: List[Dict[str, Any]] = []
        self._node_index: Dict[str, Dict[str, Any]] = {}
        self._tensors: Dict[str, Tensor] = {}
        self._ops: Dict[str, Operation] = {}
        self._names_in_use: Dict[str, int] = {}
        self._scope: List[str] = []
        self.collections: Dict[str, List[Any]] = {}
        self.variables: List[Variable] = []
        self.saver_def: Optional[Dict[str, Any]] = None
        self.seed: Optional[int] = None

    # -- default-graph stack ---------------------------------------------------------------
    @contextlib.contextmanager
    def as_default(self):
        _STATE.stack.append(self)
        try:
            yield self
        finally:
            _STATE.stack.pop()

    # -- naming ------------------------------------------------------------------------------
    def unique_name(self, name: str, mark_as_used: bool = True) -> str:
        base = "/".join(self._scope + [name]) if self._scope else name
        cnt = self._names_in_use.get(base.lower())
        if cnt is None:
            if mark_as_used:
                self._names_in_use[base.lower()] = 1
            return base
        cand = base
        while cand.lower() in self._names_in_use:
            cand = f"{base}_{cnt}"
            cnt += 1
        if mark_as_used:
            self._names_in_use[base.lower()] = cnt
            self._names_in_use[cand.lower()] = 1
        return cand

    @contextlib.contextmanager
    def name_scope(self, name: Optional[str]):
        if not name:
            yield ""
            return
        if name.endswith("/"):                      # re-enter an existing scope verbatim
            old = self._scope
            self._scope = name[:-1].split("/")
            try:
                yield name
            finally:
                self._scope = old
            return
        scoped = self.unique_name(name)
        old = self._scope
        self._scope = scoped.split("/")
        try:
            yield scoped + "/"
        finally:
            self._scope = old

    # -- node creation -----------------------------------------------------------------------
    def add_node(self, op: str, name: str, inputs: Sequence[Union[Tensor, str]] = (), attrs: Optional[Dict[str, Any]] = None,
                 out_dtypes: Sequence[DType] = (), out_shapes: Sequence[Optional[Tuple]] = (), exact_name: bool = False,
                 control_inputs: Sequence[str] = ()) -> Operation:
        full = name if exact_name else self.unique_name(name)
        if exact_name:
            self._names_in_use.setdefault(full.lower(), 1)
        node: Dict[str, Any] = {"name": full, "op": op}
        refs = [t.ref if isinstance(t, Tensor) else str(t) for t in inputs] + [f"^{c}" for c in control_inputs]
        if refs:
            node["input"] = refs
        if attrs:
            node["attr"] = attrs
        self.nodes.append(node)
        self._node_index[full] = node
        outs = []
        for i, dt in enumerate(out_dtypes):
            t = Tensor(self, full, i, dt, out_shapes[i] if i < len(out_shapes) else None)
            outs.append(t)
            self._tensors[t.name] = t
        operation = Operation(self, node, outs)
        for t in outs:
            t.op = operation
        self._ops[full] = operation
        return operation

    # -- lookup ------------------------------------------------------------------------------
    def get_tensor_by_name(self, name: str) -> Tensor:
        if name not in self._tensors:
            raise KeyError(f"The name '{name}' refers to a Tensor which does not exist in this graph.")
        return self._tensors[name]

    def get_operation_by_name(self, name: str) -> Operation:
        return self._ops[name]

    def get_operations(self) -> List[Operation]:
        return list(self._ops.values())

    def as_graph_element(self, obj):
        if isinstance(obj, (Tensor, Operation)):
            return obj
        if isinstance(obj, Variable):
            return obj.value()
        if isinstance(obj, str):
            return self._tensors[obj] if ":" in obj else self._ops[obj]
        raise TypeError(f"cannot convert {obj!r} to a graph element")

    # -- collections ---------------------------------------------------------------------------
    def add_to_collection(self, name: str, value: Any) -> None:
        self.collections.setdefault(name, []).append(value)

    def get_collection(self, name: str, scope: Optional[str] = None) -> List[Any]:
        vals = list(self.collections.get(name, []))
        if scope:
            vals = [v for v in vals if getattr(v, "name", "").startswith(scope)]
        return vals

    def get_collection_ref(self, name: str) -> List[Any]:
        return self.collections.setdefault(name, [])

    # -- export ----------------------------------------------------------------------------------
    def stripped_ops(self) -> List[str]:
        return sorted({n["op"] for n in self.nodes})

    def as_graph_def(self) -> Dict[str, Any]:
        return {"node": [dict(n) for n in self.nodes], "versions": {"producer": 26}}


class _State(threading.local):
    def __init__(self):
        self.stack: List[Graph] = [Graph()]


_STATE = _State()


def get_default_graph() -> Graph:
    return _STATE.stack[-1]


def reset_default_graph() -> None:
    if len(_STATE.stack) > 1:
        raise AssertionError("Do not use tf.reset_default_graph() to clear nested graphs.")
    _STATE.stack[0] = Graph()


def convert_to_tensor(value, dtype=None, name: str = "Const") -> Tensor:
    from . import ops

    if isinstance(value, Tensor):
        return value
    if isinstance(value, Variable):
        return value.value()
    return ops.constant(value, dtype=dtype, name=name)


# ---------------------------------------------------------------------------
# MetaGraphDef wrapper
# ---------------------------------------------------------------------------
class MetaGraphDef:
    """In-memory MetaGraphDef: a proto3-JSON shaped dict with the usual protobuf-ish methods."""

    def __init__(self, data: Optional[Dict[str, Any]] = None):
        self.data: Dict[str, Any] = data if data is not None else {}

    def to_json(self, indent: Optional[int] = 2) -> str:
        import json

        return json.dumps(self.data, indent=indent)

    def SerializeToString(self) -> bytes:
        return pbwire.encode("MetaGraphDef", self.data)

    @classmethod
    def FromString(cls, raw: bytes) -> "MetaGraphDef":
        return cls(pbwire.decode("MetaGraphDef", raw))

    def ParseFromString(self, raw: bytes) -> None:
        self.data = pbwire.decode("MetaGraphDef", raw)

    @property
    def graph_def(self) -> Dict[str, Any]:
        return self.data.get("graphDef", {})

    @property
    def collection_def(self) -> Dict[str, Any]:
        return self.data.get("collectionDef", {})


def export_meta_graph(filename: Optional[str] = None, graph: Optional[Graph] = None, as_text: bool = False,
                      collection_list: Optional[Sequence[str]] = None, **_unused) -> MetaGraphDef:
    g = graph or get_default_graph()
    coll: Dict[str, Any] = {}
    for key, vals in g.collections.items():
        if collection_list is not None and key not in collection_list:
            continue
        if not vals:
            continue
        if all(isinstance(v, Variable) for v in vals):
            coll[key] = {"bytesList": {"value": [base64.b64encode(pbwire.encode("VariableDef", v.to_proto())).decode("ascii")
                                                 for v in vals]}}
        else:
            coll[key] = {"nodeList": {"value": [v.name if hasattr(v, "name") else str(v) for v in vals]}}
    data: Dict[str, Any] = {
        "metaInfoDef": {
            "strippedOpList": {"op": [{"name": o} for o in g.stripped_ops()]},
            "tensorflowVersion": "1.10.0",
            "tensorflowGitVersion": "sparkflow_b200-tfcompat",
        },
        "graphDef": g.as_graph_def(),
        "collectionDef": coll,
    }
    if g.saver_def:
        data["saverDef"] = g.saver_def
    mg = MetaGraphDef(data)
    if filename:
        with open(filename, "w" if as_text else "wb") as fh:
            fh.write(mg.to_json() if as_text else mg.SerializeToString())
    return mg
