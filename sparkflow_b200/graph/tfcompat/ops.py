"""Graph-building ops of the TF-1.x compatible builder: constants, variables + initializers, math,
``tf.nn`` / ``tf.layers`` / ``tf.losses``.  Node/attr layouts mirror what TF-1.x emits for the same
calls (cf. the nodes decoded from lifeomic/sparkflow/tests/test_model/to_load.meta: ``dense/kernel``,
``dense/kernel/Initializer/random_uniform/{shape,min,max,RandomUniform,sub,mul}``, ``dense/kernel/
Assign``, ``dense/kernel/read``, ``dense/MatMul``, ``dense/BiasAdd``, ``dense/Tanh`` ...).
"""
from __future__ import annotations

import math
from typing import Any, Callable, Optional, Sequence, Tuple, Union

import numpy as np

from . import core
from .core import (DType, GraphKeys, Tensor, Variable, as_dtype, attr_b, attr_class, attr_f, attr_i, attr_ilist,
                   attr_s, attr_shape, attr_tensor, attr_type, convert_to_tensor, get_default_graph)

TensorLike = Union[Tensor, Variable, float, int, np.ndarray, list, tuple]


def _g():
    return get_default_graph()


def _static(shape) -> Optional[Tuple]:
    return None if shape is None else tuple(shape)


def _bshape(a, b):
    """Static broadcast of two shapes (None = unknown dim)."""
    if a is None or b is None:
        return None
    n = max(len(a), len(b))
    a = (1,) * (n - len(a)) + tuple(a)
    b = (1,) * (n - len(b)) + tuple(b)
    out = []
    for x, y in zip(a, b):
        if x == 1:
            out.append(y)
        elif y == 1 or y is None:
            out.append(x)
        else:
            out.append(y if x is None else x)
    return tuple(out)


# ---------------------------------------------------------------------------
# constants / placeholders
# ---------------------------------------------------------------------------
def constant(value, dtype=None, shape=None, name: str = "Const") -> Tensor:
    if dtype is None:
        arr = np.asarray(value)
        if arr.dtype == np.float64:
            arr = arr.astype(np.float32)
        elif arr.dtype == np.int64:
            arr = arr.astype(np.int32)
        dt = as_dtype(arr.dtype)
    else:
        dt = as_dtype(dtype)
        arr = np.asarray(value, dtype=dt.np)
    if shape is not None:
        arr = np.broadcast_to(arr, tuple(shape)).copy() if arr.size == 1 else arr.reshape(tuple(shape))
    op = _g().add_node("Const", name, attrs={"dtype": attr_type(dt), "value": attr_tensor(arr, dt)},
                       out_dtypes=[dt], out_shapes=[arr.shape])
    return op.outputs[0]


def placeholder(dtype, shape=None, name: Optional[str] = None) -> Tensor:
    dt = as_dtype(dtype)
    op = _g().add_node("Placeholder", name or "Placeholder", attrs={"dtype": attr_type(dt), "shape": attr_shape(shape)},
                       out_dtypes=[dt], out_shapes=[_static(shape)])
    return op.outputs[0]


def placeholder_with_default(input, shape=None, name: Optional[str] = None) -> Tensor:  # noqa: A002
    x = convert_to_tensor(input)
    op = _g().add_node("PlaceholderWithDefault", name or "PlaceholderWithDefault", [x],
                       {"dtype": attr_type(x.dtype), "shape": attr_shape(shape if shape is not None else x._shape)},
                       out_dtypes=[x.dtype], out_shapes=[_static(shape) if shape is not None else x._shape])
    return op.outputs[0]


# ---------------------------------------------------------------------------
# elementwise / math
# ---------------------------------------------------------------------------
def unary(op: str, x: TensorLike, name: Optional[str] = None) -> Tensor:
    x = convert_to_tensor(x)
    return _g().add_node(op, name or op, [x], {"T": attr_type(x.dtype)}, [x.dtype], [x._shape]).outputs[0]


def binary(op: str, a: TensorLike, b: TensorLike, name: Optional[str] = None) -> Tensor:
    if isinstance(a, (Tensor, Variable)):
        a = convert_to_tensor(a)
        b = convert_to_tensor(b, dtype=a.dtype, name=(name or op.lower()) + "/y")
    else:
        b = convert_to_tensor(b)
        a = convert_to_tensor(a, dtype=b.dtype, name=(name or op.lower()) + "/x")
    default = {"Add": "add", "Sub": "sub", "Mul": "mul", "RealDiv": "truediv"}.get(op, op)
    return _g().add_node(op, name or default, [a, b], {"T": attr_type(a.dtype)}, [a.dtype], [_bshape(a._shape, b._shape)]).outputs[0]


def add(a, b, name=None): return binary("Add", a, b, name)
def subtract(a, b, name=None): return binary("Sub", a, b, name)
def multiply(a, b, name=None): return binary("Mul", a, b, name)
def divide(a, b, name=None): return binary("RealDiv", a, b, name)
def maximum(a, b, name=None): return binary("Maximum", a, b, name)
def minimum(a, b, name=None): return binary("Minimum", a, b, name)
def squared_difference(a, b, name=None): return binary("SquaredDifference", a, b, name)
def pow(a, b, name=None): return binary("Pow", a, b, name)  # noqa: A001
def square(x, name=None): return unary("Square", x, name)
def sqrt(x, name=None): return unary("Sqrt", x, name)
def exp(x, name=None): return unary("Exp", x, name)
def log(x, name=None): return unary("Log", x, name)
def negative(x, name=None): return unary("Neg", x, name)
def abs(x, name=None): return unary("Abs", x, name)  # noqa: A001
def identity(x, name=None): return unary("Identity", x, name)
def stop_gradient(x, name=None): return unary("StopGradient", x, name)
def relu(x, name=None): return unary("Relu", x, name)
def sigmoid(x, name=None): return unary("Sigmoid", x, name)
def tanh(x, name=None): return unary("Tanh", x, name)
def softplus(x, name=None): return unary("Softplus", x, name)
def elu(x, name=None): return unary("Elu", x, name)


def leaky_relu(x, alpha=0.2, name=None):
    x = convert_to_tensor(x)
    return _g().add_node("LeakyRelu", name or "LeakyRelu", [x], {"T": attr_type(x.dtype), "alpha": attr_f(alpha)},
                         [x.dtype], [x._shape]).outputs[0]


def softmax(x, axis=-1, name=None):
    return unary("Softmax", x, name)


def cast(x, dtype, name=None) -> Tensor:
    x = convert_to_tensor(x)
    dt = as_dtype(dtype)
    return _g().add_node("Cast", name or "Cast", [x], {"SrcT": attr_type(x.dtype), "DstT": attr_type(dt)}, [dt], [x._shape]).outputs[0]


def matmul(a, b, transpose_a=False, transpose_b=False, name=None) -> Tensor:
    a, b = convert_to_tensor(a), convert_to_tensor(b)
    sa, sb = a._shape, b._shape
    m = None if sa is None else (sa[1] if transpose_a else sa[0])
    n = None if sb is None else (sb[0] if transpose_b else sb[1])
    return _g().add_node("MatMul", name or "MatMul", [a, b],
                         {"T": attr_type(a.dtype), "transpose_a": attr_b(transpose_a), "transpose_b": attr_b(transpose_b)},
                         [a.dtype], [(m, n)]).outputs[0]


def _reduce(op: str, x, axis, keepdims, name) -> Tensor:
    x = convert_to_tensor(x)
    scope = name or op
    with _g().name_scope(None):
        pass
    rank = None if x._shape is None else len(x._shape)
    if axis is None:
        axes = list(range(rank)) if rank is not None else [0]
    else:
        axes = [axis] if isinstance(axis, int) else list(axis)
    idx = constant(np.asarray(axes, dtype=np.int32), dtype=core.int32, name="Const")
    if x._shape is None:
        oshape = None
    else:
        norm = [a % rank for a in axes]
        oshape = tuple((1 if i in norm else d) for i, d in enumerate(x._shape) if keepdims or i not in norm)
    return _g().add_node(op, scope, [x, idx], {"T": attr_type(x.dtype), "Tidx": attr_type(core.int32), "keep_dims": attr_b(keepdims)},
                         [x.dtype], [oshape]).outputs[0]


def reduce_sum(x, axis=None, keepdims=False, name=None, keep_dims=None, reduction_indices=None):
    return _reduce("Sum", x, reduction_indices if axis is None else axis, bool(keep_dims if keep_dims is not None else keepdims), name)


def reduce_mean(x, axis=None, keepdims=False, name=None, keep_dims=None, reduction_indices=None):
    return _reduce("Mean", x, reduction_indices if axis is None else axis, bool(keep_dims if keep_dims is not None else keepdims), name)


def reduce_max(x, axis=None, keepdims=False, name=None, keep_dims=None, reduction_indices=None):
    return _reduce("Max", x, reduction_indices if axis is None else axis, bool(keep_dims if keep_dims is not None else keepdims), name)


def argmax(input, axis=None, name=None, dimension=None, output_type=core.int64) -> Tensor:  # noqa: A002
    x = convert_to_tensor(input)
    ax = dimension if axis is None else axis
    ax = 0 if ax is None else ax
    g = _g()
    node_name = g.unique_name(name or "ArgMax")
    dim = g.add_node("Const", node_name + "/dimension", attrs={"dtype": attr_type(core.int32), "value": attr_tensor(np.asarray(ax, np.int32), core.int32)},
                     out_dtypes=[core.int32], out_shapes=[()], exact_name=True).outputs[0]
    oshape = None if x._shape is None else tuple(d for i, d in enumerate(x._shape) if i != ax % len(x._shape))
    ot = as_dtype(output_type)
    return g.add_node("ArgMax", node_name, [x, dim], {"T": attr_type(x.dtype), "Tidx": attr_type(core.int32), "output_type": attr_type(ot)},
                      [ot], [oshape], exact_name=True).outputs[0]


def reshape(tensor, shape, name=None) -> Tensor:
    x = convert_to_tensor(tensor)
    g = _g()
    node_name = g.unique_name(name or "Reshape")
    if isinstance(shape, (Tensor, Variable)):
        sh = convert_to_tensor(shape)
        oshape = None
    else:
        lst = [int(s) for s in shape]
        sh = g.add_node("Const", node_name + "/shape", attrs={"dtype": attr_type(core.int32), "value": attr_tensor(np.asarray(lst, np.int32), core.int32)},
                        out_dtypes=[core.int32], out_shapes=[(len(lst),)], exact_name=True).outputs[0]
        oshape = list(None if s < 0 else s for s in lst)
        if x._shape is not None and all(d is not None for d in x._shape) and oshape.count(None) == 1:
            known = int(np.prod([d for d in oshape if d is not None])) or 1
            oshape[oshape.index(None)] = int(np.prod(x._shape)) // known
        oshape = tuple(oshape)
    return g.add_node("Reshape", node_name, [x, sh], {"T": attr_type(x.dtype), "Tshape": attr_type(core.int32)}, [x.dtype], [oshape],
                      exact_name=True).outputs[0]


def shape(input, name=None, out_type=core.int32) -> Tensor:  # noqa: A002
    x = convert_to_tensor(input)
    rank = None if x._shape is None else len(x._shape)
    return _g().add_node("Shape", name or "Shape", [x], {"T": attr_type(x.dtype), "out_type": attr_type(out_type)},
                         [as_dtype(out_type)], [(rank,)]).outputs[0]


def size(input, name=None, out_type=core.int32) -> Tensor:  # noqa: A002
    x = convert_to_tensor(input)
    return _g().add_node("Size", name or "Size", [x], {"T": attr_type(x.dtype), "out_type": attr_type(out_type)},
                         [as_dtype(out_type)], [()]).outputs[0]


def transpose(a, perm=None, name=None) -> Tensor:
    x = convert_to_tensor(a)
    rank = len(x._shape)
    perm = list(range(rank))[::-1] if perm is None else list(perm)
    p = constant(np.asarray(perm, np.int32), dtype=core.int32, name="perm")
    oshape = tuple(x._shape[i] for i in perm)
    return _g().add_node("Transpose", name or "transpose", [x, p], {"T": attr_type(x.dtype), "Tperm": attr_type(core.int32)},
                         [x.dtype], [oshape]).outputs[0]


def expand_dims(input, axis, name=None) -> Tensor:  # noqa: A002
    x = convert_to_tensor(input)
    d = constant(np.asarray(axis, np.int32), dtype=core.int32, name="dim")
    sh = None
    if x._shape is not None:
        lst = list(x._shape)
        lst.insert(axis if axis >= 0 else len(lst) + axis + 1, 1)
        sh = tuple(lst)
    return _g().add_node("ExpandDims", name or "ExpandDims", [x, d], {"T": attr_type(x.dtype), "Tdim": attr_type(core.int32)},
                         [x.dtype], [sh]).outputs[0]


def squeeze(input, axis=None, name=None) -> Tensor:  # noqa: A002
    x = convert_to_tensor(input)
    axes = [] if axis is None else ([axis] if isinstance(axis, int) else list(axis))
    sh = None
    if x._shape is not None:
        r = len(x._shape)
        norm = [a % r for a in axes]
        sh = tuple(d for i, d in enumerate(x._shape) if not ((i in norm) if axes else d == 1))
    return _g().add_node("Squeeze", name or "Squeeze", [x], {"T": attr_type(x.dtype), "squeeze_dims": attr_ilist(axes)},
                         [x.dtype], [sh]).outputs[0]


def concat(values, axis, name="concat") -> Tensor:
    vals = [convert_to_tensor(v) for v in values]
    ax = constant(np.asarray(axis, np.int32), dtype=core.int32, name="axis")
    sh = None
    if all(v._shape is not None for v in vals):
        lst = list(vals[0]._shape)
        a = axis % len(lst)
        lst[a] = None if any(v._shape[a] is None for v in vals) else sum(v._shape[a] for v in vals)
        sh = tuple(lst)
    return _g().add_node("ConcatV2", name, [*vals, ax], {"T": attr_type(vals[0].dtype), "N": attr_i(len(vals)), "Tidx": attr_type(core.int32)},
                         [vals[0].dtype], [sh]).outputs[0]


# ---------------------------------------------------------------------------
# initializers
# ---------------------------------------------------------------------------
class Initializer:
    def build(self, scope: str, shape: Tuple[int, ...], dtype: DType, var_name: str) -> Tensor:  # pragma: no cover
        raise NotImplementedError

    def __call__(self, shape, dtype=core.float32, partition_info=None):
        return self.build("Initializer", tuple(shape), as_dtype(dtype), "")


def _fans(shape: Tuple[int, ...]) -> Tuple[float, float]:
    if len(shape) < 1:
        return 1.0, 1.0
    if len(shape) == 1:
        return float(shape[0]), float(shape[0])
    if len(shape) == 2:
        return float(shape[0]), float(shape[1])
    rf = float(np.prod(shape[:-2]))
    return shape[-2] * rf, shape[-1] * rf


def _cls(var_name):
    return {"_class": attr_class(var_name)} if var_name else {}


class _Zeros(Initializer):
    value = 0.0
    tag = "zeros"

    def build(self, scope, shape, dtype, var_name):
        g = _g()
        arr = np.full(shape, self.value, dtype=dtype.np)
        # a Const with one value and a full tensorShape is TF's "splat" encoding
        t = {"dtype": dtype.enum, "tensorShape": {"dim": [{"size": str(d)} for d in shape]},
             ("floatVal" if dtype.enum == "DT_FLOAT" else "doubleVal" if dtype.enum == "DT_DOUBLE" else "intVal"): [self.value if dtype.np.kind == "f" else int(self.value)]}
        del arr
        return g.add_node("Const", f"{scope}/{self.tag}", attrs={"dtype": attr_type(dtype), "value": {"tensor": t}, **_cls(var_name)},
                          out_dtypes=[dtype], out_shapes=[shape], exact_name=True).outputs[0]


class _Ones(_Zeros):
    value = 1.0
    tag = "ones"


class _Constant(Initializer):
    def __init__(self, value=0.0):
        self.value = value

    def build(self, scope, shape, dtype, var_name):
        arr = np.broadcast_to(np.asarray(self.value, dtype=dtype.np), shape).copy()
        return _g().add_node("Const", f"{scope}/Const", attrs={"dtype": attr_type(dtype), "value": attr_tensor(arr, dtype), **_cls(var_name)},
                             out_dtypes=[dtype], out_shapes=[shape], exact_name=True).outputs[0]


class _RandomUniform(Initializer):
    def __init__(self, minval=-0.05, maxval=0.05, seed=None):
        self.minval, self.maxval, self.seed = minval, maxval, seed

    def limits(self, shape):
        return self.minval, self.maxval

    def build(self, scope, shape, dtype, var_name):
        g = _g()
        lo, hi = self.limits(shape)
        base = f"{scope}/random_uniform"
        c = _cls(var_name)

        def const(name, val, dt):
            return g.add_node("Const", name, attrs={"dtype": attr_type(dt), "value": attr_tensor(np.asarray(val, dt.np), dt), **c},
                              out_dtypes=[dt], out_shapes=[np.asarray(val).shape], exact_name=True).outputs[0]

        sh = const(base + "/shape", list(shape), core.int32)
        mn = const(base + "/min", lo, dtype)
        mx = const(base + "/max", hi, dtype)
        ru = g.add_node("RandomUniform", base + "/RandomUniform", [sh],
                        {"T": attr_type(core.int32), "dtype": attr_type(dtype), "seed": attr_i(self.seed or 0), "seed2": attr_i(0), **c},
                        [dtype], [shape], exact_name=True).outputs[0]
        sub = g.add_node("Sub", base + "/sub", [mx, mn], {"T": attr_type(dtype), **c}, [dtype], [()], exact_name=True).outputs[0]
        mul = g.add_node("Mul", base + "/mul", [ru, sub], {"T": attr_type(dtype), **c}, [dtype], [shape], exact_name=True).outputs[0]
        return g.add_node("Add", base, [mul, mn], {"T": attr_type(dtype), **c}, [dtype], [shape], exact_name=True).outputs[0]


class _GlorotUniform(_RandomUniform):
    def __init__(self, seed=None, dtype=core.float32):
        super().__init__(seed=seed)

    def limits(self, shape):
        fi, fo = _fans(shape)
        lim = math.sqrt(6.0 / (fi + fo))
        return -lim, lim


class _RandomNormal(Initializer):
    op = "RandomStandardNormal"
    tag = "random_normal"

    def __init__(self, mean=0.0, stddev=1.0, seed=None):
        self.mean, self.stddev, self.seed = mean, stddev, seed

    def std(self, shape):
        return self.stddev

    def build(self, scope, shape, dtype, var_name):
        g = _g()
        base = f"{scope}/{self.tag}"
        c = _cls(var_name)

        def const(name, val, dt):
            return g.add_node("Const", name, attrs={"dtype": attr_type(dt), "value": attr_tensor(np.asarray(val, dt.np), dt), **c},
                              out_dtypes=[dt], out_shapes=[np.asarray(val).shape], exact_name=True).outputs[0]

        sh = const(base + "/shape", list(shape), core.int32)
        mean = const(base + "/mean", self.mean, dtype)
        std = const(base + "/stddev", self.std(shape), dtype)
        rn = g.add_node(self.op, base + "/" + self.op, [sh], {"T": attr_type(core.int32), "dtype": attr_type(dtype), "seed": attr_i(self.seed or 0), "seed2": attr_i(0), **c},
                        [dtype], [shape], exact_name=True).outputs[0]
        mul = g.add_node("Mul", base + "/mul", [rn, std], {"T": attr_type(dtype), **c}, [dtype], [shape], exact_name=True).outputs[0]
        return g.add_node("Add", base, [mul, mean], {"T": attr_type(dtype), **c}, [dtype], [shape], exact_name=True).outputs[0]


class _TruncatedNormal(_RandomNormal):
    op = "TruncatedNormal"
    tag = "truncated_normal"


class _GlorotNormal(_TruncatedNormal):
    def __init__(self, seed=None, dtype=core.float32):
        super().__init__(seed=seed)

    def std(self, shape):
        fi, fo = _fans(shape)
        return math.sqrt(2.0 / (fi + fo)) / 0.87962566103423978


def zeros_initializer(dtype=core.float32): return _Zeros()
def ones_initializer(dtype=core.float32): return _Ones()
def constant_initializer(value=0.0, dtype=core.float32): return _Constant(value)
def random_uniform_initializer(minval=0.0, maxval=None, seed=None, dtype=core.float32): return _RandomUniform(minval, 1.0 if maxval is None else maxval, seed)
def random_normal_initializer(mean=0.0, stddev=1.0, seed=None, dtype=core.float32): return _RandomNormal(mean, stddev, seed)
def truncated_normal_initializer(mean=0.0, stddev=1.0, seed=None, dtype=core.float32): return _TruncatedNormal(mean, stddev, seed)
def glorot_uniform_initializer(seed=None, dtype=core.float32): return _GlorotUniform(seed)
def glorot_normal_initializer(seed=None, dtype=core.float32): return _GlorotNormal(seed)


# ---------------------------------------------------------------------------
# variables
# ---------------------------------------------------------------------------
def _make_variable(full_name: str, shape: Tuple[int, ...], dtype: DType, initializer: Union[Initializer, Tensor, np.ndarray, float, Callable],
                   trainable: bool) -> Variable:
    g = _g()
    shape = tuple(int(s) for s in shape)
    if isinstance(initializer, Initializer):
        init_val = initializer.build(f"{full_name}/Initializer", shape, dtype, full_name)
    elif isinstance(initializer, Tensor):
        init_val = initializer
    elif callable(initializer):
        init_val = convert_to_tensor(initializer(shape, dtype))
    else:
        init_val = _Constant(initializer).build(f"{full_name}/Initializer", shape, dtype, full_name)
    c = {"_class": attr_class(full_name)}
    handle = g.add_node("VariableV2", full_name, attrs={"dtype": attr_type(dtype), "shape": attr_shape(shape), "container": attr_s(""),
                                                        "shared_name": attr_s(""), **c},
                        out_dtypes=[dtype], out_shapes=[shape], exact_name=True).outputs[0]
    assign = g.add_node("Assign", f"{full_name}/Assign", [handle, init_val],
                        {"T": attr_type(dtype), "use_locking": attr_b(True), "validate_shape": attr_b(True), **c}, [dtype], [shape], exact_name=True)
    read = g.add_node("Identity", f"{full_name}/read", [handle], {"T": attr_type(dtype), **c}, [dtype], [shape], exact_name=True).outputs[0]
    var = Variable(g, full_name, dtype, shape, handle, read, init_val, assign, trainable)
    g.variables.append(var)
    g.add_to_collection(GraphKeys.GLOBAL_VARIABLES, var)
    if trainable:
        g.add_to_collection(GraphKeys.TRAINABLE_VARIABLES, var)
    return var


def get_variable(name, shape=None, dtype=core.float32, initializer=None, trainable=True, **_unused) -> Variable:
    g = _g()
    full = g.unique_name(name)
    dt = as_dtype(dtype)
    if initializer is None:
        initializer = _GlorotUniform()
    if shape is None:
        arr = np.asarray(initializer)
        shape = arr.shape
    return _make_variable(full, tuple(shape), dt, initializer, trainable)


def variable(initial_value, trainable=True, name=None, dtype=None, **_unused) -> Variable:
    g = _g()
    full = g.unique_name(name or "Variable")
    if isinstance(initial_value, Tensor):
        dt = initial_value.dtype
        shape = initial_value._shape
        return _make_variable(full, shape, dt, initial_value, trainable)
    arr = np.asarray(initial_value)
    if dtype is not None:
        arr = arr.astype(as_dtype(dtype).np)
    elif arr.dtype == np.float64:
        arr = arr.astype(np.float32)
    elif arr.dtype == np.int64:
        arr = arr.astype(np.int32)
    with g.name_scope(full + "/"):
        init = constant(arr, name="initial_value")
    return _make_variable(full, arr.shape, as_dtype(arr.dtype), init, trainable)


def trainable_variables(scope=None):
    return _g().get_collection(GraphKeys.TRAINABLE_VARIABLES, scope)


def global_variables(scope=None):
    return _g().get_collection(GraphKeys.GLOBAL_VARIABLES, scope)


def global_variables_initializer():
    g = _g()
    return g.add_node("NoOp", "init", control_inputs=[v.initializer.name for v in g.variables])


# ---------------------------------------------------------------------------
# tf.nn
# ---------------------------------------------------------------------------
def bias_add(value, bias, data_format=None, name=None) -> Tensor:
    x, b = convert_to_tensor(value), convert_to_tensor(bias)
    return _g().add_node("BiasAdd", name or "BiasAdd", [x, b], {"T": attr_type(x.dtype), "data_format": attr_s(data_format or "NHWC")},
                         [x.dtype], [x._shape]).outputs[0]


def _conv_out(n, k, s, padding):
    if n is None:
        return None
    return (n + s - 1) // s if padding == "SAME" else (n - k) // s + 1


def conv2d(input, filter, strides, padding, use_cudnn_on_gpu=True, data_format="NHWC", dilations=(1, 1, 1, 1), name=None) -> Tensor:  # noqa: A002
    x, w = convert_to_tensor(input), convert_to_tensor(filter)
    padding = padding.upper()
    kh, kw, _, co = w._shape
    n, h, wd, _ = x._shape if x._shape is not None else (None,) * 4
    oshape = (n, _conv_out(h, kh, strides[1], padding), _conv_out(wd, kw, strides[2], padding), co)
    return _g().add_node("Conv2D", name or "Conv2D", [x, w],
                         {"T": attr_type(x.dtype), "strides": attr_ilist(strides), "padding": attr_s(padding), "data_format": attr_s(data_format),
                          "dilations": attr_ilist(dilations), "use_cudnn_on_gpu": attr_b(use_cudnn_on_gpu)}, [x.dtype], [oshape]).outputs[0]


def _pool(op, value, ksize, strides, padding, data_format, name):
    x = convert_to_tensor(value)
    padding = padding.upper()
    n, h, w, c = x._shape if x._shape is not None else (None,) * 4
    oshape = (n, _conv_out(h, ksize[1], strides[1], padding), _conv_out(w, ksize[2], strides[2], padding), c)
    return _g().add_node(op, name or op, [x], {"T": attr_type(x.dtype), "ksize": attr_ilist(ksize), "strides": attr_ilist(strides),
                                             "padding": attr_s(padding), "data_format": attr_s(data_format)}, [x.dtype], [oshape]).outputs[0]


def max_pool(value, ksize, strides, padding, data_format="NHWC", name=None): return _pool("MaxPool", value, ksize, strides, padding, data_format, name)
def avg_pool(value, ksize, strides, padding, data_format="NHWC", name=None): return _pool("AvgPool", value, ksize, strides, padding, data_format, name)


def dropout(x, keep_prob=None, noise_shape=None, seed=None, name=None, rate=None) -> Tensor:
    """``tf.nn.dropout``: emits TF's ``dropout/{Shape,random_uniform,add,Floor,div,mul}`` sub-graph."""
    x = convert_to_tensor(x)
    if keep_prob is None:
        keep_prob = 1.0 - rate if not isinstance(rate, Tensor) else binary("Sub", 1.0, rate)
    g = _g()
    with g.name_scope(name or "dropout") as _:
        kp = convert_to_tensor(keep_prob, dtype=x.dtype, name="keep_prob")
        sh = shape(x)
        ru = g.add_node("RandomUniform", "random_uniform/RandomUniform", [sh],
                        {"T": attr_type(core.int32), "dtype": attr_type(x.dtype), "seed": attr_i(seed or 0), "seed2": attr_i(0)}, [x.dtype], [x._shape]).outputs[0]
        rnd = binary("Add", kp, ru, name="add")
        mask = unary("Floor", rnd, name="Floor")
        return binary("Mul", binary("RealDiv", x, kp, name="div"), mask, name="mul")


def softmax_cross_entropy_with_logits(labels=None, logits=None, dim=-1, name=None, _sentinel=None):
    logits_t, labels_t = convert_to_tensor(logits), convert_to_tensor(labels)
    op = _g().add_node("SoftmaxCrossEntropyWithLogits", name or "softmax_cross_entropy_with_logits", [logits_t, labels_t],
                       {"T": attr_type(logits_t.dtype)}, [logits_t.dtype, logits_t.dtype],
                       [None if logits_t._shape is None else (logits_t._shape[0],), logits_t._shape])
    return op.outputs[0]


def sigmoid_cross_entropy_with_logits(labels=None, logits=None, name=None, _sentinel=None):
    g = _g()
    with g.name_scope(name or "logistic_loss"):
        z, x = convert_to_tensor(labels), convert_to_tensor(logits)
        # max(x,0) - x*z + log(1+exp(-|x|))
        return binary("Add", binary("Sub", relu(x), binary("Mul", x, z)), unary("Log1p", exp(negative(abs(x)))))


# ---------------------------------------------------------------------------
# tf.layers
# ---------------------------------------------------------------------------
def _activation_name(fn) -> Optional[str]:
    if fn is None:
        return None
    table = {relu: "Relu", sigmoid: "Sigmoid", tanh: "Tanh", softmax: "Softmax", softplus: "Softplus", elu: "Elu", identity: None}
    if fn in table:
        return table[fn]
    nm = getattr(fn, "__name__", str(fn)).lower()
    for k in ("relu", "sigmoid", "tanh", "softmax", "softplus", "elu"):
        if nm == k:
            return k.capitalize()
    return "__callable__"


def _apply_activation(fn, x: Tensor) -> Tensor:
    an = _activation_name(fn)
    if an is None:
        return x
    if an == "__callable__":
        return fn(x)
    return unary(an, x, name=an)


def dense(inputs, units, activation=None, use_bias=True, kernel_initializer=None, bias_initializer=None, trainable=True,
          name=None, **_unused) -> Tensor:
    """``tf.layers.dense``: variables ``<scope>/kernel`` [in, units] and ``<scope>/bias`` [units]."""
    x = convert_to_tensor(inputs)
    g = _g()
    in_dim = x._shape[-1]
    if in_dim is None:
        raise ValueError("The last dimension of the inputs to `Dense` should be defined. Found `None`.")
    with g.name_scope(name or "dense") as scope:
        sc = scope[:-1]
        kernel = _make_variable(f"{sc}/kernel", (in_dim, units), x.dtype, kernel_initializer or _GlorotUniform(), trainable)
        bias = _make_variable(f"{sc}/bias", (units,), x.dtype, bias_initializer or _Zeros(), trainable) if use_bias else None
        if len(x._shape) > 2:
            raise NotImplementedError("dense on rank>2 inputs is not supported by the tfcompat builder")
        out = matmul(x, kernel.value(), name="MatMul")
        if bias is not None:
            out = bias_add(out, bias.value(), name="BiasAdd")
        return _apply_activation(activation, out)


def _pair(v) -> Tuple[int, int]:
    return (int(v), int(v)) if isinstance(v, int) else (int(v[0]), int(v[1]))


def conv2d_layer(inputs, filters, kernel_size, strides=(1, 1), padding="valid", activation=None, use_bias=True,
                 kernel_initializer=None, bias_initializer=None, trainable=True, name=None, **_unused) -> Tensor:
    """``tf.layers.conv2d`` (NHWC): variables ``<scope>/kernel`` [kh, kw, cin, filters], ``<scope>/bias``."""
    x = convert_to_tensor(inputs)
    g = _g()
    kh, kw = _pair(kernel_size)
    sh, sw = _pair(strides)
    cin = x._shape[-1]
    with g.name_scope(name or "conv2d") as scope:
        sc = scope[:-1]
        kernel = _make_variable(f"{sc}/kernel", (kh, kw, cin, filters), x.dtype, kernel_initializer or _GlorotUniform(), trainable)
        bias = _make_variable(f"{sc}/bias", (filters,), x.dtype, bias_initializer or _Zeros(), trainable) if use_bias else None
        out = conv2d(x, kernel.value(), (1, sh, sw, 1), padding, name="Conv2D")
        if bias is not None:
            out = bias_add(out, bias.value(), name="BiasAdd")
        return _apply_activation(activation, out)


def max_pooling2d(inputs, pool_size, strides, padding="valid", name=None, **_unused) -> Tensor:
    ph, pw = _pair(pool_size)
    sh, sw = _pair(strides)
    with _g().name_scope(name or "max_pooling2d"):
        return max_pool(inputs, (1, ph, pw, 1), (1, sh, sw, 1), padding, name="MaxPool")


def average_pooling2d(inputs, pool_size, strides, padding="valid", name=None, **_unused) -> Tensor:
    ph, pw = _pair(pool_size)
    sh, sw = _pair(strides)
    with _g().name_scope(name or "average_pooling2d"):
        return avg_pool(inputs, (1, ph, pw, 1), (1, sh, sw, 1), padding, name="AvgPool")


def flatten(inputs, name=None) -> Tensor:
    """``tf.layers.flatten``: Shape -> strided_slice -> Reshape/shape (Pack) -> Reshape."""
    x = convert_to_tensor(inputs)
    g = _g()
    with g.name_scope(name or "flatten"):
        sh = shape(x, name="Shape")

        def c(nm, v):
            return constant(np.asarray(v, np.int32), dtype=core.int32, name=nm)

        ss_name = g.unique_name("strided_slice")
        b, e, s = (g.add_node("Const", f"{ss_name}/{nm}", attrs={"dtype": attr_type(core.int32), "value": attr_tensor(np.asarray(v, np.int32), core.int32)},
                              out_dtypes=[core.int32], out_shapes=[(1,)], exact_name=True).outputs[0] for nm, v in (("stack", [0]), ("stack_1", [1]), ("stack_2", [1])))
        batch = g.add_node("StridedSlice", ss_name, [sh, b, e, s],
                           {"T": attr_type(core.int32), "Index": attr_type(core.int32), "begin_mask": attr_i(0), "end_mask": attr_i(0),
                            "ellipsis_mask": attr_i(0), "new_axis_mask": attr_i(0), "shrink_axis_mask": attr_i(1)}, [core.int32], [()], exact_name=True).outputs[0]
        rs_name = g.unique_name("Reshape")
        minus1 = g.add_node("Const", f"{rs_name}/shape/1", attrs={"dtype": attr_type(core.int32), "value": attr_tensor(np.asarray(-1, np.int32), core.int32)},
                            out_dtypes=[core.int32], out_shapes=[()], exact_name=True).outputs[0]
        packed = g.add_node("Pack", f"{rs_name}/shape", [batch, minus1], {"T": attr_type(core.int32), "N": attr_i(2), "axis": attr_i(0)},
                            [core.int32], [(2,)], exact_name=True).outputs[0]
        flat = None
        if x._shape is not None and all(d is not None for d in x._shape[1:]):
            flat = int(np.prod(x._shape[1:]))
        return g.add_node("Reshape", rs_name, [x, packed], {"T": attr_type(x.dtype), "Tshape": attr_type(core.int32)}, [x.dtype],
                          [(None if x._shape is None else x._shape[0], flat)], exact_name=True).outputs[0]


def dropout_layer(inputs, rate=0.5, noise_shape=None, seed=None, training=False, name=None) -> Tensor:
    if training is False:
        return identity(inputs, name=(name or "dropout") + "/Identity")
    return dropout(inputs, rate=rate, seed=seed, name=name or "dropout")


# ---------------------------------------------------------------------------
# tf.losses  (default reduction SUM_BY_NONZERO_WEIGHTS with weights = 1  ->  mean over elements)
# ---------------------------------------------------------------------------
def _finish_loss(scope_losses: Tensor, loss_collection: Optional[str]) -> Tensor:
    """``Sum`` over everything, divided by ``num_present`` (= element count for unit weights)."""
    total = reduce_sum(scope_losses, name="Sum")
    n = cast(size(scope_losses, name="num_present/Size"), scope_losses.dtype, name="num_present")
    value = binary("RealDiv", total, n, name="value")
    if loss_collection:
        _g().add_to_collection(loss_collection, value)
    return value


def softmax_cross_entropy(onehot_labels, logits, weights=1.0, label_smoothing=0, scope=None,
                          loss_collection=GraphKeys.LOSSES, **_unused) -> Tensor:
    if label_smoothing:
        raise NotImplementedError("label_smoothing is not supported by the tfcompat builder")
    g = _g()
    with g.name_scope(scope or "softmax_cross_entropy_loss"):
        per_row = softmax_cross_entropy_with_logits(labels=onehot_labels, logits=logits, name="xentropy")
        if not (isinstance(weights, (int, float)) and float(weights) == 1.0):
            per_row = binary("Mul", per_row, weights, name="Mul")
        return _finish_loss(per_row, loss_collection)


def mean_squared_error(labels, predictions, weights=1.0, scope=None, loss_collection=GraphKeys.LOSSES, **_unused) -> Tensor:
    g = _g()
    with g.name_scope(scope or "mean_squared_error"):
        sq = squared_difference(convert_to_tensor(predictions), convert_to_tensor(labels), name="SquaredDifference")
        if not (isinstance(weights, (int, float)) and float(weights) == 1.0):
            sq = binary("Mul", sq, weights, name="Mul")
        return _finish_loss(sq, loss_collection)


def sigmoid_cross_entropy(multi_class_labels, logits, weights=1.0, scope=None, loss_collection=GraphKeys.LOSSES, **_unused) -> Tensor:
    g = _g()
    with g.name_scope(scope or "sigmoid_cross_entropy_loss"):
        per = sigmoid_cross_entropy_with_logits(labels=multi_class_labels, logits=logits, name="xentropy")
        return _finish_loss(per, loss_collection)


def absolute_difference(labels, predictions, weights=1.0, scope=None, loss_collection=GraphKeys.LOSSES, **_unused) -> Tensor:
    g = _g()
    with g.name_scope(scope or "absolute_difference"):
        d = abs(binary("Sub", convert_to_tensor(predictions), convert_to_tensor(labels), name="Sub"), name="Abs")
        return _finish_loss(d, loss_collection)


def add_loss(loss, loss_collection=GraphKeys.LOSSES):
    _g().add_to_collection(loss_collection, convert_to_tensor(loss))


def get_losses(scope=None, loss_collection=GraphKeys.LOSSES):
    return _g().get_collection(loss_collection, scope)


# -------------------------------------------------------------------------------------------------
# More of the TF-1.x surface, emitted as the same op types real TF graphs use (all of them are executed by
# graph/executor.py; graphs that use them train on the interpreter engine unless the compiler recognises them)
# -------------------------------------------------------------------------------------------------
def relu6(x, name=None): return unary("Relu6", x, name)
def selu(x, name=None): return unary("Selu", x, name)
def softsign(x, name=None): return unary("Softsign", x, name)
def rsqrt(x, name=None): return unary("Rsqrt", x, name)
def log1p(x, name=None): return unary("Log1p", x, name)
def floor(x, name=None): return unary("Floor", x, name)
def ceil(x, name=None): return unary("Ceil", x, name)
def sign(x, name=None): return unary("Sign", x, name)
def reciprocal(x, name=None): return unary("Reciprocal", x, name)
def zeros_like(x, dtype=None, name=None): return unary("ZerosLike", x, name)
def ones_like(x, dtype=None, name=None): return unary("OnesLike", x, name)


def log_softmax(logits, axis=-1, name=None):
    return unary("LogSoftmax", logits, name)


def _compare(op: str, a, b, name) -> Tensor:
    if isinstance(a, (Tensor, Variable)):
        a = convert_to_tensor(a)
        b = convert_to_tensor(b, dtype=a.dtype, name=(name or op) + "/y")
    else:
        b = convert_to_tensor(b)
        a = convert_to_tensor(a, dtype=b.dtype, name=(name or op) + "/x")
    return _g().add_node(op, name or op, [a, b], {"T": attr_type(a.dtype)}, [core.bool_], [_bshape(a._shape, b._shape)]).outputs[0]


def greater(a, b, name=None): return _compare("Greater", a, b, name)
def greater_equal(a, b, name=None): return _compare("GreaterEqual", a, b, name)
def less(a, b, name=None): return _compare("Less", a, b, name)
def less_equal(a, b, name=None): return _compare("LessEqual", a, b, name)
def equal(a, b, name=None): return _compare("Equal", a, b, name)
def not_equal(a, b, name=None): return _compare("NotEqual", a, b, name)


def logical_not(x, name=None):
    x = convert_to_tensor(x)
    return _g().add_node("LogicalNot", name or "LogicalNot", [x], {}, [core.bool_], [x._shape]).outputs[0]


def logical_and(a, b, name=None):
    a, b = convert_to_tensor(a), convert_to_tensor(b)
    return _g().add_node("LogicalAnd", name or "LogicalAnd", [a, b], {}, [core.bool_], [_bshape(a._shape, b._shape)]).outputs[0]


def where(condition, x=None, y=None, name=None) -> Tensor:
    """Element-wise select (the three-argument form of ``tf.where``)."""
    if x is None or y is None:
        raise NotImplementedError("tf.where(condition) without x / y (index form) is not supported")
    c = convert_to_tensor(condition)
    if isinstance(x, (Tensor, Variable)):
        x = convert_to_tensor(x)
        y = convert_to_tensor(y, dtype=x.dtype, name=(name or "Select") + "/e")
    else:
        y = convert_to_tensor(y)
        x = convert_to_tensor(x, dtype=y.dtype, name=(name or "Select") + "/t")
    return _g().add_node("Select", name or "Select", [c, x, y], {"T": attr_type(x.dtype)}, [x.dtype], [_bshape(x._shape, y._shape)]).outputs[0]


def clip_by_value(t, clip_value_min, clip_value_max, name=None) -> Tensor:
    with _g().name_scope(name or "clip_by_value"):
        return binary("Maximum", binary("Minimum", t, clip_value_max, name="Minimum"), clip_value_min, name="Maximum")


def reduce_min(x, axis=None, keepdims=False, name=None, keep_dims=None, reduction_indices=None):
    return _reduce("Min", x, reduction_indices if axis is None else axis, bool(keep_dims if keep_dims is not None else keepdims), name)


def reduce_prod(x, axis=None, keepdims=False, name=None, keep_dims=None, reduction_indices=None):
    return _reduce("Prod", x, reduction_indices if axis is None else axis, bool(keep_dims if keep_dims is not None else keepdims), name)


def l2_loss(t, name=None) -> Tensor:
    """``sum(t ** 2) / 2`` (real TF has a fused L2Loss op; the composite is what its gradient expands to)."""
    with _g().name_scope(name or "L2Loss"):
        return binary("Mul", reduce_sum(square(t, name="Square"), name="Sum"), 0.5, name="mul")


def l2_normalize(x, axis=None, epsilon=1e-12, name=None, dim=None) -> Tensor:
    axis = dim if axis is None else axis
    with _g().name_scope(name or "l2_normalize"):
        sq = reduce_sum(square(x, name="Square"), axis=axis, keepdims=True, name="Sum")
        return binary("Mul", x, rsqrt(binary("Maximum", sq, epsilon, name="Maximum"), name="Rsqrt"), name="mul")


def tile(input, multiples, name=None) -> Tensor:  # noqa: A002
    x = convert_to_tensor(input)
    m = [int(v) for v in multiples]
    mt = constant(np.asarray(m, dtype=np.int32), dtype=core.int32, name="Const")
    oshape = None if x._shape is None else tuple(None if d is None else d * k for d, k in zip(x._shape, m))
    return _g().add_node("Tile", name or "Tile", [x, mt], {"T": attr_type(x.dtype), "Tmultiples": attr_type(core.int32)}, [x.dtype],
                         [oshape]).outputs[0]


def stack(values, axis=0, name="stack") -> Tensor:
    vals = [convert_to_tensor(v) for v in values]
    s0 = vals[0]._shape
    oshape = None
    if s0 is not None:
        ax = axis % (len(s0) + 1)
        oshape = tuple(list(s0[:ax]) + [len(vals)] + list(s0[ax:]))
    return _g().add_node("Pack", name or "stack", vals, {"T": attr_type(vals[0].dtype), "N": attr_i(len(vals)), "axis": attr_i(axis)},
                         [vals[0].dtype], [oshape]).outputs[0]


def log_loss(labels, predictions, weights=1.0, epsilon=1e-7, scope=None, loss_collection=GraphKeys.LOSSES, **_unused) -> Tensor:
    """``-y log(p + eps) - (1 - y) log(1 - p + eps)``, mean over elements (tf.losses.log_loss)."""
    g = _g()
    with g.name_scope(scope or "log_loss"):
        y, p = convert_to_tensor(labels), convert_to_tensor(predictions)
        pos = binary("Mul", y, log(binary("Add", p, epsilon, name="add"), name="Log"), name="mul")
        one_minus_y = binary("Sub", constant(1.0, dtype=y.dtype, name="sub/x"), y, name="sub")
        neg = binary("Mul", one_minus_y, log(binary("Add", binary("Sub", constant(1.0, dtype=p.dtype, name="sub_1/x"), p, name="sub_1"),
                                                    epsilon, name="add_1"), name="Log_1"), name="mul_1")
        per = negative(binary("Add", pos, neg, name="add_2"), name="Neg")
        if not (isinstance(weights, (int, float)) and float(weights) == 1.0):
            per = binary("Mul", per, weights, name="Mul")
        return _finish_loss(per, loss_collection)


def hinge_loss(labels, logits, weights=1.0, scope=None, loss_collection=GraphKeys.LOSSES, **_unused) -> Tensor:
    """``max(0, 1 - (2 y - 1) * logits)``, mean over elements (tf.losses.hinge_loss, labels in {0, 1})."""
    g = _g()
    with g.name_scope(scope or "hinge_loss"):
        y, z = convert_to_tensor(labels), convert_to_tensor(logits)
        signed = binary("Sub", binary("Mul", y, 2.0, name="mul"), 1.0, name="sub")
        per = relu(binary("Sub", constant(1.0, dtype=z.dtype, name="sub_1/x"), binary("Mul", signed, z, name="mul_1"), name="sub_1"), name="Relu")
        if not (isinstance(weights, (int, float)) and float(weights) == 1.0):
            per = binary("Mul", per, weights, name="Mul")
        return _finish_loss(per, loss_collection)


def huber_loss(labels, predictions, weights=1.0, delta=1.0, scope=None, loss_collection=GraphKeys.LOSSES, **_unused) -> Tensor:
    """Quadratic inside ``|e| <= delta``, linear outside (tf.losses.huber_loss), mean over elements."""
    g = _g()
    with g.name_scope(scope or "huber_loss"):
        err = binary("Sub", convert_to_tensor(predictions), convert_to_tensor(labels), name="Sub")
        a = abs(err, name="Abs")
        quad = binary("Minimum", a, delta, name="Minimum")
        lin = binary("Sub", a, quad, name="Sub_1")
        per = binary("Add", binary("Mul", binary("Mul", quad, quad, name="Mul"), 0.5, name="Mul_1"), binary("Mul", lin, delta, name="Mul_2"), name="Add")
        if not (isinstance(weights, (int, float)) and float(weights) == 1.0):
            per = binary("Mul", per, weights, name="Mul_3")
        return _finish_loss(per, loss_collection)


def batch_normalization(inputs, axis=-1, momentum=0.99, epsilon=1e-3, center=True, scale=True, beta_initializer=None,
                        gamma_initializer=None, moving_mean_initializer=None, moving_variance_initializer=None, training=False,
                        trainable=True, name=None, **_unused) -> Tensor:
    """``tf.layers.batch_normalization``: variables ``<scope>/gamma, beta`` (trainable) and ``<scope>/moving_mean,
    moving_variance`` (not trainable).  ``training=True`` normalises with the statistics of the batch, ``False`` with the
    moving statistics.  As in the reference (which only ever applies gradients of the trainable variables and never runs
    ``UPDATE_OPS``) the moving statistics keep their initial values."""
    x = convert_to_tensor(inputs)
    g = _g()
    rank = len(x._shape)
    ax = axis % rank
    c = x._shape[ax]
    if c is None:
        raise ValueError("batch_normalization needs a static size on the normalised axis")
    if training not in (True, False):
        raise NotImplementedError("batch_normalization(training=<tensor>) is not supported; pass a Python bool")
    with g.name_scope(name or "batch_normalization") as scope:
        sc = scope[:-1]
        gamma = _make_variable(f"{sc}/gamma", (c,), x.dtype, gamma_initializer or _Ones(), trainable) if scale else None
        beta = _make_variable(f"{sc}/beta", (c,), x.dtype, beta_initializer or _Zeros(), trainable) if center else None
        mm = _make_variable(f"{sc}/moving_mean", (c,), x.dtype, moving_mean_initializer or _Zeros(), False)
        mv = _make_variable(f"{sc}/moving_variance", (c,), x.dtype, moving_variance_initializer or _Ones(), False)
        red = [i for i in range(rank) if i != ax]
        bshape = [1] * rank
        bshape[ax] = c

        def per_channel(t):
            return t if ax == rank - 1 else reshape(t, bshape)

        if training:
            mean = reduce_mean(x, axis=red, keepdims=True, name="moments/mean")
            var = reduce_mean(squared_difference(x, stop_gradient(mean, name="moments/StopGradient"), name="moments/SquaredDifference"),
                              axis=red, keepdims=True, name="moments/variance")
        else:
            mean, var = per_channel(mm.value()), per_channel(mv.value())
        inv = rsqrt(binary("Add", var, epsilon, name="batchnorm/add"), name="batchnorm/Rsqrt")
        if gamma is not None:
            inv = binary("Mul", inv, per_channel(gamma.value()), name="batchnorm/mul")
        out = binary("Mul", binary("Sub", x, mean, name="batchnorm/sub"), inv, name="batchnorm/mul_1")
        if beta is not None:
            out = binary("Add", out, per_channel(beta.value()), name="batchnorm/add_1")
        return out


# ---------------------------------------------------------------------------
# more of the TF-1.x surface (embeddings, sparse labels, splits / pads, transposed and depthwise convolutions, tf.cond)
# ---------------------------------------------------------------------------
def _const_i32(value, name):
    return constant(np.asarray(value, np.int32), dtype=core.int32, name=name)


def one_hot(indices, depth, on_value=1.0, off_value=0.0, axis=-1, dtype=core.float32, name=None) -> Tensor:
    idx = convert_to_tensor(indices)
    dt = as_dtype(dtype)
    d = _const_i32(depth, "depth")
    on, off = constant(on_value, dtype=dt, name="on_value"), constant(off_value, dtype=dt, name="off_value")
    sh = None if idx._shape is None else tuple(idx._shape) + (int(depth),)
    return _g().add_node("OneHot", name or "one_hot", [idx, d, on, off], {"T": attr_type(dt), "TI": attr_type(idx.dtype), "axis": attr_i(axis)},
                         [dt], [sh]).outputs[0]


def gather(params, indices, validate_indices=None, name=None, axis=0) -> Tensor:
    p, idx = convert_to_tensor(params), convert_to_tensor(indices)
    ax = _const_i32(axis, "axis")
    sh = None
    if p._shape is not None and idx._shape is not None:
        a = axis % len(p._shape)
        sh = tuple(p._shape[:a]) + tuple(idx._shape) + tuple(p._shape[a + 1:])
    return _g().add_node("GatherV2", name or "GatherV2", [p, idx, ax],
                         {"Tparams": attr_type(p.dtype), "Tindices": attr_type(idx.dtype), "Taxis": attr_type(core.int32)}, [p.dtype], [sh]).outputs[0]


def embedding_lookup(params, ids, partition_strategy="mod", name=None, validate_indices=True, max_norm=None) -> Tensor:
    if isinstance(params, (list, tuple)):
        if len(params) != 1:
            raise NotImplementedError("embedding_lookup over a sharded list of tables")
        params = params[0]
    return gather(params, ids, name=name or "embedding_lookup")


def split(value, num_or_size_splits, axis=0, num=None, name="split"):
    x = convert_to_tensor(value)
    g = _g()
    dim = None if x._shape is None else x._shape[axis % len(x._shape)]

    def oshape(part):
        if x._shape is None:
            return None
        lst = list(x._shape)
        lst[axis % len(lst)] = part
        return tuple(lst)

    if isinstance(num_or_size_splits, int):
        k = num_or_size_splits
        ax = _const_i32(axis, "split_dim")
        part = None if dim is None else dim // k
        op = g.add_node("Split", name, [ax, x], {"T": attr_type(x.dtype), "num_split": attr_i(k)}, [x.dtype] * k, [oshape(part)] * k)
        return list(op.outputs)
    sizes = [int(s) for s in num_or_size_splits]
    sz, ax = _const_i32(sizes, "size_splits"), _const_i32(axis, "split_dim")
    op = g.add_node("SplitV", name, [x, sz, ax], {"T": attr_type(x.dtype), "Tlen": attr_type(core.int32), "num_split": attr_i(len(sizes))},
                    [x.dtype] * len(sizes), [oshape(None if s < 0 else s) for s in sizes])
    return list(op.outputs)


def unstack(value, num=None, axis=0, name="unstack"):
    x = convert_to_tensor(value)
    if num is None:
        if x._shape is None or x._shape[axis % len(x._shape)] is None:
            raise ValueError("unstack needs a static size along `axis` (or `num`)")
        num = x._shape[axis % len(x._shape)]
    sh = None if x._shape is None else tuple(d for i, d in enumerate(x._shape) if i != axis % len(x._shape))
    op = _g().add_node("Unpack", name, [x], {"T": attr_type(x.dtype), "num": attr_i(num), "axis": attr_i(axis)}, [x.dtype] * num, [sh] * num)
    return list(op.outputs)


def pad(tensor, paddings, mode="CONSTANT", name=None, constant_values=0) -> Tensor:
    x = convert_to_tensor(tensor)
    pads = np.asarray(paddings, np.int32).reshape(-1, 2)
    p = _const_i32(pads, "paddings")
    sh = None if x._shape is None else tuple(None if d is None else d + int(lo) + int(hi) for d, (lo, hi) in zip(x._shape, pads))
    mode = mode.upper()
    if mode == "CONSTANT":
        if constant_values:
            cv = constant(constant_values, dtype=x.dtype, name="constant_values")
            return _g().add_node("PadV2", name or "PadV2", [x, p, cv], {"T": attr_type(x.dtype), "Tpaddings": attr_type(core.int32)}, [x.dtype], [sh]).outputs[0]
        return _g().add_node("Pad", name or "Pad", [x, p], {"T": attr_type(x.dtype), "Tpaddings": attr_type(core.int32)}, [x.dtype], [sh]).outputs[0]
    return _g().add_node("MirrorPad", name or "MirrorPad", [x, p], {"T": attr_type(x.dtype), "Tpaddings": attr_type(core.int32), "mode": attr_s(mode)},
                         [x.dtype], [sh]).outputs[0]


def sparse_softmax_cross_entropy_with_logits(labels=None, logits=None, name=None, _sentinel=None):
    logits_t, labels_t = convert_to_tensor(logits), convert_to_tensor(labels)
    op = _g().add_node("SparseSoftmaxCrossEntropyWithLogits", name or "SparseSoftmaxCrossEntropyWithLogits", [logits_t, labels_t],
                       {"T": attr_type(logits_t.dtype), "Tlabels": attr_type(labels_t.dtype)}, [logits_t.dtype, logits_t.dtype],
                       [None if logits_t._shape is None else (logits_t._shape[0],), logits_t._shape])
    return op.outputs[0]


def sparse_softmax_cross_entropy(labels, logits, weights=1.0, scope=None, loss_collection=GraphKeys.LOSSES, reduction=None):
    with _g().name_scope(scope or "sparse_softmax_cross_entropy_loss"):
        per = sparse_softmax_cross_entropy_with_logits(labels=labels, logits=logits, name="xentropy")
        if not (isinstance(weights, (int, float)) and weights == 1.0):
            per = binary("Mul", per, weights, name="Mul")
        return _finish_loss(per, loss_collection)


def conv2d_transpose(value, filter, output_shape, strides, padding="SAME", data_format="NHWC", name=None) -> Tensor:  # noqa: A002
    """``tf.nn.conv2d_transpose``: filter is [kh, kw, out_channels, in_channels]; emitted as TF does, as the input-gradient
    op of the forward convolution."""
    y, w = convert_to_tensor(value), convert_to_tensor(filter)
    osh = [int(d) if d is not None else -1 for d in output_shape] if not isinstance(output_shape, (Tensor, Variable)) else None
    sizes = convert_to_tensor(output_shape) if osh is None else _const_i32(osh, "output_shape")
    sh = None if osh is None else tuple(None if d < 0 else d for d in osh)
    return _g().add_node("Conv2DBackpropInput", name or "conv2d_transpose", [sizes, w, y],
                         {"T": attr_type(y.dtype), "strides": attr_ilist(strides), "padding": attr_s(padding.upper()), "data_format": attr_s(data_format),
                          "dilations": attr_ilist([1, 1, 1, 1]), "use_cudnn_on_gpu": attr_b(True)}, [y.dtype], [sh]).outputs[0]


def conv2d_transpose_layer(inputs, filters, kernel_size, strides=(1, 1), padding="valid", activation=None, use_bias=True,
                           kernel_initializer=None, bias_initializer=None, name=None, trainable=True, **_unused) -> Tensor:
    """``tf.layers.conv2d_transpose`` (NHWC, static spatial sizes)."""
    x = convert_to_tensor(inputs)
    kh, kw = _pair(kernel_size)
    sh, sw = _pair(strides)
    n, h, w, cin = x._shape
    if h is None or w is None:
        raise ValueError("conv2d_transpose needs static height / width")
    padding = padding.upper()
    oh = h * sh if padding == "SAME" else h * sh + max(kh - sh, 0)
    ow = w * sw if padding == "SAME" else w * sw + max(kw - sw, 0)
    g = _g()
    with g.name_scope(name or "conv2d_transpose") as scope:
        kernel = get_variable(scope + "kernel", [kh, kw, filters, cin], x.dtype, kernel_initializer or glorot_uniform_initializer(), trainable)
        if n is None:
            bs = g.add_node("StridedSlice", "strided_slice", [shape(x), _const_i32([0], "ss/b"), _const_i32([1], "ss/e"), _const_i32([1], "ss/s")],
                            {"T": attr_type(core.int32), "Index": attr_type(core.int32), "shrink_axis_mask": attr_i(1), "begin_mask": attr_i(0),
                             "end_mask": attr_i(0), "ellipsis_mask": attr_i(0), "new_axis_mask": attr_i(0)}, [core.int32], [()]).outputs[0]
            sizes = stack([bs, _const_i32(oh, "oh"), _const_i32(ow, "ow"), _const_i32(filters, "oc")], name="output_shape")
            y = g.add_node("Conv2DBackpropInput", "conv2d_transpose", [sizes, convert_to_tensor(kernel), x],
                           {"T": attr_type(x.dtype), "strides": attr_ilist([1, sh, sw, 1]), "padding": attr_s(padding), "data_format": attr_s("NHWC"),
                            "dilations": attr_ilist([1, 1, 1, 1]), "use_cudnn_on_gpu": attr_b(True)}, [x.dtype], [(None, oh, ow, filters)]).outputs[0]
        else:
            y = conv2d_transpose(x, kernel, [n, oh, ow, filters], [1, sh, sw, 1], padding)
        if use_bias:
            bias = get_variable(scope + "bias", [filters], x.dtype, bias_initializer or zeros_initializer(), trainable)
            y = bias_add(y, bias)
        return _apply_activation(activation, y)


def depthwise_conv2d(input, filter, strides, padding, rate=None, name=None, data_format="NHWC") -> Tensor:  # noqa: A002
    x, w = convert_to_tensor(input), convert_to_tensor(filter)
    padding = padding.upper()
    kh, kw, ch, mult = w._shape
    n, h, wd, _ = x._shape if x._shape is not None else (None,) * 4
    dil = [1, 1, 1, 1] if rate is None else [1, rate[0], rate[1], 1]
    oshape = (n, _conv_out(h, (kh - 1) * dil[1] + 1, strides[1], padding), _conv_out(wd, (kw - 1) * dil[2] + 1, strides[2], padding), ch * mult)
    return _g().add_node("DepthwiseConv2dNative", name or "depthwise", [x, w],
                         {"T": attr_type(x.dtype), "strides": attr_ilist(strides), "padding": attr_s(padding), "data_format": attr_s(data_format),
                          "dilations": attr_ilist(dil)}, [x.dtype], [oshape]).outputs[0]


def erf(x, name=None): return unary("Erf", x, name)
def sin(x, name=None): return unary("Sin", x, name)
def cos(x, name=None): return unary("Cos", x, name)
def round(x, name=None): return unary("Round", x, name)  # noqa: A001
def floormod(a, b, name=None): return binary("FloorMod", a, b, name)


def logical_or(a, b, name=None):
    a, b = convert_to_tensor(a, dtype=core.bool_), convert_to_tensor(b, dtype=core.bool_)
    return _g().add_node("LogicalOr", name or "LogicalOr", [a, b], {}, [core.bool_], [_bshape(a._shape, b._shape)]).outputs[0]


def cumsum(x, axis=0, exclusive=False, reverse=False, name=None) -> Tensor:
    x = convert_to_tensor(x)
    ax = _const_i32(axis, "axis")
    return _g().add_node("Cumsum", name or "Cumsum", [x, ax], {"T": attr_type(x.dtype), "Tidx": attr_type(core.int32), "exclusive": attr_b(exclusive),
                                                            "reverse": attr_b(reverse)}, [x.dtype], [x._shape]).outputs[0]


def _bool_reduce(op, x, axis, keepdims, name):
    x = convert_to_tensor(x, dtype=core.bool_)
    rank = len(x._shape)
    axes = list(range(rank)) if axis is None else ([axis] if isinstance(axis, int) else list(axis))
    ax = _const_i32(axes, "reduction_indices")
    norm = [a % rank for a in axes]
    sh = tuple((1 if i in norm else d) for i, d in enumerate(x._shape) if keepdims or i not in norm)
    return _g().add_node(op, name or op, [x, ax], {"Tidx": attr_type(core.int32), "keep_dims": attr_b(bool(keepdims))}, [core.bool_], [sh]).outputs[0]


def reduce_any(x, axis=None, keepdims=False, name=None, keep_dims=None): return _bool_reduce("Any", x, axis, keepdims or bool(keep_dims), name)
def reduce_all(x, axis=None, keepdims=False, name=None, keep_dims=None): return _bool_reduce("All", x, axis, keepdims or bool(keep_dims), name)


def top_k(input, k=1, sorted=True, name=None):  # noqa: A002
    x = convert_to_tensor(input)
    kk = _const_i32(k, "k")
    sh = None if x._shape is None else tuple(x._shape[:-1]) + (int(k),)
    op = _g().add_node("TopKV2", name or "TopKV2", [x, kk], {"T": attr_type(x.dtype), "sorted": attr_b(sorted)}, [x.dtype, core.int32], [sh, sh])
    return op.outputs[0], op.outputs[1]


def cond(pred, true_fn=None, false_fn=None, strict=False, name=None, fn1=None, fn2=None):
    """``tf.cond``.  A python bool picks the branch at graph-construction time; a tensor predicate emits the
    ``Switch`` / ``Merge`` pair TF-1.x graphs carry (both branches are built; the engine evaluates the live one)."""
    true_fn, false_fn = true_fn or fn1, false_fn or fn2
    if isinstance(pred, (bool, np.bool_)):
        return true_fn() if pred else false_fn()
    p = convert_to_tensor(pred, dtype=core.bool_)
    g = _g()
    with g.name_scope(name or "cond"):
        t, f = true_fn(), false_fn()
        single = not isinstance(t, (list, tuple))
        ts, fs = ([t], [f]) if single else (list(t), list(f))
        outs = []
        for a, b in zip(ts, fs):
            a, b = convert_to_tensor(a), convert_to_tensor(b)
            sa = g.add_node("Switch", "Switch_t", [a, p], {"T": attr_type(a.dtype)}, [a.dtype, a.dtype], [a._shape, a._shape])
            sb = g.add_node("Switch", "Switch_f", [b, p], {"T": attr_type(b.dtype)}, [b.dtype, b.dtype], [b._shape, b._shape])
            m = g.add_node("Merge", "Merge", [sb.outputs[0], sa.outputs[1]], {"T": attr_type(a.dtype), "N": attr_i(2)}, [a.dtype, core.int32],
                           [a._shape if a._shape == b._shape else None, ()])
            outs.append(m.outputs[0])
        return outs[0] if single else outs


def strided_slice_from_key(x: Tensor, key) -> Tensor:
    """``tensor[...]`` with ints and slices (no Ellipsis / newaxis): emits the ``StridedSlice`` node TF emits, with begin /
    end / shrink masks."""
    x = convert_to_tensor(x)
    keys = key if isinstance(key, tuple) else (key,)
    if any(k is Ellipsis or k is None for k in keys):
        raise NotImplementedError("tensor[...] / tensor[None]: use tf.expand_dims / explicit slices")
    begin, end, strides = [], [], []
    bm = em = sm = 0
    shape = []
    static = x._shape
    for i, k in enumerate(keys):
        dim = None if static is None else static[i]
        if isinstance(k, slice):
            st = 1 if k.step is None else int(k.step)
            if st <= 0:
                raise NotImplementedError("negative slice steps")
            if k.start is None:
                bm |= 1 << i
            if k.stop is None:
                em |= 1 << i
            b, e = int(k.start or 0), int(k.stop or 0)
            begin.append(b); end.append(e); strides.append(st)
            if dim is None:
                shape.append(None if (k.stop is None or b < 0 or e < 0) else max((e - b + st - 1) // st, 0))
            else:
                shape.append(len(range(*k.indices(dim))))
        else:
            k = int(k)
            sm |= 1 << i
            begin.append(k); end.append(k + 1 if k != -1 else 0); strides.append(1)
            if k == -1:
                em |= 1 << i
    oshape = None if static is None else tuple(shape) + tuple(static[len(keys):])
    g = _g()
    name = g.unique_name("strided_slice")
    mk = lambda v, n: g.add_node("Const", f"{name}/{n}", attrs={"dtype": attr_type(core.int32), "value": attr_tensor(np.asarray(v, np.int32), core.int32)},  # noqa: E731
                                 out_dtypes=[core.int32], out_shapes=[(len(v),)], exact_name=True).outputs[0]
    return g.add_node("StridedSlice", name, [x, mk(begin, "stack"), mk(end, "stack_1"), mk(strides, "stack_2")],
                      {"T": attr_type(x.dtype), "Index": attr_type(core.int32), "begin_mask": attr_i(bm), "end_mask": attr_i(em),
                       "ellipsis_mask": attr_i(0), "new_axis_mask": attr_i(0), "shrink_axis_mask": attr_i(sm)}, [x.dtype], [oshape], exact_name=True).outputs[0]
