"""GraphIR -> LayerPlan: recognise the layer structure the H100 engine has hand-written kernels for.

The reference runs whatever graph the user serialised through a TF session.  The H100 engine
instead executes a *compiled* plan: the forward chain between ``tfInput`` and the loss is pattern-
matched into dense / conv / pool / reshape layers with fused bias+activation, the loss into
softmax-cross-entropy (one-hot labels or class indices), sigmoid-cross-entropy or mean-squared-error, ``tf.nn.dropout`` / ``tf.layers.dropout`` after a dense layer into a
fused Philox mask in that layer's epilogue (after a conv layer, a max-pool or the flatten of either: a mask on that
image layer, keyed by the pixel row ``b * OH * OW + oy * OW + ox`` and the channel), and ``tfOutput`` into "activation of layer k" (+ optional ArgMax /
Softmax).  Graphs outside this family (custom losses, exotic ops) are reported as unsupported so the caller can use the
generic interpreter engine instead (loudly: a RuntimeWarning names the reason).

Covers every model the reference ships (SURVEY.md section 2.3): simple_dnn, cnn_example,
autoencoder_example, the test MLPs / auto-encoder and the checkpoint fixture, and the usual TF-1.x CNN geometry beyond
them: NHWC ``Conv2D`` with VALID or SAME padding and any stride, ``MaxPool`` with a window of up to 4x4, any stride and
VALID or SAME padding (e.g. the "Deep MNIST" network).  Output sizes and pads follow TensorFlow: VALID
``out = (in - k) // s + 1``; SAME ``out = ceil(in / s)`` with ``pad_total = max((out - 1) * s + k - in, 0)`` split as
``top = pad_total // 2`` and the extra row / column at the bottom / right.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

from ..graph.ir import GraphIR, Node, split_ref

# SfAct (csrc/sf_api.h).  Every activation here has a derivative that is a function of its output, which is all the step
# stores: act'(z) is recomputed from a = act(z) in the backward kernels and the fused dropout recovers its mask from a.
ACT_IDS = {None: 0, "Relu": 1, "Sigmoid": 2, "Tanh": 3, "Elu": 4, "Selu": 5, "Softplus": 6, "Softsign": 7, "LeakyRelu": 8, "Relu6": 9}
ACT_OPS = tuple(a for a in ACT_IDS if a is not None)
# activations whose derivative needs the pre-activation, which the step does not keep
_PREACT_ACTS = ("Swish", "Gelu")


class UnsupportedGraph(ValueError):
    """The graph is valid but outside the family the compiled H100 plan covers."""


@dataclass
class Layer:
    kind: str                                   # dense | conv | pool | reshape
    kernel: Optional[str] = None                # variable node names
    bias: Optional[str] = None
    act: Optional[str] = None                   # an ACT_OPS name or None
    act_alpha: float = 0.0                      # LeakyRelu: the slope for x < 0 (0 for every other activation)
    in_shape: Tuple[int, ...] = ()              # per-sample shape (no batch dim)
    out_shape: Tuple[int, ...] = ()
    ksize: Tuple[int, int] = (0, 0)            # conv: filter taps; pool: window
    strides: Tuple[int, int] = (1, 1)           # conv / pool: (sh, sw)
    pads: Tuple[int, int, int, int] = (0, 0, 0, 0)   # conv / pool: (top, bottom, left, right), from the padding mode
    padding: str = "VALID"                      # conv / pool: TF padding mode (VALID | SAME)
    tensors: Dict[str, str] = field(default_factory=dict)   # stage -> tensor name (linear / bias / act / dropout)
    # dense / conv / pool: keep probability of a tf.nn.dropout applied to the layer's output (0 = none); a conv's dropout
    # follows its bias and activation, and a dropout on the flatten of an image layer is that layer's
    dropout_keep: float = 0.0

    @property
    def in_features(self) -> int:
        n = 1
        for d in self.in_shape:
            n *= d
        return n

    @property
    def out_features(self) -> int:
        n = 1
        for d in self.out_shape:
            n *= d
        return n


@dataclass
class OutputSpec:
    layer: int                                  # index into LayerPlan.layers whose output is fetched (-1 = the input)
    stage: str                                  # linear | bias | act
    post: Optional[str] = None                  # ArgMax | Softmax | None


@dataclass
class LayerPlan:
    layers: List[Layer]
    loss: Optional[str]                         # softmax_xent | sparse_softmax_xent | sigmoid_xent | mse | None (inference only)
    input_name: str
    label_name: Optional[str]                   # placeholder fed with labels; None if target is the input
    target_is_input: bool
    input_dim: int
    label_dim: int                              # label columns fed per row (1 for sparse_softmax_xent: the class index)
    output: Optional[OutputSpec]
    var_order: List[str]
    # L2 weight penalties of the loss: variable -> c of the term c * sum(v ** 2) (kernels and biases of the layers only)
    penalty: Dict[str, float] = field(default_factory=dict)

    def trainable_layers(self) -> List[Layer]:
        return [l for l in self.layers if l.kind in ("dense", "conv")]

    def is_mlp(self) -> bool:
        return all(l.kind in ("dense", "reshape") for l in self.layers)


_PASS = ("Identity", "StopGradient", "PlaceholderWithDefault")
MAX_POOL_WINDOW = 4


def _padding(node: Node) -> str:
    p = node.attrs.get("padding", "VALID")
    return p.decode() if isinstance(p, bytes) else str(p)


def conv_geometry(size: int, k: int, s: int, padding: str) -> Tuple[int, int, int]:
    """TensorFlow's output size and (before, after) padding of one spatial dimension."""
    if padding == "SAME":
        out = -(-size // s)
        total = max((out - 1) * s + k - size, 0)
        return out, total // 2, total - total // 2
    return (size - k) // s + 1, 0, 0


def _var_of(ir: GraphIR, ref: Tuple[str, int]) -> Optional[str]:
    node = ir.nodes[ref[0]]
    hops = 0
    while node.op in ("Identity", "ReadVariableOp") and node.inputs and hops < 4:
        node = ir.nodes[node.inputs[0][0]]
        hops += 1
    return node.name if node.op in ("VariableV2", "Variable", "VarHandleOp") else None


def _const_scalar(ir: GraphIR, ref: Tuple[str, int]) -> Optional[float]:
    """Value of a scalar that is a Const, possibly behind Identity / PlaceholderWithDefault / `1 - rate` arithmetic."""
    node = ir.nodes[ref[0]]
    hops = 0
    while node.op in ("Identity", "PlaceholderWithDefault", "Cast") and node.inputs and hops < 6:
        node = ir.nodes[node.inputs[0][0]]
        hops += 1
    if node.op == "Const":
        try:
            return float(node.attrs["value"].reshape(-1)[0])
        except Exception:
            return None
    if node.op == "Sub" and len(node.inputs) == 2:
        a, b = _const_scalar(ir, node.inputs[0]), _const_scalar(ir, node.inputs[1])
        return None if a is None or b is None else a - b
    return None


def _const_ones(ir: GraphIR, ref: Tuple[str, int]) -> bool:
    """``ref`` is a Const (possibly behind Identity / PlaceholderWithDefault / Cast) whose every element is 1"""
    node = ir.nodes[ref[0]]
    hops = 0
    while node.op in ("Identity", "PlaceholderWithDefault", "Cast") and node.inputs and hops < 6:
        node = ir.nodes[node.inputs[0][0]]
        hops += 1
    if node.op != "Const":
        return False
    try:
        v = node.attrs["value"].reshape(-1)
        return v.size > 0 and bool((v == 1).all())
    except Exception:
        return False


def _match_dropout(ir: GraphIR, node: Node) -> Optional[Tuple[Tuple[str, int], float]]:
    """``tf.nn.dropout`` sub-graph: Mul(RealDiv(x, keep), Floor(Add(keep, RandomUniform(Shape(x))))) -> (x, keep)."""
    if node.op != "Mul" or len(node.inputs) != 2:
        return None
    for a, b in ((node.inputs[0], node.inputs[1]), (node.inputs[1], node.inputs[0])):
        div, flo = ir.nodes[a[0]], ir.nodes[b[0]]
        if div.op not in ("RealDiv", "Div") or flo.op != "Floor":
            continue
        add = ir.nodes[flo.inputs[0][0]]
        if add.op not in ("Add", "AddV2") or not any(ir.nodes[i[0]].op == "RandomUniform" for i in add.inputs):
            continue
        keep = _const_scalar(ir, div.inputs[1])
        if keep is None:
            raise UnsupportedGraph(f"dropout '{node.name}': keep_prob is a placeholder without a default - it is never fed during "
                                   "training (reference: HogwildSparkModel.py never feeds tfDropout), use tf.placeholder_with_default")
        return div.inputs[0], float(keep)
    return None


def _noise_is_shape_of_x(ir: GraphIR, node: Node, x: Tuple[str, int]) -> bool:
    """the RandomUniform of dropout ``node`` (matched by ``_match_dropout``, input ``x``) draws one number per element of
    ``x``: its shape is Shape(x), not a ``noise_shape`` that broadcasts one draw over several elements"""
    for ref in node.inputs:
        flo = ir.nodes[ref[0]]
        if flo.op != "Floor":
            continue
        for i in ir.nodes[flo.inputs[0][0]].inputs:
            ru = ir.nodes[i[0]]
            if ru.op == "RandomUniform":
                sh = ir.nodes[ru.inputs[0][0]] if ru.inputs else None
                return sh is not None and sh.op == "Shape" and len(sh.inputs) == 1 and tuple(sh.inputs[0]) == tuple(x)
    return False


def _is_zeros_like(ir: GraphIR, ref: Tuple[str, int], x: Tuple[str, int]) -> bool:
    n = ir.nodes[ref[0]]
    return n.op == "ZerosLike" and len(n.inputs) == 1 and n.inputs[0] == x


def _is_nonneg_cond(ir: GraphIR, ref: Tuple[str, int], x: Tuple[str, int]) -> bool:
    """``x >= zeros_like(x)``"""
    n = ir.nodes[ref[0]]
    return n.op == "GreaterEqual" and len(n.inputs) == 2 and n.inputs[0] == x and _is_zeros_like(ir, n.inputs[1], x)


def _relu_of(ir: GraphIR, ref: Tuple[str, int]) -> Optional[Tuple[str, int]]:
    """x of ``Relu(x)`` or of TF's ``Select(x >= zeros_like(x), x, zeros_like(x))``"""
    n = ir.nodes[ref[0]]
    if n.op == "Relu" and len(n.inputs) == 1:
        return n.inputs[0]
    if n.op == "Select" and len(n.inputs) == 3:
        x = n.inputs[1]
        if _is_nonneg_cond(ir, n.inputs[0], x) and _is_zeros_like(ir, n.inputs[2], x):
            return x
    return None


def _neg_abs_of(ir: GraphIR, ref: Tuple[str, int]) -> Optional[Tuple[str, int]]:
    """x of ``Neg(Abs(x))`` or of TF's ``Select(x >= zeros_like(x), Neg(x), x)``"""
    n = ir.nodes[ref[0]]
    if n.op == "Neg" and len(n.inputs) == 1:
        a = ir.nodes[n.inputs[0][0]]
        return a.inputs[0] if a.op == "Abs" and len(a.inputs) == 1 else None
    if n.op == "Select" and len(n.inputs) == 3:
        x = n.inputs[2]
        neg = ir.nodes[n.inputs[1][0]]
        if _is_nonneg_cond(ir, n.inputs[0], x) and neg.op == "Neg" and neg.inputs == [x]:
            return x
    return None


def _match_sigmoid_xent(ir: GraphIR, node: Node) -> Optional[Tuple[Tuple[str, int], Tuple[str, int]]]:
    """``tf.nn.sigmoid_cross_entropy_with_logits``: Add(Sub(relu(x), Mul(x, z)), Log1p(Exp(-|x|))), with relu and -|x| in
    the tfcompat builder's spelling (Relu, Neg(Abs)) or TF-1.x's (Select on x >= 0) -> (logits x, labels z)."""
    if node.op not in ("Add", "AddV2") or len(node.inputs) != 2:
        return None
    for s_ref, l_ref in ((node.inputs[0], node.inputs[1]), (node.inputs[1], node.inputs[0])):
        sub, log1p = ir.nodes[s_ref[0]], ir.nodes[l_ref[0]]
        if sub.op != "Sub" or len(sub.inputs) != 2 or log1p.op != "Log1p" or len(log1p.inputs) != 1:
            continue
        ex = ir.nodes[log1p.inputs[0][0]]
        if ex.op != "Exp" or len(ex.inputs) != 1:
            continue
        x = _relu_of(ir, sub.inputs[0])
        mul = ir.nodes[sub.inputs[1][0]]
        if x is None or mul.op != "Mul" or len(mul.inputs) != 2 or _neg_abs_of(ir, ex.inputs[0]) != x:
            continue
        if mul.inputs[0] == x:
            return x, mul.inputs[1]
        if mul.inputs[1] == x:
            return x, mul.inputs[0]
    return None


_FLOAT_TYPES = ("DT_FLOAT", "DT_HALF", "DT_BFLOAT16", "DT_DOUBLE")


def _float_cast(node: Node) -> bool:
    return node.attrs.get("SrcT", "DT_FLOAT") in _FLOAT_TYPES and node.attrs.get("DstT", "DT_FLOAT") in _FLOAT_TYPES


# casts a class index may pass through: each of these types holds every index below MAX_SPARSE_CLASSES exactly, so the
# kernels, which read the placeholder's float32, see the index TF computes.  A narrower type (half, bfloat16, 8 / 16-bit
# ints) or an unsigned one can round or wrap an index.
_INDEX_CAST_TYPES = ("DT_FLOAT", "DT_DOUBLE", "DT_INT32", "DT_INT64")
# The stand-alone sparse softmax kernel (N > 32) accumulates the bias gradient of every class in shared memory, 4 bytes per
# class within the 48 KB a launch gets without opting in to more.
MAX_SPARSE_CLASSES = 12288


def _attr_ints(v) -> List[int]:
    return [int(a) for a in (v if isinstance(v, (list, tuple)) else [v])]


def _one_hot_of(ir: GraphIR, ref: Tuple[str, int]) -> Optional[Node]:
    """the OneHot node behind ``ref`` (through Identity / StopGradient / PlaceholderWithDefault), or None"""
    node = ir.nodes[ref[0]]
    while node.op in _PASS and node.inputs:
        node = ir.nodes[node.inputs[0][0]]
    return node if node.op == "OneHot" else None


def _check_one_hot(ir: GraphIR, node: Node, n_classes: int) -> None:
    """``tf.one_hot(idx, N)`` with the defaults the sparse head computes: depth N, on 1, off 0, the class axis last"""
    depth = _const_scalar(ir, node.inputs[1]) if len(node.inputs) == 4 else None
    on = _const_scalar(ir, node.inputs[2]) if len(node.inputs) == 4 else None
    off = _const_scalar(ir, node.inputs[3]) if len(node.inputs) == 4 else None
    if depth is None or int(depth) != n_classes:
        raise UnsupportedGraph(f"one_hot '{node.name}' with depth {depth} for {n_classes} logits is not covered by the compiled plan")
    if on is None or off is None:
        raise UnsupportedGraph(f"one_hot '{node.name}' with an on_value or off_value that is not a constant is not covered by the "
                               "compiled plan")
    if on != 1.0 or off != 0.0:
        raise UnsupportedGraph(f"one_hot '{node.name}' with on_value {on} / off_value {off} (label smoothing) is not covered by the "
                               "compiled plan")
    if int(node.attrs.get("axis", -1)) != -1:
        raise UnsupportedGraph(f"one_hot '{node.name}' along axis {node.attrs.get('axis')} is not covered by the compiled plan")


def _class_index_placeholder(ir: GraphIR, ref: Tuple[str, int]) -> Node:
    """Walk the class indices of a sparse softmax cross-entropy (or of its ``tf.one_hot``) back to their placeholder: through
    Identity / StopGradient / PlaceholderWithDefault, Cast between float32, float64, int32 and int64, and exactly one Reshape to [-1] or
    Squeeze of axis 1, which flattens the [None, 1] column ``ml_util`` feeds a scalar label with."""
    node = ir.nodes[ref[0]]
    flattened = False
    for _ in range(32):
        if node.op in _PASS and node.inputs:
            node = ir.nodes[node.inputs[0][0]]
        elif node.op == "Cast" and node.inputs:
            src, dst = node.attrs.get("SrcT", "DT_FLOAT"), node.attrs.get("DstT", "DT_FLOAT")
            if src not in _INDEX_CAST_TYPES or dst not in _INDEX_CAST_TYPES:
                raise UnsupportedGraph(f"Cast '{node.name}' from {src} to {dst} on the class-index path can round or wrap a class "
                                       "index; the compiled plan takes casts between float32, float64, int32 and int64")
            node = ir.nodes[node.inputs[0][0]]
        elif node.op == "Reshape" and not flattened and len(node.inputs) == 2 and ir.nodes[node.inputs[1][0]].op == "Const" \
                and [int(v) for v in ir.nodes[node.inputs[1][0]].attrs["value"].reshape(-1)] == [-1]:
            flattened = True
            node = ir.nodes[node.inputs[0][0]]
        elif node.op == "Squeeze" and not flattened and node.inputs and _attr_ints(node.attrs.get("squeeze_dims", [])) in ([1], [-1]):
            flattened = True
            node = ir.nodes[node.inputs[0][0]]
        else:
            break
    if node.op not in ("Placeholder", "PlaceholderV2"):
        raise UnsupportedGraph(f"class labels reach the loss through '{node.op}' ({node.name}): the compiled plan covers Identity, "
                               "Cast and one Reshape to [-1] or Squeeze of axis 1 of a [None, 1] label placeholder")
    shape = node.attrs.get("shape")
    if not flattened or not shape or len(shape) != 2:
        raise UnsupportedGraph(f"class labels need a rank-2 [None, 1] label placeholder flattened by a Reshape to [-1] or a Squeeze "
                               f"of axis 1; '{node.name}' has shape {shape}")
    return node


def _preact_reason(what: str) -> str:
    return (f"{what} is not covered by the compiled plan: its derivative is not a function of its output, and the step "
            "keeps only activation outputs")


def _match_leaky_maximum(ir: GraphIR, node: Node) -> Optional[Tuple[Tuple[str, int], float]]:
    """TF 1.4-1.12's ``tf.nn.leaky_relu``: Maximum(Mul(alpha, x), x), operands of both ops in either order -> (x, alpha)"""
    if node.op != "Maximum" or len(node.inputs) != 2:
        return None
    for m_ref, x in ((node.inputs[0], node.inputs[1]), (node.inputs[1], node.inputs[0])):
        mul = ir.nodes[m_ref[0]]
        if mul.op != "Mul" or len(mul.inputs) != 2 or x not in mul.inputs:
            continue
        c = mul.inputs[1] if mul.inputs[0] == x else mul.inputs[0]
        alpha = _const_scalar(ir, c)
        if alpha is None:
            raise UnsupportedGraph(f"leaky ReLU '{node.name}': alpha is not a constant, so it is not covered by the compiled plan")
        if not 0.0 <= alpha <= 1.0:
            raise UnsupportedGraph(f"Maximum(alpha * x, x) '{node.name}' with alpha {alpha} outside [0, 1] is not a leaky ReLU and is not "
                                   "covered by the compiled plan")
        return x, alpha
    return None


def _match_activation(ir: GraphIR, node: Node) -> Optional[Tuple[str, float, Tuple[str, int]]]:
    """(activation, act_alpha, input) when ``node`` is an activation the compiled plan fuses into its layer"""
    if node.op in _PREACT_ACTS:
        raise UnsupportedGraph(_preact_reason(f"activation '{node.op}' ({node.name})"))
    if node.op == "Mul" and len(node.inputs) == 2:
        for x, s in ((node.inputs[0], node.inputs[1]), (node.inputs[1], node.inputs[0])):
            sig = ir.nodes[s[0]]
            if sig.op == "Sigmoid" and sig.inputs == [x]:
                raise UnsupportedGraph(_preact_reason(f"swish x * sigmoid(x) ('{node.name}')"))
        return None
    leaky = _match_leaky_maximum(ir, node)
    if leaky is not None:
        x, alpha = leaky
        return ("Relu", 0.0, x) if alpha == 0.0 else ("LeakyRelu", float(alpha), x)
    if node.op not in ACT_OPS or len(node.inputs) != 1:
        return None
    if node.op == "LeakyRelu":
        alpha = float(node.attrs.get("alpha", 0.2))
        if alpha < 0.0:
            # the sign of the output would no longer tell the backward pass which branch the unit took
            raise UnsupportedGraph(f"leaky ReLU '{node.name}' with a negative alpha ({alpha}) is not covered by the compiled plan")
        return ("Relu", 0.0, node.inputs[0]) if alpha == 0.0 else ("LeakyRelu", alpha, node.inputs[0])
    return node.op, 0.0, node.inputs[0]


def _strip_pass(ir: GraphIR, ref: Tuple[str, int]) -> Node:
    node = ir.nodes[ref[0]]
    while node.op in _PASS and node.inputs:
        node = ir.nodes[node.inputs[0][0]]
    return node


def _sums_all_axes(ir: GraphIR, node: Node, var: str) -> bool:
    """Sum ``node`` reduces every axis of variable ``var``"""
    if len(node.inputs) != 2 or ir.nodes[node.inputs[1][0]].op != "Const":
        return False
    rank = len(ir.nodes[var].attrs.get("shape", ()))
    axes = sorted({int(a) % max(rank, 1) for a in ir.nodes[node.inputs[1][0]].attrs["value"].reshape(-1)})
    return axes == list(range(rank))


def _const_node(ir: GraphIR, ref: Tuple[str, int]) -> Node:
    node = ir.nodes[ref[0]]
    for _ in range(6):
        if node.op not in ("Identity", "PlaceholderWithDefault", "Cast") or not node.inputs:
            break
        node = ir.nodes[node.inputs[0][0]]
    return node


def _scalar_factor(ir: GraphIR, ref: Tuple[str, int]) -> Optional[float]:
    """The value of ``ref`` when it is a constant of exactly one element (a scalar, or [1], [1, 1], ...), possibly
    behind Identity / PlaceholderWithDefault / Cast or `a - b` of such constants; None otherwise.  A penalty coefficient
    must be one: a constant of several elements weighs the elements of the variable differently."""
    node = _const_node(ir, ref)
    if node.op == "Const":
        try:
            v = node.attrs["value"].reshape(-1)
        except Exception:
            return None
        return float(v[0]) if v.size == 1 else None
    if node.op == "Sub" and len(node.inputs) == 2:
        a, b = _scalar_factor(ir, node.inputs[0]), _scalar_factor(ir, node.inputs[1])
        return None if a is None or b is None else a - b
    return None


def _const_elements(ir: GraphIR, ref: Tuple[str, int]) -> int:
    """element count of the constant behind ``ref`` (0: not a constant)"""
    node = _const_node(ir, ref)
    try:
        return int(node.attrs["value"].size) if node.op == "Const" else 0
    except Exception:
        return 0


def _per_element_reason(node: Node, n: int) -> str:
    return (f"L2 penalty '{node.name}' with a coefficient that is a constant of {n} elements (per-element or masked decay) is "
            "not covered by the compiled plan: it takes one coefficient per variable")


def _l2_terms(ir: GraphIR, ref: Tuple[str, int]) -> Optional[List[Tuple[Tuple[str, int], float]]]:
    """[(x, c)] when ``ref`` is a sum of L2 penalties c * sum(x ** 2) of the accepted forms - L2Loss(x), Sum(Square(x)),
    Sum(Mul(k, Square(x))) (Keras's l2) - each, and the sum, times constant factors (the builder's l2_loss is
    Mul(Sum(Square(x)), 0.5); ``5e-4 * add_n([...])`` scales a sum), or None.  Raises for an L1 term and for a penalty
    whose coefficient is not a constant."""
    node = _strip_pass(ir, ref)
    c = 1.0
    for _ in range(16):
        if node.op != "Mul" or len(node.inputs) != 2:
            break
        a, b = node.inputs
        ka, kb = _scalar_factor(ir, a), _scalar_factor(ir, b)
        if kb is not None:
            c, node = c * kb, _strip_pass(ir, a)
        elif ka is not None:
            c, node = c * ka, _strip_pass(ir, b)
        else:
            for k_ref, t_ref in ((a, b), (b, a)):
                n = _const_elements(ir, k_ref)
                if n > 1 and _is_penalty_shaped(ir, t_ref):
                    raise UnsupportedGraph(_per_element_reason(node, n))
            if _is_penalty_shaped(ir, a) or _is_penalty_shaped(ir, b):
                raise UnsupportedGraph(f"L2 penalty '{node.name}' with a coefficient that is not a constant is not covered by the "
                                       "compiled plan")
            return None
    if node.op in ("Add", "AddV2", "AddN") and node.inputs:
        terms = []
        for i in node.inputs:
            t = _l2_terms(ir, i)
            if t is None:
                return None
            terms += [(x, c * k) for x, k in t]
        return terms
    if node.op == "L2Loss" and len(node.inputs) == 1:
        return [(node.inputs[0], 0.5 * c)]
    if node.op != "Sum" or not node.inputs:
        return None
    inner = _strip_pass(ir, node.inputs[0])
    if inner.op == "Mul" and len(inner.inputs) == 2:
        for k_ref, s_ref in ((inner.inputs[0], inner.inputs[1]), (inner.inputs[1], inner.inputs[0])):
            k, sq = _scalar_factor(ir, k_ref), _strip_pass(ir, s_ref)
            if sq.op in ("Square", "Abs") and k is None and _const_elements(ir, k_ref) > 1:
                raise UnsupportedGraph(_per_element_reason(inner, _const_elements(ir, k_ref)))
            if k is not None and sq.op in ("Square", "Abs"):
                c, inner = c * k, sq
                break
    if inner.op == "Abs":
        raise UnsupportedGraph(f"L1 penalty '{node.name}' (Abs) is not covered by the compiled plan")
    if inner.op != "Square" or len(inner.inputs) != 1:
        return None
    var = _var_of(ir, inner.inputs[0])
    if var is not None and not _sums_all_axes(ir, node, var):
        raise UnsupportedGraph(f"'{node.name}' sums the squares of a variable over some of its axes: only a penalty over the whole "
                               "variable is covered by the compiled plan")
    return [(inner.inputs[0], c)]


def _is_penalty_shaped(ir: GraphIR, ref: Tuple[str, int]) -> bool:
    try:
        return _l2_terms(ir, ref) is not None
    except UnsupportedGraph:
        return True


def _split_loss(ir: GraphIR, loss_ref: str) -> Tuple[str, Dict[str, float]]:
    """Split the training loss into its data term and its L2 weight penalties: a top-level Add / AddV2 / AddN (through
    Identity, nested in any order) of exactly one data loss and terms c * sum(v ** 2) of bare variables.  Returns the data
    term and {variable: summed c}, without the variables whose coefficients add to 0."""
    top = _strip_pass(ir, split_ref(loss_ref))
    if top.op not in ("Add", "AddV2", "AddN") or _match_sigmoid_xent(ir, top) is not None:
        return loss_ref, {}
    terms: List[Tuple[str, int]] = []

    def flatten(node: Node) -> None:
        for ref in node.inputs:
            n = _strip_pass(ir, ref)
            if n.op in ("Add", "AddV2", "AddN") and _match_sigmoid_xent(ir, n) is None:
                flatten(n)
            else:
                terms.append(ref)

    flatten(top)
    data: List[Tuple[str, int]] = []
    penalty: Dict[str, float] = {}
    for ref in terms:
        l2 = _l2_terms(ir, ref)
        if l2 is None:
            if _scalar_factor(ir, ref) == 0.0:         # tf.losses.get_regularization_loss() of a graph without regularizers
                continue
            data.append(ref)
            continue
        for x, c in l2:
            var = _var_of(ir, x)
            if var is None:
                raise UnsupportedGraph(f"L2 penalty on '{_strip_pass(ir, x).op}' ({x[0]}): the compiled plan covers penalties on bare "
                                       "variables only (no activity regularizers or penalties of expressions)")
            if not math.isfinite(c):
                raise UnsupportedGraph(f"L2 penalty on '{var}' with the coefficient {c} is not covered by the compiled plan")
            penalty[var] = penalty.get(var, 0.0) + c
    if len(data) != 1:
        raise UnsupportedGraph(f"loss '{loss_ref}' adds {len(data)} data losses: the compiled plan covers one data loss plus L2 "
                               "weight penalties")
    return f"{data[0][0]}:{data[0][1]}", {v: c for v, c in penalty.items() if c != 0.0}


def _find_loss_core(ir: GraphIR, loss_ref: str) -> Tuple[str, Node]:
    """Walk back from the scalar loss through reductions / scalings to the per-element loss node."""
    seen = set()
    frontier = [split_ref(loss_ref)[0]]
    while frontier:
        name = frontier.pop(0)
        if name in seen:
            continue
        seen.add(name)
        node = ir.nodes[name]
        if node.op in ("Add", "AddV2", "AddN") and any(_is_penalty_shaped(ir, i) for i in node.inputs):
            raise UnsupportedGraph(f"loss '{loss_ref}' adds an L2 penalty under a reduction or a scaling ('{node.name}'): the compiled "
                                   "plan covers penalties added at the top of the loss")
        if node.op == "SoftmaxCrossEntropyWithLogits":
            # tf.one_hot of class indices as the labels: the sparse head
            return ("sparse_softmax_xent" if _one_hot_of(ir, node.inputs[1]) is not None else "softmax_xent"), node
        if node.op == "SparseSoftmaxCrossEntropyWithLogits":
            return "sparse_softmax_xent", node
        if node.op == "SquaredDifference":
            return "mse", node
        if node.op == "Square" and node.inputs and ir.nodes[node.inputs[0][0]].op == "Sub":
            return "mse", ir.nodes[node.inputs[0][0]]
        if _match_sigmoid_xent(ir, node) is not None:
            return "sigmoid_xent", node
        if node.op in ("Sum", "Mean", "RealDiv", "Div", "DivNoNan", "Mul", "Identity", "Select", "Reshape", "Cast"):
            # follow data inputs that are not plain constants / shape plumbing
            for src, _ in node.inputs[: 1 if node.op in ("Sum", "Mean", "Reshape") else len(node.inputs)]:
                if ir.nodes[src].op not in ("Const", "Size", "Shape", "Fill", "Greater", "Equal", "ZerosLike", "OnesLike"):
                    frontier.append(src)
        else:
            continue
    raise UnsupportedGraph(f"loss '{loss_ref}' is neither softmax-cross-entropy, sigmoid-cross-entropy nor mean-squared-error")


def _check_mean_reduction(ir: GraphIR, loss_ref: str, kind: str, core: Node) -> None:
    """The kernels implement the *mean* over elements (tf.losses default).  Verify numerically cheap:
    the path from core to loss must contain a Sum followed by a division, or a Mean."""
    name = split_ref(loss_ref)[0]
    ops_on_path = []
    node = ir.nodes[name]
    hops = 0
    while node.name != core.name and hops < 16:
        ops_on_path.append(node.op)
        if kind in ("sigmoid_xent", "sparse_softmax_xent") and node.op == "Mul" and not any(_const_ones(ir, i) for i in node.inputs):
            raise UnsupportedGraph(f"weighted {'sigmoid' if kind == 'sigmoid_xent' else 'sparse softmax'} cross-entropy is not "
                                   "covered by the compiled plan")
        nxt = None
        for src, _ in node.inputs:
            if ir.nodes[src].op not in ("Const", "Size", "Shape", "Cast") or src == core.name:
                nxt = ir.nodes[src]
                break
        if nxt is None:
            break
        node = nxt
        hops += 1
    if "Mean" in ops_on_path:
        if kind == "mse" and "Mul" in ops_on_path:
            raise UnsupportedGraph("scaled MSE variants are not covered by the compiled plan")
        if kind == "sigmoid_xent" and "Sum" in ops_on_path:
            # e.g. reduce_mean(reduce_sum(per_element, axis=1)): a sum over the labels, N times the element mean
            raise UnsupportedGraph("a sum under a mean of sigmoid cross-entropy is not covered by the compiled plan")
        if kind == "sparse_softmax_xent" and "Sum" in ops_on_path:
            # reduce_mean(reduce_sum(per_row)): the batch total, B times the mean
            raise UnsupportedGraph("a sum under a mean of sparse softmax cross-entropy is not covered by the compiled plan")
        return
    if "Sum" in ops_on_path and any(o in ops_on_path for o in ("RealDiv", "Div", "DivNoNan")):
        return
    raise UnsupportedGraph("only mean-reduced losses are covered by the compiled plan")


def compile_graph(ir: GraphIR, tf_input: str, tf_label: Optional[str], tf_output: Optional[str] = None,
                  need_loss: bool = True) -> LayerPlan:
    input_node = split_ref(tf_input)[0]
    if input_node not in ir.nodes:
        raise KeyError(f"tfInput '{tf_input}' is not in the graph")
    in_shape = ir.nodes[input_node].attrs.get("shape")
    if not in_shape or len(in_shape) != 2 or in_shape[1] is None or in_shape[1] < 0:
        raise UnsupportedGraph("the compiled plan needs a rank-2 input placeholder [batch, features]")
    input_dim = int(in_shape[1])

    loss_kind: Optional[str] = None
    penalty: Dict[str, float] = {}
    pred_ref: Optional[Tuple[str, int]] = None
    target_ref: Optional[Tuple[str, int]] = None
    if need_loss:
        if not ir.losses:
            raise ValueError("the graph has no 'losses' collection entry; training needs tf.losses.* (or add_loss)")
        data_ref, penalty = _split_loss(ir, ir.losses[0])
        loss_kind, core = _find_loss_core(ir, data_ref)
        _check_mean_reduction(ir, data_ref, loss_kind, core)
        a, b = core.inputs[0], core.inputs[1]
        if loss_kind in ("softmax_xent", "sparse_softmax_xent"):
            pred_ref, target_ref = a, b               # (features=logits, labels / class indices / their one_hot)
        elif loss_kind == "sigmoid_xent":
            pred_ref, target_ref = _match_sigmoid_xent(ir, core)
        else:
            # mean_squared_error is symmetric: the side that is a placeholder is the target
            def is_ph(ref):
                n = ir.nodes[ref[0]]
                while n.op in _PASS and n.inputs:
                    n = ir.nodes[n.inputs[0][0]]
                return n.op in ("Placeholder", "PlaceholderV2")
            pred_ref, target_ref = (b, a) if is_ph(a) and not is_ph(b) else (a, b)
    else:
        if not tf_output:
            raise ValueError("inference compilation needs tfOutput")
        pred_ref = split_ref(tf_output)

    # ---- resolve the prediction-side post op (ArgMax / Softmax) for inference fetches ------------
    def strip_post(ref: Tuple[str, int]) -> Tuple[Tuple[str, int], Optional[str]]:
        n = ir.nodes[ref[0]]
        if n.op == "ArgMax":
            return n.inputs[0], "ArgMax"
        if n.op == "Softmax":
            return n.inputs[0], "Softmax"
        return ref, None

    chain_end = pred_ref
    post_of_end = None
    if not need_loss:
        chain_end, post_of_end = strip_post(pred_ref)

    # ---- walk the forward chain backwards -------------------------------------------------------
    layers_rev: List[Layer] = []
    cur = chain_end
    pending_act: Optional[Tuple[str, str, float]] = None   # (act, tensor name, act_alpha)
    pending_bias: Optional[Tuple[str, str]] = None     # (var, tensor name)
    # (keep_prob, tensor name, one draw per element) of a dropout above the next layer found
    pending_drop: Optional[Tuple[float, str, bool]] = None

    def image_dropout(what: str) -> Tuple[float, str]:
        """the pending dropout, landing on image layer ``what``"""
        if not pending_drop[2]:
            raise UnsupportedGraph(f"dropout '{pending_drop[1]}' on {what} draws its noise in a shape other than Shape(x) (spatial "
                                   "dropout via noise_shape), which the compiled plan does not cover")
        return pending_drop[0], pending_drop[1]

    guard = 0
    while True:
        guard += 1
        if guard > 10000:
            raise UnsupportedGraph("forward chain too long or cyclic")
        node = ir.nodes[cur[0]]
        tname = f"{node.name}:{cur[1]}"
        if node.name == input_node:
            if pending_drop:
                raise UnsupportedGraph("dropout applied directly to the input is not covered by the compiled plan")
            break
        if node.op in _PASS:
            cur = node.inputs[0]
            continue
        drop = _match_dropout(ir, node)
        if drop is not None:
            if pending_act or pending_bias or pending_drop:
                raise UnsupportedGraph(f"dropout '{node.name}' is not directly on top of a layer output")
            if drop[1] < 1.0:
                if drop[1] <= 0.0:
                    raise UnsupportedGraph("dropout with keep_prob <= 0")
                pending_drop = (drop[1], tname, _noise_is_shape_of_x(ir, node, drop[0]))
            cur = drop[0]
            continue
        act = _match_activation(ir, node)
        if act is not None:
            if pending_act or pending_bias:
                raise UnsupportedGraph(f"activation '{node.name}' is not directly on top of a linear layer")
            pending_act = (act[0], tname, act[1])
            cur = act[2]
            continue
        if node.op == "BiasAdd" or (node.op in ("Add", "AddV2") and _var_of(ir, node.inputs[1]) is not None):
            if pending_bias:
                raise UnsupportedGraph("two bias additions in a row")
            var = _var_of(ir, node.inputs[1])
            if var is None:
                raise UnsupportedGraph(f"BiasAdd '{node.name}' does not add a variable")
            pending_bias = (var, tname)
            cur = node.inputs[0]
            continue
        if node.op == "MatMul":
            if node.attrs.get("transpose_a") or node.attrs.get("transpose_b"):
                raise UnsupportedGraph("transposed MatMul is not covered by the compiled plan")
            kvar = _var_of(ir, node.inputs[1])
            if kvar is None:
                raise UnsupportedGraph(f"MatMul '{node.name}' right operand is not a variable")
            kin, kout = ir.nodes[kvar].attrs["shape"]
            tensors = {"linear": tname}
            if pending_bias:
                tensors["bias"] = pending_bias[1]
            if pending_act:
                tensors["act"] = pending_act[1]
            if pending_drop:
                tensors["dropout"] = pending_drop[1]
            layers_rev.append(Layer("dense", kernel=kvar, bias=pending_bias[0] if pending_bias else None,
                                    act=pending_act[0] if pending_act else None, act_alpha=pending_act[2] if pending_act else 0.0,
                                    in_shape=(kin,), out_shape=(kout,), tensors=tensors,
                                    dropout_keep=pending_drop[0] if pending_drop else 0.0))
            pending_act = pending_bias = pending_drop = None
            cur = node.inputs[0]
            continue
        if pending_drop and node.op not in ("Conv2D", "MaxPool", "Reshape"):
            raise UnsupportedGraph(f"dropout on top of '{node.op}' ({node.name}): the compiled plan fuses dropout into dense, conv and "
                                   "max-pool layers only")
        if node.op == "Conv2D":
            strides = [int(v) for v in node.attrs.get("strides", [1, 1, 1, 1])]
            if _padding(node) not in ("VALID", "SAME") or len(strides) != 4 or strides[0] != 1 or strides[3] != 1 or min(strides) < 1 \
                    or node.attrs.get("data_format", "NHWC") != "NHWC" or list(node.attrs.get("dilations", [1, 1, 1, 1])) != [1, 1, 1, 1]:
                raise UnsupportedGraph("only NHWC / undilated Conv2D with VALID or SAME padding and strides [1, sh, sw, 1] is covered "
                                       "by the compiled plan")
            kvar = _var_of(ir, node.inputs[1])
            if kvar is None:
                raise UnsupportedGraph(f"Conv2D '{node.name}' filter is not a variable")
            kh, kw, cin, cout = ir.nodes[kvar].attrs["shape"]
            tensors = {"linear": tname}
            if pending_bias:
                tensors["bias"] = pending_bias[1]
            if pending_act:
                tensors["act"] = pending_act[1]
            keep = 0.0
            if pending_drop:
                keep, tensors["dropout"] = image_dropout(f"conv '{node.name}'")
            layers_rev.append(Layer("conv", kernel=kvar, bias=pending_bias[0] if pending_bias else None,
                                    act=pending_act[0] if pending_act else None, act_alpha=pending_act[2] if pending_act else 0.0,
                                    in_shape=(-1, -1, cin), out_shape=(-1, -1, cout),
                                    ksize=(kh, kw), strides=(strides[1], strides[2]), padding=_padding(node), tensors=tensors,
                                    dropout_keep=keep))
            pending_act = pending_bias = pending_drop = None
            cur = node.inputs[0]
            continue
        if pending_act or pending_bias:
            raise UnsupportedGraph(f"bias/activation stacked on unsupported op '{node.op}' ({node.name})")
        if node.op == "MaxPool":
            ks = [int(v) for v in node.attrs.get("ksize", [])]
            st = [int(v) for v in node.attrs.get("strides", [])]
            if len(ks) != 4 or len(st) != 4 or ks[0] != 1 or ks[3] != 1 or st[0] != 1 or st[3] != 1 or min(ks) < 1 or min(st) < 1 \
                    or max(ks[1], ks[2]) > MAX_POOL_WINDOW or _padding(node) not in ("VALID", "SAME") \
                    or node.attrs.get("data_format", "NHWC") != "NHWC":
                raise UnsupportedGraph(f"only NHWC MaxPool with a window of at most {MAX_POOL_WINDOW}x{MAX_POOL_WINDOW}, strides "
                                       "[1, sh, sw, 1] and VALID or SAME padding is covered by the compiled plan")
            tensors, keep = {"act": tname}, 0.0
            if pending_drop:
                keep, tensors["dropout"] = image_dropout(f"max-pool '{node.name}'")
                pending_drop = None
            layers_rev.append(Layer("pool", ksize=(ks[1], ks[2]), strides=(st[1], st[2]), padding=_padding(node), tensors=tensors,
                                    dropout_keep=keep))
            cur = node.inputs[0]
            continue
        if node.op == "Reshape":
            # a pending dropout passes through: on a flatten it is the dropout of the image layer below (the same mask,
            # the flat row [OH * OW * C] being that layer's pixel rows side by side); on the input's reshape it meets the
            # input and is refused there
            layers_rev.append(Layer("reshape", tensors={"pre_dropout" if pending_drop else "act": tname,
                                                        "shape_src": f"{node.inputs[1][0]}:{node.inputs[1][1]}"}))
            cur = node.inputs[0]
            continue
        raise UnsupportedGraph(f"op '{node.op}' ({node.name}) is not covered by the compiled plan")

    layers = layers_rev[::-1]
    for i, l in enumerate(layers):
        if l.kind == "pool" and l.dropout_keep and i > 0 and layers[i - 1].kind == "conv" and layers[i - 1].dropout_keep:
            raise UnsupportedGraph(f"dropouts on both conv '{layers[i - 1].kernel}' and the max-pool after it are not covered by the "
                                   "compiled plan")

    # ---- shape propagation ---------------------------------------------------------------------
    shape: Tuple[int, ...] = (input_dim,)
    for l in layers:
        if l.kind == "reshape":
            src = ir.node_of(l.tensors["shape_src"])
            tgt: Optional[List[int]] = None
            if src.op == "Const":
                tgt = [int(v) for v in src.attrs["value"].reshape(-1)][1:]
            elif src.op == "Pack":                       # tf.layers.flatten: [batch, -1]
                tgt = [-1]
            if tgt is None:
                raise UnsupportedGraph("dynamic Reshape target")
            total = 1
            for d in shape:
                total *= d
            if tgt.count(-1) == 1:
                known = 1
                for d in tgt:
                    if d != -1:
                        known *= d
                tgt[tgt.index(-1)] = total // known
            l.in_shape, l.out_shape = shape, tuple(tgt)
        elif l.kind == "dense":
            if len(shape) != 1 or shape[0] != l.in_shape[0]:
                raise UnsupportedGraph(f"dense layer '{l.kernel}' expects {l.in_shape} features but receives {shape}")
        elif l.kind in ("conv", "pool"):
            if len(shape) != 3:
                raise UnsupportedGraph(f"{l.kind} layer on a non-image tensor (per-sample shape {shape})")
            if l.kind == "conv" and shape[2] != l.in_shape[2]:
                raise UnsupportedGraph(f"conv layer '{l.kernel}' expects NHWC input, got per-sample shape {shape}")
            oh, pt, pb = conv_geometry(shape[0], l.ksize[0], l.strides[0], l.padding)
            ow, pl, pr = conv_geometry(shape[1], l.ksize[1], l.strides[1], l.padding)
            if oh < 1 or ow < 1:
                raise UnsupportedGraph(f"{l.kind} layer: a {l.ksize[0]}x{l.ksize[1]} window does not fit its {shape[0]}x{shape[1]} input")
            l.in_shape, l.pads = shape, (pt, pb, pl, pr)
            l.out_shape = (oh, ow, l.out_shape[2] if l.kind == "conv" else shape[2])
        shape = l.out_shape

    if not any(l.kind in ("dense", "conv") for l in layers):
        raise UnsupportedGraph("no trainable layer between tfInput and the loss")

    # ---- target ----------------------------------------------------------------------------------
    label_name = None
    target_is_input = False
    label_dim = 0
    n_out = layers[-1].out_features
    if need_loss and loss_kind == "sparse_softmax_xent":
        # one class index per row: SparseSoftmaxCrossEntropyWithLogits(logits, idx) or the one-hot spelling
        # SoftmaxCrossEntropyWithLogits(logits, OneHot(idx, N, 1, 0))
        one_hot = _one_hot_of(ir, target_ref)
        if one_hot is not None:
            _check_one_hot(ir, one_hot, n_out)
            target_ref = one_hot.inputs[0]
        tnode = _class_index_placeholder(ir, target_ref)
        label_name = f"{tnode.name}:0"
        if tf_label is not None and split_ref(tf_label)[0] != tnode.name:
            raise UnsupportedGraph(f"the loss target is placeholder '{tnode.name}' but tfLabel is '{tf_label}'")
        tshape = tnode.attrs.get("shape")
        label_dim = int(tshape[1]) if tshape[1] is not None else -1
        if label_dim != 1:
            raise UnsupportedGraph(f"label width does not match: class labels take a [None, 1] placeholder, '{tnode.name}' is {tshape}")
        if n_out < 2:
            raise UnsupportedGraph("sparse softmax cross-entropy needs at least 2 classes")
        if n_out > MAX_SPARSE_CLASSES:
            raise UnsupportedGraph(f"sparse softmax cross-entropy over {n_out} classes is not covered by the compiled plan (at most "
                                   f"{MAX_SPARSE_CLASSES}: the loss kernel keeps one bias-gradient word per class in shared memory)")
    elif need_loss:
        tnode = ir.nodes[target_ref[0]]
        # tf.losses.sigmoid_cross_entropy casts the labels to the logits' dtype
        passes = _PASS + ("Cast",) if loss_kind == "sigmoid_xent" else _PASS
        while tnode.op in passes and tnode.inputs and (tnode.op != "Cast" or _float_cast(tnode)):
            tnode = ir.nodes[tnode.inputs[0][0]]
        if tnode.name == input_node:
            target_is_input = True
            label_dim = input_dim
        elif tnode.op in ("Placeholder", "PlaceholderV2"):
            label_name = f"{tnode.name}:0"
            tshape = tnode.attrs.get("shape")
            label_dim = int(tshape[1]) if tshape and len(tshape) == 2 and tshape[1] and tshape[1] > 0 else layers[-1].out_features
            if tf_label is not None and split_ref(tf_label)[0] != tnode.name:
                raise UnsupportedGraph(f"the loss target is placeholder '{tnode.name}' but tfLabel is '{tf_label}'")
        else:
            raise UnsupportedGraph("loss target must be a placeholder or the input itself")
        if label_dim != n_out:
            raise UnsupportedGraph("label width does not match the network output width")
    if need_loss:
        if loss_kind in ("softmax_xent", "sigmoid_xent", "sparse_softmax_xent") and layers[-1].act is not None:
            raise UnsupportedGraph(f"{'sigmoid' if loss_kind == 'sigmoid_xent' else 'softmax'} cross-entropy expects raw logits")
        if layers[-1].dropout_keep:
            raise UnsupportedGraph("dropout on the network output is not covered by the compiled plan")

    # ---- output fetch ------------------------------------------------------------------------------
    out_spec: Optional[OutputSpec] = None
    if tf_output:
        ref, post = strip_post(split_ref(tf_output))
        want = f"{ref[0]}:{ref[1]}"
        if split_ref(want)[0] == input_node:
            out_spec = OutputSpec(-1, "act", post)
        else:
            for i, l in enumerate(layers):
                if l.tensors.get("pre_dropout") == want:
                    raise UnsupportedGraph(f"tfOutput '{tf_output}' fetches a pre-activation tensor (the flatten below a dropout)")
                for stage in ("dropout", "act", "bias", "linear"):
                    if l.tensors.get(stage) == want:
                        # the fetched stage must be the layer's final stage (we do not keep pre-activations)
                        final = "dropout" if l.dropout_keep else ("act" if l.act or l.kind in ("pool", "reshape") else ("bias" if l.bias else "linear"))
                        if stage != final:
                            raise UnsupportedGraph(f"tfOutput '{tf_output}' fetches a pre-activation tensor")
                        out_spec = OutputSpec(i, stage, post)
            if out_spec is None and need_loss:
                out_spec = None            # tfOutput may be unrelated to training (reference cnn_example); resolved at predict time
            elif out_spec is None:
                raise UnsupportedGraph(f"tfOutput '{tf_output}' is not a tensor of the forward chain")

    layer_vars = {v for l in layers for v in (l.kernel, l.bias) if v is not None}
    for v in penalty:
        if v not in layer_vars:
            raise UnsupportedGraph(f"L2 penalty on '{v}', which is not a kernel or bias of a layer of the compiled plan")
    return LayerPlan(layers=layers, loss=loss_kind, input_name=f"{input_node}:0", label_name=label_name,
                     target_is_input=target_is_input, input_dim=input_dim, label_dim=label_dim, output=out_spec,
                     var_order=[v.name for v in ir.trainable], penalty=penalty)
