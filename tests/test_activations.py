"""ELU, SELU, softplus, softsign, leaky ReLU and ReLU6 in the compiled plan, without a GPU: the compiler accepts every
spelling that reaches it and refuses what the step cannot differentiate, with a reason; the float64 oracle of networks
using them matches the interpreter; the per-step tolerances of the GPU test reject plausible activation bugs; and the new
kernels keep no stack frame and the GEMM twins stay inside the GEMMs' register bound.

The oracle and graph helpers here are shared with tests/test_gpu_activations.py.  The oracle follows
test_step_gradients._forward (whose helpers it reuses); it differs in taking act' of the activations with a jump in it
(SELU and leaky ReLU at 0, ReLU6 at 0 and 6) on the branch the step took, and in carrying the step's stored
activations forward where they are a rounding of its own, both read from the step's stored output.
"""
import struct

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sparkflow_b200.graph import tfcompat as tf
from sparkflow_b200.graph.executor import GraphProgram
from sparkflow_b200.graph.ir import GraphIR
from sparkflow_b200.graph_utils import build_graph
from sparkflow_b200.models import zoo
from sparkflow_b200.models.compiler import ACT_IDS, UnsupportedGraph, compile_graph
from sparkflow_b200.parallel.plan_builder import act_arg, check_grammar, fused_first_conv
from kernel_usage import gemm_instances, needs_binary_utils, res_usage
from test_step_gradients import _assert_grads, _bf16, _conv, _grads, _pool_argmax, _pool_gather, _rejects

SELU = (1.0507009873554805, 1.6732632423543772)       # (lambda, alpha)
NEW_ACTS = ("Elu", "Selu", "Softplus", "Softsign", "LeakyRelu", "Relu6")
JUMP_ACTS = ("Selu", "LeakyRelu", "Relu6")            # act' jumps at 0 (and ReLU6 at 6)


# ------------------------------------------------------------------------------------------------------------------
# activation tables (float64), with the knobs the tolerance test turns into plausible bugs
# ------------------------------------------------------------------------------------------------------------------
def act_value(z, act, alpha, bug=None):
    bug = bug or {}
    lam, al = bug.get("selu", SELU)
    if act is None:
        return z
    if act == "Relu":
        return torch.relu(z)
    if act == "Sigmoid":
        return torch.sigmoid(z)
    if act == "Tanh":
        return torch.tanh(z)
    if act == "Elu":
        return F.elu(z)
    if act == "Selu":
        return lam * torch.where(z > 0, z, al * torch.expm1(z))
    if act == "Softplus":
        return F.softplus(z)
    if act == "Softsign":
        return F.softsign(z)
    if act == "LeakyRelu":
        return F.leaky_relu(z, bug.get("leaky", alpha))
    if act == "Relu6":
        return torch.clamp(z, 0.0, 6.0)
    raise KeyError(act)


def act_deriv(a, act, alpha, pos=None, top=None, bug=None):
    """act'(z) from the activation value a = act(z), as the backward kernels compute it.  ``pos`` / ``top``: the branch
    (a > 0 / a >= 6) when the step's record decides it."""
    bug = bug or {}
    lam, al = bug.get("selu", SELU)
    pos = a > 0 if pos is None else pos
    one = torch.ones_like(a)
    if act is None:
        return one
    if act == "Relu":
        return pos.to(a.dtype)
    if act == "Sigmoid":
        return a * (1 - a)
    if act == "Tanh":
        return 1 - a * a
    if act == "Elu":
        return torch.where(pos, one, a + 1)
    if act == "Selu":
        return torch.where(pos, lam * one, a + lam * al)
    if act == "Softplus":
        return torch.sigmoid(a) if bug.get("softplus_sigmoid") else -torch.expm1(-a)
    if act == "Softsign":
        return (1 - a.abs()) ** 2
    if act == "LeakyRelu":
        return torch.where(pos, one, bug.get("leaky", alpha) * one)
    if act == "Relu6":
        top = a >= 6 if top is None else top
        return (pos & ~top).to(a.dtype) if not bug.get("relu6_top") else pos.to(a.dtype)
    raise KeyError(act)


def relu6_saturation(keep=0.0):
    """(stored value of a saturated ReLU6 unit, the pre-activation from which on it is stored so) behind a dropout of keep
    probability ``keep`` (0: none): bf16(6 * (1 / keep)) with both products in fp32, as the forward epilogue computes it"""
    ik = np.float32(1.0) / np.float32(keep) if keep else np.float32(1.0)
    sat = float(_bf16(torch.tensor(float(np.float32(6.0) * ik), dtype=torch.float64)))
    half = 2.0 ** (np.frexp(sat * (1 - 2 ** -20))[1] - 1 - 8)   # half the bf16 step just below sat
    return sat, (sat - half) / float(ik)


# ------------------------------------------------------------------------------------------------------------------
# graphs
# ------------------------------------------------------------------------------------------------------------------
def _leaky(t):
    return tf.nn.leaky_relu(t, alpha=0.1)


def act_mlp():
    """one hidden layer per new activation, softmax-CE"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    h = x
    for units, act in ((64, tf.nn.elu), (48, tf.nn.selu), (40, tf.nn.softplus), (32, tf.nn.softsign), (24, _leaky), (16, tf.nn.relu6)):
        h = tf.layers.dense(h, units, activation=act)
    logits = tf.layers.dense(h, 10)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


def act_mse():
    """regression through a softsign layer to an ELU output: the MSE head differentiates an extended activation"""
    x = tf.placeholder(tf.float32, shape=[None, 20], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 5], name="y")
    h = tf.layers.dense(x, 16, activation=tf.nn.softsign)
    out = tf.layers.dense(h, 5, activation=tf.nn.elu, name="out")
    return tf.losses.mean_squared_error(y, out)


def act_cnn():
    """each new activation on a conv: with a 2x2 pool after it (ELU, softsign), with a general 3x3/2 pool (softplus) and
    with none (SELU, leaky ReLU, ReLU6)"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    h = tf.reshape(x, shape=[-1, 28, 28, 1])
    h = tf.layers.max_pooling2d(tf.layers.conv2d(h, 8, 3, padding="same", activation=tf.nn.elu), 2, 2)              # 14
    h = tf.layers.conv2d(h, 16, 3, padding="same", activation=tf.nn.selu)                                           # 14
    h = tf.layers.max_pooling2d(tf.layers.conv2d(h, 16, 3, strides=2, padding="same", activation=tf.nn.softplus), 3, 2, padding="same")  # 4
    h = tf.layers.max_pooling2d(tf.layers.conv2d(h, 16, 3, padding="same", activation=tf.nn.softsign), 2, 2)        # 2
    h = tf.layers.conv2d(h, 16, 3, padding="same", activation=_leaky)
    h = tf.layers.conv2d(h, 16, 3, padding="same", activation=tf.nn.relu6)
    logits = tf.layers.dense(tf.layers.flatten(h), 10)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


def act_drop():
    """dropout after an ELU, a SELU and a ReLU6 layer; the ReLU6 dropout's keep 0.9 makes 6 / keep inexact in bf16"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    h = tf.nn.dropout(tf.layers.dense(x, 128, activation=tf.nn.elu), keep_prob=0.5)
    h = tf.nn.dropout(tf.layers.dense(h, 64, activation=tf.nn.selu), keep_prob=0.8)
    h = tf.nn.dropout(tf.layers.dense(h, 32, activation=tf.nn.relu6), keep_prob=0.9)
    logits = tf.layers.dense(h, 10)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


# name -> (graph function, label kind: one-hot classes, regression targets, or None for an auto-encoder)
GRAPHS = {"act_mlp": (act_mlp, "onehot"), "act_mse": (act_mse, "regress"), "act_cnn": (act_cnn, "onehot"),
          "act_drop": (act_drop, "onehot"), "selu_dnn": (zoo.selu_dnn, "onehot"), "leaky_cnn": (zoo.leaky_cnn, "onehot"),
          "softplus_autoencoder": (zoo.softplus_autoencoder, None)}
CNN_GRAPHS = ("act_cnn", "leaky_cnn")

# Per graph: (relative Frobenius error, max-abs error / max|ref|) of every gradient of the GPU step against the
# bf16-emulating oracle, as test_step_gradients.TOL: about 3x the worst error tests/test_gpu_activations.py measured on
# an H100 80GB HBM3 (700 W power limit) over all plan variants and batch sizes, and never below 1e-5.
TOL = {                                   # measured
    "act_mlp": (2.5e-5, 7e-5),            # 7.2e-6, 2.3e-5
    "act_mse": (1e-5, 1e-5),              # 1.4e-7, 2.0e-7
    "act_cnn": (2.2e-3, 2e-3),            # 7.3e-4, 6.3e-4
    "act_drop": (6e-4, 1.6e-3),           # 1.9e-4, 5.2e-4 (run to run: 1.6e-7 to 1.9e-4)
    "selu_dnn": (6e-5, 1.5e-4),           # 7.7e-6, 2.7e-5
    "leaky_cnn": (2e-3, 2.7e-3),          # 6.3e-4, 8.7e-4
    "softplus_autoencoder": (5e-4, 2e-3),  # 1.7e-4, 6.4e-4
}
LOSS_TOL = 5e-5                           # relative; measured 1.9e-5 (a forward plan)
FWD_TOL = (1e-3, 4e-3)

_CACHE = {}


def act_model(name):
    """(GraphIR, LayerPlan, label tensor name or None, graph JSON)"""
    if name not in _CACHE:
        fn, kind = GRAPHS[name]
        graph = build_graph(fn)
        ir = GraphIR.from_metagraph(graph)
        label = "y:0" if kind else None
        _CACHE[name] = (ir, compile_graph(ir, "x:0", label), label, graph)
    return _CACHE[name]


def act_data(name, n, seed):
    lp = act_model(name)[1]
    kind = GRAPHS[name][1]
    rng = np.random.default_rng(seed)
    X = rng.random((n, lp.input_dim), dtype=np.float32)
    if kind == "onehot":
        return X, np.eye(lp.label_dim, dtype=np.float32)[rng.integers(0, lp.label_dim, n)]
    if kind == "regress":
        return X, rng.random((n, lp.label_dim), dtype=np.float32)
    return X, None


def act_weights(name, seed=1, scale=None):
    """the graph's initializers with small non-zero biases; ``scale``: {kernel variable: factor}"""
    ir = act_model(name)[0]
    rng = np.random.default_rng(seed + 100)
    ws = [w if w.ndim > 1 else (0.05 * rng.standard_normal(w.shape)).astype(np.float32) for w in GraphProgram(ir).init_weights(seed=seed)]
    for k, (v, w) in enumerate(zip(act_model(name)[1].var_order, ws)):
        if scale and v in scale:
            ws[k] = (w * scale[v]).astype(np.float32)
    return ws


# ------------------------------------------------------------------------------------------------------------------
# the float64 oracle
# ------------------------------------------------------------------------------------------------------------------
def act_forward(lp, weights, X, Y, emulate_bf16, argmax=None, record=None, drop_mask=None, device=torch.device("cpu"), bug=None):
    """float64 forward pass of the layer plan (test_step_gradients._forward for these networks).  Returns (loss, network
    output, parameter leaves, pools).  ``record``: {dense / conv layer with a jump activation: the step's stored output},
    from which the branch of act' is taken (checked to disagree with the oracle's own only where the pre-activation is
    zero, or 6, up to the fp32 accumulation error); ``drop_mask``: {dropout layer: kept units}; ``bug``: see act_value.
    ``record`` may hold the stored output of any dense / conv layer but the last: the oracle then carries the step's value
    forward, after checking that it is the oracle's own up to one bf16 rounding step (a value near a rounding tie - SELU's
    lambda puts many near one - is rounded either way by fp32 and float64; at B = 7 one such element moves the loss by 1e-4)."""
    assert fused_first_conv(lp) is None, "the fused first conv takes only ReLU / sigmoid / tanh"
    argmax, record, drop_mask = argmax or {}, record or {}, drop_mask or {}
    em = emulate_bf16
    bf = (lambda t: t + (_bf16(t) - t).detach()) if em else (lambda t: t)
    rg = _RG.apply if em else (lambda t: t)

    def store(z, l, i, mag):
        keep = l.dropout_keep
        kept = None
        if keep:
            kept = torch.as_tensor(np.asarray(drop_mask[i]), device=z.device).to(z.dtype)
        a = act_value(z, l.act, l.act_alpha, bug)
        if not em:
            return a if kept is None else a / keep * kept
        with torch.no_grad():
            zd = z.detach()
            a_st = _bf16(a.detach() if kept is None else a.detach() * kept / keep)
            a_d = a_st * keep if kept is not None else a_st               # the kernel takes act' at a * keep
            pos = top = None
            if i in record:
                step = record[i].to(device=z.device, dtype=torch.float64).reshape(zd.shape)
                big = torch.maximum(step.abs(), a_st.abs())
                # one bf16 rounding, plus the fp32 accumulation error of z (well below 1e-4 x its sum of |terms|)
                slack = torch.ldexp(torch.ones_like(big), torch.frexp(big)[1] - 8) + 1e-4 * mag / (keep or 1.0)
                assert bool(((step - a_st).abs() <= slack).all()), f"layer {i}: the step stored a value beyond one rounding of the oracle's"
                a_st = step
                a_d = a_st * keep if kept is not None else a_st
            if l.act == "Relu6":
                # saturation in stored units: a saturated unit holds bf16(6 / keep) (6 without a dropout), and z saturates
                # from the bf16 rounding boundary below it on
                sat, zb = relu6_saturation(keep)
                top = a_st >= sat
                if i in record:
                    live = kept.bool() if kept is not None else torch.ones_like(top)
                    off = (top != (zd >= zb)) & live
                    ratio = float(((zd[off] - zb).abs() / mag[off]).max()) if bool(off.any()) else 0.0
                    assert ratio <= 1e-3, f"layer {i}: the step's ReLU6 saturation disagrees where |z - 6| = {ratio:.1e} x sum|terms|"
            if i in record and l.act in JUMP_ACTS:
                pos = step > 0
                live = kept.bool() if kept is not None else torch.ones_like(pos)
                off = (pos != (zd > 0)) & live
                ratio = float((zd[off].abs() / mag[off]).max()) if bool(off.any()) else 0.0
                assert ratio <= 1e-3, f"layer {i}: the step's branch disagrees where |z| = {ratio:.1e} x its sum of |terms|"
            d = act_deriv(a_d, l.act, l.act_alpha, pos, top, bug)
            if kept is not None:
                d = d * kept / keep
                d = torch.where(a_st != 0, d, torch.zeros_like(d))
        return a_st + (z - zd) * d                                   # forward: the stored value; backward: d

    def magnitude(h, w, b, l):
        if not em:
            return None
        with torch.no_grad():
            m = _conv(h.abs(), w.abs(), l, lambda t: t) if l.kind == "conv" else h.abs() @ w.abs()
            return (m + b.abs() if b is not None else m).detach()

    pos_of = {n: k for k, n in enumerate(lp.var_order)}
    params = [torch.tensor(np.asarray(w), dtype=torch.float64, device=device, requires_grad=True) for w in weights]
    x = torch.as_tensor(np.asarray(X), dtype=torch.float64, device=device)
    B = x.shape[0]
    last = max(i for i, l in enumerate(lp.layers) if l.kind == "dense")
    h = bf(x)
    pools = {}
    for i, l in enumerate(lp.layers):
        if l.kind == "reshape":
            h = h.reshape(B, *l.out_shape) if len(l.out_shape) == 3 else rg(h.reshape(B, -1))
            continue
        if l.kind == "pool":
            idx = argmax.get(i)
            idx = _pool_argmax(h.detach(), l) if idx is None else idx
            pools[i] = (h.detach(), idx)
            h = _pool_gather(h, l, idx)
            continue
        w = bf(params[pos_of[l.kernel]])
        b = params[pos_of[l.bias]] if l.bias else None
        if l.kind == "conv":
            z = rg(_conv(h, w, l, rg))
            h = store(z + b if b is not None else z, l, i, magnitude(h, w, b, l))
            continue
        z = rg(h @ w)
        if b is not None:
            z = z + b
        if i != last:
            h = store(z, l, i, magnitude(h, w, b, l))
            continue
        if lp.loss == "softmax_xent":
            out = z
            yt = torch.as_tensor(np.asarray(Y), dtype=torch.float64, device=device)
            loss = -(yt * torch.log_softmax(z, 1)).sum(1).mean()
        else:
            out = act_value(z, l.act, l.act_alpha, bug)              # the MSE head works on the fp32 activation
            t = x if lp.target_is_input else torch.as_tensor(np.asarray(Y), dtype=torch.float64, device=device)
            loss = ((out - t) ** 2).mean()
        return loss, out, params, pools
    raise AssertionError("no dense layer")


class _RG(torch.autograd.Function):
    """identity forward; the gradient passing back is rounded to bf16 (a stored dz / dgrad / col2im output)"""

    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return _bf16(g)


def act_oracle(lp, weights, X, Y, emulate_bf16, **kw):
    loss, _, params, _ = act_forward(lp, weights, X, Y, emulate_bf16, **kw)
    return float(loss.detach()), _grads(loss, params)


# ------------------------------------------------------------------------------------------------------------------
# compiler
# ------------------------------------------------------------------------------------------------------------------
_TF_ACTS = {"Elu": tf.nn.elu, "Selu": tf.nn.selu, "Softplus": tf.nn.softplus, "Softsign": tf.nn.softsign,
            "LeakyRelu": lambda t: tf.nn.leaky_relu(t, alpha=0.3), "Relu6": tf.nn.relu6}


def _compile(fn, label="y:0"):
    return compile_graph(GraphIR.from_metagraph(build_graph(fn)), "x:0", label)


@pytest.mark.parametrize("spelling", ["layers_dense", "nn_op", "layers_conv2d"])
@pytest.mark.parametrize("act", NEW_ACTS)
def test_compiler_accepts_the_new_activations(act, spelling):
    def fn():
        x = tf.placeholder(tf.float32, shape=[None, 64], name="x")
        y = tf.placeholder(tf.float32, shape=[None, 4], name="y")
        if spelling == "layers_conv2d":
            h = tf.layers.conv2d(tf.reshape(x, shape=[-1, 8, 8, 1]), 8, 3, activation=_TF_ACTS[act])
            h = tf.layers.flatten(h)
        elif spelling == "layers_dense":
            h = tf.layers.dense(x, 16, activation=_TF_ACTS[act])
        else:
            h = _TF_ACTS[act](tf.layers.dense(x, 16))
        return tf.losses.softmax_cross_entropy(y, tf.layers.dense(h, 4))

    lp = _compile(fn)
    l = next(l for l in lp.layers if l.kind in ("dense", "conv"))
    assert l.kind == ("conv" if spelling == "layers_conv2d" else "dense")
    assert l.act == act and ACT_IDS[act] >= 4
    assert l.act_alpha == pytest.approx(0.3 if act == "LeakyRelu" else 0.0)
    check_grammar(lp)


def test_leaky_relu_alpha_defaults_and_zero():
    def default():
        x = tf.placeholder(tf.float32, shape=[None, 8], name="x")
        return tf.losses.mean_squared_error(x, tf.layers.dense(tf.layers.dense(x, 4, activation=tf.nn.leaky_relu), 8))

    def zero():
        x = tf.placeholder(tf.float32, shape=[None, 8], name="x")
        h = tf.nn.leaky_relu(tf.layers.dense(x, 4), alpha=0.0)
        return tf.losses.mean_squared_error(x, tf.layers.dense(h, 8))

    l = _compile(default, None).layers[0]
    assert (l.act, l.act_alpha) == ("LeakyRelu", pytest.approx(0.2))
    l = _compile(zero, None).layers[0]
    assert (l.act, l.act_alpha) == ("Relu", 0.0)


def _maximum_graph(alpha, order, alpha_node=None):
    def fn():
        x = tf.placeholder(tf.float32, shape=[None, 8], name="x")
        z = tf.layers.dense(x, 4)
        a = alpha_node() if alpha_node else tf.constant(np.float32(alpha))
        mul = tf.multiply(a, z) if order[0] == "a" else tf.multiply(z, a)
        h = tf.maximum(mul, z) if order[1] == "m" else tf.maximum(z, mul)
        return tf.losses.mean_squared_error(x, tf.layers.dense(h, 8))
    return fn


@pytest.mark.parametrize("order", ["am", "az", "zm", "zz"])
def test_compiler_accepts_the_maximum_spelling_of_leaky_relu(order):
    """TF 1.4-1.12: tf.nn.leaky_relu is Maximum(Mul(alpha, x), x); both ops' operands in either order"""
    l = _compile(_maximum_graph(0.1, order), None).layers[0]
    assert l.act == "LeakyRelu" and l.act_alpha == pytest.approx(0.1)
    assert _compile(_maximum_graph(0.0, order), None).layers[0].act == "Relu"


def _negative_alpha():
    x = tf.placeholder(tf.float32, shape=[None, 8], name="x")
    h = tf.nn.leaky_relu(tf.layers.dense(x, 4), alpha=-0.1)
    return tf.losses.mean_squared_error(x, tf.layers.dense(h, 8))


def _swish():
    x = tf.placeholder(tf.float32, shape=[None, 8], name="x")
    z = tf.layers.dense(x, 4)
    return tf.losses.mean_squared_error(x, tf.layers.dense(tf.multiply(z, tf.nn.sigmoid(z)), 8))


def _placeholder_alpha():
    return tf.placeholder(tf.float32, shape=[], name="slope")


@pytest.mark.parametrize("fn,match", [(_negative_alpha, "negative alpha"), (_maximum_graph(1.5, "am"), "outside"),
                                      (_maximum_graph(None, "zm", _placeholder_alpha), "not a constant"),
                                      (_swish, "not a function of its output")])
def test_compiler_rejects_uncovered_activations(fn, match):
    with pytest.raises(UnsupportedGraph, match=match):
        _compile(fn, None)


@pytest.mark.parametrize("act", NEW_ACTS)
def test_fused_first_conv_keeps_its_activations(act):
    """a first conv with a new activation runs the lowered im2col + GEMM path"""
    def fn(a):
        def g():
            x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
            y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
            h = tf.layers.max_pooling2d(tf.layers.conv2d(tf.reshape(x, shape=[-1, 28, 28, 1]), 32, 5, activation=a), 2, 2)
            return tf.losses.softmax_cross_entropy(y, tf.layers.dense(tf.layers.flatten(h), 10))
        return g

    assert fused_first_conv(_compile(fn(tf.nn.relu))) == 1
    assert fused_first_conv(_compile(fn(_TF_ACTS[act]))) is None


def test_fused_first_conv_fits_its_weight_gradient():
    """the planner keeps a first conv on the direct kernels only where the weight gradient's launcher takes it too: the
    padded image plus the 256 x (K + 1) fp32 group reduction within 96 KiB.  These three images fit the 64 KiB image
    rule but need 99,328, 101,376 and 103,424 B; the 62 x 62 x 3 one needs 96,304 B."""
    from conv_ref import first_conv_plan, wgrad_smem

    for h, cin, k, cout, want in [(64, 3, 4, 16, False), (112, 1, 7, 16, False), (48, 4, 4, 16, False), (62, 3, 4, 8, True),
                                  (28, 1, 5, 32, True)]:
        lp = first_conv_plan(h, h, cin, k, cout, "valid")[1]
        oh = lp.layers[1].out_shape[0]
        assert (wgrad_smem(k, k, cin, cout, oh, oh)[0] <= 96 * 1024) == want, (h, cin, k)
        assert (fused_first_conv(lp) == 1) == want, (h, cin, k)
    for name in ("cnn", "cnn_same"):
        assert fused_first_conv(compile_graph(GraphIR.from_metagraph(zoo.build(name)), "x:0", "y:0")) == 1, name


def test_act_arg_packs_the_leaky_slope():
    lp = act_model("leaky_cnn")[1]
    conv = lp.layers[1]
    assert act_arg(conv) == 8 | (struct.unpack("<I", struct.pack("<f", 0.1))[0] << 32)
    dense = [l for l in lp.layers if l.kind == "dense"]
    assert [act_arg(l) for l in dense] == [4, 0]


def test_cross_entropy_still_needs_raw_logits():
    def fn():
        x = tf.placeholder(tf.float32, shape=[None, 8], name="x")
        y = tf.placeholder(tf.float32, shape=[None, 4], name="y")
        return tf.losses.softmax_cross_entropy(y, tf.layers.dense(x, 4, activation=tf.nn.elu))

    with pytest.raises(UnsupportedGraph, match="raw logits"):
        _compile(fn)


# ------------------------------------------------------------------------------------------------------------------
# the oracle and the tolerances
# ------------------------------------------------------------------------------------------------------------------
def _feed(name, X, Y):
    _, lp, label, _ = act_model(name)
    return {"x:0": X, **({label: Y} if label else {})}


@pytest.mark.parametrize("name", [n for n in GRAPHS if n != "act_drop"])
def test_oracle_matches_interpreter(name):
    ir, lp, _, _ = act_model(name)
    X, Y = act_data(name, 7, seed=3)
    w = act_weights(name)
    l_int, g_int = GraphProgram(ir).loss_and_grads(_feed(name, X, Y), w)
    l_ora, g_ora = act_oracle(lp, w, X, Y, False)
    assert abs(l_ora - l_int) <= 1e-5 * max(1.0, abs(l_int)), (l_ora, l_int)
    _assert_grads(f"{name} exact oracle vs interpreter", lp.var_order, g_ora, [g.numpy() for g in g_int], (1e-4, 1e-4))
    l_em, _ = act_oracle(lp, w, X, Y, True)
    assert abs(l_em - l_ora) <= 2e-2 * max(1.0, abs(l_ora)), (l_em, l_ora)


# Weights that push each layer of act_mlp into the part of its activation a bug would show in: ReLU6 into saturation,
# the leaky ReLU / SELU / softplus layers onto both signs
MLP_SCALE = {"dense_5/kernel": 30.0, "dense_4/kernel": 6.0, "dense_1/kernel": 3.0, "dense_2/kernel": 3.0}


@pytest.mark.parametrize("B", [7, 129])
@pytest.mark.parametrize("what,bug", [("a SELU lambda 1 % off", dict(selu=(SELU[0] * 1.01, SELU[1]))),
                                      ("a SELU alpha 1 % off", dict(selu=(SELU[0], SELU[1] * 1.01))),
                                      ("the leaky ReLU's default slope", dict(leaky=0.2)),
                                      ("softplus' taken as sigmoid(a)", dict(softplus_sigmoid=True)),
                                      ("ReLU6 passing gradient at a = 6", dict(relu6_top=True))])
def test_tolerances_reject_plausible_activation_bugs(what, bug, B):
    name = "act_mlp"
    lp = act_model(name)[1]
    X, Y = act_data(name, B, seed=11)
    w = act_weights(name, scale=MLP_SCALE)
    _, ref = act_oracle(lp, w, X, Y, True)
    assert not _rejects(ref, ref, TOL[name])
    _, got = act_oracle(lp, w, X, Y, True, bug=bug)
    assert _rejects(got, ref, TOL[name]), f"B={B}: the tolerance {TOL[name]} accepts the gradient with {what}"


# act_drop's ReLU6 layer (behind the keep-0.9 dropout) scaled into saturation
DROP_SCALE = {"dense_2/kernel": 10.0}


def random_drop_masks(lp, B, seed):
    """{dropout layer: kept units}: any mask does for the oracle alone"""
    rng = np.random.default_rng(seed)
    return {i: rng.random((B, l.out_shape[0])) < l.dropout_keep for i, l in enumerate(lp.layers) if l.kind == "dense" and l.dropout_keep}


@pytest.mark.parametrize("B", [7, 129])
def test_tolerances_reject_relu6_gradient_at_saturation_behind_dropout(B):
    """behind a keep-0.9 dropout a saturated unit stores bf16(6 / 0.9) = 6.65625, and 6.65625 * 0.9 < 6: a backward pass
    that takes saturation from a * keep passes gradient through every saturated unit"""
    name = "act_drop"
    lp = act_model(name)[1]
    X, Y = act_data(name, B, seed=11)
    w = act_weights(name, scale=DROP_SCALE)
    masks = random_drop_masks(lp, B, seed=B)
    sat, _ = relu6_saturation(0.9)
    assert sat == 6.65625 and sat * 0.9 < 6
    _, ref = act_oracle(lp, w, X, Y, True, drop_mask=masks)
    assert not _rejects(ref, ref, TOL[name])
    _, got = act_oracle(lp, w, X, Y, True, drop_mask=masks, bug=dict(relu6_top=True))
    assert _rejects(got, ref, TOL[name]), f"B={B}: the tolerance {TOL[name]} accepts ReLU6 gradient through saturated units"


def test_relu6_saturation_in_stored_units():
    """the stored saturation value and the pre-activation boundary of relu6_saturation, against bf16(z * (1 / keep))"""
    def stored(z, ik):
        return float(_bf16(torch.tensor(float(np.float32(z) * ik), dtype=torch.float64)))

    assert relu6_saturation() == (6.0, 5.984375)
    for keep in (0.5, 0.6, 0.7, 0.75, 0.8, 0.9, 0.95):
        sat, zb = relu6_saturation(keep)
        ik = np.float32(1) / np.float32(keep)
        assert stored(6.0, ik) == sat and stored(zb + 1e-3, ik) == sat and stored(zb - 1e-3, ik) < sat, (keep, sat, zb)


def test_mlp_scale_exercises_relu6_saturation():
    lp = act_model("act_mlp")[1]
    X, Y = act_data("act_mlp", 129, seed=11)
    w = act_weights("act_mlp", scale=MLP_SCALE)
    with torch.no_grad():
        params = [torch.tensor(a, dtype=torch.float64) for a in w]
        pos = {n: k for k, n in enumerate(lp.var_order)}
        h = torch.tensor(X, dtype=torch.float64)
        for l in lp.layers[:-1]:
            h = act_value(h @ params[pos[l.kernel]] + params[pos[l.bias]], l.act, l.act_alpha)
    sat = float((h >= 6).double().mean())
    assert 0.05 < sat < 0.95, sat


# ------------------------------------------------------------------------------------------------------------------
# build artifacts
# ------------------------------------------------------------------------------------------------------------------
@needs_binary_utils
def test_ext_kernel_instances_have_no_stack_frame():
    use = res_usage()
    # the EXT instances of the GEMM kernels: the K-major generic kernel, the FWD / LOSS / DGRAD variants, the pair kernel
    gemms = [f"sf::sf_gemm_kernel<{bn}, false, 0, true, false>" for bn in (32, 64, 128, 256)] + ["sf::sf_gemm_pair_kernel<true>"]
    gemms += [f"sf::sf_gemm_kernel<{bn}, false, {epi}, true, false>" for bn in (32, 64) for epi in (1, 2, 3)]
    others = ["sf::maxpool_bwd_ext_kernel", "sf::maxpool_gen_bwd_ext_kernel", "sf::act_bwd_bias_ext_kernel", "sf::mse_ext_loss_kernel"]
    missing = [k for k in gemms + others if k not in use]
    assert not missing, (missing, sorted(use))
    spilled = {k: use[k] for k in gemms + others if use[k][1] != 0}
    assert not spilled, f"kernels with a local-memory stack frame (REG, STACK): {spilled}"
    # the EXT instances run under the GEMMs' launch bounds (384 threads, one CTA per SM): no more registers than the
    # instances without the extended activations (EXT = false, PEN = false)
    bound = max([r for (_, _, _, ext, pen), (r, _) in gemm_instances(use).items() if not ext and not pen] +
                [use["sf::sf_gemm_pair_kernel<false>"][0]])
    assert all(use[k][0] <= bound for k in gemms), {k: use[k] for k in gemms}
