"""Dropout on conv and max-pool outputs in the compiled CNN step: the compiler's placements and refusals, the fused
first conv turned off under a dropout, and a float64 oracle of image dropout checked against the interpreter and shown to
reject plausible mask and backward faults.

Mask key (one rule for kernels, oracle and docs): an image [B, OH, OW, C] is the matrix [B * OH * OW, C] its conv GEMM
writes, so the host mask of an image dropout on layer i is ``dropout_mask(B * OH * OW, C, keep, seed, i, ctr)``; a dropout
on the flatten of an image layer is that layer's dropout.
"""
import numpy as np
import pytest
import torch

import test_step_gradients as sg
from sparkflow_b200.graph import tfcompat as tf
from sparkflow_b200.graph.executor import GraphProgram
from sparkflow_b200.graph.ir import GraphIR
from sparkflow_b200.graph_utils import build_graph
from sparkflow_b200.models import zoo
from sparkflow_b200.models.compiler import UnsupportedGraph, compile_graph
from sparkflow_b200.parallel.plan_builder import check_grammar, fused_first_conv
from dropout_ref import dropout_mask
from kernel_usage import needs_binary_utils, res_usage

NAMES = ("dropout_cnn", "conv_dropout_cnn")
# (relative Frobenius error, max-abs error / max|ref|) of every gradient of the step against the bf16-emulating oracle
# (tests/test_gpu_conv_dropout.py), about 3x the worst error measured on an H100 80GB HBM3 (700 W power limit) over the
# plan variants, batch sizes and feeds there (the run-to-run spread of the atomically accumulated bias and split-K
# gradients moves it by up to 3x between runs)
TOL = {"dropout_cnn": (5.5e-3, 6e-3),             # measured 1.8e-3, 2.0e-3
       "conv_dropout_cnn": (1.5e-2, 1.4e-2)}     # measured 4.9e-3, 4.5e-3
LOSS_TOL = 7e-5                                  # relative; measured 2.1e-5

_CACHE = {}


def model(name):
    """(GraphIR, LayerPlan) of a zoo model"""
    if name not in _CACHE:
        ir = GraphIR.from_metagraph(zoo.build(name))
        _CACHE[name] = (ir, compile_graph(ir, "x:0", "y:0"))
    return _CACHE[name]


def data(name, n, seed):
    _, lp = model(name)
    rng = np.random.default_rng(seed)
    X = rng.random((n, lp.input_dim), dtype=np.float32)
    Y = np.eye(lp.label_dim, dtype=np.float32)[rng.integers(0, lp.label_dim, n)]
    return X, Y


def weights(name, seed=1):
    ir = model(name)[0]
    rng = np.random.default_rng(seed + 100)
    return [w if w.ndim > 1 else (0.05 * rng.standard_normal(w.shape)).astype(np.float32)
            for w in GraphProgram(ir).init_weights(seed=seed)]


def host_masks(lp, B, seed, ctr, streams=None):
    """{layer with a dropout: kept units}: [B, N] of a dense layer, [B * OH * OW, C] of a conv or pool layer"""
    streams = streams or {}
    out = {}
    for i, l in enumerate(lp.layers):
        if not l.dropout_keep:
            continue
        rows, cols = (B, l.out_shape[0]) if l.kind == "dense" else (B * l.out_shape[0] * l.out_shape[1], l.out_shape[2])
        out[i] = dropout_mask(rows, cols, np.float32(l.dropout_keep), seed, streams.get(i, i), ctr)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# the float64 oracle
# ----------------------------------------------------------------------------------------------------------------------
BUGS = ("per_sample_key", "no_backward_mask", "no_backward_scale", "before_pool")


class _MaskFwdOnly(torch.autograd.Function):
    """x * mask / keep forward, x / keep back: a mask that is not applied in the backward pass"""

    @staticmethod
    def forward(ctx, x, mask, keep):
        ctx.keep = keep
        return x * mask / keep

    @staticmethod
    def backward(ctx, g):
        return g / ctx.keep, None, None


class _StoreDropFault(torch.autograd.Function):
    """sg._StoreDrop (without a recorded ReLU mask) whose backward forgets the mask ('no_backward_mask') or the 1 / keep
    ('no_backward_scale')"""

    @staticmethod
    def forward(ctx, z, act, keep, mask, fault):
        a = sg._bf16(sg._ACT[act](z) * mask / keep)
        if fault == "no_backward_mask":
            d = sg._dact(sg._bf16(sg._ACT[act](z)), act) / keep
        else:
            d = sg._dact(a * keep, act) * mask
        ctx.save_for_backward(d)
        return a

    @staticmethod
    def backward(ctx, g):
        (d,) = ctx.saved_tensors
        return g * d, None, None, None, None


def forward(lp, w_np, X, Y, em, argmax=None, relu_mask=None, drop_mask=None, bug=None, bug_key=(0, 0), device=sg.DEV):
    """float64 forward pass of a CNN layer plan with dropouts on dense, conv and pool outputs; returns (loss, logits,
    parameter leaves, pools) with pools = {pool layer: (activation it pooled, winner index)}.  ``drop_mask``: host_masks
    of every dropout layer; ``em``: the step's bf16 stores (the backward of a stored dropout output as sg._StoreDrop).
    ``argmax`` / ``relu_mask``: the step's pool winners and active ReLU units (see sg.oracle).  ``bug``: one of BUGS,
    a fault the step could have, in every image dropout (and in no dense one); a faulty key draws its masks under
    ``bug_key`` = (seed, counter)."""
    assert fused_first_conv(lp) is None or not em, "the oracle does not model the fused first conv"
    argmax, relu_mask, drop_mask = argmax or {}, relu_mask or {}, drop_mask or {}
    bf = (lambda t: t + (sg._bf16(t) - t).detach()) if em else (lambda t: t)
    rg = sg._RoundGrad.apply if em else (lambda t: t)
    pos = {n: k for k, n in enumerate(lp.var_order)}
    params = [torch.tensor(np.asarray(v), dtype=torch.float64, device=device, requires_grad=True) for v in w_np]
    x = torch.as_tensor(np.asarray(X), dtype=torch.float64, device=device)
    B = x.shape[0]
    last = max(i for i, l in enumerate(lp.layers) if l.kind == "dense")

    def kept_of(i, shape):
        m = np.asarray(drop_mask[i])
        if bug == "per_sample_key" and lp.layers[i].kind != "dense":
            l = lp.layers[i]
            m = dropout_mask(B, l.out_features, np.float32(l.dropout_keep), bug_key[0], i, bug_key[1])
        return torch.as_tensor(m.reshape(shape), device=device).to(torch.float64)

    def store(z, l, i, mag):
        keep = l.dropout_keep
        mask = relu_mask.get(i) if l.act == "Relu" else None
        kept = kept_of(i, z.shape) if keep else None
        if mask is not None:
            zd, off = z.detach(), mask != (z.detach() > 0)
            if kept is not None:
                off &= kept.bool()
            ratio = float((zd[off].abs() / mag[off]).max()) if bool(off.any()) else 0.0
            assert ratio <= 1e-3, f"layer {i}: the step's ReLU mask disagrees where |z| = {ratio:.1e} x its sum of |terms|"
        if not keep:
            return sg._StoreAct.apply(z, l.act, mask) if em else sg._ACT[l.act](z)
        if not em:
            return sg._ACT[l.act](z) / keep * kept
        if bug in ("no_backward_mask", "no_backward_scale") and l.kind == "conv":
            return _StoreDropFault.apply(z, l.act, keep, kept, bug)
        return sg._StoreDrop.apply(z, l.act, keep, kept, mask)

    h = bf(x)
    pools = {}
    loss = out = None
    for i, l in enumerate(lp.layers):
        if l.kind == "reshape":
            h = h.reshape(B, *l.out_shape) if len(l.out_shape) == 3 else rg(h.reshape(B, -1))
            continue
        if l.kind == "pool":
            keep = l.dropout_keep
            if keep and bug == "before_pool":
                H, W, C = l.in_shape
                m = dropout_mask(B * H * W, C, np.float32(keep), bug_key[0], i, bug_key[1])
                h = bf(h * torch.as_tensor(m.reshape(h.shape), device=device).to(h.dtype) / keep)
            idx = argmax.get(i)
            idx = sg._pool_argmax(h.detach(), l) if idx is None else idx
            pools[i] = (h.detach(), idx)
            h = sg._pool_gather(h, l, idx)
            if keep and bug != "before_pool":
                m = kept_of(i, h.shape)
                if bug == "no_backward_mask":
                    h = bf(_MaskFwdOnly.apply(h, m, keep))
                elif bug == "no_backward_scale":
                    h = bf(h * m + (h * m / keep - h * m).detach())
                else:
                    h = bf(h * m / keep)
            continue
        w = bf(params[pos[l.kernel]])
        b = params[pos[l.bias]] if l.bias else None
        if l.kind == "conv":
            z = rg(sg._conv(h, w, l, rg))
            z = z + b if b is not None else z
            mag = None
            if em:
                with torch.no_grad():
                    mag = sg._conv(h.abs(), w.abs(), l, lambda t: t) + (b.abs() if b is not None else 0)
            h = store(z, l, i, mag)
            continue
        z = rg(h @ w)
        z = z + b if b is not None else z
        if i != last:
            mag = None
            if em:
                with torch.no_grad():
                    mag = h.abs() @ w.abs() + (b.abs() if b is not None else 0)
            h = store(z, l, i, mag)
            continue
        out = z
        yt = torch.as_tensor(np.asarray(Y), dtype=torch.float64, device=device)
        loss = -(yt * torch.log_softmax(z, 1)).sum(1).mean()
        break
    return loss, out, params, pools


def oracle(lp, w, X, Y, em, drop_mask, bug=None, **kw):
    loss, _, params, _ = forward(lp, w, X, Y, em, drop_mask=drop_mask, bug=bug, **kw)
    return float(loss.detach()), sg._grads(loss, params)


# ----------------------------------------------------------------------------------------------------------------------
# compiler
# ----------------------------------------------------------------------------------------------------------------------
def _plan(fn, output=None, need_loss=True):
    ir = GraphIR.from_metagraph(build_graph(fn))
    return ir, compile_graph(ir, "x:0", "y:0" if need_loss else None, output, need_loss=need_loss)


def _cnn(placement, spelling="nn", first=False):
    """conv 3x3x16 VALID relu -> [pool 2x2] -> conv 3x3x32 VALID tanh -> pool 2x2/2 -> flatten -> dense 10 with one dropout
    (keep 0.75) at ``placement``: conv (the tanh conv), pool, flatten, conv1 / pool1 (the first conv / its pool)"""
    def fn():
        x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
        y = tf.placeholder(tf.float32, shape=[None, 10], name="y")

        def drop(t, where):
            if where != placement:
                return t
            if spelling == "layers":
                return tf.layers.dropout(t, rate=0.25, training=True)
            if spelling == "default":
                return tf.nn.dropout(t, keep_prob=tf.placeholder_with_default(0.75, shape=[], name="kp"))
            return tf.nn.dropout(t, keep_prob=0.75)

        img = tf.reshape(x, shape=[-1, 28, 28, 1])
        c1 = drop(tf.layers.conv2d(img, 16, 3, activation=tf.nn.relu), "conv1")
        c1 = drop(tf.layers.max_pooling2d(c1, 2, 2), "pool1")
        c2 = drop(tf.layers.conv2d(c1, 32, 3, activation=tf.nn.tanh), "conv")
        p2 = drop(tf.layers.max_pooling2d(c2, 2, 2), "pool")
        logits = tf.layers.dense(drop(tf.layers.flatten(p2), "flatten"), 10, name="logits")
        tf.argmax(logits, 1, name="out")
        return tf.losses.softmax_cross_entropy(y, logits)
    return fn


def _summary(lp):
    return [(l.kind, l.out_shape, round(l.dropout_keep, 6)) for l in lp.layers]


@pytest.mark.parametrize("spelling", ["nn", "layers", "default"])
@pytest.mark.parametrize("placement,layer", [("conv", 3), ("pool", 4), ("flatten", 4), ("conv1", 1), ("pool1", 2)])
def test_compiler_attaches_image_dropouts(placement, layer, spelling):
    """every placement and spelling lands on the right layer with the right keep; a dropout after the flatten is the
    dropout of the pool below it"""
    ir, lp = _plan(_cnn(placement, spelling))
    check_grammar(lp)
    assert [i for i, l in enumerate(lp.layers) if l.dropout_keep] == [layer], _summary(lp)
    l = lp.layers[layer]
    assert abs(l.dropout_keep - 0.75) < 1e-6 and l.kind == ("conv" if placement.startswith("conv") else "pool")
    assert ir.nodes[l.tensors["dropout"].split(":")[0]].op == "Mul"
    if placement == "flatten":
        _, before = _plan(_cnn("pool", spelling))
        assert _summary(lp) == _summary(before)
    assert (fused_first_conv(lp) is None) == (placement in ("conv1", "pool1"))


def test_zoo_dropout_models_compile():
    assert _summary(model("dropout_cnn")[1]) == [
        ("reshape", (28, 28, 1), 0), ("conv", (26, 26, 32), 0), ("conv", (24, 24, 64), 0), ("pool", (12, 12, 64), 0.75),
        ("reshape", (9216,), 0), ("dense", (128,), 0.5), ("dense", (10,), 0)]
    assert _summary(model("conv_dropout_cnn")[1]) == [
        ("reshape", (28, 28, 1), 0), ("conv", (28, 28, 16), 0), ("pool", (14, 14, 16), 0.9), ("conv", (14, 14, 32), 0.8),
        ("pool", (7, 7, 32), 0), ("conv", (5, 5, 32), 0.75), ("conv", (5, 5, 16), 0.6), ("reshape", (400,), 0), ("dense", (10,), 0)]
    for name in NAMES:
        check_grammar(model(name)[1])
        assert fused_first_conv(model(name)[1]) is None


def test_fused_first_conv_is_unchanged_without_a_dropout():
    for name in ("cnn", "cnn_same"):
        lp = compile_graph(GraphIR.from_metagraph(zoo.build(name)), "x:0", "y:0")
        assert fused_first_conv(lp) == 1
    _, lp = _plan(_cnn("conv"))
    assert fused_first_conv(lp) == 1


def test_fetches_around_an_image_dropout():
    """the dropout output may be fetched; the tensor under it (pool output, conv activation, flatten) may not be a
    training graph's tfOutput"""
    _, lp = _plan(_cnn("pool"), output="dropout/mul:0", need_loss=False)
    assert lp.output.layer == 4 and lp.output.stage == "dropout"
    for placement, t in (("pool", "max_pooling2d_1/MaxPool:0"), ("conv", "conv2d_1/Tanh:0"), ("flatten", "flatten/Reshape:0")):
        with pytest.raises(UnsupportedGraph, match="pre-activation"):
            _plan(_cnn(placement), output=t)


def _conv_and_pool():
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    c = tf.nn.dropout(tf.layers.conv2d(tf.reshape(x, [-1, 28, 28, 1]), 16, 3, activation=tf.nn.relu), keep_prob=0.8)
    p = tf.nn.dropout(tf.layers.max_pooling2d(c, 2, 2), keep_prob=0.8)
    return tf.losses.softmax_cross_entropy(y, tf.layers.dense(tf.layers.flatten(p), 10))


def _on_input():
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    c = tf.layers.conv2d(tf.reshape(tf.nn.dropout(x, keep_prob=0.8), [-1, 28, 28, 1]), 16, 3)
    return tf.losses.softmax_cross_entropy(y, tf.layers.dense(tf.layers.flatten(c), 10))


def _on_input_reshape():
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    c = tf.layers.conv2d(tf.nn.dropout(tf.reshape(x, [-1, 28, 28, 1]), keep_prob=0.8), 16, 3)
    return tf.losses.softmax_cross_entropy(y, tf.layers.dense(tf.layers.flatten(c), 10))


def _on_output():
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    c = tf.layers.conv2d(tf.reshape(x, [-1, 28, 28, 1]), 16, 3)
    return tf.losses.softmax_cross_entropy(y, tf.nn.dropout(tf.layers.dense(tf.layers.flatten(c), 10), keep_prob=0.8))


def _no_default():
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    kp = tf.placeholder(tf.float32, name="keep_prob")
    c = tf.nn.dropout(tf.layers.conv2d(tf.reshape(x, [-1, 28, 28, 1]), 16, 3), keep_prob=kp)
    return tf.losses.softmax_cross_entropy(y, tf.layers.dense(tf.reshape(c, [-1, 26 * 26 * 16]), 10))


@pytest.mark.parametrize("fn,reason", [(_conv_and_pool, "both conv"), (_on_input, "input"), (_on_input_reshape, "input"),
                                       (_on_output, "network output"), (_no_default, "without a default")],
                         ids=["conv_and_pool", "input", "input_reshape", "output", "no_default"])
def test_refused_dropouts(fn, reason):
    ir = GraphIR.from_metagraph(build_graph(fn))
    with pytest.raises(UnsupportedGraph, match=reason):
        compile_graph(ir, "x:0", "y:0")


def test_spatial_dropout_is_refused():
    """a RandomUniform whose shape is not Shape(x) (noise_shape, built by hand: the builder never emits it)"""
    ir = GraphIR.from_metagraph(build_graph(_cnn("pool")))
    compile_graph(ir, "x:0", "y:0")
    ru = ir.nodes["dropout/random_uniform/RandomUniform"]
    shape_const = next(n for n in ir.nodes.values() if n.op == "Const" and n.name.endswith("Reshape/shape"))
    ru.inputs = [(shape_const.name, 0)]
    with pytest.raises(UnsupportedGraph, match="noise_shape"):
        compile_graph(ir, "x:0", "y:0")


# ----------------------------------------------------------------------------------------------------------------------
# the oracle
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_image_dropout_oracle_matches_interpreter(name):
    """The exact oracle with host masks against the interpreter running the graph's own dropout sub-graphs, each
    RandomUniform fed 0.999 where the mask keeps a unit and 0 where it drops it (floor(keep + u) is then the mask); a
    dropout on the flatten takes the mask of the layer below, reshaped to its [B, OH * OW * C] rows."""
    ir, lp = model(name)
    B = 5
    X, Y = data(name, B, seed=3)
    w = weights(name)

    def run_both(masks):
        feeds = {"x:0": X, "y:0": Y}
        for i, m in masks.items():
            feeds[sg._random_uniform_tensor(ir, lp.layers[i])] = np.where(m, 0.999, 0.0).astype(np.float32).reshape(B, -1)
        l_int, g_int = GraphProgram(ir).loss_and_grads(_shaped(ir, lp, feeds, B), w)
        l_ora, g_ora = oracle(lp, w, X, Y, False, masks)
        assert abs(l_ora - l_int) <= 1e-5 * max(1.0, abs(l_int)), (l_ora, l_int)
        sg._assert_grads(f"{name} exact oracle vs interpreter", lp.var_order, g_ora, [g.numpy() for g in g_int], (1e-4, 1e-4))
        return g_ora

    masks = host_masks(lp, B, 0x5EED, 3)
    assert len(masks) == sum(1 for l in lp.layers if l.dropout_keep) and all(0 < m.mean() < 1 for m in masks.values())
    g = run_both(masks)
    assert sg._rejects(run_both(host_masks(lp, B, 0x5EED, 4)), g, TOL[name]), "the mask does not reach the gradient"


def _shaped(ir, lp, feeds, B):
    """each fed RandomUniform in the shape of the tensor its dropout reads"""
    out = dict(feeds)
    for i, l in enumerate(lp.layers):
        t = sg._random_uniform_tensor(ir, l) if l.dropout_keep else None
        if t is None or t not in out:
            continue
        under_flatten = any(k.tensors.get("pre_dropout") for k in lp.layers[i + 1:i + 2])
        out[t] = out[t].reshape(B, -1) if (under_flatten or l.kind == "dense") else out[t].reshape(B, *l.out_shape)
    return out


@pytest.mark.parametrize("B", [5, 130])
@pytest.mark.parametrize("name", NAMES)
def test_tolerances_reject_image_dropout_bugs(name, B):
    """The step comparison rejects the oracle's gradient under each image-dropout fault: the mask keyed per sample
    [B, OH * OW * C] instead of per pixel row, a mask not applied in the backward pass, no 1 / keep in the backward pass,
    the dropout applied before the pool instead of after it (where a pool carries one).  Each fault is in the image
    dropouts only: dropout_cnn's dense dropout stays right, so the rejection comes from its pool dropout."""
    _, lp = model(name)
    X, Y = data(name, B, seed=11)
    w = weights(name)
    seed, ctr = 0x2468ACE, 7
    masks = host_masks(lp, B, seed, ctr)
    _, ref = oracle(lp, w, X, Y, True, masks)
    tol = TOL[name]
    assert not sg._rejects(ref, ref, tol)
    bugs = [b for b in BUGS if b != "before_pool" or any(l.kind == "pool" and l.dropout_keep for l in lp.layers)]
    for bug in bugs:
        # the faulty keys draw under the same seed and counter; dense dropouts stay right
        got = oracle(lp, w, X, Y, True, masks, bug=bug, bug_key=(seed, ctr))[1]
        assert sg._rejects(got, ref, tol), f"{name} B={B}: the tolerance {tol} accepts the gradient with {bug}"


@needs_binary_utils
def test_dropout_twins_keep_no_stack_frame():
    """the dropout twins of the pool and activation-gradient kernels are in the library and keep no local-memory frame"""
    use = res_usage()
    twins = {k: v for k, v in use.items() if "_drop_" in k}
    assert sorted(twins) == sorted(["sf::maxpool_drop_fwd_kernel", "sf::maxpool_gen_drop_fwd_kernel"]
                                   + [f"sf::{k}<{e}>" for k in ("maxpool_drop_bwd_kernel", "maxpool_gen_drop_bwd_kernel",
                                                                  "act_drop_bwd_bias_kernel") for e in ("false", "true")]), sorted(twins)
    assert all(v[1] == 0 for v in twins.values()), twins


def _pinned(obj):
    """name(types...) of a pybind function, an integer written int and a float float"""
    line = obj.__doc__.splitlines()[0]
    name, args = line.split("(", 1)
    types = [a.split(": ", 1)[1] for a in args.rsplit(") ->", 1)[0].split(", arg")]
    return name, tuple({"typing.SupportsInt | typing.SupportsIndex": "int", "typing.SupportsFloat | typing.SupportsIndex": "float"}
                       .get(t, t) for t in types)


_TWIN_ARGS = {   # the arguments of the direct entry points; the plan ops take the plan first and no stream
    "maxpool_drop_fwd": "in n h w c out argmax keep:f seed stream ctr",
    "maxpool_gen_drop_fwd": "in n h w c kh kw sh sw pad_top pad_left out_h out_w out argmax keep:f seed stream ctr",
    "maxpool_drop_bwd": "dout argmax n h w c act_out act pool_keep:f act_keep:f dz ld_dz dbias",
    "maxpool_gen_drop_bwd": ("dout argmax n h w c kh kw sh sw pad_top pad_left out_h out_w act_out act pool_keep:f act_keep:f dz "
                             "ld_dz dbias"),
    "act_drop_bwd_bias": "g ld_g rows c act_out act keep:f dz ld_dz dbias",
}


def test_image_dropout_bindings_keep_their_names_and_signatures():
    """_C.image_dropout holds exactly the five twins, each as the plan op add_<op>(plan, args...) and the direct entry
    point <op>(args..., stream), with the argument types above"""
    import inspect

    from sparkflow_b200.ops import native

    mod = native.cuda_ext().image_dropout
    got = dict(_pinned(o) for n, o in vars(mod).items() if inspect.isbuiltin(o))
    want = {}
    for op, spec in _TWIN_ARGS.items():
        types = tuple("float" if a.endswith(":f") else "int" for a in spec.split())
        want[op] = types + ("int",)
        want["add_" + op] = ("sparkflow_b200._C.Plan",) + types
    assert got == want


def test_every_conv_kernel_is_preloaded():
    """sf_preload_kernels names every kernel of csrc/conv.cu (each template instance a launcher uses): a kernel loaded
    lazily at its first launch would need a context-wide synchronisation in the middle of a training run"""
    import os
    import re

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    conv = open(os.path.join(root, "csrc", "conv.cu")).read()
    pre = open(os.path.join(root, "csrc", "kernels.cu")).read()
    kernels = set(re.findall(r"__global__ void __launch_bounds__\([^)]*\)\s*\n(\w+)\(", conv))
    assert {"maxpool_drop_fwd_kernel", "act_drop_bwd_bias_kernel", "maxpool_fwd_kernel"} <= kernels, kernels
    templated = {k for k in kernels if re.search(r"template <[^>]*>\s*\n__global__ void __launch_bounds__\([^)]*\)\s*\n" + k + r"\(", conv)}
    for k in sorted(kernels):
        if k.startswith("conv_first"):
            continue                # instances <KH, KW, CIN>, listed one by one
        if k in templated:
            for inst in ("false", "true"):
                assert f"sf::{k}<{inst}>" in pre, f"{k}<{inst}> is not preloaded"
        else:
            assert f"SF_PRELOAD(sf::{k})" in pre, f"{k} is not preloaded"
