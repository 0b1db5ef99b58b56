"""L2 weight penalties in the loss (``loss = data loss + sum_v c_v * sum(v ** 2)``): which spellings compile to which
penalty map and which stay on the interpreter, and the float64 oracle of the penalised step (the step oracle of
tests/test_step_gradients.py plus the closed-form penalty) against the interpreter and against plausible bugs."""
import numpy as np
import pytest

from sparkflow_b200.graph import tfcompat as tf
from sparkflow_b200.graph.executor import GraphProgram
from sparkflow_b200.graph.ir import GraphIR
from sparkflow_b200.graph.tfcompat import core
from sparkflow_b200.graph.tfcompat.ops import attr_type
from sparkflow_b200.graph_utils import build_graph
from sparkflow_b200.models import zoo
from sparkflow_b200.models.compiler import UnsupportedGraph, compile_graph
from sparkflow_b200.parallel.plan_builder import fused_first_conv
from test_step_gradients import _MODEL_CACHE, _assert_grads, _bf16, _forward, _grads, _rejects

# zoo name -> label kind (one-hot classes, or None for the auto-encoder)
L2_MODELS = {"l2_dnn": "onehot", "l2_cnn": "onehot", "l2_autoencoder": None}
# relative Frobenius / max-abs error of every gradient of the GPU step against the bf16-emulating oracle, with the strong
# penalty map of l2_model: about 3x the worst error measured on an H100 80GB HBM3 (700 W power limit) over the step test
# (every plan variant and batch size) and the delivered-gradient test (served and sharded paths).
TOL = {                                  # measured: step test; delivered-gradient test
    "l2_dnn": (7e-4, 3.1e-3),            # 1.4e-4, 2.9e-4; 2.3e-4, 1.0e-3
    "l2_cnn": (3.8e-3, 7.2e-3),          # 6.8e-4, 2.1e-3; 1.3e-3, 2.4e-3
    "l2_autoencoder": (6.5e-5, 2.9e-4),  # 1.9e-6, 1.2e-5; 2.2e-5, 9.6e-5
}


def l2_model(name, strong=True):
    """(GraphIR, LayerPlan, label tensor or None).  ``strong``: the plan's penalty coefficients raised to 4e-3 .. 1e-2
    (one per variable, so a mix-up shows), registered in the step tests' model cache so their worker helpers build the
    plan with them.  The zoo's coefficients (5e-4 .. 1e-5) put the penalty gradient below the bf16 tolerances of the
    data gradient, where no comparison could see it missing; the strong map keeps which variables are penalised."""
    if not strong:
        ir = GraphIR.from_metagraph(zoo.build(name))
        return ir, compile_graph(ir, "x:0", "y:0" if L2_MODELS[name] else None), "y:0" if L2_MODELS[name] else None
    if name not in _MODEL_CACHE:
        ir, lp, label = l2_model(name, strong=False)
        lp.penalty = {v: 4e-3 * (1 + 0.25 * k) for k, v in enumerate(lp.penalty)}
        _MODEL_CACHE[name] = (ir, lp, label)
    return _MODEL_CACHE[name]


def l2_data(name, n, seed):
    _, lp, _ = l2_model(name)
    rng = np.random.default_rng(seed)
    X = rng.random((n, lp.input_dim), dtype=np.float32)
    Y = np.eye(lp.label_dim, dtype=np.float32)[rng.integers(0, lp.label_dim, n)] if L2_MODELS[name] else None
    return X, Y


def l2_weights(name, seed=1):
    """the graph's initializers with small non-zero biases (as the step tests use them)"""
    ir = l2_model(name)[0]
    rng = np.random.default_rng(seed + 100)
    return [w if w.ndim > 1 else (0.05 * rng.standard_normal(w.shape)).astype(np.float32) for w in GraphProgram(ir).init_weights(seed=seed)]


def penalty_oracle(lp, weights, X, Y, emulate_bf16, argmax=None, relu_mask=None, coef=2.0, every_split=1, loss_scale=1.0):
    """(loss, gradients, pools) of the penalised step in float64: the step oracle's data loss plus c * sum(v ** 2) of every
    penalised variable, a kernel at its bf16 value with ``emulate_bf16`` (the step reads the bf16 replica).  The other
    arguments plant the bugs the tolerances must reject: the gradient term ``coef * c * v`` (2 is right), added
    ``every_split`` times, and the loss term times ``loss_scale``."""
    l_data, _, params, pools, _ = _forward(lp, weights, X, Y, emulate_bf16, argmax, relu_mask)
    pos = {n: k for k, n in enumerate(lp.var_order)}
    grads = _grads(l_data, params)
    loss = float(l_data.detach())
    for v, c in lp.penalty.items():
        p = params[pos[v]].detach()
        if emulate_bf16 and p.dim() > 1:
            p = _bf16(p)
        loss += loss_scale * c * float((p * p).sum())
        grads[pos[v]] = grads[pos[v]] + every_split * coef * c * p.cpu().numpy()
    return loss, grads, pools


# ------------------------------------------------------------------------------------------------------------------
# spellings
# ------------------------------------------------------------------------------------------------------------------
def _mlp():
    x = tf.placeholder(tf.float32, shape=[None, 20], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 4], name="y")
    h = tf.layers.dense(x, 16, activation=tf.nn.relu, name="h")
    logits = tf.layers.dense(h, 4, name="o")
    xent = tf.reduce_mean(tf.nn.softmax_cross_entropy_with_logits(labels=y, logits=logits))
    g = tf.get_default_graph()
    var = {v.name.split(":")[0]: v for v in tf.trainable_variables()}
    return x, y, h, logits, xent, g, var


def _l2loss_node(v):
    """TF's fused L2Loss op, which the builder's l2_loss (a composite) does not emit"""
    t = v.value()
    return tf.get_default_graph().add_node("L2Loss", "L2Loss", [t], {"T": attr_type(core.float32)}, [core.float32], [()]).outputs[0]


_MASK = np.zeros((20, 16), np.float32)
_MASK[0, 0] = 1.0


def _compile(fn):
    return compile_graph(GraphIR.from_metagraph(build_graph(fn)), "x:0", "y:0")


def _add_loss(loss):
    tf.losses.add_loss(loss)
    return loss


SPELLINGS = {
    "add_n of builder l2_loss": (lambda: (lambda x, y, h, lo, xe, g, v: _add_loss(
        xe + 5e-4 * tf.add_n([tf.nn.l2_loss(v["h/kernel"]), tf.nn.l2_loss(v["o/kernel"])])))(*_mlp()),
        {"h/kernel": 2.5e-4, "o/kernel": 2.5e-4}),
    "fused L2Loss, constant on the left": (lambda: (lambda x, y, h, lo, xe, g, v: _add_loss(
        tf.add(xe, tf.multiply(3e-3, _l2loss_node(v["o/kernel"])))))(*_mlp()), {"o/kernel": 1.5e-3}),
    "penalty first, AddV2-free Add order": (lambda: (lambda x, y, h, lo, xe, g, v: _add_loss(
        tf.add(tf.multiply(_l2loss_node(v["h/bias"]), 1e-2), xe)))(*_mlp()), {"h/bias": 5e-3}),
    "Sum(Square(v)) over all axes": (lambda: (lambda x, y, h, lo, xe, g, v: _add_loss(
        xe + 1e-3 * tf.reduce_sum(tf.square(v["h/kernel"]))))(*_mlp()), {"h/kernel": 1e-3}),
    "Keras l2: Sum(Mul(c, Square(v)))": (lambda: (lambda x, y, h, lo, xe, g, v: _add_loss(
        xe + tf.reduce_sum(tf.multiply(2e-3, tf.square(v["o/kernel"])))))(*_mlp()), {"o/kernel": 2e-3}),
    "nested adds, one variable twice": (lambda: (lambda x, y, h, lo, xe, g, v: _add_loss(
        (xe + 1e-3 * tf.nn.l2_loss(v["h/kernel"])) + tf.add_n([1e-3 * tf.nn.l2_loss(v["h/kernel"]), tf.nn.l2_loss(v["o/bias"])])))(*_mlp()),
        {"h/kernel": 1e-3, "o/bias": 0.5}),
    "coefficient 0": (lambda: (lambda x, y, h, lo, xe, g, v: _add_loss(xe + 0.0 * tf.nn.l2_loss(v["h/kernel"])))(*_mlp()), {}),
    "one-element constant factors ([1] and [1, 1])": (lambda: (lambda x, y, h, lo, xe, g, v: _add_loss(
        xe + tf.constant(np.full((1, 1), 2e-3, np.float32)) * tf.reduce_sum(tf.constant(np.full(1, 0.5, np.float32)) * tf.square(v["h/kernel"]))))(*_mlp()),
        {"h/kernel": 1e-3}),
    "add_n of one term": (lambda: (lambda x, y, h, lo, xe, g, v: _add_loss(xe + tf.add_n([1e-3 * tf.nn.l2_loss(v["o/kernel"])])))(*_mlp()),
                          {"o/kernel": 5e-4}),
    "get_regularization_loss without regularizers": (lambda: (lambda x, y, h, lo, xe, g, v: _add_loss(
        xe + tf.losses.get_regularization_loss()))(*_mlp()), {}),
}


def _regularized():
    x = tf.placeholder(tf.float32, shape=[None, 64], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 4], name="y")
    img = tf.reshape(x, [-1, 8, 8, 1])
    reg = tf.contrib.layers.l2_regularizer(1e-4)
    c = tf.layers.conv2d(img, 8, 3, activation=tf.nn.relu, kernel_regularizer=reg, bias_regularizer=tf.contrib.layers.l2_regularizer(2e-4), name="c")
    logits = tf.layers.dense(tf.layers.flatten(c), 4, kernel_regularizer=reg, bias_regularizer=tf.contrib.layers.l2_regularizer(0.0), name="d")
    return _add_loss(tf.losses.softmax_cross_entropy(y, logits, loss_collection=None) + tf.losses.get_regularization_loss())


@pytest.mark.parametrize("spelling", list(SPELLINGS))
def test_accepted_spellings_compile_to_their_penalty_map(spelling):
    fn, want = SPELLINGS[spelling]
    lp = _compile(fn)
    assert lp.loss == "softmax_xent"
    assert lp.penalty.keys() == want.keys(), (lp.penalty, want)
    for v, c in want.items():
        assert lp.penalty[v] == pytest.approx(c, rel=1e-6), (v, lp.penalty[v], c)


def test_layer_regularizers_and_get_regularization_loss():
    """kernel_regularizer / bias_regularizer on tf.layers.conv2d and dense: Mul(scale, L2Loss) in REGULARIZATION_LOSSES,
    summed by one AddN named total_regularization_loss; a scale of 0 regularizes nothing"""
    ir = GraphIR.from_metagraph(build_graph(_regularized))
    ops = {n.op for n in ir.nodes.values()}
    assert {"L2Loss", "AddN"} <= ops
    assert ir.nodes["total_regularization_loss"].op == "AddN" and len(ir.nodes["total_regularization_loss"].inputs) == 3
    lp = compile_graph(ir, "x:0", "y:0")
    assert lp.penalty == pytest.approx({"c/kernel": 5e-5, "c/bias": 1e-4, "d/kernel": 5e-5})


def test_penalty_outside_the_training_loss_is_ignored():
    """the reference trains on LOSSES[0]: a penalty added to another collection entry is not part of the step"""
    def fn():
        x, y, h, lo, xe, g, v = _mlp()
        loss = tf.losses.softmax_cross_entropy(y, lo)
        tf.losses.add_loss(1e-3 * tf.nn.l2_loss(v["h/kernel"]))
        return loss
    assert _compile(fn).penalty == {}


def _reject(build):
    def fn():
        x, y, h, lo, xe, g, v = _mlp()
        return _add_loss(build(x, y, h, lo, xe, v))
    return fn


REJECTED = {
    "L1": (_reject(lambda x, y, h, lo, xe, v: xe + 1e-3 * tf.reduce_sum(tf.abs(v["h/kernel"]))), "L1"),
    "elastic net": (_reject(lambda x, y, h, lo, xe, v: xe + tf.add_n([1e-3 * tf.nn.l2_loss(v["h/kernel"]),
                                                                       1e-3 * tf.reduce_sum(tf.abs(v["h/kernel"]))])), "L1"),
    "penalty of W - W0": (_reject(lambda x, y, h, lo, xe, v: xe + 1e-3 * tf.nn.l2_loss(tf.subtract(v["h/kernel"].value(), 0.5))), "bare variables"),
    "penalty of a transpose": (_reject(lambda x, y, h, lo, xe, v: xe + 1e-3 * tf.nn.l2_loss(tf.transpose(v["h/kernel"].value()))), "bare variables"),
    "activity regularizer": (_reject(lambda x, y, h, lo, xe, v: xe + 1e-3 * tf.nn.l2_loss(h)), "bare variables"),
    "placeholder coefficient": (_reject(lambda x, y, h, lo, xe, v: xe + tf.placeholder(tf.float32, [], name="wd") * tf.nn.l2_loss(v["h/kernel"])),
                                "not a constant"),
    "constant scaling the sum": (_reject(lambda x, y, h, lo, xe, v: 0.5 * (xe + 1e-3 * tf.nn.l2_loss(v["h/kernel"]))), "under a reduction"),
    "penalty inside the reduction": (_reject(lambda x, y, h, lo, xe, v: tf.reduce_mean(
        tf.nn.softmax_cross_entropy_with_logits(labels=y, logits=lo) + 1e-3 * tf.nn.l2_loss(v["h/kernel"]))), "under a reduction"),
    "two data losses": (_reject(lambda x, y, h, lo, xe, v: xe + tf.reduce_mean(tf.square(lo - y)) + 1e-3 * tf.nn.l2_loss(v["h/kernel"])),
                        "2 data losses"),
    "sum over some axes": (_reject(lambda x, y, h, lo, xe, v: xe + 1e-3 * tf.reduce_sum(tf.square(v["h/kernel"]), axis=0)), "some of its axes"),
    # a constant of several elements weighs the variable's elements differently: one element of the mask is 1, so taking
    # its first element as the coefficient would penalise all of W[0, :] ... W[19, :] instead of W[0, 0]
    "masked decay inside the sum": (_reject(lambda x, y, h, lo, xe, v: xe + tf.reduce_sum(tf.constant(_MASK) * tf.square(v["h/kernel"]))),
                                    "constant of 320 elements"),
    "vector factor on l2_loss": (_reject(lambda x, y, h, lo, xe, v: xe + tf.constant(np.asarray([1e-3, 0.0], np.float32)) * tf.nn.l2_loss(v["h/kernel"])),
                                 "constant of 2 elements"),
}


@pytest.mark.parametrize("case", list(REJECTED))
def test_rejected_spellings_name_their_reason(case):
    fn, reason = REJECTED[case]
    with pytest.raises(UnsupportedGraph, match=reason):
        _compile(fn)


def test_penalty_on_a_variable_outside_the_layers_is_rejected():
    def fn():
        x, y, h, lo, xe, g, v = _mlp()
        extra = tf.get_variable("extra", shape=[3, 3])
        return _add_loss(xe + 1e-3 * tf.nn.l2_loss(extra))
    with pytest.raises(UnsupportedGraph, match="not a kernel or bias"):
        _compile(fn)


def test_penalised_first_conv_is_not_fused():
    assert fused_first_conv(l2_model("l2_cnn", strong=False)[1]) is None
    assert fused_first_conv(compile_graph(GraphIR.from_metagraph(zoo.build("cnn_same")), "x:0", "y:0")) is not None


# ------------------------------------------------------------------------------------------------------------------
# the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(L2_MODELS))
def test_penalty_oracle_matches_interpreter(name):
    ir, lp, label = l2_model(name, strong=False)
    assert lp.penalty
    X, Y = l2_data(name, 7, seed=3)
    w = l2_weights(name)
    feeds = {"x:0": X}
    if label:
        feeds[label] = Y
    l_int, g_int = GraphProgram(ir).loss_and_grads(feeds, w)
    l_ora, g_ora, _ = penalty_oracle(lp, w, X, Y, emulate_bf16=False)
    assert abs(l_ora - l_int) <= 1e-5 * max(1.0, abs(l_int)), (l_ora, l_int)
    _assert_grads(f"{name} exact oracle vs interpreter", lp.var_order, g_ora, [g.numpy() for g in g_int], (1e-4, 1e-4))


LOSS_TOL = 1e-5                          # relative error of the step's loss; measured 3.5e-6


@pytest.mark.parametrize("B", [7, 129])
@pytest.mark.parametrize("name", list(L2_MODELS))
def test_tolerances_reject_penalty_bugs(name, B):
    """The step comparison rejects, one at a time: the penalty missing, c where 2c belongs, the term added by each of two
    K splits, the term of another variable of the same shape (or of none), and the loss term missing or doubled."""
    _, lp, _ = l2_model(name)
    X, Y = l2_data(name, B, seed=11)
    w = l2_weights(name)
    loss, ref, _ = penalty_oracle(lp, w, X, Y, True)
    tol = TOL[name]
    assert not _rejects(ref, ref, tol)
    grad_mutants = {"without the penalty": penalty_oracle(lp, w, X, Y, True, coef=0.0)[1],
                    "with c instead of 2c": penalty_oracle(lp, w, X, Y, True, coef=1.0)[1],
                    "with the term added by two K splits": penalty_oracle(lp, w, X, Y, True, every_split=2)[1]}
    # the term of a variable applied to another: missing on its own variable (and, where one has the same shape, added
    # to that one), one variable at a time
    no_term = penalty_oracle(lp, w, X, Y, True, coef=0.0)[1]
    for v in lp.penalty:
        k = lp.var_order.index(v)
        grads = [g if i != k else no_term[k] for i, g in enumerate(ref)]
        for i, u in enumerate(lp.var_order):
            if u != v and grads[i].shape == ref[k].shape:
                grads[i] = grads[i] + (ref[k] - no_term[k])
                break
        grad_mutants[f"with {v}'s term on the wrong variable"] = grads
    for what, grads in grad_mutants.items():
        assert _rejects(grads, ref, tol), f"{name} B={B}: the tolerance {tol} accepts the gradient {what}"
    for what, scale in (("missing", 0.0), ("doubled", 2.0)):
        l_bad = penalty_oracle(lp, w, X, Y, True, loss_scale=scale)[0]
        assert abs(l_bad - loss) / abs(loss) > LOSS_TOL, f"{name} B={B}: the loss tolerance accepts the penalty's loss term {what}"


def test_add_n_of_one_input_is_that_input():
    """as TF-1.x's add_n: no AddN node for a single input; an Identity of it when a name is given"""
    g = tf.Graph()
    with g.as_default():
        t = tf.constant(np.float32(2.0))
        assert tf.add_n([t]) is t
        named = tf.add_n([t], name="total")
        assert named.op.type == "Identity" and named.op.name == "total"
        assert tf.add_n([t, t]).op.type == "AddN"
