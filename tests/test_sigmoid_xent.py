"""Sigmoid cross-entropy in the compiled plan, without a GPU: the compiler recognises both spellings of
``tf.nn.sigmoid_cross_entropy_with_logits`` (the tfcompat builder's Relu / Neg(Abs) and TF-1.x's Select on x >= 0) and
reports the variants it does not cover; the float64 oracle of the new graphs matches the interpreter; the per-step
tolerances of the GPU test reject plausible gradient bugs; and the new kernels keep no stack frame.

The oracle and graph helpers here are shared with tests/test_gpu_sigmoid_xent.py.
"""
import dataclasses
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sparkflow_b200.graph import tfcompat as tf
from sparkflow_b200.graph.executor import GraphProgram
from sparkflow_b200.graph.ir import GraphIR
from sparkflow_b200.graph.tfcompat import ops as tfops
from sparkflow_b200.graph_utils import build_graph
from sparkflow_b200.models import zoo
from sparkflow_b200.models.compiler import UnsupportedGraph, compile_graph
from sparkflow_b200.parallel.plan_builder import loss_mode
from test_step_gradients import _assert_grads, _forward, _grads, _rejects

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "sparkflow_b200", "_C.so")


def _tf1_sigmoid_xent(labels, logits):
    """tf.nn.sigmoid_cross_entropy_with_logits as TF 1.x builds it (nn_impl.py), with the Mul operands swapped"""
    zeros = tf.zeros_like(logits)
    cond = tf.greater_equal(logits, zeros)
    relu_logits = tf.where(cond, logits, zeros)
    neg_abs_logits = tf.where(cond, tf.negative(logits), logits)
    return tf.add(tf.subtract(relu_logits, tf.multiply(labels, logits)), tf.log1p(tf.exp(neg_abs_logits)))


def tf1_mlp():
    """tf.losses.sigmoid_cross_entropy as a real TF-1.x MetaGraph carries it: labels cast to the logits' dtype, the
    TF-1.x per-element core, weights 1.0 multiplied in, Sum / DivNoNan(num_present)"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 5], name="y")
    logits = tf.layers.dense(tf.layers.dense(x, 64, activation=tf.nn.tanh), 5)
    tf.nn.sigmoid(logits, name="out")
    per = _tf1_sigmoid_xent(tf.cast(y, tf.float32), logits)
    weighted = tf.multiply(per, tf.cast(1.0, tf.float32))
    total = tf.reduce_sum(weighted)
    value = tfops.binary("DivNoNan", total, tf.cast(tf.size(weighted), tf.float32), name="value")
    tf.losses.add_loss(value)
    return value


def cnn_sigmoid():
    """cnn_same's backbone with 10 independent sigmoid outputs"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    img = tf.reshape(x, shape=[-1, 28, 28, 1])
    c1 = tf.layers.max_pooling2d(tf.layers.conv2d(img, 32, 5, padding="same", activation=tf.nn.relu), 2, 2, padding="same")
    c2 = tf.layers.max_pooling2d(tf.layers.conv2d(c1, 64, 5, padding="same", activation=tf.nn.relu), 2, 2, padding="same")
    h = tf.layers.dense(tf.layers.flatten(c2), 1024, activation=tf.nn.relu)
    logits = tf.layers.dense(h, 10)
    tf.nn.sigmoid(logits, name="out")
    return tf.losses.sigmoid_cross_entropy(y, logits)


def logreg():
    """multi-label logistic regression: the loss layer is the only dense layer, so under a sharded Hogwild master its
    GEMM also carries the read-your-writes wait"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 5], name="y")
    logits = tf.layers.dense(x, 5)
    tf.nn.sigmoid(logits, name="out")
    return tf.losses.sigmoid_cross_entropy(y, logits)


# name -> graph function; the labels are 0 / 1 except for tf1_mlp, which gets soft labels
GRAPHS = {"binary_dnn": zoo.binary_dnn, "multilabel_dnn": zoo.multilabel_dnn, "cnn_sigmoid": cnn_sigmoid, "tf1_mlp": tf1_mlp,
          "logreg": logreg}
CNN_GRAPHS = ("cnn_sigmoid",)

# Per graph: (relative Frobenius error, max-abs error / max|ref|) of every gradient of the GPU step against the
# bf16-emulating oracle, following test_step_gradients.TOL: about 3x the worst error tests/test_gpu_sigmoid_xent.py
# measured on an H100 80GB HBM3 (700 W power limit) over all plan variants, batch sizes and feeds (and, for
# multilabel_dnn, the delivered gradients).  tf1_mlp's tanh layer carries the largest bf16 rounding steps.
TOL = {                                  # measured
    "binary_dnn": (2e-4, 4e-4),          # 6.9e-5, 1.3e-4
    "multilabel_dnn": (1.5e-4, 4e-4),    # 4.9e-5, 1.3e-4
    "cnn_sigmoid": (1.8e-3, 2.1e-3),     # 5.8e-4, 7.0e-4
    "tf1_mlp": (1e-3, 4e-3),             # 2.9e-4, 1.3e-3
    "logreg": (1e-5, 1e-5),              # 7.6e-7, 9.0e-7 (floor 1e-5, as test_step_gradients.TOL)
}
LOSS_TOL = 1.5e-5                        # relative; measured 5.0e-6

_CACHE = {}


def sig_model(name):
    """(GraphIR, LayerPlan, graph JSON)"""
    if name not in _CACHE:
        graph = build_graph(GRAPHS[name])
        ir = GraphIR.from_metagraph(graph)
        _CACHE[name] = (ir, compile_graph(ir, "x:0", "y:0"), graph)
    return _CACHE[name]


def sig_data(name, n, seed):
    lp = sig_model(name)[1]
    rng = np.random.default_rng(seed)
    X = rng.random((n, lp.input_dim), dtype=np.float32)
    shape = (n, lp.label_dim)
    Y = rng.random(shape, dtype=np.float32) if name == "tf1_mlp" else rng.integers(0, 2, shape).astype(np.float32)
    return X, Y


def sig_weights(name, seed=1):
    """the graph's initializers, with small non-zero biases"""
    ir = sig_model(name)[0]
    rng = np.random.default_rng(seed + 100)
    return [w if w.ndim > 1 else (0.05 * rng.standard_normal(w.shape)).astype(np.float32)
            for w in GraphProgram(ir).init_weights(seed=seed)]


def sig_forward(lp, weights, X, Y, emulate_bf16, argmax=None, relu_mask=None, device=None, per_row=False):
    """test_step_gradients._forward with the sigmoid cross-entropy head: run on the plan with an MSE head, whose output
    is the fp32 logits of the activation-free last layer (still attached to the graph), then take the loss in float64.
    ``per_row``: normalise by the batch instead of by every element (a bug the tolerances must catch)."""
    kw = {} if device is None else dict(device=device)
    _, z, params, pools, zs = _forward(dataclasses.replace(lp, loss="mse"), weights, X, Y, emulate_bf16, argmax, relu_mask, **kw)
    y = torch.as_tensor(np.asarray(Y), dtype=torch.float64, device=z.device)
    loss = F.binary_cross_entropy_with_logits(z, y, reduction="sum") / (z.shape[0] if per_row else z.numel())
    return loss, z, params, pools, zs


def sig_oracle(lp, weights, X, Y, emulate_bf16, **kw):
    loss, _, params, _, _ = sig_forward(lp, weights, X, Y, emulate_bf16, **kw)
    return float(loss.detach()), _grads(loss, params)


# ------------------------------------------------------------------------------------------------------------------
# compiler
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(GRAPHS))
def test_compiler_accepts_sigmoid_cross_entropy(name):
    ir, lp, _ = sig_model(name)
    assert lp.loss == "sigmoid_xent" and lp.label_name == "y:0" and not lp.target_is_input
    assert lp.layers[-1].act is None and lp.label_dim == lp.layers[-1].out_features
    assert loss_mode(lp.loss) == 3
    # prediction compiles the Sigmoid as the last layer's activation
    lpi = compile_graph(ir, "x:0", None, "out:0", need_loss=False)
    assert lpi.layers[-1].act == "Sigmoid" and lpi.output.layer == len(lpi.layers) - 1


def test_loss_kinds_map_to_explicit_heads():
    assert [loss_mode(k) for k in ("softmax_xent", "mse", "sigmoid_xent")] == [1, 2, 3]
    with pytest.raises(UnsupportedGraph):
        loss_mode("hinge")


def _dense_head(n_out=5, act=None, label_dim=None):
    x = tf.placeholder(tf.float32, shape=[None, 20], name="x")
    y = tf.placeholder(tf.float32, shape=[None, label_dim or n_out], name="y")
    return x, y, tf.layers.dense(tf.layers.dense(x, 16, activation=tf.nn.relu), n_out, activation=act)


def _weighted_const():
    x, y, logits = _dense_head()
    tf.losses.add_loss(tf.reduce_mean(tf.multiply(tf.nn.sigmoid_cross_entropy_with_logits(labels=y, logits=logits), 2.0)))


def _weighted_class_vector():
    """per-class weights whose first entry is 1"""
    x, y, logits = _dense_head(n_out=4)
    per = tf.nn.sigmoid_cross_entropy_with_logits(labels=y, logits=logits)
    tf.losses.add_loss(tf.reduce_mean(tf.multiply(per, tf.constant(np.array([1., 5., 5., 5.], np.float32)))))


def _sum_over_labels():
    """reduce_mean(reduce_sum(per_element, axis=1)): N times the element mean"""
    x, y, logits = _dense_head()
    tf.losses.add_loss(tf.reduce_mean(tf.reduce_sum(tf.nn.sigmoid_cross_entropy_with_logits(labels=y, logits=logits), axis=1)))


def _weighted_placeholder():
    x, y, logits = _dense_head()
    w = tf.placeholder(tf.float32, shape=[None, 5], name="w")
    per = tf.nn.sigmoid_cross_entropy_with_logits(labels=y, logits=logits)
    tf.losses.add_loss(tf.reduce_sum(tf.multiply(w, per)) / tf.cast(tf.size(per), tf.float32))


def _activated_logits():
    x, y, out = _dense_head(act=tf.nn.sigmoid)
    tf.losses.sigmoid_cross_entropy(y, out)


def _label_smoothed():
    """TF-1.x's label_smoothing=0.1: y * (1 - 0.1) + 0.5 * 0.1"""
    x, y, logits = _dense_head()
    smoothed = tf.add(tf.multiply(y, 0.9), 0.05)
    tf.losses.add_loss(tf.reduce_mean(tf.nn.sigmoid_cross_entropy_with_logits(labels=smoothed, logits=logits)))


def _width_mismatch():
    x, y, logits = _dense_head(label_dim=1)
    tf.losses.sigmoid_cross_entropy(y, logits)


@pytest.mark.parametrize("fn,match", [(_weighted_const, "weighted"), (_weighted_placeholder, "weighted"),
                                      (_weighted_class_vector, "weighted"), (_sum_over_labels, "sum under a mean"),
                                      (_activated_logits, "raw logits"), (_label_smoothed, "placeholder"),
                                      (_width_mismatch, "width")])
def test_compiler_rejects_uncovered_variants(fn, match):
    ir = GraphIR.from_metagraph(build_graph(fn))
    with pytest.raises(UnsupportedGraph, match=match):
        compile_graph(ir, "x:0", "y:0")


def test_unit_weights_compile_as_the_element_mean():
    """a Mul by an all-ones weight vector is the unweighted loss"""
    def fn():
        x, y, logits = _dense_head(n_out=4)
        per = tf.nn.sigmoid_cross_entropy_with_logits(labels=y, logits=logits)
        tf.losses.add_loss(tf.reduce_mean(tf.multiply(per, tf.constant(np.ones(4, np.float32)))))

    assert compile_graph(GraphIR.from_metagraph(build_graph(fn)), "x:0", "y:0").loss == "sigmoid_xent"


def test_loose_add_is_not_sigmoid_cross_entropy():
    """an Add of the right shape whose parts refer to different logits tensors is not the loss"""
    def fn():
        x, y, logits = _dense_head()
        other = tf.layers.dense(x, 5)
        per = tf.add(tf.subtract(tf.nn.relu(logits), tf.multiply(logits, y)), tf.log1p(tf.exp(tf.negative(tf.abs(other)))))
        tf.losses.add_loss(tf.reduce_mean(per))

    with pytest.raises(UnsupportedGraph, match="sigmoid-cross-entropy"):
        compile_graph(GraphIR.from_metagraph(build_graph(fn)), "x:0", "y:0")


# ------------------------------------------------------------------------------------------------------------------
# the oracle and the tolerances
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(GRAPHS))
def test_oracle_matches_interpreter(name):
    ir, lp, _ = sig_model(name)
    X, Y = sig_data(name, 7, seed=3)
    w = sig_weights(name)
    l_int, g_int = GraphProgram(ir).loss_and_grads({"x:0": X, "y:0": Y}, w)
    l_ora, g_ora = sig_oracle(lp, w, X, Y, False, device=torch.device("cpu"))
    assert abs(l_ora - l_int) <= 1e-5 * max(1.0, abs(l_int)), (l_ora, l_int)
    _assert_grads(f"{name} exact oracle vs interpreter", lp.var_order, g_ora, [g.numpy() for g in g_int], (1e-4, 1e-4))
    l_em, _ = sig_oracle(lp, w, X, Y, True, device=torch.device("cpu"))
    assert abs(l_em - l_ora) <= 2e-2 * max(1.0, abs(l_ora)), (l_em, l_ora)


@pytest.mark.parametrize("B", [7, 129])
@pytest.mark.parametrize("name", ["binary_dnn", "multilabel_dnn", "tf1_mlp", "logreg"])
def test_tolerances_reject_plausible_loss_bugs(name, B):
    """The per-step comparison rejects the oracle's gradient (a) normalised per row instead of per element (a factor of
    N, so only for N > 1), (b) scaled by 1.1, (c) without the batch's last row, (d) with one label column flipped."""
    _, lp, _ = sig_model(name)
    X, Y = sig_data(name, B, seed=11)
    w = sig_weights(name)
    cpu = dict(device=torch.device("cpu"))
    _, ref = sig_oracle(lp, w, X, Y, True, **cpu)
    tol = TOL[name]
    assert not _rejects(ref, ref, tol)
    flipped = Y.copy()
    flipped[:, -1] = 1.0 - flipped[:, -1]
    mutants = {"scaled by 1.1": [1.1 * g for g in ref],
               "without the last row": sig_oracle(lp, w, X[:-1], Y[:-1], True, **cpu)[1],
               "with the last label column flipped": sig_oracle(lp, w, X, flipped, True, **cpu)[1]}
    if lp.label_dim > 1:
        mutants["normalised per row"] = sig_oracle(lp, w, X, Y, True, per_row=True, **cpu)[1]
    for what, grads in mutants.items():
        assert _rejects(grads, ref, tol), f"{name} B={B}: the tolerance {tol} accepts the gradient {what}"


# ------------------------------------------------------------------------------------------------------------------
# build artifacts
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not os.path.exists(SO) or shutil.which("cuobjdump") is None or shutil.which("c++filt") is None,
                    reason="needs the built extension and the CUDA binary utilities")
def test_sigmoid_xent_kernels_have_no_stack_frame():
    """the stand-alone kernel and the SIGMOID_LOSS GEMM variant (SfEpi 5, sf_gemm_sigmoid_loss_kernel), and the LOSS
    variants beside them"""
    txt = subprocess.run(["cuobjdump", "-res-usage", SO], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, check=True).stdout
    names = re.findall(r"Function (\S+):\n\s+REG:(\d+) STACK:(\d+)", txt)
    dem = subprocess.run(["c++filt"], input="\n".join(n for n, _, _ in names), stdout=subprocess.PIPE, text=True, check=True).stdout.splitlines()
    use = {re.sub(r"\(.*", "", d).replace("void ", ""): (int(r), int(s)) for d, (_, r, s) in zip(dem, names)}
    want = ["sf::elementwise_loss_kernel<sf::SigmoidXentHead>", "sf::elementwise_loss_kernel<sf::MseHead>"]
    want += [k for bn in (32, 64) for k in (f"sf::sf_gemm_epi_kernel<{bn}, false, 2>", f"sf::sf_gemm_sigmoid_loss_kernel<{bn}>")]
    missing = [k for k in want if k not in use]
    assert not missing, (missing, sorted(use))
    spilled = {k: use[k] for k in want if use[k][1] != 0}
    assert not spilled, f"kernels with a local-memory stack frame (REG, STACK): {spilled}"
