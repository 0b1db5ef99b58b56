"""Sparse softmax cross-entropy in the compiled plan, without a GPU: the compiler recognises class-index labels in every
spelling a numeric label column reaches the loss with (``tf.losses.sparse_softmax_cross_entropy``,
``reduce_mean(sparse_softmax_cross_entropy_with_logits)`` + ``add_loss`` and ``softmax_cross_entropy`` of a
``tf.one_hot``) and reports the variants it does not cover; the float64 oracle of the zoo models matches the
interpreter; the per-step tolerances of the GPU test reject plausible label bugs; the partition loader rejects labels
that are not class indices; and the new kernels keep no stack frame.

The oracle and graph helpers here are shared with tests/test_gpu_sparse_xent.py.
"""
import dataclasses

import numpy as np
import pytest
import torch

from sparkflow_b200.graph import tfcompat as tf
from sparkflow_b200.graph.executor import GraphProgram
from sparkflow_b200.graph.ir import GraphIR
from sparkflow_b200.graph.tfcompat import core as tfcore
from sparkflow_b200.graph.tfcompat import ops as tfops
from sparkflow_b200.graph_utils import build_graph
from sparkflow_b200.models import zoo
from sparkflow_b200.models.compiler import MAX_SPARSE_CLASSES, UnsupportedGraph, compile_graph
from sparkflow_b200.parallel.plan_builder import check_grammar, loss_mode
from sparkflow_b200.parallel.worker import check_class_labels
from kernel_usage import needs_binary_utils, res_usage
from test_step_gradients import _assert_grads, _forward, _grads, _rejects

GRAPHS = {"sparse_dnn": zoo.sparse_dnn, "onehot_cnn": zoo.onehot_cnn, "sparse_dnn100": zoo.sparse_dnn100}
CNN_GRAPHS = ("onehot_cnn",)

# Per graph: (relative Frobenius error, max-abs error / max|ref|) of every gradient of the GPU step against the
# bf16-emulating oracle, about 3x the worst error tests/test_gpu_sparse_xent.py measured on an H100 80GB HBM3 (700 W power
# limit) over all plan variants, batch sizes and feeds, following test_step_gradients.TOL; sparse_dnn and onehot_cnn
# keep the tolerances of simple_dnn and cnn, whose steps they share.
TOL = {                                  # measured
    "sparse_dnn": (5e-4, 1.2e-3),        # 1.4e-4, 2.9e-4
    "onehot_cnn": (7e-4, 2.5e-3),        # 2.2e-4, 7.6e-4
    "sparse_dnn100": (2.5e-4, 3e-3),     # 7.9e-5, 1.1e-3
}
LOSS_TOL = 5e-5                          # relative, as test_step_gradients.LOSS_TOL; measured 1.8e-6

_CACHE = {}


def sp_model(name):
    """(GraphIR, LayerPlan, graph JSON)"""
    if name not in _CACHE:
        graph = build_graph(GRAPHS[name])
        ir = GraphIR.from_metagraph(graph)
        _CACHE[name] = (ir, compile_graph(ir, "x:0", "y:0"), graph)
    return _CACHE[name]


def sp_data(name, n, seed):
    """rows X and a [n, 1] float column of class indices; a quarter of them carry a fraction (k + 0.7 truncates to k, as
    TF's Cast does)"""
    lp = sp_model(name)[1]
    rng = np.random.default_rng(seed)
    X = rng.random((n, lp.input_dim), dtype=np.float32)
    idx = rng.integers(0, lp.layers[-1].out_features, n)
    Y = (idx + np.where(rng.random(n) < 0.25, 0.7, 0.0)).astype(np.float32)[:, None]
    return X, Y


def sp_weights(name, seed=1):
    """the graph's initializers, with small non-zero biases"""
    ir = sp_model(name)[0]
    rng = np.random.default_rng(seed + 100)
    return [w if w.ndim > 1 else (0.05 * rng.standard_normal(w.shape)).astype(np.float32)
            for w in GraphProgram(ir).init_weights(seed=seed)]


def sp_forward(lp, weights, X, Y, emulate_bf16, argmax=None, relu_mask=None, device=None, bug=None):
    """test_step_gradients._forward with the sparse softmax head: run the plan with an MSE head, whose output is the
    fp32 logits of the activation-free last layer (still attached to the graph), then take the loss in float64 against
    the truncated class indices.  ``bug``: a plausible kernel bug the tolerances must catch - 'off_by_one' (label + 1),
    'per_element' (divide by B * N instead of B), 'ignore_label' (no target term), 'wrong_row' (the previous row's label)."""
    kw = {} if device is None else dict(device=device)
    _, z, params, pools, zs = _forward(dataclasses.replace(lp, loss="mse"), weights, X, Y, emulate_bf16, argmax, relu_mask, **kw)
    B, N = z.shape
    lab = np.trunc(np.asarray(Y, np.float64).reshape(-1)).astype(np.int64)
    if bug == "off_by_one":
        lab = (lab + 1) % N
    elif bug == "wrong_row":
        lab = np.roll(lab, 1)
    lse = torch.logsumexp(z, 1)
    zl = z.gather(1, torch.as_tensor(lab, device=z.device)[:, None])[:, 0]
    per = lse if bug == "ignore_label" else lse - zl
    loss = per.sum() / (B * N if bug == "per_element" else B)
    return loss, z, params, pools, zs


def sp_oracle(lp, weights, X, Y, emulate_bf16, **kw):
    loss, _, params, _, _ = sp_forward(lp, weights, X, Y, emulate_bf16, **kw)
    return float(loss.detach()), _grads(loss, params)


# ------------------------------------------------------------------------------------------------------------------
# compiler
# ------------------------------------------------------------------------------------------------------------------
def _head(n_out=5, act=None, label_shape=(None, 1)):
    x = tf.placeholder(tf.float32, shape=[None, 20], name="x")
    y = tf.placeholder(tf.float32, shape=list(label_shape), name="y")
    return x, y, tf.layers.dense(tf.layers.dense(x, 16, activation=tf.nn.relu), n_out, activation=act)


def _idx(y, dtype=tf.int32):
    return tf.cast(tf.reshape(y, [-1]), dtype)


def _losses_api():
    x, y, logits = _head()
    tf.losses.sparse_softmax_cross_entropy(_idx(y), logits)


def _mean_add_loss():
    x, y, logits = _head()
    tf.losses.add_loss(tf.reduce_mean(tf.nn.sparse_softmax_cross_entropy_with_logits(labels=_idx(y, tf.int64), logits=logits)))


def _unit_weights():
    """a Mul by an all-ones weight vector is the unweighted loss"""
    x, y, logits = _head()
    per = tf.nn.sparse_softmax_cross_entropy_with_logits(labels=_idx(y), logits=logits)
    tf.losses.add_loss(tf.reduce_mean(tf.multiply(per, tf.constant(np.ones(1, np.float32)))))


def _squeeze_identity_casts():
    """Squeeze of axis 1, Identity / StopGradient and a chain of casts through float64 and int64"""
    x, y, logits = _head()
    idx = tf.cast(tf.cast(tf.stop_gradient(tf.identity(tf.squeeze(tf.cast(y, tf.float64), axis=1))), tf.int64), tf.int32)
    tf.losses.sparse_softmax_cross_entropy(idx, logits)


def _one_hot():
    x, y, logits = _head()
    tf.losses.softmax_cross_entropy(tf.one_hot(_idx(y), 5), logits)


def _one_hot_mean():
    x, y, logits = _head(n_out=3)
    oh = tf.one_hot(tf.cast(tf.squeeze(y, axis=1), tf.int32), 3, on_value=1.0, off_value=0.0)
    tf.losses.add_loss(tf.reduce_mean(tf.nn.softmax_cross_entropy_with_logits(labels=oh, logits=logits)))


ACCEPTED = {"losses_api": _losses_api, "mean_add_loss": _mean_add_loss, "unit_weights": _unit_weights,
            "squeeze_identity_casts": _squeeze_identity_casts, "one_hot": _one_hot, "one_hot_mean": _one_hot_mean}


@pytest.mark.parametrize("name", list(ACCEPTED) + list(GRAPHS))
def test_compiler_accepts_class_index_labels(name):
    fn = ACCEPTED.get(name) or GRAPHS[name]
    ir = GraphIR.from_metagraph(build_graph(fn))
    lp = compile_graph(ir, "x:0", "y:0")
    check_grammar(lp)
    assert lp.loss == "sparse_softmax_xent" and lp.label_dim == 1 and lp.label_name == "y:0" and not lp.target_is_input
    assert lp.layers[-1].act is None and lp.layers[-1].out_features >= 2
    assert loss_mode(lp.loss) == 4


def test_loss_kinds_map_to_explicit_heads():
    assert [loss_mode(k) for k in ("softmax_xent", "mse", "sigmoid_xent")] == [1, 2, 3]
    assert loss_mode("sparse_softmax_xent") == 4


def test_one_hot_label_columns_keep_the_dense_head():
    lp = compile_graph(GraphIR.from_metagraph(zoo.build("simple_dnn")), "x:0", "y:0")
    assert lp.loss == "softmax_xent" and lp.label_dim == 10


def _weighted_const():
    x, y, logits = _head()
    tf.losses.sparse_softmax_cross_entropy(_idx(y), logits, weights=2.0)


def _weighted_placeholder():
    x, y, logits = _head()
    w = tf.placeholder(tf.float32, shape=[None], name="w")
    tf.losses.sparse_softmax_cross_entropy(_idx(y), logits, weights=w)


def _activated_logits():
    x, y, out = _head(act=tf.nn.relu)
    tf.losses.sparse_softmax_cross_entropy(_idx(y), out)


def _one_hot_smoothed():
    x, y, logits = _head()
    tf.losses.softmax_cross_entropy(tf.one_hot(_idx(y), 5, on_value=0.92, off_value=0.02), logits)


def _one_hot_depth():
    x, y, logits = _head()
    tf.losses.softmax_cross_entropy(tf.one_hot(_idx(y), 6), logits)


def _wide_placeholder():
    x, y, logits = _head(label_shape=(None, 3))
    tf.losses.sparse_softmax_cross_entropy(_idx(y), logits)


def _rank1_placeholder():
    x, y, logits = _head(label_shape=(None,))
    tf.losses.sparse_softmax_cross_entropy(tf.cast(y, tf.int32), logits)


def _rank3_placeholder():
    x, y, logits = _head(label_shape=(None, 1, 1))
    tf.losses.sparse_softmax_cross_entropy(_idx(y), logits)


def _other_op_on_index_path():
    x, y, logits = _head()
    tf.losses.sparse_softmax_cross_entropy(_idx(tf.add(y, 1.0)), logits)


def _one_class():
    x, y, logits = _head(n_out=1)
    tf.losses.sparse_softmax_cross_entropy(_idx(y), logits)


def _sum_under_mean():
    x, y, logits = _head()
    per = tf.nn.sparse_softmax_cross_entropy_with_logits(labels=_idx(y), logits=logits)
    tf.losses.add_loss(tf.reduce_mean(tf.reduce_sum(per)))


# types a real TF-1.x MetaGraph can carry that the graph builder does not name
_BF16, _INT8, _INT16 = (tfcore.DType(n, e, t) for n, e, t in (("bfloat16", "DT_BFLOAT16", np.float32), ("int8", "DT_INT8", np.int8),
                                                               ("int16", "DT_INT16", np.int16)))


def _narrowing_cast(dtype):
    """a cast through a type that rounds or wraps large indices: bfloat16 holds 257 as 256, int8 wraps 200 to -56"""
    def fn():
        x, y, logits = _head()
        tf.losses.sparse_softmax_cross_entropy(tf.cast(tf.cast(tf.reshape(y, [-1]), dtype), tf.int32), logits)
    return fn


def _one_hot_placeholder_on_value():
    x, y, logits = _head()
    on = tf.placeholder(tf.float32, shape=[], name="on")
    idx = _idx(y)
    oh = tfops._g().add_node("OneHot", "one_hot", [idx, tfops._const_i32(5, "depth"), on, tf.constant(0.0, name="off_value")],
                             {"T": tfops.attr_type(tf.float32), "TI": tfops.attr_type(tf.int32), "axis": tfops.attr_i(-1)},
                             [tf.float32], [(None, 5)]).outputs[0]
    tf.losses.softmax_cross_entropy(oh, logits)


def _too_many_classes():
    x, y, logits = _head(n_out=MAX_SPARSE_CLASSES + 1)
    tf.losses.sparse_softmax_cross_entropy(_idx(y), logits)


@pytest.mark.parametrize("fn,match", [(_weighted_const, "weighted"), (_weighted_placeholder, "weighted"),
                                      (_activated_logits, "raw logits"), (_one_hot_smoothed, "label smoothing"),
                                      (_one_hot_depth, "depth 6"), (_wide_placeholder, "width"), (_rank1_placeholder, "rank-2"),
                                      (_rank3_placeholder, "rank-2"), (_other_op_on_index_path, "through 'Add'"),
                                      (_one_class, "at least 2 classes"), (_sum_under_mean, "sum under a mean"),
                                      (_narrowing_cast(_BF16), "DT_BFLOAT16"), (_narrowing_cast(tf.float16), "DT_HALF"),
                                      (_narrowing_cast(_INT8), "DT_INT8"), (_narrowing_cast(tf.uint8), "DT_UINT8"),
                                      (_narrowing_cast(_INT16), "DT_INT16"),
                                      (_one_hot_placeholder_on_value, "not a constant"),
                                      (_too_many_classes, f"{MAX_SPARSE_CLASSES + 1} classes")])
def test_compiler_rejects_uncovered_variants(fn, match):
    ir = GraphIR.from_metagraph(build_graph(fn))
    with pytest.raises(UnsupportedGraph, match=match):
        compile_graph(ir, "x:0", "y:0")


def test_widest_class_count_compiles():
    """MAX_SPARSE_CLASSES classes (the widest whose stand-alone loss kernel fits the default shared memory) compile"""
    def fn():
        x, y, logits = _head(n_out=MAX_SPARSE_CLASSES)
        tf.losses.sparse_softmax_cross_entropy(_idx(y), logits)

    lp = compile_graph(GraphIR.from_metagraph(build_graph(fn)), "x:0", "y:0")
    assert lp.loss == "sparse_softmax_xent" and lp.layers[-1].out_features == MAX_SPARSE_CLASSES == 48 * 1024 // 4


# ------------------------------------------------------------------------------------------------------------------
# the oracle and the tolerances
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(GRAPHS))
def test_oracle_matches_interpreter(name):
    ir, lp, _ = sp_model(name)
    X, Y = sp_data(name, 7, seed=3)
    assert (Y != np.trunc(Y)).any(), "the labels must include fractions"
    w = sp_weights(name)
    l_int, g_int = GraphProgram(ir).loss_and_grads({"x:0": X, "y:0": Y}, w)
    l_ora, g_ora = sp_oracle(lp, w, X, Y, False, device=torch.device("cpu"))
    assert abs(l_ora - l_int) <= 1e-5 * max(1.0, abs(l_int)), (l_ora, l_int)
    _assert_grads(f"{name} exact oracle vs interpreter", lp.var_order, g_ora, [g.numpy() for g in g_int], (1e-4, 1e-4))
    l_em, _ = sp_oracle(lp, w, X, Y, True, device=torch.device("cpu"))
    assert abs(l_em - l_ora) <= 2e-2 * max(1.0, abs(l_ora)), (l_em, l_ora)


@pytest.mark.parametrize("B", [7, 129])
@pytest.mark.parametrize("name", list(GRAPHS))
def test_tolerances_reject_plausible_label_bugs(name, B):
    _, lp, _ = sp_model(name)
    X, Y = sp_data(name, B, seed=11)
    w = sp_weights(name)
    cpu = dict(device=torch.device("cpu"))
    _, ref = sp_oracle(lp, w, X, Y, True, **cpu)
    tol = TOL[name]
    assert not _rejects(ref, ref, tol)
    for bug in ("off_by_one", "per_element", "ignore_label", "wrong_row"):
        _, grads = sp_oracle(lp, w, X, Y, True, bug=bug, **cpu)
        assert _rejects(grads, ref, tol), f"{name} B={B}: the tolerance {tol} accepts the gradient with the bug {bug}"


# ------------------------------------------------------------------------------------------------------------------
# the partition loader's label check
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [-1.0, 10.0, np.nan, np.inf, -np.inf, 10.5])
def test_label_check_rejects_non_class_indices(bad):
    Y = np.array([[0.0], [3.0], [9.0], [bad], [1.0]], np.float32)
    with pytest.raises(ValueError, match=r"row 3\b"):
        check_class_labels(Y, 10)


def test_label_check_accepts_class_indices():
    check_class_labels(np.array([[0.0], [9.0], [2.7], [9.99], [-0.5]], np.float32), 10)     # 2.7 -> 2, -0.5 -> 0, as TF's Cast
    check_class_labels(np.array([0.0, 1.0, 2.0], np.float32), 3)
    with pytest.raises(ValueError, match="row 0"):
        check_class_labels(np.array([[-1.0], [-2.0]], np.float32), 3)


# ------------------------------------------------------------------------------------------------------------------
# build artifacts
# ------------------------------------------------------------------------------------------------------------------
@needs_binary_utils
def test_sparse_xent_kernel_instances_have_no_stack_frame():
    """the stand-alone kernel and the SPARSE_LOSS GEMM variant (SfEpi 6), which stays within the register count of the
    sigmoid loss variant it mirrors"""
    use = res_usage()
    sparse, sigmoid = "sf::sf_gemm_kernel<32, false, 6, false, false>", "sf::sf_gemm_kernel<32, false, 5, false, false>"
    want = ["sf::sparse_softmax_xent_kernel", sparse]
    missing = [k for k in want if k not in use]
    assert not missing, (missing, sorted(use))
    spilled = {k: use[k] for k in want if use[k][1] != 0}
    assert not spilled, f"kernels with a local-memory stack frame (REG, STACK): {spilled}"
    assert use[sparse][0] <= use[sigmoid][0]
