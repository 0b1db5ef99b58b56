"""Sigmoid cross-entropy on the H100: the stand-alone ``sigmoid_xent`` kernel against PyTorch, the compiled training step
of binary / multi-label classifiers against the float64 oracle of tests/test_sigmoid_xent.py in every loss placement
(fused into the last GEMM's SIGMOID_LOSS epilogue variant, with and without its transposed dz, and the stand-alone kernel),
the forward plans, a delivered gradient through the sharded push, and training end to end."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sparkflow_b200.graph.executor import GraphProgram
from sparkflow_b200.models import zoo
from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import ParamLayout, round_up
from sparkflow_b200.ops.optimizers import OptimizerSpec
from push_helpers import wait_pushes
from test_step_gradients import (DELIVERY_TOL, VARIANTS, _assert_grads, _check_pools, _errors, _grads, _recorded_argmax,
                                 _recorded_relu_mask, _run_step)
from test_sigmoid_xent import (CNN_GRAPHS, GRAPHS, LOSS_TOL, TOL, sig_data, sig_forward, sig_model, sig_weights)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SIGMOID_LOSS = 5                                   # SfEpi (csrc/sf_api.h)
DENSE_B = (1, 7, 129, 300, 1000)
CNN_B = (1, 7, 130, 300)


# ------------------------------------------------------------------------------------------------------------------
# the stand-alone kernel
# ------------------------------------------------------------------------------------------------------------------
def _kernel_case(C, rows, cols, z):
    """run C.sigmoid_xent on logits z [rows, cols] (float32, cuda) and random 0 / 1 labels; returns the outputs and the
    float64 reference"""
    g = torch.Generator(device="cuda").manual_seed(rows * 1000 + cols)
    y = torch.randint(0, 2, (rows, cols), device="cuda", generator=g).float()
    ld_dz, ld_t = round_up(cols, 8) + 8, round_up(rows, 8)
    dz = torch.full((rows, ld_dz), 3.0, dtype=torch.bfloat16, device="cuda")      # sentinel: the tail must become 0
    dzT = torch.zeros(cols, ld_t, dtype=torch.bfloat16, device="cuda")
    dbias = torch.zeros(cols, device="cuda")
    loss = torch.zeros(1, device="cuda")
    P = native.ptr
    C.sigmoid_xent(P(z), cols, P(y), cols, P(loss), P(dz), ld_dz, P(dzT), ld_t, P(dbias), rows, cols, native.current_stream())
    torch.cuda.synchronize()
    assert C.read_error_code() == 0
    z64, y64 = z.double(), y.double()
    ref_loss = F.binary_cross_entropy_with_logits(z64, y64)
    ref_dz = (torch.sigmoid(z64) - y64) / (rows * cols)
    return dict(loss=loss, dz=dz, dzT=dzT, dbias=dbias, y=y), dict(loss=ref_loss, dz=ref_dz, dbias=ref_dz.sum(0))


def _check_bf16(tag, got, ref, n):
    """one bf16 rounding step of the reference, plus the fp32 error of sigmoid(z) - y at the gradient's scale 1 / n"""
    tol = torch.ldexp(torch.ones_like(ref), torch.frexp(ref)[1] - 8) + 1e-6 / n
    err = (got.double() - ref).abs()
    assert bool((err <= tol).all()), f"{tag}: worst |got - ref| / tol = {float((err / tol).max()):.2f}"


@pytest.mark.parametrize("rows", [1, 7, 33, 300])
@pytest.mark.parametrize("cols", [1, 5, 32, 33, 100])
def test_sigmoid_xent_kernel_matches_torch(rows, cols):
    C = native.cuda_ext()
    g = torch.Generator(device="cuda").manual_seed(rows + cols)
    z = 3.0 * torch.randn(rows, cols, device="cuda", generator=g)
    out, ref = _kernel_case(C, rows, cols, z)
    # fp32 torch on the same inputs agrees with the float64 reference used below
    t32 = F.binary_cross_entropy_with_logits(z, out["y"])
    assert abs(float(t32) - float(ref["loss"])) <= 1e-5 * float(ref["loss"])
    assert abs(float(out["loss"]) - float(ref["loss"])) <= 1e-5 * float(ref["loss"]), (float(out["loss"]), float(ref["loss"]))
    n = rows * cols
    _check_bf16("dz", out["dz"][:, :cols], ref["dz"], n)
    _check_bf16("dzT", out["dzT"][:, :rows], ref["dz"].t(), n)
    assert not bool(out["dz"][:, cols:].float().any()), "the padded tail of dz is not zero"
    assert not bool(out["dzT"][:, rows:].float().any()), "dz^T past the last row was written"
    torch.testing.assert_close(out["dbias"].double(), ref["dbias"], rtol=1e-4, atol=1e-6 / cols)


@pytest.mark.parametrize("rows,cols", [(300, 100), (33, 5)])
def test_sigmoid_xent_kernel_saturated_logits(rows, cols):
    """|z| up to 60: finite everywhere; a batch whose every element is confidently right still carries its loss
    (log1p(e) with e = exp(-|z|) down to 1e-26, where log(1 + e) would give 0)"""
    C = native.cuda_ext()
    g = torch.Generator(device="cuda").manual_seed(rows)
    z = (torch.rand(rows, cols, device="cuda", generator=g) * 2 - 1) * 60
    out, ref = _kernel_case(C, rows, cols, z)
    assert all(bool(torch.isfinite(out[k].float()).all()) for k in ("loss", "dz", "dzT", "dbias"))
    assert abs(float(out["loss"]) - float(ref["loss"])) <= 1e-5 * float(ref["loss"])
    _check_bf16("dz", out["dz"][:, :cols], ref["dz"], rows * cols)
    # every element right with |z| in [20, 60]: per-element loss exp(-|z|)
    right = (2 * out["y"] - 1) * (20 + 40 * torch.rand(rows, cols, device="cuda", generator=g))
    out, ref = _kernel_case(C, rows, cols, right.contiguous())
    assert float(ref["loss"]) > 0
    rel = abs(float(out["loss"]) - float(ref["loss"])) / float(ref["loss"])
    assert rel <= 1e-4, (float(out["loss"]), float(ref["loss"]))


# ------------------------------------------------------------------------------------------------------------------
# the training step against the oracle
# ------------------------------------------------------------------------------------------------------------------
def _sig_worker(name, weights, spec=None, push="direct", shards=2):
    """a master holding ``weights`` and one worker on cuda:0; ``push``: 'direct' or 'sharded' (``shards`` shards on the
    same GPU, Hogwild)"""
    from sparkflow_b200.parallel.device_engine import DeviceWorker, MasterState, plan_publish_needs

    ir, lp, _ = sig_model(name)
    need_w, need_wt = plan_publish_needs(lp)
    lay = ParamLayout.build(ir.param_shapes(), need_w, need_wt)
    spec = spec or OptimizerSpec.from_tf_kwargs("gradient_descent", dict(learning_rate=0.0))
    if push == "sharded":
        from sparkflow_b200.parallel.dist import DistContext
        from sparkflow_b200.parallel.sharded import ShardedMaster

        master = ShardedMaster(lay, spec, DistContext(), [DEV] * shards, mb_zero=any(l.kind == "conv" for l in lp.layers))
        master.load_weights(weights)
        master.start_applier(False)
    else:
        master = MasterState(lay, spec, DEV)
        master.load_weights(weights)
    return master, DeviceWorker(ir, "x:0", "y:0", spec, master, acquire_lock=False, shared=push == "sharded", use_graphs=False)


def _compare(tag, lp, w, X, Y, got, loss, dbg, tol):
    B = X.shape[0]
    assert np.isfinite(loss), f"{tag}: loss {loss}"
    l_ref, _, params, pools, _ = sig_forward(lp, w, X, Y, True, _recorded_argmax(lp, dbg, B), _recorded_relu_mask(lp, dbg, B))
    _check_pools(tag, lp, dbg, pools, B)
    ref = _grads(l_ref, params)
    l_ref = float(l_ref.detach())
    l_err = abs(loss - l_ref) / max(abs(l_ref), 1e-30)
    assert l_err <= LOSS_TOL, f"{tag}: loss {loss} vs {l_ref} (relative error {l_err:.2e})"
    fro, mx = _assert_grads(tag, lp.var_order, got, ref, tol)
    print(f"[sigmoid-xent] {tag}: rel-Frobenius {fro:.2e} max-abs {mx:.2e} loss {l_err:.2e}")
    return fro, mx, l_err


def _check_variant(tag, variant, names, worker):
    """the loss ran where the variant puts it: a '+loss' GEMM iff fused, the 'sigmoid_xent' kernel iff not; the fused
    GEMM always runs the SIGMOID_LOSS variant (it also writes the transposed dz of the K-major path)"""
    base = [n.split("@")[0] for n in names]
    fused = variant != "unfused_loss"
    assert any(n.endswith("+loss") for n in base) == fused, (tag, names)
    assert ("sigmoid_xent" in base) != fused, (tag, names)
    assert "mse" not in base and "softmax_xent" not in base, (tag, names)
    gemms = [g for grp in worker._keep[-1] if isinstance(grp, list) for g in grp if hasattr(g, "epi")]
    assert any(g.epi == SIGMOID_LOSS for g in gemms) == fused, (tag, [g.epi for g in gemms])


STEP_CASES = [(m, v) for m in GRAPHS for v in ("default", "unfused_loss", "kmajor_wgrad") if not (m in CNN_GRAPHS and v == "kmajor_wgrad")]


@pytest.mark.parametrize("name,variant", STEP_CASES)
def test_step_gradients_match_oracle(name, variant, monkeypatch):
    """one step without push, staged and in-graph feeds: the flat gradient buffer and the loss against the
    bf16-emulating oracle"""
    for k, v in VARIANTS[variant].items():
        monkeypatch.setenv(k, v)
    _, lp, _ = sig_model(name)
    w = sig_weights(name)
    master, worker = _sig_worker(name, w)
    try:
        for B in (CNN_B if name in CNN_GRAPHS else DENSE_B):
            X, Y = sig_data(name, B, seed=B)
            for feed in ("staged", "in_graph"):
                got, loss, dbg, names = _run_step(worker, B, X, Y, feed)
                tag = f"{name}/{variant} B={B} {feed}"
                _check_variant(tag, variant, names, worker)
                _compare(tag, lp, w, X, Y, got, loss, dbg, TOL[name])
    finally:
        master.close()


@pytest.mark.parametrize("name", list(GRAPHS))
def test_forward_plans_match_oracle(name):
    """the forward + loss plan (stand-alone kernel) gives the oracle's loss"""
    _, lp, _ = sig_model(name)
    w = sig_weights(name)
    B = 129
    X, Y = sig_data(name, B, seed=41)
    with torch.no_grad():
        l_ref = float(sig_forward(lp, w, X, Y, True)[0])
    master, worker = _sig_worker(name, w)
    try:
        plan, bufs = worker.build_forward_plan(B, with_loss=True, with_pull=True)
        with torch.cuda.stream(worker.stream):
            bufs.x_stage.copy_(torch.from_numpy(X))
            bufs.y_stage.copy_(torch.from_numpy(Y))
            bufs.loss_out.zero_()
            plan.run(worker.stream.cuda_stream)
        worker.stream.synchronize()
        loss = float(bufs.loss_out[0])
        assert abs(loss - l_ref) <= LOSS_TOL * abs(l_ref), (loss, l_ref)
    finally:
        master.close()


@pytest.mark.parametrize("name", ["binary_dnn", "multilabel_dnn"])
def test_inference_runs_the_compiled_forward_plan(name, monkeypatch):
    from sparkflow_b200.ml_util import run_inference

    ir, _, graph = sig_model(name)
    w = sig_weights(name, seed=4)
    X, _ = sig_data(name, 300, seed=9)
    ref = GraphProgram(ir, "cuda").forward("out:0", {"x:0": X}, w).detach().cpu().numpy()

    def no_interpreter(*a, **k):
        raise AssertionError("prediction fell back to the interpreter")

    monkeypatch.setattr(GraphProgram, "forward", no_interpreter)
    got = run_inference(graph, w, X, "x:0", "out:0")
    assert got.size == ref.size, (got.shape, ref.shape)
    assert np.abs(got.reshape(ref.shape) - ref).max() < 1e-2, np.abs(got.reshape(ref.shape) - ref).max()


@pytest.mark.parametrize("name", ["multilabel_dnn", "logreg"])
def test_delivered_gradients_match_oracle(name):
    """through the sharded push (two Hogwild shards on one GPU): the momentum-0 tap leaves slot 0 equal to the gradient
    the appliers consumed, step by step, against the oracle and the same step without push.  logreg's only GEMM is the
    fused-loss one, so it also carries the read-your-writes wait (no pull kernel)."""
    _, lp, _ = sig_model(name)
    w = sig_weights(name)
    Bs = (1, 7, 129, 300, 7)
    X, Y = sig_data(name, sum(Bs), seed=51)
    cuts = np.cumsum((0,) + Bs)
    master, worker = _sig_worker(name, w)
    try:
        plain = [_run_step(worker, B, X[cuts[k]:cuts[k + 1]], Y[cuts[k]:cuts[k + 1]], "in_graph")[0] for k, B in enumerate(Bs)]
    finally:
        master.close()
    spec = OptimizerSpec.from_tf_kwargs("momentum", dict(learning_rate=0.0, momentum=0.0))
    master, worker = _sig_worker(name, w, spec, push="sharded")
    dbgs = {}
    try:
        for k, B in enumerate(Bs):
            rows = slice(cuts[k], cuts[k + 1])
            plan, bufs = worker.build_plan(B, 0, with_pull=True, with_push=True)
            if B not in dbgs:
                dbgs[B] = worker.last_debug
                names = [n.split("@")[0] for n in worker.last_plan_names()]
                assert not any(n.startswith("pull") or n.startswith("sync_pull") for n in names), names
                assert any(n.endswith("+loss") for n in names), names
            with torch.cuda.stream(worker.stream):
                bufs.x_stage.copy_(torch.from_numpy(X[rows]))
                bufs.y_stage.copy_(torch.from_numpy(Y[rows]))
                plan.run(worker.stream.cuda_stream)
            worker.drain()
            assert wait_pushes(master, k + 1) == k + 1
            got = master.slot_arrays()[0]
            _compare(f"{name}/sharded2 step {k} B={B}", lp, w, X[rows], Y[rows], got, float(bufs.loss_out[0]), dbgs[B], TOL[name])
            delivery = max(_errors(g, r)[0] for g, r in zip(got, plain[k]))
            assert delivery <= DELIVERY_TOL, f"step {k}: the delivered gradient differs from the step's own by {delivery:.2e}"
        for a, b, v in zip(master.weights(), w, lp.var_order):
            assert np.array_equal(a, b), f"{v} moved under a zero learning rate"
    finally:
        master.close()


# ------------------------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lock", [False, True])
def test_session_trains_binary_dnn_natively(lock):
    from sparkflow_b200.parallel.session import TrainingSession

    rng = np.random.default_rng(3)
    centers = rng.random((2, 784), dtype=np.float32)
    lab = rng.integers(0, 2, 1200)
    X = np.clip(centers[lab] + 0.2 * rng.normal(0, 1, (1200, 784)), 0, 1).astype(np.float32)
    Y = lab.astype(np.float32)[:, None]
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    sess = TrainingSession(zoo.build("binary_dnn"), "x:0", "y:0", spec, acquire_lock=lock, engine="b200", seed=0, devices=[0]).open()
    try:
        assert sess.engine_kind == "b200"
        eng = sess.make_engine(torch.device("cuda", 0))
        eng.load_partition(X, Y)
        l0 = eng.partition_loss()
        for k in range(12):
            eng.train(slice((k % 4) * 300, (k % 4) * 300 + 300), pull=True)
        eng.finish()
        l1 = eng.partition_loss()
        assert np.isfinite(l1) and l1 < 0.5 * l0, (l0, l1)
        assert sess.counters()["pushes"] == 12
    finally:
        sess.close()


def test_spark_async_dl_fits_sigmoid_cross_entropy_natively(capfd):
    """the reference suite's two-Gaussian data through SparkAsyncDL with tf.losses.sigmoid_cross_entropy"""
    from sparkflow_b200 import compat

    compat.install()
    import tensorflow as tf
    from pyspark.ml.linalg import Vectors
    from pyspark.sql import SparkSession
    from sparkflow.graph_utils import build_graph
    from sparkflow.tensorflow_async import SparkAsyncDL
    from sparkflow_b200.parallel.session import ENGINE_USES

    def create_model():
        x = tf.placeholder(tf.float32, shape=[None, 10], name="x")
        layer1 = tf.layers.dense(x, 12, activation=tf.nn.relu)
        layer2 = tf.layers.dense(layer1, 7, activation=tf.nn.relu)
        logits = tf.layers.dense(layer2, 1, name="outer")
        tf.nn.sigmoid(logits, name="prob")
        y = tf.placeholder(tf.float32, shape=[None, 1], name="y")
        return tf.losses.sigmoid_cross_entropy(y, logits)

    rng = np.random.default_rng(12345)
    dat = [(1.0, Vectors.dense(rng.normal(0, 1, 10))) for _ in range(200)]
    dat += [(0.0, Vectors.dense(rng.normal(2, 1, 10))) for _ in range(200)]
    dat = [dat[i] for i in rng.permutation(len(dat))]
    spark = SparkSession.builder.master("local[2]").appName("sparkflow").getOrCreate()
    try:
        processed = spark.createDataFrame(dat, ["label", "features"])
        before = ENGINE_USES["b200"]
        model = SparkAsyncDL(inputCol="features", tensorflowGraph=build_graph(create_model), tfInput="x:0", tfLabel="y:0",
                             tfOutput="prob:0", tfOptimizer="adam", tfLearningRate=.1, iters=20, partitions=2,
                             predictionCol="predicted", labelCol="label").fit(processed)
        data = model.transform(processed).take(10)
    finally:
        spark.stop()
    assert ENGINE_USES["b200"] > before, dict(ENGINE_USES)
    assert "engine=torch" not in capfd.readouterr().err
    wrong = sum(1 for d in data if (1 if d["predicted"] >= 0.5 else 0) != d["label"])
    assert wrong < 2, wrong
