"""Sparse softmax cross-entropy on the H100: the stand-alone kernel (``softmax_xent`` with a label row narrower than the
logits) against PyTorch and against the dense kernel fed the one-hot of the same labels; the SPARSE_LOSS GEMM epilogue
against the dense softmax head; the compiled training step of the zoo models against the float64 oracle of
tests/test_sparse_xent.py in every loss placement and feed; training and prediction end to end; and the host's label
check ahead of any kernel."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sparkflow_b200.graph.executor import GraphProgram
from sparkflow_b200.models import zoo
from sparkflow_b200.models.compiler import MAX_SPARSE_CLASSES
from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import ParamLayout, round_up
from sparkflow_b200.ops.optimizers import OptimizerSpec
from test_step_gradients import VARIANTS, _assert_grads, _check_pools, _grads, _recorded_argmax, _recorded_relu_mask, _run_step
from test_sparse_xent import CNN_GRAPHS, GRAPHS, LOSS_TOL, TOL, sp_data, sp_forward, sp_model, sp_weights

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SPARSE_LOSS = 6                                    # SfEpi (csrc/sf_api.h)
DENSE_B = (1, 7, 129, 300, 1000)
CNN_B = (1, 7, 130, 300)


# ------------------------------------------------------------------------------------------------------------------
# the stand-alone kernel
# ------------------------------------------------------------------------------------------------------------------
def _run_xent(C, z, labels, ld_labels, rows, cols):
    ld_dz, ld_t = round_up(cols, 8) + 8, round_up(rows, 8)
    dz = torch.full((rows, ld_dz), 3.0, dtype=torch.bfloat16, device="cuda")      # sentinel: the tail must become 0
    dzT = torch.zeros(cols, ld_t, dtype=torch.bfloat16, device="cuda")
    dbias = torch.zeros(cols, device="cuda")
    loss = torch.zeros(1, device="cuda")
    P = native.ptr
    C.softmax_xent(P(z), cols, P(labels), ld_labels, P(loss), P(dz), ld_dz, P(dzT), ld_t, P(dbias), rows, cols, native.current_stream())
    torch.cuda.synchronize()
    assert C.read_error_code() == 0
    return dict(loss=loss, dz=dz, dzT=dzT, dbias=dbias)


@pytest.mark.parametrize("rows", [1, 7, 33, 300])
@pytest.mark.parametrize("cols", [2, 10, 33, 100, 1000])
def test_sparse_kernel_matches_torch_and_the_dense_kernel(rows, cols):
    C = native.cuda_ext()
    g = torch.Generator(device="cuda").manual_seed(rows * 7 + cols)
    z = 3.0 * torch.randn(rows, cols, device="cuda", generator=g)
    idx = torch.randint(0, cols, (rows,), device="cuda", generator=g)
    # labels as ml_util feeds them: one float per row; a fraction truncates toward zero
    lab = (idx.float() + 0.7 * (torch.rand(rows, device="cuda", generator=g) < 0.3).float())[:, None].contiguous()
    out = _run_xent(C, z, lab, 1, rows, cols)
    ref_loss = F.cross_entropy(z, idx)                                           # fp32 torch
    ref_dz = (torch.softmax(z, 1) - F.one_hot(idx, cols).float()) / rows
    assert abs(float(out["loss"]) - float(ref_loss)) <= 1e-5 * max(1.0, float(ref_loss)), (float(out["loss"]), float(ref_loss))
    torch.testing.assert_close(out["dz"][:, :cols].float(), ref_dz, rtol=1e-2, atol=1e-6 / rows)
    torch.testing.assert_close(out["dzT"][:, :rows].float().t(), ref_dz, rtol=1e-2, atol=1e-6 / rows)
    assert not bool(out["dz"][:, cols:].float().any()), "the padded tail of dz is not zero"
    torch.testing.assert_close(out["dbias"], ref_dz.sum(0), rtol=1e-3, atol=1e-5 / rows)
    # the dense kernel on the one-hot of the same labels computes the same values
    dense = _run_xent(C, z, F.one_hot(idx, cols).float().contiguous(), cols, rows, cols)
    assert abs(float(out["loss"]) - float(dense["loss"])) <= 2e-6 * max(1.0, abs(float(dense["loss"])))
    for k in ("dz", "dzT"):
        torch.testing.assert_close(out[k].float(), dense[k].float(), rtol=8e-3, atol=1e-7)
    torch.testing.assert_close(out["dbias"], dense["dbias"], rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("rows", [7, 300])
def test_sparse_kernel_at_the_widest_compiled_class_count(rows):
    """MAX_SPARSE_CLASSES columns: the bias-gradient row fills the default 48 KB of shared memory and the launch works"""
    C = native.cuda_ext()
    cols = MAX_SPARSE_CLASSES
    g = torch.Generator(device="cuda").manual_seed(rows)
    z = 3.0 * torch.randn(rows, cols, device="cuda", generator=g)
    idx = torch.randint(0, cols, (rows,), device="cuda", generator=g)
    out = _run_xent(C, z, idx.float()[:, None].contiguous(), 1, rows, cols)
    ref_loss = F.cross_entropy(z, idx)
    ref_dz = (torch.softmax(z, 1) - F.one_hot(idx, cols).float()) / rows
    assert abs(float(out["loss"]) - float(ref_loss)) <= 1e-5 * max(1.0, float(ref_loss)), (float(out["loss"]), float(ref_loss))
    torch.testing.assert_close(out["dz"][:, :cols].float(), ref_dz, rtol=1e-2, atol=1e-6 / rows)
    torch.testing.assert_close(out["dbias"], ref_dz.sum(0), rtol=1e-3, atol=1e-5 / rows)


# ------------------------------------------------------------------------------------------------------------------
# the fused epilogue
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 129, 300])
@pytest.mark.parametrize("N", [2, 10, 32])
@pytest.mark.parametrize("with_t", [False, True], ids=["mn_major_step", "k_major_step"])
def test_fused_sparse_head_matches_the_dense_head(M, N, with_t):
    """loss_mode 4 on class indices against loss_mode 1 on their one-hot rows; with_t: the transposed dz the K-major
    weight-gradient path reads (the dense head then runs on the generic kernel), without it the MN-major path's GEMM"""
    C = native.cuda_ext()
    K = 256
    g = torch.Generator(device="cuda").manual_seed(M + N)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.3).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.3).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    idx = torch.randint(0, N, (M,), device="cuda", generator=g)
    P = native.ptr

    def run(mode, target, ld_target):
        ldn, ldt = round_up(N, 8), round_up(M, 8)
        dz = torch.full((M, ldn), 3.0, dtype=torch.bfloat16, device="cuda")
        dzT = torch.zeros(N, ldt, dtype=torch.bfloat16, device="cuda") if with_t else None
        db, loss = torch.zeros(N, device="cuda"), torch.zeros(1, device="cuda")
        gm = C.Gemm(dict(a=P(a), b=P(w), M=M, N=N, K=K, lda=K, ldb=K, bias=P(bias), loss_mode=mode, target=P(target),
                         ld_target=ld_target, loss=P(loss), out_bf16=P(dz), ld_bf16=ldn, outT_bf16=P(dzT) if with_t else 0,
                         ld_t=ldt if with_t else 0, colsum=P(db)))
        gm.launch(native.current_stream())
        torch.cuda.synchronize()
        assert C.read_error_code() == 0
        return gm, dict(loss=loss, dz=dz, dzT=dzT, db=db)

    gs, sp = run(4, (idx.float() + 0.5)[:, None].contiguous(), 1)
    _, de = run(1, F.one_hot(idx, N).float().contiguous(), N)
    assert gs.epi == SPARSE_LOSS, gs.epi
    assert abs(float(sp["loss"]) - float(de["loss"])) <= 2e-6 * max(1.0, abs(float(de["loss"])))
    torch.testing.assert_close(sp["dz"].float(), de["dz"].float(), rtol=8e-3, atol=1e-7)
    assert not bool(sp["dz"][:, N:].float().any())
    if with_t:
        torch.testing.assert_close(sp["dzT"].float(), de["dzT"].float(), rtol=8e-3, atol=1e-7)
    torch.testing.assert_close(sp["db"], de["db"], rtol=1e-5, atol=1e-7)


def test_fused_sparse_head_refuses_what_it_does_not_cover():
    """N > 32 (the row must fit one epilogue chunk) and an activation on the logits"""
    C = native.cuda_ext()
    a = torch.zeros(64, 64, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(40, 64, dtype=torch.bfloat16, device="cuda")
    t, loss, dz = torch.zeros(64, 1, device="cuda"), torch.zeros(1, device="cuda"), torch.zeros(64, 40, dtype=torch.bfloat16, device="cuda")
    P = native.ptr
    base = dict(a=P(a), b=P(w), M=64, K=64, lda=64, ldb=64, loss_mode=4, target=P(t), ld_target=1, loss=P(loss), out_bf16=P(dz), ld_bf16=40)
    with pytest.raises(RuntimeError, match="sf_gemm_prepare"):
        C.Gemm(dict(base, N=40))
    with pytest.raises(RuntimeError, match="sf_gemm_prepare"):
        C.Gemm(dict(base, N=10, act=1))


# ------------------------------------------------------------------------------------------------------------------
# the training step against the oracle
# ------------------------------------------------------------------------------------------------------------------
def _sp_worker(name, weights, lock=False):
    """a master holding ``weights`` and one worker on cuda:0; ``lock``: the worker's pull takes the read lock and copies a
    snapshot (lock mode), otherwise it pulls without the lock (Hogwild)"""
    from sparkflow_b200.parallel.device_engine import DeviceWorker, MasterState, plan_publish_needs

    ir, lp, _ = sp_model(name)
    need_w, need_wt = plan_publish_needs(lp)
    lay = ParamLayout.build(ir.param_shapes(), need_w, need_wt)
    spec = OptimizerSpec.from_tf_kwargs("gradient_descent", dict(learning_rate=0.0))
    master = MasterState(lay, spec, DEV)
    master.load_weights(weights)
    worker = DeviceWorker(ir, "x:0", "y:0", spec, master, acquire_lock=lock, use_graphs=False)
    assert worker.lock_mode == (1 if lock else 0)
    return master, worker


def _compare(tag, lp, w, X, Y, got, loss, dbg, tol):
    B = X.shape[0]
    assert np.isfinite(loss), f"{tag}: loss {loss}"
    l_ref, _, params, pools, _ = sp_forward(lp, w, X, Y, True, _recorded_argmax(lp, dbg, B), _recorded_relu_mask(lp, dbg, B))
    _check_pools(tag, lp, dbg, pools, B)
    ref = _grads(l_ref, params)
    l_ref = float(l_ref.detach())
    l_err = abs(loss - l_ref) / max(abs(l_ref), 1e-30)
    assert l_err <= LOSS_TOL, f"{tag}: loss {loss} vs {l_ref} (relative error {l_err:.2e})"
    fro, mx = _assert_grads(tag, lp.var_order, got, ref, tol)
    print(f"[sparse-xent] {tag}: rel-Frobenius {fro:.2e} max-abs {mx:.2e} loss {l_err:.2e}")


def _check_variant(tag, lp, variant, names, worker):
    """a '+loss' GEMM on the SPARSE_LOSS variant iff fused (N <= 32), the stand-alone 'softmax_xent' op iff not"""
    base = [n.split("@")[0] for n in names]
    fused = variant != "unfused_loss" and lp.layers[-1].out_features <= 32
    assert any(n.endswith("+loss") for n in base) == fused, (tag, names)
    assert ("softmax_xent" in base) != fused, (tag, names)
    gemms = [g for grp in worker._keep[-1] if isinstance(grp, list) for g in grp if hasattr(g, "epi")]
    assert any(g.epi == SPARSE_LOSS for g in gemms) == fused, (tag, [g.epi for g in gemms])


STEP_CASES = [(m, v) for m in GRAPHS for v in ("default", "unfused_loss", "kmajor_wgrad")]


@pytest.mark.parametrize("lock", [False, True], ids=["hogwild", "lock"])
@pytest.mark.parametrize("name,variant", STEP_CASES)
def test_step_gradients_match_oracle(name, variant, lock, monkeypatch):
    """one step (pull, no push), staged and in-graph feeds, with the lock on and off: the flat gradient buffer and the loss
    against the bf16-emulating oracle"""
    for k, v in VARIANTS[variant].items():
        monkeypatch.setenv(k, v)
    _, lp, _ = sp_model(name)
    w = sp_weights(name)
    master, worker = _sp_worker(name, w, lock)
    try:
        for B in (CNN_B if name in CNN_GRAPHS else DENSE_B):
            X, Y = sp_data(name, B, seed=B)
            for feed in ("staged", "in_graph"):
                got, loss, dbg, names = _run_step(worker, B, X, Y, feed)
                tag = f"{name}/{variant} B={B} {feed}{' lock' if lock else ''}"
                _check_variant(tag, lp, variant, names, worker)
                _compare(tag, lp, w, X, Y, got, loss, dbg, TOL[name])
    finally:
        master.close()


@pytest.mark.parametrize("lock", [False, True], ids=["hogwild", "lock"])
@pytest.mark.parametrize("name", list(GRAPHS))
def test_resident_gather_step_matches_oracle(name, lock):
    """HBM-resident partition: the prep plan gathers the [n, 1] label column with the permuted rows"""
    _, lp, _ = sp_model(name)
    w = sp_weights(name)
    master, worker = _sp_worker(name, w, lock)
    try:
        B = 129
        X, Y = sp_data(name, 3 * B + 5, seed=21)
        rows = np.random.default_rng(5).permutation(X.shape[0])[:B]
        perm = torch.from_numpy(rows.astype(np.int32)).to(DEV)
        got, loss, dbg, names = _run_step(worker, B, torch.from_numpy(X).to(DEV), torch.from_numpy(Y).to(DEV), "resident", perm)
        _compare(f"{name} resident B={B}{' lock' if lock else ''}", lp, w, X[rows], Y[rows], got, loss, dbg, TOL[name])
    finally:
        master.close()


@pytest.mark.parametrize("name", list(GRAPHS))
def test_forward_plans_match_oracle(name):
    """the forward + loss plan (stand-alone kernel) gives the oracle's loss"""
    _, lp, _ = sp_model(name)
    w = sp_weights(name)
    B = 129
    X, Y = sp_data(name, B, seed=41)
    with torch.no_grad():
        l_ref = float(sp_forward(lp, w, X, Y, True)[0])
    master, worker = _sp_worker(name, w)
    try:
        plan, bufs = worker.build_forward_plan(B, with_loss=True, with_pull=True)
        assert "softmax_xent" in [n.split("@")[0] for n in plan.names()]
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


# ------------------------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------------------------
def _clusters(n, classes, seed):
    rng = np.random.default_rng(seed)
    centers = rng.random((classes, 784), dtype=np.float32)
    lab = rng.integers(0, classes, n)
    X = np.clip(centers[lab] + 0.2 * rng.normal(0, 1, (n, 784)), 0, 1).astype(np.float32)
    return X, lab.astype(np.float32)[:, None]


@pytest.mark.parametrize("mode", ["pinned", "resident"])
@pytest.mark.parametrize("lock", [False, True])
@pytest.mark.parametrize("name", ["sparse_dnn", "sparse_dnn100"])
def test_session_trains_class_index_labels_natively(name, lock, mode, monkeypatch):
    from sparkflow_b200.parallel.session import TrainingSession

    monkeypatch.setenv("SPARKFLOW_PARTITION", mode)
    X, Y = _clusters(1200, 10, seed=3)
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.002))
    sess = TrainingSession(zoo.build(name), "x:0", "y:0", spec, acquire_lock=lock, engine="b200", seed=0, devices=[0]).open()
    try:
        assert sess.engine_kind == "b200"
        eng = sess.make_engine(torch.device("cuda", 0))
        eng.load_partition(X, Y)
        assert eng.resident == (mode == "resident")
        l0 = eng.partition_loss()
        for k in range(12):
            eng.train(slice((k % 4) * 300, (k % 4) * 300 + 300), pull=True)
        eng.finish()
        l1 = eng.partition_loss()
        assert np.isfinite(l1) and l1 < 0.7 * l0, (l0, l1)
        assert sess.counters()["pushes"] == 12
    finally:
        sess.close()


def test_out_of_range_label_is_refused_on_the_host():
    """a label outside [0, N) raises from load_partition, before the partition reaches the device"""
    from sparkflow_b200.parallel.session import TrainingSession

    X, Y = _clusters(600, 10, seed=4)
    Y[417, 0] = 10.0
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    sess = TrainingSession(zoo.build("sparse_dnn"), "x:0", "y:0", spec, engine="b200", seed=0, devices=[0]).open()
    try:
        eng = sess.make_engine(torch.device("cuda", 0))
        with pytest.raises(ValueError, match=r"label 10\.0 of row 417 "):
            eng.load_partition(X, Y)
        assert eng.Xd is None
        assert native.cuda_ext().read_error_code() == 0
    finally:
        sess.close()


def test_spark_async_dl_fits_a_numeric_label_column_natively(capfd, monkeypatch):
    """SparkAsyncDL on sparse_dnn with the label column as it comes out of a StringIndexer (a double per row): trains on
    the native engine, and prediction runs the compiled forward plan"""
    from sparkflow_b200 import compat

    compat.install()
    from pyspark.ml.linalg import Vectors
    from pyspark.sql import SparkSession
    from sparkflow.tensorflow_async import SparkAsyncDL
    from sparkflow_b200.parallel.session import ENGINE_USES

    X, Y = _clusters(600, 10, seed=12345)
    dat = [(float(y[0]), Vectors.dense(x)) for x, y in zip(X, Y)]
    spark = SparkSession.builder.master("local[2]").appName("sparkflow").getOrCreate()
    try:
        processed = spark.createDataFrame(dat, ["label", "features"])
        before = ENGINE_USES["b200"]
        model = SparkAsyncDL(inputCol="features", tensorflowGraph=zoo.build("sparse_dnn"), tfInput="x:0", tfLabel="y:0",
                             tfOutput="out:0", tfOptimizer="adam", tfLearningRate=.005, iters=30, partitions=2,
                             predictionCol="predicted", labelCol="label").fit(processed)

        def no_interpreter(*a, **k):
            raise AssertionError("prediction fell back to the interpreter")

        monkeypatch.setattr(GraphProgram, "forward", no_interpreter)
        data = model.transform(processed).take(100)
    finally:
        spark.stop()
    assert ENGINE_USES["b200"] > before, dict(ENGINE_USES)
    assert "engine=torch" not in capfd.readouterr().err
    wrong = sum(1 for d in data if int(d["predicted"]) != int(d["label"]))
    assert wrong <= 10, wrong
