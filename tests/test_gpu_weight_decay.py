"""L2 weight penalties on the H100: the penalised weight-gradient GEMM against float64 (2c * W added exactly once, the bias
term into a pre-filled gradient, the loss term), the compiled training step of the three zoo models against the float64
penalty oracle of tests/test_weight_decay.py in every plan variant, the gradients and loss the served and sharded push
paths deliver, a five-step update, partition_loss, and training through the session API."""
import io
import contextlib

import numpy as np
import pytest
import torch

from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import round_up
from sparkflow_b200.ops.optimizers import OptimizerSpec
from push_helpers import wait_pushes
from test_step_gradients import (UPDATE_TOL as UPDATE_TOL_DEFAULT, VARIANTS, _assert_grads, _check_pools, _recorded_argmax, _recorded_relu_mask, _run_step,
                                 _worker)
from test_weight_decay import L2_MODELS, LOSS_TOL, TOL, l2_data, l2_model, l2_weights, penalty_oracle

pytestmark = pytest.mark.gpu

GENERIC, WGRAD = 0, 4                             # SfEpi (csrc/sf_api.h)
DENSE_B = (1, 7, 129, 300, 1000)
# five-step update, relative Frobenius: the step tests' bound (2e-3), except where about 3x the worst error measured on
# an H100 80GB HBM3 (700 W power limit) is above it.  l2_cnn's SAME-padded convs carry cnn_same's larger per-step error
# into the update; Adam divides by sqrt(v), which magnifies the error of the small gradient elements.
UPDATE_TOL = {                           # measured
    ("l2_cnn", "gradient_descent"): 2.5e-2,    # 8.3e-3
    ("l2_cnn", "momentum"): 1.1e-2,            # 3.6e-3
    ("l2_cnn", "adam"): 1.3e-2,                # 4.3e-3
    ("l2_dnn", "adam"): 7e-3,                  # 2.2e-3
}
CNN_B = (1, 7, 130, 300)


# ------------------------------------------------------------------------------------------------------------------
# the penalised weight-gradient GEMM
# ------------------------------------------------------------------------------------------------------------------
# (M, N, K, mn_major, bn, W^T source, split_k): BN 64 / 128 MN-major (the WGRAD variant, also split), the generic kernel
# K-major at every width, with and without a K split (accumulate), with W and W^T sources
GEMM_CASES = [(300, 200, 129, True, 64, False, 1), (300, 200, 129, True, 128, True, 1), (520, 70, 1000, True, 64, False, 4),
              (520, 70, 1000, True, 128, True, 3), (300, 200, 129, False, 32, False, 1), (300, 200, 129, False, 64, True, 1),
              (257, 300, 700, False, 128, False, 3), (257, 300, 700, False, 256, True, 1)]


@pytest.mark.parametrize("M,N,K,mn,bn,wt,split_k", GEMM_CASES)
def test_penalised_wgrad_gemm_matches_float64(M, N, K, mn, bn, wt, split_k):
    C = native.cuda_ext()
    P = native.ptr
    g = torch.Generator(device="cuda").manual_seed(M + N + K + bn)
    a = torch.randn(K, M, device="cuda", generator=g).to(torch.bfloat16)          # a^T . b, the weight-gradient form
    b = torch.randn(K, N, device="cuda", generator=g).to(torch.bfloat16)
    if mn:
        A = torch.zeros(K, round_up(M, 8), dtype=torch.bfloat16, device="cuda")
        B = torch.zeros(K, round_up(N, 8), dtype=torch.bfloat16, device="cuda")
        A[:, :M], B[:, :N] = a, b
    else:
        A = torch.zeros(M, round_up(K, 8), dtype=torch.bfloat16, device="cuda")
        B = torch.zeros(N, round_up(K, 8), dtype=torch.bfloat16, device="cuda")
        A[:, :K], B[:, :K] = a.t(), b.t()
    W = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
    ldw = round_up(M if wt else N, 8) + 8
    Wsrc = torch.full((N if wt else M, ldw), float("nan"), dtype=torch.bfloat16, device="cuda")       # padding never read
    if wt:
        Wsrc[:, :M] = W.t()
    else:
        Wsrc[:, :N] = W
    bias = torch.randn(N, device="cuda", generator=g)
    init = torch.randn(M, N, device="cuda", generator=g)
    db0 = torch.randn(N, device="cuda", generator=g)
    c, cb = 0.75, 0.3
    out, db = init.clone(), db0.clone()
    loss = torch.full((1,), 0.5, device="cuda")
    d = dict(a=P(A), lda=A.shape[1], b=P(B), ldb=B.shape[1], M=M, N=N, K=K, mn_major=int(mn), bn=bn, split_k=split_k, pair=0,
             out_f32=P(out), ld_f32=N, accumulate=1, pen_w=P(Wsrc), pen_ld=ldw, pen_wt=int(wt), pen_w2c=2 * c, pen_b=P(bias),
             pen_b2c=2 * cb, pen_db=P(db), pen_loss=P(loss))
    gm = C.Gemm(d)
    tag = f"{M}x{N}x{K} mn={mn} bn={bn} wt={wt} split_k={split_k}"
    assert gm.bn == bn and gm.split_k == split_k and gm.pair == 0, tag
    assert gm.epi == (WGRAD if mn else GENERIC), tag
    gm.launch(native.current_stream())
    torch.cuda.synchronize()
    assert C.read_error_code() == 0, tag
    a64, b64, w64 = a.double(), b.double(), W.double()
    ref = init.double() + a64.t() @ b64 + 2 * c * w64
    scale = float((a64.abs().t() @ b64.abs()).max())
    # the term is added exactly once: a second or missing 2c * W (|W| ~ 1) is ~1.5 off, far above the fp32 error
    err = float((out.double() - ref).abs().max())
    assert err <= 2e-6 * scale + 1e-5, f"{tag}: max error {err:.2e} (scale {scale:.1f})"
    torch.testing.assert_close(db.double(), db0.double() + 2 * cb * bias.double(), rtol=1e-6, atol=1e-6, msg=tag)
    want = 0.5 + c * float((w64 * w64).sum()) + cb * float((bias.double() ** 2).sum())
    assert abs(float(loss) - want) <= 1e-5 * want, f"{tag}: loss {float(loss)} vs {want}"


@pytest.mark.parametrize("mn,split_k", [(True, 1), (True, 3), (False, 1), (False, 3)])
def test_penalised_wgrad_gemm_routes_into_mailboxes(mn, split_k):
    """Route mode (the sharded push fused into the wgrad epilogue): each 32 x 64 push tile of dW + 2c W lands in the
    mailbox of the shard that owns it, added exactly once before the store (K split 0) or the red (split-K), and nothing
    lands anywhere else.  Three shards own unequal runs of tiles; the gradient sits at an offset inside the flat
    mailboxes, as a variable after the first would."""
    C = native.cuda_ext()
    P = native.ptr
    M, N, K, off = 200, 150, 700, 96
    g = torch.Generator(device="cuda").manual_seed(11 + split_k + 2 * mn)
    a = torch.randn(K, M, device="cuda", generator=g).to(torch.bfloat16)
    b = torch.randn(K, N, device="cuda", generator=g).to(torch.bfloat16)
    if mn:
        A = torch.zeros(K, round_up(M, 8), dtype=torch.bfloat16, device="cuda")
        B = torch.zeros(K, round_up(N, 8), dtype=torch.bfloat16, device="cuda")
        A[:, :M], B[:, :N] = a, b
    else:
        A = torch.zeros(M, round_up(K, 8), dtype=torch.bfloat16, device="cuda")
        B = torch.zeros(N, round_up(K, 8), dtype=torch.bfloat16, device="cuda")
        A[:, :K], B[:, :K] = a.t(), b.t()
    W = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
    Wt = torch.zeros(N, round_up(M, 8), dtype=torch.bfloat16, device="cuda")
    Wt[:, :M] = W.t()
    tiles_c = (N + 63) // 64
    n_tiles = ((M + 31) // 32) * tiles_c
    bounds = [0, 5, 6, n_tiles]
    total = off + M * N + 64
    boxes = [torch.zeros(total, device="cuda") for _ in range(3)]
    route = torch.frombuffer(bytearray(C.pack_route(3, bounds, [P(x) for x in boxes])), dtype=torch.uint8).cuda()
    c = 0.75
    loss = torch.zeros(1, device="cuda")
    d = dict(a=P(A), lda=A.shape[1], b=P(B), ldb=B.shape[1], M=M, N=N, K=K, mn_major=int(mn), split_k=split_k, pair=0,
             accumulate=1 if split_k > 1 else 0, route=P(route), route_tile0=0, route_tiles_c=tiles_c, route_off=off, ld_f32=N,
             pen_w=P(Wt), pen_ld=Wt.shape[1], pen_wt=1, pen_w2c=2 * c, pen_loss=P(loss))
    gm = C.Gemm(d)
    tag = f"mn={mn} split_k={split_k}"
    assert gm.split_k == split_k and gm.epi == GENERIC, tag
    gm.launch(native.current_stream())
    torch.cuda.synchronize()
    assert C.read_error_code() == 0, tag
    ref = a.double().t() @ b.double() + 2 * c * W.double()
    rows, cols = torch.meshgrid(torch.arange(M, device="cuda"), torch.arange(N, device="cuda"), indexing="ij")
    owner = torch.bucketize((rows // 32) * tiles_c + cols // 64, torch.tensor(bounds[1:], device="cuda"), right=True)
    scale = float((a.double().abs().t() @ b.double().abs()).max())
    for r, box in enumerate(boxes):
        got = box[off:off + M * N].view(M, N).double()
        want = torch.where(owner == r, ref, torch.zeros_like(ref))
        err = float((got - want).abs().max())
        assert err <= 2e-6 * scale + 1e-5, f"{tag}: shard {r}: max error {err:.2e}"
        assert not bool(box[:off].any()) and not bool(box[off + M * N:].any()), f"{tag}: shard {r}: a store outside the variable"
    want = c * float((W.double() ** 2).sum())
    assert abs(float(loss) - want) <= 1e-5 * want, f"{tag}: loss {float(loss)} vs {want}"


def test_forced_pair_is_refused_for_a_penalised_gemm(monkeypatch):
    C = native.cuda_ext()
    P = native.ptr
    M = N = K = 1024
    A = torch.zeros(M, K, dtype=torch.bfloat16, device="cuda")
    B = torch.zeros(N, K, dtype=torch.bfloat16, device="cuda")
    W = torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
    out, loss = torch.zeros(M, N, device="cuda"), torch.zeros(1, device="cuda")
    d = dict(a=P(A), lda=K, b=P(B), ldb=K, M=M, N=N, K=K, out_f32=P(out), ld_f32=N, pen_w=P(W), pen_ld=N, pen_w2c=0.1, pen_loss=P(loss))
    with pytest.raises(RuntimeError, match="sf_gemm_prepare"):
        C.Gemm(dict(d, pair=1))
    monkeypatch.setenv("SPARKFLOW_GEMM_PAIR", "1")
    with pytest.raises(RuntimeError, match="sf_gemm_prepare"):
        C.Gemm(d)
    monkeypatch.delenv("SPARKFLOW_GEMM_PAIR")
    assert C.Gemm(dict(d, bn=256)).pair == 0                  # auto selection keeps it on the one-CTA kernel


# ------------------------------------------------------------------------------------------------------------------
# the step
# ------------------------------------------------------------------------------------------------------------------
def _compare(tag, lp, w, X, Y, got, loss, dbg, tol):
    B = X.shape[0]
    assert np.isfinite(loss), f"{tag}: loss {loss}"
    l_ref, ref, pools = penalty_oracle(lp, w, X, Y, True, _recorded_argmax(lp, dbg, B), _recorded_relu_mask(lp, dbg, B))
    _check_pools(tag, lp, dbg, pools, B)
    l_err = abs(loss - l_ref) / abs(l_ref)
    assert l_err <= LOSS_TOL, f"{tag}: loss {loss} vs {l_ref} (relative error {l_err:.2e})"
    fro, mx = _assert_grads(tag, lp.var_order, got, ref, tol)
    print(f"[weight-decay] {tag}: rel-Frobenius {fro:.2e} max-abs {mx:.2e} loss {l_err:.2e}")
    return fro, mx, l_err


def _pen_worker(name, w, spec=None, **kw):
    """the step tests' master + worker, the worker's plan carrying the test's (strong) penalty map"""
    master, worker = _worker(name, w, spec, **kw)
    worker.plan.penalty = dict(l2_model(name)[1].penalty)
    return master, worker


STEP_CASES = [(m, v) for m in L2_MODELS for v in ("default", "unfused_loss", "kmajor_wgrad", "no_branches")
              if not (m == "l2_cnn" and v == "kmajor_wgrad")]     # SAME convs are outside the K-major path (check_grammar)


@pytest.mark.parametrize("name,variant", STEP_CASES)
def test_penalised_step_matches_oracle(name, variant, monkeypatch):
    for k, v in VARIANTS[variant].items():
        monkeypatch.setenv(k, v)
    _, lp, _ = l2_model(name)
    w = l2_weights(name)
    master, worker = _pen_worker(name, w)
    pen_gemms = set()
    try:
        for B in (CNN_B if name == "l2_cnn" else DENSE_B):
            X, Y = l2_data(name, B, seed=B)
            got, loss, dbg, names = _run_step(worker, B, X, Y, "staged")
            assert not any(n.startswith("conv_first") for n in names), names
            _compare(f"{name}/{variant} B={B}", lp, w, X, Y, got, loss, dbg, TOL[name])
            pen_gemms |= {(dbg[i]["wgrad"].mn_major(), dbg[i]["wgrad"].split_k > 1) for i, l in enumerate(lp.layers) if "wgrad" in dbg.get(i, {})}
    finally:
        master.close()
    print(f"[weight-decay] {name}/{variant}: wgrad (mn_major, split) kinds {sorted(pen_gemms)}")


PUSH_MODES = {"served": dict(push="served"), "served_lock": dict(push="served", lock=True),
              "sharded2": dict(push="sharded", shards=2), "sharded3_lock": dict(push="sharded", shards=3, lock=True)}


@pytest.mark.parametrize("mode", list(PUSH_MODES))
@pytest.mark.parametrize("name", list(L2_MODELS))
def test_delivered_gradients_and_loss_match_oracle(name, mode):
    """the gradient tap (momentum with learning rate 0 and momentum 0: slot 0 is the consumed gradient) and the published
    loss of three steps: the penalty counted once, the first layer's bias included"""
    _, lp, _ = l2_model(name)
    w = l2_weights(name)
    Bs = (7, 130, 7) if name == "l2_cnn" else (7, 129, 7)
    X, Y = l2_data(name, sum(Bs), seed=5)
    spec = OptimizerSpec.from_tf_kwargs("momentum", dict(learning_rate=0.0, momentum=0.0))
    master, worker = _pen_worker(name, w, spec, **PUSH_MODES[mode])
    start, dbgs = 0, {}
    try:
        for k, B in enumerate(Bs):
            rows = slice(start, start + B)
            start += B
            plan, bufs = worker.build_plan(B, 0, with_pull=True, with_push=True)
            dbg = dbgs.setdefault(B, worker.last_debug)             # a cached plan leaves last_debug as it was
            with torch.cuda.stream(worker.stream):
                bufs.x_stage.copy_(torch.from_numpy(X[rows]))
                if bufs.y_stage is not None:
                    bufs.y_stage.copy_(torch.from_numpy(Y[rows]))
                plan.run(worker.stream.cuda_stream)
            worker.drain()
            assert wait_pushes(master, k + 1) == k + 1
            got = master.slot_arrays()[0]
            _compare(f"{name}/{mode} step {k} B={B}", lp, w, X[rows], None if Y is None else Y[rows], got, float(bufs.loss_out[0]), dbg,
                     TOL[name])
    finally:
        master.close()


@pytest.mark.parametrize("opt", ["gradient_descent", "momentum", "adam"])
@pytest.mark.parametrize("name", list(L2_MODELS))
def test_five_step_update_tracks_reference(name, opt):
    """Five production steps against the host ParameterServer applying the oracle's gradient of every step.  Gradient
    descent and momentum apply an update proportional to the gradient; Adam's first steps are nearly scale free
    (m / sqrt(v)), but a penalty term that is missing, halved or on the wrong variable changes the direction of every
    element it dominates, which the strong coefficients make most of them."""
    from sparkflow_b200.parallel.param_server import LocalTransport, ParameterServer
    from sparkflow_b200.parallel.worker import B200Engine

    _, lp, _ = l2_model(name)
    kw = {"gradient_descent": dict(learning_rate=0.05), "momentum": dict(learning_rate=0.02, momentum=0.9),
          "adam": dict(learning_rate=1e-3)}[opt]
    spec = OptimizerSpec.from_tf_kwargs(opt, kw)
    w0 = l2_weights(name)
    B = 130
    X, Y = l2_data(name, 2 * B, seed=9)
    master, worker = _pen_worker(name, w0, spec)
    worker.use_graphs = True
    try:
        eng = B200Engine(worker)
        eng.load_partition(X, Y)
        ref = LocalTransport(ParameterServer(w0, spec))
        for rows in (slice(0, B), slice(B, 2 * B), slice(0, B), slice(B, 2 * B), slice(0, B)):
            w_k = master.weights()
            eng.train(rows, pull=True)
            eng.finish()
            ref.push(penalty_oracle(lp, w_k, X[rows], None if Y is None else Y[rows], True)[1])
        assert wait_pushes(master, 5) == 5
        tol, worst = UPDATE_TOL.get((name, opt), UPDATE_TOL_DEFAULT), 0.0
        for a, b, a0, v in zip(master.weights(), ref.pull(), w0, lp.var_order):
            du, dr = a - a0, b - a0
            err = np.linalg.norm(du - dr) / np.linalg.norm(dr)
            assert np.isfinite(du).all() and err <= tol, f"{name}/{opt} {v}: update off by {err:.2e}"
            worst = max(worst, err)
        print(f"[weight-decay] {name}/{opt}: worst update rel-Frobenius {worst:.2e}")
    finally:
        master.close()


def test_partition_loss_includes_the_penalty():
    name = "l2_dnn"
    _, lp, _ = l2_model(name)
    w = l2_weights(name)
    X, Y = l2_data(name, 600, seed=4)
    master, worker = _pen_worker(name, w)
    try:
        worker.predict(X[:8], upto=len([l for l in lp.layers if l.kind == "dense"]) - 1, post=None)    # pulls the replica
        got = worker.partition_loss(torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda())
    finally:
        master.close()
    want = penalty_oracle(lp, w, X, Y, True)[0]
    assert abs(got - want) <= 1e-4 * want, (got, want)


def test_session_trains_l2_cnn_natively():
    from sparkflow_b200.models import zoo
    from sparkflow_b200.parallel.session import TrainingSession

    rng = np.random.default_rng(3)
    centers = rng.random((10, 784), dtype=np.float32)
    lab = rng.integers(0, 10, 1200)
    X = np.clip(centers[lab] + 0.2 * rng.normal(0, 1, (1200, 784)), 0, 1).astype(np.float32)
    Y = np.eye(10, dtype=np.float32)[lab]
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    err = io.StringIO()
    with contextlib.redirect_stderr(err):
        sess = TrainingSession(zoo.build("l2_cnn"), "x:0", "y:0", spec, acquire_lock=False, engine="b200", seed=0, devices=[0]).open()
    try:
        assert sess.engine_kind == "b200"
        assert "fall" not in err.getvalue().lower(), err.getvalue()
        eng = sess.make_engine(torch.device("cuda", 0))
        eng.load_partition(X, Y)
        l0 = eng.partition_loss()
        for k in range(12):
            eng.train(slice((k % 4) * 300, (k % 4) * 300 + 300), pull=True)
        eng.finish()
        l1 = eng.partition_loss()
        assert np.isfinite(l1) and l1 < 0.7 * l0, (l0, l1)
        assert sess.counters()["pushes"] == 12
    finally:
        sess.close()
