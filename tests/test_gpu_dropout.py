"""The fused dropout of the GEMM epilogue against the host Philox reference (tests/dropout_ref.py) and the float64 step
oracle (tests/test_step_gradients.py).

Kernel level: ``C.Gemm`` with ``drop_keep / drop_seed / drop_stream / drop_ctr`` on every tile width of the one-CTA
generic kernel and on the cluster-pair kernel, at row counts that cross 128- and 256-row tiles and column counts with
partial 32-column chunks and a partial Philox group of four; and the ``aux_keep`` dgrad that differentiates through a
stored dropout output.  Step level: the compiled training step of three graphs with dropout layers, its masks against
the host masks at the counter the step read, its gradients against the oracle, without push in every plan variant and
with push in every push mode, for two workers, and the forward-only plans.
"""
import numpy as np
import pytest
import torch

from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import round_up
from dropout_ref import dropout_mask, dropout_seed

GENERIC = 0                                   # SfEpi (csrc/sf_api.h)
ACTS = {"none": 0, "relu": 1, "sigmoid": 2, "tanh": 3}
KEEPS = (0.5, 0.75, 0.9)
CTRS = (0, 1, 2 ** 31 - 1, 2 ** 32 - 1)
STREAMS = (0, 5, 0xFFFFFFFF)
MS = (1, 129, 300, 513)
NS = (30, 130, 256, 520)
# (bn, pair): every tile width of the one-CTA kernel, and the cluster-pair kernel (it needs M, N >= 256)
CONFIGS = [(32, 0), (64, 0), (128, 0), (256, 0), (0, 1)]
CFG_IDS = ["bn32", "bn64", "bn128", "bn256", "pair"]

# Kernel-level tolerances, per element: |got - ref| <= ULP_TOL bf16 steps of ref + ACC_TOL * (sum of |terms|) / keep.
# Both sides round to bf16, so an fp32 value next to a rounding midpoint lands one step from the float64 one: the error
# comes in whole steps, and 1.5 steps accepts one and rejects two.  ACC_TOL bounds the fp32 accumulation of the tensor
# cores and the fp32 act'(aux * keep).  Measured on an H100 80GB HBM3 (400 W power limit), as a fraction of the
# tolerance: 0.66 forward (one step), 0.33 dgrad output, 0.01 dgrad column sums.
ULP_TOL = 1.5
ACC_TOL = 2e-5


def _ctr_word(ctr):
    return torch.from_numpy(np.array([ctr], dtype=np.uint32).view(np.int32)).cuda()


def _act64(z, act):
    return {"none": lambda t: t, "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}[act](z)


def _dact64(a, act):
    if act == "relu":
        return (a > 0).double()
    if act == "sigmoid":
        return a * (1 - a)
    if act == "tanh":
        return 1 - a * a
    return torch.ones_like(a)


def _operand(rows, cols, g, ints):
    """bf16 [rows, round_up(cols, 8)] (pad columns zero): small integers, or normal values"""
    if ints:
        x = torch.randint(-2, 3, (rows, cols), device="cuda", generator=g).float()
    else:
        x = torch.randn(rows, cols, device="cuda", generator=g)
    out = torch.zeros(rows, round_up(cols, 8), dtype=torch.bfloat16, device="cuda")
    out[:, :cols] = x.to(torch.bfloat16)
    return out


def _launch(C, d, cfg):
    bn, pair = cfg
    gm = C.Gemm(dict(d, bn=bn, pair=pair))
    gm.launch(native.current_stream())
    torch.cuda.synchronize()
    assert C.read_error_code() == 0
    assert gm.epi == GENERIC and gm.pair == pair, (gm.epi, gm.pair)
    if not pair:
        assert gm.bn == bn
    return gm


def _shapes(cfg):
    return [(M, N) for M in MS for N in NS if not cfg[1] or (M >= 256 and N >= 256)]


def _drop_args(k, M, N):
    """keep / counter / stream / seed of case k: the shapes of a configuration cycle through the values"""
    keep, ctr, stream = KEEPS[k % 3], CTRS[(k // 3 + k) % 4], STREAMS[k % len(STREAMS)]
    seed = (0x2545F491 * (k + 1) + M * 7919 + N) & 0xFFFFFFFF
    return keep, ctr, stream, seed, dropout_mask(M, N, np.float32(keep), seed, stream, ctr)


def _ulp(x):
    """one bf16 step at |x|: 2^(e - 8) for |x| = m 2^e, m in [0.5, 1)"""
    return torch.ldexp(torch.ones_like(x), torch.frexp(x)[1] - 8)


def _check_close(tag, got, ref, tol):
    err = (got - ref).abs()
    frac = float((err / tol).max()) if err.numel() else 0.0
    if frac > 1.0:
        bad = int((err / tol).flatten().argmax())
        pytest.fail(f"{tag}: |got - ref| / tol = {frac:.2f} at flat index {bad} (got {float(got.flatten()[bad])}, "
                    f"ref {float(ref.flatten()[bad])})")
    return frac


def _forward_case(C, cfg, k, M, N, K, act, ints, keep=None):
    g = torch.Generator(device="cuda").manual_seed(1000 * k + M + N)
    ldk, ldn, ldt = round_up(K, 8), round_up(N, 8), round_up(M, 8)
    a, b = _operand(M, K, g, ints), _operand(N, K, g, ints)
    bias = (torch.randint(-3, 4, (N,), device="cuda", generator=g).float() if ints
            else 0.3 * torch.randn(N, device="cuda", generator=g))
    kp, ctr, stream, seed, mask = _drop_args(k, M, N)
    kp = keep or kp
    if keep is not None:
        mask = dropout_mask(M, N, np.float32(kp), seed, stream, ctr)
    word = _ctr_word(ctr)
    out = torch.full((M, ldn), 3.0, dtype=torch.bfloat16, device="cuda")         # sentinel: the pad columns must become 0
    outT = torch.full((N, ldt), 3.0, dtype=torch.bfloat16, device="cuda")        # rows >= M of the transpose are not written
    _launch(C, dict(a=native.ptr(a), lda=ldk, b=native.ptr(b), ldb=ldk, M=M, N=N, K=K, bias=native.ptr(bias), act=ACTS[act],
                    out_bf16=native.ptr(out), ld_bf16=ldn, outT_bf16=native.ptr(outT), ld_t=ldt, drop_keep=kp,
                    drop_seed=seed, drop_stream=stream, drop_ctr=native.ptr(word)), cfg)
    tag = f"{CFG_IDS[CONFIGS.index(cfg)]} M={M} N={N} K={K} {act} keep={kp} ctr={ctr} stream={stream}"
    m = torch.from_numpy(mask).cuda()
    got, gotT = out[:, :N].double(), outT[:, :M].t().double()
    assert bool((out[:, N:] == 0).all()), f"{tag}: pad columns"
    assert bool((outT[:, M:] == 3.0).all()), f"{tag}: the transpose is written past row M"
    # every element the host mask drops is zero (a kept one that is zero too is checked against its value below)
    a64, b64 = a[:, :K].double(), b[:, :K].double()
    z = a64 @ b64.t() + bias.double()
    ref = (_act64(z, act) / kp).to(torch.float32).to(torch.bfloat16).double() * m
    for what, o in (("out_bf16", got), ("outT_bf16", gotT)):
        dropped_nonzero = (~m) & (o != 0)
        assert not bool(dropped_nonzero.any()), f"{tag}: {what} holds {int(dropped_nonzero.sum())} non-zero dropped elements"
    assert torch.equal(got, gotT), f"{tag}: the transpose differs from the output"
    if ints:
        assert torch.equal(got, ref), f"{tag}: not bit-exact ({int((got != ref).sum())} elements differ)"
        return 0.0
    mag = a64.abs() @ b64.abs().t() + bias.double().abs()
    return _check_close(tag, got, ref, ULP_TOL * _ulp(ref) + ACC_TOL * mag / kp + 1e-30)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_dropout_forward_matches_host_mask(cfg):
    """bias + activation + dropout of the generic epilogue: zero exactly where the host mask drops, bf16(act(z) / keep)
    to within one bf16 step where it keeps, in the row-major output and its transpose; pad columns zero."""
    C = native.cuda_ext()
    worst = 0.0
    for k, (M, N) in enumerate(_shapes(cfg)):
        for j, act in enumerate(ACTS):
            worst = max(worst, _forward_case(C, cfg, k + j, M, N, 200, act, False))
    print(f"[dropout] forward {CFG_IDS[CONFIGS.index(cfg)]}: worst error / tolerance {worst:.2f}")


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_dropout_forward_is_bit_exact_on_small_integers(cfg):
    """Small-integer operands, K <= 64, identity / ReLU, keep 0.5: the accumulation, bias, activation and the scale by 2
    are exact, so the output is the host's bit for bit - any difference is a mask or indexing fault."""
    C = native.cuda_ext()
    for k, (M, N) in enumerate(_shapes(cfg)):
        for act in ("none", "relu"):
            _forward_case(C, cfg, k, M, N, 40 if k % 2 else 64, act, True, keep=0.5)
    print(f"[dropout] bit-exact forward {CFG_IDS[CONFIGS.index(cfg)]}: every output equal")


def _dgrad_case(C, cfg, k, M, N, K, act):
    g = torch.Generator(device="cuda").manual_seed(7000 + 1000 * k + M + N)
    ldk, ldn = round_up(K, 8), round_up(N, 8)
    dz, w = _operand(M, K, g, False), _operand(N, K, g, False)
    kp, ctr, stream, seed, mask = _drop_args(k, M, N)
    m = torch.from_numpy(mask).cuda()
    z = 1.5 * torch.randn(M, N, device="cuda", generator=g, dtype=torch.float64)
    aux = torch.zeros(M, ldn, dtype=torch.bfloat16, device="cuda")
    aux[:, :N] = (_act64(z, act) * m / kp).to(torch.float32).to(torch.bfloat16)      # what the forward stored
    a_st = aux[:, :N].double()
    if act != "relu":
        assert torch.equal(a_st != 0, m)
    out = torch.full((M, ldn), 3.0, dtype=torch.bfloat16, device="cuda")
    colsum = torch.zeros(N, device="cuda")
    _launch(C, dict(a=native.ptr(dz), lda=ldk, b=native.ptr(w), ldb=ldk, M=M, N=N, K=K, aux=native.ptr(aux), ld_aux=ldn,
                    aux_act=ACTS[act], aux_keep=kp, out_bf16=native.ptr(out), ld_bf16=ldn, colsum=native.ptr(colsum)), cfg)
    tag = f"{CFG_IDS[CONFIGS.index(cfg)]} dgrad M={M} N={N} K={K} {act} keep={kp}"
    assert bool((out[:, N:] == 0).all()), f"{tag}: pad columns"
    a64, b64 = dz[:, :K].double(), w[:, :K].double()
    d = _dact64(a_st * kp, act) * m / kp                                           # g W^T . mask / keep . act'(aux keep)
    ref = (a64 @ b64.t()) * d
    mag = (a64.abs() @ b64.abs().t()) / kp
    got = out[:, :N].double()
    assert not bool(((~m) & (got != 0)).any()), f"{tag}: gradient through a dropped element"
    f_out = _check_close(tag + " out_bf16", got, ref, ULP_TOL * _ulp(ref) + ACC_TOL * mag + 1e-30)
    f_col = _check_close(tag + " colsum", colsum.double(), ref.sum(0), ACC_TOL * mag.sum(0) + 1e-30)
    return f_out, f_col


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_dropout_dgrad_matches_float64(cfg):
    """The dgrad through a dropout layer (aux_keep): the mask recovered from the stored activation, 1 / keep and act'
    at aux * keep, in the bf16 output and the fp32 column sums (the bias gradient)."""
    C = native.cuda_ext()
    worst = [0.0, 0.0]
    for k, (M, N) in enumerate(_shapes(cfg)):
        for j, act in enumerate(ACTS):
            worst = [max(a, b) for a, b in zip(worst, _dgrad_case(C, cfg, k + j, M, N, 200, act))]
    print(f"[dropout] dgrad {CFG_IDS[CONFIGS.index(cfg)]}: worst error / tolerance {worst[0]:.2f} (out), {worst[1]:.2f} (colsum)")


# ----------------------------------------------------------------------------------------------------------------------
# the compiled training step
# ----------------------------------------------------------------------------------------------------------------------
from push_helpers import wait_pushes  # noqa: E402
from test_step_gradients import (DROP_LOSS_TOL, FWD_TOL, TOL, VARIANTS, _compare_step, _data, _errors, _forward,  # noqa: E402
                                 _model, _run_step, _weights, _worker, host_drop_masks)

STEP_VARIANTS = dict(VARIANTS, pair={"SPARKFLOW_GEMM_PAIR": "1"})
# cnn_drop is cnn_same: SAME-padded convs have no K-major weight gradient; ae_drop has no GEMM the pair kernel takes
STEP_CASES = ([("mlp_drop", v) for v in ("default", "unfused_loss", "kmajor_wgrad", "no_branches", "pair")]
              + [("ae_drop", v) for v in ("default", "unfused_loss", "kmajor_wgrad", "no_branches")]
              + [("cnn_drop", v) for v in ("default", "unfused_loss", "pair")])


def _dropout_layers(lp):
    """{dense layer with a dropout: the dense layer that reads its output}"""
    dense = [i for i, l in enumerate(lp.layers) if l.kind == "dense"]
    return {i: min(j for j in dense if j > i) for i in dense if lp.layers[i].dropout_keep}


def _ctr(t):
    return int(t.cpu().view(-1)[0]) & 0xFFFFFFFF


def _step_masks(tag, lp, dbg, B, worker_index, ctr=None):
    """The plan's dropout parameters as ``plan_builder`` records them, checked against the seed formula; returns
    (host masks at the counter the step read, that counter).  ``ctr``: the counter value, read from the plan's counter
    word when not given (the step must have read the same)."""
    seeds = set()
    for i in _dropout_layers(lp):
        r = dbg[i]["drop"]
        assert r["keep"] == lp.layers[i].dropout_keep and r["stream"] == i, (tag, i, r)
        assert r["seed"] == dropout_seed(worker_index, native.ptr(r["ctr"])), f"{tag}: layer {i} seed"
        seeds.add(r["seed"])
        word = r["ctr"]
    assert len(seeds) == 1, f"{tag}: the layers of one plan use different seeds"
    if ctr is None:
        ctr = _ctr(word)
    return host_drop_masks(lp, B, seeds.pop(), ctr), ctr


def _check_stored_masks(tag, lp, dbg, masks, B):
    """The input of the layer after each dropout - and its transposed copy where the plan keeps one - is zero exactly
    where the host mask drops (a kept unit may be zero too: a ReLU that is off)."""
    for i, nxt in _dropout_layers(lp).items():
        N = lp.layers[i].out_shape[0]
        m = torch.from_numpy(masks[i])
        copies = [("a_in", dbg[nxt]["a_in"][:, :N])]
        if dbg[nxt]["a_inT"] is not None:
            copies.append(("a_inT", dbg[nxt]["a_inT"][:N, :B].t()))
        for what, a in copies:
            a = a.cpu()
            assert a.shape == m.shape, (tag, what, a.shape, m.shape)
            bad = (~m) & (a != 0)
            assert not bool(bad.any()), f"{tag}: layer {i} {what}: {int(bad.sum())} units the host mask drops are non-zero"
            if lp.layers[i].act not in ("Relu", None):
                # a kept tanh / sigmoid unit is non-zero: its zeros are exactly the dropped units
                assert torch.equal(a != 0, m), f"{tag}: layer {i} {what}: {int(((a == 0) & m).sum())} kept units are zero"
        if lp.layers[i].act == "Relu":
            kept_on = (dbg[nxt]["a_in"][:, :N].cpu() != 0)
            assert float(kept_on.double().mean()) > 0.2 * float(m.double().mean()), f"{tag}: layer {i}: hardly any unit kept"


def _pair_gemms(worker):
    return [g for grp in worker._keep[-1] if isinstance(grp, list) for g in grp if hasattr(g, "pair") and g.pair == 1]


@pytest.mark.gpu
@pytest.mark.parametrize("name,variant", STEP_CASES)
def test_dropout_step_matches_oracle(name, variant, monkeypatch):
    """One step without push, staged and in-graph feeds: the stored dropout outputs against the host masks of the
    plan's seed at counter 0, then every gradient and the loss against the bf16-emulating oracle with those masks."""
    for k, v in STEP_VARIANTS[variant].items():
        monkeypatch.setenv(k, v)
    _, lp, _ = _model(name)
    w = _weights(name)
    master, worker = _worker(name, w)
    worst = [0.0, 0.0, 0.0]
    pair_seen = False
    try:
        # 513: two 256-row tiles of the pair kernel (not on cnn_drop: at that batch the pool check's float64 winners
        # meet bf16 ties the step broke one rounding step apart)
        for B in (1, 7, 129, 300) + ((513,) if variant == "pair" and name != "cnn_drop" else ()):
            X, Y = _data(name, B, seed=B + 60)
            for feed in ("staged", "in_graph"):
                tag = f"{name}/{variant} B={B} {feed}"
                got, loss, dbg, names = _run_step(worker, B, X, Y, feed)
                masks, ctr = _step_masks(tag, lp, dbg, B, 0)
                assert ctr == 0, f"{tag}: a step without push moved its counter to {ctr}"
                _check_stored_masks(tag, lp, dbg, masks, B)
                e = _compare_step(tag, lp, w, X, Y, got, loss, dbg, TOL[name], masks, DROP_LOSS_TOL[name])
                worst = [max(a, b) for a, b in zip(worst, e)]
                pair_seen |= bool(_pair_gemms(worker))
    finally:
        master.close()
    assert pair_seen == (variant == "pair"), f"{name}/{variant}: the cluster-pair kernel ran: {pair_seen}"
    print(f"[dropout] {name}/{variant}: worst rel-Frobenius {worst[0] / TOL[name][0]:.2f}, max-abs {worst[1] / TOL[name][1]:.2f} "
          f"of the tolerance; loss {worst[2] / DROP_LOSS_TOL[name]:.2f}")


# push modes of the pushed steps: the worker's own push with and without the lock, a served master, 2 shards
PUSH_MODES = {"direct_lock": dict(lock=True), "direct": {}, "served": dict(push="served"), "sharded2": dict(push="sharded", shards=2)}
PUSH_GRAPHS = {"direct_lock": True, "direct": False, "served": False, "sharded2": True}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(PUSH_MODES))
def test_pushed_dropout_steps_advance_the_mask(mode):
    """Five production steps with push (CUDA graph replay in the direct-lock and sharded modes).  The gradient tap:
    momentum with learning rate 0 and momentum 0 leaves slot 0 equal to the gradient the push delivered.  Each step
    reads the counter its predecessor's push left; its masks are the host masks at that counter, differ from the
    previous step's, and its gradient is the oracle's with them.  In the direct modes a second worker on the same master
    draws its own masks."""
    from sparkflow_b200.ops.optimizers import OptimizerSpec
    from sparkflow_b200.parallel.device_engine import DeviceWorker

    name, B, steps = "mlp_drop", 129, 5
    ir, lp, label = _model(name)
    w = _weights(name)
    X, Y = _data(name, steps * B, seed=77)
    spec = OptimizerSpec.from_tf_kwargs("momentum", dict(learning_rate=0.0, momentum=0.0))
    master, worker = _worker(name, w, spec, **PUSH_MODES[mode])
    worker.use_graphs = PUSH_GRAPHS[mode]
    worst = [0.0, 0.0, 0.0]
    try:
        plan, bufs = worker.build_plan(B, 0, with_pull=True, with_push=True)
        dbg = worker.last_debug
        prev = None
        for k in range(steps):
            rows = slice(k * B, (k + 1) * B)
            tag = f"{name}/{mode} step {k}"
            masks, ctr = _step_masks(tag, lp, dbg, B, 0)
            assert ctr == k, f"{tag}: the counter reads {ctr} after {k} pushes"
            with torch.cuda.stream(worker.stream):
                bufs.x_stage.copy_(torch.from_numpy(X[rows]))
                bufs.y_stage.copy_(torch.from_numpy(Y[rows]))
            worker.run_plan(plan)
            worker.drain()
            assert wait_pushes(master, k + 1) == k + 1
            assert _ctr(dbg[0]["drop"]["ctr"]) == ctr + 1, f"{tag}: the push did not advance the counter"
            _check_stored_masks(tag, lp, dbg, masks, B)
            if prev is not None:
                for i in masks:
                    assert not np.array_equal(masks[i], prev[i]), f"{tag}: layer {i} drew the previous step's mask"
            prev = masks
            got = master.slot_arrays()[0]
            e = _compare_step(tag, lp, w, X[rows], Y[rows], got, float(bufs.loss_out[0]), dbg, TOL[name], masks, DROP_LOSS_TOL[name])
            worst = [max(a, b) for a, b in zip(worst, e)]
        if mode.startswith("direct"):
            w1 = DeviceWorker(ir, "x:0", label, spec, master, acquire_lock=mode == "direct_lock", shared=False, use_graphs=False,
                              worker_index=1)
            plan1, bufs1 = w1.build_plan(B, 0, with_pull=True, with_push=True)
            dbg1 = w1.last_debug
            rows = slice(0, B)
            m1, ctr1 = _step_masks(f"{name}/{mode} worker 1", lp, dbg1, B, 1)
            m0, _ = _step_masks(f"{name}/{mode} worker 0", lp, dbg, B, 0, ctr=ctr1)
            with torch.cuda.stream(w1.stream):
                bufs1.x_stage.copy_(torch.from_numpy(X[rows]))
                bufs1.y_stage.copy_(torch.from_numpy(Y[rows]))
            w1.run_plan(plan1)
            w1.drain()
            assert wait_pushes(master, steps + 1) == steps + 1
            _check_stored_masks(f"{name}/{mode} worker 1", lp, dbg1, m1, B)
            for i in m1:
                assert not np.array_equal(m1[i], m0[i]), f"{mode}: layer {i}: worker 1 drew worker 0's mask"
            e = _compare_step(f"{name}/{mode} worker 1", lp, w, X[rows], Y[rows], master.slot_arrays()[0],
                              float(bufs1.loss_out[0]), dbg1, TOL[name], m1, DROP_LOSS_TOL[name])
            worst = [max(a, b) for a, b in zip(worst, e)]
        for a, b, v in zip(master.weights(), w, lp.var_order):
            assert np.array_equal(a, b), f"{name}/{mode}: {v} moved under a zero learning rate"
    finally:
        master.close()
    print(f"[dropout] {name}/{mode} pushed: worst rel-Frobenius {worst[0] / TOL[name][0]:.2f}, max-abs "
          f"{worst[1] / TOL[name][1]:.2f} of the tolerance; loss {worst[2] / DROP_LOSS_TOL[name]:.2f}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mlp_drop", "ae_drop"])
def test_dropout_forward_plans_match_oracle(name):
    """predict and the forward + loss plan have no step counter: their masks are the host masks at counter 0 under the
    seed without the counter's address (the keep placeholder is not fed, so TensorFlow drops units here too).  Measured
    output error on an H100 80GB HBM3 (400 W power limit): mlp_drop 2.1e-4 / 1.2e-3 of FWD_TOL's 1e-3 / 4e-3."""
    _, lp, _ = _model(name)
    w = _weights(name)
    B = 129
    X, Y = _data(name, B, seed=41)
    masks = host_drop_masks(lp, B, dropout_seed(0), 0)
    with torch.no_grad():
        l_ref, out_ref = _forward(lp, w, X, Y, True, drop_mask=masks)[:2]
    with torch.no_grad():
        other = _forward(lp, w, X, Y, True, drop_mask=host_drop_masks(lp, B, dropout_seed(0), 1))[1]
    master, worker = _worker(name, w)
    try:
        out = worker.predict(X, upto=None, post=None)
        assert out.shape == tuple(out_ref.shape) and np.isfinite(out).all()
        fro, mx = _errors(out, out_ref.cpu().numpy())
        assert fro <= FWD_TOL[0] and mx <= FWD_TOL[1], (fro, mx)
        assert _errors(out, other.cpu().numpy())[0] > 0.1, "the output does not depend on the mask"
        plan, bufs = worker.build_forward_plan(B, with_loss=True, with_pull=True)
        with torch.cuda.stream(worker.stream):
            bufs.x_stage.copy_(torch.from_numpy(X))
            if bufs.y_stage is not None:
                bufs.y_stage.copy_(torch.from_numpy(Y))
            bufs.loss_out.zero_()
            plan.run(worker.stream.cuda_stream)
        worker.stream.synchronize()
        loss, l_ref = float(bufs.loss_out[0]), float(l_ref)
        assert abs(loss - l_ref) <= DROP_LOSS_TOL[name] * abs(l_ref), (loss, l_ref)
        print(f"[dropout] {name} forward B={B}: output rel-Frobenius {fro / FWD_TOL[0]:.2f}, max-abs {mx / FWD_TOL[1]:.2f} of the "
              f"tolerance; loss {abs(loss - l_ref) / abs(l_ref) / DROP_LOSS_TOL[name]:.2f}")
    finally:
        master.close()
