"""ELU, SELU, softplus, softsign, leaky ReLU and ReLU6 on the H100: the GEMM twins (FWD, LOSS with MSE, DGRAD, the
generic kernel with the dropout derivative, the cluster-pair kernel) and the stand-alone backward / MSE kernels against
float64, the compiled training step against the bf16-emulating oracle of tests/test_activations.py, the forward plans, a
sharded Hogwild step whose first GEMM carries the read-your-writes wait, and training end to end."""
import numpy as np
import pytest
import torch

from sparkflow_b200.graph.executor import GraphProgram
from sparkflow_b200.models.compiler import ACT_IDS
from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import round_up
from sparkflow_b200.ops.optimizers import OptimizerSpec
from sparkflow_b200.parallel.plan_builder import act_arg
from push_helpers import wait_pushes
from test_step_gradients import (DELIVERY_TOL, VARIANTS, _MODEL_CACHE, _assert_grads, _check_pools, _errors, _grads,
                                 _recorded_argmax, _run_step, _worker, host_drop_masks)
from test_activations import (CNN_GRAPHS, DROP_SCALE, FWD_TOL, GRAPHS, JUMP_ACTS, LOSS_TOL, MLP_SCALE, NEW_ACTS, TOL, act_data, act_deriv,
                              act_forward, act_model, act_value, act_weights, relu6_saturation)

# weights that drive act_mlp's layers and act_drop's ReLU6 layer into the regions a bug shows in
SCALES = {"act_mlp": MLP_SCALE, "act_drop": DROP_SCALE}

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
ALPHA = 0.1                                         # leaky ReLU slope of the kernel cases
GENERIC, FWD, LOSS, DGRAD = 0, 1, 2, 3              # SfEpi


class _Layer:
    def __init__(self, act):
        self.act, self.act_alpha = act, (ALPHA if act == "LeakyRelu" else 0.0)


def _bf16_step(ref):
    return torch.ldexp(torch.ones_like(ref), torch.frexp(ref)[1] - 8)


def _operand(rows, k, g, scale=0.05):
    ld = round_up(k, 8)
    t = torch.zeros(rows, ld, dtype=torch.bfloat16, device=DEV)
    t[:, :k] = (scale * torch.randn(rows, k, device=DEV, generator=g)).to(torch.bfloat16)
    return t


def _bias(n, g):
    """column values spanning |x| up to 60, and packed around 0 and 6"""
    v = torch.empty(n, device=DEV)
    k = torch.arange(n, device=DEV) % 4
    v = torch.where(k == 0, (torch.rand(n, device=DEV, generator=g) * 2 - 1) * 60, v)
    v = torch.where(k == 1, (torch.rand(n, device=DEV, generator=g) * 2 - 1) * 1e-2, v)
    v = torch.where(k == 2, 6 + (torch.rand(n, device=DEV, generator=g) * 2 - 1) * 5e-2, v)
    v = torch.where(k == 3, (torch.rand(n, device=DEV, generator=g) * 2 - 1) * 3, v)
    return v


def _gemm(d):
    C = native.cuda_ext()
    g = C.Gemm(d)
    g.launch(native.current_stream())
    torch.cuda.synchronize()
    assert C.read_error_code() == 0
    return g


def _near_jump(z, act):
    """elements whose pre-activation sits within fp32 accumulation error of a jump of act'"""
    if act not in JUMP_ACTS:
        return torch.zeros_like(z, dtype=torch.bool)
    near = z.abs() < 1e-4
    return near | ((z - 6).abs() < 1e-4) if act == "Relu6" else near


# ------------------------------------------------------------------------------------------------------------------
# GEMM kernels
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K", [(7, 40, 64), (130, 72, 200)])
@pytest.mark.parametrize("act", NEW_ACTS)
def test_forward_gemm_matches_float64(act, M, N, K):
    """bias + activation -> bf16 on the FWD twin, the generic twin (with a transposed copy) and, for a large shape, the pair
    twin"""
    g = torch.Generator(device=DEV).manual_seed(M * 31 + N)
    a, b, bias = _operand(M, K, g), _operand(N, K, g), _bias(N, g)
    z = a[:, :K].double() @ b[:, :K].double().t() + bias.double()
    ref = act_value(z, act, ALPHA)
    for want, extra in ((FWD, {}), (GENERIC, dict(outT=True))):
        ldn = round_up(N, 8)
        out = torch.full((M, ldn), 3.0, dtype=torch.bfloat16, device=DEV)
        outT = torch.zeros(N, round_up(M, 8), dtype=torch.bfloat16, device=DEV)
        d = dict(a=native.ptr(a), lda=a.shape[1], b=native.ptr(b), ldb=b.shape[1], M=M, N=N, K=K, bias=native.ptr(bias),
                 act=ACT_IDS[act],
                 act_alpha=ALPHA if act == "LeakyRelu" else 0.0, out_bf16=native.ptr(out), ld_bf16=ldn)
        if extra:
            d.update(outT_bf16=native.ptr(outT), ld_t=outT.shape[1])
        gm = _gemm(d)
        assert gm.epi == want, (act, gm.epi)
        got = out[:, :N].double()
        tol = _bf16_step(ref) + 2e-5 * (1 + z.abs())
        err = (got - ref).abs()
        assert bool((err <= tol).all()), f"{act} epi={want}: worst err/tol {float((err / tol).max()):.2f}"
        assert not bool(out[:, N:].float().any())
        if extra:
            assert torch.equal(outT[:, :M].t(), out[:, :N])


@pytest.mark.parametrize("act", NEW_ACTS)
def test_pair_gemm_matches_float64(act):
    M, N, K = 512, 384, 512
    g = torch.Generator(device=DEV).manual_seed(7)
    a, b, bias = _operand(M, K, g, 0.02), _operand(N, K, g, 0.02), _bias(N, g)
    out = torch.zeros(M, N, dtype=torch.bfloat16, device=DEV)
    gm = _gemm(dict(a=native.ptr(a), lda=K, b=native.ptr(b), ldb=K, M=M, N=N, K=K, bias=native.ptr(bias), act=ACT_IDS[act],
                    act_alpha=ALPHA if act == "LeakyRelu" else 0.0, out_bf16=native.ptr(out), ld_bf16=N, pair=1))
    assert gm.pair == 1
    z = a.double() @ b.double().t() + bias.double()
    ref = act_value(z, act, ALPHA)
    err = (out.double() - ref).abs()
    tol = _bf16_step(ref) + 2e-5 * (1 + z.abs())
    assert bool((err <= tol).all()), f"{act}: worst err/tol {float((err / tol).max()):.2f}"


@pytest.mark.parametrize("keep", [0.0, 0.6, 0.9])
@pytest.mark.parametrize("act", NEW_ACTS)
def test_dgrad_gemm_matches_float64(act, keep):
    """dz = (g . W) * act'(aux): the DGRAD twin, and with a dropout's aux_keep the generic twin.  The reference takes the
    branches of act' (a unit's sign, ReLU6's saturation) from the pre-activation z, not from the stored value: behind keep
    0.9 a saturated ReLU6 unit stores bf16(6 / 0.9) = 6.65625, whose a * keep is below 6."""
    M, N, K = 130, 72, 96
    g = torch.Generator(device=DEV).manual_seed(11)
    dz, w = _operand(M, K, g, 0.5), _operand(N, K, g, 0.5)
    zpre = _bias(N, g).double().expand(M, N) + 0.5 * torch.randn(M, N, device=DEV, generator=g, dtype=torch.float64)
    a = act_value(zpre, act, ALPHA)
    mask = None
    if keep:
        mask = (torch.rand(M, N, device=DEV, generator=g) < keep).double()
        a = a * mask / keep
    ld = round_up(N, 8)
    aux = torch.zeros(M, ld, dtype=torch.bfloat16, device=DEV)
    aux[:, :N] = a.to(torch.bfloat16)
    out = torch.zeros(M, ld, dtype=torch.bfloat16, device=DEV)
    colsum = torch.zeros(N, device=DEV)
    gm = _gemm(dict(a=native.ptr(dz), lda=dz.shape[1], b=native.ptr(w), ldb=w.shape[1], M=M, N=N, K=K, aux=native.ptr(aux), ld_aux=ld,
                    aux_act=ACT_IDS[act], aux_act_alpha=ALPHA if act == "LeakyRelu" else 0.0, aux_keep=keep,
                    out_bf16=native.ptr(out), ld_bf16=ld, colsum=native.ptr(colsum)))
    assert gm.epi == (GENERIC if keep else DGRAD), gm.epi
    a_st = aux[:, :N].double()
    pos, top = zpre > 0, zpre >= 6
    if keep:
        d = torch.where(a_st != 0, act_deriv(a_st * keep, act, ALPHA, pos, top) / keep, torch.zeros_like(a_st))
    else:
        d = act_deriv(a_st, act, ALPHA, pos, top)
    # a z within rounding of a jump of act' (0, or ReLU6's bf16 boundary below 6 / keep) may be stored on either side
    _, zb = relu6_saturation(keep)
    ok = zpre.abs() >= 1e-3
    if act == "Relu6":
        ok &= ((zpre - zb).abs() >= 2e-2) & ((zpre - 6).abs() >= 2e-2)
    ref = (dz[:, :K].double() @ w[:, :K].double().t()) * d
    err = (out[:, :N].double() - ref).abs()
    tol = _bf16_step(ref) + 1e-5 * ref.abs().max()
    assert bool((err <= tol)[ok].all()), f"{act} keep={keep}: worst err/tol {float((err / tol)[ok].max()):.2f}"
    if act == "Relu6":
        assert bool((top & ok & (a_st != 0)).any()), "no saturated unit survived the dropout"
    # the column sums add the fp32 values: where an element is taken from the bf16 output, allow its rounding (2^-9)
    ref_ok = torch.where(ok, ref, out[:, :N].double())
    slack = 2.0 ** -8 * torch.where(ok, torch.zeros_like(ref), ref_ok.abs()).sum(0) + 1e-3 * ref_ok.abs().sum(0) + 1e-6
    assert bool(((colsum.double() - ref_ok.sum(0)).abs() <= slack).all()), f"{act} keep={keep}: column sums"


@pytest.mark.parametrize("act", NEW_ACTS)
def test_mse_loss_gemm_and_kernel_match_float64(act):
    """the fused MSE head (LOSS twin) and the stand-alone MSE kernel: loss and dz = 2 (a - t) / (M N) * act'(a)"""
    C = native.cuda_ext()
    M, N, K = 129, 40, 64
    g = torch.Generator(device=DEV).manual_seed(13)
    a, b, bias = _operand(M, K, g), _operand(N, K, g), _bias(N, g)
    tgt = torch.rand(M, N, device=DEV, generator=g)
    z = a[:, :K].double() @ b[:, :K].double().t() + bias.double()
    av = act_value(z, act, ALPHA)
    ok = ~_near_jump(z, act)
    ref_loss = float(((av - tgt.double()) ** 2).mean())
    ref_dz = 2 * (av - tgt.double()) / (M * N) * act_deriv(av, act, ALPHA, pos=z > 0, top=z >= 6)
    ld = round_up(N, 8)
    dz, loss = torch.zeros(M, ld, dtype=torch.bfloat16, device=DEV), torch.zeros(1, device=DEV)
    gm = _gemm(dict(a=native.ptr(a), lda=a.shape[1], b=native.ptr(b), ldb=b.shape[1], M=M, N=N, K=K, bias=native.ptr(bias),
                    act=ACT_IDS[act], act_alpha=ALPHA if act == "LeakyRelu" else 0.0, loss_mode=2, target=native.ptr(tgt), ld_target=N,
                    loss=native.ptr(loss), out_bf16=native.ptr(dz), ld_bf16=ld))
    assert gm.epi == LOSS
    # the stand-alone kernel on the fp32 activation the fused head saw
    out32 = av.float().contiguous()
    dz2, loss2 = torch.zeros(M, ld, dtype=torch.bfloat16, device=DEV), torch.zeros(1, device=DEV)
    C.mse_loss(native.ptr(out32), N, native.ptr(tgt), N, act_arg(_Layer(act)), native.ptr(loss2), native.ptr(dz2), ld, 0, 0, 0, M, N,
               native.current_stream())
    torch.cuda.synchronize()
    for tag, got, lo in (("fused", dz, loss), ("stand-alone", dz2, loss2)):
        assert abs(float(lo) - ref_loss) <= 1e-5 * ref_loss, (tag, float(lo), ref_loss)
        err = (got[:, :N].double() - ref_dz).abs()[ok]
        tol = (_bf16_step(ref_dz) + 1e-4 * ref_dz.abs().max())[ok]
        assert bool((err <= tol).all()), f"{act} {tag}: worst err/tol {float((err / tol).max()):.2f}"


@pytest.mark.parametrize("act", NEW_ACTS)
def test_conv_backward_kernels_match_float64(act):
    """maxpool_bwd (2x2), maxpool_gen_bwd (3x3/2 SAME) and act_bwd_bias: g * act'(a) and the bias gradient"""
    C = native.cuda_ext()
    P, st = native.ptr, native.current_stream()
    n, h, w, c = 3, 8, 8, 16
    M = n * h * w
    g = torch.Generator(device=DEV).manual_seed(17)
    zpre = _bias(c, g).double().expand(M, c) + torch.randn(M, c, device=DEV, generator=g, dtype=torch.float64)
    a = act_value(zpre, act, ALPHA).to(torch.bfloat16).contiguous()
    d = act_deriv(a.double(), act, ALPHA)
    code = act_arg(_Layer(act))
    # act_bwd_bias
    grad = torch.randn(M, c, device=DEV, generator=g).to(torch.bfloat16)
    dz, db = torch.zeros(M, c, dtype=torch.bfloat16, device=DEV), torch.zeros(c, device=DEV)
    C.act_bwd_bias(P(grad), c, M, c, P(a), code, P(dz), c, P(db), st)
    torch.cuda.synchronize()
    ref = grad.double() * d
    assert bool(((dz.double() - ref).abs() <= _bf16_step(ref) + 1e-6).all()), act
    torch.testing.assert_close(db.double(), ref.sum(0), rtol=1e-4, atol=1e-4)
    # 2x2 max-pool backward: every window's winner is its first cell here
    am = torch.zeros(n * 4 * 4 * c, dtype=torch.uint8, device=DEV)
    dout = torch.randn(n * 4 * 4 * c, device=DEV, generator=g).to(torch.bfloat16)
    dz, db = torch.zeros(M, c, dtype=torch.bfloat16, device=DEV), torch.zeros(c, device=DEV)
    C.maxpool_bwd(P(dout), P(am), n, h, w, c, P(a), code, P(dz), c, 0, 0, P(db), st)
    torch.cuda.synchronize()
    up = torch.zeros(n, h, w, c, dtype=torch.float64, device=DEV)
    up[:, ::2, ::2, :] = dout.double().reshape(n, 4, 4, c)
    ref = up.reshape(M, c) * d
    assert bool(((dz.double() - ref).abs() <= _bf16_step(ref) + 1e-6).all()), act
    torch.testing.assert_close(db.double(), ref.sum(0), rtol=1e-4, atol=1e-4)
    # general 3x3 / 2 SAME pool: the winner of window (py, px) is in-window index 4 (its centre, input (2py, 2px) + pad 1)
    oh = ow = 4
    am = torch.full((n * oh * ow * c,), 4, dtype=torch.uint8, device=DEV)
    dz, db = torch.zeros(M, c, dtype=torch.bfloat16, device=DEV), torch.zeros(c, device=DEV)
    C.maxpool_gen_bwd(P(dout), P(am), n, h, w, c, 3, 3, 2, 2, 0, 0, oh, ow, P(a), code, P(dz), c, P(db), st)
    torch.cuda.synchronize()
    up = torch.zeros(n, h, w, c, dtype=torch.float64, device=DEV)
    up[:, 1::2, 1::2, :] = dout.double().reshape(n, oh, ow, c)
    ref = up.reshape(M, c) * d
    assert bool(((dz.double() - ref).abs() <= _bf16_step(ref) + 1e-6).all()), act
    torch.testing.assert_close(db.double(), ref.sum(0), rtol=1e-4, atol=1e-4)


# ------------------------------------------------------------------------------------------------------------------
# the training step against the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def registered(monkeypatch):
    """the graphs of test_activations in test_step_gradients' model cache, so its worker / step helpers run them"""
    for name in GRAPHS:
        ir, lp, label, _ = act_model(name)
        monkeypatch.setitem(_MODEL_CACHE, name, (ir, lp, label))


def _record(lp, dbg, B):
    """{dense / conv layer but the last: its output as the step stored it}"""
    out = {}
    dense = [i for i, l in enumerate(lp.layers) if l.kind == "dense"]
    for i, l in enumerate(lp.layers):
        if l.kind == "dense" and i != dense[-1]:
            nxt = min(j for j in dense if j > i)
            out[i] = dbg[nxt]["a_in"][:, :l.out_shape[0]].to(DEV)
        elif l.kind == "conv":
            out[i] = dbg[i]["act_out"].to(DEV).reshape(B, *l.out_shape)
    return out


def _drop_masks(lp, dbg, B):
    seeds = {dbg[i]["drop"]["seed"] for i, l in enumerate(lp.layers) if l.kind == "dense" and l.dropout_keep}
    return host_drop_masks(lp, B, seeds.pop(), 0) if seeds else None


def _compare(tag, name, lp, w, X, Y, got, loss, dbg):
    B = X.shape[0]
    assert np.isfinite(loss), f"{tag}: loss {loss}"
    l_ref, _, params, pools = act_forward(lp, w, X, Y, True, _recorded_argmax(lp, dbg, B), _record(lp, dbg, B), _drop_masks(lp, dbg, B),
                                          device=DEV)
    _check_pools(tag, lp, dbg, pools, B)
    ref = _grads(l_ref, params)
    l_ref = float(l_ref.detach())
    l_err = abs(loss - l_ref) / max(abs(l_ref), 1e-30)
    print(f"[activations] {tag}: loss {loss} vs {l_ref} ({l_err:.2e})")
    fro, mx = _assert_grads(tag, lp.var_order, got, ref, TOL[name])
    print(f"[activations] {tag}: rel-Frobenius {fro:.2e} max-abs {mx:.2e} loss {l_err:.2e}")
    assert l_err <= LOSS_TOL, f"{tag}: loss {loss} vs {l_ref} (relative error {l_err:.2e})"


def _ext_gemms(worker):
    return [g for grp in worker._keep[-1] if isinstance(grp, list) for g in grp if hasattr(g, "epi")]


STEP_CASES = ([(m, v) for m in GRAPHS if m not in CNN_GRAPHS for v in ("default", "unfused_loss", "kmajor_wgrad", "no_branches")]
              + [(m, v) for m in CNN_GRAPHS for v in ("default", "unfused_loss", "lowered_conv1", "no_branches")])


@pytest.mark.parametrize("name,variant", STEP_CASES)
def test_step_gradients_match_oracle(name, variant, registered, monkeypatch):
    for k, v in VARIANTS[variant].items():
        monkeypatch.setenv(k, v)
    lp = act_model(name)[1]
    w = act_weights(name, scale=SCALES.get(name))
    master, worker = _worker(name, w)
    try:
        for B in (1, 7, 129):
            X, Y = act_data(name, B, seed=B)
            for feed in ("staged", "in_graph"):
                got, loss, dbg, names = _run_step(worker, B, X, Y, feed)
                base = [n.split("@")[0] for n in names]
                assert "conv_first_fwd" not in base, names
                _compare(f"{name}/{variant} B={B} {feed}", name, lp, w, X, Y, got, loss, dbg)
    finally:
        master.close()


def test_large_batch_step_runs_the_pair_twin(registered, monkeypatch):
    """B = 4353 through selu_dnn: the SELU layers' forward and dgrad GEMMs land on the cluster-pair twin"""
    monkeypatch.setenv("SPARKFLOW_GEMM_PAIR", "1")
    name = "selu_dnn"
    lp = act_model(name)[1]
    w = act_weights(name)
    master, worker = _worker(name, w)
    try:
        B = 4353
        X, Y = act_data(name, B, seed=5)
        got, loss, dbg, names = _run_step(worker, B, X, Y, "in_graph")
        dense = [i for i, l in enumerate(lp.layers) if l.kind == "dense"]
        assert dbg[dense[1]]["fwd"].pair == 1 and dbg[dense[1]]["dgrad"].pair == 1, "the SELU GEMMs did not run on the pair kernel"
        _compare(f"{name} B={B}", name, lp, w, X, Y, got, loss, dbg)
    finally:
        master.close()


@pytest.mark.parametrize("name", list(GRAPHS))
def test_forward_plans_match_oracle(name, registered):
    lp = act_model(name)[1]
    if any(l.dropout_keep for l in lp.layers):
        pytest.skip("the forward plan of a dropout graph draws its own mask (tests/test_gpu_dropout.py)")
    w = act_weights(name)
    B = 129
    X, Y = act_data(name, B, seed=41)
    with torch.no_grad():
        l_ref, out_ref = act_forward(lp, w, X, Y, True, device=DEV)[:2]
    master, worker = _worker(name, w)
    try:
        out = worker.predict(X, upto=None, post=None)
        fro, mx = _errors(out, out_ref.cpu().numpy())
        assert fro <= FWD_TOL[0] and mx <= FWD_TOL[1], (fro, mx)
        plan, bufs = worker.build_forward_plan(B, with_loss=True, with_pull=True)
        with torch.cuda.stream(worker.stream):
            bufs.x_stage.copy_(torch.from_numpy(X))
            if bufs.y_stage is not None:
                bufs.y_stage.copy_(torch.from_numpy(Y))
            bufs.loss_out.zero_()
            plan.run(worker.stream.cuda_stream)
        worker.stream.synchronize()
        assert abs(float(bufs.loss_out[0]) - float(l_ref)) <= LOSS_TOL * abs(float(l_ref)), (float(bufs.loss_out[0]), float(l_ref))
    finally:
        master.close()


@pytest.mark.parametrize("name", ["selu_dnn", "leaky_cnn"])
def test_inference_runs_the_compiled_forward_plan(name, monkeypatch):
    """prediction of the logits and of their argmax on the compiled forward plan: the logits against the bf16-emulating
    oracle, the argmax equal to the oracle's except where its top two logits are within that tolerance"""
    from sparkflow_b200.ml_util import run_inference

    ir, lp, _, graph = act_model(name)
    logits = lp.layers[-1].tensors["bias"]
    w = act_weights(name, seed=4)
    X, Y = act_data(name, 300, seed=9)
    with torch.no_grad():
        ref = act_forward(lp, w, X, Y, True, device=DEV)[1].cpu().numpy()

    def no_interpreter(*a, **k):
        raise AssertionError("prediction fell back to the interpreter")

    monkeypatch.setattr(GraphProgram, "forward", no_interpreter)
    got = run_inference(graph, w, X, "x:0", logits).reshape(ref.shape)
    fro, mx = _errors(got, ref)
    assert fro <= FWD_TOL[0] and mx <= FWD_TOL[1], (fro, mx)
    got_arg = run_inference(graph, w, X, "x:0", "out:0").reshape(-1)
    top2 = np.sort(ref, axis=1)[:, -2:]
    near_tie = (top2[:, 1] - top2[:, 0]) <= 2 * FWD_TOL[1] * np.abs(ref).max()
    wrong = got_arg != ref.argmax(1)
    assert not (wrong & ~near_tie).any(), np.flatnonzero(wrong & ~near_tie)


def test_sharded_hogwild_first_gemm_carries_the_wait(registered):
    """two Hogwild shards on one GPU: selu_dnn's first GEMM (SELU) carries the read-your-writes wait on the generic twin;
    the delivered gradients match the oracle and the same step without push"""
    name = "selu_dnn"
    lp = act_model(name)[1]
    w = act_weights(name)
    Bs = (7, 129, 7)
    X, Y = act_data(name, sum(Bs), seed=51)
    cuts = np.cumsum((0,) + Bs)
    master, worker = _worker(name, w)
    try:
        plain = [_run_step(worker, B, X[cuts[k]:cuts[k + 1]], Y[cuts[k]:cuts[k + 1]], "in_graph")[0] for k, B in enumerate(Bs)]
    finally:
        master.close()
    spec = OptimizerSpec.from_tf_kwargs("momentum", dict(learning_rate=0.0, momentum=0.0))
    master, worker = _worker(name, w, spec, push="sharded")
    dbgs = {}
    try:
        for k, B in enumerate(Bs):
            rows = slice(cuts[k], cuts[k + 1])
            plan, bufs = worker.build_plan(B, 0, with_pull=True, with_push=True)
            if B not in dbgs:                   # a plan is built once per batch size; its record stays with it
                dbgs[B] = worker.last_debug
                names = [n.split("@")[0] for n in worker.last_plan_names()]
                assert not any(n.startswith("pull") or n.startswith("sync_pull") for n in names), names
                assert dbgs[B][0]["fwd"].epi == GENERIC
            dbg = dbgs[B]
            with torch.cuda.stream(worker.stream):
                bufs.x_stage.copy_(torch.from_numpy(X[rows]))
                bufs.y_stage.copy_(torch.from_numpy(Y[rows]))
                plan.run(worker.stream.cuda_stream)
            worker.drain()
            assert wait_pushes(master, k + 1) == k + 1
            got = master.slot_arrays()[0]
            delivery = max(_errors(g, r)[0] for g, r in zip(got, plain[k]))
            print(f"[activations] {name}/sharded2 step {k}: delivery {delivery:.2e}")
            assert delivery <= DELIVERY_TOL, f"step {k}: the delivered gradient differs from the step's own by {delivery:.2e}"
            _compare(f"{name}/sharded2 step {k} B={B}", name, lp, w, X[rows], Y[rows], got, float(bufs.loss_out[0]), dbg)
    finally:
        master.close()


def test_session_trains_selu_dnn_natively():
    """selu_dnn on a learnable seeded dataset (ten noisy class centres) on the native engine: the loss falls"""
    from sparkflow_b200.models import zoo
    from sparkflow_b200.parallel.session import TrainingSession

    rng = np.random.default_rng(3)
    centers = rng.random((10, 784), dtype=np.float32)
    lab = rng.integers(0, 10, 1200)
    X = np.clip(centers[lab] + 0.2 * rng.normal(0, 1, (1200, 784)), 0, 1).astype(np.float32)
    Y = np.eye(10, dtype=np.float32)[lab]
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    sess = TrainingSession(zoo.build("selu_dnn"), "x:0", "y:0", spec, acquire_lock=False, engine="b200", seed=0, devices=[0]).open()
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
