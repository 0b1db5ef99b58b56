"""64-row tiles of the one-CTA GEMM (csrc/gemm_sm90.cu, ``SfGemm.bm``).

A specialized epilogue variant whose grid of 64-row tiles is still one wave runs with 64-row tiles: half the A operand
bytes per CTA, twice the CTAs, and the first consumer warpgroup alone runs the main loop.  Each output element comes from
the same m64 x BN x k16 wgmma sequence over the same k-blocks as in a 128-row tile, so:

* the bf16 outputs and the non-accumulating fp32 outputs at ``bm=64`` equal those at ``bm=128`` bit for bit;
* the column sums and the loss, atomic sums over 32-row groups, agree within an fp32 reordering bound;
* every output agrees with float64 (``gemm_ref``).

``sf_gemm_prepare`` picks 64 rows by itself for every dense GEMM of the flagship's training step, and keeps 128 for the
generic kernel, split-K, multi-wave and pair GEMMs.
"""
import math
import re

import pytest
import torch

from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import round_up
from gemm_ref import U, _aux, _operands, _reference

GENERIC, FWD, LOSS, DGRAD, WGRAD, SIGMOID_LOSS, SPARSE_LOSS = range(7)      # SfEpi (csrc/sf_api.h)
SOFTMAX, MSE, SIGMOID_XENT, SPARSE = 1, 2, 3, 4                             # SfLossMode
ACT = {None: 0, "relu": 1, "sigmoid": 2, "tanh": 3}
ROWS = (1, 63, 64, 65, 300)

# (name, variant, N, K, bn, options): the flagship's GEMMs (simple_dnn 784-256-256-10), N tails and the loss heads.
# WGRAD: M is the row count of dW (the layer's fan-in), K the batch; the others take M from ROWS.
KMAJOR_CASES = [
    ("fwd0", FWD, 256, 784, 32, dict(act="relu")),
    ("fwd1", FWD, 256, 256, 32, dict(act="relu")),
    ("fwd-tail", FWD, 40, 37, 64, dict(act="tanh")),
    ("fwd-bn64", FWD, 250, 256, 64, dict(act="sigmoid")),
    ("xent", LOSS, 10, 256, 32, dict(loss=SOFTMAX)),
    ("mse", LOSS, 40, 256, 64, dict(loss=MSE)),
    ("dgrad2", DGRAD, 256, 10, 32, dict(aux_act="relu")),
    ("dgrad1", DGRAD, 256, 256, 32, dict(aux_act="relu")),
    ("dgrad-tail", DGRAD, 70, 37, 64, dict(aux_act="sigmoid")),
    ("sigmoid-xent", SIGMOID_LOSS, 10, 256, 32, dict(loss=SIGMOID_XENT)),
    ("sigmoid-xent-bn64", SIGMOID_LOSS, 40, 256, 64, dict(loss=SIGMOID_XENT)),
    ("sparse-xent", SPARSE_LOSS, 10, 256, 32, dict(loss=SPARSE)),
]
# (M, N, K, bn): the flagship's weight gradients and tails
WGRAD_CASES = [(784, 256, 300, 64), (256, 256, 300, 64), (256, 10, 300, 64), (65, 70, 17, 128), (1, 256, 300, 128), (63, 64, 1, 64)]


@pytest.fixture(scope="module")
def C():
    return native.cuda_ext()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _targets(loss, M, N, g):
    """label rows [M, ld] (fp32) for a loss head"""
    if loss == SOFTMAX:
        return torch.eye(N)[torch.randint(0, N, (M,), generator=g)]
    if loss == SPARSE:
        t = torch.zeros(M, 8)
        t[:, 0] = torch.randint(0, N, (M,), generator=g).float()
        return t
    return torch.rand(M, N, generator=g)


def _head64(loss, z, t):
    """float64 dz and loss of a head on the logits z [M, N]"""
    M, N = z.shape
    if loss == SOFTMAX:
        lse = torch.logsumexp(z, 1, keepdim=True)
        ysum = t.sum(1, keepdim=True)
        return (torch.softmax(z, 1) * ysum - t) / M, float(((lse * ysum).squeeze(1) - (t * z).sum(1)).sum() / M)
    if loss == SPARSE:
        y = torch.nn.functional.one_hot(t[:, 0].long(), N).double()
        return (torch.softmax(z, 1) - y) / M, float((torch.logsumexp(z, 1) - (y * z).sum(1)).sum() / M)
    if loss == MSE:
        d = z - t
        return 2 * d / (M * N), float((d * d).sum() / (M * N))
    per = torch.clamp_min(z, 0) - z * t + torch.log1p(torch.exp(-z.abs()))
    return (torch.sigmoid(z) - t) / (M * N), float(per.sum() / (M * N))


def _launch(C, d, bm):
    """one launch of the GEMM `d` (fresh outputs) at tile height bm; returns (Gemm, outputs)"""
    M, N = d["M"], d["N"]
    out = {}
    if d.get("mn_major"):
        out["f32"] = torch.full((M, N), 1234.5, device="cuda")
        dd = dict(out_f32=native.ptr(out["f32"]), ld_f32=N)
    else:
        ldn = round_up(N, 8)
        out["bf16"] = torch.full((M, ldn), 99.0, dtype=torch.bfloat16, device="cuda")
        dd = dict(out_bf16=native.ptr(out["bf16"]), ld_bf16=ldn)
        if d.get("want_colsum"):
            out["colsum"] = torch.zeros(N, device="cuda")
            dd["colsum"] = native.ptr(out["colsum"])
        if d.get("loss_mode"):
            out["loss"] = torch.zeros(1, device="cuda")
            dd["loss"] = native.ptr(out["loss"])
    gm = C.Gemm(dict({k: v for k, v in d.items() if k != "want_colsum"}, **dd, bm=bm, pair=0))
    gm.launch(native.current_stream())
    torch.cuda.synchronize()
    assert C.read_error_code() == 0
    return gm, out


def _check_pair(tag, g128, o128, g64, o64, d, epi):
    M, N = d["M"], d["N"]
    assert (g128.bm, g64.bm) == (128, 64), tag
    for gm, bm in ((g128, 128), (g64, 64)):
        assert gm.epi == epi and gm.pair == 0 and gm.split_k == 1, (tag, gm.epi)
        assert tuple(gm.grid) == ((N + gm.bn - 1) // gm.bn, (M + bm - 1) // bm, 1), (tag, gm.grid)
    for k in ("bf16", "f32"):
        if k in o64:
            assert torch.equal(o64[k], o128[k]), f"{tag}: {k} output differs between 64- and 128-row tiles"
    if "bf16" in o64:
        assert torch.all(o64["bf16"][:, N:] == 0), f"{tag}: bf16 pad columns"


def _reorder_bound(parts):
    """|sum| of atomic adds of 32-row partial sums in any order: one fp32 rounding per add, each of at most the total
    of the magnitudes"""
    n = parts.shape[0]
    return (math.ceil(n / 32) + 1) * 2 * U * parts.abs().sum(0) + 1e-30


@pytest.mark.gpu
@pytest.mark.parametrize("M", ROWS)
@pytest.mark.parametrize("name,epi,N,K,bn,opt", KMAJOR_CASES, ids=[c[0] for c in KMAJOR_CASES])
def test_rows64_kmajor_variant_matches_rows128_and_float64(C, name, epi, N, K, bn, opt, M):
    tag = f"{name} {M}x{N}x{K} bn={bn}"
    a16, b16, bias = _operands(M, N, K, False, seed=M * 7 + N + K, dev="cuda")
    g = torch.Generator().manual_seed(M + K)
    act, aux_act, loss = opt.get("act"), opt.get("aux_act"), opt.get("loss")
    d = dict(a=native.ptr(a16), b=native.ptr(b16), M=M, N=N, K=K, lda=a16.shape[1], ldb=b16.shape[1], bn=bn, act=ACT[act])
    keep = [a16, b16]
    if epi != DGRAD:
        d["bias"] = native.ptr(bias)
    if epi == DGRAD:
        aux = _aux(M, N, aux_act, False, seed=M + N, dev="cuda")
        keep.append(aux)
        d.update(aux=native.ptr(aux), ld_aux=aux.shape[1], aux_act=ACT[aux_act], want_colsum=True)
    if loss:
        t = _targets(loss, M, N, g).cuda()
        keep.append(t)
        d.update(loss_mode=loss, target=native.ptr(t), ld_target=t.shape[1], want_colsum=True)
    g128, o128 = _launch(C, d, 128)
    g64, o64 = _launch(C, d, 64)
    assert g128.bn == bn, tag
    _check_pair(tag, g128, o128, g64, o64, d, epi)

    # float64
    got = o64["bf16"][:, :N].double()
    if loss:
        z, _ = _reference(a16, b16, K, bias, 1.0, None)
        f, loss64 = _head64(loss, z, t.double()[:, :N] if loss != SPARSE else t.double())
        bound = 2.0 ** -8 * f.abs() + 1e-3 * float(f.abs().max())
        assert bool(((got - f).abs() <= bound).all()), f"{tag}: dz against float64"
        for o in (o64, o128):
            assert abs(float(o["loss"]) - loss64) <= 1e-3 * abs(loss64) + 1e-6, (tag, float(o["loss"]), loss64)
        # every head's per-row loss is >= 0, and the total is an atomic sum of the same per-warp row sums at both heights
        assert abs(float(o64["loss"]) - float(o128["loss"])) <= (math.ceil(M / 32) + 1) * 2 * U * abs(loss64) * 1.01 + 1e-12, tag
    else:
        f, e = _reference(a16, b16, K, bias if epi != DGRAD else torch.zeros_like(bias), 1.0, act,
                          aux if epi == DGRAD else None, aux_act)
        assert bool(((got - f).abs() <= 1.01 * e + 2.0 ** -8 * f.abs()).all()), f"{tag}: bf16 output against float64"
    if "colsum" in o64:
        cs = o64["colsum"].double()
        assert bool(((cs - f.sum(0)).abs() <= 1e-3 * f.abs().sum(0) + 1e-6).all()), f"{tag}: column sums against float64"
        # both heights sum each column over the same 32-row groups, in the same order within a group: only the order of
        # the groups' atomic adds differs
        diff = (cs - o128["colsum"].double()).abs()
        assert bool((diff <= 1.01 * _reorder_bound(f)).all()), f"{tag}: column sums differ beyond reordering"


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,bn", WGRAD_CASES, ids=["x".join(map(str, c)) for c in WGRAD_CASES])
def test_rows64_wgrad_variant_matches_rows128_and_float64(C, M, N, K, bn):
    tag = f"WGRAD {M}x{N}x{K} bn={bn}"
    a16, b16, _ = _operands(M, N, K, False, seed=M + N * 3 + K, dev="cuda", mn_major=True)
    d = dict(a=native.ptr(a16), b=native.ptr(b16), M=M, N=N, K=K, lda=a16.shape[1], ldb=b16.shape[1], bn=bn, mn_major=1)
    g128, o128 = _launch(C, d, 128)
    g64, o64 = _launch(C, d, 64)
    assert g128.mn_major() == 1 and g128.bn == bn, tag
    _check_pair(tag, g128, o128, g64, o64, d, WGRAD)
    f, e = _reference(a16, b16, K, torch.zeros(N, device="cuda"), 1.0, None, N=N, M=M, mn_major=True)
    assert bool(((o64["f32"].double() - f).abs() <= e).all()), f"{tag}: fp32 output against float64"


@pytest.mark.gpu
def test_auto_tile_height(C):
    """64 rows only where the kernel has them and the grid stays one wave; the launch grid follows the height."""
    sms = _sms()

    def gemm(M, N, K, **kw):
        a16, b16, bias = _operands(M, N, K, False, seed=1, dev="cuda", mn_major=bool(kw.get("mn_major")))
        ob = torch.zeros(M, round_up(N, 8), dtype=torch.bfloat16, device="cuda")
        of = torch.zeros(M, N, device="cuda")
        d = dict(a=native.ptr(a16), b=native.ptr(b16), M=M, N=N, K=K, lda=a16.shape[1], ldb=b16.shape[1], bias=native.ptr(bias))
        if kw.get("mn_major"):
            d.update(out_f32=native.ptr(of), ld_f32=N, bias=0)
        else:
            d.update(out_bf16=native.ptr(ob), ld_bf16=ob.shape[1])
        d.update(kw)
        gm = C.Gemm(d)
        assert tuple(gm.grid)[1] == (M + gm.bm - 1) // gm.bm
        return gm

    g = gemm(300, 256, 784, act=1)
    assert (g.epi, g.bn, g.bm, tuple(g.grid)) == (FWD, 32, 64, (8, 5, 1))
    g = gemm(784, 256, 300, mn_major=1)
    assert (g.epi, g.bn, g.bm, tuple(g.grid)) == (WGRAD, 64, 64, (4, 13, 1))
    # the generic kernel (forced, or a feature only it has) keeps 128 rows and refuses 64
    assert gemm(300, 256, 784, act=1, epi=GENERIC).bm == 128
    assert gemm(300, 256, 784, act=1, drop_keep=0.5, drop_seed=3).bm == 128
    with pytest.raises(RuntimeError):
        gemm(300, 256, 784, act=1, epi=GENERIC, bm=64)
    # split-K
    g = gemm(288, 64, 30000, mn_major=1, split_k=8)
    assert g.split_k > 1 and g.epi == WGRAD and g.bm == 128
    with pytest.raises(RuntimeError):
        gemm(288, 64, 30000, mn_major=1, split_k=8, bm=64)
    # one wave at 128 rows but not at 64, and several waves at either
    m = 64 * (sms // 8 + 1)                      # 8 column tiles at BN 32: one wave of 128-row tiles only
    g = gemm(m, 256, 64, act=1, bn=32)
    assert g.epi == FWD and g.bm == 128 and g.grid[0] * ((m + 63) // 64) > sms >= g.grid[0] * g.grid[1]
    assert gemm(30000, 64, 288, act=1).bm == 128
    # a forced height is kept
    assert gemm(30000, 64, 288, act=1, bm=64).bm == 64
    assert gemm(300, 256, 784, act=1, bm=128).bm == 128
    # the cluster-pair kernel
    g = gemm(4096, 4096, 1024, pair=1)
    assert g.pair == 1 and g.bm == 128
    with pytest.raises(RuntimeError):
        gemm(4096, 4096, 1024, pair=1, bm=64)


@pytest.mark.gpu
def test_flagship_plan_runs_every_dense_gemm_on_64_row_tiles():
    from sparkflow_b200.graph.executor import GraphProgram
    from sparkflow_b200.graph.ir import GraphIR
    from sparkflow_b200.models import zoo
    from sparkflow_b200.models.compiler import compile_graph
    from sparkflow_b200.ops.layout import ParamLayout
    from sparkflow_b200.ops.optimizers import OptimizerSpec
    from sparkflow_b200.parallel.device_engine import DeviceWorker, MasterState, plan_publish_needs

    ir = GraphIR.from_metagraph(zoo.build("simple_dnn"))
    lp = compile_graph(ir, "x:0", "y:0")
    need_w, need_wt = plan_publish_needs(lp)
    lay = ParamLayout.build(ir.param_shapes(), need_w, need_wt)
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    master = MasterState(lay, spec, torch.device("cuda:0"))
    master.load_weights(GraphProgram(ir).init_weights(seed=1))
    worker = DeviceWorker(ir, "x:0", "y:0", spec, master, acquire_lock=True, shared=False)
    plan, _ = worker.build_plan(300, 0)
    gemms = [g for grp in worker._keep[-1] if isinstance(grp, list) for g in grp if hasattr(g, "epi")]
    n_dense = sum(1 for n in plan.names() if re.match(r"(fwd|dgrad|wgrad)\d", n))
    assert len(gemms) == n_dense >= 6, plan.names()
    assert all(g.epi != GENERIC and g.bm == 64 for g in gemms), (plan.names(), [(g.epi, g.bm, tuple(g.grid)) for g in gemms])
    master.close()
