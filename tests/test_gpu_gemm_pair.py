"""The persistent cluster-pair GEMM (csrc/gemm_pair_sm90.cu) against a float64 product, at the tile tails and with every
epilogue the training plans run on it.

``sf_gemm_prepare`` sends a large un-split GEMM to this kernel on its own (a 4096-wide layer of the benchmark's
``wide_dnn`` from B = 1025 on 132 SMs), so the step's forward and dgrad GEMMs run it once the batch is large.  Two kinds of
case:

* exact: bf16 operands that are small integers, a dyadic alpha, integer biases and act'(aux) values that are short
  dyadic fractions.  Every value the kernel produces is then exact in fp32 whatever the summation order, so the fp32
  output and the column sums must equal the float64 reference bit for bit, the bf16 output must be bf16(reference), and
  the transposed bf16 output must be the row-major one transposed.
* real-valued: Gaussian operands, compared under an element-wise bound derived from the fp32 arithmetic
  (``_reference``); ``test_pair_bound_rejects_plausible_faults`` shows on the CPU that the bound is tight enough to fail.
"""
import math

import pytest
import torch

from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import round_up
from gemm_ref import U, _aux, _check_layout, _colsum_bound, _exact_bf16, _fraction, _operands, _reference, _run

# (M, N, K, pair_ctas): M % 256 = 1 (the last pair tile has one valid row) / 200 / 128 (the rank-1 CTA of the last tile
# row is entirely out of bounds) / 0; N % 128 = 40 (the second multicast half of B is entirely out of bounds) / 100 / 44
# / 104, N % 8 != 0 twice (pad columns in the bf16 output); K = 40 (one partial k-block), 1000 (a partial tail block),
# 4096; one CTA pair walking all 16 tiles (the stage phase carries across tiles), an odd CTA count, one CTA pair per two
# SMs, and more CTAs than twice the tile count.
GEOMETRY = [(513, 296, 1000, 0), (968, 484, 40, 2), (640, 300, 4096, 7), (1280, 1000, 1000, 10000)]


@pytest.fixture(scope="module")
def C():
    return native.cuda_ext()


# ------------------------------------------------------------------------------------------------------------------
# exact cases
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,ctas", GEOMETRY)
def test_pair_exact_forward_epilogues(C, M, N, K, ctas):
    """bias + each activation -> bf16 + transposed bf16 + fp32 (vector stores at pitch N, scalar ones at a pitch past N),
    alpha = 1 / 2, and an fp32 accumulate onto a non-zero buffer: every output exactly the float64 reference"""
    a16, b16, bias = _operands(M, N, K, True, seed=M + N + K, dev="cuda")
    pitches = (N, N + 3)
    for k, (act, alpha) in enumerate([(None, 1.0), ("relu", 0.5), ("sigmoid", 1.0), ("tanh", 0.5)]):
        tag = f"{M}x{N}x{K} ctas={ctas} act={act} alpha={alpha}"
        gm, out = _run(C, a16, b16, M, N, K, pair_ctas=ctas, bias=bias, act=act, alpha=alpha, f32=pitches[k % 2])
        assert gm.pair == 1, tag
        _check_layout(tag, out, M, N, pitches[k % 2])
        ref, bound = _reference(a16, b16, K, bias, alpha, act)
        if act in (None, "relu"):
            assert torch.equal(out["f32"][:, :N].double(), ref), tag
            assert torch.equal(out["bf16"][:, :N], _exact_bf16(ref)), tag
        else:                                   # the fast sigmoid / tanh are the only inexact step
            frac = _fraction(out["f32"][:, :N], ref, bound)
            print(f"[gemm-pair] exact operands {tag}: worst error {frac:.3f} of the bound")
            assert frac <= 1.0, tag
    init = torch.randint(-50, 51, (M, N), generator=torch.Generator().manual_seed(5)).float().cuda()
    gm, out = _run(C, a16, b16, M, N, K, pair_ctas=ctas, bias=bias, alpha=0.5, f32=N, bf16=False, transposed=False, init=init)
    ref, _ = _reference(a16, b16, K, bias, 0.5, None)
    assert torch.equal(out["f32"].double(), ref + init.double()), f"{M}x{N}x{K}: accumulate"


@pytest.mark.gpu
@pytest.mark.parametrize("aux_act", [None, "relu", "sigmoid", "tanh"])
@pytest.mark.parametrize("M,N,K,ctas", GEOMETRY[:3])
def test_pair_exact_dgrad_epilogue(C, M, N, K, ctas, aux_act):
    """dgrad: the product times act'(aux) -> bf16 + transposed bf16, and its column sums (the bias gradient)"""
    a16, b16, _ = _operands(M, N, K, True, seed=3 * M + N + K, dev="cuda")
    aux = _aux(M, N, aux_act, True, seed=M, dev="cuda")
    gm, out = _run(C, a16, b16, M, N, K, pair_ctas=ctas, aux=aux, aux_act=aux_act, colsum=True, f32=N)
    tag = f"{M}x{N}x{K} ctas={ctas} aux_act={aux_act}"
    assert gm.pair == 1, tag
    _check_layout(tag, out, M, N, N)
    ref, _ = _reference(a16, b16, K, torch.zeros(N, device="cuda"), 1.0, None, aux, aux_act)
    assert torch.equal(out["f32"][:, :N].double(), ref), tag
    assert torch.equal(out["bf16"][:, :N], _exact_bf16(ref)), tag
    assert torch.equal(out["colsum"].double(), ref.sum(0)), tag


# ------------------------------------------------------------------------------------------------------------------
# real-valued cases
# ------------------------------------------------------------------------------------------------------------------
REAL_CASES = [("bias", None, None), ("sigmoid", "sigmoid", None), ("tanh", "tanh", None), ("dgrad-sigmoid", None, "sigmoid"),
              ("dgrad-tanh", None, "tanh")]


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,ctas", GEOMETRY)
def test_pair_real_valued_within_derived_bound(C, M, N, K, ctas):
    """Gaussian operands: the fp32 output and the column sums within the bound of ``_reference``, the bf16 outputs the rounding
    of the fp32 one; and the one-CTA kernel (BN 128 and 256) computes the same bits on the same operands"""
    a16, b16, bias = _operands(M, N, K, False, seed=7 * M + N + K, dev="cuda")
    worst = {}
    for name, act, aux_act in REAL_CASES:
        aux = _aux(M, N, aux_act, False, seed=N, dev="cuda") if aux_act else None
        kw = dict(bias=None if aux_act else bias, act=act, alpha=1.0 if aux_act else 0.75, aux=aux, aux_act=aux_act,
                  colsum=aux_act is not None, f32=N)
        tag = f"{M}x{N}x{K} ctas={ctas} {name}"
        gm, out = _run(C, a16, b16, M, N, K, pair_ctas=ctas, **kw)
        assert gm.pair == 1, tag
        _check_layout(tag, out, M, N, N)
        ref, bound = _reference(a16, b16, K, bias if not aux_act else torch.zeros(N, device="cuda"), kw["alpha"], act, aux, aux_act)
        frac = _fraction(out["f32"][:, :N], ref, bound)
        worst[name] = frac
        assert frac <= 1.0, f"{tag}: error {frac:.2f} x the bound"
        if aux_act:
            cf = _fraction(out["colsum"], ref.sum(0), _colsum_bound(ref, bound))
            worst[name + " colsum"] = cf
            assert cf <= 1.0, f"{tag}: column sums {cf:.2f} x the bound"
        # both kernels run the same k-block order and the same epilogue code: on an H100 their outputs agree bit for bit
        for bn in (128, 256):
            g1, o1 = _run(C, a16, b16, M, N, K, pair=0, bn=bn, **kw)
            assert g1.pair == 0 and g1.bn == bn
            for k in ("f32", "bf16", "T"):                # not the column sums: their atomic adds land in any order
                assert torch.equal(o1[k], out[k]), f"{tag}: the one-CTA kernel (BN {bn}) differs from the pair kernel in {k}"
    print(f"[gemm-pair] {M}x{N}x{K} ctas={ctas}: worst error / bound " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


def _with_fault(ref, what, a16, b16, K, bias):
    """the reference with one fault a pair kernel could plausibly have"""
    got = ref.clone()
    M, N = ref.shape
    if what == "a K column dropped":
        k = K - 1
        got -= a16[:, k:k + 1].double() @ b16[:N, k:k + 1].double().t()
    elif what == "the last valid row of the partial pair tile zeroed":
        got[M - 1] = 0
    elif what == "the bias shifted by one column":
        got += torch.roll(bias.double(), 1) - bias.double()
    elif what == "a 64-column multicast half of one tile zeroed":
        got[256:512, 64:128] = 0
    return got


@pytest.mark.parametrize("M,N,K", [(513, 296, 1000), (640, 300, 4096)])
def test_pair_bound_rejects_plausible_faults(M, N, K):
    """The real-valued comparison can fail: computed on the CPU, the fp32 rounding of the reference passes and the
    reference with (a) one K column dropped, (b) the last valid row of a partial pair tile zeroed, (c) the bias shifted by
    one column, (d) the second 64-column multicast half of one tile zeroed is rejected."""
    a16, b16, bias = _operands(M, N, K, False, seed=7 * M + N + K, dev="cpu")
    ref, bound = _reference(a16, b16, K, bias, 1.0, None)
    assert _fraction(ref.float(), ref, bound) <= 1.0
    assert 0 < M % 256 <= 128, "the fault (b) needs a last pair tile whose second CTA has no rows"
    for what in ("a K column dropped", "the last valid row of the partial pair tile zeroed", "the bias shifted by one column",
                 "a 64-column multicast half of one tile zeroed"):
        frac = _fraction(_with_fault(ref, what, a16, b16, K, bias).float(), ref, bound)
        print(f"[gemm-pair] {M}x{N}x{K} with {what}: {frac:.1f} x the bound")
        assert frac > 1.0, f"{M}x{N}x{K}: the bound accepts the output with {what}"


# ------------------------------------------------------------------------------------------------------------------
# eligibility (no launches)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_read_your_writes_gemm_stays_on_the_one_cta_kernel(C, monkeypatch):
    """The fused read-your-writes wait (SfGemmEpilogue.ryw) exists only in the one-CTA kernel, so a GEMM carrying it is
    never sent to the pair kernel: not automatically, not with pair=1, not with SPARKFLOW_GEMM_PAIR=1.  Only built,
    never launched: the wait would spin on counters nobody advances."""
    M = N = 4096
    K = 1024
    a = torch.zeros(M, K, dtype=torch.bfloat16, device="cuda")
    b = torch.zeros(N, K, dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
    words = torch.zeros(64, dtype=torch.int32, device="cuda")
    ryw = torch.frombuffer(bytearray(C.pack_ryw(1, [1], native.ptr(words), native.ptr(words) + 128, 0)), dtype=torch.uint8).cuda()
    base = dict(a=native.ptr(a), b=native.ptr(b), M=M, N=N, K=K, out_bf16=native.ptr(out), ld_bf16=N)
    for pair in (-1, 1):
        assert C.Gemm(dict(base, pair=pair)).pair == 1, "the shape must be pair-eligible without the wait"
        g = C.Gemm(dict(base, pair=pair, ryw=native.ptr(ryw)))
        assert g.pair == 0, f"pair={pair}: a GEMM with the read-your-writes wait went to the pair kernel"
    monkeypatch.setenv("SPARKFLOW_GEMM_PAIR", "1")
    assert C.Gemm(dict(base, pair=-1, ryw=native.ptr(ryw))).pair == 0


@pytest.mark.gpu
def test_gemm_refuses_more_row_tiles_than_the_grid_holds(C):
    """the one-CTA kernel puts M tiles on grid.y (at most 65535): a larger M is refused when the GEMM is built"""
    a = torch.zeros(64, 64, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="sf_gemm_prepare"):
        C.Gemm(dict(a=native.ptr(a), b=native.ptr(a), M=65535 * 128 + 1, N=64, K=64, pair=0, out_bf16=native.ptr(a), ld_bf16=64))


# ------------------------------------------------------------------------------------------------------------------
# 2x2 max-pool past the old grid.y limit
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_maxpool2_backward_at_large_batch(C):
    """n * h * w = 2,131,200 rows: more 32-row blocks than grid.y holds.  Forward winners, pooled values and the
    transposed copy; backward dz (exact: bf16 dout times a 0 / 1 ReLU derivative), its transpose and the bias gradient."""
    n, h, w, c = 3700, 24, 24, 32
    M = n * h * w
    assert (M + 31) // 32 > 65535
    g = torch.Generator(device="cuda").manual_seed(9)
    a = torch.relu(torch.randn(n, h, w, c, device="cuda", generator=g)).to(torch.bfloat16)
    oh, ow = h // 2, w // 2
    out = torch.zeros(n, oh, ow, c, dtype=torch.bfloat16, device="cuda")
    am = torch.zeros(n, oh, ow, c, dtype=torch.uint8, device="cuda")
    ldB = round_up(n, 8)
    outT = torch.zeros(oh * ow * c, ldB, dtype=torch.bfloat16, device="cuda")
    st = native.current_stream()
    C.maxpool_fwd(native.ptr(a), n, h, w, c, native.ptr(out), native.ptr(am), native.ptr(outT), ldB, st)
    torch.cuda.synchronize()
    # window cells in row-major order; the first maximum wins
    win = torch.stack([a[:, dy::2, dx::2, :] for dy in (0, 1) for dx in (0, 1)], -1)
    best, idx = win.float().max(-1)
    first = (win.float() == best.unsqueeze(-1)).int().argmax(-1)
    assert torch.equal(out.float(), best)
    assert torch.equal(am.long(), first)
    assert torch.equal(outT[:, :n].t(), out.reshape(n, -1))
    dout = torch.randn(n, oh, ow, c, device="cuda", generator=g).to(torch.bfloat16)
    ldM = round_up(M, 8)
    dz = torch.full((M, c), 7.0, dtype=torch.bfloat16, device="cuda")
    dzT = torch.zeros(c, ldM, dtype=torch.bfloat16, device="cuda")
    db = torch.zeros(c, device="cuda")
    C.maxpool_bwd(native.ptr(dout), native.ptr(am), n, h, w, c, native.ptr(a), 1, native.ptr(dz), c, native.ptr(dzT), ldM, native.ptr(db), st)
    torch.cuda.synchronize()
    ref = torch.zeros(n, h, w, c, device="cuda")
    for dy in (0, 1):
        for dx in (0, 1):
            hit = first == dy * 2 + dx
            ref[:, dy::2, dx::2, :] = torch.where(hit, dout.float(), torch.zeros((), device="cuda"))
    ref = (ref * (a.float() > 0)).reshape(M, c)
    assert torch.equal(dz.float(), ref), "dz"
    assert torch.equal(dzT[:, :M].t(), dz), "dz transposed"
    ref_db = ref.double().sum(0)
    bound = (12 + math.ceil(M / 32)) * U * ref.double().abs().sum(0)     # 4 rows per thread, 8 per shared atomic, one global per 32
    assert bool(((db.double() - ref_db).abs() <= bound).all()), (db, ref_db)
