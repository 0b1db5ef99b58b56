"""The one-CTA GEMM (sf_gemm_kernel and its epilogue variants, csrc/gemm_sm90.cu) against a float64 product, at every
tile width, operand layout, K split and tail, and with the fused loss heads.

This kernel runs every GEMM too small for the cluster-pair kernel: all of the dense training step's GEMMs at the
flagship batch, every CNN and autoencoder GEMM and every split-K weight gradient.  Each launch passes ``pair=0`` and an
explicit ``bn`` and asserts the width, K split, epilogue variant and operand layout that ``Gemm`` reports, so a case
pins its kernel instantiation whatever the SM count.  Three kinds of case:

* exact: bf16 operands that are small integers, alpha 1 or 1/2, integer biases and start values, act'(aux) values that
  are short dyadic fractions.  ``_exact_in_fp32`` first shows that every partial sum the kernel can form is an fp32
  number; then the fp32 output and the column sums must equal float64 bit for bit and the bf16 output must be
  bf16(float64).  The operand pad columns hold NaN: the tensor maps' extents exclude them, so none may reach an output.
* real-valued: Gaussian operands, under the element-wise bound of ``_reference`` and ``_colsum_bound``.
* loss heads: softmax cross-entropy and MSE, under bounds derived below from __expf, __logf and __fdividef.

``test_bounds_reject_plausible_faults`` shows on the CPU that the bounds fail on faults this kernel could have.
"""
import math

import pytest
import torch

from sparkflow_b200.ops import native
from gemm_ref import (U, _aux, _check_layout, _colsum_bound, _dact64, _exact_bf16, _fraction, _logical, _operands, _reference,
                      _run)

GENERIC, FWD, LOSS, DGRAD, WGRAD = 0, 1, 2, 3, 4         # SfEpi (csrc/sf_api.h)
SOFTMAX, MSE, SPARSE = 1, 2, 4                            # SfLossMode
NAN = float("nan")
BNS = (32, 64, 128, 256)
BF16_HALF_STEP = 2.0 ** -8                                # bf16 rounding: at most 2^-8 of the value

# K-major (M, N, K): one row and K below one k-block; M % 128 = 1 and N % 32 = 8; N % 8 != 0, a 16-wide K tail and more
# k-blocks than stages at every width (the ring phase wraps); a large one; no tails; the flagship's last-layer dgrad
# (K = 10) and M % 128 = 1 at K = 37; and "waves": more CTAs than SMs at every width, so the multi-wave PDL trigger path
# runs.  K % 8 != 0 in three of them: their operands have NaN pad columns between K and the row pitch, which only a tensor
# map whose K extent is the pitch would read.
KMAJOR = [(1, 10, 8), (129, 40, 40), (300, 250, 784), (1000, 520, 4096), (128, 256, 64), (300, 256, 10), (129, 40, 37), "waves"]
# MN-major (M, N, K, split_k): the weight-gradient shapes of the training plans, a batch of one (K = 1), K = 7, N % 8 != 0
MNMAJOR = [(784, 256, 300, 1), (256, 256, 300, 1), (256, 10, 300, 1), (1600, 10, 300, 1), (288, 64, 30000, 8), (25, 32, 4000, 1),
           (4096, 4096, 300, 1), (130, 70, 17, 1), (100, 50, 1, 1), (64, 27, 7, 1)]
# (M, N, K, split_k requested, the K splits in k-blocks that sf_gemm_prepare settles on): each with a short last split,
# K % 8 != 0 (NaN pad columns)
SPLITS = [(300, 250, 1001, 3, (6, 6, 4)), (300, 250, 1001, 6, (3, 3, 3, 3, 3, 1)), (129, 40, 29999, 8, (59,) * 7 + (56,))]


@pytest.fixture(scope="module")
def C():
    return native.cuda_ext()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def _geometry(geo):
    return (128 * _sms() + 1, 72, 131) if geo == "waves" else geo


def _ids(geos):
    return [g if isinstance(g, str) else "x".join(map(str, g)) for g in geos]


# ------------------------------------------------------------------------------------------------------------------
# exactness condition
# ------------------------------------------------------------------------------------------------------------------
def _exponent(t):
    """the least e >= 0 such that every value of t is a multiple of 2^-e"""
    t = torch.as_tensor(t, dtype=torch.float64)
    for e in range(40):
        s = t * 2.0 ** e
        if torch.equal(s, torch.round(s)):
            return e
    raise AssertionError("not a short dyadic fraction")


def _exact_in_fp32(tag, a16, b16, M, N, K, mn_major=False, alpha=1.0, bias=None, init=None, aux=None, aux_act=None, colsum=False):
    """Asserts that every value the kernel forms on these operands is an fp32 number, whatever the order of its sums: a
    multiple of 2^-e below 2^(24 - e) in magnitude.  The values and their worst-case magnitudes:
      * the main loop's partial sums: integers, at most S = sum_k |a_k b_k|;
      * alpha * acc + bias, summed with the start value and the other K splits' partial results by atomic adds: multiples
        of 2^-e(alpha, bias, start), at most |alpha| S + |bias| + |start|;
      * the product with act'(aux) (itself a short fraction: act' of a short fraction is formed exactly): e grows by
        e(act'), the magnitude is scaled by |act'|;
      * the column sums: any partial sum of a column, at most the column's sum of magnitudes."""
    A, B = _logical(a16, b16, K, N, M, mn_major)
    assert _exponent(A) == 0 and _exponent(B) == 0, f"{tag}: the operands must be integers"
    S = A.abs() @ B.abs().t()
    checks = [("main-loop partial sums", S, 0)]
    e = _exponent(alpha)
    mag = abs(alpha) * S
    for t in (bias, init):
        if t is not None:
            e = max(e, _exponent(t))
            mag = mag + t.double().abs()
    checks.append(("epilogue and accumulate", mag, e))
    if aux is not None:
        d = _dact64(aux[:, :N].double(), aux_act).abs()
        e += _exponent(d)
        mag = mag * d
        checks.append(("act'(aux) product", mag, e))
    if colsum:
        checks.append(("column sums", mag.sum(0), e))
    for what, m, ex in checks:
        assert float(m.max()) * 2.0 ** ex < 2.0 ** 24, f"{tag}: {what} reach {float(m.max())} at a 2^-{ex} step: not exact in fp32"


# ------------------------------------------------------------------------------------------------------------------
# exact cases: the launches
# ------------------------------------------------------------------------------------------------------------------
def _kmajor_runs(M, N, bn_index):
    """(name, launch kwargs) of the exact K-major runs of one geometry at one width: fp32 at pitch N (vector stores) and
    N + 3 (scalar stores), bf16 + transposed bf16, column sums, each activation, an accumulate onto a non-zero start, a
    dgrad (the act'(aux) of its width).  The dgrad sums its columns up to 300 rows: over more, at act' steps of 1/16, the
    column sums could outgrow fp32's 24 bits."""
    init = torch.randint(-50, 51, (M, N), generator=torch.Generator().manual_seed(5)).float()
    aux_act = ("relu", "sigmoid", "tanh", None)[bn_index]
    return [("bias", dict(bias=True, act=None, alpha=1.0, f32=N, colsum=True)),
            ("relu", dict(bias=True, act="relu", alpha=0.5, f32=N + 3)),
            ("sigmoid", dict(bias=True, act="sigmoid", alpha=1.0, f32=N + 3)),
            ("tanh", dict(bias=True, act="tanh", alpha=0.5, f32=N)),
            ("accumulate", dict(bias=True, act=None, alpha=0.5, f32=N + 3, bf16=False, transposed=False, init=init)),
            (f"dgrad-{aux_act}", dict(bias=False, act=None, alpha=1.0, f32=N, colsum=M <= 300, aux_act=aux_act))]


def _exact_kmajor_inputs(geo, dev):
    M, N, K = _geometry(geo)
    a16, b16, bias = _operands(M, N, K, True, seed=M + N + K, dev=dev, pad=NAN)
    return M, N, K, a16, b16, bias


def _resolve(kw, bias, M, N, dev, seed):
    """launch kwargs with the bias, start value and aux operand in place"""
    kw = dict(kw)
    kw["bias"] = bias if kw.pop("bias") else None
    if kw.get("init") is not None:
        kw["init"] = kw["init"].to(dev)
    if "aux_act" in kw:
        kw["aux"] = _aux(M, N, kw["aux_act"], True, seed=seed, dev=dev)
    return kw


def _check_exact(tag, gm_out, ref, kw, M, N):
    gm, out = gm_out
    _check_layout(tag, out, M, N, kw.get("f32"))
    if "f32" in out:
        got = out["f32"][:, :N].double()
        want = ref + kw["init"].double() if kw.get("init") is not None else ref
        assert torch.equal(got, want), f"{tag}: fp32 output != float64"
    if "bf16" in out:
        assert torch.equal(out["bf16"][:, :N], _exact_bf16(ref)), f"{tag}: bf16 output != bf16(float64)"
    if "colsum" in out:
        assert torch.equal(out["colsum"].double(), ref.sum(0)), f"{tag}: column sums != float64"


@pytest.mark.gpu
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("geo", KMAJOR, ids=_ids(KMAJOR))
def test_cta_exact_kmajor(C, geo, bn):
    M, N, K, a16, b16, bias = _exact_kmajor_inputs(geo, "cuda")
    for name, kw in _kmajor_runs(M, N, BNS.index(bn)):
        tag = f"{M}x{N}x{K} bn={bn} {name}"
        kw = _resolve(kw, bias, M, N, "cuda", seed=M + bn)
        _exact_in_fp32(tag, a16, b16, M, N, K, alpha=kw["alpha"], bias=kw["bias"], init=kw.get("init"), aux=kw.get("aux"),
                       aux_act=kw.get("aux_act"), colsum=kw.get("colsum", False))
        gm, out = _run(C, a16, b16, M, N, K, pair=0, bn=bn, **kw)
        assert (gm.pair, gm.bn, gm.split_k, gm.epi, gm.mn_major()) == (0, bn, 1, GENERIC, 0), tag
        ref, bound = _reference(a16, b16, K, bias if kw["bias"] is not None else torch.zeros(N, device="cuda"), kw["alpha"],
                                kw["act"], kw.get("aux"), kw.get("aux_act"))
        if kw["act"] in ("sigmoid", "tanh"):          # the fast sigmoid / tanh are the only inexact step
            _check_layout(tag, out, M, N, kw["f32"])
            frac = _fraction(out["f32"][:, :N], ref, bound)
            print(f"[gemm-cta] exact operands {tag}: worst error {frac:.3f} of the bound")
            assert frac <= 1.0, tag
        else:
            _check_exact(tag, (gm, out), ref, kw, M, N)


def _split_inputs(M, N, K, dev):
    a16, b16, bias = _operands(M, N, K, True, seed=K + N, dev=dev, pad=NAN)
    init = torch.randint(-50, 51, (M, N), generator=torch.Generator().manual_seed(6)).float().to(dev)
    return a16, b16, bias, init


@pytest.mark.gpu
@pytest.mark.parametrize("bn", (32, 128))
@pytest.mark.parametrize("M,N,K,split_k,kblocks", SPLITS)
def test_cta_exact_split_k(C, M, N, K, split_k, kblocks, bn):
    """K splits atomically added onto a non-zero start, the bias added by split 0 alone, at the split counts whose last
    split is short; fp32 at a pitch past N"""
    assert sum(kblocks) == math.ceil(K / 64) and len(kblocks) == split_k and kblocks[-1] < kblocks[0]
    a16, b16, bias, init = _split_inputs(M, N, K, "cuda")
    tag = f"{M}x{N}x{K} split_k={split_k} bn={bn}"
    _exact_in_fp32(tag, a16, b16, M, N, K, alpha=0.5, bias=bias, init=init)
    gm, out = _run(C, a16, b16, M, N, K, pair=0, bn=bn, bias=bias, alpha=0.5, f32=N + 3, bf16=False, transposed=False,
                   init=init, split_k=split_k)
    assert (gm.pair, gm.bn, gm.split_k, gm.epi, gm.mn_major()) == (0, bn, split_k, GENERIC, 0), tag
    assert gm.kblocks_per_split == kblocks[0], tag
    ref, _ = _reference(a16, b16, K, bias, 0.5, None)
    _check_exact(tag, (gm, out), ref, dict(f32=N + 3, init=init), M, N)


def _mn_inputs(M, N, K, exact, dev):
    return _operands(M, N, K, exact, seed=M + 3 * N + K, dev=dev, mn_major=True, pad=NAN)


def _mn_runs(M, N, split_k):
    """(name, expected variant, launch kwargs): the generic kernel with column sums (a K split accumulates instead), and
    the weight-gradient variant"""
    init = torch.randint(-50, 51, (M, N), generator=torch.Generator().manual_seed(7)).float() if split_k > 1 else None
    if split_k > 1:
        gen = dict(alpha=1.0, f32=N + 3, bf16=False, transposed=False, init=init, epi=GENERIC)
    else:
        gen = dict(alpha=1.0, f32=N + 3, colsum=True, transposed=M * N <= 1 << 22)
    return [("generic", GENERIC, gen),
            ("wgrad", WGRAD, dict(alpha=0.5, f32=N, bf16=False, transposed=False, init=init))]


@pytest.mark.gpu
@pytest.mark.parametrize("bn", (64, 128))
@pytest.mark.parametrize("M,N,K,split_k", MNMAJOR)
def test_cta_exact_mn_major(C, M, N, K, split_k, bn):
    """D = a^T . b with a [K, M] and b [K, N] row-major: the weight-gradient form, read straight from the row-major
    activation and dz buffers"""
    a16, b16, _ = _mn_inputs(M, N, K, True, "cuda")
    zero = torch.zeros(N, device="cuda")
    for name, epi, kw in _mn_runs(M, N, split_k):
        tag = f"{M}x{N}x{K} split_k={split_k} bn={bn} {name}"
        if kw.get("init") is not None:
            kw["init"] = kw["init"].cuda()
        _exact_in_fp32(tag, a16, b16, M, N, K, mn_major=True, alpha=kw["alpha"], init=kw.get("init"), colsum=kw.get("colsum", False))
        gm, out = _run(C, a16, b16, M, N, K, pair=0, bn=bn, split_k=split_k, mn_major=True, **kw)
        assert (gm.pair, gm.bn, gm.split_k, gm.epi, gm.mn_major()) == (0, bn, split_k, epi, 1), tag
        ref, _ = _reference(a16, b16, K, zero, kw["alpha"], None, M=M, N=N, mn_major=True)
        _check_exact(tag, (gm, out), ref, kw, M, N)


@pytest.mark.gpu
def test_cta_mn_major_width_clamp(C):
    """the MN-major kernel exists at BN 64 and 128: no width and BN 32 come back as 64, BN 256 as 128"""
    M, N, K = 130, 70, 17
    a16, b16, _ = _mn_inputs(M, N, K, True, "cuda")
    ref, _ = _reference(a16, b16, K, torch.zeros(N, device="cuda"), 1.0, None, M=M, N=N, mn_major=True)
    for bn, want in ((0, 64), (32, 64), (256, 128)):
        gm, out = _run(C, a16, b16, M, N, K, pair=0, bn=bn, mn_major=True, f32=N, bf16=False, transposed=False)
        assert gm.bn == want and gm.mn_major() == 1, (bn, gm.bn)
        assert torch.equal(out["f32"].double(), ref), bn


# ------------------------------------------------------------------------------------------------------------------
# exact cases: the specialized epilogue variants against float64, not only against the generic kernel
# ------------------------------------------------------------------------------------------------------------------
VARIANT_GEOMETRY = [(300, 250, 784), (129, 40, 40), (300, 256, 10), (129, 40, 37)]


@pytest.mark.gpu
@pytest.mark.parametrize("bn", (32, 64))
@pytest.mark.parametrize("M,N,K", VARIANT_GEOMETRY)
def test_cta_exact_fwd_and_dgrad_variants(C, M, N, K, bn):
    a16, b16, bias = _operands(M, N, K, True, seed=M * N + K, dev="cuda", pad=NAN)
    zero = torch.zeros(N, device="cuda")
    for act, alpha in ((None, 0.5), ("relu", 1.0)):
        tag = f"{M}x{N}x{K} bn={bn} FWD act={act}"
        _exact_in_fp32(tag, a16, b16, M, N, K, alpha=alpha, bias=bias)
        gm, out = _run(C, a16, b16, M, N, K, pair=0, bn=bn, bias=bias, act=act, alpha=alpha, transposed=False)
        assert (gm.bn, gm.split_k, gm.epi, gm.mn_major()) == (bn, 1, FWD, 0), tag
        ref, _ = _reference(a16, b16, K, bias, alpha, act)
        _check_exact(tag, (gm, out), ref, {}, M, N)
    for aux_act in (None, "relu", "sigmoid", "tanh"):
        tag = f"{M}x{N}x{K} bn={bn} DGRAD aux_act={aux_act}"
        aux = _aux(M, N, aux_act, True, seed=K + bn, dev="cuda")
        _exact_in_fp32(tag, a16, b16, M, N, K, aux=aux, aux_act=aux_act, colsum=True)
        gm, out = _run(C, a16, b16, M, N, K, pair=0, bn=bn, aux=aux, aux_act=aux_act, colsum=True, transposed=False)
        assert (gm.bn, gm.split_k, gm.epi, gm.mn_major()) == (bn, 1, DGRAD, 0), tag
        ref, _ = _reference(a16, b16, K, zero, 1.0, None, aux, aux_act)
        _check_exact(tag, (gm, out), ref, {}, M, N)


def _mse_exact_inputs(M, N, K, dev):
    a16, b16, bias = _operands(M, N, K, True, seed=M + N, dev=dev, pad=NAN, lim=1)
    ld_t = N + 5
    tgt = torch.full((M, ld_t), NAN)
    tgt[:, :N] = torch.randint(-4, 5, (M, N), generator=torch.Generator().manual_seed(8)).float()
    return a16, b16, bias, tgt.to(dev), ld_t


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,bn", [(256, 32, 784, 32), (128, 64, 37, 64), (128, 64, 37, 32)])
def test_cta_exact_loss_variant(C, M, N, K, bn):
    """The LOSS variant's MSE head on integer logits and integer targets, where M * N is a power of two: the gradient
    scale 2 / (M N) is then a power of two too and the head is exact."""
    a16, b16, bias, tgt, ld_t = _mse_exact_inputs(M, N, K, "cuda")
    tag = f"{M}x{N}x{K} bn={bn} LOSS mse"
    _exact_in_fp32(tag, a16, b16, M, N, K, bias=bias)
    z, _ = _reference(a16, b16, K, bias, 1.0, None)
    d = z - tgt[:, :N].double()
    scale = 2.0 / (M * N)
    assert _exponent(scale) > 0 and scale == 2.0 ** -_exponent(scale)
    assert float(d.abs().max()) < 2 ** 24 and float((d * d).sum()) < 2 ** 24 and float(d.abs().sum(0).max()) < 2 ** 24, tag
    loss = torch.zeros(1, device="cuda")
    gm, out = _run(C, a16, b16, M, N, K, pair=0, bn=bn, bias=bias, colsum=True, transposed=False,
                   extra=dict(loss_mode=MSE, target=native.ptr(tgt), ld_target=ld_t, loss=native.ptr(loss)))
    assert (gm.bn, gm.split_k, gm.epi, gm.mn_major()) == (bn, 1, LOSS, 0), tag
    _check_exact(tag, (gm, out), d * scale, dict(colsum=True), M, N)
    assert float(loss) == float((d * d).sum() * scale / 2), tag


# ------------------------------------------------------------------------------------------------------------------
# real-valued cases
# ------------------------------------------------------------------------------------------------------------------
REAL_CASES = [("bias", None, None), ("sigmoid", "sigmoid", None), ("tanh", "tanh", None), ("dgrad-sigmoid", None, "sigmoid"),
              ("dgrad-tanh", None, "tanh")]


def _check_real(tag, out, ref, bound, M, N, worst, name):
    frac = _fraction(out["f32"][:, :N], ref, bound)
    worst[name] = max(worst.get(name, 0.0), frac)
    assert frac <= 1.0, f"{tag}: error {frac:.2f} x the bound"
    if "colsum" in out:
        cf = _fraction(out["colsum"], ref.sum(0), _colsum_bound(ref, bound))
        worst[name + " colsum"] = max(worst.get(name + " colsum", 0.0), cf)
        assert cf <= 1.0, f"{tag}: column sums {cf:.2f} x the bound"


@pytest.mark.gpu
@pytest.mark.parametrize("geo", KMAJOR, ids=_ids(KMAJOR))
def test_cta_real_valued_kmajor(C, geo):
    M, N, K = _geometry(geo)
    a16, b16, bias = _operands(M, N, K, False, seed=7 * M + N + K, dev="cuda", pad=NAN)
    zero = torch.zeros(N, device="cuda")
    worst = {}
    for bn in BNS:
        for name, act, aux_act in REAL_CASES:
            aux = _aux(M, N, aux_act, False, seed=N, dev="cuda") if aux_act else None
            kw = dict(bias=None if aux_act else bias, act=act, alpha=1.0 if aux_act else 0.75, aux=aux, aux_act=aux_act,
                      colsum=aux_act is not None, f32=N)
            tag = f"{M}x{N}x{K} bn={bn} {name}"
            gm, out = _run(C, a16, b16, M, N, K, pair=0, bn=bn, **kw)
            assert (gm.pair, gm.bn, gm.split_k, gm.epi) == (0, bn, 1, GENERIC), tag
            _check_layout(tag, out, M, N, N)
            ref, bound = _reference(a16, b16, K, zero if aux_act else bias, kw["alpha"], act, aux, aux_act)
            _check_real(tag, out, ref, bound, M, N, worst, name)
    print(f"[gemm-cta] {M}x{N}x{K}: worst error / bound " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,split_k,kblocks", SPLITS)
def test_cta_real_valued_split_k(C, M, N, K, split_k, kblocks):
    a16, b16, bias = _operands(M, N, K, False, seed=M + N + K, dev="cuda", pad=NAN)
    worst = {}
    for bn in (32, 128):
        tag = f"{M}x{N}x{K} split_k={split_k} bn={bn}"
        gm, out = _run(C, a16, b16, M, N, K, pair=0, bn=bn, bias=bias, alpha=0.75, f32=N, bf16=False, transposed=False,
                       init=torch.zeros(M, N, device="cuda"), split_k=split_k)
        assert (gm.bn, gm.split_k) == (bn, split_k), tag
        ref, bound = _reference(a16, b16, K, bias, 0.75, None, splits=split_k)
        _check_real(tag, out, ref, bound, M, N, worst, f"bn {bn}")
    print(f"[gemm-cta] {M}x{N}x{K} split_k={split_k}: worst error / bound " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,split_k", MNMAJOR)
def test_cta_real_valued_mn_major(C, M, N, K, split_k):
    a16, b16, _ = _mn_inputs(M, N, K, False, "cuda")
    zero = torch.zeros(N, device="cuda")
    worst = {}
    for bn in (64, 128):
        tag = f"{M}x{N}x{K} split_k={split_k} bn={bn}"
        init = torch.zeros(M, N, device="cuda") if split_k > 1 else None
        gm, out = _run(C, a16, b16, M, N, K, pair=0, bn=bn, alpha=0.5, f32=N, bf16=False, transposed=False, colsum=split_k == 1,
                       init=init, split_k=split_k, mn_major=True)
        assert (gm.bn, gm.split_k, gm.mn_major()) == (bn, split_k, 1), tag
        ref, bound = _reference(a16, b16, K, zero, 0.5, None, M=M, N=N, mn_major=True, splits=split_k)
        _check_real(tag, out, ref, bound, M, N, worst, f"bn {bn}")
    print(f"[gemm-cta] MN-major {M}x{N}x{K}: worst error / bound " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


# ------------------------------------------------------------------------------------------------------------------
# fused loss heads: float64 references and bounds
# ------------------------------------------------------------------------------------------------------------------
TINY = 2.0 ** -126           # absolute slack for a result that leaves the normal fp32 range


def _g(n):
    """gamma_n: the relative error bound of n fp32 roundings"""
    return n * U / (1 - n * U)


def _mul(x, ex, y, ey):
    """x * y, one rounding, from x and y known to within ex and ey"""
    return x * y, abs(x) * ey + abs(y) * ex + ex * ey + U * (abs(x) + ex) * (abs(y) + ey) + TINY


def _add(x, ex, y, ey):
    """x + y, one rounding"""
    return x + y, ex + ey + U * (abs(x + y) + ex + ey)


def _expf(x, ex):
    """__expf: the input error through exp, then at most 2 + 1.173 |x| ulp, an ulp being at most 2u of the value"""
    hi = torch.exp(x + ex)
    return torch.exp(x), torch.exp(x) * torch.expm1(ex) + (2 + 1.173 * (x.abs() + ex)) * 2 * U * hi + TINY


def _rcp(y, ey):
    """__fdividef(1, y) for y > ey >= 0: the input error through 1 / y, then 2 ulp"""
    lo = y - ey
    return 1 / y, ey / (y * lo) + 4 * U / lo


def _logf(y, ey):
    """__logf for y > ey >= 0: the input error through log, then at most 2^-21.41 absolute on [0.5, 2] and 3 ulp elsewhere"""
    v = torch.log(y)
    ein = torch.log(y / (y - ey))
    return v, ein + 2.0 ** -21.41 + 6 * U * (v.abs() + ein)


def _softmax_xent_ref(z, ez, y):
    """float64 loss and dz of the softmax cross-entropy head on logits z (known to within ez, see ``_reference``) and label
    rows y, with their bounds; the head's arithmetic, row by row (it holds a whole row, N <= 32):
      mx = max z;  ex = __expf(z - mx);  se = sum ex;  ysum = sum y;  zy = sum y z
      loss_row = ((mx + __logf(se)) ysum - zy) / M;   dz = (ex __fdividef(1, se) ysum - y) / M
    1 / M is __fdividef's (2 ulp); the row losses are summed by a 32-lane shuffle tree and one atomic add per 32 rows."""
    M, N = z.shape
    mx = z.max(1, keepdim=True).values
    emx = ez.max(1, keepdim=True).values                  # the computed maximum is one of the computed logits
    t, et = _add(z, ez, -mx, emx)
    ex, eex = _expf(t, et)
    se = ex.sum(1, keepdim=True)
    ese = eex.sum(1, keepdim=True) + _g(N) * (ex + eex).sum(1, keepdim=True)
    ysum = y.sum(1, keepdim=True)
    eys = _g(N) * y.abs().sum(1, keepdim=True)
    yz, eyz = _mul(y, 0, z, ez)
    zy = yz.sum(1, keepdim=True)
    ezy = eyz.sum(1, keepdim=True) + _g(N) * (yz.abs() + eyz).sum(1, keepdim=True)
    inv_b, einv_b = 1.0 / M, 4 * U / M
    lse, else_ = _logf(se, ese)
    s, es = _add(mx, emx, lse, else_)
    s, es = _mul(s, es, ysum, eys)
    s, es = _add(s, es, -zy, ezy)
    lrow, elrow = _mul(s, es, inv_b, einv_b)
    loss = float(lrow.sum())
    eloss = float(elrow.sum() + _g(5 + math.ceil(M / 32)) * (lrow.abs() + elrow).sum())
    inv_se, einv = _rcp(se, ese)
    p, ep = _mul(ex, eex, inv_se, einv)
    q, eq = _mul(p, ep, ysum, eys)
    r, er = _add(q, eq, -y, 0)
    dz, edz = _mul(r, er, inv_b, einv_b)
    return loss, eloss, dz, edz


def _mse_ref(f, ef, t, act):
    """float64 loss and dz of the MSE head on outputs f (after the activation, known to within ef) and targets t, with
    their bounds: scale = 2 / (M N) (an IEEE division), d = f - t, dz = d scale (times a (1 - a) after a sigmoid); the loss
    sums d^2 over each row's 32-column chunk, a 32-row shuffle tree and one atomic add of sum * 0.5 * scale per chunk and
    32 rows."""
    M, N = f.shape
    scale = 2.0 / (M * N)
    d, ed = _add(f, ef, -t, 0)
    dz, edz = _mul(d, ed, scale, U * scale)
    if act == "sigmoid":
        om, eom = _add(1.0, 0, -f, ef)
        da, eda = _mul(f, ef, om, eom)
        dz, edz = _mul(dz, edz, da, eda)
    sq, esq = _mul(d, ed, d, ed)
    depth = 32 + 5 + math.ceil(M / 32) * math.ceil(N / 32)
    total = float(sq.sum())
    etotal = float(esq.sum() + _g(depth) * (sq + esq).sum())
    return total * 0.5 * scale, (etotal + 3 * U * (total + etotal)) * 0.5 * scale + TINY, dz, edz


def _labels(M, N, seed):
    """label rows cycling through one-hot, soft rows summing to 0.5, soft rows summing to 1.7 and all-zero rows (the first
    kind moves with N, so that one-row cases see each)"""
    g = torch.Generator().manual_seed(seed)
    kind = (torch.arange(M) + N) % 4
    w = torch.rand(M, N, generator=g) + 0.05
    w = w / w.sum(1, keepdim=True)
    hot = torch.nn.functional.one_hot(torch.randint(0, N, (M,), generator=g), N).float()
    y = torch.where((kind == 0)[:, None], hot, torch.zeros(M, N))
    y = torch.where((kind == 1)[:, None], 0.5 * w, y)
    y = torch.where((kind == 2)[:, None], 1.7 * w, y)
    return y


def _head_logit_operands(M, N, dev, seed):
    """real-valued operands whose logits alpha A B^T + bias spread over tens of units: alpha 3, a bias in [-20, 20]"""
    K = 90
    a16, b16, _ = _operands(M, N, K, False, seed=seed, dev=dev, pad=NAN)
    bias = (torch.rand(N, generator=torch.Generator().manual_seed(seed + 2)) * 40 - 20).to(dev)
    return a16, b16, bias, K, 3.0


def _padded(t, ld):
    out = torch.full((t.shape[0], ld), NAN, device=t.device)
    out[:, :t.shape[1]] = t
    return out


def _check_head(tag, out, loss, M, N, ref_loss, eloss, dz, edz):
    """bf16 dz within the fp32 bound plus half a bf16 step, its pads zero; column sums of the fp32 dz; the loss"""
    _check_layout(tag, out, M, N)
    bound = edz + BF16_HALF_STEP * (dz.abs() + edz)
    fd = _fraction(out["bf16"][:, :N], dz, bound)
    fc = _fraction(out["colsum"], dz.sum(0), _colsum_bound(dz, edz))
    fl = abs(float(loss) - ref_loss) / eloss
    assert fd <= 1.0 and fc <= 1.0 and fl <= 1.0, f"{tag}: dz {fd:.2f}, column sums {fc:.2f}, loss {fl:.2f} x the bound"
    return fd, fc, fl


SOFTMAX_N = (1, 2, 10, 31, 32)
MSE_N = (10, 784, 1000)
HEAD_M = (1, 129, 1000)


@pytest.mark.gpu
@pytest.mark.parametrize("M", HEAD_M)
@pytest.mark.parametrize("N", SOFTMAX_N)
def test_cta_softmax_xent_head(C, N, M):
    """softmax cross-entropy through the LOSS variant and through the generic kernel (with the transposed dz), one-hot,
    soft (rows summing to 0.5 and 1.7) and all-zero label rows"""
    a16, b16, bias, K, alpha = _head_logit_operands(M, N, "cuda", seed=M + 40 * N)
    y = _labels(M, N, seed=M + N).cuda()
    ld_y = N + 3
    yp = _padded(y, ld_y)
    z, ez = _reference(a16, b16, K, bias, alpha, None)
    ref = _softmax_xent_ref(z, ez, y.double())
    for path, epi, want in (("LOSS variant", -1, LOSS), ("generic", GENERIC, GENERIC)):
        tag = f"{M}x{N} softmax {path}"
        loss = torch.zeros(1, device="cuda")
        gm, out = _run(C, a16, b16, M, N, K, pair=0, bn=32, bias=bias, alpha=alpha, colsum=True, transposed=epi == GENERIC,
                       epi=epi, extra=dict(loss_mode=SOFTMAX, target=native.ptr(yp), ld_target=ld_y, loss=native.ptr(loss)))
        assert (gm.bn, gm.split_k, gm.epi) == (32, 1, want), tag
        fr = _check_head(tag, out, loss, M, N, *ref)
        print(f"[gemm-cta] {tag}: worst error / bound dz {fr[0]:.3f}, column sums {fr[1]:.3f}, loss {fr[2]:.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("act", [None, "sigmoid"])
@pytest.mark.parametrize("M", HEAD_M)
@pytest.mark.parametrize("N", MSE_N)
def test_cta_mse_head(C, N, M, act):
    """MSE through the LOSS variant (BN 64) and the generic kernel (BN 128, with the transposed dz), targets at a pitch
    past N"""
    K = 196
    a16, b16, bias = _operands(M, N, K, False, seed=M + N, dev="cuda", pad=NAN)
    t = torch.rand(M, N, generator=torch.Generator().manual_seed(N)).cuda()
    ld_t = N + 5
    tp = _padded(t, ld_t)
    f, ef = _reference(a16, b16, K, bias, 1.0, act)
    ref = _mse_ref(f, ef, t.double(), act)
    for path, bn, epi, want in (("LOSS variant", 64, -1, LOSS), ("generic", 128, GENERIC, GENERIC)):
        tag = f"{M}x{N} mse act={act} {path}"
        loss = torch.zeros(1, device="cuda")
        gm, out = _run(C, a16, b16, M, N, K, pair=0, bn=bn, bias=bias, act=act, colsum=True, transposed=epi == GENERIC, epi=epi,
                       extra=dict(loss_mode=MSE, target=native.ptr(tp), ld_target=ld_t, loss=native.ptr(loss)))
        assert (gm.bn, gm.split_k, gm.epi) == (bn, 1, want), tag
        fr = _check_head(tag, out, loss, M, N, *ref)
        print(f"[gemm-cta] {tag}: worst error / bound dz {fr[0]:.3f}, column sums {fr[1]:.3f}, loss {fr[2]:.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [SOFTMAX, SPARSE])
def test_softmax_heads_run_at_bn_32_whatever_width_is_requested(C, mode):
    """Both softmax heads hold a whole row in one 32-column chunk: a wider requested tile comes back as BN 32 (with the B
    tensor map built for it) and computes exactly what the default width does"""
    M, N = 129, 10
    a16, b16, bias, K, alpha = _head_logit_operands(M, N, "cuda", seed=11)
    cls = torch.randint(0, N, (M,), generator=torch.Generator().manual_seed(12))
    y = torch.nn.functional.one_hot(cls, N).float().cuda()
    target, ld = (y, N) if mode == SOFTMAX else (cls.float().cuda(), 1)
    z, ez = _reference(a16, b16, K, bias, alpha, None)
    ref = _softmax_xent_ref(z, ez, y.double())
    first = None
    for bn in (0, 64, 128, 256):
        tag = f"loss_mode={mode} bn={bn}"
        loss = torch.zeros(1, device="cuda")
        gm, out = _run(C, a16, b16, M, N, K, pair=0, bn=bn, bias=bias, alpha=alpha, colsum=True,
                       extra=dict(loss_mode=mode, target=native.ptr(target), ld_target=ld, loss=native.ptr(loss)))
        # gm.bn was 32 before the B tensor map was built at that width too (the width used to be forced afterwards):
        # this assertion does not pin the map's box height, the bit-identical outputs below do
        assert gm.bn == 32 and gm.split_k == 1, tag
        _check_head(tag, out, loss, M, N, *ref)
        if first is None:
            first = out
        for k in ("bf16", "T"):
            assert torch.equal(out[k], first[k]), f"{tag}: {k} differs from the default width's"


# ------------------------------------------------------------------------------------------------------------------
# CPU: the exactness condition of every exact case, and the bounds against plausible faults
# ------------------------------------------------------------------------------------------------------------------
def test_exact_cases_are_exact_in_fp32():
    """every exact case above meets the condition its GPU test asserts before it demands bit equality"""
    for geo in KMAJOR:
        M, N, K, a16, b16, bias = _exact_kmajor_inputs(geo, "cpu")
        for bn_index, bn in enumerate(BNS):
            for name, kw in _kmajor_runs(M, N, bn_index):
                kw = _resolve(kw, bias, M, N, "cpu", seed=M + bn)
                _exact_in_fp32(f"{M}x{N}x{K} bn={bn} {name}", a16, b16, M, N, K, alpha=kw["alpha"], bias=kw["bias"],
                               init=kw.get("init"), aux=kw.get("aux"), aux_act=kw.get("aux_act"), colsum=kw.get("colsum", False))
    for M, N, K, split_k, _ in SPLITS:
        a16, b16, bias, init = _split_inputs(M, N, K, "cpu")
        _exact_in_fp32(f"{M}x{N}x{K} split_k={split_k}", a16, b16, M, N, K, alpha=0.5, bias=bias, init=init)
    for M, N, K, split_k in MNMAJOR:
        a16, b16, _ = _mn_inputs(M, N, K, True, "cpu")
        for name, _, kw in _mn_runs(M, N, split_k):
            _exact_in_fp32(f"MN {M}x{N}x{K} {name}", a16, b16, M, N, K, mn_major=True, alpha=kw["alpha"], init=kw.get("init"),
                           colsum=kw.get("colsum", False))
    for M, N, K in VARIANT_GEOMETRY:
        for bn in (32, 64):
            a16, b16, bias = _operands(M, N, K, True, seed=M * N + K, dev="cpu", pad=NAN)
            for alpha in (0.5, 1.0):
                _exact_in_fp32(f"FWD {M}x{N}x{K}", a16, b16, M, N, K, alpha=alpha, bias=bias)
            for aux_act in (None, "relu", "sigmoid", "tanh"):
                aux = _aux(M, N, aux_act, True, seed=K + bn, dev="cpu")
                _exact_in_fp32(f"DGRAD {M}x{N}x{K} {aux_act}", a16, b16, M, N, K, aux=aux, aux_act=aux_act, colsum=True)


def _faults(M, N, K, split_k):
    """(what, got, ref, bound) for each fault, computed on the CPU"""
    a16, b16, bias = _operands(M, N, K, False, seed=M + N + K, dev="cpu", pad=NAN)
    A, B = _logical(a16, b16, K, N)
    ref, bound = _reference(a16, b16, K, bias, 0.75, None, splits=split_k)
    kb = -(-math.ceil(K / 64) // split_k)                       # k-blocks per split
    last = (split_k - 1) * kb * 64
    yield "the bias added on every K split", ref + (split_k - 1) * bias.double(), ref, bound
    yield "the short last K split dropped", ref - 0.75 * A[:, last:] @ B[:, last:].t(), ref, bound
    got = ref.clone()
    got[127] = 0
    yield "the last row of a 128-row tile missing", got, ref, bound
    aux = _aux(M, N, "sigmoid", False, seed=N, dev="cpu")
    f, e = _reference(a16, b16, K, torch.zeros(N), 1.0, None, aux, "sigmoid")
    tiles = (M // 128) * 128
    yield "the column sums missing the last partial row tile", f[:tiles].sum(0), f.sum(0), _colsum_bound(f, e)
    za16, zb16, zbias, zK, alpha = _head_logit_operands(M, 10, "cpu", seed=3)
    z, ez = _reference(za16, zb16, zK, zbias, alpha, None)
    y = _labels(M, 10, seed=4).double()
    _, _, dz, edz = _softmax_xent_ref(z, ez, y)
    p = torch.softmax(z, 1)
    yield "softmax dz computed as p - y", (p - y) / M, dz, edz + BF16_HALF_STEP * (dz.abs() + edz)


@pytest.mark.parametrize("M,N,K,split_k,kblocks", SPLITS[:2])
def test_bounds_reject_plausible_faults(M, N, K, split_k, kblocks):
    """The real-valued comparisons can fail: the fp32 rounding of each reference passes its bound, and the reference with
    (a) the bias added by every K split, (b) the short last K split dropped, (c) the last row of a 128-row tile missing,
    (d) the column sums missing the last partial row tile, (e) the softmax dz computed as p - y instead of p sum(y) - y is
    rejected."""
    assert M % 128 != 0 and kblocks[-1] < kblocks[0]
    for what, got, ref, bound in _faults(M, N, K, split_k):
        assert _fraction(ref.float(), ref, bound) <= 1.0, what
        frac = _fraction(got.float(), ref, bound)
        print(f"[gemm-cta] {M}x{N}x{K} split_k={split_k} with {what}: {frac:.1f} x the bound")
        assert frac > 1.0, f"{M}x{N}x{K}: the bound accepts the output with {what}"
