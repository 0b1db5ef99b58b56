"""float64 references of the GEMM kernels (csrc/gemm_sm90.cu, csrc/gemm_pair_sm90.cu) and element-wise error bounds
derived from their fp32 arithmetic.  The operand, reference and bound helpers are device-agnostic: the CPU tests use them
too.  ``_run`` launches one GEMM."""
import math

import torch

from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import round_up

ACT = {None: 0, "relu": 1, "sigmoid": 2, "tanh": 3}
U = 2.0 ** -24                      # fp32 unit roundoff


def _operands(M, N, K, exact, seed, dev, mn_major=False, pad=0.0, lim=3):
    """bf16 operands and an fp32 bias [N].  K-major: A [M, round_up(K, 8)], B [N, round_up(K, 8)]; MN-major: A
    [K, round_up(M, 8)], B [K, round_up(N, 8)].  `pad` fills the columns between the logical extent and the row pitch.
    exact: integer operands in [-lim, lim] and an integer bias."""
    g = torch.Generator().manual_seed(seed)
    if exact:
        a = torch.randint(-lim, lim + 1, (M, K), generator=g).float()
        b = torch.randint(-lim, lim + 1, (N, K), generator=g).float()
        bias = torch.randint(-8, 9, (N,), generator=g).float()
    else:
        a = torch.randn(M, K, generator=g) * 0.5
        b = torch.randn(N, K, generator=g) * 0.5
        bias = torch.randn(N, generator=g)
    if mn_major:
        a16 = torch.full((K, round_up(M, 8)), pad, dtype=torch.bfloat16)
        b16 = torch.full((K, round_up(N, 8)), pad, dtype=torch.bfloat16)
        a16[:, :M], b16[:, :N] = a.t().to(torch.bfloat16), b.t().to(torch.bfloat16)
    else:
        a16 = torch.full((M, round_up(K, 8)), pad, dtype=torch.bfloat16)
        b16 = torch.full((N, round_up(K, 8)), pad, dtype=torch.bfloat16)
        a16[:, :K], b16[:, :K] = a.to(torch.bfloat16), b.to(torch.bfloat16)
    return a16.to(dev), b16.to(dev), bias.to(dev)


def _logical(a16, b16, K, N=None, M=None, mn_major=False):
    """the float64 operands A [M, K] and B [N, K] without their pads"""
    if mn_major:
        return a16[:K, :M].t().double(), b16[:K, :N].t().double()
    N = N or b16.shape[0]
    return a16[:, :K].double(), b16[:N, :K].double()


# act'(aux) exact in fp32 at these stored activations: relu 0 / 1, sigmoid a(1 - a) = 3/16 or 1/4, tanh 1 - a^2 = 1, 15/16,
# 3/4; any value with no activation (act' = 1)
AUX_EXACT = {None: (-1.5, 0.0, 2.0), "relu": (0.0, 0.5, 1.0, 2.0), "sigmoid": (0.25, 0.5, 0.75), "tanh": (-0.5, 0.0, 0.25, 0.5)}


def _aux(M, N, aux_act, exact, seed, dev):
    g = torch.Generator().manual_seed(seed + 1)
    if exact:
        vals = torch.tensor(AUX_EXACT[aux_act])
        a = vals[torch.randint(0, len(vals), (M, N), generator=g)]
    else:
        z = torch.randn(M, N, generator=g) * 2
        a = {None: lambda v: v, "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}[aux_act](z)
    out = torch.zeros(M, round_up(N, 8), dtype=torch.bfloat16)
    out[:, :N] = a.to(torch.bfloat16)
    return out.to(dev)


def _dact64(a, aux_act):
    if aux_act == "relu":
        return (a > 0).double()
    if aux_act == "sigmoid":
        return a * (1 - a)
    if aux_act == "tanh":
        return 1 - a * a
    return torch.ones_like(a)


def _reference(a16, b16, K, bias, alpha, act, aux=None, aux_act=None, N=None, M=None, mn_major=False, splits=1):
    """float64 epilogue output f (before any accumulate) and its element-wise error bound for fp32 arithmetic.

    The bound adds up, per element:
      * the main loop: ceil(K / 16) + 1 fp32 roundings of the accumulator (one per 16-deep tensor-core step, each allowed
        to truncate: 2u relative) of partial sums no larger than S = sum_k |a_k b_k|;
      * alpha * acc + bias: 2u of |alpha| S + |bias|;
      * `splits` K splits atomically added onto a zero start: each further split starts a new accumulator chain (one more
        rounding of its partial sum), scales it and adds it to the running total: 4u of |alpha| S + |bias| per split;
      * the activation: relu and none pass the error on; sigmoid_fast halves it twice (slope <= 1/4) and adds its own
        relative error, __expf's (2 + 1.17 |z|) ulp plus one add and __fdividef's 2 ulp, below 2^-20 (1 + |z|) of the
        value; tanh_fast passes the error on (slope <= 1) and adds the same 2^-20 (1 + |z|), but absolutely: near 0 it
        is the difference 1 - e^{-2|z|} that carries __expf's error;
      * act'(aux): act' rounded in fp32 and the product rounded: 4u of |f| (1 + |act'|)."""
    A, B = _logical(a16, b16, K, N, M, mn_major)
    N = B.shape[0]
    acc = A @ B.t()
    S = A.abs() @ B.abs().t()
    bias = bias.double()
    z = alpha * acc + bias
    e = abs(alpha) * (math.ceil(K / 16) + 1) * 2 * U * S + 2 * U * (abs(alpha) * S + bias.abs())
    e = e + (splits - 1) * 4 * U * (abs(alpha) * S + bias.abs())
    if act == "relu":
        f = torch.relu(z)
    elif act == "sigmoid":
        f = torch.sigmoid(z)
        e = e / 4 + 2.0 ** -20 * (1 + z.abs()) * f
    elif act == "tanh":
        f = torch.tanh(z)
        e = e + 2.0 ** -20 * (1 + z.abs())
    else:
        f = z
    if aux is not None:
        d = _dact64(aux[:, :N].double(), aux_act)
        rounded = aux_act in ("sigmoid", "tanh")
        e = e * d.abs() + (4 * U * f.abs() * (1 + d.abs()) if rounded else 0)
        f = f * d
    return f, e


def _colsum_bound(f, e):
    """column sums: the rows' own errors plus a 32-row shuffle tree (5 roundings) and one atomic add per 32-row group"""
    M = f.shape[0]
    return e.sum(0) + (5 + math.ceil(M / 32)) * U * (f.abs() + e).sum(0)


def _fraction(got, ref, bound):
    """worst |got - ref| / bound (0 where both are 0)"""
    d = (got.double() - ref).abs()
    return float((d / bound.clamp_min(1e-300)).max())


def _run(C, a16, b16, M, N, K, pair=1, pair_ctas=0, bn=0, bias=None, act=None, alpha=1.0, aux=None, aux_act=None,
         colsum=False, f32=None, bf16=True, transposed=True, init=None, split_k=1, mn_major=False, epi=-1, extra=None):
    """One launch.  ``f32``: None (no fp32 output) or the fp32 row pitch; ``init``: start value of the fp32 output for an
    accumulating launch; ``extra``: further Gemm fields (a loss head's).  Returns (the Gemm, dict of outputs)."""
    dev = a16.device
    ldn, ldt = round_up(N, 8), round_up(M, 8)
    out = {}
    if f32 is not None:
        buf = torch.full((M, f32), 1234.5, device=dev)
        if init is not None:
            buf[:, :N] = init
        out["f32"] = buf
    if bf16:
        out["bf16"] = torch.full((M, ldn), 99.0, dtype=torch.bfloat16, device=dev)   # pad columns: must come back 0
    if transposed:
        out["T"] = torch.zeros(N, ldt, dtype=torch.bfloat16, device=dev)
    if colsum:
        out["colsum"] = torch.zeros(N, device=dev)
    d = dict(a=native.ptr(a16), b=native.ptr(b16), M=M, N=N, K=K, lda=a16.shape[1], ldb=b16.shape[1], bn=bn, pair=pair,
             pair_ctas=pair_ctas, bias=native.ptr(bias), act=ACT[act], alpha=alpha, aux=native.ptr(aux),
             ld_aux=aux.shape[1] if aux is not None else 0, aux_act=ACT[aux_act], colsum=native.ptr(out.get("colsum")),
             out_f32=native.ptr(out.get("f32")), ld_f32=f32 or N, accumulate=int(init is not None),
             out_bf16=native.ptr(out.get("bf16")), ld_bf16=ldn if bf16 else 0, outT_bf16=native.ptr(out.get("T")),
             ld_t=ldt if transposed else 0, split_k=split_k, mn_major=int(mn_major), epi=epi, **(extra or {}))
    gm = C.Gemm(d)
    gm.launch(native.current_stream())
    torch.cuda.synchronize()
    assert C.read_error_code() == 0
    return gm, out


def _check_layout(tag, out, M, N, f32=None):
    """what every case asserts beyond the values: pads, untouched fp32 pitch, transposed == row-major"""
    if "bf16" in out:
        assert torch.all(out["bf16"][:, N:] == 0), f"{tag}: bf16 pad columns"
        if "T" in out:
            assert torch.equal(out["T"][:, :M].t(), out["bf16"][:, :N]), f"{tag}: transposed != row-major"
            assert torch.all(out["T"][:, M:] == 0), f"{tag}: transposed pad columns written"
        if "f32" in out:
            assert torch.equal(out["bf16"][:, :N], out["f32"][:, :N].to(torch.bfloat16)), f"{tag}: bf16 != bf16(fp32 output)"
    if f32 is not None and f32 > N:
        assert torch.all(out["f32"][:, N:] == 1234.5), f"{tag}: fp32 columns past N written"


def _exact_bf16(ref):
    return ref.float().to(torch.bfloat16)
