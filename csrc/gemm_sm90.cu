// wgmma / TMA GEMM for sm_90a with fused training epilogues.
//
//   D[M,N] = alpha * A[M,K] . B[N,K]^T          (both operands K-major, bf16, fp32 accumulate)
//
// One CTA computes one 128 x BN output tile (optionally one K-split of it):
//   warp 0       : TMA producer  (cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier tx-count)
//   warps 1-3    : bias tile loader
//   warpgroups 1-2: wgmma main loop, 64 rows each, accumulator in registers; then both stage the fp32 tile in the
//                  drained operand ring and run the epilogue (one row per thread, 32-column chunks -> fused math -> global)
//
// Fused epilogues cover everything a dense layer needs in training (reference ops K1/K2 of
// SURVEY.md section 2.4: MatMul+BiasAdd+{Relu,Sigmoid,Tanh}, their gradients and BiasAddGrad):
//   * bias add + activation, bf16 output and its transpose (the transpose feeds the K-major
//     operand of the next wgrad GEMM, so no separate transpose kernel exists),
//   * dgrad: multiply by act'(previous activation) read from the forward buffer,
//   * column sums (bias gradient) via an in-register transpose-reduce + one red per column,
//   * fp32 store or atomic accumulate (split-K / straight into the flat gradient buffer that the
//     push kernel consumes).
// The generic kernel (sf_gemm_kernel) tests each of these at run time.  The training GEMMs run specialized variants
// (sf_gemm_epi_kernel, one per SfEpi kind, sf_gemm_sigmoid_loss_kernel and sf_gemm_sparse_loss_kernel) that contain only their own epilogue code, a
// fifth to a half of the generic kernel's; the DGRAD / loss variants also fetch their act'(aux) / label rows before the
// main loop.
//
// The B operand may live in *peer* GPU memory: the tensor map simply carries the peer-mapped
// address, and the TMA engine pulls weight tiles over NVLink while the MMA pipeline runs
// (the "pull-fused" first dense layer of the parameter-server design).
#include <cstdlib>
#include "sm90_ptx.cuh"
#include "sf_api.h"

namespace sf {

constexpr int kBM = 128;
constexpr int kBK = 64;           // 64 bf16 = 128 B = one swizzle row
constexpr int kWgmmaK = 16;
constexpr int kGemmThreads = 384;
constexpr int kPairBN = 128;      // tile columns of the persistent cluster-pair kernel (gemm_pair_sm90.cu)

// Fast forms: the results are rounded to bf16 (or feed a loss) - a slow-path division per element would triple the
// epilogue's code size, and the epilogue is instruction-fetch bound (it runs once per launch on a cold I-cache).
__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
__device__ __forceinline__ float tanh_fast(float x) {
  const float t = __expf(-2.f * fabsf(x));
  return copysignf(__fdividef(1.f - t, 1.f + t), x);
}
__device__ __forceinline__ float act_fwd(float x, int act) {
  switch (act) {
    case SF_ACT_RELU: return fmaxf(x, 0.f);
    case SF_ACT_SIGMOID: return sigmoid_fast(x);
    case SF_ACT_TANH: return tanh_fast(x);
    default: return x;
  }
}
// derivative expressed through the activation *output* a
__device__ __forceinline__ float act_bwd_from_out(float a, int act) {
  switch (act) {
    case SF_ACT_RELU: return a > 0.f ? 1.f : 0.f;
    case SF_ACT_SIGMOID: return a * (1.f - a);
    case SF_ACT_TANH: return 1.f - a * a;
    default: return 1.f;
  }
}
// Whole-chunk forms of the extended activations (SfAct 4-9): one loop per kind, so the kind is tested once per chunk.
template <int ACT>
__device__ __forceinline__ void act_ext_fwd_chunk(float (&f)[32], float alpha) {
#pragma unroll
  for (int j = 0; j < 32; ++j) f[j] = act_ext_fwd(f[j], ACT, alpha);
}
template <int ACT>
__device__ __forceinline__ void act_ext_bwd_chunk(float (&f)[32], const float (&a)[32], float keep, float alpha) {
  if (keep > 0.f && keep < 1.f) {
    const float ik = __fdividef(1.f, keep);
    if constexpr (ACT == SF_ACT_RELU6) {
      // saturation is decided in stored units: a saturated unit holds bf16(6 * ik), rounded exactly as the forward
      // epilogue rounded it, and a * keep of that value is not 6 for most keep (keep 0.9: 6.65625 * 0.9 = 5.9906)
      const float sat = __bfloat162float(__float2bfloat16(6.f * ik));
#pragma unroll
      for (int j = 0; j < 32; ++j) f[j] *= (a[j] > 0.f && a[j] < sat) ? ik : 0.f;
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) f[j] *= a[j] != 0.f ? act_ext_dact(a[j] * keep, ACT, alpha) * ik : 0.f;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] *= act_ext_dact(a[j], ACT, alpha);
  }
}
__device__ __forceinline__ void act_ext_fwd32(float (&f)[32], int act, float alpha) {
  switch (act) {
    case SF_ACT_ELU: act_ext_fwd_chunk<SF_ACT_ELU>(f, alpha); break;
    case SF_ACT_SELU: act_ext_fwd_chunk<SF_ACT_SELU>(f, alpha); break;
    case SF_ACT_SOFTPLUS: act_ext_fwd_chunk<SF_ACT_SOFTPLUS>(f, alpha); break;
    case SF_ACT_SOFTSIGN: act_ext_fwd_chunk<SF_ACT_SOFTSIGN>(f, alpha); break;
    case SF_ACT_LEAKY_RELU: act_ext_fwd_chunk<SF_ACT_LEAKY_RELU>(f, alpha); break;
    case SF_ACT_RELU6: act_ext_fwd_chunk<SF_ACT_RELU6>(f, alpha); break;
    default: break;
  }
}
__device__ __forceinline__ void act_ext_bwd32(float (&f)[32], const float (&a)[32], int act, float keep, float alpha) {
  switch (act) {
    case SF_ACT_ELU: act_ext_bwd_chunk<SF_ACT_ELU>(f, a, keep, alpha); break;
    case SF_ACT_SELU: act_ext_bwd_chunk<SF_ACT_SELU>(f, a, keep, alpha); break;
    case SF_ACT_SOFTPLUS: act_ext_bwd_chunk<SF_ACT_SOFTPLUS>(f, a, keep, alpha); break;
    case SF_ACT_SOFTSIGN: act_ext_bwd_chunk<SF_ACT_SOFTSIGN>(f, a, keep, alpha); break;
    case SF_ACT_LEAKY_RELU: act_ext_bwd_chunk<SF_ACT_LEAKY_RELU>(f, a, keep, alpha); break;
    case SF_ACT_RELU6: act_ext_bwd_chunk<SF_ACT_RELU6>(f, a, keep, alpha); break;
    default: break;
  }
}

// whole-chunk forms: ONE (uniform) branch on the activation kind instead of one per element.  EXT: the kernel is a twin
// that also carries the extended set (act >= SF_ACT_ELU); without it these are the ReLU / sigmoid / tanh code alone.
template <bool EXT>
__device__ __forceinline__ void act_fwd32(float (&f)[32], int act, float alpha) {
  if (EXT && act >= SF_ACT_ELU) {
    act_ext_fwd32(f, act, alpha);
  } else if (act == SF_ACT_RELU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] = fmaxf(f[j], 0.f);
  } else if (act == SF_ACT_SIGMOID) {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] = sigmoid_fast(f[j]);
  } else if (act == SF_ACT_TANH) {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] = tanh_fast(f[j]);
  }
}
// f[j] *= act'(a[j]) (a = activation output); keep in (0, 1): a = act(z) * mask / keep (fused dropout), mask = a != 0
template <bool EXT>
__device__ __forceinline__ void act_bwd32(float (&f)[32], const float (&a)[32], int act, float keep, float alpha) {
  if (EXT && act >= SF_ACT_ELU) {
    act_ext_bwd32(f, a, act, keep, alpha);
  } else if (keep > 0.f && keep < 1.f) {
    const float ik = __fdividef(1.f, keep);
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] *= a[j] != 0.f ? act_bwd_from_out(a[j] * keep, act) * ik : 0.f;
  } else if (act == SF_ACT_RELU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] = a[j] > 0.f ? f[j] : 0.f;
  } else if (act == SF_ACT_SIGMOID) {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] *= a[j] * (1.f - a[j]);
  } else if (act == SF_ACT_TANH) {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] *= 1.f - a[j] * a[j];
  }
}

// One level of the column-sum transpose-reduce: lanes exchange half of their W live partial sums with lane ^ W.  W is a
// template parameter so every index into `r` is a constant (an indexed access would put `r` in local memory).
template <int W>
__device__ __forceinline__ void colsum_step(float (&r)[32], int lane) {
  const bool upper = (lane & W) != 0;
#pragma unroll
  for (int j = 0; j < W; ++j) {
    // opaque copies: a select between two elements of `r` would also be compiled into an indexed local-memory access
    float lo, hi;
    asm("mov.b32 %0, %1;" : "=f"(lo) : "f"(r[j]));
    asm("mov.b32 %0, %1;" : "=f"(hi) : "f"(r[j + W]));
    const float send = upper ? lo : hi;
    const float keep = upper ? hi : lo;
    r[j] = keep + __shfl_xor_sync(0xffffffffu, send, W);
  }
}

// Epilogue feature sets.  EPI is an SfEpi value, or kEpiPair: the generic set without the loss heads (the cluster-pair
// kernel never runs a loss).  The generic sets test every feature at run time; a specialized variant compiles in only
// its own features, and sf_gemm_prepare selects it only when the features it leaves out are absent and the ones it
// keeps unconditionally (the bf16 / fp32 output, the aux operand) are present.
constexpr int kEpiPair = -1;
template <int EPI>
struct EpiFeatures {
  static constexpr bool kGeneric = EPI == SF_EPI_GENERIC || EPI == kEpiPair;
  static constexpr bool kAct = kGeneric || EPI == SF_EPI_FWD || EPI == SF_EPI_LOSS;
  static constexpr bool kLoss = EPI == SF_EPI_GENERIC || EPI == SF_EPI_LOSS;                  // softmax-CE / MSE heads
  // sigmoid-CE head: only in its own variant, which therefore also carries the transposed bf16 output and the fused
  // read-your-writes wait that otherwise only the generic kernel has (so the generic kernel stays as it was)
  static constexpr bool kSigmoidLoss = EPI == SF_EPI_SIGMOID_LOSS;
  // sparse softmax-CE head (one class index per row): likewise only in its own variant, with the same extras
  static constexpr bool kSparseLoss = EPI == SF_EPI_SPARSE_LOSS;
  static constexpr bool kOutT = kGeneric || EPI == SF_EPI_SIGMOID_LOSS || EPI == SF_EPI_SPARSE_LOSS;
  static constexpr bool kRyw = kGeneric || EPI == SF_EPI_SIGMOID_LOSS || EPI == SF_EPI_SPARSE_LOSS;
  static constexpr bool kAux = kGeneric || EPI == SF_EPI_DGRAD;
  static constexpr bool kColsum = kGeneric || EPI == SF_EPI_LOSS || EPI == SF_EPI_SIGMOID_LOSS || EPI == SF_EPI_SPARSE_LOSS ||
                                  EPI == SF_EPI_DGRAD;
  static constexpr bool kF32 = kGeneric || EPI == SF_EPI_WGRAD;
  static constexpr bool kBf16 = kGeneric || EPI == SF_EPI_FWD || EPI == SF_EPI_LOSS || EPI == SF_EPI_SIGMOID_LOSS ||
                                EPI == SF_EPI_SPARSE_LOSS || EPI == SF_EPI_DGRAD;
  // the thread's act'(aux) chunk / label row / class index are fetched before the main loop (epi_prefetch)
  static constexpr bool kPrefetch = EPI == SF_EPI_LOSS || EPI == SF_EPI_SIGMOID_LOSS || EPI == SF_EPI_SPARSE_LOSS || EPI == SF_EPI_DGRAD;
};

// One 32-column chunk of a thread's output row: everything between the accumulator (v, already in registers) and
// global memory.  `aux_pref` / `tgt_pref` are the act'(a) operand / label row of this chunk when the caller fetched
// them before the accumulator wait (nullptr: read here).  EXT: the extended activations (twin kernels only).
template <int EPI, bool EXT>
__device__ __forceinline__ void epi_chunk(const SfGemmEpilogue& ep, const uint32_t (&v)[32], const float* s_bias32, int row, bool row_ok,
                                          int col0, int M, int N, int lane, const uint4* aux_pref, const float* tgt_pref,
                                          unsigned long long* tq = nullptr) {
    using F = EpiFeatures<EPI>;
    float f[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] = __uint_as_float(v[j]) * ep.alpha + s_bias32[j];
    if (tq != nullptr) tq[0] = trace_now();
    if (F::kAct) act_fwd32<EXT>(f, ep.act, ep.act_alpha);
    if (tq != nullptr) tq[1] = trace_now();
    if (F::kGeneric && ep.drop_keep > 0.f && ep.drop_keep < 1.f) {
      // fused dropout: keep with probability drop_keep, scale the survivors by 1 / drop_keep
      const float inv_keep = __fdividef(1.f, ep.drop_keep);
      const uint32_t thr = static_cast<uint32_t>(fminf(ep.drop_keep * 4294967296.f, 4294967040.f));
      const uint32_t stepc = ep.drop_ctr != nullptr ? *ep.drop_ctr : 0u;
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        const uint4 rnd = philox4x32_10(make_uint4(static_cast<uint32_t>(row), static_cast<uint32_t>(col0 >> 2) + g, stepc, ep.drop_stream),
                                        make_uint2(ep.drop_seed, 0x5F3759DFu));
        f[4 * g + 0] = rnd.x < thr ? f[4 * g + 0] * inv_keep : 0.f;
        f[4 * g + 1] = rnd.y < thr ? f[4 * g + 1] * inv_keep : 0.f;
        f[4 * g + 2] = rnd.z < thr ? f[4 * g + 2] * inv_keep : 0.f;
        f[4 * g + 3] = rnd.w < thr ? f[4 * g + 3] * inv_keep : 0.f;
      }
    }
    if (tq != nullptr) tq[2] = trace_now();
    if (F::kLoss && ep.loss_mode == SF_LOSS_SOFTMAX_XENT) {
      // whole row lives in this thread (host guarantees N <= 32): softmax + CE + gradient in registers
      const float* yv = tgt_pref;                         // N <= 32: the single chunk was prefetched
      const int nvalid = row_ok ? (N - col0 < 32 ? N - col0 : 32) : 0;
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 32; ++j) mx = fmaxf(mx, j < nvalid ? f[j] : -INFINITY);
      float se = 0.f, ysum = 0.f, zy = 0.f;
      float ex[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const bool ok = j < nvalid;
        ex[j] = ok ? __expf(f[j] - mx) : 0.f;
        const float y = ok ? yv[j] : 0.f;
        se += ex[j];
        ysum += y;
        zy += ok ? y * f[j] : 0.f;
      }
      const float inv_b = __fdividef(1.f, static_cast<float>(M));
      float lrow = row_ok ? ((mx + __logf(se)) * ysum - zy) * inv_b : 0.f;
      const float inv_se = row_ok ? __fdividef(1.f, se) : 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) f[j] = j < nvalid ? (ex[j] * inv_se * ysum - yv[j]) * inv_b : 0.f;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) lrow += __shfl_xor_sync(0xffffffffu, lrow, o);
      if (lane == 0 && lrow != 0.f) atomicAdd(ep.loss, lrow);
    } else if (F::kLoss && ep.loss_mode == SF_LOSS_MSE) {
      const float scale = 2.f / (static_cast<float>(M) * static_cast<float>(N));
      const float* tp = ep.target + static_cast<size_t>(row_ok ? row : 0) * ep.ld_target + col0;
      float lrow = 0.f;
      float a_out[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        a_out[j] = f[j];
        if (row_ok && col0 + j < N) {
          const float d = f[j] - (tgt_pref != nullptr ? tgt_pref[j] : tp[j]);
          lrow += d * d;
          f[j] = d * scale;
        } else {
          f[j] = 0.f;
        }
      }
      act_bwd32<EXT>(f, a_out, ep.act, 0.f, ep.act_alpha);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) lrow += __shfl_xor_sync(0xffffffffu, lrow, o);
      if (lane == 0 && lrow != 0.f) atomicAdd(ep.loss, lrow * 0.5f * scale);
    } else if (F::kSigmoidLoss && ep.loss_mode == SF_LOSS_SIGMOID_XENT) {
      // f holds raw logits (the host rejects an activation); the caller fetched the chunk's labels
      const float scale = __fdividef(1.f, static_cast<float>(M) * static_cast<float>(N));
      float lrow = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        float g = 0.f;
        if (row_ok && col0 + j < N) lrow += sigmoid_xent_elem(f[j], tgt_pref[j], g);
        f[j] = g * scale;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) lrow += __shfl_xor_sync(0xffffffffu, lrow, o);
      if (lane == 0 && lrow != 0.f) atomicAdd(ep.loss, lrow * scale);
    } else if (F::kSparseLoss && ep.loss_mode == SF_LOSS_SPARSE_SOFTMAX_XENT) {
      // whole row in this thread (N <= 32, raw logits); tgt_pref[0] is the row's class index, truncated toward zero like
      // TF's Cast.  It is only compared with column indices, so a label outside [0, N) reads nothing out of bounds.
      const int label = static_cast<int>(tgt_pref[0]);
      const int nvalid = row_ok ? (N - col0 < 32 ? N - col0 : 32) : 0;
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 32; ++j) mx = fmaxf(mx, j < nvalid ? f[j] : -INFINITY);
      float se = 0.f, zl = 0.f;
      float ex[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const bool ok = j < nvalid;
        ex[j] = ok ? __expf(f[j] - mx) : 0.f;
        se += ex[j];
        zl += ok && col0 + j == label ? f[j] : 0.f;
      }
      const float inv_b = __fdividef(1.f, static_cast<float>(M));
      float lrow = row_ok ? (mx + __logf(se) - zl) * inv_b : 0.f;
      const float inv_se = row_ok ? __fdividef(1.f, se) : 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) f[j] = j < nvalid ? (ex[j] * inv_se - (col0 + j == label ? 1.f : 0.f)) * inv_b : 0.f;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) lrow += __shfl_xor_sync(0xffffffffu, lrow, o);
      if (lane == 0 && lrow != 0.f) atomicAdd(ep.loss, lrow);
    }
    if (tq != nullptr) tq[3] = trace_now();
    if (F::kAux && (!F::kGeneric || ep.aux != nullptr) && row_ok) {
      const __nv_bfloat16* ap = ep.aux + static_cast<size_t>(row) * ep.ld_aux + col0;
      float a32[32];
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        uint4 q = make_uint4(0u, 0u, 0u, 0u);
        if (col0 + g * 8 < ep.ld_aux) q = (aux_pref != nullptr) ? aux_pref[g] : *reinterpret_cast<const uint4*>(ap + g * 8);
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 a2 = __bfloat1622float2(h[t]);
          a32[g * 8 + 2 * t] = a2.x;
          a32[g * 8 + 2 * t + 1] = a2.y;
        }
      }
      act_bwd32<EXT>(f, a32, ep.aux_act, F::kGeneric ? ep.aux_keep : 0.f, ep.aux_act_alpha);
    }
    if (tq != nullptr) tq[4] = trace_now();
    // padded columns / rows contribute exact zeros everywhere below
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (col0 + j >= N || !row_ok) f[j] = 0.f;

    if (F::kColsum && ep.colsum != nullptr) {
      // transpose-reduce over the 32 rows held by this warp: 31 shuffles, lane j ends up with
      // the sum of column col0 + j.
      float r[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) r[j] = f[j];
      colsum_step<16>(r, lane);
      colsum_step<8>(r, lane);
      colsum_step<4>(r, lane);
      colsum_step<2>(r, lane);
      colsum_step<1>(r, lane);
      // after the butterfly lane l holds column bitrev-free index: position is l itself
      if (col0 + lane < N) atomicAdd(ep.colsum + col0 + lane, r[0]);
    }

    if (tq != nullptr) tq[5] = trace_now();          // tracer: math done, stores follow
    if (F::kF32 && (!F::kGeneric || ep.out_f32 != nullptr || ep.route != nullptr) && row_ok) {
      float* op;
      if (F::kGeneric && ep.route != nullptr) {
        // push fused into the wgrad epilogue: this 32-column chunk lies inside ONE 32 x 64 push tile; its gradient goes
        // straight into this worker's mailbox on the GPU that owns the tile (NVLink peer stores / reds)
        const int tile = ep.route_tile0 + (row >> 5) * ep.route_tiles_c + (col0 >> 6);
        int owner = 0;
#pragma unroll
        for (int r = 1; r < SF_MAX_SHARDS; ++r) owner += (r < ep.route->n_shards && tile >= ep.route->bounds[r]) ? 1 : 0;
        op = ep.route->mailbox[owner] + ep.route_off + static_cast<size_t>(row) * ep.ld_f32 + col0;
      } else {
        op = ep.out_f32 + static_cast<size_t>(row) * ep.ld_f32 + col0;
      }
      if (ep.accumulate) {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (col0 + j < N) atomicAdd(op + j, f[j]);
      } else if ((ep.ld_f32 & 3) == 0 && col0 + 32 <= N &&
                 (reinterpret_cast<uintptr_t>(op) & 15) == 0) {
#pragma unroll
        for (int g = 0; g < 8; ++g)
          *reinterpret_cast<float4*>(op + 4 * g) =
              make_float4(f[4 * g], f[4 * g + 1], f[4 * g + 2], f[4 * g + 3]);
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (col0 + j < N) op[j] = f[j];
      }
    }
    if (tq != nullptr) tq[6] = trace_now();
    if (F::kBf16 && (!F::kGeneric || ep.out_bf16 != nullptr) && row_ok) {
      __nv_bfloat16* op = ep.out_bf16 + static_cast<size_t>(row) * ep.ld_bf16 + col0;
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        if (col0 + g * 8 < ep.ld_bf16) {
          uint4 q;
          q.x = pack_bf16x2(f[g * 8 + 0], f[g * 8 + 1]);
          q.y = pack_bf16x2(f[g * 8 + 2], f[g * 8 + 3]);
          q.z = pack_bf16x2(f[g * 8 + 4], f[g * 8 + 5]);
          q.w = pack_bf16x2(f[g * 8 + 6], f[g * 8 + 7]);
          *reinterpret_cast<uint4*>(op + g * 8) = q;
        }
      }
    }
    if (tq != nullptr) tq[7] = trace_now();
    if (F::kOutT && ep.outT_bf16 != nullptr && row_ok) {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (col0 + j < N)
          ep.outT_bf16[static_cast<size_t>(col0 + j) * ep.ld_t + row] = __float2bfloat16(f[j]);
    }
}

template <int BN>
struct GemmSmem {
  // ~200 KB of operand ring per CTA: small-N tiles are latency bound, so they get the deepest ring
  // (all 13 k-blocks of the flagship's 784-wide layer are in flight at once)
  static constexpr int kStages = (BN >= 256) ? 4 : (BN >= 128) ? 6 : (BN >= 64) ? 8 : 10;
  static constexpr int kABytes = kBM * kBK * 2;
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  // the epilogue stages the fp32 accumulator tile in the (then idle) ring: pitch BN + 1 floats, so the 32 lanes of a warp
  // reading 32 consecutive rows of one column hit 32 different banks
  static constexpr int kStgPitch = BN + 1;
  static_assert(kBM * kStgPitch * 4 <= kStages * kStageBytes, "accumulator staging must fit the operand ring");
  // + barriers (full, empty per stage) + bias tile (BN floats) + 1024 alignment slack
  static constexpr int kBarBytes = 256;
  static constexpr int kBytes = kStages * kStageBytes + kBarBytes + BN * 4 + 1024;
};

// Main loop of one consumer warpgroup: rows 64 * wg .. + 64 of the 128-row tile, all BN columns, over the k-blocks
// [it, it + num_kb) of the stage ring.  One wgmma batch stays in flight; a stage is released (one arrive per warpgroup,
// plus one on the same barrier of CTA `peer` when the stage is filled by cluster multicast) once the MMAs reading it
// have retired.
template <int BN, bool MN, int kStages, int kStageBytes, int kABytes>
__device__ __forceinline__ void mma_mainloop(float (&acc)[BN / 2], uint8_t* stage_base, uint64_t* full_bar, uint64_t* empty_bar,
                                             uint32_t it, int num_kb, int wg, bool signal, uint32_t code, int peer = -1) {
#pragma unroll
  for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
  int prev = -1;
  for (int i = 0; i < num_kb; ++i) {
    const uint32_t gi = it + static_cast<uint32_t>(i);
    const int s = static_cast<int>(gi % kStages);
    mbar_wait(&full_bar[s], (gi / kStages) & 1, code + s);
    const uint32_t a_addr = smem_u32(stage_base + s * kStageBytes) + wg * 8192;   // 64 rows (K-major) / one 64-row atom (MN-major)
    const uint32_t b_addr = smem_u32(stage_base + s * kStageBytes) + kABytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBK / kWgmmaK; ++k) {
      if constexpr (MN) {
        // 16 K rows of 128 B per MMA: +2 KB; the next 64 MN elements are one 8 KB atom away
        wgmma_bf16<BN, 1, 1>(acc, wgmma_desc_sw128(a_addr + k * 2048, 8192), wgmma_desc_sw128(b_addr + k * 2048, 8192), 1u);
      } else {
        // 16 elements (32 B) along K inside the swizzle atom
        wgmma_bf16<BN, 0, 0>(acc, wgmma_desc_sw128(a_addr + k * 32, 16), wgmma_desc_sw128(b_addr + k * 32, 16), 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && signal) {
      mbar_arrive(&empty_bar[prev]);
      if (peer >= 0) mbar_arrive_cluster(&empty_bar[prev], static_cast<uint32_t>(peer));
    }
    prev = s;
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
  if (prev >= 0 && signal) {
    mbar_arrive(&empty_bar[prev]);
    if (peer >= 0) mbar_arrive_cluster(&empty_bar[prev], static_cast<uint32_t>(peer));
  }
}

// consumer thread ct (0..255) writes its accumulator fragment into the staged tile stg[128][BN + 1]
template <int BN>
__device__ __forceinline__ void stage_acc(float* stg, const float (&acc)[BN / 2], int ct) {
  const int r0 = 64 * (ct >> 7) + 16 * ((ct >> 5) & 3) + ((ct & 31) >> 2);
  const int c0 = 2 * (ct & 3);
#pragma unroll
  for (int j = 0; j < BN / 2; ++j) stg[(r0 + 8 * ((j >> 1) & 1)) * (BN + 1) + 8 * (j >> 2) + c0 + (j & 1)] = acc[j];
}

// The act'(aux) chunk (DGRAD), label row (LOSS) or class index (SPARSE_LOSS, into tgt[0]) that consumer thread ct's
// epilogue reads, fetched before the main loop
// so that the load's latency hides under it.  Earlier launches wrote both, and everything upstream of this grid is
// complete once pdl_wait has returned.  BN <= 64: a thread owns at most one chunk (c = q / 4, see epilogue_tile).
template <int BN, int EPI>
__device__ __forceinline__ void epi_prefetch(const SfGemmEpilogue& ep, uint4 (&aux)[4], float (&tgt)[32], int m0, int n0, int M, int N,
                                             int ct) {
  static_assert(BN <= 64, "one 32-column chunk per consumer thread");
  const int q = ct >> 5, lane = ct & 31;
  const int row = m0 + (q & 3) * 32 + lane;
  const int col0 = n0 + (q >> 2) * 32;
  const bool live = row < M && (q >> 2) < BN / 32 && col0 < ep.n_store_limit;
  if constexpr (EPI == SF_EPI_DGRAD) {
    const __nv_bfloat16* ap = ep.aux + static_cast<size_t>(live ? row : 0) * ep.ld_aux + col0;
#pragma unroll
    for (int g = 0; g < 4; ++g)
      aux[g] = (live && col0 + g * 8 < ep.ld_aux) ? *reinterpret_cast<const uint4*>(ap + g * 8) : make_uint4(0u, 0u, 0u, 0u);
  } else if constexpr (EPI == SF_EPI_SPARSE_LOSS) {
    tgt[0] = live ? ep.target[static_cast<size_t>(row) * ep.ld_target] : 0.f;     // the row's class index
  } else {
    const float* tp = ep.target + static_cast<size_t>(live ? row : 0) * ep.ld_target + col0;
#pragma unroll
    for (int j = 0; j < 32; ++j) tgt[j] = (live && col0 + j < N) ? tp[j] : 0.f;
  }
}

// Epilogue of one 128 x BN tile from the staged accumulator, by the 256 consumer threads: warp q owns rows
// 32 * (q % 4) .. + 32 (one row per lane) and every other 32-column chunk starting at chunk q / 4.  aux_pref / tgt_pref:
// the thread's chunk fetched by epi_prefetch (variants with EpiFeatures::kPrefetch only).
template <int BN, int EPI, bool EXT>
__device__ __forceinline__ void epilogue_tile(const SfGemmEpilogue& ep, const float* stg, const float* s_bias, int m0, int n0, int M,
                                              int N, int ct, const uint4* aux_pref = nullptr, const float* tgt_pref = nullptr) {
  using F = EpiFeatures<EPI>;
  const int q = ct >> 5, lane = ct & 31;
  const int r = (q & 3) * 32 + lane;
  const int row = m0 + r;
  const bool row_ok = row < M;
  const float* srow = stg + r * (BN + 1);
#pragma unroll 1
  for (int c = q >> 2; c < BN / 32; c += 2) {
    const int col0 = n0 + c * 32;
    if (col0 >= ep.n_store_limit) break;   // whole chunk outside every output pitch
    uint32_t v[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = __float_as_uint(srow[c * 32 + j]);
    if constexpr (F::kPrefetch) {
      epi_chunk<EPI, EXT>(ep, v, s_bias + c * 32, row, row_ok, col0, M, N, lane, aux_pref, tgt_pref);
    } else {
      float tgt[32];
      if (F::kLoss && ep.loss_mode != SF_LOSS_NONE) {
        const float* tp = ep.target + static_cast<size_t>(row_ok ? row : 0) * ep.ld_target + col0;
#pragma unroll
        for (int j = 0; j < 32; ++j) tgt[j] = (row_ok && col0 + j < N) ? tp[j] : 0.f;
      }
      epi_chunk<EPI, EXT>(ep, v, s_bias + c * 32, row, row_ok, col0, M, N, lane, nullptr, F::kLoss ? tgt : nullptr);
    }
  }
}

// Thread roles (384 threads): warp 0 lane 0 is the TMA producer, warps 1-3 load the bias tile, warpgroups 1 and 2 each
// run the wgmma main loop for 64 rows of the tile and then, together, the epilogue.
// MN: both operands MN-major (D = a^T . b with a [K, M], b [K, N] row-major): the stage buffers have the same size, but a
// stage is filled with {64 MN elements, 64 K rows} boxes and described to the tensor core as MN-major.
// EPI: epilogue feature set (SfEpi); only the generic kernel handles the fused read-your-writes wait.  EXT: the extended
// activations are compiled in (the twin kernels below).
template <int BN, bool MN, int EPI, bool EXT = false>
__device__ __forceinline__ void gemm_cta(const CUtensorMap& tmA, const CUtensorMap& tmB, const SfGemmEpilogue& ep, int M, int N,
                                         int K, int kblocks_per_split) {
  static_assert(!MN || BN % 64 == 0, "MN-major B needs whole 64-element swizzle atoms");
  using F = EpiFeatures<EPI>;
  using S = GemmSmem<BN>;
  extern __shared__ uint8_t smem_raw[];
  // 128B swizzle needs 1024-byte aligned stage bases
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stage_base = smem;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::kStages * S::kStageBytes);
  uint64_t* empty_bar = full_bar + S::kStages;
  float* s_bias = reinterpret_cast<float*>(smem + S::kStages * S::kStageBytes + S::kBarBytes);

  TraceScope trace;
  // When a successor may launch (PDL trigger): a GEMM that carries the fused read-your-writes wait never triggers (its
  // successors launch when it completes) - they must not sit on SMs that the shard applier whose acknowledgement it
  // waits for needs for its own CTAs.  A grid of several waves triggers at entry: its successor's CTAs only get SMs as
  // this grid drains.  A one-wave grid triggers after its main loop, see there.
  if ((!F::kRyw || ep.ryw == nullptr) && !ep.one_wave) pdl_launch_dependents();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * BN;
  const int m0 = blockIdx.y * kBM;
  const int total_kb = (K + kBK - 1) / kBK;
  const int kb_begin = blockIdx.z * kblocks_per_split;
  int kb_end = kb_begin + kblocks_per_split;
  if (kb_end > total_kb) kb_end = total_kb;
  const int num_kb = kb_end - kb_begin;   // host guarantees >= 1

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < S::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);        // one arrive per consumer warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();
  pdl_wait();      // everything above overlapped the previous kernel; global memory is touched below
  trace.mark();

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      if (F::kRyw && ep.ryw != nullptr) {
        // pull fused into this GEMM: read-your-writes wait before the first weight tile is fetched (local spin)
        const SfRyw& w = *ep.ryw;
        const uint32_t posted = *w.my_posted;
        const unsigned long long t0 = sf_globaltimer();
        for (int r = 0; r < w.n_shards; ++r) {
          const uint32_t want = posted * static_cast<uint32_t>(w.ack_grid[r] ? w.ack_grid[r] : 1);
          while (static_cast<int32_t>(ld_relaxed_sys(w.applied + r * 16) - want) < 0) {
            if (sf_globaltimer() - t0 > 20000000000ull) sf_fail(0x405);
          }
        }
        if (w.stats != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
          const unsigned long long t1 = sf_globaltimer(), t_post = w.stats[0];
          if (t_post != 0 && t0 > t_post) {
            w.stats[8] += t0 - t_post;
            w.stats[9] += t1 - t0;
            w.stats[11] += 1ull;
          }
        }
      }
      // weights (B) are re-read by every M tile: keep them in L2; activations stream through.
      const uint64_t hintA = ep.a_evict_first ? kEvictFirst : kEvictNormal;
      const uint64_t hintB = kEvictLast;
      for (int i = 0; i < num_kb; ++i) {
        const int s = i % S::kStages;
        const uint32_t ph = (i / S::kStages) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1, 0x100 + s);
        uint8_t* a_dst = stage_base + s * S::kStageBytes;
        uint8_t* b_dst = a_dst + S::kABytes;
        mbar_expect_tx(&full_bar[s], S::kStageBytes);
        const int kc = (kb_begin + i) * kBK;
        if constexpr (MN) {
#pragma unroll
          for (int h = 0; h < kBM / 64; ++h) tma_load_2d(a_dst + h * 8192, &tmA, &full_bar[s], m0 + h * 64, kc, hintA);
#pragma unroll
          for (int h = 0; h < BN / 64; ++h) tma_load_2d(b_dst + h * 8192, &tmB, &full_bar[s], n0 + h * 64, kc, hintB);
        } else {
          tma_load_2d(a_dst, &tmA, &full_bar[s], kc, m0, hintA);
          tma_load_2d(b_dst, &tmB, &full_bar[s], kc, n0, hintB);
        }
      }
    }
  } else if (warp < 4) {
    // ===================== bias tile, loaded while the main loop runs =====================
    const bool is_split0 = (blockIdx.z == 0);
    for (int j = threadIdx.x - 32; j < BN; j += 96)
      s_bias[j] = (ep.bias != nullptr && is_split0 && n0 + j < N) ? ep.bias[n0 + j] : 0.f;
    asm volatile("bar.arrive 2, 352;" ::: "memory");
  } else {
    // ===================== wgmma main loop + epilogue =====================
    const int ct = threadIdx.x - 128;
    uint4 aux_pref[4];
    float tgt_pref[32];
    if constexpr (F::kPrefetch) epi_prefetch<BN, EPI>(ep, aux_pref, tgt_pref, m0, n0, M, N, ct);
    float acc[BN / 2];
    mma_mainloop<BN, MN, S::kStages, S::kStageBytes, S::kABytes>(acc, stage_base, full_bar, empty_bar, 0, num_kb, ct >> 7,
                                                                 (ct & 127) == 0, 0x200);
    // One-wave grid: the successor launches once every CTA is past its main loop, so its launch and prologue overlap
    // this epilogue.  A trigger at entry would let a chain of small GEMMs pre-launch in a cascade, and those waiting
    // CTAs (one per SM at this register / shared-memory size, 149 for the push) hold SMs the GEMMs ahead of them need.
    if ((!F::kRyw || ep.ryw == nullptr) && ep.one_wave) pdl_launch_dependents();
    // every stage has been consumed by both warpgroups: the ring holds the staged accumulator tile from here on
    float* stg = reinterpret_cast<float*>(stage_base);
    asm volatile("bar.sync 1, 256;" ::: "memory");
    stage_acc<BN>(stg, acc, ct);
    asm volatile("bar.sync 1, 256;" ::: "memory");
    asm volatile("bar.sync 2, 352;" ::: "memory");      // bias tile in shared memory
    if constexpr (F::kPrefetch) {
      epilogue_tile<BN, EPI, EXT>(ep, stg, s_bias, m0, n0, M, N, ct, aux_pref, tgt_pref);
    } else {
      epilogue_tile<BN, EPI, EXT>(ep, stg, s_bias, m0, n0, M, N, ct);
    }
  }
  trace.end(KID_GEMM);
}

// The generic kernel: every epilogue feature, each behind a runtime test.
template <int BN, bool MN = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
sf_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const SfGemmEpilogue ep, int M, int N, int K, int kblocks_per_split) {
  gemm_cta<BN, MN, SF_EPI_GENERIC>(tmA, tmB, ep, M, N, K, kblocks_per_split);
}

// A specialized epilogue variant (EPI != SF_EPI_GENERIC): a fraction of the generic kernel's code, which matters because
// the epilogue runs once per launch on a cold instruction cache.
template <int BN, bool MN, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
sf_gemm_epi_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const SfGemmEpilogue ep, int M, int N, int K, int kblocks_per_split) {
  static_assert(EPI != SF_EPI_GENERIC, "the generic epilogue is sf_gemm_kernel");
  gemm_cta<BN, MN, EPI>(tmA, tmB, ep, M, N, K, kblocks_per_split);
}

// The sigmoid cross-entropy head (SF_EPI_SIGMOID_LOSS, K-major) runs only here: as a runtime branch of the LOSS variant
// it raised that variant's register count, and in the generic kernel it added a quarter to the code every generic GEMM
// of the training step fetches.  It carries what a loss GEMM may need beyond the LOSS variant: the transposed dz of the
// K-major weight-gradient path and the read-your-writes wait of a network whose only dense layer is the loss layer.
template <int BN>
__global__ void __launch_bounds__(kGemmThreads, 1)
sf_gemm_sigmoid_loss_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                            const SfGemmEpilogue ep, int M, int N, int K, int kblocks_per_split) {
  gemm_cta<BN, false, SF_EPI_SIGMOID_LOSS>(tmA, tmB, ep, M, N, K, kblocks_per_split);
}

// The sparse softmax cross-entropy head (SF_EPI_SPARSE_LOSS, K-major, BN 32: the row fits one chunk) runs only here, so
// that the LOSS variant and the generic kernel keep their code; it carries the same extras as the sigmoid kernel.
__global__ void __launch_bounds__(kGemmThreads, 1)
sf_gemm_sparse_loss_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                           const SfGemmEpilogue ep, int M, int N, int K, int kblocks_per_split) {
  gemm_cta<32, false, SF_EPI_SPARSE_LOSS>(tmA, tmB, ep, M, N, K, kblocks_per_split);
}

// Twins of the generic kernel (K-major) and of the FWD / LOSS / DGRAD variants that also carry the extended activations
// (SfAct 4-9): their code would otherwise sit in every ReLU / sigmoid / tanh GEMM's epilogue, which is instruction-fetch
// bound.  sf_gemm_launch picks a twin exactly when ep.act or ep.aux_act is one of them.
template <int BN>
__global__ void __launch_bounds__(kGemmThreads, 1)
sf_gemm_ext_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const SfGemmEpilogue ep, int M, int N, int K, int kblocks_per_split) {
  gemm_cta<BN, false, SF_EPI_GENERIC, true>(tmA, tmB, ep, M, N, K, kblocks_per_split);
}
template <int BN, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
sf_gemm_epi_ext_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const SfGemmEpilogue ep, int M, int N, int K, int kblocks_per_split) {
  static_assert(EPI == SF_EPI_FWD || EPI == SF_EPI_LOSS || EPI == SF_EPI_DGRAD, "only these variants apply an activation");
  gemm_cta<BN, false, EPI, true>(tmA, tmB, ep, M, N, K, kblocks_per_split);
}

// ---------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

}  // namespace sf

extern "C" int sf_make_tmap_bf16_kmajor(CUtensorMap* out, const void* base, uint64_t rows,
                                        uint64_t cols, uint64_t ld_elems, uint32_t box_rows) {
  auto fn = sf::get_encode();
  if (!fn) return -1;
  cuuint64_t dims[2] = {cols, rows};                 // innermost first
  cuuint64_t strides[1] = {ld_elems * 2};            // bytes, dim 1
  cuuint32_t box[2] = {static_cast<cuuint32_t>(sf::kBK), box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : static_cast<int>(r);
}

// SMs of the current device (132 on an H100 SXM when no device is visible, e.g. while a plan is prepared on a CPU host)
extern "C" int sf_num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0, v = 0;
    n = (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0)
            ? v : 132;
  }
  return n;
}

extern "C" int sf_gemm_pick_bn(int M, int N) {
  // Small problems are latency bound: prefer more CTAs (smaller BN) until the grid covers every
  // SM; big problems want the widest tile for operand reuse.
  const int m_tiles = (M + sf::kBM - 1) / sf::kBM;
  const int sms = sf_num_sms();
  const int cands[4] = {256, 128, 64, 32};
  for (int i = 0; i < 4; ++i) {
    const int bn = cands[i];
    if (bn > 32 && bn / 2 >= N) continue;              // tile mostly padding
    const int n_tiles = (N + bn - 1) / bn;
    if (m_tiles * n_tiles >= sms || bn == 32) return bn;
  }
  return 32;
}

// The specialized epilogue variant that computes exactly what the generic kernel would for this GEMM, or SF_EPI_GENERIC.
// Variants exist only at the tile shapes the dense training plans use: K-major BN 32 / 64, MN-major (WGRAD) BN 64 / 128.
static int pick_epi(const SfGemm* g) {
  const SfGemmEpilogue& e = g->ep;
  const bool dropout = e.drop_keep > 0.f && e.drop_keep < 1.f;
  const bool aux_dropout = e.aux_keep > 0.f && e.aux_keep < 1.f;
  if (e.loss_mode == SF_LOSS_SIGMOID_XENT) {
    // the sigmoid head exists only in its own variant: K-major, BN 32 / 64, raw logits, bf16 dz (+ transpose)
    const bool ok = !g->pair && !g->mn_major && !dropout && e.route == nullptr && e.aux == nullptr && e.out_f32 == nullptr &&
                    e.out_bf16 != nullptr && e.act == SF_ACT_NONE && (g->bn == 32 || g->bn == 64);
    return ok ? SF_EPI_SIGMOID_LOSS : SF_EPI_GENERIC;
  }
  if (e.loss_mode == SF_LOSS_SPARSE_SOFTMAX_XENT) {
    // likewise the sparse softmax head: K-major, BN 32, raw logits, bf16 dz (+ transpose)
    const bool ok = !g->pair && !g->mn_major && !dropout && e.route == nullptr && e.aux == nullptr && e.out_f32 == nullptr &&
                    e.out_bf16 != nullptr && e.act == SF_ACT_NONE && g->bn == 32;
    return ok ? SF_EPI_SPARSE_LOSS : SF_EPI_GENERIC;
  }
  if (g->pair || dropout || e.route != nullptr || e.ryw != nullptr || e.outT_bf16 != nullptr) return SF_EPI_GENERIC;
  if (g->mn_major) {
    const bool wgrad = (g->bn == 64 || g->bn == 128) && e.out_f32 != nullptr && e.out_bf16 == nullptr && e.aux == nullptr &&
                       e.colsum == nullptr && e.act == SF_ACT_NONE && e.loss_mode == SF_LOSS_NONE;
    return wgrad ? SF_EPI_WGRAD : SF_EPI_GENERIC;
  }
  if ((g->bn != 32 && g->bn != 64) || e.out_bf16 == nullptr || e.out_f32 != nullptr) return SF_EPI_GENERIC;
  if (e.loss_mode != SF_LOSS_NONE) return e.aux == nullptr ? SF_EPI_LOSS : SF_EPI_GENERIC;
  if (e.aux != nullptr) return (!aux_dropout && e.act == SF_ACT_NONE) ? SF_EPI_DGRAD : SF_EPI_GENERIC;
  return e.colsum == nullptr ? SF_EPI_FWD : SF_EPI_GENERIC;
}

// the epilogue applies (or differentiates) one of the extended activations: the GEMM runs on a twin kernel
static bool uses_ext_act(const SfGemmEpilogue& e) { return e.act >= SF_ACT_ELU || e.aux_act >= SF_ACT_ELU; }

extern "C" int sf_gemm_prepare(SfGemm* g) {
  if (g->M <= 0 || g->N <= 0 || g->K <= 0) return -2;
  if (g->ep.act < SF_ACT_NONE || g->ep.act > SF_ACT_RELU6 || g->ep.aux_act < SF_ACT_NONE || g->ep.aux_act > SF_ACT_RELU6) return -5;
  if (g->mn_major && uses_ext_act(g->ep)) return -7;     // no MN-major twin: the weight-gradient GEMMs apply no activation
  if (g->ep.loss_mode < SF_LOSS_NONE || g->ep.loss_mode > SF_LOSS_SPARSE_SOFTMAX_XENT) return -5;
  if (g->bn == 0) g->bn = sf_gemm_pick_bn(g->M, g->N);
  if (g->ep.loss_mode == SF_LOSS_SIGMOID_XENT && g->bn > 64) g->bn = 64;    // the widest tile of its variant
  if (g->ep.loss_mode == SF_LOSS_SOFTMAX_XENT || g->ep.loss_mode == SF_LOSS_SPARSE_SOFTMAX_XENT) {
    // the row must fit one epilogue chunk; settled before the B tensor map, whose box height is the tile width
    if (g->N > 32) return -5;
    g->bn = 32;
  }
  if (g->split_k <= 0) g->split_k = 1;
  // large, un-split problems go to the persistent cluster-pair kernel (gemm_pair_sm90.cu): 256 x 128 tiles per CTA pair.
  // A GEMM that carries the fused read-your-writes wait stays on the one-CTA kernel, the only one that implements it.
  {
    const long long pair_tiles = static_cast<long long>((g->M + 255) / 256) * ((g->N + sf::kPairBN - 1) / sf::kPairBN);
    const bool eligible = g->split_k == 1 && g->ep.loss_mode == SF_LOSS_NONE && g->ep.ryw == nullptr && g->M >= 256 && g->N >= 256;
    const char* env = getenv("SPARKFLOW_GEMM_PAIR");
    int want = g->pair;
    if (env != nullptr && want < 0) want = atoi(env);
    if (want < 0) want = (g->bn == 256 && pair_tiles >= sf_num_sms() / 2 && g->K >= 512) ? 1 : 0;
    g->pair = (want > 0 && eligible && !g->mn_major) ? 1 : 0;
    if (g->pair) g->bn = sf::kPairBN;
  }
  if (!g->pair && (g->M + sf::kBM - 1) / sf::kBM > 65535) return -2;     // the one-CTA grid puts M tiles on grid.y
  int rc;
  if (g->mn_major) {
    // a is [K, lda] (M contiguous), b is [K, ldb] (N contiguous): boxes of {64 MN elements, 64 K rows}
    if (g->pair || g->ep.loss_mode != SF_LOSS_NONE) return -7;
    if (g->bn < 64) g->bn = 64;
    if (g->bn > 128) g->bn = 128;
    rc = sf_make_tmap_bf16_kmajor(&g->tmA, g->a, g->K, g->M, g->lda, 64);
    if (rc) return rc;
    rc = sf_make_tmap_bf16_kmajor(&g->tmB, g->b, g->K, g->N, g->ldb, 64);
    if (rc) return rc;
  } else {
    rc = sf_make_tmap_bf16_kmajor(&g->tmA, g->a, g->M, g->K, g->lda, sf::kBM);
    if (rc) return rc;
    rc = sf_make_tmap_bf16_kmajor(&g->tmB, g->b, g->N, g->K, g->ldb, g->pair ? sf::kPairBN / 2 : g->bn);
    if (rc) return rc;
  }
  const int total_kb = (g->K + sf::kBK - 1) / sf::kBK;
  if (g->split_k > total_kb) g->split_k = total_kb;
  g->kblocks_per_split = (total_kb + g->split_k - 1) / g->split_k;
  g->split_k = (total_kb + g->kblocks_per_split - 1) / g->kblocks_per_split;
  if (g->split_k > 1) g->ep.accumulate = 1;
  // a loss head needs the finished logits: no K split
  if (g->ep.loss_mode != SF_LOSS_NONE && (g->split_k > 1 || !g->ep.target || !g->ep.loss)) return -5;
  // largest column any output can hold
  int lim = g->N;
  if (g->ep.out_bf16 && g->ep.ld_bf16 > lim) lim = g->ep.ld_bf16;
  g->ep.n_store_limit = lim;
  g->ep.one_wave = static_cast<long long>((g->N + g->bn - 1) / g->bn) * ((g->M + sf::kBM - 1) / sf::kBM) * g->split_k <= sf_num_sms();
  g->epi = g->epi == SF_EPI_GENERIC ? SF_EPI_GENERIC : pick_epi(g);
  if (g->ep.loss_mode == SF_LOSS_SIGMOID_XENT && g->epi != SF_EPI_SIGMOID_LOSS) return -5;
  if (g->ep.loss_mode == SF_LOSS_SPARSE_SOFTMAX_XENT && g->epi != SF_EPI_SPARSE_LOSS) return -5;
  return 0;
}

template <int BN, bool MN = false, int EPI = SF_EPI_GENERIC, bool EXT = false>
static cudaError_t launch_bn(const SfGemm* g, cudaStream_t st) {
  using S = sf::GemmSmem<BN>;
  auto kernel = [] {
    if constexpr (EXT && EPI == SF_EPI_GENERIC) return sf::sf_gemm_ext_kernel<BN>;
    else if constexpr (EXT) return sf::sf_gemm_epi_ext_kernel<BN, EPI>;
    else if constexpr (EPI == SF_EPI_GENERIC) return sf::sf_gemm_kernel<BN, MN>;
    else if constexpr (EPI == SF_EPI_SIGMOID_LOSS) return sf::sf_gemm_sigmoid_loss_kernel<BN>;
    else if constexpr (EPI == SF_EPI_SPARSE_LOSS) return sf::sf_gemm_sparse_loss_kernel;
    else return sf::sf_gemm_epi_kernel<BN, MN, EPI>;
  }();
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kBytes);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  dim3 grid((g->N + BN - 1) / BN, (g->M + sf::kBM - 1) / sf::kBM, g->split_k);
  return sf::launch(kernel, grid, dim3(sf::kGemmThreads), S::kBytes, st, g->tmA, g->tmB, g->ep,
                    g->M, g->N, g->K, g->kblocks_per_split);
}

// K-major epilogue variants exist at BN 32 and 64 (pick_epi)
template <int EPI, bool EXT = false>
static cudaError_t launch_kmajor_variant(const SfGemm* g, cudaStream_t st) {
  return g->bn == 32 ? launch_bn<32, false, EPI, EXT>(g, st) : launch_bn<64, false, EPI, EXT>(g, st);
}

// the twins of the extended activations (K-major only, see sf_gemm_prepare)
static int launch_ext(const SfGemm* g, cudaStream_t st) {
  cudaError_t e;
  switch (g->epi) {
    case SF_EPI_GENERIC: break;
    case SF_EPI_FWD: return static_cast<int>(launch_kmajor_variant<SF_EPI_FWD, true>(g, st));
    case SF_EPI_LOSS: return static_cast<int>(launch_kmajor_variant<SF_EPI_LOSS, true>(g, st));
    case SF_EPI_DGRAD: return static_cast<int>(launch_kmajor_variant<SF_EPI_DGRAD, true>(g, st));
    default: return -3;
  }
  if (g->mn_major) return -3;
  switch (g->bn) {
    case 32: e = launch_bn<32, false, SF_EPI_GENERIC, true>(g, st); break;
    case 64: e = launch_bn<64, false, SF_EPI_GENERIC, true>(g, st); break;
    case 128: e = launch_bn<128, false, SF_EPI_GENERIC, true>(g, st); break;
    case 256: e = launch_bn<256, false, SF_EPI_GENERIC, true>(g, st); break;
    default: return -3;
  }
  return static_cast<int>(e);
}

extern "C" int sf_gemm_launch(const SfGemm* g, cudaStream_t st) {
  if (g->pair) return sf_gemm_pair_launch(g, st);
  if (uses_ext_act(g->ep)) return launch_ext(g, st);
  cudaError_t e;
  switch (g->epi) {
    case SF_EPI_GENERIC: break;
    case SF_EPI_FWD: return static_cast<int>(launch_kmajor_variant<SF_EPI_FWD>(g, st));
    case SF_EPI_LOSS: return static_cast<int>(launch_kmajor_variant<SF_EPI_LOSS>(g, st));
    case SF_EPI_DGRAD: return static_cast<int>(launch_kmajor_variant<SF_EPI_DGRAD>(g, st));
    case SF_EPI_SIGMOID_LOSS: return static_cast<int>(launch_kmajor_variant<SF_EPI_SIGMOID_LOSS>(g, st));
    case SF_EPI_SPARSE_LOSS: return static_cast<int>(launch_bn<32, false, SF_EPI_SPARSE_LOSS>(g, st));
    case SF_EPI_WGRAD:
      e = g->bn == 64 ? launch_bn<64, true, SF_EPI_WGRAD>(g, st) : launch_bn<128, true, SF_EPI_WGRAD>(g, st);
      return static_cast<int>(e);
    default: return -3;
  }
  if (g->mn_major) {
    switch (g->bn) {
      case 64: e = launch_bn<64, true>(g, st); break;
      case 128: e = launch_bn<128, true>(g, st); break;
      default: return -3;
    }
    return static_cast<int>(e);
  }
  switch (g->bn) {
    case 32: e = launch_bn<32>(g, st); break;
    case 64: e = launch_bn<64>(g, st); break;
    case 128: e = launch_bn<128>(g, st); break;
    case 256: e = launch_bn<256>(g, st); break;
    default: return -3;
  }
  return static_cast<int>(e);
}

extern "C" void sf_set_pdl(int enabled) { sf::pdl_enabled() = enabled ? 1 : 0; }

// tracing: `buf` is a device buffer of `cap` 32-byte records (or nullptr to disable)
extern "C" int sf_trace_enable(void* buf, unsigned int cap) {
  sf::TraceRec* b = static_cast<sf::TraceRec*>(buf);
  unsigned int zero = 0;
  cudaError_t e = cudaMemcpyToSymbol(sf::g_trace_buf, &b, sizeof(b));
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(sf::g_trace_cap, &cap, sizeof(cap));
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(sf::g_trace_n, &zero, sizeof(zero));
  return static_cast<int>(e);
}
extern "C" unsigned int sf_trace_count() {
  unsigned int n = 0;
  cudaMemcpyFromSymbol(&n, sf::g_trace_n, sizeof(n));
  return n;
}

static unsigned int* g_err_host_ptr = nullptr;

// allocate the host-visible error word for the current device and point the device symbol at it
extern "C" int sf_init_error_channel() {
  if (g_err_host_ptr == nullptr) {
    void* raw = nullptr;
    cudaError_t e = cudaHostAlloc(&raw, sizeof(unsigned int), cudaHostAllocMapped | cudaHostAllocPortable);
    if (e != cudaSuccess) return static_cast<int>(e);
    g_err_host_ptr = static_cast<unsigned int*>(raw);
    *g_err_host_ptr = 0;
  }
  unsigned int* dptr = nullptr;
  cudaError_t e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&dptr), g_err_host_ptr, 0);
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(sf::g_sf_error_host, &dptr, sizeof(dptr));
  return static_cast<int>(e);
}
extern "C" unsigned int sf_read_host_error_code() { return g_err_host_ptr ? *g_err_host_ptr : 0u; }

extern "C" unsigned int sf_read_error_code() {
  unsigned int v = 0;
  cudaMemcpyFromSymbol(&v, sf::g_sf_error_code, sizeof(v));
  return v;
}
