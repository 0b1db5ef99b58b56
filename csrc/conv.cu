// Convolution building blocks for the compiled CNN plan (reference ops K3/K4 of SURVEY.md section 2.4:
// Conv2D + BiasAdd + Relu, MaxPool and their gradients; examples/cnn_example.py:10-22).
//
// Convolutions are lowered to the wgmma GEMM of gemm_sm90.cu:
//   forward   out[M, Cout]   = patches[M, K] . W^T[Cout, K]^T  (+bias, ReLU in the GEMM epilogue)
//   wgrad     dW[K, Cout]    = patches^T[K, M] . dz^T[Cout, M]^T      (split-K, atomic accumulate)
//   dgrad     dpatch[M, K]   = dz[M, Cout] . W[K, Cout]^T             -> col2im gather
// with M = batch * out_h * out_w and K = kh * kw * Cin in (kh, kw, cin) order, i.e. exactly the flattening
// of TensorFlow's HWIO filter layout.  The kernels here produce the K-major operands those GEMMs need:
// im2col writes patches AND patches^T; max-pool backward applies the ReLU derivative, scatters through
// the arg-max mask and writes dz, dz^T and the bias gradient in one pass.
#include "sm90_ptx.cuh"
#include "sf_api.h"

namespace sf {

// ------------------------------------------------------------------------------------------------
// im2col (NHWC, VALID, stride 1): out[m, k] = in[b, oh+kh, ow+kw, c];  32x32 tiles through smem so
// that the row-major store (along k) and the transposed store (along m) are both coalesced.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
im2col_kernel(const __nv_bfloat16* __restrict__ in, int n, int h, int w, int c, int kh, int kw,
              __nv_bfloat16* __restrict__ out, int ld_out, __nv_bfloat16* __restrict__ outT, int ld_t) {
  __shared__ __nv_bfloat16 tile[32][34];
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int oh = h - kh + 1, ow = w - kw + 1;
  const int M = n * oh * ow, K = kh * kw * c;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int k0 = blockIdx.y * 32, m0 = blockIdx.x * 32;      // M tiles on x: a 4096-row evaluation chunk has > 65535 of them
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty + 8 * i, k = k0 + tx;
    __nv_bfloat16 v = __float2bfloat16(0.f);
    if (m < M && k < K) {
      const int b = m / (oh * ow), r = m - b * (oh * ow);
      const int y = r / ow, x = r - y * ow;
      const int cc = k % c, t = k / c;
      const int dx = t % kw, dy = t / kw;
      v = in[((static_cast<size_t>(b) * h + (y + dy)) * w + (x + dx)) * c + cc];
    }
    tile[ty + 8 * i][tx] = v;
    if (out != nullptr && m < M && k < ld_out) out[static_cast<size_t>(m) * ld_out + k] = v;
  }
  if (outT != nullptr) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = k0 + ty + 8 * i, m = m0 + tx;
      if (k < K && m < M) outT[static_cast<size_t>(k) * ld_t + m] = tile[tx][ty + 8 * i];
    }
  }
  trace.end(KID_IM2COL);
}

// Fast path (C % 8 == 0, ld_out % 8 == 0, no transposed copy - the MN-major wgrad reads `out` itself): one 16-byte
// vector = 8 channels of one filter tap per thread; loads and stores are both contiguous along k.
__global__ void __launch_bounds__(256)
im2col_vec8_kernel(const uint4* __restrict__ in, int n, int h, int w, int c8, int kh, int kw, uint4* __restrict__ out, int ld8) {
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int oh = h - kh + 1, ow = w - kw + 1;
  const int M = n * oh * ow, K8 = kh * kw * c8;
  const long long total = static_cast<long long>(M) * ld8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int m = static_cast<int>(i / ld8), q = static_cast<int>(i - static_cast<long long>(m) * ld8);
    uint4 v = make_uint4(0u, 0u, 0u, 0u);                    // pad columns carry zeros
    if (q < K8) {
      const int tap = q / c8, cc = q - tap * c8;
      const int dy = tap / kw, dx = tap - dy * kw;
      const int b = m / (oh * ow), r = m - b * (oh * ow);
      const int y = r / ow, x = r - y * ow;
      v = in[(static_cast<size_t>(b * h + y + dy) * w + (x + dx)) * c8 + cc];
    }
    out[i] = v;
  }
  trace.end(KID_IM2COL);
}

__device__ __forceinline__ void acc_bf16x8(float (&acc)[8], const uint4& q) {
  const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const float2 f = __bfloat1622float2(h2[t]);
    acc[2 * t] += f.x;
    acc[2 * t + 1] += f.y;
  }
}

// col2im gather, 8 channels per thread (C % 8 == 0, ld_cols % 8 == 0)
__global__ void __launch_bounds__(256)
col2im_vec8_kernel(const uint4* __restrict__ dcols, int ld8, int n, int h, int w, int c8, int kh, int kw, uint4* __restrict__ din) {
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int oh = h - kh + 1, ow = w - kw + 1;
  const int total = n * h * w * c8;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int cc = i % c8;
    int t = i / c8;
    const int x = t % w;
    t /= w;
    const int y = t % h;
    const int b = t / h;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const int dy_lo = y - (oh - 1) > 0 ? y - (oh - 1) : 0, dy_hi = y < kh - 1 ? y : kh - 1;
    const int dx_lo = x - (ow - 1) > 0 ? x - (ow - 1) : 0, dx_hi = x < kw - 1 ? x : kw - 1;
    for (int dy = dy_lo; dy <= dy_hi; ++dy) {
      const uint4* row = dcols + (static_cast<size_t>(b * oh + (y - dy)) * ow + x) * ld8 + (dy * kw) * c8 + cc;
      for (int dx = dx_lo; dx <= dx_hi; ++dx) acc_bf16x8(acc, row[dx * c8 - static_cast<long long>(dx) * ld8]);
    }
    uint4 q;
    q.x = pack_bf16x2(acc[0], acc[1]);
    q.y = pack_bf16x2(acc[2], acc[3]);
    q.z = pack_bf16x2(acc[4], acc[5]);
    q.w = pack_bf16x2(acc[6], acc[7]);
    din[i] = q;
  }
  trace.end(KID_COL2IM);
}

// ------------------------------------------------------------------------------------------------
// col2im as a gather (no atomics): din[b, y, x, c] = sum_{dy,dx} dcols[(b, y-dy, x-dx), (dy*kw+dx)*C + c]
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
col2im_kernel(const __nv_bfloat16* __restrict__ dcols, int ld_cols, int n, int h, int w, int c, int kh, int kw,
              __nv_bfloat16* __restrict__ din) {
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int oh = h - kh + 1, ow = w - kw + 1;
  const size_t total = static_cast<size_t>(n) * h * w * c;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cc = static_cast<int>(i % c);
    size_t t = i / c;
    const int x = static_cast<int>(t % w);
    t /= w;
    const int y = static_cast<int>(t % h);
    const int b = static_cast<int>(t / h);
    float acc = 0.f;
    for (int dy = 0; dy < kh; ++dy) {
      const int yy = y - dy;
      if (yy < 0 || yy >= oh) continue;
      for (int dx = 0; dx < kw; ++dx) {
        const int xx = x - dx;
        if (xx < 0 || xx >= ow) continue;
        const size_t m = (static_cast<size_t>(b) * oh + yy) * ow + xx;
        acc += __bfloat162float(dcols[m * ld_cols + (dy * kw + dx) * c + cc]);
      }
    }
    din[i] = __float2bfloat16(acc);
  }
  trace.end(KID_COL2IM);
}

// ------------------------------------------------------------------------------------------------
// 2x2 / stride-2 max pool (VALID).  argmax stores the winner's position inside the window (0..3).
// Optional outT[(y*ow + x)*C + c][b] is the transposed flattened activation (K-major operand of the
// following dense layer's wgrad).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
maxpool_fwd_kernel(const __nv_bfloat16* __restrict__ in, int n, int h, int w, int c, __nv_bfloat16* __restrict__ out,
                   uint8_t* __restrict__ argmax, __nv_bfloat16* __restrict__ outT, int ld_t) {
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int oh = h / 2, ow = w / 2;
  const size_t total = static_cast<size_t>(n) * oh * ow * c;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cc = static_cast<int>(i % c);
    size_t t = i / c;
    const int x = static_cast<int>(t % ow);
    t /= ow;
    const int y = static_cast<int>(t % oh);
    const int b = static_cast<int>(t / oh);
    const __nv_bfloat16* p = in + ((static_cast<size_t>(b) * h + 2 * y) * w + 2 * x) * c + cc;
    float best = __bfloat162float(p[0]);
    int bi = 0;
    const float v1 = __bfloat162float(p[c]);
    const float v2 = __bfloat162float(p[static_cast<size_t>(w) * c]);
    const float v3 = __bfloat162float(p[static_cast<size_t>(w) * c + c]);
    if (v1 > best) { best = v1; bi = 1; }
    if (v2 > best) { best = v2; bi = 2; }
    if (v3 > best) { best = v3; bi = 3; }
    out[i] = __float2bfloat16(best);
    argmax[i] = static_cast<uint8_t>(bi);
    if (outT != nullptr) outT[static_cast<size_t>((y * ow + x) * c + cc) * ld_t + b] = __float2bfloat16(best);
  }
  trace.end(KID_POOL_FWD);
}

// ------------------------------------------------------------------------------------------------
// max-pool backward fused with the activation derivative of the conv output it pooled:
//   dz[b, y, x, c] = (argmax(window) == position) ? dout[window] * act'(a[b, y, x, c]) : 0
// written row-major [M, ld_dz] (dgrad A operand), transposed [C, ld_t] (wgrad B operand) and reduced
// over M into dbias[C].  One 32(m) x 32(c) tile per CTA.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float pool_dact(float a, int act) {
  switch (act) {
    case SF_ACT_RELU: return a > 0.f ? 1.f : 0.f;
    case SF_ACT_SIGMOID: return a * (1.f - a);
    case SF_ACT_TANH: return 1.f - a * a;
    default: return 1.f;
  }
}

__global__ void __launch_bounds__(256)
maxpool_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const uint8_t* __restrict__ argmax, int n, int h, int w, int c,
                   const __nv_bfloat16* __restrict__ act_out, int act, __nv_bfloat16* __restrict__ dz, int ld_dz,
                   __nv_bfloat16* __restrict__ dzT, int ld_t, float* __restrict__ dbias) {
  __shared__ __nv_bfloat16 tile[32][34];
  __shared__ float s_col[32];
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int oh = h / 2, ow = w / 2;
  const int M = n * h * w;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 32, m0 = blockIdx.y * 32;
  if (threadIdx.x < 32) s_col[threadIdx.x] = 0.f;
  __syncthreads();
  float cacc = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty + 8 * i, cc = c0 + tx;
    float g = 0.f;
    if (m < M && cc < c) {
      const int b = m / (h * w), r = m - b * (h * w);
      const int y = r / w, x = r - y * w;
      const int py = y >> 1, px = x >> 1;
      if (py < oh && px < ow) {
        const size_t o = ((static_cast<size_t>(b) * oh + py) * ow + px) * c + cc;
        if (argmax[o] == ((y & 1) * 2 + (x & 1)))
          g = __bfloat162float(dout[o]) * pool_dact(__bfloat162float(act_out[static_cast<size_t>(m) * c + cc]), act);
      }
    }
    const __nv_bfloat16 gb = __float2bfloat16(g);
    tile[ty + 8 * i][tx] = gb;
    cacc += g;
    if (dz != nullptr && m < M && cc < ld_dz) dz[static_cast<size_t>(m) * ld_dz + cc] = gb;
  }
  if (dbias != nullptr) atomicAdd(&s_col[tx], cacc);
  __syncthreads();
  if (dbias != nullptr && threadIdx.x < 32 && c0 + threadIdx.x < c && s_col[threadIdx.x] != 0.f)
    atomicAdd(dbias + c0 + threadIdx.x, s_col[threadIdx.x]);
  if (dzT != nullptr) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int cc = c0 + ty + 8 * i, m = m0 + tx;
      if (cc < c && m < M) dzT[static_cast<size_t>(cc) * ld_t + m] = tile[tx][ty + 8 * i];
    }
  }
  trace.end(KID_POOL_BWD);
}

}  // namespace sf

static inline int grid_1d(size_t total) {
  size_t b = (total + 255) / 256;
  if (b > sf_num_sms() * 16) b = sf_num_sms() * 16;
  return static_cast<int>(b < 1 ? 1 : b);
}

extern "C" int sf_im2col_nhwc(const __nv_bfloat16* in, int n, int h, int w, int c, int kh, int kw, __nv_bfloat16* out,
                              int ld_out, __nv_bfloat16* outT, int ld_t, cudaStream_t st) {
  const int M = n * (h - kh + 1) * (w - kw + 1), K = kh * kw * c;
  if (outT == nullptr && out != nullptr && (c & 7) == 0 && (ld_out & 7) == 0 && ld_out >= K && (reinterpret_cast<uintptr_t>(in) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(out) & 15) == 0) {
    const size_t total = static_cast<size_t>(M) * (ld_out / 8);
    return static_cast<int>(sf::launch(sf::im2col_vec8_kernel, dim3(grid_1d(total)), dim3(256), 0, st, reinterpret_cast<const uint4*>(in), n, h, w,
                                       c / 8, kh, kw, reinterpret_cast<uint4*>(out), ld_out / 8));
  }
  const int span_k = (out && ld_out > K) ? ld_out : K;
  dim3 grid((M + 31) / 32, (span_k + 31) / 32);
  return static_cast<int>(sf::launch(sf::im2col_kernel, grid, dim3(256), 0, st, in, n, h, w, c, kh, kw, out, ld_out, outT, ld_t));
}

extern "C" int sf_col2im_nhwc(const __nv_bfloat16* dcols, int ld_cols, int n, int h, int w, int c, int kh, int kw,
                              __nv_bfloat16* din, cudaStream_t st) {
  const size_t total = static_cast<size_t>(n) * h * w * c;
  if ((c & 7) == 0 && (ld_cols & 7) == 0 && total / 8 < (1u << 30) && (reinterpret_cast<uintptr_t>(dcols) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(din) & 15) == 0)
    return static_cast<int>(sf::launch(sf::col2im_vec8_kernel, dim3(grid_1d(total / 8)), dim3(256), 0, st, reinterpret_cast<const uint4*>(dcols),
                                       ld_cols / 8, n, h, w, c / 8, kh, kw, reinterpret_cast<uint4*>(din)));
  return static_cast<int>(sf::launch(sf::col2im_kernel, dim3(grid_1d(total)), dim3(256), 0, st, dcols, ld_cols, n, h, w, c, kh, kw, din));
}

extern "C" int sf_maxpool2_fwd(const __nv_bfloat16* in, int n, int h, int w, int c, __nv_bfloat16* out, uint8_t* argmax,
                               __nv_bfloat16* outT, int ld_t, cudaStream_t st) {
  const size_t total = static_cast<size_t>(n) * (h / 2) * (w / 2) * c;
  return static_cast<int>(sf::launch(sf::maxpool_fwd_kernel, dim3(grid_1d(total)), dim3(256), 0, st, in, n, h, w, c, out, argmax, outT, ld_t));
}

extern "C" int sf_maxpool2_bwd(const __nv_bfloat16* dout, const uint8_t* argmax, int n, int h, int w, int c,
                               const __nv_bfloat16* act_out, int act, __nv_bfloat16* dz, int ld_dz, __nv_bfloat16* dzT, int ld_t,
                               float* dbias, cudaStream_t st) {
  const int M = n * h * w;
  const int span_c = (dz && ld_dz > c) ? ld_dz : c;
  dim3 grid((span_c + 31) / 32, (M + 31) / 32);
  return static_cast<int>(sf::launch(sf::maxpool_bwd_kernel, grid, dim3(256), 0, st, dout, argmax, n, h, w, c, act_out, act, dz,
                                     ld_dz, dzT, ld_t, dbias));
}

namespace sf {

// ------------------------------------------------------------------------------------------------
// First convolution of a network, fused with its bias, activation and 2x2 max-pool - forward and weight gradient.
// (reference workload: examples/cnn_example.py:14-15: 5x5x1 -> 32, ReLU, max_pooling2d(2, 2).)
// With K = kh * kw * cin <= 64 the layer is a poor tensor-core GEMM (K = 25 padded to 64, 172,800 x 32 outputs in 1,350
// latency-bound 128-row tiles, plus an im2col matrix and a pooling pass through HBM: ~110 us of a 350 us step); as a
// direct CUDA-core kernel it is ~0.3 GFLOP that never leaves shared memory: one CTA per image holds the image and
// the filter bank on chip, every thread owns one output channel (lane = channel: filter reads are conflict free, pixel
// reads are warp broadcasts) and produces whole pooled pixels, so the un-pooled activation is never written at all.
// The backward kernel recomputes nothing: the gradient of a pooled pixel goes to the arg-max position if the pooled
// value passed the activation (ReLU: pooled > 0), and is correlated with the input patch there.
// ------------------------------------------------------------------------------------------------
constexpr int kConv1Threads = 256;
constexpr int kConv1MaxK = 64;

__device__ __forceinline__ float conv1_act(float v, int act) {
  switch (act) {
    case SF_ACT_RELU: return fmaxf(v, 0.f);
    case SF_ACT_SIGMOID: return 1.f / (1.f + __expf(-v));
    case SF_ACT_TANH: return tanhf(v);
    default: return v;
  }
}

// x [n, h, w, cin] bf16; wT [cout, ld_w] bf16 (row c = filter of channel c, k = (dy * kw + dx) * cin + ci); bias fp32 [cout]
// pooled [n, oh/2, ow/2, cout] bf16; argmax uint8 (position 0..3 of the winner inside its 2x2 window)
// KH / KW / CIN are compile-time (0 = runtime): with constant taps the filter lives in registers and the window loop unrolls.
template <int KH, int KW, int CIN>
__global__ void __launch_bounds__(kConv1Threads)
conv_first_fwd_kernel(const __nv_bfloat16* __restrict__ x, int n, int h, int w, int cin_rt, int kh_rt, int kw_rt, int cout,
                      const __nv_bfloat16* __restrict__ wT, int ld_w, const float* __restrict__ bias, int act,
                      __nv_bfloat16* __restrict__ pooled, uint8_t* __restrict__ argmax, int parts) {
  extern __shared__ float conv1_smem[];
  TraceScope trace;
  pdl_launch_dependents();
  const int kh = KH ? KH : kh_rt, kw = KW ? KW : kw_rt, cin = CIN ? CIN : cin_rt;
  const int K = kh * kw * cin;
  float* s_w = conv1_smem;                       // [K][cout]  (runtime-shape path only)
  float* s_x = conv1_smem + (KH ? 0 : K * cout); // [h * w * cin]
  const int tid = threadIdx.x;
  const int oh = h - kh + 1, ow = w - kw + 1, ph = oh / 2, pw = ow / 2;
  const int c = tid % cout, grp = tid / cout, n_grp = kConv1Threads / cout;
  pdl_wait();
  trace.mark();
  constexpr int KC = KH ? KH * KW * CIN : 1;
  float wr[KC];
  if constexpr (KH != 0) {
#pragma unroll
    for (int k = 0; k < KC; ++k) wr[k] = __bfloat162float(wT[static_cast<size_t>(c) * ld_w + k]);
  } else {
    for (int i = tid; i < K * cout; i += kConv1Threads) s_w[i] = __bfloat162float(wT[static_cast<size_t>(i % cout) * ld_w + i / cout]);
  }
  const float b = bias != nullptr ? bias[c] : 0.f;
  // `parts` CTAs share an image (each takes every parts-th pooled pixel group): more resident warps to hide latency
  for (int item = blockIdx.x; item < n * parts; item += gridDim.x) {
    const int img = item / parts, part = item - img * parts;
    __syncthreads();                               // previous image fully consumed (and s_w complete on the first pass)
    const __nv_bfloat16* xi = x + static_cast<size_t>(img) * h * w * cin;
    for (int i = tid; i < h * w * cin; i += kConv1Threads) s_x[i] = __bfloat162float(xi[i]);
    __syncthreads();
    for (int p = grp + part * n_grp; p < ph * pw; p += n_grp * parts) {
      const int py = p / pw, px = p - py * pw;
      float a00 = b, a01 = b, a10 = b, a11 = b;
      if constexpr (KH != 0) {
        // (KH + 1) x (KW + 1) input window of the 2x2 output quad, one row at a time, filter taps from registers
#pragma unroll
        for (int iy = 0; iy <= KH; ++iy) {
          float row[(KW + 1) * CIN];
          const float* rp = s_x + ((2 * py + iy) * w + 2 * px) * CIN;
#pragma unroll
          for (int j = 0; j < (KW + 1) * CIN; ++j) row[j] = rp[j];
#pragma unroll
          for (int dx = 0; dx < KW; ++dx)
#pragma unroll
            for (int ci = 0; ci < CIN; ++ci) {
              if (iy < KH) {                        // this input row is filter row iy of the upper outputs
                const float wv = wr[(iy * KW + dx) * CIN + ci];
                a00 = fmaf(wv, row[dx * CIN + ci], a00);
                a01 = fmaf(wv, row[(dx + 1) * CIN + ci], a01);
              }
              if (iy >= 1) {                        // ... and filter row iy - 1 of the lower outputs
                const float wv = wr[((iy - 1) * KW + dx) * CIN + ci];
                a10 = fmaf(wv, row[dx * CIN + ci], a10);
                a11 = fmaf(wv, row[(dx + 1) * CIN + ci], a11);
              }
            }
        }
      } else {
        for (int dy = 0; dy < kh; ++dy) {
          const float* r0 = s_x + ((2 * py + dy) * w + 2 * px) * cin;
          const float* r1 = r0 + w * cin;
          for (int dx = 0; dx < kw; ++dx) {
            for (int ci = 0; ci < cin; ++ci) {
              const float wv = s_w[((dy * kw + dx) * cin + ci) * cout + c];
              const int o = dx * cin + ci;
              a00 = fmaf(wv, r0[o], a00);
              a01 = fmaf(wv, r0[o + cin], a01);
              a10 = fmaf(wv, r1[o], a10);
              a11 = fmaf(wv, r1[o + cin], a11);
            }
          }
        }
      }
      a00 = conv1_act(a00, act); a01 = conv1_act(a01, act); a10 = conv1_act(a10, act); a11 = conv1_act(a11, act);
      float m = a00;
      int am = 0;
      if (a01 > m) { m = a01; am = 1; }
      if (a10 > m) { m = a10; am = 2; }
      if (a11 > m) { m = a11; am = 3; }
      const size_t o = (static_cast<size_t>(img) * ph * pw + p) * cout + c;
      pooled[o] = __float2bfloat16(m);
      argmax[o] = static_cast<uint8_t>(am);
    }
  }
  trace.end(KID_IM2COL);
}

// g_pool [n, ph, pw, cout] bf16 = dL/d(pooled); dW [K, cout] fp32 and db [cout] are ACCUMULATED with atomics
template <int KH, int KW, int CIN>
__global__ void __launch_bounds__(kConv1Threads)
conv_first_wgrad_kernel(const __nv_bfloat16* __restrict__ x, int n, int h, int w, int cin_rt, int kh_rt, int kw_rt, int cout,
                        const __nv_bfloat16* __restrict__ g_pool, const __nv_bfloat16* __restrict__ pooled,
                        const uint8_t* __restrict__ argmax, int act, float* __restrict__ dW, float* __restrict__ db, int stage) {
  extern __shared__ float conv1_smem[];
  TraceScope trace;
  pdl_launch_dependents();
  const int kh = KH ? KH : kh_rt, kw = KW ? KW : kw_rt, cin = CIN ? CIN : cin_rt;
  const int K = kh * kw * cin;
  float* s_x = conv1_smem;                         // [h * w * cin]
  float* s_red = conv1_smem + h * w * cin;         // [n_grp][K + 1][cout]
  __shared__ int s_off[kConv1MaxK];                // input offset of filter tap k relative to the window origin (runtime shapes)
  const int tid = threadIdx.x;
  if (KH == 0 && tid < kConv1MaxK) {
    const int k = tid < K ? tid : 0, ci = k % cin, t = k / cin;
    s_off[tid] = ((t / kw) * w + (t % kw)) * cin + ci;
  }
  const int oh = h - kh + 1, ow = w - kw + 1, ph = oh / 2, pw = ow / 2;
  const int c = tid % cout, grp = tid / cout, n_grp = kConv1Threads / cout;
  constexpr int KA = KH ? KH * KW * CIN : kConv1MaxK;
  float acc[KA];
#pragma unroll
  for (int k = 0; k < KA; ++k) acc[k] = 0.f;
  float bacc = 0.f;
  pdl_wait();
  trace.mark();
  // s_g / s_am: this image's dL/dz at the pooling winners (gradient x activation derivative) and the winner positions,
  // staged with coalesced loads (three dependent global loads per pooled pixel were the kernel's critical path)
  float* s_g = s_red + n_grp * (K + 1) * cout;
  uint8_t* s_am = reinterpret_cast<uint8_t*>(s_g + (stage ? ph * pw * cout : 0));
  for (int img = blockIdx.x; img < n; img += gridDim.x) {
    __syncthreads();
    const __nv_bfloat16* xi = x + static_cast<size_t>(img) * h * w * cin;
    for (int i = tid; i < h * w * cin; i += kConv1Threads) s_x[i] = __bfloat162float(xi[i]);
    if (stage) {
      const size_t o0 = static_cast<size_t>(img) * ph * pw * cout;
      for (int i = tid; i < ph * pw * cout; i += kConv1Threads) {
        const float a = __bfloat162float(pooled[o0 + i]);
        s_g[i] = __bfloat162float(g_pool[o0 + i]) * pool_dact(a, act);
        s_am[i] = argmax[o0 + i];
      }
    }
    __syncthreads();
    for (int p = grp; p < ph * pw; p += n_grp) {
      float g;
      int am;
      if (stage) {
        g = s_g[p * cout + c];
        am = s_am[p * cout + c];
      } else {
        const size_t o = (static_cast<size_t>(img) * ph * pw + p) * cout + c;
        g = __bfloat162float(g_pool[o]) * pool_dact(__bfloat162float(pooled[o]), act);
        am = argmax[o];
      }
      if (g == 0.f) continue;
      const int py = p / pw, px = p - py * pw;
      const float* r = s_x + ((2 * py + (am >> 1)) * w + 2 * px + (am & 1)) * cin;
      bacc += g;
      if constexpr (KH != 0) {
#pragma unroll
        for (int dy = 0; dy < KH; ++dy)
#pragma unroll
          for (int j = 0; j < KW * CIN; ++j) acc[dy * KW * CIN + j] = fmaf(g, r[dy * w * CIN + j], acc[dy * KW * CIN + j]);
      } else {
#pragma unroll
        for (int k = 0; k < kConv1MaxK; ++k)
          if (k < K) acc[k] = fmaf(g, r[s_off[k]], acc[k]);
      }
    }
  }
  // reduce the groups that share a channel, then one atomic per (k, channel) and CTA
  __syncthreads();
#pragma unroll
  for (int k = 0; k < KA; ++k)
    if (k < K) s_red[(grp * (K + 1) + k) * cout + c] = acc[k];
  s_red[(grp * (K + 1) + K) * cout + c] = bacc;
  __syncthreads();
  for (int i = tid; i < (K + 1) * cout; i += kConv1Threads) {
    float v = 0.f;
    for (int g = 0; g < n_grp; ++g) v += s_red[g * (K + 1) * cout + i];
    if (v != 0.f) {
      if (i < K * cout) atomicAdd(dW + i, v);
      else if (db != nullptr) atomicAdd(db + (i - K * cout), v);
    }
  }
  trace.end(KID_POOL_BWD);
}

}  // namespace sf

template <int KH, int KW, int CIN>
static int conv_first_fwd_launch(const __nv_bfloat16* x, int n, int h, int w, int cin, int kh, int kw, int cout, const __nv_bfloat16* wT, int ld_w,
                                 const float* bias, int act, __nv_bfloat16* pooled, uint8_t* argmax, cudaStream_t st) {
  const int K = kh * kw * cin;
  const size_t smem = ((KH ? 0 : static_cast<size_t>(K) * cout) + static_cast<size_t>(h) * w * cin) * sizeof(float);
  if (smem > 96 * 1024) return -8;
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    cudaError_t e = cudaFuncSetAttribute(sf::conv_first_fwd_kernel<KH, KW, CIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return static_cast<int>(e);
    attr = smem;
  }
  // work items = (image, part): pick the split whose wave count x pixels-per-thread is smallest on every SM x 4 resident CTAs
  const int slots = sf_num_sms() * 4, n_grp = sf::kConv1Threads / cout, P = ((h - kh + 1) / 2) * ((w - kw + 1) / 2);
  int parts = 1;
  float best = 1e30f;
  for (int p = 1; p <= 8; ++p) {
    const int items = n * p, waves = (items + slots - 1) / slots;
    const float util = items < slots ? static_cast<float>(items) / slots : 1.f;
    const float cost = waves * ((P + n_grp * p - 1) / (n_grp * p) + 2.f) / util;
    if (cost < best) { best = cost; parts = p; }
  }
  const int grid = n * parts < slots ? n * parts : slots;
  return static_cast<int>(sf::launch(sf::conv_first_fwd_kernel<KH, KW, CIN>, dim3(grid), dim3(sf::kConv1Threads), smem, st, x, n, h, w, cin, kh, kw,
                                     cout, wT, ld_w, bias, act, pooled, argmax, parts));
}

template <int KH, int KW, int CIN>
static int conv_first_wgrad_launch(const __nv_bfloat16* x, int n, int h, int w, int cin, int kh, int kw, int cout, const __nv_bfloat16* g_pool,
                                   const __nv_bfloat16* pooled, const uint8_t* argmax, int act, float* dW, float* db, cudaStream_t st) {
  const int K = kh * kw * cin;
  const int n_grp = sf::kConv1Threads / cout;
  size_t smem = (static_cast<size_t>(h) * w * cin + static_cast<size_t>(n_grp) * (K + 1) * cout) * sizeof(float);
  if (smem > 96 * 1024) return -8;
  const size_t pc = static_cast<size_t>((h - kh + 1) / 2) * ((w - kw + 1) / 2) * cout;
  const size_t stage_bytes = pc * sizeof(float) + ((pc + 15) / 16) * 16;
  const int stage = smem + stage_bytes <= 96 * 1024 ? 1 : 0;
  if (stage) smem += stage_bytes;
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    cudaError_t e = cudaFuncSetAttribute(sf::conv_first_wgrad_kernel<KH, KW, CIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return static_cast<int>(e);
    attr = smem;
  }
  int grid = n < sf_num_sms() * 2 ? n : sf_num_sms() * 2;          // one (or a few) images per CTA; one atomic per gradient word and CTA
  if (grid < 1) grid = 1;
  return static_cast<int>(sf::launch(sf::conv_first_wgrad_kernel<KH, KW, CIN>, dim3(grid), dim3(sf::kConv1Threads), smem, st, x, n, h, w, cin, kh, kw,
                                     cout, g_pool, pooled, argmax, act, dW, db, stage));
}

#define SF_CONV1_DISPATCH(FN, ...)                                             \
  do {                                                                         \
    if (kh == 5 && kw == 5 && cin == 1) return FN<5, 5, 1>(__VA_ARGS__);       \
    if (kh == 3 && kw == 3 && cin == 1) return FN<3, 3, 1>(__VA_ARGS__);       \
    if (kh == 3 && kw == 3 && cin == 3) return FN<3, 3, 3>(__VA_ARGS__);       \
    return FN<0, 0, 0>(__VA_ARGS__);                                           \
  } while (0)

extern "C" int sf_conv_first_fwd(const __nv_bfloat16* x, int n, int h, int w, int cin, int kh, int kw, int cout, const __nv_bfloat16* wT,
                                 int ld_w, const float* bias, int act, __nv_bfloat16* pooled, uint8_t* argmax, cudaStream_t st) {
  const int K = kh * kw * cin;
  if (K > sf::kConv1MaxK || cout < 8 || cout > 64 || (sf::kConv1Threads % cout) != 0) return -8;
  SF_CONV1_DISPATCH(conv_first_fwd_launch, x, n, h, w, cin, kh, kw, cout, wT, ld_w, bias, act, pooled, argmax, st);
}

extern "C" int sf_conv_first_wgrad(const __nv_bfloat16* x, int n, int h, int w, int cin, int kh, int kw, int cout, const __nv_bfloat16* g_pool,
                                   const __nv_bfloat16* pooled, const uint8_t* argmax, int act, float* dW, float* db, cudaStream_t st) {
  const int K = kh * kw * cin;
  if (K > sf::kConv1MaxK || cout < 8 || cout > 64 || (sf::kConv1Threads % cout) != 0) return -8;
  SF_CONV1_DISPATCH(conv_first_wgrad_launch, x, n, h, w, cin, kh, kw, cout, g_pool, pooled, argmax, act, dW, db, st);
}
