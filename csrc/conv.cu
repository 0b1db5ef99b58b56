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
//
// Geometry follows TensorFlow: stride (sh, sw) and a zero border of pad_top / pad_left rows and columns in front of the
// image (SAME padding puts the odd extra row / column at the bottom / right, which only shows up in the output size).
// Padded conv taps read zero; padded pool cells never win.  VALID stride 1 is pad 0, stride 1, out = in - k + 1.
#include "sm90_ptx.cuh"
#include "sf_api.h"

namespace sf {

// ------------------------------------------------------------------------------------------------
// im2col (NHWC): out[m, k] = in[b, y * sh - pad_top + dy, x * sw - pad_left + dx, c] (zero outside the image);  32x32 tiles
// through smem so that the row-major store (along k) and the transposed store (along m) are both coalesced.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
im2col_kernel(const __nv_bfloat16* __restrict__ in, int n, int h, int w, int c, int kh, int kw, int sh, int sw, int pt, int pl,
              int oh, int ow, __nv_bfloat16* __restrict__ out, int ld_out, __nv_bfloat16* __restrict__ outT, int ld_t) {
  __shared__ __nv_bfloat16 tile[32][34];
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
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
      const int iy = y * sh - pt + dy, ix = x * sw - pl + dx;
      if (iy >= 0 && iy < h && ix >= 0 && ix < w) v = in[((static_cast<size_t>(b) * h + iy) * w + ix) * c + cc];
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
im2col_vec8_kernel(const uint4* __restrict__ in, int n, int h, int w, int c8, int kh, int kw, int sh, int sw, int pt, int pl, int oh,
                   int ow, uint4* __restrict__ out, int ld8) {
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int M = n * oh * ow, K8 = kh * kw * c8;
  const long long total = static_cast<long long>(M) * ld8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int m = static_cast<int>(i / ld8), q = static_cast<int>(i - static_cast<long long>(m) * ld8);
    uint4 v = make_uint4(0u, 0u, 0u, 0u);                    // pad columns and out-of-image taps carry zeros
    if (q < K8) {
      const int tap = q / c8, cc = q - tap * c8;
      const int dy = tap / kw, dx = tap - dy * kw;
      const int b = m / (oh * ow), r = m - b * (oh * ow);
      const int y = r / ow, x = r - y * ow;
      const int iy = y * sh - pt + dy, ix = x * sw - pl + dx;
      if (iy >= 0 && iy < h && ix >= 0 && ix < w) v = in[(static_cast<size_t>(b * h + iy) * w + ix) * c8 + cc];
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
col2im_vec8_kernel(const uint4* __restrict__ dcols, int ld8, int n, int h, int w, int c8, int kh, int kw, int sh, int sw, int pt, int pl,
                   int oh, int ow, uint4* __restrict__ din) {
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int total = n * h * w * c8;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int cc = i % c8;
    int t = i / c8;
    const int x = t % w;
    t /= w;
    const int y = t % h;
    const int b = t / h;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    // taps dy whose output row (y + pt - dy) / sh is a whole number inside [0, oh): the first one of the right residue,
    // then every sh-th, with the output row stepping down by one
    const int yp = y + pt, xp = x + pl;
    const int dy_lo = yp - (oh - 1) * sh > 0 ? yp - (oh - 1) * sh : 0, dy_hi = yp < kh - 1 ? yp : kh - 1;
    const int dx_lo = xp - (ow - 1) * sw > 0 ? xp - (ow - 1) * sw : 0, dx_hi = xp < kw - 1 ? xp : kw - 1;
    const int dy0 = dy_lo + (yp - dy_lo) % sh, dx0 = dx_lo + (xp - dx_lo) % sw;
    int oy = (yp - dy0) / sh;
    const int ox0 = (xp - dx0) / sw;
    for (int dy = dy0; dy <= dy_hi; dy += sh, --oy) {
      const uint4* row = dcols + static_cast<size_t>((b * oh + oy) * ow) * ld8 + (dy * kw) * c8 + cc;
      int ox = ox0;
      for (int dx = dx0; dx <= dx_hi; dx += sw, --ox) acc_bf16x8(acc, row[ox * ld8 + dx * c8]);
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
// col2im as a gather (no atomics): din[b, y, x, c] = sum_{dy,dx} dcols[(b, oy, ox), (dy*kw+dx)*C + c] over the taps with
// oy * sh = y + pad_top - dy and ox * sw = x + pad_left - dx inside the output
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
col2im_kernel(const __nv_bfloat16* __restrict__ dcols, int ld_cols, int n, int h, int w, int c, int kh, int kw, int sh, int sw,
              int pt, int pl, int oh, int ow, __nv_bfloat16* __restrict__ din) {
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
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
      const int ty = y + pt - dy;
      if (ty < 0 || ty % sh != 0 || ty / sh >= oh) continue;
      const int yy = ty / sh;
      for (int dx = 0; dx < kw; ++dx) {
        const int tx = x + pl - dx;
        if (tx < 0 || tx % sw != 0 || tx / sw >= ow) continue;
        const int xx = tx / sw;
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
// EXT: the backward kernels' twins for the extended activations (SfAct 4-9, alpha = a leaky ReLU's slope); the launchers
// pick a twin exactly when act is one of them, so the ReLU / sigmoid / tanh kernels keep their code.
template <bool EXT>
__device__ __forceinline__ float pool_dact(float a, int act, float alpha) {
  return EXT ? act_ext_dact(a, act, alpha) : pool_dact(a, act);
}

template <bool EXT>
__device__ __forceinline__ void maxpool_bwd_tile(const __nv_bfloat16* __restrict__ dout, const uint8_t* __restrict__ argmax, int n, int h,
                                                 int w, int c, const __nv_bfloat16* __restrict__ act_out, int act, float alpha,
                                                 __nv_bfloat16* __restrict__ dz, int ld_dz, __nv_bfloat16* __restrict__ dzT, int ld_t,
                                                 float* __restrict__ dbias) {
  __shared__ __nv_bfloat16 tile[32][34];
  __shared__ float s_col[32];
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int oh = h / 2, ow = w / 2;
  const int M = n * h * w;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int m0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
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
          g = __bfloat162float(dout[o]) * pool_dact<EXT>(__bfloat162float(act_out[static_cast<size_t>(m) * c + cc]), act, alpha);
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

__global__ void __launch_bounds__(256)
maxpool_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const uint8_t* __restrict__ argmax, int n, int h, int w, int c,
                   const __nv_bfloat16* __restrict__ act_out, int act, __nv_bfloat16* __restrict__ dz, int ld_dz,
                   __nv_bfloat16* __restrict__ dzT, int ld_t, float* __restrict__ dbias) {
  maxpool_bwd_tile<false>(dout, argmax, n, h, w, c, act_out, act, 0.f, dz, ld_dz, dzT, ld_t, dbias);
}
__global__ void __launch_bounds__(256)
maxpool_bwd_ext_kernel(const __nv_bfloat16* __restrict__ dout, const uint8_t* __restrict__ argmax, int n, int h, int w, int c,
                       const __nv_bfloat16* __restrict__ act_out, int act, float alpha, __nv_bfloat16* __restrict__ dz, int ld_dz,
                       __nv_bfloat16* __restrict__ dzT, int ld_t, float* __restrict__ dbias) {
  maxpool_bwd_tile<true>(dout, argmax, n, h, w, c, act_out, act, alpha, dz, ld_dz, dzT, ld_t, dbias);
}

// ------------------------------------------------------------------------------------------------
// General max pool: kh x kw window (<= 4x4), stride (sh, sw), pad_top / pad_left cells in front (SAME or VALID).  argmax
// stores the winner's in-window index dy * kw + dx; padded cells never win; ties go to the first cell in row-major order,
// as in maxpool_fwd_kernel.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
maxpool_gen_fwd_kernel(const __nv_bfloat16* __restrict__ in, int n, int h, int w, int c, int kh, int kw, int sh, int sw, int pt, int pl,
                       int oh, int ow, __nv_bfloat16* __restrict__ out, uint8_t* __restrict__ argmax) {
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const size_t total = static_cast<size_t>(n) * oh * ow * c;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cc = static_cast<int>(i % c);
    size_t t = i / c;
    const int x = static_cast<int>(t % ow);
    t /= ow;
    const int y = static_cast<int>(t % oh);
    const int b = static_cast<int>(t / oh);
    const int y0 = y * sh - pt, x0 = x * sw - pl;
    float best = -INFINITY;
    int bi = 0;
    for (int dy = 0; dy < kh; ++dy) {
      const int iy = y0 + dy;
      if (iy < 0 || iy >= h) continue;
      const __nv_bfloat16* row = in + (static_cast<size_t>(b) * h + iy) * w * c + cc;
      for (int dx = 0; dx < kw; ++dx) {
        const int ix = x0 + dx;
        if (ix < 0 || ix >= w) continue;
        const float v = __bfloat162float(row[static_cast<size_t>(ix) * c]);
        if (v > best) { best = v; bi = dy * kw + dx; }
      }
    }
    out[i] = __float2bfloat16(best);
    argmax[i] = static_cast<uint8_t>(bi);
  }
  trace.end(KID_POOL_GEN_FWD);
}

// General max-pool backward, a gather over the conv-output positions fused with act'(a) and the bias gradient:
//   dz[b, y, x, c] = act'(a[b, y, x, c]) * sum over the windows (py, px) that contain (y, x) and whose arg-max is (y, x)
//                    of dout[b, py, px, c]
// (overlapping windows: a position collects the gradient of every window it won).  Row-major dz [M, ld_dz] and the
// column sums over M into dbias[C]; one 32(m) x 32(c) tile per CTA, M tiles on x.
template <bool EXT>
__device__ __forceinline__ void maxpool_gen_bwd_tile(const __nv_bfloat16* __restrict__ dout, const uint8_t* __restrict__ argmax, int n,
                                                     int h, int w, int c, int kh, int kw, int sh, int sw, int pt, int pl, int oh, int ow,
                                                     const __nv_bfloat16* __restrict__ act_out, int act, float alpha,
                                                     __nv_bfloat16* __restrict__ dz, int ld_dz, float* __restrict__ dbias) {
  __shared__ float s_col[32];
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int M = n * h * w;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int m0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
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
      const int yp = y + pt, xp = x + pl;
      // windows py with py * sh <= yp < py * sh + kh, inside [0, oh)
      const int py_lo = yp - kh + 1 > 0 ? (yp - kh + sh) / sh : 0, py_hi = yp / sh < oh - 1 ? yp / sh : oh - 1;
      const int px_lo = xp - kw + 1 > 0 ? (xp - kw + sw) / sw : 0, px_hi = xp / sw < ow - 1 ? xp / sw : ow - 1;
      for (int py = py_lo; py <= py_hi; ++py) {
        const int dy = yp - py * sh;
        for (int px = px_lo; px <= px_hi; ++px) {
          const size_t o = static_cast<size_t>((b * oh + py) * ow + px) * c + cc;
          if (argmax[o] == dy * kw + (xp - px * sw)) g += __bfloat162float(dout[o]);
        }
      }
      if (g != 0.f) g *= pool_dact<EXT>(__bfloat162float(act_out[static_cast<size_t>(m) * c + cc]), act, alpha);
    }
    cacc += g;
    if (dz != nullptr && m < M && cc < ld_dz) dz[static_cast<size_t>(m) * ld_dz + cc] = __float2bfloat16(g);
  }
  if (dbias != nullptr) atomicAdd(&s_col[tx], cacc);
  __syncthreads();
  if (dbias != nullptr && threadIdx.x < 32 && c0 + threadIdx.x < c && s_col[threadIdx.x] != 0.f)
    atomicAdd(dbias + c0 + threadIdx.x, s_col[threadIdx.x]);
  trace.end(KID_POOL_GEN_BWD);
}

__global__ void __launch_bounds__(256)
maxpool_gen_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const uint8_t* __restrict__ argmax, int n, int h, int w, int c, int kh, int kw,
                       int sh, int sw, int pt, int pl, int oh, int ow, const __nv_bfloat16* __restrict__ act_out, int act,
                       __nv_bfloat16* __restrict__ dz, int ld_dz, float* __restrict__ dbias) {
  maxpool_gen_bwd_tile<false>(dout, argmax, n, h, w, c, kh, kw, sh, sw, pt, pl, oh, ow, act_out, act, 0.f, dz, ld_dz, dbias);
}
// (256, 4): under the plain bound ptxas kept this twin at 32 registers and spilled 48 bytes; it needs 52
__global__ void __launch_bounds__(256, 4)
maxpool_gen_bwd_ext_kernel(const __nv_bfloat16* __restrict__ dout, const uint8_t* __restrict__ argmax, int n, int h, int w, int c, int kh,
                           int kw, int sh, int sw, int pt, int pl, int oh, int ow, const __nv_bfloat16* __restrict__ act_out, int act,
                           float alpha, __nv_bfloat16* __restrict__ dz, int ld_dz, float* __restrict__ dbias) {
  maxpool_gen_bwd_tile<true>(dout, argmax, n, h, w, c, kh, kw, sh, sw, pt, pl, oh, ow, act_out, act, alpha, dz, ld_dz, dbias);
}

// ------------------------------------------------------------------------------------------------
// Activation gradient of a conv with no pool after it: dz[m, c] = g[m, c] * act'(a[m, c]) written row-major [M, ld_dz], and
// the column sums over M added into dbias[C].  g is the gradient wrt the conv's activation output: col2im of the next conv
// or the flatten dgrad of the dense layer above.  Same 32(m) x 32(c) tile and s_col reduction as maxpool_bwd_kernel.
// ------------------------------------------------------------------------------------------------
template <bool EXT>
__device__ __forceinline__ void act_bwd_bias_tile(const __nv_bfloat16* __restrict__ g, int ld_g, int M, int c,
                                                  const __nv_bfloat16* __restrict__ act_out, int act, float alpha,
                                                  __nv_bfloat16* __restrict__ dz, int ld_dz, float* __restrict__ dbias) {
  __shared__ float s_col[32];
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int m0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  if (threadIdx.x < 32) s_col[threadIdx.x] = 0.f;
  __syncthreads();
  float cacc = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty + 8 * i, cc = c0 + tx;
    float v = 0.f;
    if (m < M && cc < c)
      v = __bfloat162float(g[static_cast<size_t>(m) * ld_g + cc]) *
          pool_dact<EXT>(__bfloat162float(act_out[static_cast<size_t>(m) * c + cc]), act, alpha);
    cacc += v;
    if (dz != nullptr && m < M && cc < ld_dz) dz[static_cast<size_t>(m) * ld_dz + cc] = __float2bfloat16(v);
  }
  if (dbias != nullptr) atomicAdd(&s_col[tx], cacc);
  __syncthreads();
  if (dbias != nullptr && threadIdx.x < 32 && c0 + threadIdx.x < c && s_col[threadIdx.x] != 0.f)
    atomicAdd(dbias + c0 + threadIdx.x, s_col[threadIdx.x]);
  trace.end(KID_ACT_BWD);
}

__global__ void __launch_bounds__(256)
act_bwd_bias_kernel(const __nv_bfloat16* __restrict__ g, int ld_g, int M, int c, const __nv_bfloat16* __restrict__ act_out, int act,
                    __nv_bfloat16* __restrict__ dz, int ld_dz, float* __restrict__ dbias) {
  act_bwd_bias_tile<false>(g, ld_g, M, c, act_out, act, 0.f, dz, ld_dz, dbias);
}
__global__ void __launch_bounds__(256)
act_bwd_bias_ext_kernel(const __nv_bfloat16* __restrict__ g, int ld_g, int M, int c, const __nv_bfloat16* __restrict__ act_out, int act,
                        float alpha, __nv_bfloat16* __restrict__ dz, int ld_dz, float* __restrict__ dbias) {
  act_bwd_bias_tile<true>(g, ld_g, M, c, act_out, act, alpha, dz, ld_dz, dbias);
}

}  // namespace sf

static inline int grid_1d(size_t total) {
  size_t b = (total + 255) / 256;
  if (b > sf_num_sms() * 16) b = sf_num_sms() * 16;
  return static_cast<int>(b < 1 ? 1 : b);
}

// out_h / out_w <= 0: the VALID output size (in - k) / s + 1
static inline void conv_out_size(int h, int w, int kh, int kw, int sh, int sw, int& oh, int& ow) {
  if (oh <= 0) oh = (h - kh) / sh + 1;
  if (ow <= 0) ow = (w - kw) / sw + 1;
}

extern "C" int sf_im2col_nhwc(const __nv_bfloat16* in, int n, int h, int w, int c, int kh, int kw, int sh, int sw, int pad_top, int pad_left,
                              int out_h, int out_w, __nv_bfloat16* out, int ld_out, __nv_bfloat16* outT, int ld_t, cudaStream_t st) {
  if (sh < 1 || sw < 1) return -8;
  conv_out_size(h, w, kh, kw, sh, sw, out_h, out_w);
  const int M = n * out_h * out_w, K = kh * kw * c;
  if (outT == nullptr && out != nullptr && (c & 7) == 0 && (ld_out & 7) == 0 && ld_out >= K && (reinterpret_cast<uintptr_t>(in) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(out) & 15) == 0) {
    const size_t total = static_cast<size_t>(M) * (ld_out / 8);
    return static_cast<int>(sf::launch(sf::im2col_vec8_kernel, dim3(grid_1d(total)), dim3(256), 0, st, reinterpret_cast<const uint4*>(in), n, h, w,
                                       c / 8, kh, kw, sh, sw, pad_top, pad_left, out_h, out_w, reinterpret_cast<uint4*>(out), ld_out / 8));
  }
  const int span_k = (out && ld_out > K) ? ld_out : K;
  dim3 grid((M + 31) / 32, (span_k + 31) / 32);
  return static_cast<int>(sf::launch(sf::im2col_kernel, grid, dim3(256), 0, st, in, n, h, w, c, kh, kw, sh, sw, pad_top, pad_left, out_h, out_w,
                                     out, ld_out, outT, ld_t));
}

extern "C" int sf_col2im_nhwc(const __nv_bfloat16* dcols, int ld_cols, int n, int h, int w, int c, int kh, int kw, int sh, int sw, int pad_top,
                              int pad_left, int out_h, int out_w, __nv_bfloat16* din, cudaStream_t st) {
  if (sh < 1 || sw < 1) return -8;
  conv_out_size(h, w, kh, kw, sh, sw, out_h, out_w);
  const size_t total = static_cast<size_t>(n) * h * w * c;
  if ((c & 7) == 0 && (ld_cols & 7) == 0 && total / 8 < (1u << 30) && (reinterpret_cast<uintptr_t>(dcols) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(din) & 15) == 0)
    return static_cast<int>(sf::launch(sf::col2im_vec8_kernel, dim3(grid_1d(total / 8)), dim3(256), 0, st, reinterpret_cast<const uint4*>(dcols),
                                       ld_cols / 8, n, h, w, c / 8, kh, kw, sh, sw, pad_top, pad_left, out_h, out_w, reinterpret_cast<uint4*>(din)));
  return static_cast<int>(sf::launch(sf::col2im_kernel, dim3(grid_1d(total)), dim3(256), 0, st, dcols, ld_cols, n, h, w, c, kh, kw, sh, sw, pad_top,
                                     pad_left, out_h, out_w, din));
}

extern "C" int sf_maxpool2_fwd(const __nv_bfloat16* in, int n, int h, int w, int c, __nv_bfloat16* out, uint8_t* argmax,
                               __nv_bfloat16* outT, int ld_t, cudaStream_t st) {
  const size_t total = static_cast<size_t>(n) * (h / 2) * (w / 2) * c;
  return static_cast<int>(sf::launch(sf::maxpool_fwd_kernel, dim3(grid_1d(total)), dim3(256), 0, st, in, n, h, w, c, out, argmax, outT, ld_t));
}

extern "C" int sf_maxpool2_bwd(const __nv_bfloat16* dout, const uint8_t* argmax, int n, int h, int w, int c,
                               const __nv_bfloat16* act_out, int act, float act_alpha, __nv_bfloat16* dz, int ld_dz, __nv_bfloat16* dzT,
                               int ld_t, float* dbias, cudaStream_t st) {
  const int M = n * h * w;
  const int span_c = (dz && ld_dz > c) ? ld_dz : c;
  dim3 grid((M + 31) / 32, (span_c + 31) / 32);     // rows on grid.x: a large batch outgrows grid.y's 65535 blocks
  if (act >= SF_ACT_ELU)
    return static_cast<int>(sf::launch(sf::maxpool_bwd_ext_kernel, grid, dim3(256), 0, st, dout, argmax, n, h, w, c, act_out, act, act_alpha,
                                       dz, ld_dz, dzT, ld_t, dbias));
  return static_cast<int>(sf::launch(sf::maxpool_bwd_kernel, grid, dim3(256), 0, st, dout, argmax, n, h, w, c, act_out, act, dz,
                                     ld_dz, dzT, ld_t, dbias));
}

extern "C" int sf_maxpool_fwd(const __nv_bfloat16* in, int n, int h, int w, int c, int kh, int kw, int sh, int sw, int pad_top, int pad_left,
                              int out_h, int out_w, __nv_bfloat16* out, uint8_t* argmax, cudaStream_t st) {
  if (kh < 1 || kw < 1 || kh > 4 || kw > 4 || sh < 1 || sw < 1) return -8;
  conv_out_size(h, w, kh, kw, sh, sw, out_h, out_w);
  const size_t total = static_cast<size_t>(n) * out_h * out_w * c;
  return static_cast<int>(sf::launch(sf::maxpool_gen_fwd_kernel, dim3(grid_1d(total)), dim3(256), 0, st, in, n, h, w, c, kh, kw, sh, sw, pad_top,
                                     pad_left, out_h, out_w, out, argmax));
}

extern "C" int sf_maxpool_bwd(const __nv_bfloat16* dout, const uint8_t* argmax, int n, int h, int w, int c, int kh, int kw, int sh, int sw,
                              int pad_top, int pad_left, int out_h, int out_w, const __nv_bfloat16* act_out, int act, float act_alpha,
                              __nv_bfloat16* dz, int ld_dz, float* dbias, cudaStream_t st) {
  if (kh < 1 || kw < 1 || kh > 4 || kw > 4 || sh < 1 || sw < 1) return -8;
  conv_out_size(h, w, kh, kw, sh, sw, out_h, out_w);
  const int M = n * h * w;
  const int span_c = (dz && ld_dz > c) ? ld_dz : c;
  dim3 grid((M + 31) / 32, (span_c + 31) / 32);
  if (act >= SF_ACT_ELU)
    return static_cast<int>(sf::launch(sf::maxpool_gen_bwd_ext_kernel, grid, dim3(256), 0, st, dout, argmax, n, h, w, c, kh, kw, sh, sw,
                                       pad_top, pad_left, out_h, out_w, act_out, act, act_alpha, dz, ld_dz, dbias));
  return static_cast<int>(sf::launch(sf::maxpool_gen_bwd_kernel, grid, dim3(256), 0, st, dout, argmax, n, h, w, c, kh, kw, sh, sw, pad_top,
                                     pad_left, out_h, out_w, act_out, act, dz, ld_dz, dbias));
}

extern "C" int sf_act_bwd_bias(const __nv_bfloat16* g, int ld_g, int rows, int c, const __nv_bfloat16* act_out, int act, float act_alpha,
                               __nv_bfloat16* dz, int ld_dz, float* dbias, cudaStream_t st) {
  const int span_c = (dz && ld_dz > c) ? ld_dz : c;
  dim3 grid((rows + 31) / 32, (span_c + 31) / 32);
  if (act >= SF_ACT_ELU)
    return static_cast<int>(sf::launch(sf::act_bwd_bias_ext_kernel, grid, dim3(256), 0, st, g, ld_g, rows, c, act_out, act, act_alpha, dz,
                                       ld_dz, dbias));
  return static_cast<int>(sf::launch(sf::act_bwd_bias_kernel, grid, dim3(256), 0, st, g, ld_g, rows, c, act_out, act, dz, ld_dz, dbias));
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
// Stride 1 with SAME padding: the CTA stages the image inside a zero border (pad_top rows above, pad_left columns to the
// left, the rest below / right) of (oh + kh - 1) x (ow + kw - 1) pixels and runs the VALID loops over it; pads of 0
// stage the plain image.
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

// image `xi` [h, w, cin] -> s_x [hp, wp, cin] fp32 inside a zero border (pt rows above, pl columns to the left)
__device__ __forceinline__ void conv1_stage_image(float* s_x, const __nv_bfloat16* __restrict__ xi, int h, int w, int cin, int hp, int wp,
                                                  int pt, int pl) {
  if (hp == h && wp == w) {
    for (int i = threadIdx.x; i < h * w * cin; i += kConv1Threads) s_x[i] = __bfloat162float(xi[i]);
    return;
  }
  const int row = wp * cin, shift = pl * cin;      // one padded row; the image row starts `shift` floats into it
#pragma unroll 1                                   // kept rolled: the VALID fast path above must not pay for its code
  for (int i = threadIdx.x; i < hp * row; i += kConv1Threads) {
    const int y = i / row - pt, j = i - (y + pt) * row - shift;
    s_x[i] = (y >= 0 && y < h && j >= 0 && j < w * cin) ? __bfloat162float(xi[y * w * cin + j]) : 0.f;
  }
}

// x [n, h, w, cin] bf16; wT [cout, ld_w] bf16 (row c = filter of channel c, k = (dy * kw + dx) * cin + ci); bias fp32 [cout]
// pooled [n, oh/2, ow/2, cout] bf16; argmax uint8 (position 0..3 of the winner inside its 2x2 window)
// KH / KW / CIN are compile-time (0 = runtime): with constant taps the filter lives in registers and the window loop unrolls.
template <int KH, int KW, int CIN>
__global__ void __launch_bounds__(kConv1Threads)
conv_first_fwd_kernel(const __nv_bfloat16* __restrict__ x, int n, int h, int w, int cin_rt, int kh_rt, int kw_rt, int cout, int pt, int pl,
                      int oh, int ow, const __nv_bfloat16* __restrict__ wT, int ld_w, const float* __restrict__ bias, int act,
                      __nv_bfloat16* __restrict__ pooled, uint8_t* __restrict__ argmax, int parts) {
  extern __shared__ float conv1_smem[];
  TraceScope trace;
  pdl_launch_dependents();
  const int kh = KH ? KH : kh_rt, kw = KW ? KW : kw_rt, cin = CIN ? CIN : cin_rt;
  const int K = kh * kw * cin;
  float* s_w = conv1_smem;                       // [K][cout]  (runtime-shape path only)
  float* s_x = conv1_smem + (KH ? 0 : K * cout); // [hp * wp * cin]
  const int tid = threadIdx.x;
  const int hp = oh + kh - 1, wp = ow + kw - 1, ph = oh / 2, pw = ow / 2;
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
    conv1_stage_image(s_x, x + static_cast<size_t>(img) * h * w * cin, h, w, cin, hp, wp, pt, pl);
    __syncthreads();
    for (int p = grp + part * n_grp; p < ph * pw; p += n_grp * parts) {
      const int py = p / pw, px = p - py * pw;
      float a00 = b, a01 = b, a10 = b, a11 = b;
      if constexpr (KH != 0) {
        // (KH + 1) x (KW + 1) input window of the 2x2 output quad, one row at a time, filter taps from registers
#pragma unroll
        for (int iy = 0; iy <= KH; ++iy) {
          float row[(KW + 1) * CIN];
          const float* rp = s_x + ((2 * py + iy) * wp + 2 * px) * CIN;
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
          const float* r0 = s_x + ((2 * py + dy) * wp + 2 * px) * cin;
          const float* r1 = r0 + wp * cin;
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
conv_first_wgrad_kernel(const __nv_bfloat16* __restrict__ x, int n, int h, int w, int cin_rt, int kh_rt, int kw_rt, int cout, int pt, int pl,
                        int oh, int ow, const __nv_bfloat16* __restrict__ g_pool, const __nv_bfloat16* __restrict__ pooled,
                        const uint8_t* __restrict__ argmax, int act, float* __restrict__ dW, float* __restrict__ db, int stage) {
  extern __shared__ float conv1_smem[];
  TraceScope trace;
  pdl_launch_dependents();
  const int kh = KH ? KH : kh_rt, kw = KW ? KW : kw_rt, cin = CIN ? CIN : cin_rt;
  const int K = kh * kw * cin;
  const int hp = oh + kh - 1, wp = ow + kw - 1, ph = oh / 2, pw = ow / 2;
  float* s_x = conv1_smem;                         // [hp * wp * cin]
  float* s_red = conv1_smem + hp * wp * cin;       // [n_grp][K + 1][cout]
  __shared__ int s_off[kConv1MaxK];                // input offset of filter tap k relative to the window origin (runtime shapes)
  const int tid = threadIdx.x;
  if (KH == 0 && tid < kConv1MaxK) {
    const int k = tid < K ? tid : 0, ci = k % cin, t = k / cin;
    s_off[tid] = ((t / kw) * wp + (t % kw)) * cin + ci;
  }
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
    conv1_stage_image(s_x, x + static_cast<size_t>(img) * h * w * cin, h, w, cin, hp, wp, pt, pl);
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
      const float* r = s_x + ((2 * py + (am >> 1)) * wp + 2 * px + (am & 1)) * cin;
      bacc += g;
      if constexpr (KH != 0) {
#pragma unroll
        for (int dy = 0; dy < KH; ++dy)
#pragma unroll
          for (int j = 0; j < KW * CIN; ++j) acc[dy * KW * CIN + j] = fmaf(g, r[dy * wp * CIN + j], acc[dy * KW * CIN + j]);
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
static int conv_first_fwd_launch(const __nv_bfloat16* x, int n, int h, int w, int cin, int kh, int kw, int cout, int pt, int pl, int oh, int ow,
                                 const __nv_bfloat16* wT, int ld_w, const float* bias, int act, __nv_bfloat16* pooled, uint8_t* argmax,
                                 cudaStream_t st) {
  const int K = kh * kw * cin;
  const size_t smem = ((KH ? 0 : static_cast<size_t>(K) * cout) + static_cast<size_t>(oh + kh - 1) * (ow + kw - 1) * cin) * sizeof(float);
  if (smem > 96 * 1024) return -8;
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    cudaError_t e = cudaFuncSetAttribute(sf::conv_first_fwd_kernel<KH, KW, CIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return static_cast<int>(e);
    attr = smem;
  }
  // work items = (image, part): pick the split whose wave count x pixels-per-thread is smallest on every SM x 4 resident CTAs
  const int slots = sf_num_sms() * 4, n_grp = sf::kConv1Threads / cout, P = (oh / 2) * (ow / 2);
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
                                     cout, pt, pl, oh, ow, wT, ld_w, bias, act, pooled, argmax, parts));
}

template <int KH, int KW, int CIN>
static int conv_first_wgrad_launch(const __nv_bfloat16* x, int n, int h, int w, int cin, int kh, int kw, int cout, int pt, int pl, int oh,
                                   int ow, const __nv_bfloat16* g_pool, const __nv_bfloat16* pooled, const uint8_t* argmax, int act, float* dW,
                                   float* db, cudaStream_t st) {
  const int K = kh * kw * cin;
  const int n_grp = sf::kConv1Threads / cout;
  size_t smem = (static_cast<size_t>(oh + kh - 1) * (ow + kw - 1) * cin + static_cast<size_t>(n_grp) * (K + 1) * cout) * sizeof(float);
  if (smem > 96 * 1024) return -8;
  const size_t pc = static_cast<size_t>(oh / 2) * (ow / 2) * cout;
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
                                     cout, pt, pl, oh, ow, g_pool, pooled, argmax, act, dW, db, stage));
}

#define SF_CONV1_DISPATCH(FN, ...)                                             \
  do {                                                                         \
    if (kh == 5 && kw == 5 && cin == 1) return FN<5, 5, 1>(__VA_ARGS__);       \
    if (kh == 3 && kw == 3 && cin == 1) return FN<3, 3, 1>(__VA_ARGS__);       \
    if (kh == 3 && kw == 3 && cin == 3) return FN<3, 3, 3>(__VA_ARGS__);       \
    return FN<0, 0, 0>(__VA_ARGS__);                                           \
  } while (0)

// out_h / out_w <= 0: VALID (pads 0, out = in - k + 1); otherwise stride 1 with pad_top / pad_left zero rows / columns in front
static inline bool conv1_geometry(int h, int w, int kh, int kw, int pad_top, int pad_left, int& oh, int& ow) {
  if (oh <= 0) oh = h - kh + 1;
  if (ow <= 0) ow = w - kw + 1;
  return pad_top >= 0 && pad_left >= 0 && pad_top < kh && pad_left < kw && oh >= 2 && ow >= 2 && oh + kh - 1 >= h + pad_top &&
         ow + kw - 1 >= w + pad_left;
}

extern "C" int sf_conv_first_fwd(const __nv_bfloat16* x, int n, int h, int w, int cin, int kh, int kw, int cout, const __nv_bfloat16* wT,
                                 int ld_w, const float* bias, int act, __nv_bfloat16* pooled, uint8_t* argmax, int pad_top, int pad_left,
                                 int out_h, int out_w, cudaStream_t st) {
  const int K = kh * kw * cin;
  if (K > sf::kConv1MaxK || cout < 8 || cout > 64 || (sf::kConv1Threads % cout) != 0) return -8;
  if (!conv1_geometry(h, w, kh, kw, pad_top, pad_left, out_h, out_w)) return -8;
  SF_CONV1_DISPATCH(conv_first_fwd_launch, x, n, h, w, cin, kh, kw, cout, pad_top, pad_left, out_h, out_w, wT, ld_w, bias, act, pooled, argmax, st);
}

extern "C" int sf_conv_first_wgrad(const __nv_bfloat16* x, int n, int h, int w, int cin, int kh, int kw, int cout, const __nv_bfloat16* g_pool,
                                   const __nv_bfloat16* pooled, const uint8_t* argmax, int act, float* dW, float* db, int pad_top, int pad_left,
                                   int out_h, int out_w, cudaStream_t st) {
  const int K = kh * kw * cin;
  if (K > sf::kConv1MaxK || cout < 8 || cout > 64 || (sf::kConv1Threads % cout) != 0) return -8;
  if (!conv1_geometry(h, w, kh, kw, pad_top, pad_left, out_h, out_w)) return -8;
  SF_CONV1_DISPATCH(conv_first_wgrad_launch, x, n, h, w, cin, kh, kw, cout, pad_top, pad_left, out_h, out_w, g_pool, pooled, argmax, act, dW, db,
                    st);
}
