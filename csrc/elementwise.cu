// Elementwise / reduction kernels of the training step that are not GEMMs:
// input cast+transpose (K11 feeder), softmax-cross-entropy against one-hot / soft labels or class indices (K5), MSE and
// sigmoid-cross-entropy (K6), argmax (K7).
// Reference semantics: tf.losses.softmax_cross_entropy / mean_squared_error / sigmoid_cross_entropy with the default
// SUM_BY_NONZERO_WEIGHTS reduction (examples/simple_dnn.py:20, autoencoder_example.py:15).
#include "sm90_ptx.cuh"
#include "sf_api.h"

namespace sf {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float dact_from_out(float a, int act) {
  switch (act) {
    case SF_ACT_RELU: return a > 0.f ? 1.f : 0.f;
    case SF_ACT_SIGMOID: return a * (1.f - a);
    case SF_ACT_TANH: return 1.f - a * a;
    default: return 1.f;
  }
}
// with the extended set (SfAct 4-9)
__device__ __forceinline__ float dact_from_out(float a, int act, float alpha) {
  return act >= SF_ACT_ELU ? act_ext_dact(a, act, alpha) : dact_from_out(a, act);
}

// ---------------------------------------------------------------------------
// fp32 -> bf16 cast with optional row gather and transposed copy.  32x32 tiles through smem so
// that both the row-major and the transposed stores are coalesced.
// ---------------------------------------------------------------------------
template <bool GATHER>
__global__ void __launch_bounds__(256)
cast_transpose_kernel(const float* __restrict__ in, int ld_in, const int32_t* __restrict__ idx,
                      __nv_bfloat16* __restrict__ out, int ld_out, __nv_bfloat16* __restrict__ outT,
                      int ld_t, int rows, int cols) {
  __shared__ float tile[32][33];
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + ty + 8 * i, c = c0 + tx;
    float v = 0.f;
    if (r < rows && c < cols) {
      const int src_r = GATHER ? idx[r] : r;
      v = in[static_cast<size_t>(src_r) * ld_in + c];
    }
    tile[ty + 8 * i][tx] = v;
    if (out != nullptr && r < rows && c < ld_out) out[static_cast<size_t>(r) * ld_out + c] = __float2bfloat16(v);
  }
  if (outT == nullptr) {
    trace.end(KID_CAST);
    return;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + 8 * i, r = r0 + tx;       // outT[c][r]
    if (c < cols && r < ld_t)
      outT[static_cast<size_t>(c) * ld_t + r] = __float2bfloat16(r < rows ? tile[tx][ty + 8 * i] : 0.f);
  }
  trace.end(KID_CAST);
}

// ---------------------------------------------------------------------------
// Softmax cross-entropy: one warp per row.
//   loss  += sum_j y_j (lse - z_j) / B
//   dz_j   = (softmax_j * sum(y) - y_j) / B
// dbias (column sums of dz) is accumulated per block in shared memory, then one atomic per column.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
softmax_xent_kernel(const float* __restrict__ logits, int ld_logits, const float* __restrict__ labels,
                    int ld_labels, float* __restrict__ loss, __nv_bfloat16* __restrict__ dz, int ld_dz,
                    __nv_bfloat16* __restrict__ dzT, int ld_t, float* __restrict__ dbias, int rows,
                    int cols) {
  extern __shared__ float s_db[];   // [cols]
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) s_db[c] = 0.f;
  __syncthreads();
  const float inv_b = 1.f / static_cast<float>(rows);
  float loss_acc = 0.f;
  for (int r = blockIdx.x * warps_per_block + warp; r < rows; r += gridDim.x * warps_per_block) {
    const float* z = logits + static_cast<size_t>(r) * ld_logits;
    const float* y = labels + static_cast<size_t>(r) * ld_labels;
    float mx = -INFINITY;
    for (int c = lane; c < cols; c += 32) mx = fmaxf(mx, z[c]);
    mx = warp_max(mx);
    float se = 0.f, sy = 0.f, szy = 0.f;
    for (int c = lane; c < cols; c += 32) {
      const float zc = z[c], yc = y[c];
      se += __expf(zc - mx);
      sy += yc;
      szy += yc * zc;
    }
    se = warp_sum(se);
    sy = warp_sum(sy);
    szy = warp_sum(szy);
    const float lse = mx + __logf(se);
    loss_acc += (lse * sy - szy);
    const float inv_se = 1.f / se;
    for (int c = lane; c < cols; c += 32) {
      const float p = __expf(z[c] - mx) * inv_se;
      const float g = (p * sy - y[c]) * inv_b;
      if (dz) dz[static_cast<size_t>(r) * ld_dz + c] = __float2bfloat16(g);
      if (dzT) dzT[static_cast<size_t>(c) * ld_t + r] = __float2bfloat16(g);
      if (dbias) atomicAdd(&s_db[c], g);
    }
    // zero the padded tail of the row so the K-major GEMM operand is clean
    if (dz)
      for (int c = cols + lane; c < ld_dz; c += 32) dz[static_cast<size_t>(r) * ld_dz + c] = __float2bfloat16(0.f);
  }
  if (lane == 0 && loss_acc != 0.f) atomicAdd(loss, loss_acc * inv_b);
  __syncthreads();
  if (dbias)
    for (int c = threadIdx.x; c < cols; c += blockDim.x)
      if (s_db[c] != 0.f) atomicAdd(dbias + c, s_db[c]);
  trace.end(KID_SOFTMAX);
}

// ---------------------------------------------------------------------------
// Sparse softmax cross-entropy: one warp per row, one class index per row (labels[r * ld_labels], truncated toward zero).
//   loss  += (lse - z_label) / B
//   dz_j   = (softmax_j - [j == label]) / B
// The label is compared with the column index inside the column loops and never used as an address.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
sparse_softmax_xent_kernel(const float* __restrict__ logits, int ld_logits, const float* __restrict__ labels,
                           int ld_labels, float* __restrict__ loss, __nv_bfloat16* __restrict__ dz, int ld_dz,
                           __nv_bfloat16* __restrict__ dzT, int ld_t, float* __restrict__ dbias, int rows,
                           int cols) {
  extern __shared__ float s_db[];   // [cols]
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) s_db[c] = 0.f;
  __syncthreads();
  const float inv_b = 1.f / static_cast<float>(rows);
  float loss_acc = 0.f;
  for (int r = blockIdx.x * warps_per_block + warp; r < rows; r += gridDim.x * warps_per_block) {
    const float* z = logits + static_cast<size_t>(r) * ld_logits;
    float mx = -INFINITY;
    for (int c = lane; c < cols; c += 32) mx = fmaxf(mx, z[c]);
    mx = warp_max(mx);
    // truncation toward zero; loaded after the max pass (loaded before it, the kernel keeps a 16-byte stack frame)
    const int label = static_cast<int>(labels[static_cast<size_t>(r) * ld_labels]);
    float se = 0.f, zl = 0.f;
    for (int c = lane; c < cols; c += 32) {
      const float zc = z[c];
      se += __expf(zc - mx);
      zl += c == label ? zc : 0.f;
    }
    se = warp_sum(se);
    zl = warp_sum(zl);
    loss_acc += mx + __logf(se) - zl;
    const float inv_se = 1.f / se;
    for (int c = lane; c < cols; c += 32) {
      const float p = __expf(z[c] - mx) * inv_se;
      const float g = (p - (c == label ? 1.f : 0.f)) * inv_b;
      if (dz) dz[static_cast<size_t>(r) * ld_dz + c] = __float2bfloat16(g);
      if (dzT) dzT[static_cast<size_t>(c) * ld_t + r] = __float2bfloat16(g);
      if (dbias) atomicAdd(&s_db[c], g);
    }
    // zero the padded tail of the row so the K-major GEMM operand is clean
    if (dz)
      for (int c = cols + lane; c < ld_dz; c += 32) dz[static_cast<size_t>(r) * ld_dz + c] = __float2bfloat16(0.f);
  }
  if (lane == 0 && loss_acc != 0.f) atomicAdd(loss, loss_acc * inv_b);
  __syncthreads();
  if (dbias)
    for (int c = threadIdx.x; c < cols; c += blockDim.x)
      if (s_db[c] != 0.f) atomicAdd(dbias + c, s_db[c]);
  trace.end(KID_SPARSE_SOFTMAX);
}

// ---------------------------------------------------------------------------
// Element-wise losses over all elements (32x32 tiles; transposed store through smem; column sums for dbias).  The
// head maps (network output o, target t) to a loss term and dz:
//   MseHead          loss += mean((o - t)^2), dz = 2 (o - t) / (rows * cols) * act'(o)   (o after activation `act`)
//   SigmoidXentHead  loss += mean(max(o, 0) - o t + log1p(exp(-|o|))), dz = (sigmoid(o) - t) / (rows * cols)  (raw logits)
//   MseExtHead       MseHead for the extended activations (SfAct 4-9; alpha: a leaky ReLU's slope), its own kernel so
//                    that the MSE kernel of ReLU / sigmoid / tanh outputs keeps its code
// ---------------------------------------------------------------------------
struct MseHead {
  static constexpr int kKid = KID_MSE;
  __device__ static float scale(int rows, int cols) { return 2.f / (static_cast<float>(rows) * static_cast<float>(cols)); }
  __device__ static float grad(float o, float t, int act, float, float scale, float& lacc) {
    const float d = o - t;
    lacc += d * d;
    return d * scale * dact_from_out(o, act);
  }
  __device__ static float loss(float sum, float scale) { return sum * 0.5f * scale; }
};

struct MseExtHead {
  static constexpr int kKid = KID_MSE;
  __device__ static float scale(int rows, int cols) { return 2.f / (static_cast<float>(rows) * static_cast<float>(cols)); }
  __device__ static float grad(float o, float t, int act, float alpha, float scale, float& lacc) {
    const float d = o - t;
    lacc += d * d;
    return d * scale * dact_from_out(o, act, alpha);
  }
  __device__ static float loss(float sum, float scale) { return sum * 0.5f * scale; }
};

struct SigmoidXentHead {
  static constexpr int kKid = KID_SIGMOID_XENT;
  __device__ static float scale(int rows, int cols) { return 1.f / (static_cast<float>(rows) * static_cast<float>(cols)); }
  __device__ static float grad(float o, float t, int, float, float scale, float& lacc) {
    float g;
    lacc += sigmoid_xent_elem(o, t, g);
    return g * scale;
  }
  __device__ static float loss(float sum, float scale) { return sum * scale; }
};

template <class Head>
__device__ __forceinline__ void elementwise_loss_tile(const float* __restrict__ out, int ld_out, const float* __restrict__ target,
                                                      int ld_target, int act, float act_alpha, float* __restrict__ loss,
                                                      __nv_bfloat16* __restrict__ dz, int ld_dz, __nv_bfloat16* __restrict__ dzT, int ld_t,
                                                      float* __restrict__ dbias, int rows, int cols) {
  __shared__ float tile[32][33];
  __shared__ float s_col[32];
  __shared__ float s_loss[8];
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  if (threadIdx.x < 32) s_col[threadIdx.x] = 0.f;
  __syncthreads();
  const float scale = Head::scale(rows, cols);
  float lacc = 0.f, cacc = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + ty + 8 * i, c = c0 + tx;
    float g = 0.f;
    if (r < rows && c < cols)
      g = Head::grad(out[static_cast<size_t>(r) * ld_out + c], target[static_cast<size_t>(r) * ld_target + c], act, act_alpha, scale,
                     lacc);
    tile[ty + 8 * i][tx] = g;
    cacc += g;
    if (dz != nullptr && r < rows && c < ld_dz) dz[static_cast<size_t>(r) * ld_dz + c] = __float2bfloat16(g);
  }
  if (dbias) atomicAdd(&s_col[tx], cacc);
  lacc = warp_sum(lacc);
  if (tx == 0) s_loss[ty] = lacc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += s_loss[i];
    if (t != 0.f) atomicAdd(loss, Head::loss(t, scale));
  }
  if (dbias && threadIdx.x < 32 && c0 + threadIdx.x < cols && s_col[threadIdx.x] != 0.f)
    atomicAdd(dbias + c0 + threadIdx.x, s_col[threadIdx.x]);
  if (dzT != nullptr) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = c0 + ty + 8 * i, r = r0 + tx;
      if (c < cols && r < rows) dzT[static_cast<size_t>(c) * ld_t + r] = __float2bfloat16(tile[tx][ty + 8 * i]);
    }
  }
  trace.end(Head::kKid);
}

template <class Head>
__global__ void __launch_bounds__(256)
elementwise_loss_kernel(const float* __restrict__ out, int ld_out, const float* __restrict__ target, int ld_target,
                        int act, float* __restrict__ loss, __nv_bfloat16* __restrict__ dz, int ld_dz,
                        __nv_bfloat16* __restrict__ dzT, int ld_t, float* __restrict__ dbias, int rows, int cols) {
  elementwise_loss_tile<Head>(out, ld_out, target, ld_target, act, 0.f, loss, dz, ld_dz, dzT, ld_t, dbias, rows, cols);
}
// MSE of an output with an extended activation (MseExtHead); act_alpha: a leaky ReLU's slope
__global__ void __launch_bounds__(256)
mse_ext_loss_kernel(const float* __restrict__ out, int ld_out, const float* __restrict__ target, int ld_target, int act, float act_alpha,
                    float* __restrict__ loss, __nv_bfloat16* __restrict__ dz, int ld_dz, __nv_bfloat16* __restrict__ dzT, int ld_t,
                    float* __restrict__ dbias, int rows, int cols) {
  elementwise_loss_tile<MseExtHead>(out, ld_out, target, ld_target, act, act_alpha, loss, dz, ld_dz, dzT, ld_t, dbias, rows, cols);
}

__global__ void __launch_bounds__(256)
argmax_rows_kernel(const float* __restrict__ in, int ld, float* __restrict__ out, int rows, int cols) {
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const float* z = in + static_cast<size_t>(warp) * ld;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int c = lane; c < cols; c += 32) {
    const float v = z[c];
    if (v > best) { best = v; bi = c; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) out[warp] = static_cast<float>(bi);
  trace.end(KID_ARGMAX);
}

}  // namespace sf

extern "C" int sf_cast_transpose(const float* in, int ld_in, __nv_bfloat16* out, int ld_out,
                                 __nv_bfloat16* outT, int ld_t, int rows, int cols, cudaStream_t st) {
  const int span_c = (out && ld_out > cols) ? ld_out : cols;
  const int span_r = (outT && ld_t > rows) ? ld_t : rows;
  dim3 grid((span_c + 31) / 32, (span_r + 31) / 32);
  return static_cast<int>(sf::launch(sf::cast_transpose_kernel<false>, grid, dim3(256), 0, st, in, ld_in,
                                     static_cast<const int32_t*>(nullptr), out, ld_out, outT, ld_t, rows, cols));
}

namespace sf {
// fp32 row gather out[r, :] = in[idx[r], :] (label rows / fp32 targets of a minibatch drawn from an HBM-resident partition)
__global__ void __launch_bounds__(256)
gather_rows_f32_kernel(const float* __restrict__ in, int ld_in, const int32_t* __restrict__ idx, float* __restrict__ out, int ld_out,
                       int rows, int cols) {
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int r = warp; r < rows; r += nwarps) {
    const float* src = in + static_cast<size_t>(idx[r]) * ld_in;
    float* dst = out + static_cast<size_t>(r) * ld_out;
    for (int c = lane; c < cols; c += 32) dst[c] = src[c];
  }
  trace.end(KID_CAST);
}
}  // namespace sf

extern "C" int sf_gather_rows_f32(const float* in, int ld_in, const int32_t* idx, float* out, int ld_out, int rows, int cols,
                                  cudaStream_t st) {
  int grid = (rows + 7) / 8;
  if (grid > 296) grid = 296;
  if (grid < 1) grid = 1;
  return static_cast<int>(sf::launch(sf::gather_rows_f32_kernel, dim3(grid), dim3(256), 0, st, in, ld_in, idx, out, ld_out, rows, cols));
}

extern "C" int sf_gather_cast_transpose(const float* in, int ld_in, const int32_t* idx,
                                        __nv_bfloat16* out, int ld_out, __nv_bfloat16* outT, int ld_t,
                                        int rows, int cols, cudaStream_t st) {
  const int span_c = (out && ld_out > cols) ? ld_out : cols;
  const int span_r = (outT && ld_t > rows) ? ld_t : rows;
  dim3 grid((span_c + 31) / 32, (span_r + 31) / 32);
  return static_cast<int>(sf::launch(sf::cast_transpose_kernel<true>, grid, dim3(256), 0, st, in, ld_in, idx, out,
                                     ld_out, outT, ld_t, rows, cols));
}

extern "C" int sf_softmax_xent(const float* logits, int ld_logits, const float* labels, int ld_labels,
                               float* loss, __nv_bfloat16* dz, int ld_dz, __nv_bfloat16* dzT, int ld_t,
                               float* dbias, int rows, int cols, cudaStream_t st) {
  int blocks = (rows + 7) / 8;
  if (blocks > sf_num_sms() * 4) blocks = sf_num_sms() * 4;
  return static_cast<int>(sf::launch(sf::softmax_xent_kernel, dim3(blocks), dim3(256), cols * sizeof(float), st,
                                     logits, ld_logits, labels, ld_labels, loss, dz, ld_dz, dzT, ld_t, dbias, rows, cols));
}

extern "C" int sf_sparse_softmax_xent(const float* logits, int ld_logits, const float* labels, int ld_labels,
                                      float* loss, __nv_bfloat16* dz, int ld_dz, __nv_bfloat16* dzT, int ld_t,
                                      float* dbias, int rows, int cols, cudaStream_t st) {
  int blocks = (rows + 7) / 8;
  if (blocks > sf_num_sms() * 4) blocks = sf_num_sms() * 4;
  return static_cast<int>(sf::launch(sf::sparse_softmax_xent_kernel, dim3(blocks), dim3(256), cols * sizeof(float), st,
                                     logits, ld_logits, labels, ld_labels, loss, dz, ld_dz, dzT, ld_t, dbias, rows, cols));
}

// the grid spans ld_dz columns, so the padded tail of every dz row is written (with zeros)
static dim3 elementwise_loss_grid(__nv_bfloat16* dz, int ld_dz, int rows, int cols) {
  const int span_c = (dz && ld_dz > cols) ? ld_dz : cols;
  return dim3((span_c + 31) / 32, (rows + 31) / 32);
}
template <class Head>
static int launch_elementwise_loss(const float* out, int ld_out, const float* target, int ld_target, int act, float* loss,
                                   __nv_bfloat16* dz, int ld_dz, __nv_bfloat16* dzT, int ld_t, float* dbias, int rows, int cols,
                                   cudaStream_t st) {
  return static_cast<int>(sf::launch(sf::elementwise_loss_kernel<Head>, elementwise_loss_grid(dz, ld_dz, rows, cols), dim3(256), 0, st, out,
                                     ld_out, target, ld_target, act, loss, dz, ld_dz, dzT, ld_t, dbias, rows, cols));
}

extern "C" int sf_mse_loss(const float* out, int ld_out, const float* target, int ld_target, int act, float act_alpha,
                           float* loss, __nv_bfloat16* dz, int ld_dz, __nv_bfloat16* dzT, int ld_t,
                           float* dbias, int rows, int cols, cudaStream_t st) {
  if (act >= SF_ACT_ELU)
    return static_cast<int>(sf::launch(sf::mse_ext_loss_kernel, elementwise_loss_grid(dz, ld_dz, rows, cols), dim3(256), 0, st, out, ld_out,
                                       target, ld_target, act, act_alpha, loss, dz, ld_dz, dzT, ld_t, dbias, rows, cols));
  return launch_elementwise_loss<sf::MseHead>(out, ld_out, target, ld_target, act, loss, dz, ld_dz, dzT, ld_t, dbias, rows, cols, st);
}

extern "C" int sf_sigmoid_xent(const float* logits, int ld_logits, const float* labels, int ld_labels, float* loss,
                               __nv_bfloat16* dz, int ld_dz, __nv_bfloat16* dzT, int ld_t, float* dbias, int rows, int cols,
                               cudaStream_t st) {
  return launch_elementwise_loss<sf::SigmoidXentHead>(logits, ld_logits, labels, ld_labels, SF_ACT_NONE, loss, dz, ld_dz, dzT, ld_t,
                                                      dbias, rows, cols, st);
}

extern "C" int sf_argmax_rows(const float* in, int ld, float* out, int rows, int cols, cudaStream_t st) {
  const int blocks = (rows * 32 + 255) / 256;
  return static_cast<int>(sf::launch(sf::argmax_rows_kernel, dim3(blocks), dim3(256), 0, st, in, ld, out, rows, cols));
}

extern "C" int sf_fill_zero(void* p, size_t bytes, cudaStream_t st) {
  return static_cast<int>(cudaMemsetAsync(p, 0, bytes, st));
}
