// C ABI between the sm_90a kernels (csrc/*.cu) and the host runtime (plan.cpp / bindings.cpp).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

// 4-9: the extended set.  Each derivative is a function of the activation's output a = act(z), which is all the backward
// pass stores; LeakyRelu takes its slope from the epilogue's act_alpha / aux_act_alpha (the kernels' alpha argument).  The
// GEMMs run them on kernel instances of their own (EXT, gemm_sm90.cu), so the kernels of ReLU / sigmoid / tanh models are
// unchanged.
enum SfAct {
  SF_ACT_NONE = 0,
  SF_ACT_RELU = 1,
  SF_ACT_SIGMOID = 2,
  SF_ACT_TANH = 3,
  SF_ACT_ELU = 4,          // x > 0 ? x : exp(x) - 1                           act' = a > 0 ? 1 : a + 1
  SF_ACT_SELU = 5,         // lambda * (x > 0 ? x : alpha (exp(x) - 1))         act' = a > 0 ? lambda : a + lambda alpha
  SF_ACT_SOFTPLUS = 6,     // max(x, 0) + log1p(exp(-|x|))                     act' = 1 - exp(-a)
  SF_ACT_SOFTSIGN = 7,     // x / (1 + |x|)                                    act' = (1 - |a|)^2
  SF_ACT_LEAKY_RELU = 8,   // x > 0 ? x : alpha x, alpha > 0                    act' = a > 0 ? 1 : alpha
  SF_ACT_RELU6 = 9,        // min(max(x, 0), 6)                                 act' = 0 < a < 6 ? 1 : 0
};

enum SfOptimizer {
  SF_OPT_SGD = 0,
  SF_OPT_MOMENTUM = 1,
  SF_OPT_ADAM = 2,
  SF_OPT_RMSPROP = 3,
  SF_OPT_ADAGRAD = 4,
  SF_OPT_ADADELTA = 5,
  SF_OPT_ADAGRAD_DA = 6,
  SF_OPT_FTRL = 7,
  SF_OPT_PROXIMAL_ADAGRAD = 8,
  SF_OPT_PROXIMAL_SGD = 9,
};

enum SfLockMode { SF_LOCK_NONE = 0 /* Hogwild */, SF_LOCK_RW = 1 /* writer-priority RW lock */ };

// ---------------------------------------------------------------------------
// GEMM
// ---------------------------------------------------------------------------
// Sharded master: the flat parameter state is partitioned by push tile (32 x 64 elements of one variable); shard r
// (living on GPU r) owns push tiles [bounds[r], bounds[r + 1]).  A worker's gradient tile is written straight into its
// mailbox on the owning GPU (peer-mapped NVLink stores from the wgrad epilogue: the "push" is fused into the GEMM).
#define SF_MAX_SHARDS 8
struct SfRoute {
  int n_shards;
  int bounds[SF_MAX_SHARDS + 1];
  float* mailbox[SF_MAX_SHARDS];  // this worker's mailbox on every shard owner (flat gradient layout)
};

// Pull fused into the first GEMM of a step (sharded master, Hogwild): the TMA producer of every CTA waits until every
// shard's applier has acknowledged this worker's last push (read-your-writes; the words live in LOCAL memory, the
// appliers write them over NVLink) before it fetches the first weight tile - from the inbox replica the appliers
// publish into with multimem.st.  The wait overlaps everything the step does before its first GEMM.
struct SfRyw {
  int n_shards;
  int ack_grid[SF_MAX_SHARDS];    // acknowledgements per push of shard r (CTAs of its applier)
  const uint32_t* applied;        // local: word r * 16
  const uint32_t* my_posted;      // local: sequence number of my last post
  unsigned long long* stats;      // optional latency accounting, same layout as SfSyncPullArgs.stats
};

struct SfGemmEpilogue {
  float* out_f32;                 // [M, ld_f32] optional
  __nv_bfloat16* out_bf16;        // [M, ld_bf16] optional (ld multiple of 8, pad columns get 0)
  __nv_bfloat16* outT_bf16;       // [N, ld_t]   optional transpose
  const float* bias;              // [N] optional
  const __nv_bfloat16* aux;       // [M, ld_aux] optional: multiply by act'(aux) (dgrad)
  float* colsum;                  // [N] optional: atomicAdd column sums (bias gradient)
  float alpha;
  int ld_f32, ld_bf16, ld_t, ld_aux;
  int act;                        // SfAct applied after bias
  int aux_act;                    // SfAct whose derivative is taken at aux
  int accumulate;                 // atomicAdd into out_f32
  int n_store_limit;              // filled by sf_gemm_prepare
  int one_wave;                   // filled by sf_gemm_prepare: the grid fits on the SMs at once (PDL trigger placement)
  int a_evict_first;
  // fused loss (last dense layer): the epilogue turns the activation into dL/dz in registers, so
  // out_bf16 / outT_bf16 / colsum receive dz, dz^T and the bias gradient directly.
  int loss_mode;                  // SfLossMode: 0 none, 1 softmax cross-entropy (N <= 32), 2 mean squared error,
                                  // 3 sigmoid cross-entropy (raw logits, any N), 4 sparse softmax cross-entropy (N <= 32)
  const float* target;            // [M, ld_target] labels (one-hot / soft) or regression targets; loss mode 4: one class
                                  // index per row in column 0
  int ld_target;
  float* loss;                    // scalar accumulator (mean loss)
  // sharded push fused into a wgrad epilogue: when `route` is set the fp32 output element (row, col) is stored to
  // route->mailbox[owner] + route_off + row * ld_f32 + col, owner = shard of push tile
  // route_tile0 + (row / 32) * route_tiles_c + col / 64 (out_f32 is ignored).
  const SfRoute* route;           // device memory
  int route_tile0, route_tiles_c;
  long long route_off;
  // fused dropout (reference: the tfDropout keep-prob placeholder of tf.nn.dropout, ml_util.py:70-71): after the
  // activation every element is kept with probability drop_keep and scaled by 1 / drop_keep.  The mask is
  // Philox4x32-10 keyed by (drop_seed, 0x5F3759DF) over the counter (row, column / 4, *drop_ctr, drop_stream), lane
  // column % 4 kept iff it is below keep * 2^32: a pure function of (sample row, feature, step number, layer, seed).
  // The training plans mix the worker index and the address of the plan's step counter into the seed, so workers and
  // plans of one worker draw different masks; forward-only plans have no counter (step number 0).  No mask tensor is
  // stored: the backward pass recovers it from the stored activation (aux_keep: aux holds act(z) * mask / keep, so
  // mask = aux != 0).
  float drop_keep;                // 0 or >= 1: no dropout
  unsigned int drop_seed, drop_stream;
  const unsigned int* drop_ctr;   // device word that changes every step (nullptr: 0)
  float aux_keep;                 // dgrad: keep probability of the dropout that produced aux (0 = none)
  const SfRyw* ryw;               // device memory; nullptr = no wait
  // slope of a leaky ReLU `act` / `aux_act` (SF_ACT_LEAKY_RELU); appended last so every field above keeps its offset
  float act_alpha, aux_act_alpha;
  // L2 weight penalty c * sum(W^2) + c_b * sum(b^2) of the layer whose weight gradient this GEMM computes (appended last,
  // like act_alpha).  Set only on weight-gradient GEMMs; they then run the PEN kernel instances (sf_gemm_prepare).
  //   weight: K split 0 adds pen_w2c * W to every fp32 output element (before the store, atomic add or routed red), W
  //           read from the bf16 replica the step computed with: W [M, pen_ld] or, pen_wt = 1, W^T [N, pen_ld]
  //   bias:   the CTAs of row tile 0, split 0 atomically add pen_b2c * b[n] into pen_db[n]
  //   loss:   pen_w2c / 2 * sum(W^2) + pen_b2c / 2 * sum(b^2) over the elements a CTA covers, atomically added to pen_loss
  float pen_w2c;                  // 2c (0 with pen_w = nullptr: no weight term)
  const __nv_bfloat16* pen_w;
  int pen_ld, pen_wt;
  const float* pen_b;             // fp32 bias [N] (nullptr: no bias term)
  float pen_b2c;                  // 2c_b
  float* pen_db;                  // bias gradient [N]
  float* pen_loss;                // loss accumulator (required with a penalty)
  int bm;                         // filled by sf_gemm_prepare: rows of the one-CTA kernel's output tile (SfGemm.bm)
};

enum SfLossMode { SF_LOSS_NONE = 0, SF_LOSS_SOFTMAX_XENT = 1, SF_LOSS_MSE = 2, SF_LOSS_SIGMOID_XENT = 3, SF_LOSS_SPARSE_SOFTMAX_XENT = 4 };

// Epilogue variant of the one-CTA GEMM kernel.  The generic kernel carries every epilogue feature behind runtime tests;
// each specialized variant compiles in only the features of one kind of training GEMM (sf_gemm_prepare picks it):
//   FWD   bias + activation -> bf16
//   LOSS  bias (+ activation) + softmax-CE / MSE head -> dz bf16, loss, optional column sum
//   DGRAD act'(aux) -> bf16, optional column sum
//   WGRAD fp32 store or atomic accumulate (MN-major operands)
//   SIGMOID_LOSS  bias + sigmoid-CE head on raw logits -> dz bf16 (+ transpose), loss, optional column sum, optional
//                 read-your-writes wait; the only kernel with this head (the generic kernel has none)
//   SPARSE_LOSS   bias + softmax-CE head on raw logits against one class index per row (N <= 32, BN 32) -> the same
//                 outputs as SIGMOID_LOSS; the only kernel with this head
enum SfEpi { SF_EPI_GENERIC = 0, SF_EPI_FWD = 1, SF_EPI_LOSS = 2, SF_EPI_DGRAD = 3, SF_EPI_WGRAD = 4, SF_EPI_SIGMOID_LOSS = 5,
             SF_EPI_SPARSE_LOSS = 6 };


struct SfGemm {
  CUtensorMap tmA, tmB;           // filled by sf_gemm_prepare
  const void* a;                  // bf16 [M, lda]  (K contiguous)
  const void* b;                  // bf16 [N, ldb]  (K contiguous); may be a peer-mapped address
  int M, N, K;
  int lda, ldb;
  int bn;                         // 0 = auto
  int bm;                         // in: 0 = auto, 64 or 128 = forced; out: rows of the one-CTA kernel's output tile.  64
                                  // only on a specialized epilogue variant without a K split (auto: when the grid of
                                  // 64-row tiles is still one wave); the pair kernel's value is 128
  int split_k;                    // 0/1 = none
  int kblocks_per_split;          // filled
  int mn_major;                   // 1: BOTH operands are MN-major: a is [K, lda] with M contiguous, b is [K, ldb] with N contiguous
                                  // (D = a^T . b, the weight-gradient form: activations / dz are consumed as they are
                                  // stored, no transposed copies); 0: both K-major (a [M, lda], b [N, ldb])
  int pair;                       // in: -1 = auto, 0 = one-CTA kernel, 1 = force the persistent cluster-pair kernel; out: 0 / 1
  int pair_ctas;                  // CTAs of the persistent cluster-pair kernel (0 = one per SM)
  int epi;                        // in: -1 = auto, SF_EPI_GENERIC = force the generic kernel; out: the SfEpi variant launched
  SfGemmEpilogue ep;
  int kernel;                     // filled by sf_gemm_prepare: the one-CTA kernel instance launched (kGemmKernels, gemm_sm90.cu)
};

#ifdef __cplusplus
extern "C" {
#endif

int sf_gemm_prepare(SfGemm* g);
int sf_gemm_launch(const SfGemm* g, cudaStream_t st);
int sf_gemm_pair_launch(const SfGemm* g, cudaStream_t st);
int sf_gemm_pick_bn(int M, int N);
int sf_num_sms();
unsigned int sf_read_error_code();
int sf_init_error_channel();
unsigned int sf_read_host_error_code();
void sf_set_pdl(int enabled);
int sf_trace_enable(void* buf, unsigned int cap);
unsigned int sf_trace_count();

// ---------------------------------------------------------------------------
// Elementwise / reduction kernels (elementwise.cu)
// ---------------------------------------------------------------------------
// fp32 [rows, cols] (ld_in) -> bf16 [rows, ld_out] and optional transpose bf16 [cols, ld_t]
int sf_gather_rows_f32(const float* in, int ld_in, const int32_t* idx, float* out, int ld_out, int rows, int cols, cudaStream_t st);
int sf_cast_transpose(const float* in, int ld_in, __nv_bfloat16* out, int ld_out,
                      __nv_bfloat16* outT, int ld_t, int rows, int cols, cudaStream_t st);
// gather rows by index then cast/transposes (minibatch assembly on the device)
int sf_gather_cast_transpose(const float* in, int ld_in, const int32_t* idx, __nv_bfloat16* out,
                             int ld_out, __nv_bfloat16* outT, int ld_t, int rows, int cols,
                             cudaStream_t st);
// softmax cross-entropy with (soft) labels: mean loss (atomicAdd into loss[0]), dlogits = (p*sum(y) - y)/B
int sf_softmax_xent(const float* logits, int ld_logits, const float* labels, int ld_labels,
                    float* loss, __nv_bfloat16* dz, int ld_dz, __nv_bfloat16* dzT, int ld_t,
                    float* dbias, int rows, int cols, cudaStream_t st);
// softmax cross-entropy against one class index per row, labels[r * ld_labels] (a float, truncated toward zero like TF's
// Cast): mean loss (lse - z_label) / B, dlogits = (p - [j == label]) / B.  The label is only compared with the column
// index, never used as an address: a label outside [0, cols) reads nothing out of bounds (its row then has no target).
int sf_sparse_softmax_xent(const float* logits, int ld_logits, const float* labels, int ld_labels,
                           float* loss, __nv_bfloat16* dz, int ld_dz, __nv_bfloat16* dzT, int ld_t,
                           float* dbias, int rows, int cols, cudaStream_t st);
// mean squared error over all elements of out (after activation `act`, out is post-activation; act_alpha: the slope of a
// leaky ReLU): loss += mean((out-target)^2); dz = 2*(out-target)/(rows*cols) * act'(out)
int sf_mse_loss(const float* out, int ld_out, const float* target, int ld_target, int act, float act_alpha,
                float* loss, __nv_bfloat16* dz, int ld_dz, __nv_bfloat16* dzT, int ld_t,
                float* dbias, int rows, int cols, cudaStream_t st);
// sigmoid cross-entropy of raw logits z against labels y in [0, 1] over all elements:
// loss += mean(max(z, 0) - z * y + log1p(exp(-|z|))); dz = (sigmoid(z) - y) / (rows * cols)
int sf_sigmoid_xent(const float* logits, int ld_logits, const float* labels, int ld_labels, float* loss,
                    __nv_bfloat16* dz, int ld_dz, __nv_bfloat16* dzT, int ld_t, float* dbias, int rows, int cols,
                    cudaStream_t st);
int sf_argmax_rows(const float* in, int ld, float* out, int rows, int cols, cudaStream_t st);
int sf_fill_zero(void* p, size_t bytes, cudaStream_t st);

// conv building blocks (NHWC; stride (sh, sw), pad_top / pad_left zero rows / columns in front of the image, output
// out_h x out_w; out_h / out_w <= 0 = the VALID size) and max-pools (conv.cu)
int sf_im2col_nhwc(const __nv_bfloat16* in, int n, int h, int w, int c, int kh, int kw, int sh, int sw, int pad_top, int pad_left,
                   int out_h, int out_w, __nv_bfloat16* out, int ld_out, __nv_bfloat16* outT, int ld_t, cudaStream_t st);
int sf_col2im_nhwc(const __nv_bfloat16* dcols, int ld_cols, int n, int h, int w, int c, int kh, int kw, int sh, int sw,
                   int pad_top, int pad_left, int out_h, int out_w, __nv_bfloat16* din, cudaStream_t st);
// 2x2 / stride-2 / unpadded max-pool (the fast path)
int sf_maxpool2_fwd(const __nv_bfloat16* in, int n, int h, int w, int c, __nv_bfloat16* out,
                    uint8_t* argmax, __nv_bfloat16* outT, int ld_t, cudaStream_t st);
int sf_maxpool2_bwd(const __nv_bfloat16* dout, const uint8_t* argmax, int n, int h, int w, int c,
                    const __nv_bfloat16* act_out, int act, float act_alpha, __nv_bfloat16* dz, int ld_dz,
                    __nv_bfloat16* dzT, int ld_t, float* dbias, cudaStream_t st);
// general max-pool: kh x kw <= 4x4 window, any stride, VALID or SAME (argmax = dy * kw + dx of the winner); the backward
// pass is fused with act'(a) of the pooled conv output and the bias gradient and writes row-major dz [M, ld_dz]
int sf_maxpool_fwd(const __nv_bfloat16* in, int n, int h, int w, int c, int kh, int kw, int sh, int sw, int pad_top, int pad_left,
                   int out_h, int out_w, __nv_bfloat16* out, uint8_t* argmax, cudaStream_t st);
int sf_maxpool_bwd(const __nv_bfloat16* dout, const uint8_t* argmax, int n, int h, int w, int c, int kh, int kw, int sh, int sw,
                   int pad_top, int pad_left, int out_h, int out_w, const __nv_bfloat16* act_out, int act, float act_alpha,
                   __nv_bfloat16* dz, int ld_dz, float* dbias, cudaStream_t st);
// activation gradient of a conv with no pool after it: dz = g * act'(a) [rows, ld_dz], dbias += column sums
int sf_act_bwd_bias(const __nv_bfloat16* g, int ld_g, int rows, int c, const __nv_bfloat16* act_out, int act, float act_alpha,
                    __nv_bfloat16* dz, int ld_dz, float* dbias, cudaStream_t st);

// dropout twins for an image dropout (keep in (0, 1), mask key of the GEMM epilogue's dropout over the pooled tensor as the
// matrix [n * out_h * out_w, c] (c % 4 == 0 for the 2x2 one), ctr: the step's counter word, nullptr = 0): the forward kernels scale the pooled value by
// mask / keep and set bit 7 of its argmax byte to the mask (the 2x2 one writes no transposed copy); the backward kernels
// take pool_keep, a dropout on the pooled output (gradient * mask / keep to the winner, the mask from argmax bit 7), or
// act_keep / keep, one on the conv output act_out = act(z) * mask / keep (mask = act_out != 0, act' at act_out * keep,
// times 1 / keep), and write no dz^T
int sf_maxpool2_drop_fwd(const __nv_bfloat16* in, int n, int h, int w, int c, __nv_bfloat16* out, uint8_t* argmax, float keep,
                         unsigned int seed, unsigned int stream, const unsigned int* ctr, cudaStream_t st);
int sf_maxpool2_drop_bwd(const __nv_bfloat16* dout, const uint8_t* argmax, int n, int h, int w, int c, const __nv_bfloat16* act_out,
                         int act, float act_alpha, float pool_keep, float act_keep, __nv_bfloat16* dz, int ld_dz, float* dbias,
                         cudaStream_t st);
int sf_maxpool_drop_fwd(const __nv_bfloat16* in, int n, int h, int w, int c, int kh, int kw, int sh, int sw, int pad_top, int pad_left,
                        int out_h, int out_w, __nv_bfloat16* out, uint8_t* argmax, float keep, unsigned int seed, unsigned int stream,
                        const unsigned int* ctr, cudaStream_t st);
int sf_maxpool_drop_bwd(const __nv_bfloat16* dout, const uint8_t* argmax, int n, int h, int w, int c, int kh, int kw, int sh, int sw,
                        int pad_top, int pad_left, int out_h, int out_w, const __nv_bfloat16* act_out, int act, float act_alpha,
                        float pool_keep, float act_keep, __nv_bfloat16* dz, int ld_dz, float* dbias, cudaStream_t st);
int sf_act_drop_bwd_bias(const __nv_bfloat16* g, int ld_g, int rows, int c, const __nv_bfloat16* act_out, int act, float act_alpha,
                         float keep, __nv_bfloat16* dz, int ld_dz, float* dbias, cudaStream_t st);

// first convolution of a network (K = kh * kw * cin <= 64, cout in {8, 16, 32, 64}) fused with bias, activation and the
// 2x2 max-pool that follows it: direct CUDA-core kernels, one CTA per image, nothing but the pooled tensor is written.
// Stride 1; out_h / out_w <= 0 = VALID, otherwise the conv output size with pad_top / pad_left zero rows / columns in front
int sf_conv_first_fwd(const __nv_bfloat16* x, int n, int h, int w, int cin, int kh, int kw, int cout, const __nv_bfloat16* wT,
                      int ld_w, const float* bias, int act, __nv_bfloat16* pooled, uint8_t* argmax, int pad_top, int pad_left,
                      int out_h, int out_w, cudaStream_t st);
int sf_conv_first_wgrad(const __nv_bfloat16* x, int n, int h, int w, int cin, int kh, int kw, int cout, const __nv_bfloat16* g_pool,
                        const __nv_bfloat16* pooled, const uint8_t* argmax, int act, float* dW, float* db, int pad_top, int pad_left,
                        int out_h, int out_w, cudaStream_t st);

// ---------------------------------------------------------------------------
// Fused push: optimizer step on the (possibly remote) master shard + bf16 publish (optim_push.cu)
// ---------------------------------------------------------------------------
struct SfTensorSeg {              // one trainable variable inside the flat buffers
  int64_t offset;                 // element offset in the flat fp32 buffers
  int rows, cols;                 // [in, out] (bias: rows = 1)
  int64_t w_off;   int w_ld;      // bf16 copy   [rows, w_ld]   (-1 = none)
  int64_t wt_off;  int wt_ld;     // bf16 transpose [cols, wt_ld] (-1 = none)
};

#define SF_MAX_INLINE_SEGS 32

struct SfHyper {
  float lr, beta1, beta2, eps;    // adam: beta1/beta2/eps ; rmsprop: decay=beta1 momentum=beta2
  float momentum, rho, decay;
  float l1, l2, lr_power, init_accum;
  float l2_shrinkage;
  int nesterov, centered;
};

struct SfPushArgs {
  // master state (peer-mapped address when the master is another GPU): one float4 per parameter
  // (.x = value, .y/.z/.w = optimizer slots).  A push reads and writes each element's tuple with ONE
  // 16-byte access, so concurrent Hogwild pushes can lose updates but never tear a (p, m, v) tuple.
  float4* state;
  uint32_t* ctrl;                 // control block in master memory (see SfCtrl offsets)
  // bf16 publish destinations: master copy first, then any replicas that are pushed to directly.
  // With NVLS a single multicast alias covers every replica (shadow_is_mc = 1).
  __nv_bfloat16* shadow_dst[8];
  int n_shadow_dst;
  float* vec_pub[2];              // optional fp32 publish of the 1-D variables (double-buffered publish), indexed from
  int n_vec_pub;                  // vec_offset; the worker-applied push writes both copies, the applier one per pass
  long long vec_offset;
  int shadow_is_mc;
  float* vec_dst[8];              // sharded master: fp32 publish of the 1-D variables into every replica (one multicast
  int n_vec_dst;                  // alias when shadow_is_mc); indexed from vec_offset.  0 = use vec_pub
  int mb_zero;                    // applier: zero the consumed mailbox elements (accumulating wgrad epilogues add into them)
  float* grad;                    // local flat gradient (consumed, then zeroed for the next step)
  float* loss_acc;                // local: loss accumulated by the loss kernel (consumed + zeroed)
  float* loss_out;                // last step's loss for the host to read (device or pinned host memory)
  unsigned int* done_dev;         // optional device counter: incremented per push, its value is also stored to
                                  // ((uint32*)loss_out)[1] (after the loss) so a host can spin on step completion
  const SfTensorSeg* segs;        // device array
  const int32_t* tile_map;        // device array [num_tiles * 3] = (seg, tile_row, tile_col)
  int num_tiles;
  // the same tables in kernel-parameter (constant) space when the model has <= SF_MAX_INLINE_SEGS variables:
  // no dependent global loads before the data loads can be issued
  int n_inline_segs;              // 0 = use the global tables
  int tile_prefix[SF_MAX_INLINE_SEGS + 1];
  SfTensorSeg inline_segs[SF_MAX_INLINE_SEGS];
  int optimizer;
  int lock_mode;
  int drop;                       // fault injection: consume the gradient but do not apply it
  int scope_sys;                  // 1: lock / counters use .sys scope (multi-GPU world); 0: .gpu (single GPU)
  float grad_scale;
  SfHyper h;
  // lock mode, worker-applied push that also publishes into the pushing worker's replica (shadow_dst[1], vec_pub[0]):
  // local word that receives the SF_CTRL_VERSION value this push creates, so the worker's next pull can skip its copy
  uint32_t* replica_version;
};

// control block layout (uint32 words) living in master memory
enum SfCtrl {
  SF_CTRL_LOCK = 0,         // RW lock word: [0,16) readers, bit 16 writer, [17,32) writers waiting
  SF_CTRL_VERSION = 1,      // bumped once per applied push (seqlock-style version)
  SF_CTRL_STEP = 2,         // global optimizer step count (adam beta powers)
  SF_CTRL_PUSHES = 3,       // total pushes applied
  SF_CTRL_ERRORS = 4,
  SF_CTRL_DROPPED = 5,
  SF_CTRL_PUB = 6,          // double-buffered publish: bit 31 = current buffer, [0,16) = pulls in flight (either buffer)
  SF_CTRL_WORDS = 64
};

// local_sync: 8 uint32 words in the *worker's own* memory used for in-grid coordination
int sf_push_launch(const SfPushArgs* a, uint32_t* local_sync, int grid, cudaStream_t st);

struct SfPullArgs {
  const __nv_bfloat16* src;       // master publish buffer (peer-mapped)
  __nv_bfloat16* dst;             // local replica
  const float4* src_state;        // optional: master state (element-interleaved), first 1-D variable
  float* dst_f32;                 // optional local fp32 copy of the 1-D variables (biases)
  size_t n_bf16;                  // elements (multiple of 8)
  size_t n_f32;                   // elements (multiple of 4)
  uint32_t* ctrl;                 // master control block
  uint32_t* seen_version;         // local: version observed by this pull
  int lock_mode;
  int scope_sys;
  // served push: wait until the applier has consumed this worker's last posted gradient, so a pull after a
  // push always observes the worker's own update (the reference's POST /update is synchronous)
  const uint32_t* wait_applied;   // master flag word (peer mapped) or nullptr
  const uint32_t* my_posted;      // local word holding the sequence number of my last post
  // double-buffered publish (served push, lock mode): instead of the RW lock the pull registers in SF_CTRL_PUB with
  // ONE remote atomic, learns which of the two complete publish buffers is current and copies that one; the applier
  // writes the other buffer and flips.  Pulls never wait for an update in progress and still never see a torn one.
  int dbuf;
  const __nv_bfloat16* src_alt;   // publish buffer 1 (src is buffer 0)
  const float* vec_pub[2];        // fp32 copies of the 1-D variables, one per buffer
  // lock mode: local word naming the version the replica (dst, dst_f32) already holds (SfPushArgs.replica_version).
  // While no writer holds or waits for the lock and SF_CTRL_VERSION equals it, the pull takes no lock and copies nothing.
  const uint32_t* replica_version;
};
int sf_pull_launch(const SfPullArgs* a, uint32_t* local_sync, int grid, cudaStream_t st);

// ---------------------------------------------------------------------------
// Served push ("mailbox + master-resident applier"): the worker's push kernel only streams its gradient
// into its mailbox in master memory (4 B / parameter over NVLink instead of 36 B) and posts a sequence
// number; a persistent applier kernel on the master GPU applies the mailboxes one at a time at HBM speed.
// ---------------------------------------------------------------------------
enum SfMailFlag { SF_MB_POSTED = 0, SF_MB_APPLIED = 16, SF_MB_WORDS = 32 };   // uint32 words per worker, 64 B apart

struct SfPostArgs {
  float* grad;                    // local gradient (consumed + zeroed)
  float* mailbox;                 // this worker's mailbox in master memory (peer mapped)
  uint32_t* flags;                // this worker's flag words in master memory
  float* loss_acc; float* loss_out;
  unsigned int* done_dev;         // see SfPushArgs
  size_t n;                       // floats (multiple of 4)
  int drop;                       // fault injection: consume the gradient, post nothing
};
int sf_post_launch(const SfPostArgs* a, uint32_t* local_sync, int grid, cudaStream_t st);

struct SfApplierArgs {
  SfPushArgs push;                // master-local pointers; push.grad is ignored
  float* mailboxes;               // [n_workers][mailbox_stride]
  size_t mailbox_stride;          // floats
  uint32_t* flags;                // [n_workers][SF_MB_WORDS]
  int n_workers;
  uint32_t* sync;                 // 12 words of master-local memory for the in-grid protocol (applier_kernel)
  unsigned long long idle_timeout_ns;   // listening window: a launch exits after this long without any posted mailbox
  int linger;                           // 1: keep listening after a pass (warm instruction cache / TLB for the next one: the
                                        // pass is latency bound); 0: a launch exits as soon as nothing more is posted
  int dbuf;                       // double-buffered publish: passes alternate between (push.shadow_dst[0], push.vec_pub[0])
  __nv_bfloat16* shadow_alt;      // and (shadow_alt, vec_pub_alt); SF_CTRL_PUB bit 31 names the complete one
  float* vec_pub_alt;
  int max_batch;                  // pushes fused into one pass over the state (1..8; 0 = 8)
  // ---- sharded master: this applier owns push tiles [tile_begin, tile_end) (0, 0 = all) ----
  int tile_begin, tile_end;
  uint32_t* ack[8];               // per worker: acknowledgement word of THIS shard inside the worker's own memory (peer
                                  // mapped), one per worker or none.  Given: every CTA adds 1 to the word of each consumed
                                  // worker right after its own tiles (one NVLink flush per CTA, all in parallel) - the
                                  // worker waits for posts * gridDim acknowledgements
  // seqlock stamps of this shard in every replica's publish segment (lock mode; needs ack words, ver_local and the slot
  // offsets): `begin` counts the passes STARTED (stamped by the leader before the first publish store), `end` counts CTA
  // completions (every CTA adds 1 after its own fence): the shard is quiescent iff end == begin * gridDim.
  // n_ver = 1 + ver_mc: one multimem.st reaches every replica; else one store per peer.
  uint32_t* ver_begin[8];
  uint32_t* ver_end[8];
  int n_ver;
  int ver_mc;
  const uint32_t* ver_local;      // this shard's begin stamp in the OWN replica (unicast address; survives applier restarts)
  // two publish slots per replica: pass v writes slot v & 1 = every publish destination advanced by these element
  // offsets, so a reader can always copy the newest COMPLETE pass while the next one is landing in the other slot
  long long slot_off_bf16, slot_off_f32;
  unsigned long long* stats;      // optional: [0] sum(ns decide -> tiles done), [1] sum(ns decide -> acknowledged), [2] passes, [3] pushes
};
int sf_applier_launch(const SfApplierArgs* a, unsigned int seq, int grid, cudaStream_t st);

// ---------------------------------------------------------------------------
// Sharded master, worker side.
// sync_pull: the step's "pull".  Per shard: wait until that shard's applier has acknowledged this worker's last post
// (read-your-writes, a LOCAL spin: the applier stores the acknowledgement into this worker's memory), then - lock mode -
// take a consistent snapshot of the shard's slice of the multicast-fed inbox replica into the working replica
// (seqlock; all CTAs of a shard agree on one version).  Hogwild: no copy at all, the GEMMs read the inbox in place.
// post_flags: the step's "push" epilogue.  The wgrad epilogues already stored the matrix gradients into the owners'
// mailboxes; this forwards the (tiny) 1-D tail, then publishes the post with one release store per shard.
// ---------------------------------------------------------------------------
struct SfSyncPullArgs {
  int n_shards;
  int bounds[SF_MAX_SHARDS + 1];
  const uint32_t* applied;        // local: word r * 16 = acknowledgement word of shard r for this worker
  const uint32_t* my_posted;      // local: sequence number of my last post
  int ack_grid[SF_MAX_SHARDS];    // CTAs of shard r's applier (>= 1): the word counts CTA acknowledgements
  int copy;                       // 1: snapshot inbox -> working replica
  const uint32_t* ver_begin;      // local inbox stamps: word r * ver_stride
  const uint32_t* ver_end;
  int ver_stride;
  long long slot_off_bf16, slot_off_f32;   // second publish slot (SfApplierArgs), required with copy
  const __nv_bfloat16* src;       // inbox publish buffer (local copy fed by the appliers' multicast stores)
  __nv_bfloat16* dst;             // working replica
  const float* src_vec;           // inbox fp32 copy of the 1-D tail (indexed from vec_offset)
  float* dst_vec;
  long long vec_offset;
  const SfTensorSeg* segs;        // device tables
  const int32_t* tile_map;
  int ctas_per_shard;
  uint32_t* sync;                 // local: 8 words per shard (arrivals, min version, max version, result, round)
  // optional latency accounting (%globaltimer ns): [0] = time of my last post (written by post_flags), per shard s:
  // [8 + 4s] sum(wait start - post), [9 + 4s] sum(ack seen - wait start), [10 + 4s] sum(snapshot done - ack seen), [11 + 4s] steps
  unsigned long long* stats;
};
int sf_sync_pull_launch(const SfSyncPullArgs* a, cudaStream_t st);

struct SfPostFlagsArgs {
  int n_shards;
  int bounds[SF_MAX_SHARDS + 1];
  uint32_t* posted[SF_MAX_SHARDS];   // POSTED word of this worker on every shard owner (peer mapped)
  float* mailbox[SF_MAX_SHARDS];     // this worker's mailbox on every shard owner
  float* grad;                       // local flat gradient buffer (only the 1-D tail is accumulated here)
  const long long* vec_tiles;        // device: [n_vec_tiles][3] = (push tile index, flat element offset, count <= 64)
  int n_vec_tiles;
  float* loss_acc; float* loss_out;
  unsigned int* done_dev;
  uint32_t* my_posted;               // local sequence word (incremented here)
  int drop;                          // fault injection: consume the gradient, post nothing
  long long total;                   // mailbox elements (drop + accumulate mode re-zeroes the mailboxes)
  int mb_zero;
  unsigned long long* heartbeat;     // optional: 2 words in this worker's symmetric segment (time of last post, posts)
  unsigned long long* stats;         // optional: [0] = %globaltimer of this post (see SfSyncPullArgs.stats)
  int phase;                         // 0: everything; 1: only forward the 1-D tail (runs beside the last wgrad); 2: only post
                                     // (every gradient store belongs to a COMPLETED kernel: no fence on the critical path)
};
int sf_post_flags_launch(const SfPostFlagsArgs* a, cudaStream_t st);
int sf_preload_kernels();

// host-visible lock helpers for tests (single-thread kernels)
int sf_lock_test(uint32_t* ctrl, int op, cudaStream_t st);

#ifdef __cplusplus
}
#endif
