// Unity translation unit for all device code (one copy of the sf::g_sf_error_code symbol).
#include "gemm_sm90.cu"
#include "gemm_pair_sm90.cu"
#include "elementwise.cu"
#include "optim_push.cu"
#include "conv.cu"

// Force the (lazy) load of EVERY kernel of this library up front: CUDA's lazy module loading needs a context-wide
// synchronisation the first time a kernel is used, which must never happen in the middle of a training run.
#define SF_PRELOAD(k)                                                   \
  do {                                                                  \
    cudaFuncAttributes fa;                                              \
    cudaError_t e_ = cudaFuncGetAttributes(&fa, k);                     \
    if (e_ != cudaSuccess) return static_cast<int>(e_);                 \
  } while (0)
#define SF_PRELOAD_OPT(K, SYS)                                                                          \
  SF_PRELOAD((sf::K<SF_OPT_SGD, SYS>)); SF_PRELOAD((sf::K<SF_OPT_MOMENTUM, SYS>)); SF_PRELOAD((sf::K<SF_OPT_ADAM, SYS>)); \
  SF_PRELOAD((sf::K<SF_OPT_RMSPROP, SYS>)); SF_PRELOAD((sf::K<SF_OPT_ADAGRAD, SYS>)); SF_PRELOAD((sf::K<SF_OPT_ADADELTA, SYS>)); \
  SF_PRELOAD((sf::K<SF_OPT_ADAGRAD_DA, SYS>)); SF_PRELOAD((sf::K<SF_OPT_FTRL, SYS>)); SF_PRELOAD((sf::K<SF_OPT_PROXIMAL_ADAGRAD, SYS>)); \
  SF_PRELOAD((sf::K<SF_OPT_PROXIMAL_SGD, SYS>))

#define SF_PRELOAD_SMEM(k, bytes)                                                                   \
  do {                                                                                              \
    cudaError_t e_ = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);    \
    if (e_ != cudaSuccess) return static_cast<int>(e_);                                             \
    SF_PRELOAD(k);                                                                                  \
  } while (0)
#define SF_PRELOAD_CONV1(KH, KW, CIN)                                                               \
  SF_PRELOAD_SMEM((sf::conv_first_fwd_kernel<KH, KW, CIN>), sf::kConv1MaxSmem);                     \
  SF_PRELOAD_SMEM((sf::conv_first_wgrad_kernel<KH, KW, CIN>), sf::kConv1MaxSmem)

extern "C" int sf_preload_kernels() {
  // the GEMMs' opt-in shared memory sizes are set here too, so a plan can be CAPTURED without ever having run eagerly
  if (const int rc = sf_gemm_preload()) return rc;
  SF_PRELOAD(sf::gather_rows_f32_kernel); SF_PRELOAD(sf::cast_transpose_kernel<false>); SF_PRELOAD(sf::cast_transpose_kernel<true>);
  SF_PRELOAD(sf::softmax_xent_kernel); SF_PRELOAD(sf::sparse_softmax_xent_kernel); SF_PRELOAD(sf::elementwise_loss_kernel<sf::MseHead>);
  SF_PRELOAD(sf::elementwise_loss_kernel<sf::SigmoidXentHead>); SF_PRELOAD(sf::argmax_rows_kernel);
  SF_PRELOAD(sf::im2col_kernel); SF_PRELOAD(sf::col2im_kernel); SF_PRELOAD(sf::maxpool_fwd_kernel); SF_PRELOAD(sf::maxpool_bwd_kernel);
  SF_PRELOAD(sf::im2col_vec8_kernel); SF_PRELOAD(sf::col2im_vec8_kernel);
  SF_PRELOAD(sf::maxpool_gen_fwd_kernel); SF_PRELOAD(sf::maxpool_gen_bwd_kernel); SF_PRELOAD(sf::act_bwd_bias_kernel);
  // the twins of the extended activations (SfAct 4-9)
  SF_PRELOAD(sf::mse_ext_loss_kernel);
  SF_PRELOAD(sf::maxpool_bwd_ext_kernel); SF_PRELOAD(sf::maxpool_gen_bwd_ext_kernel); SF_PRELOAD(sf::act_bwd_bias_ext_kernel);
  // the dropout twins of the pool and activation-gradient kernels (an image dropout), with and without the extended set
  SF_PRELOAD(sf::maxpool_drop_fwd_kernel); SF_PRELOAD(sf::maxpool_gen_drop_fwd_kernel);
  SF_PRELOAD(sf::maxpool_drop_bwd_kernel<false>); SF_PRELOAD(sf::maxpool_drop_bwd_kernel<true>);
  SF_PRELOAD(sf::maxpool_gen_drop_bwd_kernel<false>); SF_PRELOAD(sf::maxpool_gen_drop_bwd_kernel<true>);
  SF_PRELOAD(sf::act_drop_bwd_bias_kernel<false>); SF_PRELOAD(sf::act_drop_bwd_bias_kernel<true>);
  // the fused first conv's opt-in shared memory is a per-device setting too: every instance gets the launchers' cap
  SF_PRELOAD_CONV1(5, 5, 1); SF_PRELOAD_CONV1(3, 3, 1); SF_PRELOAD_CONV1(3, 3, 3); SF_PRELOAD_CONV1(0, 0, 0);
  SF_PRELOAD(sf::pull_kernel<true>); SF_PRELOAD(sf::pull_kernel<false>); SF_PRELOAD(sf::post_kernel); SF_PRELOAD(sf::lock_test_kernel);
  SF_PRELOAD(sf::sync_pull_kernel); SF_PRELOAD(sf::post_flags_kernel);
  SF_PRELOAD_OPT(push_kernel, true); SF_PRELOAD_OPT(push_kernel, false);
  SF_PRELOAD_OPT(applier_kernel, true); SF_PRELOAD_OPT(applier_kernel, false);
  return 0;
}
