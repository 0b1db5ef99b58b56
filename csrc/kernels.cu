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

#define SF_SMEM_ATTR(k, bytes)                                                                              \
  do {                                                                                                      \
    cudaError_t e_ = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);           \
    if (e_ != cudaSuccess) return static_cast<int>(e_);                                                     \
  } while (0)

extern "C" int sf_preload_kernels() {
  // opt-in shared memory sizes are set here too, so a plan can be CAPTURED without ever having run eagerly
  SF_SMEM_ATTR(sf::sf_gemm_kernel<32>, sf::GemmSmem<32>::kBytes); SF_SMEM_ATTR(sf::sf_gemm_kernel<64>, sf::GemmSmem<64>::kBytes);
  SF_SMEM_ATTR(sf::sf_gemm_kernel<128>, sf::GemmSmem<128>::kBytes); SF_SMEM_ATTR(sf::sf_gemm_kernel<256>, sf::GemmSmem<256>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_kernel<64, true>), sf::GemmSmem<64>::kBytes); SF_SMEM_ATTR((sf::sf_gemm_kernel<128, true>), sf::GemmSmem<128>::kBytes);
  SF_PRELOAD((sf::sf_gemm_kernel<64, true>)); SF_PRELOAD((sf::sf_gemm_kernel<128, true>));
  SF_SMEM_ATTR((sf::sf_gemm_epi_kernel<32, false, SF_EPI_FWD>), sf::GemmSmem<32>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_epi_kernel<64, false, SF_EPI_FWD>), sf::GemmSmem<64>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_epi_kernel<32, false, SF_EPI_LOSS>), sf::GemmSmem<32>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_epi_kernel<64, false, SF_EPI_LOSS>), sf::GemmSmem<64>::kBytes);
  SF_SMEM_ATTR(sf::sf_gemm_sigmoid_loss_kernel<32>, sf::GemmSmem<32>::kBytes);
  SF_SMEM_ATTR(sf::sf_gemm_sigmoid_loss_kernel<64>, sf::GemmSmem<64>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_epi_kernel<32, false, SF_EPI_DGRAD>), sf::GemmSmem<32>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_epi_kernel<64, false, SF_EPI_DGRAD>), sf::GemmSmem<64>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_epi_kernel<64, true, SF_EPI_WGRAD>), sf::GemmSmem<64>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_epi_kernel<128, true, SF_EPI_WGRAD>), sf::GemmSmem<128>::kBytes);
  SF_PRELOAD((sf::sf_gemm_epi_kernel<32, false, SF_EPI_FWD>)); SF_PRELOAD((sf::sf_gemm_epi_kernel<64, false, SF_EPI_FWD>));
  SF_PRELOAD((sf::sf_gemm_epi_kernel<32, false, SF_EPI_LOSS>)); SF_PRELOAD((sf::sf_gemm_epi_kernel<64, false, SF_EPI_LOSS>));
  SF_PRELOAD(sf::sf_gemm_sigmoid_loss_kernel<32>); SF_PRELOAD(sf::sf_gemm_sigmoid_loss_kernel<64>);
  SF_SMEM_ATTR(sf::sf_gemm_sparse_loss_kernel, sf::GemmSmem<32>::kBytes); SF_PRELOAD(sf::sf_gemm_sparse_loss_kernel);
  SF_PRELOAD((sf::sf_gemm_epi_kernel<32, false, SF_EPI_DGRAD>)); SF_PRELOAD((sf::sf_gemm_epi_kernel<64, false, SF_EPI_DGRAD>));
  SF_PRELOAD((sf::sf_gemm_epi_kernel<64, true, SF_EPI_WGRAD>)); SF_PRELOAD((sf::sf_gemm_epi_kernel<128, true, SF_EPI_WGRAD>));
  SF_SMEM_ATTR(sf::sf_gemm_pair_kernel, sf::kPairSmemBytes);
  SF_PRELOAD(sf::sf_gemm_kernel<32>); SF_PRELOAD(sf::sf_gemm_kernel<64>); SF_PRELOAD(sf::sf_gemm_kernel<128>); SF_PRELOAD(sf::sf_gemm_kernel<256>); SF_PRELOAD(sf::sf_gemm_pair_kernel);
  SF_PRELOAD(sf::gather_rows_f32_kernel); SF_PRELOAD(sf::cast_transpose_kernel<false>); SF_PRELOAD(sf::cast_transpose_kernel<true>);
  SF_PRELOAD(sf::softmax_xent_kernel); SF_PRELOAD(sf::sparse_softmax_xent_kernel); SF_PRELOAD(sf::elementwise_loss_kernel<sf::MseHead>);
  SF_PRELOAD(sf::elementwise_loss_kernel<sf::SigmoidXentHead>); SF_PRELOAD(sf::argmax_rows_kernel);
  SF_PRELOAD(sf::im2col_kernel); SF_PRELOAD(sf::col2im_kernel); SF_PRELOAD(sf::maxpool_fwd_kernel); SF_PRELOAD(sf::maxpool_bwd_kernel);
  SF_PRELOAD(sf::im2col_vec8_kernel); SF_PRELOAD(sf::col2im_vec8_kernel);
  SF_PRELOAD(sf::maxpool_gen_fwd_kernel); SF_PRELOAD(sf::maxpool_gen_bwd_kernel); SF_PRELOAD(sf::act_bwd_bias_kernel);
  // the twins of the extended activations (SfAct 4-9)
  SF_SMEM_ATTR(sf::sf_gemm_ext_kernel<32>, sf::GemmSmem<32>::kBytes); SF_SMEM_ATTR(sf::sf_gemm_ext_kernel<64>, sf::GemmSmem<64>::kBytes);
  SF_SMEM_ATTR(sf::sf_gemm_ext_kernel<128>, sf::GemmSmem<128>::kBytes); SF_SMEM_ATTR(sf::sf_gemm_ext_kernel<256>, sf::GemmSmem<256>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_epi_ext_kernel<32, SF_EPI_FWD>), sf::GemmSmem<32>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_epi_ext_kernel<64, SF_EPI_FWD>), sf::GemmSmem<64>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_epi_ext_kernel<32, SF_EPI_LOSS>), sf::GemmSmem<32>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_epi_ext_kernel<64, SF_EPI_LOSS>), sf::GemmSmem<64>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_epi_ext_kernel<32, SF_EPI_DGRAD>), sf::GemmSmem<32>::kBytes);
  SF_SMEM_ATTR((sf::sf_gemm_epi_ext_kernel<64, SF_EPI_DGRAD>), sf::GemmSmem<64>::kBytes);
  SF_SMEM_ATTR(sf::sf_gemm_pair_ext_kernel, sf::kPairSmemBytes);
  SF_PRELOAD(sf::sf_gemm_ext_kernel<32>); SF_PRELOAD(sf::sf_gemm_ext_kernel<64>); SF_PRELOAD(sf::sf_gemm_ext_kernel<128>);
  SF_PRELOAD(sf::sf_gemm_ext_kernel<256>); SF_PRELOAD(sf::sf_gemm_pair_ext_kernel);
  SF_PRELOAD((sf::sf_gemm_epi_ext_kernel<32, SF_EPI_FWD>)); SF_PRELOAD((sf::sf_gemm_epi_ext_kernel<64, SF_EPI_FWD>));
  SF_PRELOAD((sf::sf_gemm_epi_ext_kernel<32, SF_EPI_LOSS>)); SF_PRELOAD((sf::sf_gemm_epi_ext_kernel<64, SF_EPI_LOSS>));
  SF_PRELOAD((sf::sf_gemm_epi_ext_kernel<32, SF_EPI_DGRAD>)); SF_PRELOAD((sf::sf_gemm_epi_ext_kernel<64, SF_EPI_DGRAD>));
  SF_PRELOAD(sf::mse_ext_loss_kernel);
  SF_PRELOAD(sf::maxpool_bwd_ext_kernel); SF_PRELOAD(sf::maxpool_gen_bwd_ext_kernel); SF_PRELOAD(sf::act_bwd_bias_ext_kernel);
  SF_PRELOAD((sf::conv_first_fwd_kernel<5, 5, 1>)); SF_PRELOAD((sf::conv_first_wgrad_kernel<5, 5, 1>));
  SF_PRELOAD((sf::conv_first_fwd_kernel<3, 3, 1>)); SF_PRELOAD((sf::conv_first_wgrad_kernel<3, 3, 1>));
  SF_PRELOAD((sf::conv_first_fwd_kernel<3, 3, 3>)); SF_PRELOAD((sf::conv_first_wgrad_kernel<3, 3, 3>));
  SF_PRELOAD((sf::conv_first_fwd_kernel<0, 0, 0>)); SF_PRELOAD((sf::conv_first_wgrad_kernel<0, 0, 0>));
  SF_PRELOAD(sf::pull_kernel<true>); SF_PRELOAD(sf::pull_kernel<false>); SF_PRELOAD(sf::post_kernel); SF_PRELOAD(sf::lock_test_kernel);
  SF_PRELOAD(sf::sync_pull_kernel); SF_PRELOAD(sf::post_flags_kernel);
  SF_PRELOAD_OPT(push_kernel, true); SF_PRELOAD_OPT(push_kernel, false);
  SF_PRELOAD_OPT(applier_kernel, true); SF_PRELOAD_OPT(applier_kernel, false);
  return 0;
}
