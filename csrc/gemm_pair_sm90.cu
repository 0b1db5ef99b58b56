// Persistent cluster-pair GEMM for the large layers.
//
//   D[M,N] = alpha * A[M,K] . B[N,K]^T     same operands / epilogue contract as gemm_sm90.cu
//
// Why a second kernel: with one tile per CTA nothing overlaps a tile's epilogue with the next tile's loads, and every
// CTA fetches its own copy of the weight tile.  Here
//   * a cluster of two CTAs computes one 256 x 128 tile: each CTA owns 128 rows of A, and each loads HALF of the shared
//     128 x 64 B tile per k-block and multicasts it into both CTAs' shared memory (half the L2 -> SM traffic for B);
//   * the kernel is persistent (one CTA per SM, tiles walked in an L2-friendly grouped order), so the TMA producer
//     already streams the next tile's operands while the consumer warpgroups run the current tile's epilogue;
//   * the fp32 accumulator is staged in a region of its own, not in the operand ring the producer keeps filling.
//
// Barriers (same shared-memory offsets in both CTAs):
//   full[s]   count 1: the local producer's arrive.expect_tx of the stage's bytes (own A, both B halves).
//   empty[s]  count 4: one arrive per consumer warpgroup of BOTH CTAs - a stage is refilled by both CTAs' multicasts,
//             so it is free only when both CTAs have consumed it.
#include "sm90_ptx.cuh"
#include "sf_api.h"

namespace sf {

constexpr int kPairHalfN = kPairBN / 2;
constexpr int kPairStages = 4;
constexpr int kPairABytes = kBM * kBK * 2;          // 16 KB
constexpr int kPairBBytes = kPairBN * kBK * 2;      // 16 KB, half of it multicast by each CTA
constexpr int kPairStageBytes = kPairABytes + kPairBBytes;
constexpr int kPairStgBytes = kBM * (kPairBN + 1) * 4;
constexpr int kPairBarBytes = 256;
constexpr int kPairSmemBytes = kPairStages * kPairStageBytes + kPairStgBytes + kPairBarBytes + kPairBN * 4 + 1024;

__device__ __forceinline__ void pair_tile_coords(int t, int tiles_m, int tiles_n, int group_m, int& tm, int& tn) {
  const int per_group = group_m * tiles_n;
  const int g = t / per_group;
  const int first_m = g * group_m;
  const int gm = (tiles_m - first_m) < group_m ? (tiles_m - first_m) : group_m;
  const int r = t - g * per_group;
  tm = first_m + r % gm;
  tn = r / gm;
}

// One CTA of the pair kernel.  EXT: the extended activations (SfAct 4-9) are compiled into the epilogue.
template <bool EXT>
__device__ __forceinline__ void pair_cta(const CUtensorMap& tmA, const CUtensorMap& tmB, const SfGemmEpilogue& ep, int M, int N, int K,
                                         int tiles_m, int tiles_n, int group_m) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stage_base = smem;
  float* stg = reinterpret_cast<float*>(smem + kPairStages * kPairStageBytes);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kPairStages * kPairStageBytes + kPairStgBytes);
  uint64_t* empty_bar = full_bar + kPairStages;
  float* s_bias = reinterpret_cast<float*>(smem + kPairStages * kPairStageBytes + kPairStgBytes + kPairBarBytes);

  TraceScope trace;
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = cluster_ctarank();
  const int pair = static_cast<int>(cluster_id_x());
  const int n_pairs = static_cast<int>(cluster_nctaid_x());
  const int num_kb = (K + kBK - 1) / kBK;
  const int num_tiles = tiles_m * tiles_n;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < kPairStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);
    }
    mbar_fence_init();
  }
  cluster_sync_all();                      // both CTAs' barriers exist before any multicast or remote arrive
  pdl_wait();
  trace.mark();

  if (warp == 0) {
    // ===================== TMA producer (both CTAs) =====================
    if (lane == 0) {
      const uint64_t hintA = ep.a_evict_first ? kEvictFirst : kEvictNormal;
      const uint64_t hintB = kEvictLast;
      uint32_t it = 0;
      for (int t = pair; t < num_tiles; t += n_pairs) {
        int tm, tn;
        pair_tile_coords(t, tiles_m, tiles_n, group_m, tm, tn);
        const int m_row = tm * 2 * kBM + static_cast<int>(rank) * kBM;
        const int n_row = tn * kPairBN + static_cast<int>(rank) * kPairHalfN;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % kPairStages;
          const uint32_t ph = (it / kPairStages) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1, 0x500 + s);
          uint8_t* a_dst = stage_base + s * kPairStageBytes;
          uint8_t* b_dst = a_dst + kPairABytes + rank * (kPairHalfN * kBK * 2);
          mbar_expect_tx(&full_bar[s], kPairStageBytes);
          tma_load_2d(a_dst, &tmA, &full_bar[s], kb * kBK, m_row, hintA);
          tma_load_2d_multicast(b_dst, &tmB, &full_bar[s], kb * kBK, n_row, 0b11, hintB);
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== wgmma main loop + epilogue (rows rank * 128 .. + 128 of the pair tile) =====================
    const int ct = threadIdx.x - 128;
    uint32_t it = 0;
    for (int t = pair; t < num_tiles; t += n_pairs) {
      int tm, tn;
      pair_tile_coords(t, tiles_m, tiles_n, group_m, tm, tn);
      const int m0 = tm * 2 * kBM + static_cast<int>(rank) * kBM;
      const int n0 = tn * kPairBN;
      float acc[kPairBN / 2];
      mma_mainloop<kPairBN, false, kPairStages, kPairStageBytes, kPairABytes>(acc, stage_base, full_bar, empty_bar, it, num_kb, ct >> 7,
                                                                              (ct & 127) == 0, 0x5a0, static_cast<int>(rank ^ 1u));
      it += static_cast<uint32_t>(num_kb);
      asm volatile("bar.sync 1, 256;" ::: "memory");          // the previous tile's epilogue is done with stg / s_bias
      if (ct < kPairBN) s_bias[ct] = (ep.bias != nullptr && n0 + ct < N) ? ep.bias[n0 + ct] : 0.f;
      stage_acc<kPairBN>(stg, acc, ct);
      asm volatile("bar.sync 1, 256;" ::: "memory");
      epilogue_tile<kPairBN, kEpiPair, EXT>(ep, stg, s_bias, m0, n0, M, N, ct);
    }
  }

  __syncwarp();
  cluster_sync_all();                      // no CTA exits while its peer may still arrive on its barriers
  trace.end(KID_GEMM);
}

template <bool EXT>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kGemmThreads, 1)
sf_gemm_pair_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const SfGemmEpilogue ep,
                    int M, int N, int K, int tiles_m, int tiles_n, int group_m) {
  pair_cta<EXT>(tmA, tmB, ep, M, N, K, tiles_m, tiles_n, group_m);
}

}  // namespace sf

extern "C" int sf_gemm_pair_launch(const SfGemm* g, cudaStream_t st) {
  const bool ext = g->ep.act >= SF_ACT_ELU || g->ep.aux_act >= SF_ACT_ELU;
  const int tiles_m = (g->M + 2 * sf::kBM - 1) / (2 * sf::kBM);
  const int tiles_n = (g->N + sf::kPairBN - 1) / sf::kPairBN;
  const int tiles = tiles_m * tiles_n;
  int pairs = (g->pair_ctas > 0 ? g->pair_ctas : sf_num_sms()) / 2;
  if (pairs > tiles) pairs = tiles;
  if (pairs < 1) pairs = 1;
  // a wave of `pairs` concurrent tiles should cover a near-square block of the output: group_m tile rows at a time
  static const int env_group = [] { const char* v = getenv("SPARKFLOW_PAIR_GROUP_M"); return v ? atoi(v) : 0; }();
  int group_m = env_group > 0 ? env_group : 8;
  if (group_m > tiles_m) group_m = tiles_m;
  return static_cast<int>(sf::launch(ext ? sf::sf_gemm_pair_kernel<true> : sf::sf_gemm_pair_kernel<false>, dim3(2 * pairs),
                                     dim3(sf::kGemmThreads), sf::kPairSmemBytes, st, g->tmA, g->tmB, g->ep, g->M, g->N, g->K, tiles_m,
                                     tiles_n, group_m));
}

// Sets a GEMM kernel's opt-in shared-memory size and forces its module load
template <typename Fn>
static int preload_gemm(Fn* fn, int smem) {
  cudaFuncAttributes fa;
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, fn);
  return static_cast<int>(e);
}

// Every GEMM kernel instance: the one-CTA kernels of kGemmKernels (gemm_sm90.cu) and both pair instances.  Nothing else
// grants a GEMM its shared memory (every instance needs more than the default 48 KB), so an instance missing here fails
// its first launch.  Called by sf_preload_kernels, once per device.
static int sf_gemm_preload() {
  for (const sf::GemmKernel& k : sf::kGemmKernels)
    if (const int rc = preload_gemm(k.fn, k.smem)) return rc;
  if (const int rc = preload_gemm(sf::sf_gemm_pair_kernel<false>, sf::kPairSmemBytes)) return rc;
  return preload_gemm(sf::sf_gemm_pair_kernel<true>, sf::kPairSmemBytes);
}
