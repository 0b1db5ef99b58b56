// Whole-chain GEMM kernel: one persistent launch runs the forward / dgrad / wgrad GEMMs of a dense network.
//
// Why: the flagship step is 8 dependent GEMM launches deep; each boundary costs hardware dependency latency plus a
// kernel prologue (barrier init, descriptor prefetch), and those dependent launches are exactly what host->device
// traffic stretches in the end-to-end loop.  Here the chain is ONE launch: barriers are set up once per CTA, a stage boundary is a release / acquire pair on a counter in L2.
//
// Scheduling: tiles of all GEMMs form one ticket sequence in a topological order (critical path first).  A CTA draws
// a ticket, waits until every GEMM its tile depends on is complete, runs the tile with the same thread roles as
// sf_gemm_kernel<32> (TMA producer / bias loader / two wgmma warpgroups that then run the fused training epilogues),
// and publishes it.  A waiting CTA only ever waits for lower tickets, all of which are held by running CTAs, so the
// scheme cannot deadlock whatever the grid size.
#include "sm90_ptx.cuh"
#include "sf_api.h"

namespace sf {

constexpr int kMegaBN = 32;

__device__ __forceinline__ void red_release_gpu_add(unsigned int* p, unsigned int v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__global__ void __launch_bounds__(kGemmThreads, 1)
sf_mega_kernel(const SfMegaArgs a) {
  using S = GemmSmem<kMegaBN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stage_base = smem;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::kStages * S::kStageBytes);
  uint64_t* empty_bar = full_bar + S::kStages;
  float* s_bias = reinterpret_cast<float*>(smem + S::kStages * S::kStageBytes + S::kBarBytes);
  __shared__ int s_ticket;
  __shared__ int s_begin[SF_MEGA_MAX_GEMMS + 1];

  TraceScope trace;
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tid = threadIdx.x;

  if (tid == 0) {
    for (int s = 0; s < S::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);
    }
    mbar_fence_init();
  }
  __syncthreads();
  pdl_wait();      // the chain's inputs (cast / pull) are complete; global memory is touched below
  trace.mark();
  if (tid <= a.n_gemms) s_begin[tid] = (tid < a.n_gemms) ? a.gemms[tid].tile_begin : a.total_tiles;

  uint32_t it = 0;          // k-blocks consumed so far by this CTA (every role advances it identically)
  while (true) {
    __syncthreads();        // previous tile fully retired (staged tile read, s_ticket / s_bias reusable); s_begin visible
    if (tid == 0) s_ticket = static_cast<int>(atomicAdd(a.ctr + 0, 1u));
    __syncthreads();
    const int t = s_ticket;
    if (t >= a.total_tiles) break;
    int g = 0;
    while (g + 1 < a.n_gemms && t >= s_begin[g + 1]) ++g;
    const SfMegaGemm& G = a.gemms[g];
    const int local = t - s_begin[g];
    const int n0 = (local % G.tiles_n) * kMegaBN;
    const int m0 = (local / G.tiles_n) * kBM;
    const int M = G.M, N = G.N;
    const int num_kb = (G.K + kBK - 1) / kBK;
    const SfGemmEpilogue& ep = G.ep;

    // ---- dependencies: every tile of the producing GEMMs has been published ----
    if (tid == 0) {
      for (int d = 0; d < G.n_deps; ++d) {
        const int dg = G.deps[d];
        const unsigned int need = static_cast<unsigned int>(s_begin[dg + 1] - s_begin[dg]);
        const unsigned long long t0 = sf_globaltimer();
        unsigned int spins = 0;
        while (true) {
          unsigned int v;
          asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.ctr + 2 + dg) : "memory");
          if (v >= need) break;
          if ((++spins & 0x3F) == 0 && sf_globaltimer() - t0 > 2000000000ull) sf_fail(0x600 + dg);
        }
      }
      // the producers wrote through the generic proxy; this thread's TMA loads go through the async proxy
      fence_proxy_async_global();
    }
    __syncthreads();

    if (warp == 0) {
      // ===================== TMA producer =====================
      if (lane == 0) {
        tma_prefetch_desc(&G.tmA);
        tma_prefetch_desc(&G.tmB);
        const uint64_t hintA = ep.a_evict_first ? kEvictFirst : kEvictNormal;
        for (int i = 0; i < num_kb; ++i) {
          const uint32_t gi = it + i;
          const int s = gi % S::kStages;
          const uint32_t ph = (gi / S::kStages) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1, 0x610 + s);
          uint8_t* a_dst = stage_base + s * S::kStageBytes;
          uint8_t* b_dst = a_dst + S::kABytes;
          mbar_expect_tx(&full_bar[s], S::kStageBytes);
          tma_load_2d(a_dst, &G.tmA, &full_bar[s], i * kBK, m0, hintA);
          tma_load_2d(b_dst, &G.tmB, &full_bar[s], i * kBK, n0, kEvictLast);
        }
      }
    } else if (warp < 4) {
      // ===================== bias tile =====================
      const int j = tid - 32;
      if (j < kMegaBN) s_bias[j] = (ep.bias != nullptr && n0 + j < N) ? ep.bias[n0 + j] : 0.f;
      asm volatile("bar.arrive 2, 352;" ::: "memory");
    } else {
      // ===================== wgmma main loop + epilogue =====================
      const int ct = tid - 128;
      float acc[kMegaBN / 2];
      mma_mainloop<kMegaBN, false, S::kStages, S::kStageBytes, S::kABytes>(acc, stage_base, full_bar, empty_bar, it, num_kb, ct >> 7,
                                                                           (ct & 127) == 0, 0x620);
      float* stg = reinterpret_cast<float*>(stage_base);   // every stage of this tile has been consumed
      asm volatile("bar.sync 1, 256;" ::: "memory");
      stage_acc<kMegaBN>(stg, acc, ct);
      asm volatile("bar.sync 1, 256;" ::: "memory");
      asm volatile("bar.sync 2, 352;" ::: "memory");
      if (n0 < ep.n_store_limit) epilogue_tile<kMegaBN, true>(ep, stg, s_bias, m0, n0, M, N, ct);
      // the staged tile was written through the generic proxy; the next tile's TMA loads refill the same bytes
      fence_proxy_async_smem();
    }
    it += static_cast<uint32_t>(num_kb);
    __syncthreads();        // every output store of this tile has been issued by its thread
    if (tid == 0) {
      __threadfence();
      red_release_gpu_add(a.ctr + 2 + g, 1u);
    }
  }

  if (tid == 0) {
    // the last CTA out re-arms the counters for the next launch (stream order separates the launches)
    const unsigned int prev = atomicAdd(a.ctr + 1, 1u);
    if (prev == gridDim.x - 1) {
      __threadfence();
      for (int i = 0; i < 2 + a.n_gemms; ++i) a.ctr[i] = 0u;
    }
  }
  trace.end(KID_GEMM);
}

}  // namespace sf

extern "C" int sf_mega_launch(const SfMegaArgs* a, int grid, cudaStream_t st) {
  using S = sf::GemmSmem<sf::kMegaBN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(sf::sf_mega_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kBytes);
    if (e != cudaSuccess) return static_cast<int>(e);
    attr_set = true;
  }
  if (a->n_gemms < 1 || a->n_gemms > SF_MEGA_MAX_GEMMS || a->total_tiles < 1) return -9;
  if (grid <= 0) grid = 64;           // the widest stage of the flagship is 56 tiles; leave SMs to the applier
  if (grid > a->total_tiles) grid = a->total_tiles;
  if (grid > sf_num_sms()) grid = sf_num_sms();
  return static_cast<int>(sf::launch(sf::sf_mega_kernel, dim3(grid), dim3(sf::kGemmThreads), S::kBytes, st, *a));
}
