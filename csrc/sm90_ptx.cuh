// sm_90a PTX wrappers used by every sparkflow_b200 kernel.
//
// Everything here is raw inline PTX (no CUTLASS/CuTe dependency): mbarrier,
// TMA (cp.async.bulk.tensor, with cluster multicast), wgmma, cluster barriers,
// system-scope acquire/release memory operations used by the NVLink push/pull
// paths, and the NVLS multimem stores.  Bit layouts of the wgmma shared-memory
// descriptors follow the PTX ISA.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include "sf_api.h"

namespace sf {

// ---------------------------------------------------------------------------
// Error reporting for bounded spin loops.  A kernel that would otherwise hang
// (bad descriptor, lost arrive) writes a code here and traps, so the host sees
// a launch failure instead of a dead GPU.
// ---------------------------------------------------------------------------
__device__ unsigned int g_sf_error_code = 0;
__device__ unsigned int* g_sf_error_host = nullptr;     // mapped pinned host word: survives the dead context

__device__ __forceinline__ void sf_fail(unsigned int code) {
  atomicExch(&g_sf_error_code, code);
  if (g_sf_error_host != nullptr) {
    // code | blockIdx.x << 12 so the host can see WHICH bounded wait fired even though the trap kills the context
    *reinterpret_cast<volatile unsigned int*>(g_sf_error_host) = code | (blockIdx.x << 12);
  }
  __threadfence_system();
  asm volatile("trap;");
}

// ---------------------------------------------------------------------------
// Device-side timeline tracer: when enabled, thread 0 of every CTA appends
// (kernel id, block, t_entry, t_after_pdl_wait, t_exit) in %globaltimer ns.
// ---------------------------------------------------------------------------
struct TraceRec {
  unsigned long long t0, t1, t2;
  unsigned int kernel_id, block;
};
__device__ TraceRec* g_trace_buf = nullptr;
__device__ unsigned int g_trace_cap = 0;
__device__ unsigned int g_trace_n = 0;

enum KernelId { KID_GEMM = 1, KID_CAST = 2, KID_SOFTMAX = 3, KID_MSE = 4, KID_ARGMAX = 5, KID_PUSH = 6, KID_PULL = 7,
                KID_IM2COL = 8, KID_COL2IM = 9, KID_POOL_FWD = 10, KID_POOL_BWD = 11, KID_POOL_GEN_FWD = 12, KID_POOL_GEN_BWD = 13,
                KID_ACT_BWD = 14, KID_SIGMOID_XENT = 15, KID_SPARSE_SOFTMAX = 16,
                // phase stamps (ids 100 and up): one extra record of three stamps in t0 / t1 / t2
                KID_PUSH_LEAD = 106,      // push, block 0: grant seen, gradient loads returned, optimizer math done
                KID_PUSH_TAIL = 107 };    // push, last CTA: stores issued, done-counter arrival returned, tail done

__device__ __forceinline__ unsigned long long trace_now() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
struct TraceScope {
  unsigned long long t0, t1;
  bool on;
  __device__ __forceinline__ TraceScope() : t0(0), t1(0), on(false) {
    if (threadIdx.x == 0 && g_trace_buf != nullptr) {
      on = true;
      t0 = trace_now();
    }
  }
  __device__ __forceinline__ void mark() {
    if (on) t1 = trace_now();
  }
  __device__ __forceinline__ void end(unsigned int kid) {
    if (on) {
      const unsigned int i = atomicAdd(&g_trace_n, 1u);
      if (i < g_trace_cap) {
        const unsigned int b = blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z);
        g_trace_buf[i] = TraceRec{t0, t1, trace_now(), kid, b};
      }
    }
  }
  // one phase-stamp record (kid >= 100) written by the thread that holds the scope
  __device__ __forceinline__ void phases(unsigned int kid, unsigned long long a, unsigned long long b, unsigned long long c) {
    if (on) {
      const unsigned int i = atomicAdd(&g_trace_n, 1u);
      if (i < g_trace_cap) g_trace_buf[i] = TraceRec{a, b, c, kid, blockIdx.x};
    }
  }
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() {
  uint32_t l;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
  return l;
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: traps with `code` after ~2 s instead of hanging the GPU.
__device__ __forceinline__ unsigned long long sf_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, uint32_t code) {
  if (mbar_try_wait(bar, parity)) return;
  const unsigned long long t0 = sf_globaltimer();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0xFF) == 0 && sf_globaltimer() - t0 > 2000000000ull) sf_fail(code);
  }
}

// ---------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}

// L2 cache-hint policies (the createpolicy encodings of evict_normal / evict_first / evict_last).
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar,
                                            int32_t c0, int32_t c1, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)),
        "r"(c0), "r"(c1), "l"(hint)
      : "memory");
}

__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem_src,
                                             int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
      :
      : "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}


// ---------------------------------------------------------------------------
// Clusters: CTA rank, remote mbarrier arrive, cluster-wide barrier
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_id_x() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_nctaid_x() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset as `bar` in CTA `cta` of this cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t"
      ".reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(cta)
      : "memory");
}
// TMA tile load written to the same shared-memory offset in every CTA of `cta_mask`; each destination CTA's
// mbarrier at the offset of `bar` receives the bytes that landed in it
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0, int32_t c1,
                                                      uint16_t cta_mask, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5, %6;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask),
        "l"(hint)
      : "memory");
}

// ---------------------------------------------------------------------------
// wgmma: warpgroup-wide asynchronous MMA, operands in shared memory, fp32 accumulator in registers
// ---------------------------------------------------------------------------
// Shared-memory matrix descriptor, 128-byte swizzle (layout type 1).  K-major operand: rows 128 B apart, 8-row
// swizzle atoms SBO = 1024 B apart (LBO unused).  MN-major operand (the tile is K rows of 64 consecutive M / N
// elements, what a TMA box {64 elements, K rows} of a row-major [K, MN] tensor produces): 8-row k-groups are
// SBO = 1024 B apart and the next 64 MN elements are LBO bytes away.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keep the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] . B[N x 16]^T; TA / TB = 1: the operand is MN-major.  Accumulator fragment: register j of
// thread t holds row 16 * (t / 32) + (t % 32) / 4 + 8 * ((j / 2) % 2), column 8 * (j / 4) + 2 * (t % 4) + j % 2.

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n32(float (&d)[16], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n64(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n256(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}

template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  if constexpr (N == 32) wgmma_bf16_n32<TA, TB>(d, a_desc, b_desc, scale_d);
  else if constexpr (N == 64) wgmma_bf16_n64<TA, TB>(d, a_desc, b_desc, scale_d);
  else if constexpr (N == 128) wgmma_bf16_n128<TA, TB>(d, a_desc, b_desc, scale_d);
  else wgmma_bf16_n256<TA, TB>(d, a_desc, b_desc, scale_d);
}


// ---------------------------------------------------------------------------
// System-scope memory operations for the NVLink push/pull paths
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t atom_cas_acqrel_sys(uint32_t* p, uint32_t cmp, uint32_t val) {
  uint32_t old;
  asm volatile("atom.acq_rel.sys.global.cas.b32 %0, [%1], %2, %3;"
               : "=r"(old)
               : "l"(p), "r"(cmp), "r"(val)
               : "memory");
  return old;
}
__device__ __forceinline__ uint32_t atom_add_acqrel_sys(uint32_t* p, uint32_t val) {
  uint32_t old;
  asm volatile("atom.acq_rel.sys.global.add.u32 %0, [%1], %2;"
               : "=r"(old)
               : "l"(p), "r"(val)
               : "memory");
  return old;
}
__device__ __forceinline__ uint32_t atom_xor_release_sys(uint32_t* p, uint32_t val) {
  uint32_t old;
  asm volatile("atom.release.sys.global.xor.b32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(val) : "memory");
  return old;
}
__device__ __forceinline__ float ld_relaxed_sys_f32(const float* p) {
  float v;
  asm volatile("ld.global.relaxed.sys.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t atom_add_relaxed_sys(uint32_t* p, uint32_t val) {
  uint32_t old;
  asm volatile("atom.relaxed.sys.global.add.u32 %0, [%1], %2;"
               : "=r"(old)
               : "l"(p), "r"(val)
               : "memory");
  return old;
}

// Streaming 16-byte accesses (peer memory is not cached in the local L2; keep it out of L1 too).
__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.relaxed.sys.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ void st_stream_f4(float4* p, const float4& v) {
  asm volatile("st.global.relaxed.sys.L1::no_allocate.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p),
               "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ uint4 ld_stream_u4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.relaxed.sys.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ void st_stream_u4(uint4* p, const uint4& v) {
  asm volatile("st.global.relaxed.sys.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p),
               "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

// NVLS: one store, replicated by the NVSwitch into every GPU bound to the multicast object.
__device__ __forceinline__ void multimem_st_f4(float4* mc_ptr, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_ptr),
               "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void multimem_st_u4(uint4* mc_ptr, const uint4& v) {
  // bf16x2-packed payload; the switch only replicates, so the element type is irrelevant.
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_ptr),
               "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)),
               "f"(__uint_as_float(v.w))
               : "memory");
}

// Programmatic dependent launch: the next kernel's prologue (barrier init, descriptor
// prefetch) overlaps this kernel's tail; `pdl_wait` blocks until every prerequisite grid has
// completed and its memory is visible.  Both are no-ops for launches without the PDL attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// Philox4x32-10 counter-based generator (Salmon et al., SC'11): 4 x 32 random bits per (counter, key)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

// Sigmoid cross-entropy of one raw logit z against label y (tf.nn.sigmoid_cross_entropy_with_logits), shared by the
// fused-loss GEMM epilogue and the stand-alone loss kernel: returns max(z, 0) - z y + log1p(e) and sets g = sigmoid(z) - y,
// with e = exp(-|z|) <= 1 on both sides of 0.  log1pf, not log(1 + e): 1 + e rounds to 1 for |z| > 17, which would drop
// the loss of every saturated element.
__device__ __forceinline__ float sigmoid_xent_elem(float z, float y, float& g) {
  const float e = __expf(-fabsf(z));
  const float r = __fdividef(1.f, 1.f + e);
  g = (z >= 0.f ? r : e * r) - y;
  return fmaxf(z, 0.f) - z * y + log1pf(e);
}

// The extended activations (SfAct 4-9), shared by the GEMM epilogue twins and the stand-alone backward / loss kernels.
// act_ext_dact takes the derivative from the stored output a = act(z), never from z.  Softplus: 1 - exp(-a) = -expm1(-a),
// below a = 1/4 from its series (1 - exp(-a) would cancel there; the series' first omitted term is a^6 / 720 <= 1.5e-6 a),
// so the kernels need no expm1f (its slow path gave the general pool-backward kernel a stack frame).  ReLU6 passes no
// gradient at a = 0 or a = 6 (TF's Relu6Grad).
constexpr float kSeluLambda = 1.0507009873554805f;
constexpr float kSeluAlpha = 1.6732632423543772f;
__device__ __forceinline__ float act_ext_fwd(float x, int act, float alpha) {
  switch (act) {
    case SF_ACT_ELU: return x > 0.f ? x : expm1f(x);
    case SF_ACT_SELU: return kSeluLambda * (x > 0.f ? x : kSeluAlpha * expm1f(x));
    case SF_ACT_SOFTPLUS: return fmaxf(x, 0.f) + log1pf(__expf(-fabsf(x)));
    case SF_ACT_SOFTSIGN: return __fdividef(x, 1.f + fabsf(x));
    case SF_ACT_LEAKY_RELU: return x > 0.f ? x : alpha * x;
    case SF_ACT_RELU6: return fminf(fmaxf(x, 0.f), 6.f);
    default: return x;
  }
}
__device__ __forceinline__ float act_ext_dact(float a, int act, float alpha) {
  switch (act) {
    case SF_ACT_ELU: return a > 0.f ? 1.f : a + 1.f;
    case SF_ACT_SELU: return a > 0.f ? kSeluLambda : a + kSeluLambda * kSeluAlpha;
    case SF_ACT_SOFTPLUS:
      if (a < 0.25f) return a * (1.f - a * (0.5f - a * (1.f / 6.f - a * (1.f / 24.f - a * (1.f / 120.f)))));
      return 1.f - __expf(-a);
    case SF_ACT_SOFTSIGN: {
      const float t = 1.f - fabsf(a);
      return t * t;
    }
    case SF_ACT_LEAKY_RELU: return a > 0.f ? 1.f : alpha;
    case SF_ACT_RELU6: return (a > 0.f && a < 6.f) ? 1.f : 0.f;
    default: return 1.f;
  }
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

// Host-side launch helper: every kernel of the step is launched with the programmatic stream
// serialization attribute (unless disabled), which stream capture turns into programmatic graph edges.
inline int& pdl_enabled() {
  static int v = 1;
  return v;
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                          Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace sf
