// Fused parameter-server push / pull for sm_90a.
//
// push  (reference: POST /update -> optimizer.apply_gradients, one optimizer step PER PUSH,
//        sparkflow/HogwildSparkModel.py:219-242): the *worker* launches this kernel.  It streams
//        its local gradient, loads the master's p / slot tiles through peer-mapped NVLink
//        addresses, applies the optimizer rule in registers, stores p / slots back to the master
//        and publishes the bf16 copies (row-major and transposed, i.e. both K-major GEMM operand
//        layouts) to the master and - through an NVLS multicast alias or explicit peer stores -
//        to the replicas.  No NCCL, no host, no master-side SMs.
//        Hogwild (acquire_lock=False): no lock, racing read-modify-writes over NVLink.
//        Lock mode: device writer-priority RW lock (mirror of sparkflow/RWLock.py semantics) held
//        in the master's control block, taken by CTA 0 and released by the last CTA to finish.
// pull  (reference: GET /parameters): copies the master's bf16 publish buffer (and optionally the
//        fp32 params) into the local replica under the read side of the same lock.  A locked worker-applied push
//        also publishes into the pushing worker's replica, so its next pull copies nothing while no other push
//        came in between (replica_is_current).
//
// All ten TF-1.x optimizers of tensorflow_async.py:19-30 are implemented as update functors.
#include "sm90_ptx.cuh"
#include "sf_api.h"

namespace sf {

constexpr uint32_t kLockWriter = 1u << 16;
constexpr uint32_t kLockWaitOne = 1u << 17;
constexpr uint32_t kLockReaders = 0xFFFFu;
constexpr unsigned long long kLockTimeoutNs = 20ull * 1000 * 1000 * 1000;  // 20 s
constexpr unsigned long long kStaleReaderNs = 2ull * 1000 * 1000 * 1000;   // 2 s: a registered pull that never finishes is dead

__device__ __forceinline__ unsigned long long gtime_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---- writer-priority readers/writer lock on one 32-bit word -------------------------------------
// Scope: .sys when more than one GPU shares the master (NVLink peers), .gpu for a single-GPU world
// (every participant must use the same scope for the operations to be morally strong).
// Uncontended acquires are ONE atomic round trip (optimistic add / cas); the slow paths keep the
// writer-priority contract of the reference lock: a waiting writer blocks new readers.
template <bool SYS> __device__ __forceinline__ uint32_t lk_ld_acquire(const uint32_t* p) {
  uint32_t v;
  if (SYS) asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  else asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
template <bool SYS> __device__ __forceinline__ uint32_t lk_add_acquire(uint32_t* p, uint32_t x) {
  uint32_t old;
  if (SYS) asm volatile("atom.acquire.sys.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(x) : "memory");
  else asm volatile("atom.acquire.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(x) : "memory");
  return old;
}
template <bool SYS> __device__ __forceinline__ uint32_t lk_add_release(uint32_t* p, uint32_t x) {
  uint32_t old;
  if (SYS) asm volatile("atom.release.sys.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(x) : "memory");
  else asm volatile("atom.release.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(x) : "memory");
  return old;
}
template <bool SYS> __device__ __forceinline__ uint32_t lk_add_relaxed(uint32_t* p, uint32_t x) {
  uint32_t old;
  if (SYS) asm volatile("atom.relaxed.sys.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(x) : "memory");
  else asm volatile("atom.relaxed.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(x) : "memory");
  return old;
}
// fire-and-forget counter bump (no return value -> no NVLink round trip on the critical path)
template <bool SYS> __device__ __forceinline__ void lk_red_relaxed(uint32_t* p, uint32_t x) {
  if (SYS) asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(x) : "memory");
  else asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(x) : "memory");
}
template <bool SYS> __device__ __forceinline__ void lk_red_release(uint32_t* p, uint32_t x) {
  if (SYS) asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(x) : "memory");
  else asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(x) : "memory");
}
template <bool SYS> __device__ __forceinline__ uint32_t lk_cas_acquire(uint32_t* p, uint32_t cmp, uint32_t val) {
  uint32_t old;
  if (SYS) asm volatile("atom.acquire.sys.global.cas.b32 %0, [%1], %2, %3;" : "=r"(old) : "l"(p), "r"(cmp), "r"(val) : "memory");
  else asm volatile("atom.acquire.gpu.global.cas.b32 %0, [%1], %2, %3;" : "=r"(old) : "l"(p), "r"(cmp), "r"(val) : "memory");
  return old;
}

template <bool SYS> __device__ void rw_acquire_write(uint32_t* lock) {
  if (lk_cas_acquire<SYS>(lock, 0u, kLockWriter) == 0u) return;          // uncontended: one round trip
  lk_add_relaxed<SYS>(lock, kLockWaitOne);                               // announce: blocks new readers
  const unsigned long long t0 = gtime_ns();
  while (true) {
    const uint32_t v = lk_ld_acquire<SYS>(lock);
    if ((v & (kLockReaders | kLockWriter)) == 0) {
      if (lk_cas_acquire<SYS>(lock, v, v - kLockWaitOne + kLockWriter) == v) return;
    } else {
      __nanosleep(32);
    }
    if (gtime_ns() - t0 > kLockTimeoutNs) sf_fail(0x401);
  }
}
template <bool SYS> __device__ void rw_release_write(uint32_t* lock) { lk_red_release<SYS>(lock, 0u - kLockWriter); }
template <bool SYS> __device__ void rw_acquire_read(uint32_t* lock) {
  const unsigned long long t0 = gtime_ns();
  while (true) {
    const uint32_t old = lk_add_acquire<SYS>(lock, 1u);                 // optimistic: register as a reader
    if ((old & kLockWriter) == 0 && (old >> 17) == 0) return;            // no writer active, none waiting
    lk_add_relaxed<SYS>(lock, 0u - 1u);                                  // back out and wait our turn
    while (true) {
      const uint32_t v = lk_ld_acquire<SYS>(lock);
      if ((v & kLockWriter) == 0 && (v >> 17) == 0) break;
      __nanosleep(32);
      if (gtime_ns() - t0 > kLockTimeoutNs) sf_fail(0x402);
    }
  }
}
template <bool SYS> __device__ void rw_release_read(uint32_t* lock) { lk_red_release<SYS>(lock, 0u - 1u); }

// Does a locked pull's snapshot equal what the replica already holds?  `mine` is the SF_CTRL_VERSION value the worker's
// own last push created (its push publishes into the replica too); `ver` receives the version read.
// Seqlock-style read with the lock word as the sequence: the lock word first, then the version, both acquire.
//  - Every writer bumps SF_CTRL_VERSION before its release of the write bit, and every later change of the lock word is
//    an atomic RMW, so an acquire load of the lock word that reads any value coherence-after a writer's release
//    synchronizes with it: the version load that follows sees that writer's bump.  A version equal to `mine` therefore
//    means no push was applied after the worker's own one and before the lock word was read.
//  - Only the writer that set bit 16 clears it, so a lock word without it (and without waiting writers) means no push
//    was in progress when it was read.
// Together: at the instant the lock word was read the publish buffer held exactly the worker's own last push, i.e. the
// replica.  A writer that takes the lock after that instant is ordered after this pull, as it would be had the pull
// taken the read lock first; a second read of the lock word after the version would only reject such writers.
template <bool SYS> __device__ __forceinline__ bool replica_is_current(uint32_t* ctrl, uint32_t mine, uint32_t& ver) {
  if ((lk_ld_acquire<SYS>(ctrl + SF_CTRL_LOCK) & ~kLockReaders) != 0u) return false;      // a writer holds or awaits the lock
  ver = lk_ld_acquire<SYS>(ctrl + SF_CTRL_VERSION);
  return ver == mine;
}

// ---- in-grid coordination on the worker's own memory --------------------------------------
// local_sync words: 0 = grant epoch, 1 = granted value (optimizer step t), 2 = done counter,
//                   3 = launch counter, 5 = (push) the version the push creates when it publishes into the worker's
//                   replica, 6 = (push) count of pushes whose early tuple loads were stale (push_grant).
//                   All CTAs of the grid must be co-resident (grid <= #SMs).
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// The launch counter (word 3) of a locked push / pull is read RELAXED: the previous launch that wrote it completed before
// this grid started, and this launch's last CTA rewrites it only after every CTA's release-ordered arrival on the done
// counter.  A relaxed load does not hold back the lock / version round trip that follows it, so the two overlap.
__device__ __forceinline__ uint32_t ld_launch_epoch(const uint32_t* local_sync) {
  uint32_t v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(local_sync + 3) : "memory");
  return v;
}
// Arrival on the done counter (word 2): release for this CTA's stores (bar.sync makes it cumulative over the CTA), acquire
// for the last CTA, which then sees every CTA's stores without a second round trip.
__device__ __forceinline__ uint32_t arrive_done(uint32_t* local_sync) {
  uint32_t old;
  asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(old) : "l"(local_sync + 2) : "memory");
  return old;
}

// Locked push with a replica_version word: the grant and the first tile's master-tuple loads run BEFORE the
// programmatic-dependency wait (under the predecessor's tail: the push pre-launches once the last weight-gradient GEMM
// has passed its main loop); only the gradient, the loss words and what the tuples feed wait for it.  Block 0 reads
// SF_CTRL_VERSION under the write lock; the early tuple loads are used when it equals the replica_version `mine` of the
// worker's own last push, and reloaded after the wait otherwise (the first push, `mine` = -1; after another worker's push
// or a host write of the master state).  Why a match means the early loads saw the current state:
//  - The tuple loads are performed before the worker's previous push could still store: that push completed before this
//    grid started (the same premise as ld_launch_epoch: kernels of a step plan let their successor launch only after
//    their own wait, and steps are separate launches).  Every CTA's tuple loads are consumed before its release-ordered
//    arrival on the done counter, and the last arrival precedes the lock release, so a writer that takes the lock after
//    this push cannot affect them.
//  - VERSION == mine, read under the write lock, means no push was applied between the worker's own last push and this
//    acquire: every applied push (worker-applied or applier) bumps VERSION before it releases the write bit, and this
//    acquire synchronizes with that release; a dropped push writes no state, and host writes of the master state bump
//    VERSION themselves (MasterState.load_weights / load_slots).  A writer whose stores overlapped the early loads released
//    the lock before this acquire, so its bump is seen and the tuples are reloaded.
//  - No new deadlock: the lock is now held while the kernel waits for its predecessor, the last weight-gradient GEMM.
//    By then the graph has completed every other dependency of the push, and that GEMM's CTAs are resident (one wave: it
//    lets the push launch only after its main loop), so it completes without this push.  Without programmatic launch the
//    wait returns at once and the order is the plain one.
// The lock is held for at most the predecessor's remaining epilogue longer; the part of the push after the wait gets
// shorter by about as much.
template <bool SYS>
__device__ __forceinline__ void push_grant(const SfPushArgs& a, uint32_t* local_sync, bool early, uint32_t* s_t, uint32_t* s_epoch,
                                           uint32_t* s_valid) {
  if (threadIdx.x == 0) {
    const uint32_t mine = early ? *a.replica_version : 0u;
    const uint32_t epoch = ld_launch_epoch(local_sync);
    uint32_t t, ver = 0;
    if (blockIdx.x == 0) {
      rw_acquire_write<SYS>(a.ctrl + SF_CTRL_LOCK);
      t = ld_relaxed_sys(a.ctrl + SF_CTRL_STEP) + 1;
      if (early) local_sync[5] = ver = ld_relaxed_sys(a.ctrl + SF_CTRL_VERSION) + 1;     // this push's version
      local_sync[1] = t;
      st_release_gpu(local_sync + 0, epoch + 1);
    } else {
      const unsigned long long t0 = gtime_ns();
      while (ld_acquire_gpu(local_sync + 0) != epoch + 1) {
        if (early) __nanosleep(32);      // before the wait the poll shares the SM with the predecessor's epilogue
        if (gtime_ns() - t0 > kLockTimeoutNs) sf_fail(0x403);
      }
      t = local_sync[1];
      if (early) ver = local_sync[5];
    }
    *s_epoch = epoch;
    *s_t = t;
    *s_valid = early && ver - 1u == mine;
  }
  __syncthreads();
}

// ---- optimizer rules (TF 1.x training_ops semantics) ---------------------------------------
struct Upd {
  float p, s0, s1, s2;
};

__device__ __forceinline__ float sgnf(float x) { return (x > 0.f) - (x < 0.f); }

template <int OPT>
__device__ __forceinline__ void apply_rule(Upd& u, float g, const SfHyper& h, float t, float lr_t) {
  if constexpr (OPT == SF_OPT_SGD) {
    u.p -= h.lr * g;
  } else if constexpr (OPT == SF_OPT_MOMENTUM) {
    u.s0 = h.momentum * u.s0 + g;
    u.p -= h.nesterov ? (h.lr * g + h.lr * h.momentum * u.s0) : (h.lr * u.s0);
  } else if constexpr (OPT == SF_OPT_ADAM) {
    u.s0 = h.beta1 * u.s0 + (1.f - h.beta1) * g;
    u.s1 = h.beta2 * u.s1 + (1.f - h.beta2) * g * g;
    u.p -= __fdividef(lr_t * u.s0, __fsqrt_rn(u.s1) + h.eps);
  } else if constexpr (OPT == SF_OPT_RMSPROP) {
    u.s0 = h.decay * u.s0 + (1.f - h.decay) * g * g;            // ms
    float denom = u.s0 + h.eps;
    if (h.centered) {
      u.s2 = h.decay * u.s2 + (1.f - h.decay) * g;              // mg
      denom -= u.s2 * u.s2;
    }
    u.s1 = h.momentum * u.s1 + h.lr * g * rsqrtf(denom);        // mom
    u.p -= u.s1;
  } else if constexpr (OPT == SF_OPT_ADAGRAD) {
    u.s0 += g * g;
    u.p -= h.lr * g * rsqrtf(u.s0);
  } else if constexpr (OPT == SF_OPT_ADADELTA) {
    u.s0 = h.rho * u.s0 + (1.f - h.rho) * g * g;
    const float upd = sqrtf(u.s1 + h.eps) * rsqrtf(u.s0 + h.eps) * g;
    u.s1 = h.rho * u.s1 + (1.f - h.rho) * upd * upd;
    u.p -= h.lr * upd;
  } else if constexpr (OPT == SF_OPT_ADAGRAD_DA) {
    u.s0 += g;                                                  // gradient accumulator
    u.s1 += g * g;                                              // squared accumulator
    float tmp = u.s0;
    if (h.l1 > 0.f) tmp = sgnf(u.s0) * fmaxf(fabsf(u.s0) - h.l1 * t, 0.f);
    u.p = (-h.lr * tmp) / (h.l2 * t * h.lr + sqrtf(u.s1));
  } else if constexpr (OPT == SF_OPT_FTRL) {
    const float gs = g + 2.f * h.l2_shrinkage * u.p;
    const float acc_new = u.s0 + g * g;
    float pow_new, pow_old;
    if (h.lr_power == -0.5f) {
      pow_new = sqrtf(acc_new);
      pow_old = sqrtf(u.s0);
    } else {
      pow_new = __powf(acc_new, -h.lr_power);
      pow_old = __powf(u.s0, -h.lr_power);
    }
    const float sigma = (pow_new - pow_old) / h.lr;
    u.s1 += gs - sigma * u.p;                                   // linear
    const float quad = pow_new / h.lr + 2.f * h.l2;
    u.p = fabsf(u.s1) > h.l1 ? (sgnf(u.s1) * h.l1 - u.s1) / quad : 0.f;
    u.s0 = acc_new;
  } else if constexpr (OPT == SF_OPT_PROXIMAL_ADAGRAD) {
    u.s0 += g * g;
    const float lr_a = h.lr * rsqrtf(u.s0);
    const float prox = u.p - lr_a * g;
    u.p = (h.l1 > 0.f ? sgnf(prox) * fmaxf(fabsf(prox) - lr_a * h.l1, 0.f) : prox) / (1.f + h.l2 * lr_a);
  } else if constexpr (OPT == SF_OPT_PROXIMAL_SGD) {
    const float prox = u.p - h.lr * g;
    u.p = (h.l1 > 0.f ? sgnf(prox) * fmaxf(fabsf(prox) - h.lr * h.l1, 0.f) : prox) / (1.f + h.l2 * h.lr);
  }
}

template <int OPT> struct Slots { static constexpr int n = 0; };
template <> struct Slots<SF_OPT_MOMENTUM> { static constexpr int n = 1; };
template <> struct Slots<SF_OPT_ADAM> { static constexpr int n = 2; };
template <> struct Slots<SF_OPT_RMSPROP> { static constexpr int n = 3; };
template <> struct Slots<SF_OPT_ADAGRAD> { static constexpr int n = 1; };
template <> struct Slots<SF_OPT_ADADELTA> { static constexpr int n = 2; };
template <> struct Slots<SF_OPT_ADAGRAD_DA> { static constexpr int n = 2; };
template <> struct Slots<SF_OPT_FTRL> { static constexpr int n = 2; };
template <> struct Slots<SF_OPT_PROXIMAL_ADAGRAD> { static constexpr int n = 1; };

// weak (non-atomic) 16-byte streaming accesses: L1 is invalidated at launch boundaries and every element is
// touched once per kernel, so no stronger ordering than the end-of-push release is needed.
__device__ __forceinline__ float4 ld_weak_f4(const float* p) {
  float4 r;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_weak_f4(float* p, float a, float b, float c, float d) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

constexpr int kTileR = 32;
constexpr int kTileC = 64;
constexpr int kPushThreads = 256;

__device__ __forceinline__ void st_shadow8(__nv_bfloat16* dst, uint2 q, bool mc) {
  if (mc) {
    asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" ::"l"(dst),
                 "f"(__uint_as_float(q.x)), "f"(__uint_as_float(q.y))
                 : "memory");
  } else {
    asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1, %2};" ::"l"(dst), "r"(q.x),
                 "r"(q.y)
                 : "memory");
  }
}
__device__ __forceinline__ void st_vec_f32(float* dst, float v, bool mc) {
  if (mc) asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(dst), "f"(v) : "memory");
  else asm volatile("st.global.relaxed.sys.f32 [%0], %1;" ::"l"(dst), "f"(v) : "memory");
}
__device__ __forceinline__ void st_u32_pub(uint32_t* dst, uint32_t v, bool mc) {
  if (mc) asm volatile("multimem.st.relaxed.sys.global.u32 [%0], %1;" ::"l"(dst), "r"(v) : "memory");
  else asm volatile("st.global.relaxed.sys.u32 [%0], %1;" ::"l"(dst), "r"(v) : "memory");
}
__device__ __forceinline__ void st_shadow16(__nv_bfloat16* dst, uint4 q, bool mc) {
  if (mc) multimem_st_u4(reinterpret_cast<uint4*>(dst), q);
  else asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "r"(q.x), "r"(q.y), "r"(q.z), "r"(q.w) : "memory");
}
// One 32x64 parameter tile: load the master tuples ONCE, then apply `n_grads` pushes to them back to back in
// registers (push k uses step number t+k and its own bias-corrected rate: bit-for-bit the result of n_grads
// separate optimizer steps, one per push, in that order), store the tuples back, publish bf16 W / W^T.
// Shared by the worker-side push kernel (n_grads = 1, master tuples over NVLink, ZERO: the consumed gradient is
// cleared for the next step's accumulating epilogues) and the master-resident applier (gradients from up to 8
// worker mailboxes: state traffic and publish are paid once per batch instead of once per push).
// `pub0` / `vec0`: publish targets standing in for a.shadow_dst[0] / a.vec_pub[0] (the applier alternates buffers).
// HALVES: half-rows per thread (2: 256 threads per tile, 1: 512 threads per tile - the applier: a pass is bound by the
// per-thread instruction chain, not by memory, so it spreads the tile over twice the warps)
// Everything one thread holds for one tile between "loads issued" and "apply": the applier keeps TWO of these alive
// (software pipeline: the next tile's tuples and first gradient are in flight while the current tile is applied).
template <int HALVES>
struct TileRegs {
  SfTensorSeg sg;
  int r0, c0, c;
  bool vec;
  int nv[HALVES];
  int64_t e[HALVES];
  float g[HALVES][4];
  Upd u[HALVES][4];
};

__device__ __forceinline__ void tile_load_grad(const float* grad, int64_t e, int nv, bool vec, float (&g)[4]) {
  g[0] = g[1] = g[2] = g[3] = 0.f;
  if (nv == 0) return;
  if (vec) {
    const float4 gv = *reinterpret_cast<const float4*>(grad + e);
    g[0] = gv.x; g[1] = gv.y; g[2] = gv.z; g[3] = gv.w;
  } else {
    // compile-time indices only: a runtime-bounded loop here would index g[] dynamically and push the whole tile
    // state (gradient, tuples, geometry) into local memory
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (j < nv) g[j] = grad[e + j];
  }
}

// the master-tuple loads of one half-row (geometry already in T)
template <int HALVES>
__device__ __forceinline__ void tile_load_state(const SfPushArgs& a, TileRegs<HALVES>& T, int half) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!a.drop && j < T.nv[half]) v = ld_weak_f4(reinterpret_cast<const float*>(a.state + T.e[half] + j));
    T.u[half][j] = Upd{v.x, v.y, v.z, v.w};
  }
}
// ZERO: the gradient of one half-row is consumed: zero it for the next step's accumulating epilogues
template <bool ZERO, int HALVES>
__device__ __forceinline__ void tile_clear_grad(float* grad0, TileRegs<HALVES>& T, int half) {
  if (ZERO && T.nv[half] > 0) {
    if (T.vec) {
      *reinterpret_cast<float4*>(grad0 + T.e[half]) = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (j < T.nv[half]) grad0[T.e[half] + j] = 0.f;
    }
  }
}

// the tile's geometry: segment, origin and the thread's half-rows
template <int HALVES>
__device__ __forceinline__ void push_tile_geometry(const SfPushArgs& a, int tile, TileRegs<HALVES>& T) {
  const int tid = threadIdx.x;
  if (a.n_inline_segs > 0) {                         // tables live in constant (parameter) space
    int si = 0;
    while (si + 1 < a.n_inline_segs && tile >= a.tile_prefix[si + 1]) ++si;
    T.sg = a.inline_segs[si];
    const int local = tile - a.tile_prefix[si];
    const int tiles_c = (T.sg.cols + kTileC - 1) / kTileC;
    T.r0 = (local / tiles_c) * kTileR;
    T.c0 = (local % tiles_c) * kTileC;
  } else {
    const int seg_i = a.tile_map[tile * 3 + 0];
    T.r0 = a.tile_map[tile * 3 + 1] * kTileR;
    T.c0 = a.tile_map[tile * 3 + 2] * kTileC;
    T.sg = a.segs[seg_i];
  }
  const SfTensorSeg& sg = T.sg;
  T.vec = ((sg.cols & 3) == 0) && ((sg.offset & 3) == 0);
  const int tx = tid & 15, ty = tid >> 4;
  T.c = T.c0 + tx * 4;
#pragma unroll
  for (int half = 0; half < HALVES; ++half) {
    const int r = T.r0 + ty + 16 * half;
    T.nv[half] = (r < sg.rows && T.c < sg.cols) ? ((sg.cols - T.c) >= 4 ? 4 : (sg.cols - T.c)) : 0;
    T.e[half] = sg.offset + static_cast<int64_t>(r) * sg.cols + T.c;
  }
}

// phase 1a of a tile: geometry + the master-tuple loads.  Nothing here depends on the pushing step's results.
template <int HALVES>
__device__ __forceinline__ void push_tile_state(const SfPushArgs& a, int tile, TileRegs<HALVES>& T) {
  push_tile_geometry(a, tile, T);
#pragma unroll
  for (int half = 0; half < HALVES; ++half) tile_load_state(a, T, half);
}

// phase 1b of a tile: the first gradient's loads and (ZERO) its clear
template <bool ZERO, int HALVES>
__device__ __forceinline__ void push_tile_grad(float* grad0, TileRegs<HALVES>& T) {
#pragma unroll
  for (int half = 0; half < HALVES; ++half) {
    tile_load_grad(grad0, T.e[half], T.nv[half], T.vec, T.g[half]);
    tile_clear_grad<ZERO>(grad0, T, half);
  }
}

// phase 1 of a tile: geometry + every load of the thread's half-rows (tuples and the first gradient), nothing consumed yet
template <bool ZERO, int HALVES>
__device__ __forceinline__ void push_tile_load(const SfPushArgs& a, float* grad0, int tile, TileRegs<HALVES>& T) {
  push_tile_geometry(a, tile, T);
#pragma unroll
  for (int half = 0; half < HALVES; ++half) {
    tile_load_grad(grad0, T.e[half], T.nv[half], T.vec, T.g[half]);
    tile_load_state(a, T, half);
    tile_clear_grad<ZERO>(grad0, T, half);
  }
}

// phases 2 + 3 of a tile: n_grads optimizer steps in registers, then the tuple stores and the bf16 / fp32 publish
template <int OPT, bool ZERO, int HALVES>
__device__ __forceinline__ void push_tile_apply(const SfPushArgs& a, float* const* grads, int n_grads, TileRegs<HALVES>& T,
                                                const uint32_t* s_t_ptr, bool sync_for_t, __nv_bfloat16 (*s_tr)[kTileR + 8],
                                                __nv_bfloat16* pub0, float* vec0, unsigned long long* tp, long long off_bf16,
                                                long long off_f32) {
  constexpr int NS = Slots<OPT>::n;
  const int tid = threadIdx.x;
  const bool mc = a.shadow_is_mc != 0;
  const SfTensorSeg& sg = T.sg;
  const int tx = tid & 15, ty = tid >> 4;
  const int r0 = T.r0, c0 = T.c0, c = T.c;
  // ---- step number: under the lock it was granted above; Hogwild read it at kernel entry ----
  if (sync_for_t) __syncthreads();     // the step count was written to shared memory by thread 0
  const float t0 = static_cast<float>(*s_t_ptr);
  // ---- phase 2: n_grads optimizer steps in registers (the next push's gradient is in flight meanwhile) ----
  if (!a.drop) {
    for (int k = 0; k < n_grads; ++k) {
      float gn[HALVES][4];
      if (k + 1 < n_grads) {
#pragma unroll
        for (int half = 0; half < HALVES; ++half) tile_load_grad(grads[k + 1], T.e[half], T.nv[half], T.vec, gn[half]);
      }
      const float t = t0 + static_cast<float>(k);
      float lr_t = a.h.lr;
      if constexpr (OPT == SF_OPT_ADAM) {
        lr_t = a.h.lr * sqrtf(1.f - __powf(a.h.beta2, t)) / (1.f - __powf(a.h.beta1, t));
      }
#pragma unroll
      for (int half = 0; half < HALVES; ++half)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (j < T.nv[half]) apply_rule<OPT>(T.u[half][j], T.g[half][j] * a.grad_scale, a.h, t, lr_t);
      if (k + 1 < n_grads) {
#pragma unroll
        for (int half = 0; half < HALVES; ++half)
#pragma unroll
          for (int j = 0; j < 4; ++j) T.g[half][j] = gn[half][j];
      }
    }
  }
  if (a.mb_zero) {
    // accumulating wgrad epilogues (split-K conv) add into the mailbox: hand it back zeroed
    for (int k = 0; k < n_grads; ++k)
#pragma unroll
      for (int half = 0; half < HALVES; ++half) {
        if (T.nv[half] == 0) continue;
        if (T.vec) {
          *reinterpret_cast<float4*>(grads[k] + T.e[half]) = make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (j < T.nv[half]) grads[k][T.e[half] + j] = 0.f;
        }
      }
  }
  if (tp != nullptr) tp[1] = gtime_ns() + static_cast<unsigned long long>(T.u[0][0].p == 12345.678f);      // optimizer math done (loads consumed)
  // ---- phase 3: stores ----
#pragma unroll
  for (int half = 0; half < HALVES; ++half) {
    const int rl = ty + 16 * half;
    const int r = r0 + rl;
    float w[4] = {0.f, 0.f, 0.f, 0.f};
    if (T.nv[half] > 0 && !a.drop) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (j < T.nv[half]) {
          const Upd& q = T.u[half][j];
          w[j] = q.p;
          float* dst = reinterpret_cast<float*>(a.state + T.e[half] + j);
          st_weak_f4(dst, q.p, NS >= 1 ? q.s0 : 0.f, NS >= 2 ? q.s1 : 0.f, NS >= 3 ? q.s2 : 0.f);
          if (a.n_vec_dst > 0) {                                      // sharded master: every replica's fp32 tail
            if (T.e[half] + j >= a.vec_offset) {
              const long long vi = T.e[half] + j - a.vec_offset;
              for (int d = 0; d < a.n_vec_dst; ++d) st_vec_f32(a.vec_dst[d] + off_f32 + vi, q.p, mc);
            }
          } else if (a.n_vec_pub > 0 && T.e[half] + j >= a.vec_offset) {       // 1-D variables: fp32 publish copy / copies
            const long long vi = T.e[half] + j - a.vec_offset;
            vec0[vi] = q.p;
            if (a.n_vec_pub > 1) a.vec_pub[1][vi] = q.p;
          }
        }
      }
      // row-major bf16 publish: [rows, w_ld]; w_ld is a multiple of 8 and c of 4, pads carry zeros
      if (sg.w_off >= 0) {
        const int64_t wo = sg.w_off + static_cast<int64_t>(r) * sg.w_ld + c;
        const uint2 q = make_uint2(pack_bf16x2(w[0], w[1]), pack_bf16x2(w[2], w[3]));
        for (int d = 0; d < a.n_shadow_dst; ++d) st_shadow8((d == 0 ? pub0 : a.shadow_dst[d] + off_bf16) + wo, q, mc && d == 0);
      }
    }
    if (sg.wt_off >= 0 && !a.drop) {
#pragma unroll
      for (int j = 0; j < 4; ++j) s_tr[tx * 4 + j][rl] = __float2bfloat16(w[j]);
    }
  }
  if (tp != nullptr) tp[2] = gtime_ns();      // state + row-major publish stores issued
  if (sg.wt_off >= 0 && !a.drop) {
    __syncthreads();
    // transposed bf16 publish: [cols, wt_ld]; each thread owns 8 consecutive rows of one column
    const int cl = tid >> 2, part = tid & 3;
    const int cc = c0 + cl, rr = r0 + part * 8;
    if (cl < kTileC && cc < sg.cols && rr < sg.rows) {
      const int64_t to = sg.wt_off + static_cast<int64_t>(cc) * sg.wt_ld + rr;
      const uint4 q = *reinterpret_cast<const uint4*>(&s_tr[cl][part * 8]);
      for (int d = 0; d < a.n_shadow_dst; ++d) st_shadow16((d == 0 ? pub0 : a.shadow_dst[d] + off_bf16) + to, q, mc && d == 0);
    }
    __syncthreads();
  }
}

// A run of tiles on one CTA with the NEXT tile's loads in flight while the current one is applied (the applier of a big
// shard: ~60 tiles per CTA; without this every tile pays a full HBM round trip with nothing else outstanding).  With at
// most one tile per CTA it is the plain sequence: load the tile, apply it.
template <int OPT, int HALVES>
__device__ __forceinline__ void push_tiles_pipelined(const SfPushArgs& a, float* const* grads, int n_grads, int tile, int tile_hi, int stride,
                                                     const uint32_t* s_t_ptr, __nv_bfloat16 (*s_tr)[kTileR + 8], __nv_bfloat16* pub0,
                                                     float* vec0, unsigned long long* tp, long long off_bf16, long long off_f32) {
  TileRegs<HALVES> cur, nxt;
  if (tile >= tile_hi) return;
  push_tile_load<false, HALVES>(a, grads[0], tile, cur);
  for (; tile < tile_hi; tile += stride) {
    const bool more = tile + stride < tile_hi;
    if (more) push_tile_load<false, HALVES>(a, grads[0], tile + stride, nxt);
    if (tp != nullptr) tp[0] = gtime_ns();      // loads issued
    push_tile_apply<OPT, false, HALVES>(a, grads, n_grads, cur, s_t_ptr, false, s_tr, pub0, vec0, tp, off_bf16, off_f32);
    if (more) cur = nxt;
  }
}

// End-of-step hand-off to the host: the mean loss `l` and the step count, with *loss_acc and *done_dev (`done`) loaded by
// the caller.  With a spinning host (done_dev) both travel in ONE aligned 8-byte store to the pinned word pair
// {loss, count} - single-copy atomic, so no system fence (measured several us, on the critical path of every step) is
// needed to order "loss before count".  Without a loss, ((uint32*)loss_out)[1] = ++*done_dev after a system fence.
__device__ __forceinline__ void publish_loss(float* loss_out, float* loss_acc, unsigned int* done_dev, float l, unsigned int done) {
  if (loss_acc != nullptr) *loss_acc = 0.f;
  if (done_dev == nullptr) {
    if (loss_acc != nullptr) *loss_out = l;
    return;
  }
  const unsigned int v = done + 1;
  *done_dev = v;
  if (loss_acc != nullptr) {
    const unsigned long long w = static_cast<unsigned long long>(__float_as_uint(l)) | (static_cast<unsigned long long>(v) << 32);
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(loss_out), "l"(w) : "memory");
    return;
  }
  asm volatile("fence.acq_rel.sys;" ::: "memory");
  st_release_sys(reinterpret_cast<uint32_t*>(loss_out) + 1, v);
}

template <int OPT, bool SYS>
__global__ void __launch_bounds__(kPushThreads, 2)
push_kernel(const SfPushArgs a, uint32_t* local_sync) {
  __shared__ uint32_t s_t;
  __shared__ uint32_t s_epoch;
  __shared__ uint32_t s_valid;
  __shared__ unsigned long long s_ph[3];      // trace: phase stamps of block 0's first tile
  __shared__ __align__(16) __nv_bfloat16 s_tr[kTileC][kTileR + 8];
  TraceScope trace;
  pdl_launch_dependents();
  const int tid = threadIdx.x;
  const bool locked = a.lock_mode == SF_LOCK_RW;
  const bool early = a.replica_version != nullptr;      // lock mode (runtime.cpp): see push_grant
  TileRegs<2> T;
  unsigned long long t_grant = 0ull, t_grad = 0ull;
  // Hogwild reads the global step count racily; it does not depend on this step's kernels, so the
  // round trip to the master overlaps the predecessor's tail (before the programmatic-dependency wait).
  if (!locked && tid == 0) s_t = ld_relaxed_sys(a.ctrl + SF_CTRL_STEP) + 1;
  if (early) {
    if (static_cast<int>(blockIdx.x) < a.num_tiles) push_tile_state(a, blockIdx.x, T);      // in flight during the grant
    push_grant<SYS>(a, local_sync, true, &s_t, &s_epoch, &s_valid);
    if (trace.on) t_grant = gtime_ns();
  }
  pdl_wait();
  trace.mark();
  float loss = 0.f;
  unsigned int done = 0;
  if (tid == 0) {                  // any CTA may be the last: each loads the two words the last one publishes
    if (a.loss_acc != nullptr) loss = *a.loss_acc;
    if (a.done_dev != nullptr) done = *a.done_dev;
  }

  // ---------------- acquire / step number ----------------
  if (locked && !early) {
    push_grant<SYS>(a, local_sync, false, &s_t, &s_epoch, &s_valid);
    if (trace.on) t_grant = gtime_ns();
  }

  // ---------------- tiles ----------------
  float* const grads[1] = {a.grad};
  for (int tile = blockIdx.x; tile < a.num_tiles; tile += gridDim.x) {
    const bool first = tile == static_cast<int>(blockIdx.x);
    const bool lead = trace.on && blockIdx.x == 0 && first;
    if (!early || !first) {
      push_tile_load<true>(a, a.grad, tile, T);
    } else {
      if (!s_valid)      // the early loads may predate another writer's push: reload
#pragma unroll
        for (int half = 0; half < 2; ++half) tile_load_state(a, T, half);
      push_tile_grad<true>(a.grad, T);
    }
    if (lead) t_grad = gtime_ns() + static_cast<unsigned long long>(T.g[0][0] == 12345.678f);      // gradient loads returned
    push_tile_apply<OPT, true, 2>(a, grads, 1, T, &s_t, !locked && first, s_tr, a.shadow_dst[0], a.vec_pub[0], lead ? s_ph : nullptr,
                                  0, 0);
  }

  // ---------------- completion ----------------
  __syncthreads();
  if (tid == 0) {
    const unsigned long long t_st = trace.on ? gtime_ns() : 0ull;
    // lock mode: the arrival orders this CTA's stores before the lock release performed by the last CTA; Hogwild
    // promises no ordering at all, so the counter is relaxed.
    const uint32_t prev = locked ? arrive_done(local_sync) : atomicAdd(local_sync + 2, 1u);
    if (prev == gridDim.x - 1) {                  // last CTA of this push
      const unsigned long long t_arr = trace.on ? gtime_ns() : 0ull;
      local_sync[2] = 0;
      publish_loss(a.loss_out, a.loss_acc, a.done_dev, loss, done);
      if (a.drop) {
        lk_red_relaxed<SYS>(a.ctrl + SF_CTRL_DROPPED, 1u);
      } else {
        lk_red_relaxed<SYS>(a.ctrl + SF_CTRL_STEP, 1u);
        lk_red_relaxed<SYS>(a.ctrl + SF_CTRL_PUSHES, 1u);
        lk_red_relaxed<SYS>(a.ctrl + SF_CTRL_VERSION, 1u);
        // the pushing worker's replica holds this version; only its next pull or push, a later kernel, reads the word
        if (early) *a.replica_version = local_sync[5];
        if (early && !s_valid) local_sync[6] += 1u;      // pushes that reloaded their tuples after the wait
      }
      if (locked) {
        rw_release_write<SYS>(a.ctrl + SF_CTRL_LOCK);
        st_release_gpu(local_sync + 3, s_epoch + 1);
      }
      trace.phases(KID_PUSH_TAIL, t_st, t_arr, gtime_ns());
    }
    if (blockIdx.x == 0) trace.phases(KID_PUSH_LEAD, t_grant, t_grad, s_ph[1]);
  }
  trace.end(KID_PUSH);
}

// ---------------------------------------------------------------------------
// pull: master publish buffer -> local replica (16-byte streaming copies over NVLink)
// ---------------------------------------------------------------------------
template <bool SYS>
__global__ void __launch_bounds__(256, 1)
pull_kernel(const SfPullArgs a, uint32_t* local_sync) {
  __shared__ uint32_t s_epoch;
  TraceScope trace;
  pdl_wait();
  trace.mark();
  const int tid = threadIdx.x;
  const bool locked = a.lock_mode == SF_LOCK_RW;
  if (a.wait_applied != nullptr) {
    if (tid == 0) {
      const uint32_t want = *a.my_posted;
      const unsigned long long t0 = gtime_ns();
      while (static_cast<int32_t>(ld_acquire_sys(a.wait_applied) - want) < 0) {
        __nanosleep(64);
        if (gtime_ns() - t0 > kLockTimeoutNs) sf_fail(0x405);
      }
    }
    __syncthreads();
  }
  const bool dbuf = locked && a.dbuf != 0;
  __shared__ uint32_t s_cur;
  constexpr uint32_t kElided = 2u;      // local_sync[1]: the replica is current, no lock is taken and nothing copied
  uint32_t ver = 0;
  if (locked) {
    if (tid == 0) {
      const uint32_t mine = (blockIdx.x == 0 && a.replica_version != nullptr) ? *a.replica_version : 0u;
      const uint32_t epoch = ld_launch_epoch(local_sync);
      if (blockIdx.x == 0) {
        uint32_t cur = 0;
        if (dbuf) cur = atom_add_acqrel_sys(a.ctrl + SF_CTRL_PUB, 1u) >> 31;      // register + learn the complete buffer
        else if (a.replica_version != nullptr && replica_is_current<SYS>(a.ctrl, mine, ver)) cur = kElided;
        else rw_acquire_read<SYS>(a.ctrl + SF_CTRL_LOCK);
        local_sync[1] = cur;
        st_release_gpu(local_sync + 0, epoch + 1);
        s_cur = cur;
      } else {
        const unsigned long long t0 = gtime_ns();
        while (ld_acquire_gpu(local_sync + 0) != epoch + 1) {
          if (gtime_ns() - t0 > kLockTimeoutNs) sf_fail(0x404);
        }
        s_cur = local_sync[1];
      }
      s_epoch = epoch;
    }
    __syncthreads();
  }
  // successors may pre-launch only once the waits above are over: while this kernel spins on the applier or on a writer's
  // lock, their CTAs (one per SM at GEMM shared-memory sizes) would hold the SMs the kernel it waits for needs
  pdl_launch_dependents();
  const bool elided = locked && s_cur == kElided;
  const uint32_t cur = dbuf ? s_cur : 0u;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t gid = static_cast<size_t>(blockIdx.x) * blockDim.x + tid;
  if (!elided) {
    {
      const uint4* s = reinterpret_cast<const uint4*>(cur ? a.src_alt : a.src);
      uint4* d = reinterpret_cast<uint4*>(a.dst);
      const size_t n16 = a.n_bf16 / 8;
      // 4 independent 16-byte loads in flight per thread to cover the ~2 us NVLink latency
      size_t i = gid;
      for (; i + 3 * stride < n16; i += 4 * stride) {
        const uint4 v0 = ld_stream_u4(s + i), v1 = ld_stream_u4(s + i + stride),
                    v2 = ld_stream_u4(s + i + 2 * stride), v3 = ld_stream_u4(s + i + 3 * stride);
        d[i] = v0; d[i + stride] = v1; d[i + 2 * stride] = v2; d[i + 3 * stride] = v3;
      }
      for (; i < n16; i += stride) d[i] = ld_stream_u4(s + i);
    }
    if (dbuf) {                        // 1-D variables: the fp32 copy that belongs to the same published version
      const float* vp = a.vec_pub[cur];
      for (size_t i = gid; i < a.n_f32; i += stride) a.dst_f32[i] = ld_relaxed_sys_f32(vp + i);
    } else if (a.src_state != nullptr) {      // 1-D variables: gather .x of the interleaved master state
      for (size_t i = gid; i < a.n_f32; i += stride) a.dst_f32[i] = ld_stream_f4(a.src_state + i).x;
    }
  }
  if (gid == 0 && a.seen_version != nullptr) *a.seen_version = elided ? ver : ld_relaxed_sys(a.ctrl + SF_CTRL_VERSION);
  if (locked) {
    __syncthreads();                 // every load of this CTA has returned (values were stored to the replica)
    if (tid == 0) {
      if (arrive_done(local_sync) == gridDim.x - 1) {
        local_sync[2] = 0;
        if (dbuf) lk_red_release<SYS>(a.ctrl + SF_CTRL_PUB, 0u - 1u);
        else if (!elided) rw_release_read<SYS>(a.ctrl + SF_CTRL_LOCK);
        st_release_gpu(local_sync + 3, s_epoch + 1);
      }
    }
  }
  trace.end(KID_PULL);
}

// ---------------------------------------------------------------------------
// post: worker-side half of a served push.  local_sync[4] holds this worker's posted sequence number.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 1)
post_kernel(const SfPostArgs a, uint32_t* local_sync) {
  __shared__ uint32_t s_seq;
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int tid = threadIdx.x;
  if (tid == 0) {
    // the mailbox may only be overwritten once the applier has consumed the previous post
    const uint32_t posted = ld_acquire_gpu(local_sync + 4);
    if (!a.drop) {
      const unsigned long long t0 = gtime_ns();
      while (static_cast<int32_t>(ld_acquire_sys(a.flags + SF_MB_APPLIED) - posted) < 0) {
        __nanosleep(64);
        if (gtime_ns() - t0 > kLockTimeoutNs) sf_fail(0x406);
      }
    }
    s_seq = posted;
  }
  __syncthreads();
  const size_t n4 = a.n / 4;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  float4* g = reinterpret_cast<float4*>(a.grad);
  float4* mb = reinterpret_cast<float4*>(a.mailbox);
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + tid; i < n4; i += stride) {
    const float4 v = g[i];
    g[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!a.drop) st_weak_f4(reinterpret_cast<float*>(mb + i), v.x, v.y, v.z, v.w);
  }
  __syncthreads();
  if (tid == 0) {
    // release: this CTA's mailbox stores (ordered by bar.sync) become visible before the last CTA posts
    asm volatile("fence.acq_rel.sys;" ::: "memory");
    const uint32_t prev = lk_add_release<false>(local_sync + 2, 1u);
    if (prev == gridDim.x - 1) {
      (void)ld_acquire_gpu(local_sync + 2);
      local_sync[2] = 0;
      publish_loss(a.loss_out, a.loss_acc, a.done_dev, a.loss_acc != nullptr ? *a.loss_acc : 0.f, a.done_dev != nullptr ? *a.done_dev : 0u);
      if (!a.drop) {
        st_release_gpu(local_sync + 4, s_seq + 1);
        st_release_sys(a.flags + SF_MB_POSTED, s_seq + 1);
      }
    }
  }
  trace.end(KID_PUSH);
}

// ---------------------------------------------------------------------------
// applier: master-GPU side of a served push.  A host thread keeps a few of these *finite* kernels queued on a
// dedicated stream; each one listens for posted mailboxes for at most `poll_ns`, applies what is posted and
// exits.  (A truly persistent kernel is not an option inside a PyTorch process: CUDA's lazy module loading
// needs a context-wide synchronisation the first time any kernel is used, which would stall behind it.)
// CTA 0 is the leader: its first warp scans every worker's POSTED / APPLIED words in one round trip
// (lane = worker), (lock mode) takes the write lock ONCE for the whole batch, and publishes (epoch, ready mask,
// step) to the other CTAs through master-local memory; every CTA then runs its share of the tiles, applying the
// posted gradients one after the other IN REGISTERS (push_tiles_pipelined): each push is still its own optimizer step
// with its own step number - exactly the reference's parameter server, one update per push in arrival (round-robin)
// order - but the tuples and the bf16 publish move once per batch.  The leader bumps the counters by the batch
// size, releases the lock and acknowledges every consumed mailbox through its APPLIED word.  A shard's applier (ack
// words given) also has every CTA acknowledge the consumed workers in their own memory as soon as its tiles are out.
// sync words: 0 = epoch of the published decision, 1 = ready mask (0 = nothing), 2 = first step number,
//             3 = done counter, 4 = round-robin cursor, 5 = publish buffer / slot of the pass;
//             stats only: 8-9 = time of the decision, 10-11 = time of the last acknowledged decision.
// ---------------------------------------------------------------------------
constexpr int kApplierThreads = 512;
// 120 registers: a 512-thread CTA leaves 4K of its SM's registers to the kernels beside it.  The tile loop needs no more
// (no spill at this bound); with only a 512-thread launch bound ptxas takes up to 124, and the SM has none left over.
template <int OPT, bool SYS>
__global__ void __maxnreg__(120)
applier_kernel(const SfApplierArgs a, const uint32_t seq) {
  __shared__ uint32_t s_t;
  __shared__ uint32_t s_mask;
  __shared__ uint32_t s_buf;
  __shared__ int s_n;
  __shared__ float* s_grads[8];
  __shared__ __align__(16) __nv_bfloat16 s_tr[kTileC][kTileR + 8];
  const int tid = threadIdx.x;
  const bool leader = blockIdx.x == 0;
  const bool locked = a.push.lock_mode == SF_LOCK_RW;
  // One launch serves up to kMaxBatches passes.  With `linger` it keeps listening between passes: the same resident CTAs
  // (instruction cache, TLB warm) serve the next push - a cold pass spends microseconds just fetching code.
  constexpr int kMaxBatches = 256;
  for (int k = 0; k < kMaxBatches; ++k) {
    const uint32_t epoch = seq * 256u + static_cast<uint32_t>(k);
    uint32_t posted = 0;                    // leader warp: lane w holds worker w's POSTED word
    if (leader) {
      if (tid < 32) {
        unsigned m_ready = 0;
        const unsigned long long t0 = gtime_ns();
        while (true) {
          bool ready = false;
          if (tid < a.n_workers) {
            posted = ld_acquire_sys(a.flags + tid * SF_MB_WORDS + SF_MB_POSTED);
            const uint32_t ap = ld_relaxed_sys(a.flags + tid * SF_MB_WORDS + SF_MB_APPLIED);
            ready = posted != ap;
          }
          m_ready = __ballot_sync(0xffffffffu, ready);
          if (m_ready) break;
          // the first decision listens for a whole window; follow-ups only take what is already there
          const bool over = (k > 0 && !a.linger) || (gtime_ns() - t0 > a.idle_timeout_ns);
          if (__ballot_sync(0xffffffffu, over) & 1u) break;      // lane 0 decides for the whole warp
          __nanosleep(40);
        }
        if (a.max_batch > 0 && a.max_batch < 8) {                // keep only the first max_batch workers after the cursor
          const int rr = static_cast<int>(a.sync[4]) % a.n_workers;
          unsigned keep = 0;
          int cnt = 0;
          for (int i = 0; i < a.n_workers && cnt < a.max_batch; ++i) {
            const int w = (rr + i) % a.n_workers;
            if (m_ready >> w & 1u) { keep |= 1u << w; ++cnt; }
          }
          m_ready = keep;
        }
        if (tid == 0) {
          uint32_t t = 0, buf = 0;
          if (m_ready) {
            if (locked) rw_acquire_write<SYS>(a.push.ctrl + SF_CTRL_LOCK);       // vs. worker-applied / external pushes
            if (a.dbuf) {
              // write the buffer that is NOT current.  Pulls still copying it registered before the last flip: one
              // instant with no pull in flight (any time after that flip) means they are all gone.
              const unsigned long long t0 = gtime_ns();
              uint32_t pub;
              while (((pub = ld_acquire_sys(a.push.ctrl + SF_CTRL_PUB)) & 0xFFFFu) != 0u) {
                if (gtime_ns() - t0 > kStaleReaderNs) {
                  // watchdog: a pull registered and never deregistered (its worker died mid-pull).  Drop the stale
                  // registrations instead of stalling every other worker: clear the reader count, record the event
                  // (the reference tolerates dead workers the same way: the server simply stops hearing from them).
                  (void)atomicAnd(a.push.ctrl + SF_CTRL_PUB, 0xFFFF0000u);
                  lk_red_relaxed<SYS>(a.push.ctrl + SF_CTRL_ERRORS, 1u);
                  pub = ld_acquire_sys(a.push.ctrl + SF_CTRL_PUB);
                  break;
                }
              }
              buf = (pub >> 31) ^ 1u;
            }
            t = ld_relaxed_sys(a.push.ctrl + SF_CTRL_STEP) + 1;
            if (a.n_ver > 0) {
              // seqlock: stamp `begin` in every replica before the first publish store of this pass can land
              const uint32_t ver = ld_relaxed_sys(a.ver_local) + 1;
              for (int d = 0; d < a.n_ver; ++d) st_u32_pub(a.ver_begin[d], ver, a.ver_mc != 0);
              asm volatile("fence.acq_rel.sys;" ::: "memory");
              buf = ver & 1u;                                    // two publish slots: this pass lands in slot ver & 1
            }
          }
          if (a.stats != nullptr) a.sync[8] = static_cast<uint32_t>(gtime_ns()), a.sync[9] = static_cast<uint32_t>(gtime_ns() >> 32);
          a.sync[1] = m_ready;
          a.sync[2] = t;
          a.sync[5] = buf;
          st_release_gpu(a.sync + 0, epoch);
          s_mask = m_ready;
          s_t = t;
          s_buf = buf;
        }
      }
    } else if (tid == 0) {
      const unsigned long long t0 = gtime_ns();
      while (ld_acquire_gpu(a.sync + 0) != epoch) {
        __nanosleep(20);
        if (gtime_ns() - t0 > a.idle_timeout_ns + kLockTimeoutNs) sf_fail(0x408);
      }
    }
    if (!leader && tid == 0) {
      s_mask = a.sync[1];
      s_t = a.sync[2];
      s_buf = a.sync[5];
    }
    __syncthreads();
    const uint32_t mask = s_mask;
    if (mask == 0) return;                              // nothing (more) is posted: this launch is done
    const bool probe = a.stats != nullptr && blockIdx.x == gridDim.x - 1 && tid == 0;      // phase timing of one follower CTA
    const unsigned long long tp0 = probe ? gtime_ns() : 0ull;
    if (tid == 0) {
      // application order: round-robin from the cursor, so no worker's push is always last in a batch
      const int rr = static_cast<int>(a.sync[4]) % a.n_workers;
      int n = 0;
      for (int i = 0; i < a.n_workers; ++i) {
        const int w = (rr + i) % a.n_workers;
        if (mask >> w & 1u) s_grads[n++] = a.mailboxes + static_cast<size_t>(w) * a.mailbox_stride;
      }
      s_n = n;
    }
    __syncthreads();
    const int n = s_n;
    const long long off_bf16 = s_buf ? a.slot_off_bf16 : 0;      // two publish slots (0 without)
    const long long off_f32 = s_buf ? a.slot_off_f32 : 0;
    __nv_bfloat16* const pub0 = ((a.dbuf && s_buf) ? a.shadow_alt : a.push.shadow_dst[0]) + off_bf16;
    float* const vec0 = (a.dbuf && s_buf) ? a.vec_pub_alt : a.push.vec_pub[0];
    const int tile_lo = a.tile_end > a.tile_begin ? a.tile_begin : 0;
    const int tile_hi = a.tile_end > a.tile_begin ? a.tile_end : a.push.num_tiles;
    // probe timestamps in shared memory: a thread-local array whose address is passed down would get a stack frame
    __shared__ unsigned long long tpt[3];
    if (probe) tpt[0] = tpt[1] = tpt[2] = 0ull;
    const unsigned long long tpa = probe ? gtime_ns() : 0ull;          // s_grads built, barrier passed
    push_tiles_pipelined<OPT, 1>(a.push, s_grads, n, tile_lo + static_cast<int>(blockIdx.x), tile_hi, static_cast<int>(gridDim.x), &s_t, s_tr,
                                 pub0, vec0, probe ? tpt : nullptr, off_bf16, off_f32);
    __syncthreads();
    const unsigned long long tp1 = probe ? gtime_ns() : 0ull;
    if (probe && tpt[0] != 0ull) {
      a.stats[8] += tpa - tp0;             // build the mailbox list + barrier
      a.stats[9] += tpt[0] - tpa;          // tile header + loads issued
      a.stats[10] += tpt[1] - tpt[0];      // loads returned + optimizer math
      a.stats[11] += tpt[2] - tpt[1];      // state / W stores issued
      a.stats[12] += tp1 - tpt[2];         // transpose through smem + W^T stores + barriers
      const unsigned long long q0 = gtime_ns(), q1 = gtime_ns();
      a.stats[13] += q1 - q0;              // cost of one %globaltimer read
    }
    const bool counting = a.ack[0] != nullptr;          // a shard's applier: every CTA acknowledges (runtime.cpp)
    if (counting) {
      // distributed acknowledgement: this CTA is done with the consumed mailboxes and its share of the publish is on its
      // way.  ONE system fence per CTA (thread 0; bar.sync makes it cumulative over the CTA's stores), then relaxed
      // counts: every CTA pays its NVLink flush in parallel instead of the leader paying it after all of them.
      if (tid == 0) asm volatile("fence.acq_rel.sys;" ::: "memory");
      __syncthreads();
      if (tid < 8 && (mask >> tid & 1u) && a.ack[tid] != nullptr)
        asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(a.ack[tid]), "r"(1u) : "memory");
      // seqlock `end`: count this CTA's completion in every replica (after the fence: its publish stores are performed)
      if (tid >= 8 && tid < 8 + a.n_ver) {
        if (a.ver_mc) asm volatile("multimem.red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(a.ver_end[tid - 8]), "r"(1u) : "memory");
        else asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(a.ver_end[tid - 8]), "r"(1u) : "memory");
      }
    }
    if (tid == 0) {
      if (counting) lk_red_relaxed<false>(a.sync + 3, 1u);       // ordered after the fence above
      else lk_red_release<false>(a.sync + 3, 1u);
      if (probe) {
        const unsigned long long tp2 = gtime_ns();
        const unsigned long long t_dec = static_cast<unsigned long long>(a.sync[8]) | (static_cast<unsigned long long>(a.sync[9]) << 32);
        a.stats[4] += tp0 - t_dec;          // decision -> this CTA saw it
        a.stats[5] += tp1 - tp0;            // tiles: loads, optimizer, stores issued
        a.stats[6] += tp2 - tp1;            // acknowledgement red + arrive (the NVLink flush)
      }
    }
    if (leader && tid < 32) {
      if (tid == 0) {
        const unsigned long long t0 = gtime_ns();
        while (ld_acquire_gpu(a.sync + 3) != gridDim.x) {
          if (gtime_ns() - t0 > kLockTimeoutNs) sf_fail(0x407);
        }
        const unsigned long long t_tiles = a.stats != nullptr ? gtime_ns() : 0ull;
        a.sync[3] = 0;                                  // everybody has arrived; the next decision is published after this
        a.sync[4] = static_cast<uint32_t>(32 - __clz(mask));     // cursor: one past the highest worker served
        // the freshly written buffer becomes the current one (release: after every CTA's publish stores, which the
        // acquire of the done counter above made visible to this thread)
        if (a.dbuf) (void)atom_xor_release_sys(a.push.ctrl + SF_CTRL_PUB, 0x80000000u);
        lk_red_relaxed<SYS>(a.push.ctrl + SF_CTRL_STEP, static_cast<uint32_t>(n));
        lk_red_relaxed<SYS>(a.push.ctrl + SF_CTRL_PUSHES, static_cast<uint32_t>(n));
        lk_red_relaxed<SYS>(a.push.ctrl + SF_CTRL_VERSION, static_cast<uint32_t>(n));
        if (locked) rw_release_write<SYS>(a.push.ctrl + SF_CTRL_LOCK);
        if (a.stats != nullptr) {
          const unsigned long long t_dec = static_cast<unsigned long long>(a.sync[8]) | (static_cast<unsigned long long>(a.sync[9]) << 32);
          a.stats[0] += t_tiles - t_dec;
          a.stats[2] += 1ull;
          a.stats[3] += static_cast<unsigned long long>(n);
          a.sync[10] = static_cast<uint32_t>(t_dec), a.sync[11] = static_cast<uint32_t>(t_dec >> 32);
        }
      }
      __syncwarp();
      // lane w acknowledges worker w (release: ordered after lane 0's acquire of the done counter by the warp barrier)
      if (mask >> tid & 1u) {
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
        st_release_sys(a.flags + tid * SF_MB_WORDS + SF_MB_APPLIED, posted);
      }
      if (a.stats != nullptr) {
        __syncwarp();
        if (tid == 0) {
          const unsigned long long t_dec = static_cast<unsigned long long>(a.sync[10]) | (static_cast<unsigned long long>(a.sync[11]) << 32);
          a.stats[1] += gtime_ns() - t_dec;
        }
      }
    }
    __syncthreads();
  }
}


// ---------------------------------------------------------------------------
// Sharded master, worker side (see sf_api.h).
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint4 ld_local_u4(const uint4* p) {
  // the inbox replica is LOCAL memory written by remote multimem / peer stores: bypass L1 (may hold a stale line)
  uint4 r;
  asm volatile("ld.global.relaxed.sys.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}

// copy the publish slices (W block, W^T block, fp32 tail elements) of up to kCopyBatch push tiles: inbox -> working
// replica.  All loads of the batch are issued before the first store (the copy is latency-, not bandwidth-bound).
constexpr int kCopyBatch = 4;
__device__ __forceinline__ void copy_tiles_publish(const SfSyncPullArgs& a, int tile0, int tile_end, int stride, long long soff_bf16,
                                                   long long soff_f32) {
  const int tid = threadIdx.x;
  const __nv_bfloat16* const src = a.src + soff_bf16;
  const float* const src_vec = a.src_vec != nullptr ? a.src_vec + soff_f32 : nullptr;
  uint4 vw[kCopyBatch], vt[kCopyBatch];
  float vv[kCopyBatch];
  int64_t ow[kCopyBatch], ot[kCopyBatch];
  long long ov[kCopyBatch];
#pragma unroll
  for (int b = 0; b < kCopyBatch; ++b) {
    const int tile = tile0 + b * stride;
    ow[b] = ot[b] = -1;
    ov[b] = -1;
    if (tile >= tile_end) continue;
    const SfTensorSeg sg = a.segs[a.tile_map[tile * 3 + 0]];
    const int r0 = a.tile_map[tile * 3 + 1] * kTileR, c0 = a.tile_map[tile * 3 + 2] * kTileC;
    if (sg.w_off >= 0) {
      const int row = r0 + (tid >> 3), col = c0 + (tid & 7) * 8;
      if (row < sg.rows && col < sg.w_ld) {
        ow[b] = sg.w_off + static_cast<int64_t>(row) * sg.w_ld + col;
        vw[b] = ld_local_u4(reinterpret_cast<const uint4*>(src + ow[b]));
      }
    }
    if (sg.wt_off >= 0) {
      const int trow = c0 + (tid >> 2), el = r0 + (tid & 3) * 8;
      if (trow < sg.cols && el < sg.wt_ld) {
        ot[b] = sg.wt_off + static_cast<int64_t>(trow) * sg.wt_ld + el;
        vt[b] = ld_local_u4(reinterpret_cast<const uint4*>(src + ot[b]));
      }
    }
    if (sg.rows == 1 && a.dst_vec != nullptr && tid < kTileC && c0 + tid < sg.cols) {
      ov[b] = sg.offset + c0 + tid - a.vec_offset;
      vv[b] = ld_relaxed_sys_f32(src_vec + ov[b]);
    }
  }
#pragma unroll
  for (int b = 0; b < kCopyBatch; ++b) {
    if (ow[b] >= 0) *reinterpret_cast<uint4*>(a.dst + ow[b]) = vw[b];
    if (ot[b] >= 0) *reinterpret_cast<uint4*>(a.dst + ot[b]) = vt[b];
    if (ov[b] >= 0) a.dst_vec[ov[b]] = vv[b];
  }
}

__global__ void __launch_bounds__(256, 1)
sync_pull_kernel(const SfSyncPullArgs a) {
  __shared__ uint32_t s_e;
  __shared__ uint32_t s_ok;
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int tid = threadIdx.x;
  const int cps = a.ctas_per_shard;
  const int shard = blockIdx.x / cps, part = blockIdx.x % cps;
  // ---- read-your-writes: this shard's applier has consumed my last post (it acknowledges into MY memory) ----
  unsigned long long t_seen = 0;
  if (tid == 0) {
    const uint32_t want = *a.my_posted * static_cast<uint32_t>(a.ack_grid[shard]);
    const unsigned long long t0 = gtime_ns();
    // relaxed polling (the word lives in local memory, remote appliers write it); the data the acknowledgement covers is
    // consumed by LATER kernels (kernel boundary) or validated by the seqlock below
    while (static_cast<int32_t>(ld_relaxed_sys(a.applied + shard * 16) - want) < 0) {
      __nanosleep(20);
      if (gtime_ns() - t0 > kLockTimeoutNs) sf_fail(0x405);
    }
    if (a.stats != nullptr && part == 0) {
      t_seen = gtime_ns();
      const unsigned long long t_post = a.stats[0];
      if (t_post != 0 && t0 > t_post) {
        a.stats[8 + 4 * shard] += t0 - t_post;
        a.stats[9 + 4 * shard] += t_seen - t0;
        a.stats[11 + 4 * shard] += 1ull;
      }
    }
  }
  __syncthreads();
  if (!a.copy) {
    trace.end(KID_PULL);
    return;
  }
  // ---- consistent snapshot of the shard (seqlock; every CTA of the shard must have copied the SAME version) ----
  uint32_t* sy = a.sync + shard * 8;          // 0 arrivals, 1 min version, 2 max version / dirty, 3 result (round << 1 | ok), 4 round
  const unsigned long long t0 = gtime_ns();
  while (true) {
    uint32_t round = 0;
    if (tid == 0 && cps > 1) round = ld_acquire_gpu(sy + 4);
    if (tid == 0 && cps > 1 && part != 0) {
      // the shard's first CTA picks the version for all of them (independent picks disagree whenever a pass completes
      // between two CTAs' reads - which is exactly when the acknowledgements they just waited for arrive)
      while (ld_acquire_gpu(sy + 6) != round + 1) {
        if (gtime_ns() - t0 > kLockTimeoutNs) sf_fail(0x40D);
      }
      s_e = sy[5];
    } else if (tid == 0) {
      // seqlock reader without fences: the stamp loads are relaxed.sys (served by L2, the coherence point of local
      // memory); the copy's loads cannot issue before the version is known (bar.sync below) and the re-check of `begin`
      // is issued after the copy's values were consumed by its stores (bar.sync), i.e. in program order.
      // `begin` = passes started, `end` = CTA completions (ack_grid per pass).
      // Two slots: never wait.  Quiescent -> the newest pass is complete; a pass in flight -> the one before it is
      // (the leader starts a pass only after every CTA of the previous one fenced its publish stores)
      uint32_t b = ld_relaxed_sys(a.ver_begin + shard * a.ver_stride);
      if (ld_relaxed_sys(a.ver_end + shard * a.ver_stride) != b * static_cast<uint32_t>(a.ack_grid[shard])) b -= 1u;
      s_e = b;
      if (cps > 1) {
        sy[5] = b;
        st_release_gpu(sy + 6, round + 1);
      }
    }
    __syncthreads();
    {
      const uint32_t ver = s_e;
      const long long so_b = (ver & 1u) ? a.slot_off_bf16 : 0, so_f = (ver & 1u) ? a.slot_off_f32 : 0;
      for (int tile = a.bounds[shard] + part; tile < a.bounds[shard + 1]; tile += cps * kCopyBatch)
        copy_tiles_publish(a, tile, a.bounds[shard + 1], cps, so_b, so_f);
    }
    __syncthreads();
    if (tid == 0) {
      const uint32_t e = s_e;
      // slot e & 1 is rewritten by pass e + 2
      const uint32_t b2 = ld_relaxed_sys(a.ver_begin + shard * a.ver_stride);
      const bool clean = static_cast<int32_t>(b2 - e) <= 1;
      uint32_t ok;
      if (cps == 1) {
        ok = clean ? 1u : 0u;
      } else {
        // agreement round: min / max over the CTAs' versions (a dirty CTA poisons max), last arriver publishes the verdict
        atomicMin(sy + 1, e);
        atomicMax(sy + 2, clean ? e : 0xFFFFFFFFu);
        if (lk_add_release<false>(sy + 0, 1u) == static_cast<uint32_t>(cps) - 1u) {
          (void)ld_acquire_gpu(sy + 0);
          ok = (sy[1] == sy[2]) ? 1u : 0u;
          sy[0] = 0; sy[1] = 0xFFFFFFFFu; sy[2] = 0;
          st_release_gpu(sy + 4, round + 1);
          st_release_gpu(sy + 3, ((round + 1) << 1) | ok);
        } else {
          uint32_t r;
          while (((r = ld_acquire_gpu(sy + 3)) >> 1) != round + 1) {
            if (gtime_ns() - t0 > kLockTimeoutNs) sf_fail(0x40B);
          }
          ok = r & 1u;
        }
      }
      s_ok = ok;
    }
    __syncthreads();
    if (s_ok) break;
    if (gtime_ns() - t0 > kLockTimeoutNs) sf_fail(0x40C);
  }
  if (tid == 0 && a.stats != nullptr && part == 0 && t_seen != 0) a.stats[10 + 4 * shard] += gtime_ns() - t_seen;
  trace.end(KID_PULL);
}

__global__ void __launch_bounds__(256, 1)
post_flags_kernel(const SfPostFlagsArgs a) {
  TraceScope trace;
  pdl_launch_dependents();
  pdl_wait();
  trace.mark();
  const int tid = threadIdx.x;
  // ---- 1-D tail (bias gradients were accumulated locally by atomics): forward each 64-element tile to its owner ----
  for (int i = tid >> 6; i < (a.phase == 2 ? 0 : a.n_vec_tiles); i += blockDim.x >> 6) {
    const long long tile = a.vec_tiles[i * 3 + 0], off = a.vec_tiles[i * 3 + 1], cnt = a.vec_tiles[i * 3 + 2];
    int owner = 0;
    for (int r = 1; r < a.n_shards; ++r) owner += tile >= a.bounds[r] ? 1 : 0;
    const int l = tid & 63;
    if (l < cnt) {
      const float g = a.grad[off + l];
      a.grad[off + l] = 0.f;
      if (!a.drop) asm volatile("st.global.relaxed.sys.f32 [%0], %1;" ::"l"(a.mailbox[owner] + off + l), "f"(g) : "memory");
    }
  }
  if (a.drop && a.mb_zero) {
    // the wgrad epilogues already ADDED this step's tiles into the mailboxes: a dropped push must take them out again
    for (int r = 0; r < a.n_shards; ++r)
      for (long long i = tid; i < a.total / 4; i += blockDim.x)
        st_weak_f4(a.mailbox[r] + i * 4, 0.f, 0.f, 0.f, 0.f);
  }
  __syncthreads();
  if (a.phase == 1) {                  // forwarding only: the post comes from a later launch
    trace.end(KID_PUSH);
    return;
  }
  if (tid == 0) {
    publish_loss(a.loss_out, a.loss_acc, a.done_dev, a.loss_acc != nullptr ? *a.loss_acc : 0.f, a.done_dev != nullptr ? *a.done_dev : 0u);
  }
  if (!a.drop && a.phase == 2 && tid < a.n_shards) {
    // every gradient store (wgrad epilogues, tail forwarding) belongs to a kernel that COMPLETED before this one started
    // (griddepcontrol.wait / graph edges): completed kernels' writes are performed system-wide, no fence needed here
    const uint32_t seq = *a.my_posted + 1;
    asm volatile("st.global.relaxed.sys.u32 [%0], %1;" ::"l"(a.posted[tid]), "r"(seq) : "memory");
  }
  if (!a.drop && a.phase != 2 && tid < a.n_shards) {
    // the matrix gradients were stored by the wgrad kernels this kernel depends on (kernel boundary = performed);
    // the release below orders them, and the tail stores above (bar.sync), before the post becomes visible
    const uint32_t seq = *a.my_posted + 1;
    asm volatile("fence.acq_rel.sys;" ::: "memory");
    st_release_sys(a.posted[tid], seq);
  }
  __syncthreads();
  if (!a.drop && tid == 0) *a.my_posted = *a.my_posted + 1;
  if (tid == 0 && a.stats != nullptr) a.stats[0] = gtime_ns();
  if (tid == 0 && a.heartbeat != nullptr) {
    // liveness: (%globaltimer ns, steps so far) in this worker's symmetric segment, readable by every peer / the host
    a.heartbeat[0] = gtime_ns();
    a.heartbeat[1] = a.heartbeat[1] + 1ull;
  }
  trace.end(KID_PUSH);
}

// single-thread lock exerciser used by the GPU tests (op: 0 = acquire_read, 1 = release_read,
// 2 = acquire_write, 3 = release_write)
__global__ void lock_test_kernel(uint32_t* ctrl, int op) {
  switch (op) {
    case 0: rw_acquire_read<true>(ctrl + SF_CTRL_LOCK); break;
    case 1: rw_release_read<true>(ctrl + SF_CTRL_LOCK); break;
    case 2: rw_acquire_write<true>(ctrl + SF_CTRL_LOCK); break;
    case 3: rw_release_write<true>(ctrl + SF_CTRL_LOCK); break;
  }
}

}  // namespace sf

template <int OPT>
static int launch_push(const SfPushArgs* a, uint32_t* ls, int grid, cudaStream_t st) {
  if (a->scope_sys)
    return static_cast<int>(sf::launch(sf::push_kernel<OPT, true>, dim3(grid), dim3(sf::kPushThreads), 0, st, *a, ls));
  return static_cast<int>(sf::launch(sf::push_kernel<OPT, false>, dim3(grid), dim3(sf::kPushThreads), 0, st, *a, ls));
}

extern "C" int sf_push_launch(const SfPushArgs* a, uint32_t* local_sync, int grid, cudaStream_t st) {
  // lock mode needs every CTA resident: at most two 256-thread CTAs per SM (launch bounds); big models use both for
  // twice the loads in flight per SM
  if (grid <= 0) grid = a->num_tiles < 296 ? a->num_tiles : 296;
  if (grid > 296) grid = 296;
  if (grid < 1) grid = 1;
  switch (a->optimizer) {
    case SF_OPT_SGD: return launch_push<SF_OPT_SGD>(a, local_sync, grid, st);
    case SF_OPT_MOMENTUM: return launch_push<SF_OPT_MOMENTUM>(a, local_sync, grid, st);
    case SF_OPT_ADAM: return launch_push<SF_OPT_ADAM>(a, local_sync, grid, st);
    case SF_OPT_RMSPROP: return launch_push<SF_OPT_RMSPROP>(a, local_sync, grid, st);
    case SF_OPT_ADAGRAD: return launch_push<SF_OPT_ADAGRAD>(a, local_sync, grid, st);
    case SF_OPT_ADADELTA: return launch_push<SF_OPT_ADADELTA>(a, local_sync, grid, st);
    case SF_OPT_ADAGRAD_DA: return launch_push<SF_OPT_ADAGRAD_DA>(a, local_sync, grid, st);
    case SF_OPT_FTRL: return launch_push<SF_OPT_FTRL>(a, local_sync, grid, st);
    case SF_OPT_PROXIMAL_ADAGRAD: return launch_push<SF_OPT_PROXIMAL_ADAGRAD>(a, local_sync, grid, st);
    case SF_OPT_PROXIMAL_SGD: return launch_push<SF_OPT_PROXIMAL_SGD>(a, local_sync, grid, st);
  }
  return -4;
}

extern "C" int sf_pull_launch(const SfPullArgs* a, uint32_t* local_sync, int grid, cudaStream_t st) {
  if (grid <= 0) {
    const size_t n16 = a->n_bf16 / 8 + a->n_f32 / 4;
    grid = static_cast<int>((n16 + 256 * 4 - 1) / (256 * 4));
    if (grid > sf_num_sms()) grid = sf_num_sms();
    if (grid < 1) grid = 1;
  }
  if (a->scope_sys) return static_cast<int>(sf::launch(sf::pull_kernel<true>, dim3(grid), dim3(256), 0, st, *a, local_sync));
  return static_cast<int>(sf::launch(sf::pull_kernel<false>, dim3(grid), dim3(256), 0, st, *a, local_sync));
}

extern "C" int sf_post_launch(const SfPostArgs* a, uint32_t* local_sync, int grid, cudaStream_t st) {
  if (grid <= 0) {
    grid = static_cast<int>((a->n / 4 + 256 * 8 - 1) / (256 * 8));
    if (grid > sf_num_sms()) grid = sf_num_sms();
    if (grid < 1) grid = 1;
  }
  return static_cast<int>(sf::launch(sf::post_kernel, dim3(grid), dim3(256), 0, st, *a, local_sync));
}

template <int OPT>
static int launch_applier(const SfApplierArgs* a, unsigned int seq, int grid, cudaStream_t st) {
  if (a->push.scope_sys) sf::applier_kernel<OPT, true><<<grid, sf::kApplierThreads, 0, st>>>(*a, seq);
  else sf::applier_kernel<OPT, false><<<grid, sf::kApplierThreads, 0, st>>>(*a, seq);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int sf_applier_launch(const SfApplierArgs* a, unsigned int seq, int grid, cudaStream_t st) {
  if (grid <= 0) grid = 96;
  if (grid > sf_num_sms()) grid = sf_num_sms();       // co-resident with the training kernels: 256 threads, ~5 KB smem per CTA
  if (a->n_workers < 1 || a->n_workers > 8) return -6;
  switch (a->push.optimizer) {
    case SF_OPT_SGD: return launch_applier<SF_OPT_SGD>(a, seq, grid, st);
    case SF_OPT_MOMENTUM: return launch_applier<SF_OPT_MOMENTUM>(a, seq, grid, st);
    case SF_OPT_ADAM: return launch_applier<SF_OPT_ADAM>(a, seq, grid, st);
    case SF_OPT_RMSPROP: return launch_applier<SF_OPT_RMSPROP>(a, seq, grid, st);
    case SF_OPT_ADAGRAD: return launch_applier<SF_OPT_ADAGRAD>(a, seq, grid, st);
    case SF_OPT_ADADELTA: return launch_applier<SF_OPT_ADADELTA>(a, seq, grid, st);
    case SF_OPT_ADAGRAD_DA: return launch_applier<SF_OPT_ADAGRAD_DA>(a, seq, grid, st);
    case SF_OPT_FTRL: return launch_applier<SF_OPT_FTRL>(a, seq, grid, st);
    case SF_OPT_PROXIMAL_ADAGRAD: return launch_applier<SF_OPT_PROXIMAL_ADAGRAD>(a, seq, grid, st);
    case SF_OPT_PROXIMAL_SGD: return launch_applier<SF_OPT_PROXIMAL_SGD>(a, seq, grid, st);
  }
  return -4;
}


extern "C" int sf_sync_pull_launch(const SfSyncPullArgs* a, cudaStream_t st) {
  if (a->n_shards < 1 || a->n_shards > SF_MAX_SHARDS || a->ctas_per_shard < 1) return -6;
  const int grid = a->n_shards * a->ctas_per_shard;
  if (grid > sf_num_sms()) return -6;            // the agreement round needs every CTA of a shard resident
  return static_cast<int>(sf::launch(sf::sync_pull_kernel, dim3(grid), dim3(256), 0, st, *a));
}

extern "C" int sf_post_flags_launch(const SfPostFlagsArgs* a, cudaStream_t st) {
  if (a->n_shards < 1 || a->n_shards > SF_MAX_SHARDS) return -6;
  return static_cast<int>(sf::launch(sf::post_flags_kernel, dim3(1), dim3(256), 0, st, *a));
}

extern "C" int sf_lock_test(uint32_t* ctrl, int op, cudaStream_t st) {
  sf::lock_test_kernel<<<1, 1, 0, st>>>(ctrl, op);
  return static_cast<int>(cudaGetLastError());
}
