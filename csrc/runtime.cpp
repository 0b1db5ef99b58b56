// Host runtime of sparkflow_b200 (C++): step-plan runner with CUDA-graph capture, prepared GEMM
// objects (TMA descriptors are encoded once per buffer set), the CUDA-IPC symmetric-memory helper
// that maps the master's buffers into every worker process, and thin pybind11 entry points for
// every kernel.  Python hands over raw device addresses (torch owns the allocations); nothing in
// here depends on libtorch.
#include <pybind11/pybind11.h>
#include <pybind11/numpy.h>
#include <pybind11/stl.h>

#include <array>
#include <atomic>
#include <map>
#include <mutex>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <thread>
#include <functional>
#include <memory>
#include <stdexcept>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "sf_api.h"
#include "vmm.h"

namespace py = pybind11;

namespace {

inline void ck(cudaError_t e, const char* what) {
  if (e != cudaSuccess) {
    throw std::runtime_error(std::string("sparkflow_b200 CUDA error in ") + what + ": " +
                             cudaGetErrorString(e));
  }
}
inline void ck_rc(int rc, const char* what) {
  if (rc != 0) {
    const char* msg = rc > 0 ? cudaGetErrorString(static_cast<cudaError_t>(rc)) : "invalid argument";
    throw std::runtime_error(std::string("sparkflow_b200: ") + what + " failed (rc=" +
                             std::to_string(rc) + ", " + msg + ")");
  }
}

template <class T>
inline T* P(uintptr_t v) { return reinterpret_cast<T*>(v); }
inline cudaStream_t S(uintptr_t v) { return reinterpret_cast<cudaStream_t>(v); }

template <class T>
T getd(const py::dict& d, const char* k, T dflt) {
  if (d.contains(k) && !d[k].is_none()) return d[k].cast<T>();
  return dflt;
}

// the device addresses listed under `k`, cast into `out` (more than `out` holds: `what` is the error); returns how many
template <class T, size_t N>
int getd_ptrs(const py::dict& d, const char* k, const char* what, T* (&out)[N]) {
  const auto v = getd<std::vector<uintptr_t>>(d, k, {});
  if (v.size() > N) throw std::runtime_error(what);
  for (size_t i = 0; i < v.size(); ++i) out[i] = P<T>(v[i]);
  return static_cast<int>(v.size());
}

// one (offset, rows, cols, w_off, w_ld, wt_off, wt_ld) row of a variable table (any other length: `what` is the error)
void fill_seg(SfTensorSeg& sg, const std::vector<int64_t>& r, const char* what) {
  if (r.size() != 7) throw std::runtime_error(what);
  std::memset(&sg, 0, sizeof(sg));
  sg.offset = r[0];
  sg.rows = static_cast<int>(r[1]);
  sg.cols = static_cast<int>(r[2]);
  sg.w_off = r[3];
  sg.w_ld = static_cast<int>(r[4]);
  sg.wt_off = r[5];
  sg.wt_ld = static_cast<int>(r[6]);
}

// ---------------------------------------------------------------------------
// Prepared GEMM
// ---------------------------------------------------------------------------
struct Gemm {
  SfGemm g;
  explicit Gemm(const py::dict& d) {
    std::memset(&g, 0, sizeof(g));
    g.a = P<void>(getd<uintptr_t>(d, "a", 0));
    g.b = P<void>(getd<uintptr_t>(d, "b", 0));
    g.M = getd<int>(d, "M", 0);
    g.N = getd<int>(d, "N", 0);
    g.K = getd<int>(d, "K", 0);
    g.lda = getd<int>(d, "lda", g.K);
    g.ldb = getd<int>(d, "ldb", g.K);
    g.bn = getd<int>(d, "bn", 0);
    g.split_k = getd<int>(d, "split_k", 1);
    g.pair = getd<int>(d, "pair", -1);
    g.mn_major = getd<int>(d, "mn_major", 0);
    g.pair_ctas = getd<int>(d, "pair_ctas", 0);
    g.epi = getd<int>(d, "epi", -1);
    g.ep.out_f32 = P<float>(getd<uintptr_t>(d, "out_f32", 0));
    g.ep.ld_f32 = getd<int>(d, "ld_f32", g.N);
    g.ep.out_bf16 = P<__nv_bfloat16>(getd<uintptr_t>(d, "out_bf16", 0));
    g.ep.ld_bf16 = getd<int>(d, "ld_bf16", 0);
    g.ep.outT_bf16 = P<__nv_bfloat16>(getd<uintptr_t>(d, "outT_bf16", 0));
    g.ep.ld_t = getd<int>(d, "ld_t", 0);
    g.ep.bias = P<const float>(getd<uintptr_t>(d, "bias", 0));
    g.ep.aux = P<const __nv_bfloat16>(getd<uintptr_t>(d, "aux", 0));
    g.ep.ld_aux = getd<int>(d, "ld_aux", 0);
    g.ep.aux_act = getd<int>(d, "aux_act", 0);
    g.ep.colsum = P<float>(getd<uintptr_t>(d, "colsum", 0));
    g.ep.alpha = getd<float>(d, "alpha", 1.0f);
    g.ep.act = getd<int>(d, "act", 0);
    g.ep.accumulate = getd<int>(d, "accumulate", 0);
    g.ep.a_evict_first = getd<int>(d, "a_evict_first", 0);
    g.ep.loss_mode = getd<int>(d, "loss_mode", 0);
    g.ep.target = P<const float>(getd<uintptr_t>(d, "target", 0));
    g.ep.ld_target = getd<int>(d, "ld_target", 0);
    g.ep.loss = P<float>(getd<uintptr_t>(d, "loss", 0));
    g.ep.drop_keep = getd<float>(d, "drop_keep", 0.0f);
    g.ep.drop_seed = getd<unsigned int>(d, "drop_seed", 0u);
    g.ep.drop_stream = getd<unsigned int>(d, "drop_stream", 0u);
    g.ep.drop_ctr = P<const unsigned int>(getd<uintptr_t>(d, "drop_ctr", 0));
    g.ep.aux_keep = getd<float>(d, "aux_keep", 0.0f);
    g.ep.act_alpha = getd<float>(d, "act_alpha", 0.0f);
    g.ep.aux_act_alpha = getd<float>(d, "aux_act_alpha", 0.0f);
    g.ep.ryw = P<const SfRyw>(getd<uintptr_t>(d, "ryw", 0));
    g.ep.route = P<const SfRoute>(getd<uintptr_t>(d, "route", 0));
    g.ep.route_tile0 = getd<int>(d, "route_tile0", 0);
    g.ep.route_tiles_c = getd<int>(d, "route_tiles_c", 1);
    g.ep.route_off = getd<long long>(d, "route_off", 0);
    if ((g.lda % 8) || (g.ldb % 8)) throw std::runtime_error("gemm: lda/ldb must be multiples of 8 (16-byte TMA strides)");
    if (g.ep.out_bf16 && (g.ep.ld_bf16 % 8)) throw std::runtime_error("gemm: ld_bf16 must be a multiple of 8");
    if (g.ep.aux && (g.ep.ld_aux % 8)) throw std::runtime_error("gemm: ld_aux must be a multiple of 8");
    ck_rc(sf_gemm_prepare(&g), "sf_gemm_prepare (cuTensorMapEncodeTiled)");
  }
  void launch(uintptr_t stream) const { ck_rc(sf_gemm_launch(&g, S(stream)), "sf_gemm_launch"); }
  int bn() const { return g.bn; }
  int split_k() const { return g.split_k; }
  int kblocks_per_split() const { return g.kblocks_per_split; }
  int pair() const { return g.pair; }
  int epi() const { return g.epi; }
  py::tuple grid() const {
    return py::make_tuple((g.N + g.bn - 1) / g.bn, (g.M + 127) / 128, g.split_k);
  }
  int mn_major() const { return g.mn_major; }
};

// ---------------------------------------------------------------------------
// push / pull argument parsing
// ---------------------------------------------------------------------------
SfHyper parse_hyper(const py::dict& d) {
  SfHyper h;
  std::memset(&h, 0, sizeof(h));
  h.lr = getd<float>(d, "lr", 0.01f);
  h.beta1 = getd<float>(d, "beta1", 0.9f);
  h.beta2 = getd<float>(d, "beta2", 0.999f);
  h.eps = getd<float>(d, "eps", 1e-8f);
  h.momentum = getd<float>(d, "momentum", 0.0f);
  h.rho = getd<float>(d, "rho", 0.95f);
  h.decay = getd<float>(d, "decay", 0.9f);
  h.l1 = getd<float>(d, "l1", 0.0f);
  h.l2 = getd<float>(d, "l2", 0.0f);
  h.lr_power = getd<float>(d, "lr_power", -0.5f);
  h.init_accum = getd<float>(d, "init_accum", 0.1f);
  h.l2_shrinkage = getd<float>(d, "l2_shrinkage", 0.0f);
  h.nesterov = getd<int>(d, "nesterov", 0);
  h.centered = getd<int>(d, "centered", 0);
  return h;
}

SfPushArgs parse_push(const py::dict& d) {
  SfPushArgs a;
  std::memset(&a, 0, sizeof(a));
  a.state = P<float4>(getd<uintptr_t>(d, "state", 0));
  a.ctrl = P<uint32_t>(getd<uintptr_t>(d, "ctrl", 0));
  a.n_shadow_dst = getd_ptrs(d, "shadow_dst", "push: at most 8 publish destinations", a.shadow_dst);
  a.n_vec_pub = getd_ptrs(d, "vec_pub", "push: at most 2 vec_pub targets", a.vec_pub);
  a.vec_offset = getd<long long>(d, "vec_offset", 0);
  a.shadow_is_mc = getd<int>(d, "shadow_is_mc", 0);
  a.n_vec_dst = getd_ptrs(d, "vec_dst", "push: at most 8 vec_dst targets", a.vec_dst);
  a.mb_zero = getd<int>(d, "mb_zero", 0);
  a.grad = P<float>(getd<uintptr_t>(d, "grad", 0));
  a.loss_acc = P<float>(getd<uintptr_t>(d, "loss_acc", 0));
  a.loss_out = P<float>(getd<uintptr_t>(d, "loss_out", 0));
  a.done_dev = P<unsigned int>(getd<uintptr_t>(d, "done_dev", 0));
  a.segs = P<const SfTensorSeg>(getd<uintptr_t>(d, "segs", 0));
  a.tile_map = P<const int32_t>(getd<uintptr_t>(d, "tile_map", 0));
  a.num_tiles = getd<int>(d, "num_tiles", 0);
  a.optimizer = getd<int>(d, "optimizer", SF_OPT_SGD);
  a.lock_mode = getd<int>(d, "lock_mode", 0);
  a.drop = getd<int>(d, "drop", 0);
  a.scope_sys = getd<int>(d, "scope_sys", 1);
  a.grad_scale = getd<float>(d, "grad_scale", 1.0f);
  a.h = parse_hyper(getd<py::dict>(d, "hyper", py::dict()));
  a.replica_version = P<uint32_t>(getd<uintptr_t>(d, "replica_version", 0));
  if (a.replica_version && (a.lock_mode != SF_LOCK_RW || a.n_shadow_dst != 2 || a.shadow_is_mc))
    throw std::runtime_error("push: replica_version needs lock mode and the replica as the second of two publish destinations");
  {
    auto rows = getd<std::vector<std::vector<int64_t>>>(d, "seg_rows", {});
    if (!rows.empty() && rows.size() <= SF_MAX_INLINE_SEGS) {
      int acc = 0;
      for (size_t i = 0; i < rows.size(); ++i) {
        SfTensorSeg& sg = a.inline_segs[i];
        fill_seg(sg, rows[i], "push: seg_rows entries are (offset, rows, cols, w_off, w_ld, wt_off, wt_ld)");
        a.tile_prefix[i] = acc;
        acc += ((sg.rows + 31) / 32) * ((sg.cols + 63) / 64);
      }
      a.tile_prefix[rows.size()] = acc;
      a.n_inline_segs = static_cast<int>(rows.size());
      if (acc != a.num_tiles) throw std::runtime_error("push: seg_rows do not match num_tiles");
    }
  }
  if (!a.grad && getd<int>(d, "applier", 0)) a.grad = reinterpret_cast<float*>(16);   // never dereferenced by the applier
  if (!a.state || !a.ctrl || !a.grad || !a.segs || !a.tile_map || a.num_tiles <= 0)
    throw std::runtime_error("push: state/ctrl/grad/segs/tile_map/num_tiles are required");
  return a;
}

SfPostArgs parse_post(const py::dict& d) {
  SfPostArgs a;
  std::memset(&a, 0, sizeof(a));
  a.grad = P<float>(getd<uintptr_t>(d, "grad", 0));
  a.mailbox = P<float>(getd<uintptr_t>(d, "mailbox", 0));
  a.flags = P<uint32_t>(getd<uintptr_t>(d, "flags", 0));
  a.loss_acc = P<float>(getd<uintptr_t>(d, "loss_acc", 0));
  a.loss_out = P<float>(getd<uintptr_t>(d, "loss_out", 0));
  a.done_dev = P<unsigned int>(getd<uintptr_t>(d, "done_dev", 0));
  a.n = getd<size_t>(d, "n", 0);
  a.drop = getd<int>(d, "drop", 0);
  if (!a.grad || !a.mailbox || !a.flags || a.n == 0 || (a.n % 4)) throw std::runtime_error("post: grad/mailbox/flags/n (multiple of 4) are required");
  return a;
}

void fill_bounds(const py::dict& d, int n_shards, int* bounds) {
  auto b = getd<std::vector<int>>(d, "bounds", {});
  if (static_cast<int>(b.size()) != n_shards + 1) throw std::runtime_error("sharded: bounds must have n_shards + 1 entries");
  for (int i = 0; i <= n_shards; ++i) bounds[i] = b[i];
  for (int i = n_shards + 1; i <= SF_MAX_SHARDS; ++i) bounds[i] = b[n_shards];
}

SfSyncPullArgs parse_sync_pull(const py::dict& d) {
  SfSyncPullArgs a;
  std::memset(&a, 0, sizeof(a));
  a.n_shards = getd<int>(d, "n_shards", 0);
  if (a.n_shards < 1 || a.n_shards > SF_MAX_SHARDS) throw std::runtime_error("sync_pull: n_shards in [1, 8]");
  fill_bounds(d, a.n_shards, a.bounds);
  a.applied = P<const uint32_t>(getd<uintptr_t>(d, "applied", 0));
  a.my_posted = P<const uint32_t>(getd<uintptr_t>(d, "my_posted", 0));
  a.copy = getd<int>(d, "copy", 0);
  a.ver_begin = P<const uint32_t>(getd<uintptr_t>(d, "ver_begin", 0));
  a.ver_end = P<const uint32_t>(getd<uintptr_t>(d, "ver_end", 0));
  a.ver_stride = getd<int>(d, "ver_stride", 16);
  a.slot_off_bf16 = getd<long long>(d, "slot_off_bf16", 0);
  a.slot_off_f32 = getd<long long>(d, "slot_off_f32", 0);
  a.src = P<const __nv_bfloat16>(getd<uintptr_t>(d, "src", 0));
  a.dst = P<__nv_bfloat16>(getd<uintptr_t>(d, "dst", 0));
  a.src_vec = P<const float>(getd<uintptr_t>(d, "src_vec", 0));
  a.dst_vec = P<float>(getd<uintptr_t>(d, "dst_vec", 0));
  a.vec_offset = getd<long long>(d, "vec_offset", 0);
  a.segs = P<const SfTensorSeg>(getd<uintptr_t>(d, "segs", 0));
  a.tile_map = P<const int32_t>(getd<uintptr_t>(d, "tile_map", 0));
  a.ctas_per_shard = getd<int>(d, "ctas_per_shard", 1);
  a.sync = P<uint32_t>(getd<uintptr_t>(d, "sync", 0));
  a.stats = P<unsigned long long>(getd<uintptr_t>(d, "stats", 0));
  {
    auto ag = getd<std::vector<int>>(d, "ack_grid", {});
    if (static_cast<int>(ag.size()) != a.n_shards) throw std::runtime_error("sync_pull: one ack_grid entry per shard");
    for (int i = 0; i < a.n_shards; ++i) {
      if (ag[i] < 1) throw std::runtime_error("sync_pull: ack_grid entries must be >= 1");
      a.ack_grid[i] = ag[i];
    }
  }
  if (!a.applied || !a.my_posted) throw std::runtime_error("sync_pull: applied / my_posted are required");
  if (a.copy && (!a.ver_begin || !a.ver_end || !a.src || !a.dst || !a.segs || !a.tile_map || !a.sync || !a.slot_off_bf16 || !a.slot_off_f32))
    throw std::runtime_error("sync_pull: copy needs ver_begin/ver_end/src/dst/segs/tile_map/sync/slot_off_bf16/slot_off_f32");
  return a;
}

SfPostFlagsArgs parse_post_flags(const py::dict& d) {
  SfPostFlagsArgs a;
  std::memset(&a, 0, sizeof(a));
  a.n_shards = getd<int>(d, "n_shards", 0);
  if (a.n_shards < 1 || a.n_shards > SF_MAX_SHARDS) throw std::runtime_error("post_flags: n_shards in [1, 8]");
  fill_bounds(d, a.n_shards, a.bounds);
  const char* per_shard = "post_flags: one posted word and one mailbox per shard";
  if (getd_ptrs(d, "posted", per_shard, a.posted) != a.n_shards || getd_ptrs(d, "mailbox", per_shard, a.mailbox) != a.n_shards)
    throw std::runtime_error(per_shard);
  a.grad = P<float>(getd<uintptr_t>(d, "grad", 0));
  a.vec_tiles = P<const long long>(getd<uintptr_t>(d, "vec_tiles", 0));
  a.n_vec_tiles = getd<int>(d, "n_vec_tiles", 0);
  a.loss_acc = P<float>(getd<uintptr_t>(d, "loss_acc", 0));
  a.loss_out = P<float>(getd<uintptr_t>(d, "loss_out", 0));
  a.done_dev = P<unsigned int>(getd<uintptr_t>(d, "done_dev", 0));
  a.my_posted = P<uint32_t>(getd<uintptr_t>(d, "my_posted", 0));
  a.drop = getd<int>(d, "drop", 0);
  a.total = getd<long long>(d, "total", 0);
  a.mb_zero = getd<int>(d, "mb_zero", 0);
  a.phase = getd<int>(d, "phase", 0);
  a.heartbeat = P<unsigned long long>(getd<uintptr_t>(d, "heartbeat", 0));
  a.stats = P<unsigned long long>(getd<uintptr_t>(d, "stats", 0));
  if (!a.grad || !a.my_posted || (a.n_vec_tiles > 0 && !a.vec_tiles)) throw std::runtime_error("post_flags: grad / my_posted / vec_tiles are required");
  return a;
}

py::bytes pack_ryw(int n_shards, const std::vector<int>& ack_grid, uintptr_t applied, uintptr_t my_posted, uintptr_t stats) {
  SfRyw r;
  std::memset(&r, 0, sizeof(r));
  if (n_shards < 1 || n_shards > SF_MAX_SHARDS || static_cast<int>(ack_grid.size()) != n_shards) throw std::runtime_error("pack_ryw: n_shards in [1, 8], one grid size per shard");
  r.n_shards = n_shards;
  for (int i = 0; i < n_shards; ++i) {
    if (ack_grid[i] < 1) throw std::runtime_error("pack_ryw: grid sizes must be >= 1");
    r.ack_grid[i] = ack_grid[i];
  }
  r.applied = P<const uint32_t>(applied);
  r.my_posted = P<const uint32_t>(my_posted);
  r.stats = P<unsigned long long>(stats);
  return py::bytes(reinterpret_cast<const char*>(&r), sizeof(r));
}

// device-resident routing table of one worker (kept alive by the Python side)
py::bytes pack_route(int n_shards, const std::vector<int>& bounds, const std::vector<uintptr_t>& mailboxes) {
  SfRoute r;
  std::memset(&r, 0, sizeof(r));
  if (n_shards < 1 || n_shards > SF_MAX_SHARDS || static_cast<int>(bounds.size()) != n_shards + 1 || static_cast<int>(mailboxes.size()) != n_shards)
    throw std::runtime_error("pack_route: n_shards in [1, 8], n_shards + 1 bounds, n_shards mailboxes");
  r.n_shards = n_shards;
  for (int i = 0; i <= n_shards; ++i) r.bounds[i] = bounds[i];
  for (int i = n_shards + 1; i <= SF_MAX_SHARDS; ++i) r.bounds[i] = bounds[n_shards];
  for (int i = 0; i < n_shards; ++i) r.mailbox[i] = P<float>(mailboxes[i]);
  return py::bytes(reinterpret_cast<const char*>(&r), sizeof(r));
}

SfPullArgs parse_pull(const py::dict& d) {
  SfPullArgs a;
  std::memset(&a, 0, sizeof(a));
  a.src = P<const __nv_bfloat16>(getd<uintptr_t>(d, "src", 0));
  a.dst = P<__nv_bfloat16>(getd<uintptr_t>(d, "dst", 0));
  a.src_state = P<const float4>(getd<uintptr_t>(d, "src_state", 0));
  a.dst_f32 = P<float>(getd<uintptr_t>(d, "dst_f32", 0));
  a.n_bf16 = getd<size_t>(d, "n_bf16", 0);
  a.n_f32 = getd<size_t>(d, "n_f32", 0);
  a.ctrl = P<uint32_t>(getd<uintptr_t>(d, "ctrl", 0));
  a.seen_version = P<uint32_t>(getd<uintptr_t>(d, "seen_version", 0));
  a.lock_mode = getd<int>(d, "lock_mode", 0);
  a.scope_sys = getd<int>(d, "scope_sys", 1);
  a.wait_applied = P<const uint32_t>(getd<uintptr_t>(d, "wait_applied", 0));
  a.my_posted = P<const uint32_t>(getd<uintptr_t>(d, "my_posted", 0));
  a.dbuf = getd<int>(d, "dbuf", 0);
  a.src_alt = P<const __nv_bfloat16>(getd<uintptr_t>(d, "src_alt", 0));
  a.vec_pub[0] = P<const float>(getd<uintptr_t>(d, "vec_pub0", 0));
  a.vec_pub[1] = P<const float>(getd<uintptr_t>(d, "vec_pub1", 0));
  a.replica_version = P<const uint32_t>(getd<uintptr_t>(d, "replica_version", 0));
  if (a.replica_version && (a.lock_mode != SF_LOCK_RW || a.dbuf || a.wait_applied))
    throw std::runtime_error("pull: replica_version needs lock mode and a worker-applied push");
  if (a.dbuf && (!a.src_alt || (a.n_f32 && (!a.vec_pub[0] || !a.vec_pub[1])))) throw std::runtime_error("pull: dbuf needs src_alt and vec_pub0/1");
  if (a.wait_applied && !a.my_posted) throw std::runtime_error("pull: wait_applied needs my_posted");
  if (a.n_bf16 % 8) throw std::runtime_error("pull: bf16 size must be a 16-byte multiple");
  if (!a.ctrl) throw std::runtime_error("pull: ctrl is required");
  return a;
}

// ---------------------------------------------------------------------------
// Step plan: an ordered list of kernel launches, replayable as a CUDA graph.
// ---------------------------------------------------------------------------
class Plan {
 public:
  using Op = std::function<int(cudaStream_t)>;
  static constexpr int kMaxBranches = 3;
  Plan() {
    for (int i = 0; i < kMaxBranches; ++i) ev_[i] = nullptr;
  }
  ~Plan() {
    reset_graph();
    for (int i = 0; i < kMaxBranches; ++i) {
      if (ev_[i]) cudaEventDestroy(ev_[i]);      // branch streams are pooled per main stream and live for the process
    }
    if (ev_main_) cudaEventDestroy(ev_main_);
  }

  // ops added after branch(b) run on side stream b (0 = the caller's stream)
  void branch(int b) {
    if (b < 0 || b >= kMaxBranches) throw std::runtime_error("plan: bad branch id");
    cur_branch_ = b;
  }
  // side stream b waits for everything issued so far on the main stream
  void fork(int b) { add_ctl(1, b, "fork"); }
  // the main stream waits for everything issued so far on side stream b
  void join(int b) { add_ctl(2, b, "join"); }

  void add(std::string name, Op op) {
    items_.push_back(Item{std::move(name), std::move(op), cur_branch_, 0});
    reset_graph();
  }
  void add_gemm(std::shared_ptr<Gemm> g, const std::string& name) {
    add(name, [g](cudaStream_t st) { return sf_gemm_launch(&g->g, st); });
  }
  size_t size() const {
    size_t n = 0;
    for (auto& it : items_) n += it.kind == 0;
    return n;
  }
  std::vector<std::string> names() const {
    std::vector<std::string> v;
    for (auto& it : items_)
      if (it.kind == 0) v.push_back(it.branch ? it.name + "@" + std::to_string(it.branch) : it.name);
    return v;
  }

  void run(uintptr_t stream) {
    cudaStream_t main = S(stream);
    cur_main_ = main;
    for (auto& it : items_) {
      if (it.kind == 0) {
        const int rc = it.op(it.branch ? side(it.branch) : main);
        if (rc != 0) ck_rc(rc, it.name.c_str());
      } else if (it.kind == 1) {
        if (!ev_main_) ck(cudaEventCreateWithFlags(&ev_main_, cudaEventDisableTiming), "cudaEventCreate");
        ck(cudaEventRecord(ev_main_, main), "cudaEventRecord(fork)");
        ck(cudaStreamWaitEvent(side(it.branch), ev_main_, 0), "cudaStreamWaitEvent(fork)");
      } else {
        if (!ev_[it.branch]) ck(cudaEventCreateWithFlags(&ev_[it.branch], cudaEventDisableTiming), "cudaEventCreate");
        ck(cudaEventRecord(ev_[it.branch], side(it.branch)), "cudaEventRecord(join)");
        ck(cudaStreamWaitEvent(main, ev_[it.branch], 0), "cudaStreamWaitEvent(join)");
      }
    }
  }
  // Capture the op list once; later steps are a single cudaGraphLaunch.
  void capture(uintptr_t stream) {
    reset_graph();
    cudaStream_t st = S(stream);
    ck(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal), "cudaStreamBeginCapture");
    try {
      run(stream);
    } catch (...) {
      cudaGraph_t dead = nullptr;
      cudaStreamEndCapture(st, &dead);
      if (dead) cudaGraphDestroy(dead);
      throw;
    }
    ck(cudaStreamEndCapture(st, &graph_), "cudaStreamEndCapture");
    ck(cudaGraphInstantiate(&exec_, graph_, 0), "cudaGraphInstantiate");
  }
  bool captured() const { return exec_ != nullptr; }
  void replay(uintptr_t stream) {
    if (!exec_) throw std::runtime_error("plan not captured");
    ck(cudaGraphLaunch(exec_, S(stream)), "cudaGraphLaunch");
  }
  void replay_n(uintptr_t stream, int n) {
    if (!exec_) throw std::runtime_error("plan not captured");
    for (int i = 0; i < n; ++i) ck(cudaGraphLaunch(exec_, S(stream)), "cudaGraphLaunch");
  }
  size_t graph_nodes() const {
    size_t n = 0;
    if (graph_) cudaGraphGetNodes(graph_, nullptr, &n);
    return n;
  }

 private:
  struct Item {
    std::string name;
    Op op;
    int branch;
    int kind;   // 0 = kernel op, 1 = fork, 2 = join
  };
  void add_ctl(int kind, int b, const char* name) {
    if (b <= 0 || b >= kMaxBranches) throw std::runtime_error("plan: fork/join need a side branch id in [1,2]");
    items_.push_back(Item{name, nullptr, b, kind});
    reset_graph();
  }
  // Branch streams are POOLED per main stream (not per plan): a worker owns a handful of plans (staging slots, batch
  // shapes, forward-only variants) and the GPU has a limited number of hardware launch queues
  // (CUDA_DEVICE_MAX_CONNECTIONS): when more streams than queues exist, unrelated streams share a queue, and a kernel
  // that spins on a flag (a pull waiting for an applier) at the head of a queue blocks the launch of the very applier
  // kernel it is waiting for, if that one was mapped to the same queue.  Few streams -> no aliasing.
  static cudaStream_t pooled_side(cudaStream_t main, int b) {
    static std::mutex mu;
    static std::map<cudaStream_t, std::array<cudaStream_t, kMaxBranches>> pool;
    std::lock_guard<std::mutex> lk(mu);
    auto& arr = pool[main];          // value-initialised to nullptr on first use
    if (!arr[b]) ck(cudaStreamCreateWithFlags(&arr[b], cudaStreamNonBlocking), "cudaStreamCreate(side)");
    return arr[b];
  }
  cudaStream_t side(int b) { return pooled_side(cur_main_, b); }
  void reset_graph() {
    if (exec_) { cudaGraphExecDestroy(exec_); exec_ = nullptr; }
    if (graph_) { cudaGraphDestroy(graph_); graph_ = nullptr; }
  }
  std::vector<Item> items_;
  int cur_branch_ = 0;
  cudaStream_t cur_main_ = nullptr;
  cudaEvent_t ev_[kMaxBranches];
  cudaEvent_t ev_main_ = nullptr;
  cudaGraph_t graph_ = nullptr;
  cudaGraphExec_t exec_ = nullptr;
};

// ---------------------------------------------------------------------------
// StepDriver: the native inner loop of a worker.  For every step it copies the minibatch rows from
// the pinned host partition to the plan's staging buffers on the copy stream, makes the compute stream
// wait for that copy, replays the step's CUDA graph and reads the step's loss back into a pinned ring.
// Staging buffers are double-buffered by registering two plans (slot 0 / slot 1) per batch shape.
// ---------------------------------------------------------------------------
class StepDriver {
 public:
  StepDriver(uintptr_t compute_stream, uintptr_t copy_stream, uintptr_t x_host, size_t x_row_bytes, uintptr_t y_host,
             size_t y_row_bytes, uintptr_t loss_ring, int ring_len)
      : compute_(S(compute_stream)), copy_(S(copy_stream)), x_host_(P<const char>(x_host)), x_row_(x_row_bytes),
        y_host_(P<const char>(y_host)), y_row_(y_row_bytes), ring_(P<float>(loss_ring)), ring_len_(ring_len) {
    auto flag = [](const char* n) { const char* v = getenv(n); return v != nullptr && v[0] == '1'; };
    probe_ = flag("SPARKFLOW_DRV_PROBE");
    if (probe_) ck(cudaEventCreate(&base_), "cudaEventCreate(base)");
  }
  ~StepDriver() {
    for (auto& e : entries_) {
      if (e.ready) cudaEventDestroy(e.ready);
      if (e.free_) cudaEventDestroy(e.free_);
    }
  }
  // `prep` (optional, captured): prepares the step's operands from what was just staged; replayed on the copy stream
  // after the staging copies and before the step's ready event, so it overlaps the steps still in flight
  int add_plan(py::object plan, uintptr_t x_stage, uintptr_t y_stage, uintptr_t loss_out, int batch, py::object prep) {
    Entry e;
    e.keep = plan;
    e.plan = plan.cast<Plan*>();
    if (!e.plan->captured()) throw std::runtime_error("StepDriver: plan must be captured first");
    if (!prep.is_none()) {
      e.keep_prep = prep;
      e.prep = prep.cast<Plan*>();
      if (!e.prep->captured()) throw std::runtime_error("StepDriver: prep plan must be captured first");
    }
    e.x_stage = P<char>(x_stage);
    e.y_stage = P<char>(y_stage);
    e.loss_out = P<float>(loss_out);
    e.batch = batch;
    const unsigned int evf = probe_ ? cudaEventDefault : cudaEventDisableTiming;
    ck(cudaEventCreateWithFlags(&e.ready, evf), "cudaEventCreate");
    ck(cudaEventCreateWithFlags(&e.free_, evf), "cudaEventCreate");
    if (probe_) ck(cudaEventCreateWithFlags(&e.start, evf), "cudaEventCreate");
    entries_.push_back(e);
    return static_cast<int>(entries_.size()) - 1;
  }
  // contiguous minibatches: step k uses plan ids[k] on rows [starts[k], starts[k] + batch)
  void run(py::array_t<int32_t, py::array::c_style | py::array::forcecast> ids,
           py::array_t<int64_t, py::array::c_style | py::array::forcecast> starts) {
    const int n = static_cast<int>(ids.size());
    if (starts.size() != n) throw std::runtime_error("StepDriver.run: ids/starts length mismatch");
    const int32_t* ip = ids.data();
    const int64_t* sp = starts.data();
    py::gil_scoped_release nogil;
    using clk = std::chrono::steady_clock;
    auto ns = [](clk::time_point a, clk::time_point b) { return std::chrono::duration_cast<std::chrono::nanoseconds>(b - a).count(); };
    for (int k = 0; k < n; ++k) {
      if (ip[k] < 0 || ip[k] >= static_cast<int>(entries_.size())) throw std::runtime_error("StepDriver.run: bad plan id");
      Entry& e = entries_[ip[k]];
      const auto t0 = clk::now();
      if (e.primed) {
        wait_free(e);
        harvest(e);
      }
      const auto t1 = clk::now();
      if (probe_ && !base_recorded_) {
        ck(cudaEventRecord(base_, compute_), "cudaEventRecord(base)");
        base_recorded_ = true;
      }
      ck(cudaMemcpyAsync(e.x_stage, x_host_ + static_cast<size_t>(sp[k]) * x_row_, static_cast<size_t>(e.batch) * x_row_,
                         cudaMemcpyHostToDevice, copy_), "cudaMemcpyAsync(x)");
      if (e.y_stage && y_host_)
        ck(cudaMemcpyAsync(e.y_stage, y_host_ + static_cast<size_t>(sp[k]) * y_row_, static_cast<size_t>(e.batch) * y_row_,
                           cudaMemcpyHostToDevice, copy_), "cudaMemcpyAsync(y)");
      if (e.prep) e.prep->replay(reinterpret_cast<uintptr_t>(copy_));
      const auto t2 = clk::now();
      ck(cudaEventRecord(e.ready, copy_), "cudaEventRecord(ready)");
      ck(cudaStreamWaitEvent(compute_, e.ready, 0), "cudaStreamWaitEvent");
      if (probe_) ck(cudaEventRecord(e.start, compute_), "cudaEventRecord(start)");
      const auto t3 = clk::now();
      e.plan->replay(reinterpret_cast<uintptr_t>(compute_));
      const auto t4 = clk::now();
      // the step's last kernel stores the loss straight into this entry's pinned host word (zero-copy D2H: no
      // copy-engine operation on the compute stream); it is moved into the ring once the step has retired
      ck(cudaEventRecord(e.free_, compute_), "cudaEventRecord(free)");
      const auto t5 = clk::now();
      host_ns_[0] += ns(t0, t1); host_ns_[1] += ns(t1, t2); host_ns_[2] += ns(t2, t3); host_ns_[3] += ns(t3, t4); host_ns_[4] += ns(t4, t5);
      e.pending = step_;
      e.primed = true;
      ++step_;
    }
  }
  // ---- resident mode: the partition lives in HBM; a step's minibatch is `perm[start : start + batch]` (device int32
  // row ids), copied device-to-device into the plan's index buffer right before its graph, which gathers the rows
  // itself.  No PCIe traffic per step; completion is the pinned word written by the step's last kernel.
  void run_resident(py::array_t<int32_t, py::array::c_style | py::array::forcecast> ids,
                    py::array_t<int64_t, py::array::c_style | py::array::forcecast> starts, uintptr_t perm_dev) {
    const int n = static_cast<int>(ids.size());
    if (starts.size() != n) throw std::runtime_error("StepDriver.run_resident: ids/starts length mismatch");
    if (n == 0) return;
    const int32_t* ip = ids.data();
    const int64_t* sp = starts.data();
    const int32_t* perm = P<const int32_t>(perm_dev);
    py::gil_scoped_release nogil;
    // plans may also have been replayed by other paths: re-baseline the completion counters once per call
    ck(cudaStreamSynchronize(compute_), "cudaStreamSynchronize(resident)");
    for (auto& e : entries_) {
      harvest(e);
      e.launched = *(reinterpret_cast<volatile unsigned int*>(e.loss_out) + 1);
    }
    using clk = std::chrono::steady_clock;
    auto ns = [](clk::time_point a, clk::time_point b) { return std::chrono::duration_cast<std::chrono::nanoseconds>(b - a).count(); };
    for (int k = 0; k < n; ++k) {
      if (ip[k] < 0 || ip[k] >= static_cast<int>(entries_.size())) throw std::runtime_error("StepDriver.run_resident: bad plan id");
      Entry& e = entries_[ip[k]];
      const auto t0 = clk::now();
      if (e.primed && e.pending >= 0) wait_done(e);
      const auto t1 = clk::now();
      // the row ids of step k are staged on the COPY stream (the slot is free: its previous step has retired), so the
      // copy overlaps the steps still in flight and the step graph only waits on an event that has usually fired already
      ck(cudaMemcpyAsync(e.x_stage, perm + sp[k], static_cast<size_t>(e.batch) * sizeof(int32_t), cudaMemcpyDeviceToDevice, copy_),
         "cudaMemcpyAsync(minibatch row ids)");
      if (e.prep) e.prep->replay(reinterpret_cast<uintptr_t>(copy_));
      ck(cudaEventRecord(e.ready, copy_), "cudaEventRecord(ready)");
      ck(cudaStreamWaitEvent(compute_, e.ready, 0), "cudaStreamWaitEvent");
      const auto t2 = clk::now();
      e.plan->replay(reinterpret_cast<uintptr_t>(compute_));
      const auto t3 = clk::now();
      host_ns_[0] += ns(t0, t1); host_ns_[1] += ns(t1, t2); host_ns_[3] += ns(t2, t3);
      ++e.launched;
      e.pending = step_;
      e.primed = true;
      done_mode_ = true;
      ++step_;
    }
  }
  // host nanoseconds spent per phase since construction: wait-for-slot, H2D enqueue, event hand-off, graph launch, record
  std::vector<long long> host_ns() const { return std::vector<long long>(host_ns_, host_ns_ + 5); }
  std::vector<float> probe() const { return probe_rows_; }
  long long steps() const { return step_; }
  // wait for every in-flight step and move their losses into the ring
  void flush() {
    py::gil_scoped_release nogil;
    for (auto& e : entries_)
      if (e.primed && e.pending >= 0) {
        if (done_mode_) wait_done(e);
        else ck(cudaEventSynchronize(e.free_), "cudaEventSynchronize(flush)");
        harvest(e);
      }
  }

 private:
  struct Entry;
  // The loop thread never sleeps: a blocked thread's wake-up (tens of microseconds, more inside a VM) would land on
  // the critical path of the next step.  SPARKFLOW_DRIVER_BLOCK=1 restores cudaEventSynchronize.
  void wait_free(Entry& e) {
    static const bool block = [] { const char* v = getenv("SPARKFLOW_DRIVER_BLOCK"); return v != nullptr && v[0] == '1'; }();
    if (block) {
      ck(cudaEventSynchronize(e.free_), "cudaEventSynchronize(slot free)");
      return;
    }
    cudaError_t q;
    while ((q = cudaEventQuery(e.free_)) == cudaErrorNotReady) {
#if defined(__x86_64__)
      __builtin_ia32_pause();
#endif
    }
    ck(q, "cudaEventQuery(slot free)");
  }
  // resident mode: spin on the pinned completion word written by the step's last kernel (no CUDA call at all)
  void wait_done(Entry& e) {
    if (e.launched == 0) return;
    volatile unsigned int* done = reinterpret_cast<volatile unsigned int*>(e.loss_out) + 1;
    const auto t0 = std::chrono::steady_clock::now();
    unsigned long long spins = 0;
    while (static_cast<int>(*done - static_cast<unsigned int>(e.launched)) < 0) {
#if defined(__x86_64__)
      __builtin_ia32_pause();
#endif
      if ((++spins & 0xFFFFF) == 0) {
        if (cudaStreamQuery(compute_) != cudaErrorNotReady && static_cast<int>(*done - static_cast<unsigned int>(e.launched)) < 0 &&
            std::chrono::steady_clock::now() - t0 > std::chrono::seconds(5))
          throw std::runtime_error("StepDriver: the step's completion word never arrived (device error?)");
      }
    }
    if (e.pending >= 0) ring_[e.pending % ring_len_] = *const_cast<volatile float*>(e.loss_out);
    e.pending = -1;
  }
  void harvest(Entry& e) {
    if (probe_ && e.pending >= 0 && probe_rows_.size() < 4096 * 4) {
      float a = 0.f, b = 0.f, c = 0.f;
      cudaEventElapsedTime(&a, base_, e.ready);
      cudaEventElapsedTime(&b, base_, e.start);
      cudaEventElapsedTime(&c, base_, e.free_);
      probe_rows_.push_back(static_cast<float>(e.pending));
      probe_rows_.push_back(a * 1e3f);
      probe_rows_.push_back(b * 1e3f);
      probe_rows_.push_back(c * 1e3f);
    }
    if (e.pending >= 0) ring_[e.pending % ring_len_] = *const_cast<volatile float*>(e.loss_out);
    e.pending = -1;
  }
  struct Entry {
    long long pending = -1;
    unsigned long long launched = 0;      // resident mode: graph launches so far (the completion word counts them)
    py::object keep, keep_prep;
    Plan* plan = nullptr;
    Plan* prep = nullptr;
    char* x_stage = nullptr;
    char* y_stage = nullptr;
    float* loss_out = nullptr;
    int batch = 0;
    cudaEvent_t ready = nullptr, free_ = nullptr, start = nullptr;
    bool primed = false;
  };
  cudaStream_t compute_, copy_;
  const char* x_host_;
  size_t x_row_;
  const char* y_host_;
  size_t y_row_;
  float* ring_;
  int ring_len_;
  long long step_ = 0;
  long long host_ns_[5] = {0, 0, 0, 0, 0};
  bool probe_ = false, base_recorded_ = false, done_mode_ = false;
  cudaEvent_t base_ = nullptr;
  std::vector<float> probe_rows_;      // (step, H2D done, graph may start, graph done) in us since the first step
  std::vector<Entry> entries_;
};

// ---------------------------------------------------------------------------
// Applier: master side of the served push mode.  A host thread keeps `depth` finite poll-and-apply kernels
// queued on a dedicated high-priority stream (see applier_kernel in optim_push.cu).
// ---------------------------------------------------------------------------
class Applier {
 public:
  Applier(const py::dict& push, uintptr_t mailboxes, size_t mailbox_stride, uintptr_t flags, int n_workers, uintptr_t sync,
          double poll_window_s, int grid, int depth, int max_batch, uintptr_t shadow_alt, uintptr_t vec_pub_alt, const py::dict& shard)
      : grid_(grid), depth_(depth < 1 ? 1 : (depth > 16 ? 16 : depth)) {
    py::dict d(push);
    std::memset(&args_, 0, sizeof(args_));
    args_.push = parse_push(d);
    args_.mailboxes = P<float>(mailboxes);
    args_.mailbox_stride = mailbox_stride;
    args_.flags = P<uint32_t>(flags);
    args_.n_workers = n_workers;
    args_.sync = P<uint32_t>(sync);
    args_.idle_timeout_ns = static_cast<unsigned long long>(poll_window_s * 1e9);
    args_.max_batch = max_batch;
    args_.shadow_alt = P<__nv_bfloat16>(shadow_alt);
    args_.vec_pub_alt = P<float>(vec_pub_alt);
    args_.dbuf = shadow_alt != 0 ? 1 : 0;
    if (args_.dbuf && args_.push.n_vec_pub > 0 && !args_.vec_pub_alt) throw std::runtime_error("applier: dbuf needs vec_pub_alt");
    // sharded master (optional): tile range, remote acknowledgement words, seqlock stamps
    args_.tile_begin = getd<int>(shard, "tile_begin", 0);
    args_.tile_end = getd<int>(shard, "tile_end", 0);
    {
      const int n_ack = getd_ptrs(shard, "ack", "applier: at most 8 ack words", args_.ack);
      if (n_ack && n_ack != n_workers) throw std::runtime_error("applier: one ack word per worker, or none");
      for (int i = 0; i < n_ack; ++i)
        if (!args_.ack[i]) throw std::runtime_error("applier: ack words must be non-null");
      const char* ver = "applier: ver_begin / ver_end lists must match (<= 8)";
      args_.n_ver = getd_ptrs(shard, "ver_begin", ver, args_.ver_begin);
      if (getd_ptrs(shard, "ver_end", ver, args_.ver_end) != args_.n_ver) throw std::runtime_error(ver);
      args_.ver_mc = getd<int>(shard, "ver_mc", 0);
      args_.stats = P<unsigned long long>(getd<uintptr_t>(shard, "stats", 0));
      args_.linger = getd<int>(shard, "linger", 0);
      args_.ver_local = P<const uint32_t>(getd<uintptr_t>(shard, "ver_local", 0));
      args_.slot_off_bf16 = getd<long long>(shard, "slot_off_bf16", 0);
      args_.slot_off_f32 = getd<long long>(shard, "slot_off_f32", 0);
      if (args_.n_ver > 0 && (!n_ack || !args_.ver_local || !args_.slot_off_bf16 || !args_.slot_off_f32))
        throw std::runtime_error("applier: seqlock stamps need ack words, ver_local and both slot offsets");
    }
    ck(cudaGetDevice(&device_), "cudaGetDevice");
    int lo = 0, hi = 0;
    ck(cudaDeviceGetStreamPriorityRange(&lo, &hi), "cudaDeviceGetStreamPriorityRange");
    ck(cudaStreamCreateWithPriority(&stream_, cudaStreamNonBlocking, hi), "cudaStreamCreate(applier)");
    ck(cudaMemsetAsync(args_.sync, 0, 8 * sizeof(uint32_t), stream_), "cudaMemsetAsync(applier sync)");
    ck(cudaStreamSynchronize(stream_), "applier init");
    ck_rc(sf_preload_kernels(), "preload kernels");
    events_.resize(depth_);
    for (auto& e : events_) ck(cudaEventCreateWithFlags(&e, cudaEventDisableTiming), "cudaEventCreate");
    stop_.store(false);
    thread_ = std::thread([this]() { this->loop(); });
  }
  ~Applier() {
    try { stop(); } catch (...) {}
    for (auto& e : events_) if (e) cudaEventDestroy(e);
    if (stream_) cudaStreamDestroy(stream_);
  }
  bool alive() const { return thread_.joinable() && !failed_.load(); }
  long long launches() const { return static_cast<long long>(seq_.load()); }
  void stop() {
    if (!thread_.joinable()) return;
    stop_.store(true);
    {
      py::gil_scoped_release nogil;
      thread_.join();
    }
    if (failed_.load()) throw std::runtime_error("sparkflow_b200 applier thread failed: " + error_);
  }

 private:
  void loop() {
    if (cudaSetDevice(device_) != cudaSuccess) { failed_.store(true); error_ = "cudaSetDevice"; return; }
    unsigned int seq = 0;
    while (!stop_.load(std::memory_order_relaxed)) {
      const int slot = seq % depth_;
      if (seq >= static_cast<unsigned int>(depth_)) {
        const cudaError_t e = cudaEventSynchronize(events_[slot]);      // the launch `depth` ago has retired
        if (e != cudaSuccess) { failed_.store(true); error_ = cudaGetErrorString(e); return; }
      }
      ++seq;
      const int rc = sf_applier_launch(&args_, seq, grid_, stream_);
      if (rc != 0) { failed_.store(true); error_ = "applier launch failed"; return; }
      cudaEventRecord(events_[slot], stream_);
      seq_.store(seq);
    }
    cudaStreamSynchronize(stream_);
  }
  SfApplierArgs args_;
  int grid_, depth_, device_ = 0;
  cudaStream_t stream_ = nullptr;
  std::vector<cudaEvent_t> events_;
  std::thread thread_;
  std::atomic<bool> stop_{false}, failed_{false};
  std::atomic<unsigned int> seq_{0};
  std::string error_;
};

// ---------------------------------------------------------------------------
// CUDA-IPC symmetric memory: cudaMalloc'ed segments exported to the peer processes of the box.
// ---------------------------------------------------------------------------
uintptr_t ipc_alloc(size_t bytes) {
  void* p = nullptr;
  ck(cudaMalloc(&p, bytes), "cudaMalloc(symmetric segment)");
  ck(cudaMemset(p, 0, bytes), "cudaMemset(symmetric segment)");
  return reinterpret_cast<uintptr_t>(p);
}
void ipc_free(uintptr_t p) { cudaFree(P<void>(p)); }
py::bytes ipc_get_handle(uintptr_t p) {
  cudaIpcMemHandle_t h;
  ck(cudaIpcGetMemHandle(&h, P<void>(p)), "cudaIpcGetMemHandle");
  return py::bytes(reinterpret_cast<const char*>(&h), sizeof(h));
}
uintptr_t ipc_open_handle(const std::string& raw) {
  if (raw.size() != sizeof(cudaIpcMemHandle_t)) throw std::runtime_error("bad IPC handle size");
  cudaIpcMemHandle_t h;
  std::memcpy(&h, raw.data(), sizeof(h));
  void* p = nullptr;
  ck(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle");
  return reinterpret_cast<uintptr_t>(p);
}
void ipc_close_handle(uintptr_t p) { cudaIpcCloseMemHandle(P<void>(p)); }

bool enable_peer_access(int peer) {
  int dev = 0;
  ck(cudaGetDevice(&dev), "cudaGetDevice");
  if (dev == peer) return true;
  int can = 0;
  ck(cudaDeviceCanAccessPeer(&can, dev, peer), "cudaDeviceCanAccessPeer");
  if (!can) return false;
  cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return true; }
  ck(e, "cudaDeviceEnablePeerAccess");
  return true;
}

py::bytes pack_segs(const std::vector<std::vector<int64_t>>& rows) {
  std::vector<SfTensorSeg> v(rows.size());
  for (size_t i = 0; i < rows.size(); ++i) {
    fill_seg(v[i], rows[i], "pack_segs: (offset, rows, cols, w_off, w_ld, wt_off, wt_ld)");
    if (v[i].w_off >= 0 && ((v[i].w_ld % 8) || (v[i].w_off % 8))) throw std::runtime_error("pack_segs: w_ld / w_off must be multiples of 8");
    if (v[i].wt_off >= 0 && ((v[i].wt_ld % 8) || (v[i].wt_off % 8))) throw std::runtime_error("pack_segs: wt_ld / wt_off must be multiples of 8");
  }
  return py::bytes(reinterpret_cast<const char*>(v.data()), v.size() * sizeof(SfTensorSeg));
}

// ---------------------------------------------------------------------------
// Kernel launchers: each takes a kernel's Python-facing arguments (device addresses, sizes; the dict-driven ops parse
// and check their dict here, once) and returns the launch as a callable of the stream that returns the sf_* rc.  A plan
// keeps the callable and calls it on every run; the direct entry point calls it right away (see def_kernel).
// ---------------------------------------------------------------------------
namespace launch {

// The `act` argument of the stand-alone backward / loss kernels: the SfAct in its low 32 bits and, for a leaky ReLU, the
// fp32 bits of its slope in the high 32 (0 otherwise), so these bindings keep their signatures.
int act_kind(long long act) { return static_cast<int>(act & 0xffffffffLL); }
float act_alpha(long long act) {
  const uint32_t bits = static_cast<uint32_t>(static_cast<unsigned long long>(act) >> 32);
  float a;
  std::memcpy(&a, &bits, sizeof(a));
  return a;
}

auto cast_transpose(uintptr_t in, int ld_in, uintptr_t idx, uintptr_t out, int ld_out, uintptr_t outT, int ld_t, int rows, int cols) {
  return [=](cudaStream_t st) {
    return idx ? sf_gather_cast_transpose(P<const float>(in), ld_in, P<const int32_t>(idx), P<__nv_bfloat16>(out), ld_out,
                                          P<__nv_bfloat16>(outT), ld_t, rows, cols, st)
               : sf_cast_transpose(P<const float>(in), ld_in, P<__nv_bfloat16>(out), ld_out, P<__nv_bfloat16>(outT), ld_t, rows, cols, st);
  };
}
// softmax_xent takes one-hot / soft label rows, or one class index per row: a label row narrower than the logits row
// (ld_labels < cols) cannot be a distribution over the classes, so it is read as one class index per row, at stride
// ld_labels (sf_sparse_softmax_xent), and this binding keeps its signature.
auto softmax_xent(uintptr_t logits, int ld_logits, uintptr_t labels, int ld_labels, uintptr_t loss, uintptr_t dz, int ld_dz,
                  uintptr_t dzT, int ld_t, uintptr_t dbias, int rows, int cols) {
  return [=](cudaStream_t st) {
    if (ld_labels < cols)
      return sf_sparse_softmax_xent(P<const float>(logits), ld_logits, P<const float>(labels), ld_labels, P<float>(loss),
                                    P<__nv_bfloat16>(dz), ld_dz, P<__nv_bfloat16>(dzT), ld_t, P<float>(dbias), rows, cols, st);
    return sf_softmax_xent(P<const float>(logits), ld_logits, P<const float>(labels), ld_labels, P<float>(loss), P<__nv_bfloat16>(dz),
                           ld_dz, P<__nv_bfloat16>(dzT), ld_t, P<float>(dbias), rows, cols, st);
  };
}
auto mse(uintptr_t out, int ld_out, uintptr_t target, int ld_target, long long act, uintptr_t loss, uintptr_t dz, int ld_dz, uintptr_t dzT,
         int ld_t, uintptr_t dbias, int rows, int cols) {
  return [=](cudaStream_t st) {
    return sf_mse_loss(P<const float>(out), ld_out, P<const float>(target), ld_target, act_kind(act), act_alpha(act), P<float>(loss), P<__nv_bfloat16>(dz), ld_dz,
                       P<__nv_bfloat16>(dzT), ld_t, P<float>(dbias), rows, cols, st);
  };
}
auto sigmoid_xent(uintptr_t logits, int ld_logits, uintptr_t labels, int ld_labels, uintptr_t loss, uintptr_t dz, int ld_dz,
                  uintptr_t dzT, int ld_t, uintptr_t dbias, int rows, int cols) {
  return [=](cudaStream_t st) {
    return sf_sigmoid_xent(P<const float>(logits), ld_logits, P<const float>(labels), ld_labels, P<float>(loss), P<__nv_bfloat16>(dz),
                           ld_dz, P<__nv_bfloat16>(dzT), ld_t, P<float>(dbias), rows, cols, st);
  };
}
auto argmax(uintptr_t in, int ld, uintptr_t out, int rows, int cols) {
  return [=](cudaStream_t st) { return sf_argmax_rows(P<const float>(in), ld, P<float>(out), rows, cols, st); };
}
auto im2col(uintptr_t in, int n, int h, int w, int c, int kh, int kw, uintptr_t out, int ld_out, uintptr_t outT, int ld_t, int sh, int sw,
            int pad_top, int pad_left, int out_h, int out_w) {
  return [=](cudaStream_t st) {
    return sf_im2col_nhwc(P<const __nv_bfloat16>(in), n, h, w, c, kh, kw, sh, sw, pad_top, pad_left, out_h, out_w, P<__nv_bfloat16>(out),
                          ld_out, P<__nv_bfloat16>(outT), ld_t, st);
  };
}
auto col2im(uintptr_t dcols, int ld_cols, int n, int h, int w, int c, int kh, int kw, uintptr_t din, int sh, int sw, int pad_top,
            int pad_left, int out_h, int out_w) {
  return [=](cudaStream_t st) {
    return sf_col2im_nhwc(P<const __nv_bfloat16>(dcols), ld_cols, n, h, w, c, kh, kw, sh, sw, pad_top, pad_left, out_h, out_w,
                          P<__nv_bfloat16>(din), st);
  };
}
auto maxpool_fwd(uintptr_t in, int n, int h, int w, int c, uintptr_t out, uintptr_t argmax, uintptr_t outT, int ld_t) {
  return [=](cudaStream_t st) {
    return sf_maxpool2_fwd(P<const __nv_bfloat16>(in), n, h, w, c, P<__nv_bfloat16>(out), P<uint8_t>(argmax), P<__nv_bfloat16>(outT), ld_t, st);
  };
}
auto maxpool_bwd(uintptr_t dout, uintptr_t argmax, int n, int h, int w, int c, uintptr_t act_out, long long act, uintptr_t dz, int ld_dz,
                 uintptr_t dzT, int ld_t, uintptr_t dbias) {
  return [=](cudaStream_t st) {
    return sf_maxpool2_bwd(P<const __nv_bfloat16>(dout), P<const uint8_t>(argmax), n, h, w, c, P<const __nv_bfloat16>(act_out), act_kind(act),
                           act_alpha(act), P<__nv_bfloat16>(dz), ld_dz, P<__nv_bfloat16>(dzT), ld_t, P<float>(dbias), st);
  };
}
auto maxpool_gen_fwd(uintptr_t in, int n, int h, int w, int c, int kh, int kw, int sh, int sw, int pad_top, int pad_left, int out_h,
                     int out_w, uintptr_t out, uintptr_t argmax) {
  return [=](cudaStream_t st) {
    return sf_maxpool_fwd(P<const __nv_bfloat16>(in), n, h, w, c, kh, kw, sh, sw, pad_top, pad_left, out_h, out_w, P<__nv_bfloat16>(out),
                          P<uint8_t>(argmax), st);
  };
}
auto maxpool_gen_bwd(uintptr_t dout, uintptr_t argmax, int n, int h, int w, int c, int kh, int kw, int sh, int sw, int pad_top,
                     int pad_left, int out_h, int out_w, uintptr_t act_out, long long act, uintptr_t dz, int ld_dz, uintptr_t dbias) {
  return [=](cudaStream_t st) {
    return sf_maxpool_bwd(P<const __nv_bfloat16>(dout), P<const uint8_t>(argmax), n, h, w, c, kh, kw, sh, sw, pad_top, pad_left, out_h,
                          out_w, P<const __nv_bfloat16>(act_out), act_kind(act), act_alpha(act), P<__nv_bfloat16>(dz), ld_dz,
                          P<float>(dbias), st);
  };
}
auto act_bwd_bias(uintptr_t g, int ld_g, int rows, int c, uintptr_t act_out, long long act, uintptr_t dz, int ld_dz, uintptr_t dbias) {
  return [=](cudaStream_t st) {
    return sf_act_bwd_bias(P<const __nv_bfloat16>(g), ld_g, rows, c, P<const __nv_bfloat16>(act_out), act_kind(act), act_alpha(act),
                           P<__nv_bfloat16>(dz), ld_dz,
                           P<float>(dbias), st);
  };
}
auto conv_first_fwd(uintptr_t x, int n, int h, int w, int cin, int kh, int kw, int cout, uintptr_t wT, int ld_w, uintptr_t bias, int act,
                    uintptr_t pooled, uintptr_t argmax, int pad_top, int pad_left, int out_h, int out_w) {
  return [=](cudaStream_t st) {
    return sf_conv_first_fwd(P<const __nv_bfloat16>(x), n, h, w, cin, kh, kw, cout, P<const __nv_bfloat16>(wT), ld_w, P<const float>(bias),
                             act, P<__nv_bfloat16>(pooled), P<uint8_t>(argmax), pad_top, pad_left, out_h, out_w, st);
  };
}
auto conv_first_wgrad(uintptr_t x, int n, int h, int w, int cin, int kh, int kw, int cout, uintptr_t g_pool, uintptr_t pooled,
                      uintptr_t argmax, int act, uintptr_t dW, uintptr_t db, int pad_top, int pad_left, int out_h, int out_w) {
  return [=](cudaStream_t st) {
    return sf_conv_first_wgrad(P<const __nv_bfloat16>(x), n, h, w, cin, kh, kw, cout, P<const __nv_bfloat16>(g_pool),
                               P<const __nv_bfloat16>(pooled), P<const uint8_t>(argmax), act, P<float>(dW), P<float>(db), pad_top, pad_left,
                               out_h, out_w, st);
  };
}
auto push(const py::dict& d, uintptr_t local_sync, int grid) {
  const SfPushArgs a = parse_push(d);
  return [=](cudaStream_t st) { return sf_push_launch(&a, P<uint32_t>(local_sync), grid, st); };
}
auto post(const py::dict& d, uintptr_t local_sync, int grid) {
  const SfPostArgs a = parse_post(d);
  return [=](cudaStream_t st) { return sf_post_launch(&a, P<uint32_t>(local_sync), grid, st); };
}
auto pull(const py::dict& d, uintptr_t local_sync, int grid) {
  const SfPullArgs a = parse_pull(d);
  return [=](cudaStream_t st) { return sf_pull_launch(&a, P<uint32_t>(local_sync), grid, st); };
}
auto sync_pull(const py::dict& d) {
  const SfSyncPullArgs a = parse_sync_pull(d);
  return [=](cudaStream_t st) { return sf_sync_pull_launch(&a, st); };
}
auto post_flags(const py::dict& d) {
  const SfPostFlagsArgs a = parse_post_flags(d);
  return [=](cudaStream_t st) { return sf_post_flags_launch(&a, st); };
}

}  // namespace launch

// the direct entry point of `launch`: its arguments with the stream inserted before the last sizeof...(J) of them
template <class L, class... A, size_t... I, size_t... J>
auto direct_entry(const char* name, L (*launch)(A...), std::index_sequence<I...>, std::index_sequence<J...>) {
  using Args = std::tuple<A...>;
  return [name, launch](std::tuple_element_t<I, Args>... lead, uintptr_t stream,
                        std::tuple_element_t<sizeof...(I) + J, Args>... trail) { ck_rc(launch(lead..., trail...)(S(stream)), name); };
}

// Binds one kernel's launcher twice: as the plan op Plan.add_<plan_name>(args...) and as the direct entry point
// <direct_name>(args..., stream), which launches at once and raises if the launch fails.  `names` are the keyword names
// of the leading arguments and `defaults` those of the trailing defaulted ones; the direct form takes its stream between
// the two.  Bound without them, the arguments are positional and the stream comes last.
template <class L, class... A, class... N, class... D>
void def_kernel(py::module_& m, py::class_<Plan>& plan, const char* plan_name, const char* direct_name, L (*launch)(A...),
                std::tuple<N...> names, std::tuple<D...> defaults) {
  auto add = [plan_name, launch](Plan& p, A... a) { p.add(plan_name, launch(a...)); };
  auto now = direct_entry(direct_name, launch, std::make_index_sequence<sizeof...(A) - sizeof...(D)>(),
                          std::make_index_sequence<sizeof...(D)>());
  const std::string add_name = std::string("add_") + plan_name;
  std::apply([&](const auto&... x) { plan.def(add_name.c_str(), add, x...); }, std::tuple_cat(names, defaults));
  if constexpr (sizeof...(N) + sizeof...(D) == 0)
    m.def(direct_name, now);
  else
    std::apply([&](const auto&... x) { m.def(direct_name, now, x...); }, std::tuple_cat(names, std::make_tuple(py::arg("stream")), defaults));
}
template <class L, class... A>
void def_kernel(py::module_& m, py::class_<Plan>& plan, const char* plan_name, const char* direct_name, L (*launch)(A...)) {
  def_kernel(m, plan, plan_name, direct_name, launch, std::tuple<>(), std::tuple<>());
}

}  // namespace

PYBIND11_MODULE(_C, m) {
  m.doc() = "sparkflow_b200 native runtime (sm_90a kernels + step-plan runner)";
  m.attr("ARCH") = "sm_90a";
  m.attr("CTRL_WORDS") = static_cast<int>(SF_CTRL_WORDS);
  m.attr("CTRL_PUB") = static_cast<int>(SF_CTRL_PUB);
  m.attr("SEG_BYTES") = static_cast<int>(sizeof(SfTensorSeg));
  m.attr("PUSH_TILE_R") = 32;
  m.attr("PUSH_TILE_C") = 64;

  py::class_<Gemm, std::shared_ptr<Gemm>>(m, "Gemm")
      .def(py::init<const py::dict&>())
      .def("launch", &Gemm::launch)
      .def_property_readonly("bn", &Gemm::bn)
      .def_property_readonly("split_k", &Gemm::split_k)
      .def_property_readonly("kblocks_per_split", &Gemm::kblocks_per_split)
      .def_property_readonly("pair", &Gemm::pair)
      .def_property_readonly("epi", &Gemm::epi)
      .def("mn_major", &Gemm::mn_major)
      .def_property_readonly("grid", &Gemm::grid);

  py::class_<Plan> plan(m, "Plan");
  plan.def(py::init<>())
      .def("__len__", &Plan::size)
      .def("names", &Plan::names)
      .def("run", &Plan::run)
      .def("capture", &Plan::capture)
      .def("captured", &Plan::captured)
      .def("replay", &Plan::replay)
      .def("replay_n", &Plan::replay_n, py::call_guard<py::gil_scoped_release>())
      .def("branch", &Plan::branch)
      .def("fork", &Plan::fork)
      .def("join", &Plan::join)
      .def("graph_nodes", &Plan::graph_nodes)
      .def("add_gemm", &Plan::add_gemm, py::arg("gemm"), py::arg("name") = "gemm")
      .def("add_gather_rows",
           [](Plan& p, uintptr_t in, int ld_in, uintptr_t idx, uintptr_t out, int ld_out, int rows, int cols) {
             p.add("gather_rows", [=](cudaStream_t st) {
               return sf_gather_rows_f32(P<const float>(in), ld_in, P<const int32_t>(idx), P<float>(out), ld_out, rows, cols, st);
             });
           });

  // every kernel below is a plan op (Plan.add_<first name>) and a direct entry point (_C.<second name>, used by tests and
  // the eager paths)
  def_kernel(m, plan, "cast_transpose", "cast_transpose", launch::cast_transpose);
  def_kernel(m, plan, "softmax_xent", "softmax_xent", launch::softmax_xent);
  def_kernel(m, plan, "mse", "mse_loss", launch::mse);
  def_kernel(m, plan, "sigmoid_xent", "sigmoid_xent", launch::sigmoid_xent);
  def_kernel(m, plan, "argmax", "argmax_rows", launch::argmax);
  def_kernel(m, plan, "maxpool_fwd", "maxpool_fwd", launch::maxpool_fwd);
  def_kernel(m, plan, "maxpool_bwd", "maxpool_bwd", launch::maxpool_bwd);
  def_kernel(m, plan, "maxpool_gen_fwd", "maxpool_gen_fwd", launch::maxpool_gen_fwd);
  def_kernel(m, plan, "maxpool_gen_bwd", "maxpool_gen_bwd", launch::maxpool_gen_bwd);
  def_kernel(m, plan, "act_bwd_bias", "act_bwd_bias", launch::act_bwd_bias);
  def_kernel(m, plan, "push", "push", launch::push);
  def_kernel(m, plan, "post", "post", launch::post);
  def_kernel(m, plan, "pull", "pull", launch::pull);
  def_kernel(m, plan, "sync_pull", "sync_pull", launch::sync_pull);
  def_kernel(m, plan, "post_flags", "post_flags", launch::post_flags);
  // conv geometry (stride, pad_top / pad_left, output size) trails the stream argument; the defaults are VALID stride 1
  const auto pads = std::make_tuple(py::arg("pad_top") = 0, py::arg("pad_left") = 0, py::arg("out_h") = 0, py::arg("out_w") = 0);
  const auto geometry = std::tuple_cat(std::make_tuple(py::arg("sh") = 1, py::arg("sw") = 1), pads);
  def_kernel(m, plan, "im2col", "im2col", launch::im2col,
             std::make_tuple(py::arg("in"), py::arg("n"), py::arg("h"), py::arg("w"), py::arg("c"), py::arg("kh"), py::arg("kw"), py::arg("out"),
                             py::arg("ld_out"), py::arg("outT"), py::arg("ld_t")),
             geometry);
  def_kernel(m, plan, "col2im", "col2im", launch::col2im,
             std::make_tuple(py::arg("dcols"), py::arg("ld_cols"), py::arg("n"), py::arg("h"), py::arg("w"), py::arg("c"), py::arg("kh"),
                             py::arg("kw"), py::arg("din")),
             geometry);
  def_kernel(m, plan, "conv_first_fwd", "conv_first_fwd", launch::conv_first_fwd,
             std::make_tuple(py::arg("x"), py::arg("n"), py::arg("h"), py::arg("w"), py::arg("cin"), py::arg("kh"), py::arg("kw"), py::arg("cout"),
                             py::arg("wT"), py::arg("ld_w"), py::arg("bias"), py::arg("act"), py::arg("pooled"), py::arg("argmax")),
             pads);
  def_kernel(m, plan, "conv_first_wgrad", "conv_first_wgrad", launch::conv_first_wgrad,
             std::make_tuple(py::arg("x"), py::arg("n"), py::arg("h"), py::arg("w"), py::arg("cin"), py::arg("kh"), py::arg("kw"), py::arg("cout"),
                             py::arg("g_pool"), py::arg("pooled"), py::arg("argmax"), py::arg("act"), py::arg("dW"), py::arg("db")),
             pads);

  py::class_<Applier>(m, "Applier")
      .def(py::init<const py::dict&, uintptr_t, size_t, uintptr_t, int, uintptr_t, double, int, int, int, uintptr_t, uintptr_t, const py::dict&>(), py::arg("push"), py::arg("mailboxes"),
           py::arg("mailbox_stride"), py::arg("flags"), py::arg("n_workers"), py::arg("sync"), py::arg("poll_window_s") = 30e-6,
           py::arg("grid") = 96, py::arg("depth") = 3, py::arg("max_batch") = 8, py::arg("shadow_alt") = 0, py::arg("vec_pub_alt") = 0,
           py::arg("shard") = py::dict())
      .def("alive", &Applier::alive)
      .def("launches", &Applier::launches)
      .def("stop", &Applier::stop);
  m.attr("MB_WORDS") = static_cast<int>(SF_MB_WORDS);
  m.attr("MB_APPLIED") = static_cast<int>(SF_MB_APPLIED);

  py::class_<StepDriver>(m, "StepDriver")
      .def(py::init<uintptr_t, uintptr_t, uintptr_t, size_t, uintptr_t, size_t, uintptr_t, int>())
      .def("add_plan", &StepDriver::add_plan, py::arg("plan"), py::arg("x_stage"), py::arg("y_stage"), py::arg("loss_out"),
           py::arg("batch"), py::arg("prep") = py::none())
      .def("run", &StepDriver::run)
      .def("steps", &StepDriver::steps)
      .def("flush", &StepDriver::flush)
      .def("run_resident", &StepDriver::run_resident)
      .def("host_ns", &StepDriver::host_ns)
      .def("probe", &StepDriver::probe);

  m.def("lock_op", [](uintptr_t ctrl, int op, uintptr_t stream) {
    ck_rc(sf_lock_test(P<uint32_t>(ctrl), op, S(stream)), "lock_op");
  });
  m.def("gemm_pick_bn", &sf_gemm_pick_bn);
  m.def("set_pdl", &sf_set_pdl);
  m.def("trace_enable", [](uintptr_t buf, unsigned int cap) { ck_rc(sf_trace_enable(P<void>(buf), cap), "trace_enable"); });
  m.def("trace_count", &sf_trace_count);
  m.attr("TRACE_REC_BYTES") = 32;
  m.def("read_error_code", &sf_read_error_code);
  m.def("init_error_channel", []() {
    ck_rc(sf_init_error_channel(), "init_error_channel");
    ck_rc(sf_preload_kernels(), "preload kernels");        // no lazy module load in the middle of a run
  });
  m.def("read_host_error_code", &sf_read_host_error_code);
  m.def("pack_segs", &pack_segs);

  m.def("pack_route", &pack_route);
  m.def("pack_ryw", &pack_ryw);
  m.attr("MAX_SHARDS") = static_cast<int>(SF_MAX_SHARDS);
  // symmetric (VMM) memory + NVSwitch multicast
  m.def("vmm_granularity", &sfvmm::granularity, py::arg("device"), py::arg("multicast") = false, py::arg("n_devices") = 1);
  m.def("vmm_multicast_supported", &sfvmm::multicast_supported);
  m.def("vmm_create", &sfvmm::create);
  m.def("vmm_release", &sfvmm::release);
  m.def("vmm_export_fd", &sfvmm::export_fd);
  m.def("vmm_import_fd", &sfvmm::import_fd);
  m.def("vmm_map", &sfvmm::map);
  m.def("vmm_unmap", &sfvmm::unmap);
  m.def("mc_create", &sfvmm::mc_create);
  m.def("mc_add_device", &sfvmm::mc_add_device);
  m.def("mc_bind", &sfvmm::mc_bind);
  m.def("mc_unbind", &sfvmm::mc_unbind);
  m.def("memset_d8", [](uintptr_t p, int value, size_t bytes) { ck(cudaMemset(P<void>(p), value, bytes), "cudaMemset"); });

  m.def("ipc_alloc", &ipc_alloc);
  m.def("ipc_free", &ipc_free);
  m.def("ipc_get_handle", &ipc_get_handle);
  m.def("ipc_open_handle", &ipc_open_handle);
  m.def("ipc_close_handle", &ipc_close_handle);
  m.def("enable_peer_access", &enable_peer_access);
  m.def("device_count", []() { int n = 0; return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0; });
}
