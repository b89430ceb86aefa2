// capi_frontier.cu — demi_dpor_frontier: one DPORwHeuristics search as a frontier of backtrack points (K3F), and the
// communicator behind it.  Host side of frontier_kernel.cuh: the round loop, the queue directory (a round's points
// are one sorted run; the queue is the runs, indexed by branch depth), the steal plan and its NCCL exchange.
// Semantics: include/demi_b200.h (the tests hold a sequential CPU restatement of the same protocol).
#include <dlfcn.h>
#include <deque>
#include <thread>
#include <chrono>
#include <nccl.h>                    // types only: the library is bound with dlopen (no link-time dependency)
#include "frontier_kernel.cuh"
#include "models/model_ir.cuh"
#include "engine.hpp"

using namespace demi;

// --------------------------------------------------------------------------------------------------- NCCL binding
namespace {
struct NcclApi {
  void* lib = nullptr;
  decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
  decltype(&ncclCommInitRank) CommInitRank = nullptr;
  decltype(&ncclCommDestroy) CommDestroy = nullptr;
  decltype(&ncclAllGather) AllGather = nullptr;
  decltype(&ncclSend) Send = nullptr;
  decltype(&ncclRecv) Recv = nullptr;
  decltype(&ncclGroupStart) GroupStart = nullptr;
  decltype(&ncclGroupEnd) GroupEnd = nullptr;
  decltype(&ncclGetErrorString) GetErrorString = nullptr;
  std::string err;
};
NcclApi* nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (tried) return &api;
  tried = true;
  // a host that already loaded NCCL (torch ships its own) gets that copy: same soname
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) { api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (api.lib) break; }
  if (!api.lib) { api.err = "libnccl.so.2 not found"; return &api; }
#define BIND(name) api.name = (decltype(api.name))dlsym(api.lib, "nccl" #name); if (!api.name) api.err = "nccl" #name " missing";
  BIND(GetUniqueId) BIND(CommInitRank) BIND(CommDestroy) BIND(AllGather) BIND(Send) BIND(Recv) BIND(GroupStart) BIND(GroupEnd)
  BIND(GetErrorString)
#undef BIND
  return &api;
}
#define NCCL_TRY(h, expr) do { ncclResult_t r_ = (expr); if (r_ != ncclSuccess) \
  return fail((h), DEMI_ERR_CUDA, "%s: %s", #expr, nccl_api()->GetErrorString(r_)); } while (0)
}  // namespace
struct FrComm { ncclComm_t comm = nullptr; int rank = 0, world = 1; };

extern "C" int32_t demi_comm_unique_id(uint8_t id[DEMI_COMM_ID_BYTES]) {
  NcclApi* a = nccl_api();
  if (!a->err.empty()) return fail(nullptr, DEMI_ERR_NO_DEVICE, "demi_comm_unique_id: %s", a->err.c_str());
  static_assert(sizeof(ncclUniqueId) == DEMI_COMM_ID_BYTES, "ncclUniqueId size");
  ncclUniqueId u;
  ncclResult_t r = a->GetUniqueId(&u);
  if (r != ncclSuccess) return fail(nullptr, DEMI_ERR_CUDA, "ncclGetUniqueId: %s", a->GetErrorString(r));
  memcpy(id, &u, sizeof(u));
  return DEMI_OK;
}
extern "C" int32_t demi_comm_init(demi_handle* h, const uint8_t id[DEMI_COMM_ID_BYTES], int32_t rank, int32_t world) {
  if (!h || !id) return DEMI_ERR_INVALID;
  if (world < 1 || world > 64 || rank < 0 || rank >= world) return fail(h, DEMI_ERR_INVALID, "demi_comm_init: rank %d of %d", rank, world);
  if (h->comm) return fail(h, DEMI_ERR_STATE, "demi_comm_init: the handle already has a communicator");
  NcclApi* a = nccl_api();
  if (!a->err.empty()) return fail(h, DEMI_ERR_NO_DEVICE, "demi_comm_init: %s", a->err.c_str());
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  ncclUniqueId u; memcpy(&u, id, sizeof(u));
  FrComm* c = new FrComm();
  c->rank = rank; c->world = world;
  ncclResult_t r = a->CommInitRank(&c->comm, world, u, rank);
  if (r != ncclSuccess) { delete c; return fail(h, DEMI_ERR_CUDA, "ncclCommInitRank: %s", a->GetErrorString(r)); }
  h->comm = c;
  return DEMI_OK;
}
extern "C" int32_t demi_comm_rank(const demi_handle* h, int32_t* rank, int32_t* world) {
  if (!h) return DEMI_ERR_INVALID;
  const FrComm* c = h->comm;
  if (rank) *rank = c ? c->rank : 0;
  if (world) *world = c ? c->world : 1;
  return DEMI_OK;
}
void demi_comm_free(demi_handle* h) {
  FrComm* c = h->comm;
  if (!c) return;
  if (c->comm) nccl_api()->CommDestroy(c->comm);
  delete c;
  h->comm = nullptr;
}
extern "C" int32_t demi_create_multi(const demi_config* cfg, const int32_t* devices, int32_t n, demi_handle** out) {
  if (!cfg || !devices || !out || n < 1 || n > 64) return fail(nullptr, DEMI_ERR_INVALID, "demi_create_multi: bad arguments");
  for (int i = 0; i < n; i++) out[i] = nullptr;
  int32_t rc = DEMI_OK;
  for (int i = 0; i < n && rc == DEMI_OK; i++) { demi_config c = *cfg; c.device = devices[i]; rc = demi_create(&c, &out[i]); }
  if (rc == DEMI_OK && n > 1) {
    uint8_t id[DEMI_COMM_ID_BYTES];
    rc = demi_comm_unique_id(id);
    if (rc == DEMI_OK) {
      std::vector<int32_t> rcs(n, DEMI_OK);
      std::vector<std::thread> th;
      for (int i = 0; i < n; i++) th.emplace_back([&, i] { rcs[i] = demi_comm_init(out[i], id, i, n); });
      for (auto& t : th) t.join();
      for (int i = 0; i < n; i++) if (rcs[i] != DEMI_OK) { rc = rcs[i]; g_create_error = demi_last_error(out[i]); }
    }
  }
  if (rc != DEMI_OK) { for (int i = 0; i < n; i++) { demi_destroy(out[i]); out[i] = nullptr; } }
  return rc;
}

// --------------------------------------------------------------------------------------------------- kernel table
namespace {
typedef void (*fr_exec_fn)(const FrArgs);
struct FrVariant { int model; int bd; fr_exec_fn fn; size_t smem; };
template <class MODEL, int BD>
FrVariant make_frv() { return FrVariant{MODEL::ID, BD, fr_exec_kernel<MODEL, BD>, (size_t)FrExec<MODEL, BD>::WORDS * BD * sizeof(uint32_t)}; }
const FrVariant* pick_frv(int model) {
  static const std::vector<FrVariant> v = { make_frv<PingPong3, 128>(), make_frv<Raft5, 128>(), make_frv<Bcast32, 64>(), make_frv<IrModel, 64>() };
  for (const FrVariant& d : v) if (d.model == model) return &d;
  return nullptr;
}
constexpr int SCAN_WPB = 4;

struct FrRun { std::vector<unsigned long long> lo, hi; };      // per branch: the not yet dequeued part of the run, [lo, hi) in the queue array

struct FrState {
  demi_handle* h = nullptr; FrComm* comm = nullptr; const FrVariant* v = nullptr;
  demi_frontier_params F{}; uint32_t W = 0, win_cap = 0, segs_cap = 0;
  size_t scan_smem = 0, cnt_smem = 0;             // dynamic shared memory of the scan kernel; of the count and scatter kernels
  cudaStream_t s = nullptr;
  std::vector<DevBuf> allocs;
  // the device buffers, each in the argument struct of the kernels that use it (fr_setup binds them once): A for the
  // executor and the enqueue, S for the select kernels (per window: the segments, the quota and where winners go),
  // X for the steal round's pack and unpack (per batch: the records and where they go)
  FrArgs A{};
  FrSelArgs S{};
  FrXArgs X{};
  // NCCL buffers
  uint4* sendbuf = nullptr; uint4* recvbuf = nullptr; unsigned long long* gather_dev = nullptr;
  unsigned long long* log_all = nullptr; unsigned long long* log_counts = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  // host: the queue directory
  std::vector<FrRun> runs;
  std::vector<std::deque<uint32_t>> brq;          // per branch: runs with points left, creation order
  std::vector<unsigned long long> branch_live;
  unsigned long long pool_top = 0, pool_live = 0, n_exec = 0;
  uint32_t n_slots = 0;
  unsigned long long explored_sel = 0;            // explored pairs after the last getNext (history on)
  bool round_failed = false;                      // a round ended in a capacity status: R.explored_pairs is final
  demi_frontier_result R{};

  template <class T> int32_t dalloc(T*& p, size_t n) {
    allocs.emplace_back();
    const int32_t rc = allocs.back().grow(h, std::max<size_t>(n * sizeof(T), 256));
    p = allocs.back().get<T>();
    return rc;
  }
  ~FrState() { for (auto& e : ev) if (e) cudaEventDestroy(e); }
};

// device buffers are kept in the handle between calls with the same geometry (a search of a few hundred
// interleavings takes a millisecond; allocating its tables takes longer)
struct FrGeom { int model, world; demi_frontier_params F; uint32_t n_sends, ext_cap; };
bool fr_same_geom(const FrGeom& a, const FrGeom& b, uint32_t n_ext) {
  return a.model == b.model && a.world == b.world && a.F.max_messages == b.F.max_messages && a.F.width == b.F.width &&
         a.F.max_interleavings == b.F.max_interleavings && a.F.explored_slots == b.F.explored_slots && a.F.pool_cap == b.F.pool_cap &&
         a.F.trace_cap == b.F.trace_cap && a.F.steal_max == b.F.steal_max && a.F.flags == b.F.flags &&   // flags: the explored-key log
         a.n_sends == b.n_sends && n_ext <= a.ext_cap;
}

int32_t fr_setup(FrState& st, const demi_ext_event* ext, uint32_t n_ext, bool reuse) {
  demi_handle* h = st.h;
  const demi_frontier_params& F = st.F;
  FrArgs& A = st.A; FrSelArgs& S = st.S; FrXArgs& X = st.X;
  const uint32_t T1 = (uint32_t)F.max_messages + 2;
  uint32_t n_sends = 0;
  for (uint32_t i = 0; i < n_ext; i++) if (ext[i].kind == DEMI_EXT_SEND) n_sends++;
  A.cap_pend = demi_fr_pool_entries(demi_model_key(h), F.max_messages, n_sends);
  if (A.cap_pend >= 0xFFFFu) return fail(h, DEMI_ERR_CAPACITY, "demi_dpor_frontier: %u pending entries per interleaving exceed the 16-bit links", A.cap_pend);
  st.s = h->stream;
  if (!reuse) {
    const int world = st.comm ? st.comm->world : 1;
    st.W = F.width;
    st.win_cap = std::min<uint32_t>(std::max<uint32_t>(4 * st.W, 4096), 1u << 22);
    st.segs_cap = 1 << 16;
    st.scan_smem = (size_t)SCAN_WPB * fr_scan_words(T1) * 4; st.cnt_smem = (size_t)SCAN_WPB * fr_cnt_words(T1) * 4;
    A.T1 = T1; A.rcap = T1 * (T1 - 1) / 2; A.e_slots = F.explored_slots; A.no_history = (F.flags & DEMI_FR_NO_HISTORY) ? 1u : 0u;
    S.s_slots = 1; while (S.s_slots < 2 * st.win_cap) S.s_slots <<= 1;
    X.rec_u4 = T1 + 2;
    const unsigned long long cap_exec = F.max_interleavings + st.W + 1;
    const size_t warps = (st.W + 31) / 32;
    int32_t rc = DEMI_OK;
    auto da = [&](auto*& p, size_t n) { if (rc == DEMI_OK) rc = st.dalloc(p, n); };
    da(A.tr, (size_t)F.trace_cap * T1); da(A.tr_meta, F.trace_cap); da(A.E, F.explored_slots); da(A.pool, F.pool_cap);
    da(S.sel, std::max<uint32_t>(st.W, F.steal_max)); da(A.out_hash, cap_exec); da(A.out_viol, cap_exec);
    da(A.pendA, warps * A.cap_pend * 32); da(A.pendP1, warps * A.cap_pend * 32); da(A.pendNX, warps * A.cap_pend * 32);
    da(A.races, (size_t)st.W * A.rcap); da(A.n_races, st.W); da(A.counts, (size_t)T1 * st.W); da(A.tot, T1); da(A.base, T1);
    da(A.tile_tot, (size_t)T1 * ((st.W + FR_TILE - 1) / FR_TILE + 1));
    da(A.ctr, FRC_N); da(A.info, 1);
    da(S.win, st.win_cap); da(S.flag, st.win_cap); da(S.skey, S.s_slots); da(S.sidx, S.s_slots); da(S.blockcnt, (st.win_cap + 255) / 256 + 1);
    da(S.segs, st.segs_cap);
    if (world > 1) {
      da(st.sendbuf, (size_t)F.steal_max * (world - 1) * X.rec_u4); da(st.recvbuf, (size_t)F.steal_max * (world - 1) * X.rec_u4);
      da(st.gather_dev, (size_t)world * std::max(world, 8));
      if (!A.no_history) {                                       // explored pairs to share
        A.log.cap = (unsigned int)std::min<unsigned long long>(F.explored_slots / 2, 1ull << 22);
        da(A.log.keys, A.log.cap); da(A.log.n, 4); da(st.log_all, (size_t)world * A.log.cap); da(st.log_counts, world);
      }
    }
    da(X.hist, T1);
    da(A.ext, std::max<uint32_t>(n_ext, 64));
    if (rc != DEMI_OK) return rc;
    for (auto& e : st.ev) CUDA_TRY(h, cudaEventCreate(&e));
    A.sel = S.sel;
    S.pool = A.pool; S.E = A.E; S.e_slots = A.e_slots; S.info = A.info; S.ctr = A.ctr; S.no_history = A.no_history; S.log = A.log;
    X.sel = S.sel; X.tr = A.tr; X.tr_meta = A.tr_meta; X.T1 = T1; X.pool = A.pool;
  }
  A.model_flags = h->cfg.model_flags; A.blocked_mask = h->cfg.blocked_mask;
  A.max_messages = F.max_messages; A.looking_for = F.looking_for; A.n_ext = n_ext;
  st.runs.clear(); st.pool_top = st.pool_live = st.n_exec = 0; st.n_slots = 0;
  st.explored_sel = 0; st.round_failed = false;
  memset(&st.R, 0, sizeof(st.R));
  if (!A.no_history) CUDA_TRY(h, cudaMemsetAsync(A.E, 0, F.explored_slots * 8, st.s));
  CUDA_TRY(h, cudaMemsetAsync(A.ctr, 0, FRC_N * 8, st.s));
  if (A.log.n) CUDA_TRY(h, cudaMemsetAsync(A.log.n, 0, 16, st.s));
  CUDA_TRY(h, cudaMemsetAsync(A.info, 0, sizeof(FrInfo), st.s));
  if (n_ext) CUDA_TRY(h, cudaMemcpyAsync(const_cast<uint4*>(A.ext), ext, n_ext * sizeof(demi_ext_event), cudaMemcpyHostToDevice, st.s));
  CUDA_TRY(h, cudaFuncSetAttribute(st.v->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)st.v->smem));
  CUDA_TRY(h, cudaFuncSetAttribute(fr_scan_kernel<SCAN_WPB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)st.scan_smem));
  CUDA_TRY(h, cudaFuncSetAttribute(fr_count_kernel<SCAN_WPB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)st.cnt_smem));
  CUDA_TRY(h, cudaFuncSetAttribute(fr_scatter_kernel<SCAN_WPB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)st.cnt_smem));
  st.brq.assign(T1, {}); st.branch_live.assign(T1, 0);
  return DEMI_OK;
}

// a new sorted run of `tot[b]` points per branch, laid out deeper-branch-first from `start`
void fr_add_run(FrState& st, unsigned long long start, const uint32_t* tot) {
  FrRun run; run.lo.assign(st.A.T1, 0); run.hi.assign(st.A.T1, 0);
  unsigned long long off = start;
  const uint32_t idx = (uint32_t)st.runs.size();
  bool any = false;
  for (uint32_t b = st.A.T1; b-- > 0;) {
    run.lo[b] = off; off += tot[b]; run.hi[b] = off;
    if (tot[b]) { st.brq[b].push_back(idx); st.branch_live[b] += tot[b]; st.pool_live += tot[b]; any = true; }
  }
  if (any) st.runs.push_back(std::move(run));
}

// the select kernels over one window given as ascending segments; `quota` winners at most are taken, written to
// the selection from index `sel_base`
int32_t fr_select_window(FrState& st, const std::vector<FrSeg>& segs, uint32_t win_n, uint32_t quota, uint32_t sel_base,
                         uint32_t* taken, uint32_t* cut) {
  demi_handle* h = st.h;
  FrSelArgs& S = st.S;
  if (segs.size() > st.segs_cap) return fail(h, DEMI_ERR_CAPACITY, "demi_dpor_frontier: %zu queue segments in one window", segs.size());
  CUDA_TRY(h, cudaMemcpyAsync(const_cast<FrSeg*>(S.segs), segs.data(), segs.size() * sizeof(FrSeg), cudaMemcpyHostToDevice, st.s));
  CUDA_TRY(h, cudaMemsetAsync(S.skey, 0, (size_t)S.s_slots * 8, st.s));
  CUDA_TRY(h, cudaMemsetAsync(S.sidx, 0xFF, (size_t)S.s_slots * 4, st.s));
  S.n_segs = (uint32_t)segs.size(); S.win_n = win_n; S.n_blocks = (win_n + 255) / 256;
  S.sel_base = sel_base; S.quota = quota;
  fr_sel_probe_kernel<<<S.n_blocks, 256, 0, st.s>>>(S);
  fr_sel_winner_kernel<<<S.n_blocks, 256, 0, st.s>>>(S);
  fr_sel_blockscan_kernel<<<1, 1024, 0, st.s>>>(S);
  fr_sel_assign_kernel<<<S.n_blocks, 256, 0, st.s>>>(S);
  CUDA_TRY(h, cudaGetLastError());
  FrInfo info;
  CUDA_TRY(h, cudaMemcpyAsync(&info, S.info, sizeof(info), cudaMemcpyDeviceToHost, st.s));
  if (!S.no_history) CUDA_TRY(h, cudaMemcpyAsync(&st.explored_sel, S.ctr + FRC_EXPLORED, 8, cudaMemcpyDeviceToHost, st.s));
  CUDA_TRY(h, cudaStreamSynchronize(st.s));
  *taken = info.taken; *cut = info.cut;
  h->perf.kernel_launches += 4;
  return DEMI_OK;
}

// getNext for a round (DPORwHeuristics.scala:1142-1162, `quota` times): the first `quota` unexplored points in queue order
int32_t fr_select_front(FrState& st, uint32_t quota, uint32_t* n_sel) {
  *n_sel = 0;
  std::vector<FrSeg> segs;
  std::vector<std::pair<uint32_t, uint32_t>> src;          // (branch, run) of every segment
  while (*n_sel < quota && st.pool_live > 0) {
    segs.clear(); src.clear();
    uint32_t win_n = 0;
    for (uint32_t b = st.A.T1; b-- > 0 && win_n < st.win_cap;) {
      if (!st.branch_live[b]) continue;
      for (uint32_t r : st.brq[b]) {
        const FrRun& run = st.runs[r];
        const unsigned long long avail = run.hi[b] - run.lo[b];
        if (!avail) continue;
        const uint32_t take = (uint32_t)std::min<unsigned long long>(avail, st.win_cap - win_n);
        segs.push_back(FrSeg{run.lo[b], win_n, take}); src.emplace_back(b, r);
        win_n += take;
        if (win_n >= st.win_cap) break;
      }
    }
    uint32_t taken = 0, cut = 0;
    int32_t rc = fr_select_window(st, segs, win_n, quota - *n_sel, *n_sel, &taken, &cut);
    if (rc != DEMI_OK) return rc;
    uint32_t left = cut;                                    // dequeue the first `cut` points of the window
    for (size_t i = 0; i < segs.size() && left; i++) {
      const uint32_t c = std::min(left, segs[i].count);
      const uint32_t b = src[i].first; FrRun& run = st.runs[src[i].second];
      run.lo[b] += c; st.branch_live[b] -= c; st.pool_live -= c; left -= c;
      if (run.lo[b] == run.hi[b]) {                        // exhausted runs leave the branch's list (they are at its front)
        auto& q = st.brq[b];
        while (!q.empty() && st.runs[q.front()].lo[b] == st.runs[q.front()].hi[b]) q.pop_front();
      }
    }
    st.R.keys_dropped += cut - taken;
    *n_sel += taken;
  }
  return DEMI_OK;
}

// the LAST m points of the queue (shallowest branch), filtered and marked like a dequeue; survivors -> the selection [0, n)
int32_t fr_select_tail(FrState& st, unsigned long long m, uint32_t* n_out) {
  *n_out = 0;
  std::vector<FrSeg> segs;
  unsigned long long need = m;
  for (uint32_t b = 0; b < st.A.T1 && need; b++) {
    if (!st.branch_live[b]) continue;
    auto& q = st.brq[b];
    for (auto it = q.rbegin(); it != q.rend() && need; ++it) {
      FrRun& run = st.runs[*it];
      const unsigned long long avail = run.hi[b] - run.lo[b];
      if (!avail) continue;
      const unsigned long long take = std::min(avail, need);
      run.hi[b] -= take;
      segs.push_back(FrSeg{run.hi[b], 0, (uint32_t)take});
      st.branch_live[b] -= take; st.pool_live -= take; need -= take;
    }
    while (!q.empty() && st.runs[q.back()].lo[b] == st.runs[q.back()].hi[b]) q.pop_back();
  }
  std::reverse(segs.begin(), segs.end());                  // ascending queue order
  // windows of at most win_cap points, in order (the first point of a pair wins)
  size_t i = 0; uint32_t off_in_seg = 0;
  while (i < segs.size()) {
    std::vector<FrSeg> w; uint32_t win_n = 0;
    while (i < segs.size() && win_n < st.win_cap) {
      const uint32_t c = std::min<uint32_t>(segs[i].count - off_in_seg, st.win_cap - win_n);
      w.push_back(FrSeg{segs[i].src + off_in_seg, win_n, c});
      win_n += c; off_in_seg += c;
      if (off_in_seg == segs[i].count) { i++; off_in_seg = 0; }
    }
    uint32_t taken = 0, cut = 0;
    int32_t rc = fr_select_window(st, w, win_n, win_n, *n_out, &taken, &cut);
    if (rc != DEMI_OK) return rc;
    st.R.keys_dropped += win_n - taken;
    *n_out += taken;
  }
  return DEMI_OK;
}

// a round that ends in a capacity status adds nothing to the executed work (st.R still holds the last completed
// round's counters); keys_dropped and pool_left already are the failed round's getNext, explored_pairs becomes it
int32_t fr_round_fail(FrState& st, uint32_t status) {
  st.R.status = status;
  st.R.explored_pairs = st.explored_sel;
  st.round_failed = true;
  return DEMI_OK;
}

// execute st.A.n_sel points (or the root), scan the new traces, enqueue their backtrack points as a new run
int32_t fr_execute_and_scan(FrState& st, uint32_t n_sel, bool root) {
  demi_handle* h = st.h;
  if ((unsigned long long)st.n_slots + n_sel > st.F.trace_cap) return fr_round_fail(st, DEMI_DS_TRACE_OVF);   // the whole round, before it runs
  FrArgs& A = st.A;
  A.n_sel = n_sel; A.root = root ? 1u : 0u; A.first_slot = st.n_slots; A.exec_base = st.n_exec; A.pool_top = st.pool_top;
  if (h->cfg.model == DEMI_MODEL_IR) CUDA_TRY(h, ir_bind(h->ir_dev, st.s));
  CUDA_TRY(h, cudaEventRecord(st.ev[0], st.s));
  st.v->fn<<<(n_sel + st.v->bd - 1) / st.v->bd, st.v->bd, st.v->smem, st.s>>>(A);
  CUDA_TRY(h, cudaEventRecord(st.ev[1], st.s));
  const uint32_t wb = (n_sel + SCAN_WPB - 1) / SCAN_WPB;
  fr_scan_kernel<SCAN_WPB><<<wb, SCAN_WPB * 32, st.scan_smem, st.s>>>(A);    // every race of the round is marked explored ...
  fr_count_kernel<SCAN_WPB><<<wb, SCAN_WPB * 32, st.cnt_smem, st.s>>>(A);     // ... before any of its points is enqueued
  const uint32_t n_tiles = (n_sel + FR_TILE - 1) / FR_TILE;
  fr_rowscan_kernel<<<dim3(A.T1, n_tiles), 256, 0, st.s>>>(A);
  fr_base_kernel<<<1, 1024, 0, st.s>>>(A, n_tiles);
  fr_scatter_kernel<SCAN_WPB><<<wb, SCAN_WPB * 32, st.cnt_smem, st.s>>>(A, st.F.pool_cap);
  CUDA_TRY(h, cudaGetLastError());
  CUDA_TRY(h, cudaEventRecord(st.ev[2], st.s));
  h->perf.kernel_launches += 6;
  std::vector<uint32_t> tot(A.T1);
  unsigned long long ctr[FRC_N];
  CUDA_TRY(h, cudaMemcpyAsync(tot.data(), A.tot, A.T1 * 4, cudaMemcpyDeviceToHost, st.s));
  CUDA_TRY(h, cudaMemcpyAsync(ctr, A.ctr, sizeof(ctr), cudaMemcpyDeviceToHost, st.s));
  CUDA_TRY(h, cudaStreamSynchronize(st.s));
  float ms = 0;
  cudaEventElapsedTime(&ms, st.ev[0], st.ev[1]); st.R.exec_ms += ms;
  cudaEventElapsedTime(&ms, st.ev[1], st.ev[2]); st.R.scan_ms += ms;
  if (ctr[FRC_STATUS]) return fr_round_fail(st, (uint32_t)ctr[FRC_STATUS]);
  if (ctr[FRC_EXPLORED] * 2 >= st.F.explored_slots) return fr_round_fail(st, DEMI_DS_EXPLORED_OVF);   // after the round's scan
  unsigned long long added = 0;
  for (uint32_t b = 0; b < A.T1; b++) added += tot[b];
  if (st.pool_top + added > st.F.pool_cap) return fr_round_fail(st, DEMI_DS_HEAP_OVF);   // pool_cap bounds the arena: every point enqueued or received
  fr_add_run(st, st.pool_top, tot.data());
  st.pool_top += added;
  st.R.keys_enqueued += added;
  st.n_slots += n_sel; st.n_exec += n_sel;
  st.R.interleavings = st.n_exec; st.R.deliveries = ctr[FRC_DELIVERIES]; st.R.violations = ctr[FRC_VIOLATIONS];
  st.R.races = ctr[FRC_RACES]; st.R.explored_pairs = ctr[FRC_EXPLORED];
  st.R.rounds++;
  return DEMI_OK;
}

// the pair keys every rank marked explored since the last exchange become known to all ranks (a set union, so the
// order in which they were logged does not matter): the rank-local explored sets stop diverging
int32_t fr_share_explored(FrState& st, const std::vector<unsigned long long>& n_new) {
  demi_handle* h = st.h; NcclApi* nc = nccl_api(); FrComm* cm = st.comm;
  const FrLog& log = st.A.log;
  const int G = cm->world, me = cm->rank;
  unsigned long long maxn = 0;
  for (int q = 0; q < G; q++) maxn = std::max(maxn, n_new[q]);
  if (!maxn) return DEMI_OK;
  if (maxn > log.cap) { st.R.status = DEMI_DS_EXPLORED_OVF; return DEMI_OK; }
  // equal-size all-gather: every rank contributes `maxn` slots of its log (the tail beyond its own count is ignored)
  CUDA_TRY(h, cudaMemcpyAsync(st.log_counts, n_new.data(), (size_t)G * 8, cudaMemcpyHostToDevice, st.s));
  NCCL_TRY(h, nc->AllGather(log.keys, st.log_all, (size_t)maxn, ncclUint64, cm->comm, st.s));
  fr_merge_keys_kernel<<<dim3((unsigned)((maxn + 255) / 256), (unsigned)G), 256, 0, st.s>>>(st.log_all, (unsigned int)maxn, st.log_counts, (unsigned)G, (unsigned)me,
                                                                                          st.A.E, st.F.explored_slots, st.A.ctr);
  CUDA_TRY(h, cudaGetLastError());
  CUDA_TRY(h, cudaMemsetAsync(log.n, 0, 4, st.s));
  h->perf.kernel_launches++;
  st.R.bytes_sent += n_new[me] * 8ull * (unsigned long long)(G - 1);
  return DEMI_OK;
}

// one steal exchange; `have` = every rank's queue length (all-gathered).  The plan is a pure function of the all-gathered lengths, so every rank computes the same one.
int32_t fr_exchange(FrState& st, const std::vector<unsigned long long>& have_in, unsigned long long total_pool,
                    std::vector<unsigned long long>& have_after) {
  demi_handle* h = st.h; NcclApi* nc = nccl_api(); FrComm* cm = st.comm;
  const int G = cm->world, me = cm->rank;
  const uint32_t rec_u4 = st.X.rec_u4, T1 = st.A.T1;
  const unsigned long long S = st.F.rounds_per_exchange ? st.F.rounds_per_exchange : 1;
  const unsigned long long need = S * st.F.width;
  const unsigned long long share = (total_pool + G - 1) / G;
  const unsigned long long target = need < share ? need : share;
  std::vector<unsigned long long> have = have_in, give(G);
  for (int q = 0; q < G; q++) give[q] = have[q] > target ? have[q] - target : 0;
  std::vector<uint32_t> planned((size_t)G * G, 0);          // planned[don * G + rcv]
  for (int rcv = 0; rcv < G; rcv++) {
    unsigned long long want = have[rcv] < target ? target - have[rcv] : 0;
    for (int don = 0; don < G && want; don++) {
      if (don == rcv || !give[don]) continue;
      unsigned long long m = std::min(want, give[don]);
      m = std::min<unsigned long long>(m, st.F.steal_max);
      if (!m) continue;
      give[don] -= m; want -= m;
      planned[(size_t)don * G + rcv] = (uint32_t)m;
    }
  }
  st.R.exchanges++;
  // donor side: dequeue the tail, pack the survivors
  std::vector<uint32_t> my_row(G, 0);
  std::vector<size_t> send_off(G, 0);
  size_t off = 0;
  for (int rcv = 0; rcv < G; rcv++) {
    const uint32_t m = planned[(size_t)me * G + rcv];
    if (!m) continue;
    uint32_t n = 0;
    int32_t rc = fr_select_tail(st, m, &n);
    if (rc != DEMI_OK) return rc;
    send_off[rcv] = off;
    if (n) {
      FrXArgs X = st.X; X.n = n; X.buf = st.sendbuf + off * rec_u4;
      fr_pack_kernel<<<n, 128, 0, st.s>>>(X);
      CUDA_TRY(h, cudaGetLastError());
      h->perf.kernel_launches++;
    }
    my_row[rcv] = n; off += n;
    st.R.records_sent += n; st.R.bytes_sent += (unsigned long long)n * rec_u4 * 16;
  }
  // every rank learns how many records really travel (points found explored on the donor are dropped there)
  std::vector<unsigned long long> row64(G), mat((size_t)G * G);
  for (int q = 0; q < G; q++) row64[q] = my_row[q];
  CUDA_TRY(h, cudaMemcpyAsync(st.gather_dev + (size_t)me * G, row64.data(), G * 8, cudaMemcpyHostToDevice, st.s));
  NCCL_TRY(h, nc->AllGather(st.gather_dev + (size_t)me * G, st.gather_dev, G, ncclUint64, cm->comm, st.s));
  CUDA_TRY(h, cudaMemcpyAsync(mat.data(), st.gather_dev, (size_t)G * G * 8, cudaMemcpyDeviceToHost, st.s));
  CUDA_TRY(h, cudaStreamSynchronize(st.s));
  // every rank's queue length after the exchange: a donor loses what was planned (explored points are dropped on the
  // way out), a receiver gains what really arrived
  have_after = have_in;
  for (int don = 0; don < G; don++) for (int rcv = 0; rcv < G; rcv++) {
    have_after[don] -= planned[(size_t)don * G + rcv];
    have_after[rcv] += mat[(size_t)don * G + rcv];
  }
  std::vector<size_t> recv_off(G, 0);
  size_t roff = 0;
  for (int don = 0; don < G; don++) { recv_off[don] = roff; roff += (size_t)mat[(size_t)don * G + me]; }
  NCCL_TRY(h, nc->GroupStart());
  for (int rcv = 0; rcv < G; rcv++) if (my_row[rcv])
    NCCL_TRY(h, nc->Send(st.sendbuf + send_off[rcv] * rec_u4, (size_t)my_row[rcv] * rec_u4 * 16, ncclUint8, rcv, cm->comm, st.s));
  for (int don = 0; don < G; don++) if (mat[(size_t)don * G + me])
    NCCL_TRY(h, nc->Recv(st.recvbuf + recv_off[don] * rec_u4, (size_t)mat[(size_t)don * G + me] * rec_u4 * 16, ncclUint8, don, cm->comm, st.s));
  NCCL_TRY(h, nc->GroupEnd());
  // receiver side: every donor's batch becomes trace slots + one sorted run
  for (int don = 0; don < G; don++) {
    const uint32_t n = (uint32_t)mat[(size_t)don * G + me];
    if (!n) continue;
    if ((unsigned long long)st.n_slots + n > st.F.trace_cap) { st.R.status = DEMI_DS_TRACE_OVF; break; }
    if (st.pool_top + n > st.F.pool_cap) { st.R.status = DEMI_DS_HEAP_OVF; break; }
    CUDA_TRY(h, cudaMemsetAsync(st.X.hist, 0, T1 * 4, st.s));
    FrXArgs X = st.X; X.n = n; X.buf = st.recvbuf + recv_off[don] * rec_u4; X.first_slot = st.n_slots; X.pool_top = st.pool_top;
    // the batch arrives in the donor's queue order (branch desc, then its slot order), which the new slots preserve;
    // the run lays branches out deepest first, so the records of one branch must be contiguous: they are.
    fr_unpack_kernel<<<n, 128, 0, st.s>>>(X);
    CUDA_TRY(h, cudaGetLastError());
    h->perf.kernel_launches++;
    std::vector<uint32_t> tot(T1);
    CUDA_TRY(h, cudaMemcpyAsync(tot.data(), X.hist, T1 * 4, cudaMemcpyDeviceToHost, st.s));
    CUDA_TRY(h, cudaStreamSynchronize(st.s));
    fr_add_run(st, st.pool_top, tot.data());
    st.pool_top += n; st.n_slots += n; st.R.records_received += n;
  }
  CUDA_TRY(h, cudaStreamSynchronize(st.s));
  return DEMI_OK;
}

int32_t fr_run(FrState& st, demi_dpor_violation* viol, uint32_t cap_viol, uint64_t* hashes, uint64_t cap_hashes) {
  demi_handle* h = st.h;
  const demi_frontier_params& F = st.F;
  const int G = st.comm ? st.comm->world : 1, me = st.comm ? st.comm->rank : 0;
  const uint32_t S = F.rounds_per_exchange ? F.rounds_per_exchange : 1;
  int32_t rc;
  // the first execution: no nextTrace (DPORwHeuristics.scala:1219-1221 with an empty backtrack set), on rank 0
  if (me == 0 && F.max_interleavings >= 1) { if ((rc = fr_execute_and_scan(st, 1, true)) != DEMI_OK) return rc; }
  int exhausted = 0, budget = 0;
  for (;;) {
    // ---- what every rank learns at an exchange point
    unsigned long long mine[8] = {st.pool_live, st.n_exec, st.R.violations, st.R.status, 0, 0, 0, 0};
    std::vector<unsigned long long> all((size_t)G * 8);
    if (G > 1) {
      const auto t0 = std::chrono::steady_clock::now();
      NcclApi* nc = nccl_api();
      if (st.A.log.n) {                                                       // how many pair keys this rank has to share
        unsigned int nn = 0;
        CUDA_TRY(h, cudaMemcpyAsync(&nn, st.A.log.n, 4, cudaMemcpyDeviceToHost, st.s));
        CUDA_TRY(h, cudaStreamSynchronize(st.s));
        mine[4] = nn;
      }
      CUDA_TRY(h, cudaMemcpyAsync(st.gather_dev + (size_t)me * 8, mine, sizeof(mine), cudaMemcpyHostToDevice, st.s));
      NCCL_TRY(h, nc->AllGather(st.gather_dev + (size_t)me * 8, st.gather_dev, 8, ncclUint64, st.comm->comm, st.s));
      CUDA_TRY(h, cudaMemcpyAsync(all.data(), st.gather_dev, (size_t)G * 64, cudaMemcpyDeviceToHost, st.s));
      CUDA_TRY(h, cudaStreamSynchronize(st.s));
      st.R.exchange_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    } else memcpy(all.data(), mine, sizeof(mine));
    unsigned long long executed = 0, total_pool = 0; bool any_status = false, found = false;
    std::vector<unsigned long long> have(G), n_new(G);
    for (int q = 0; q < G; q++) { have[q] = all[q * 8]; total_pool += have[q]; executed += all[q * 8 + 1]; found |= all[q * 8 + 2] != 0; any_status |= all[q * 8 + 3] != 0; n_new[q] = all[q * 8 + 4]; }
    if (any_status) break;
    if (F.stop_if_found && found) break;                                      // :1147
    if (executed >= F.max_interleavings) { budget = 1; break; }
    if (!total_pool) { exhausted = 1; break; }
    std::vector<unsigned long long> have_after = have;
    if (G > 1) {
      const auto t0 = std::chrono::steady_clock::now();
      if (st.A.log.n && (rc = fr_share_explored(st, n_new)) != DEMI_OK) return rc;
      if (st.R.status) continue;
      if ((rc = fr_exchange(st, have, total_pool, have_after)) != DEMI_OK) return rc;
      st.R.exchange_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
      if (st.R.status) continue;                                              // reported at the next exchange point
    }
    // ---- S rounds.  What is left of the budget goes to the ranks in rank order, each taking what its queue (as every
    // rank knows it after the exchange) could use in S rounds — so the budget follows the work
    unsigned long long left = F.max_interleavings - executed, allow = 0;
    for (int q = 0; q <= me; q++) {
      const unsigned long long cap = std::min<unsigned long long>((unsigned long long)S * F.width, have_after[q]);
      allow = std::min(cap, left);
      left -= allow;
    }
    for (uint32_t r = 0; r < S && allow && st.pool_live && !st.R.status; r++) {
      const uint32_t quota = (uint32_t)std::min<unsigned long long>(allow, st.W);
      uint32_t n_sel = 0;
      const auto ts0 = std::chrono::steady_clock::now();
      if ((rc = fr_select_front(st, quota, &n_sel)) != DEMI_OK) return rc;      // ends with a stream sync (the cut)
      st.R.select_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - ts0).count();
      if (n_sel) { if ((rc = fr_execute_and_scan(st, n_sel, false)) != DEMI_OK) return rc; }
      else st.R.rounds++;
      allow -= n_sel;
      if (F.stop_if_found && st.R.violations) break;
    }
  }
  // results
  if (!st.round_failed) {
    unsigned long long ctr[FRC_N];                          // a steal round marks the points it hands over
    CUDA_TRY(h, cudaMemcpy(ctr, st.A.ctr, sizeof(ctr), cudaMemcpyDeviceToHost));
    st.R.explored_pairs = ctr[FRC_EXPLORED];
  }
  st.R.pool_left = st.pool_live; st.R.trace_slots = st.n_slots;
  st.R.exhausted = (uint32_t)exhausted; st.R.budget_exhausted = (uint32_t)budget;
  if (st.n_exec) {
    // only what the caller asked for crosses PCIe: the schedule hashes if wanted, and the violating records (compacted
    // on the device, then put back in execution order)
    if (hashes) CUDA_TRY(h, cudaMemcpy(hashes, st.A.out_hash, std::min<unsigned long long>(st.n_exec, cap_hashes) * 8, cudaMemcpyDeviceToHost));
    if (viol && cap_viol) {
      DevBuf buf;
      if ((rc = buf.grow(h, (size_t)cap_viol * sizeof(demi_dpor_violation) + 16)) != DEMI_OK) return rc;
      demi_dpor_violation* vd = buf.get<demi_dpor_violation>();
      unsigned int* cnt = (unsigned int*)(vd + cap_viol);
      CUDA_TRY(h, cudaMemsetAsync(cnt, 0, 4, st.s));
      fr_collect_viol_kernel<<<(unsigned)((st.n_exec + 255) / 256), 256, 0, st.s>>>(st.A.out_hash, st.A.out_viol, st.n_exec, vd, cap_viol, cnt);
      CUDA_TRY(h, cudaGetLastError());
      unsigned int nv = 0;
      CUDA_TRY(h, cudaMemcpyAsync(&nv, cnt, 4, cudaMemcpyDeviceToHost, st.s));
      CUDA_TRY(h, cudaStreamSynchronize(st.s));
      const unsigned int got = std::min<unsigned int>(nv, cap_viol);
      if (got) CUDA_TRY(h, cudaMemcpy(viol, vd, (size_t)got * sizeof(demi_dpor_violation), cudaMemcpyDeviceToHost));
      std::sort(viol, viol + got, [](const demi_dpor_violation& a, const demi_dpor_violation& b) { return a.interleaving < b.interleaving; });
      h->perf.kernel_launches++;
    }
  }
  return DEMI_OK;
}
}  // namespace

struct FrCache { FrGeom geom; FrState st; };

void demi_frontier_free(demi_handle* h) {
  if (!h->frontier) return;
  cudaSetDevice(h->cfg.device);
  delete h->frontier;
  h->frontier = nullptr;
}

extern "C" int32_t demi_dpor_frontier(demi_handle* h, const demi_ext_event* ext, uint32_t n_ext,
                                      const demi_frontier_params* params, demi_frontier_result* result,
                                      demi_dpor_violation* viol, uint32_t cap_viol, uint64_t* hashes, uint64_t cap_hashes) {
  if (!h) return DEMI_ERR_INVALID;
  if (!params || !result || (!ext && n_ext)) return fail(h, DEMI_ERR_INVALID, "demi_dpor_frontier: null argument");
  const demi_frontier_params& F = *params;
  if (F.max_messages < 1 || F.max_messages > 1000) return fail(h, DEMI_ERR_INVALID, "demi_dpor_frontier: max_messages must be in [1, 1000]");
  if (!F.width || F.width > (1u << 20)) return fail(h, DEMI_ERR_INVALID, "demi_dpor_frontier: width must be in [1, 2^20]");
  if (F.explored_slots < 1024 || (F.explored_slots & (F.explored_slots - 1))) return fail(h, DEMI_ERR_INVALID, "demi_dpor_frontier: explored_slots must be a power of two >= 1024");
  if (!F.pool_cap || !F.trace_cap || F.trace_cap >= (1u << 28)) return fail(h, DEMI_ERR_INVALID, "demi_dpor_frontier: pool_cap / trace_cap (below 2^28) must be positive");
  { int32_t mrc = demi_need_model(h); if (mrc != DEMI_OK) return mrc; }
  { int32_t vrc = demi_check_dpor_program(h, "demi_dpor_frontier", ext, n_ext); if (vrc != DEMI_OK) return vrc; }
  FrComm* cm = h->comm;
  if (cm && cm->world > 1 && !F.steal_max) return fail(h, DEMI_ERR_INVALID, "demi_dpor_frontier: steal_max must be positive on %d ranks", cm->world);
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  uint32_t n_sends = 0;
  for (uint32_t i = 0; i < n_ext; i++) if (ext[i].kind == DEMI_EXT_SEND) n_sends++;
  FrGeom g{h->cfg.model, (cm && cm->world > 1) ? cm->world : 1, F, n_sends, std::max<uint32_t>(n_ext, 64)};
  FrCache* cache = h->frontier;
  bool reuse = cache && fr_same_geom(cache->geom, g, n_ext);
  if (!reuse) { delete cache; cache = new FrCache(); cache->geom = g; h->frontier = cache; }
  FrState& st = cache->st;
  st.h = h; st.comm = (cm && cm->world > 1) ? cm : nullptr; st.F = F;
  st.v = pick_frv(h->cfg.model);
  if (!st.v) return fail(h, DEMI_ERR_INVALID, "demi_dpor_frontier: no kernel for model %d", h->cfg.model);
  memset(result, 0, sizeof(*result));
  h->perf.kernel_launches = 0;
  int32_t rc = fr_setup(st, ext, n_ext, reuse);
  if (rc != DEMI_OK) { delete cache; h->frontier = nullptr; return rc; }
  if (rc == DEMI_OK) rc = fr_run(st, viol, cap_viol, hashes, cap_hashes);
  *result = st.R;
  if (rc != DEMI_OK) return rc;
  h->perf.prefixes = st.n_exec; h->perf.deliveries = st.R.deliveries; h->perf.violations = st.R.violations;
  h->perf.kernel_ms = st.R.exec_ms + st.R.scan_ms + st.R.select_ms;
  if (st.R.status) return fail(h, DEMI_ERR_CAPACITY, "demi_dpor_frontier: status %u", st.R.status);
  return DEMI_OK;
}

extern "C" int32_t demi_dpor_frontier_multi(demi_handle** hs, int32_t n, const demi_ext_event* ext, uint32_t n_ext,
                                            const demi_frontier_params* params, demi_frontier_result* results,
                                            demi_dpor_violation* viol, uint32_t cap_viol, uint64_t* hashes, uint64_t cap_hashes) {
  if (!hs || n < 1 || !results) return DEMI_ERR_INVALID;
  std::vector<int32_t> rcs(n, DEMI_OK);
  std::vector<std::thread> th;
  for (int i = 0; i < n; i++)
    th.emplace_back([&, i] {
      rcs[i] = demi_dpor_frontier(hs[i], ext, n_ext, params, &results[i], viol ? viol + (size_t)i * cap_viol : nullptr, cap_viol,
                                  hashes ? hashes + (size_t)i * cap_hashes : nullptr, cap_hashes);
    });
  for (auto& t : th) t.join();
  for (int i = 0; i < n; i++) if (rcs[i] != DEMI_OK) return rcs[i];
  return DEMI_OK;
}
