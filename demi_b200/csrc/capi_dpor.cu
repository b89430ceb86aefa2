// capi_dpor.cu — C ABI for batched DPORwHeuristics searches (K3), the edit-distance bounded / resumable
// configuration of RunnerUtils.editDistanceDporDDMin, and IncrementalDDMin on top of it, for one trace or many.
#include "dpor_kernel.cuh"
#include "models/model_ir.cuh"
#include "engine.hpp"
#include "incddmin_driver.hpp"
#include "many_rendezvous.hpp"

using namespace demi;

typedef void (*dpor_fn)(const DporArgs);
// fn: one seed per launch; fn_multi: every search reads the seed of its own trace (DporArgs::seeds)
struct DporVariant { int model; int bd; dpor_fn fn; size_t smem; int nq; dpor_fn fn_multi; };
template <class MODEL, int BD>
static DporVariant make_dv() {
  using M = DporMachine<MODEL, BD>;
  return DporVariant{MODEL::ID, BD, dpor_kernel<MODEL, BD>, (size_t)M::WORDS * BD * sizeof(uint32_t), M::NQ,
                     dpor_kernel<MODEL, BD, true>};
}
// A loaded model (IrModel) has the geometry of DEMI_IR_ACTORS actors, whatever it loads: 16 x 8 state words and a
// staged outbox of 16 x 3 words per search (22 528 B of shared memory per block of 32), and NQ = 17 * 16 FIFOs per
// search in HBM.  The canonical order of getPendingEvent (the scan over q = src * 16 + dst, deadLetters in row 16) is
// the oracle's (src * DEMI_MAX_ACTORS + dst, deadLetters in row n_actors): no queue whose sender or receiver lies in
// [n_actors, 16) ever holds a message, because the interpreter drops a SEND to such an index and every external is
// range-checked against the loaded actor count, so both scans meet the non-empty queues in the same order.
static const DporVariant* pick_dv(int model) {
  static const std::vector<DporVariant> v = { make_dv<PingPong3, 32>(), make_dv<Raft5, 32>(), make_dv<Bcast32, 32>(),
                                              make_dv<IrModel, 32>() };
  for (const DporVariant& d : v) if (d.model == model) return &d;
  return nullptr;
}

namespace {

// setInitialDepGraph / setInitialTrace / ArvindDistanceOrdering.init from a recorded execution
struct SeedHost {
  std::vector<uint4> nodes;          // {src|dst<<8|type<<16, p0, p1, parent | depth << 20}
  std::vector<uint32_t> trace;       // DepTracker.initialTrace: root, then the delivered Uniques
  std::vector<int32_t> orig_index;   // originalIndices (BacktrackOrdering.scala:110-116): later occurrences overwrite
};
int32_t build_seed(demi_handle* h, const demi_dpor_seed* seed, SeedHost& out) {
  if (!seed->events || !seed->dep_parent || !seed->n_nodes) return fail(h, DEMI_ERR_INVALID, "demi_dpor_seed: events and dep_parent are required");
  if (seed->n_nodes > (1u << 16)) return fail(h, DEMI_ERR_INVALID, "demi_dpor_seed: node ids are 16-bit");
  { int32_t vrc = demi_check_events(h, "demi_dpor_seed", seed->events, seed->n_events, seed->n_nodes); if (vrc != DEMI_OK) return vrc;
    vrc = demi_check_parents(h, "demi_dpor_seed", seed->dep_parent, seed->n_nodes); if (vrc != DEMI_OK) return vrc; }
  out.nodes.assign(seed->n_nodes, make_uint4(0, 0, 0, 0));
  out.orig_index.assign(seed->n_nodes, -1);
  out.trace.assign(1, 0u);
  std::vector<char> have(seed->n_nodes, 0);
  have[0] = 1;
  for (uint32_t i = 0; i < seed->n_events; i++) {
    const demi_event& e = seed->events[i];
    if (e.kind == DEMI_EV_MSG_SEND) {                        // the Unique was allocated when the message was sent
      if (e.node == 0 || e.node >= seed->n_nodes) return fail(h, DEMI_ERR_INVALID, "demi_dpor_seed: event %u names node %u outside the tree", i, (unsigned)e.node);
      // timer markers and externals are "deadLetters" messages for both DepTracker and DPORwHeuristics
      const uint32_t src = e.src >= DEMI_MAX_ACTORS ? (uint32_t)DEMI_DEADLETTERS : e.src;
      out.nodes[e.node] = make_uint4(src | ((uint32_t)e.dst << 8) | ((uint32_t)e.type << 16), e.p0, e.p1, seed->dep_parent[e.node]);
      have[e.node] = 1;
    } else if (e.kind == DEMI_EV_MSG_EVENT) {
      if (e.node >= seed->n_nodes) return fail(h, DEMI_ERR_INVALID, "demi_dpor_seed: event %u names node %u outside the tree", i, (unsigned)e.node);
      out.trace.push_back(e.node);
    }
  }
  for (uint32_t v = 1; v < seed->n_nodes; v++) {             // a parent is created before its children
    if (!have[v]) return fail(h, DEMI_ERR_INVALID, "demi_dpor_seed: node %u has no MsgSend event", v);
    const uint32_t par = out.nodes[v].w;
    if (par >= v) return fail(h, DEMI_ERR_INVALID, "demi_dpor_seed: node %u has parent %u", v, par);
    out.nodes[v].w = par | (((out.nodes[par].w >> 20) + 1) << 20);
  }
  for (size_t i = 0; i < out.trace.size(); i++) out.orig_index[out.trace[i]] = (int32_t)i;
  return DEMI_OK;
}

// The parameters every search of a launch shares
int32_t check_shared_params(demi_handle* h, const demi_dpor_params& P) {
  if (P.node_cap < 2 || P.node_cap > (1u << 20)) return fail(h, DEMI_ERR_INVALID, "node_cap must be in [2, 2^20]");
  if (P.explored_slots < 2 || (P.explored_slots & (P.explored_slots - 1))) return fail(h, DEMI_ERR_INVALID, "explored_slots must be a power of two");
  return DEMI_OK;
}
int32_t check_max_messages(demi_handle* h, int32_t max_messages) {
  if (max_messages < 0 || max_messages > 1022) return fail(h, DEMI_ERR_INVALID, "max_messages must be in [0, 1022] (setMaxMessagesToSchedule)");
  return DEMI_OK;
}
int32_t check_budget_params(demi_handle* h, const demi_dpor_params& P) {
  if (!P.heap_cap || !P.max_interleavings) return fail(h, DEMI_ERR_INVALID, "heap_cap / max_interleavings must be positive");
  if (P.max_interleavings >= (1u << 20)) return fail(h, DEMI_ERR_INVALID, "max_interleavings must be below 2^20 (backtrack key packing)");
  return DEMI_OK;
}
// what a search needs of its seed: the ordering's original trace, and a graph within node_cap
int32_t check_seed(demi_handle* h, const demi_dpor_params& P, uint32_t flags, const SeedHost* seed) {
  if ((flags & DEMI_DF_ARVIND_ORDERING) && !seed) return fail(h, DEMI_ERR_INVALID, "ArvindDistanceOrdering needs the original trace (demi_dpor_seed)");
  if (seed && seed->nodes.size() > P.node_cap) return fail(h, DEMI_ERR_CAPACITY, "node_cap %u is below the seed graph's %zu nodes", P.node_cap, seed->nodes.size());
  return DEMI_OK;
}

// Device bytes one search of a launch owns (the per-search buffers of dpor_run), for T1 = max_messages + 2
size_t dpor_search_bytes(const demi_dpor_params& P, uint32_t T1, int nq, bool arv, bool use_buckets) {
  const size_t NI = (size_t)P.max_interleavings + 1;
  return sizeof(demi_dpor_result) + (size_t)P.node_cap * (sizeof(uint4) + sizeof(uint32_t)) +
         (size_t)demi_pow2_at_least(2 * P.node_cap, 4, 1u << 22) * sizeof(uint32_t) + (size_t)nq * DPOR_QCAP * sizeof(uint32_t) +
         (size_t)P.explored_slots * sizeof(uint64_t) + (size_t)P.heap_cap * sizeof(DporKey) + NI * (T1 + 1) * sizeof(uint32_t) +
         3 * (size_t)T1 * sizeof(uint32_t) + ((arv || use_buckets) ? (size_t)P.heap_cap * sizeof(uint32_t) : 0) +
         (arv ? (2 * (size_t)T1 + 4) * sizeof(int32_t) : 0) + (use_buckets ? 2 * (size_t)T1 * sizeof(uint32_t) : 0) +
         2 * sizeof(uint32_t);
}

// A multi-trace launch (dpor_kernel<..., true>): the seeds of the call, on the device once per call, and the trace of
// each search of the launch (host, n_searches entries)
struct MultiSeeds {
  const DporSeedView* views;
  const uint4* nodes; const uint32_t* trace; const int32_t* orig_index;
  const uint32_t* trace_of_search;
};

// One K3 launch of n_searches searches.  With `multi`, params->max_messages is the largest of the launch's traces (it
// sets the strides) and the seed checks are the caller's, per trace.
int32_t dpor_run(demi_handle* h, const demi_ext_event* ext, const uint32_t* ext_offsets, uint32_t n_searches,
                 const demi_dpor_params* params, uint32_t flags, const SeedHost* seed,
                 const int32_t* caps, const uint32_t* cap_offsets, demi_dpor_result* results,
                 demi_dpor_violation* viol, uint32_t cap_viol, uint64_t* hashes, uint32_t cap_hashes,
                 const MultiSeeds* multi = nullptr) {
  const demi_dpor_params& P = *params;
  int32_t vrc;
  if ((vrc = check_shared_params(h, P)) != DEMI_OK || (vrc = check_max_messages(h, P.max_messages)) != DEMI_OK ||
      (vrc = check_budget_params(h, P)) != DEMI_OK || (!multi && (vrc = check_seed(h, P, flags, seed)) != DEMI_OK))
    return vrc;
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  const DporVariant* dv = pick_dv(h->cfg.model);
  if (!dv) return fail(h, DEMI_ERR_INVALID, "no DPOR kernel for model %d", h->cfg.model);
  const uint32_t n_ext = ext_offsets[n_searches];
  { int32_t vrc = demi_check_dpor_program(h, "demi_dpor_batch", ext, n_ext); if (vrc != DEMI_OK) return vrc; }
  DporArgs a{};
  a.model_flags = h->cfg.model_flags; a.blocked_mask = h->cfg.blocked_mask;
  a.P = P; a.n_searches = n_searches; a.cap_viol = cap_viol; a.cap_hashes = cap_hashes;
  a.T1 = (uint32_t)P.max_messages + 2;
  a.child_slots = demi_pow2_at_least(2 * P.node_cap, 4, 1u << 22);
  a.flags = flags;
  const bool arv = (flags & DEMI_DF_ARVIND_ORDERING) != 0;
  // a single uncapped test with the default ordering (the classic batch) uses the bucket queue; instances that are
  // resumed re-enqueue keys, and for those the binary heap keeps the oracle's order among the duplicates
  const bool use_buckets = !arv && !caps;
  const size_t S = n_searches, NI = (size_t)P.max_interleavings + 1;
  const size_t n_caps = caps ? cap_offsets[n_searches] : 0;
  const size_t n_seed_nodes = seed ? seed->nodes.size() : 0, n_seed_trace = seed ? seed->trace.size() : 0;
  a.n_init_nodes = (uint32_t)n_seed_nodes; a.n_init_trace = (uint32_t)n_seed_trace;
  // Every per-search buffer once: the field it binds, its bytes, its fill (-1: none) and whether the field is bound
  // (an unbound one stays null).  The buffers live in the handle, one per entry, and only grow: a DDMin run issues many
  // launches of similar size.
  int32_t rc = DEMI_OK;
  cudaError_t e = cudaSuccess;
  size_t nb = 0;
  auto buf = [&](auto*& field, size_t bytes, int fill, bool bound = true) {
    if (nb == h->dpor_buf.size()) h->dpor_buf.emplace_back();
    DevBuf& d = h->dpor_buf[nb++];
    if (rc == DEMI_OK) rc = d.grow(h, bytes);
    if (rc != DEMI_OK) return;
    if (fill >= 0 && e == cudaSuccess) e = cudaMemsetAsync(d.get(), fill, bytes, h->stream);
    field = bound ? d.get<std::remove_reference_t<decltype(*field)>>() : nullptr;
  };
  buf(a.ext, std::max<size_t>(n_ext, 1) * sizeof(demi_ext_event), -1);
  buf(a.ext_offsets, (S + 1) * sizeof(uint32_t), -1);
  buf(a.results, S * sizeof(demi_dpor_result), 0);
  buf(a.viol, std::max<size_t>(S * cap_viol, 1) * sizeof(demi_dpor_violation), 0, viol != nullptr);
  buf(a.hashes, std::max<size_t>(S * cap_hashes, 1) * sizeof(uint64_t), 0, hashes != nullptr);
  buf(a.nodes, S * P.node_cap * sizeof(uint4), -1);
  buf(a.child_hash, S * a.child_slots * sizeof(uint32_t), 0);
  buf(a.queues, S * dv->nq * DPOR_QCAP * sizeof(uint32_t), -1);
  buf(a.explored, S * P.explored_slots * sizeof(uint64_t), 0xFF);
  buf(a.heap, S * P.heap_cap * sizeof(DporKey), -1);
  buf(a.traces, S * NI * a.T1 * sizeof(uint32_t), -1);
  buf(a.trace_len, S * NI * sizeof(uint32_t), -1);
  buf(a.cur_trace, S * a.T1 * sizeof(uint32_t), -1);
  buf(a.next_trace, S * a.T1 * sizeof(uint32_t), -1);
  buf(a.node_pos, S * P.node_cap * sizeof(uint32_t), 0);
  buf(a.scan, S * a.T1 * sizeof(uint32_t), -1);
  buf(a.heap_dist, (arv || use_buckets) ? S * P.heap_cap * sizeof(uint32_t) : 16, -1, arv || use_buckets);
  buf(a.path, arv ? S * (2 * (size_t)a.T1 + 4) * sizeof(int32_t) : 16, -1, arv);
  buf(a.caps, std::max<size_t>(n_caps, 1) * sizeof(int32_t), -1, caps != nullptr);
  buf(a.cap_offsets, (S + 1) * sizeof(uint32_t), -1);
  buf(a.init_nodes, std::max<size_t>(n_seed_nodes, 1) * sizeof(uint4), -1);
  buf(a.init_trace, std::max<size_t>(n_seed_trace, 1) * sizeof(uint32_t), -1);
  buf(a.orig_index, std::max<size_t>(n_seed_nodes, 1) * sizeof(int32_t), -1);
  buf(a.buckets, use_buckets ? S * 2 * (size_t)a.T1 * sizeof(uint32_t) : 16, -1, use_buckets);
  buf(a.trace_of_search, multi ? S * sizeof(uint32_t) : 16, -1, multi != nullptr);
  if (rc != DEMI_OK) {
    for (DevBuf& d : h->dpor_buf) d.reset();       // all of them: a smaller retry then finds the memory free
    return rc;
  }
  auto up = [&](const void* dst, const void* src, size_t bytes) {
    if (e == cudaSuccess && bytes) e = cudaMemcpyAsync(const_cast<void*>(dst), src, bytes, cudaMemcpyHostToDevice, h->stream);
  };
  up(a.ext, ext, n_ext * sizeof(demi_ext_event));
  up(a.ext_offsets, ext_offsets, (S + 1) * sizeof(uint32_t));
  if (caps) { up(a.caps, caps, n_caps * sizeof(int32_t)); up(a.cap_offsets, cap_offsets, (S + 1) * sizeof(uint32_t)); }
  if (multi) {
    up(a.trace_of_search, multi->trace_of_search, S * sizeof(uint32_t));
    a.seeds = multi->views; a.init_nodes = multi->nodes; a.init_trace = multi->trace; a.orig_index = multi->orig_index;
  }
  if (seed) {
    up(a.init_nodes, seed->nodes.data(), n_seed_nodes * sizeof(uint4));
    up(a.init_trace, seed->trace.data(), n_seed_trace * sizeof(uint32_t));
    up(a.orig_index, seed->orig_index.data(), n_seed_nodes * sizeof(int32_t));
  }
  if (e == cudaSuccess && h->cfg.model == DEMI_MODEL_IR) e = ir_bind(h->ir_dev, h->stream);   // this unit's copy of g_ir
  // the race scan's position table goes to shared memory when it leaves room for >= 8 blocks per SM
  const dpor_fn fn = multi ? dv->fn_multi : dv->fn;
  size_t smem = dv->smem;
  const size_t scan_bytes = (size_t)a.T1 * dv->bd * sizeof(uint32_t);
  a.scan_in_smem = (dv->smem + scan_bytes <= 27 * 1024) ? 1u : 0u;
  if (a.scan_in_smem) smem += scan_bytes;
  if (e == cudaSuccess) e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e == cudaSuccess) e = cudaEventRecord(h->ev0, h->stream);
  if (e == cudaSuccess) {
    fn<<<(n_searches + dv->bd - 1) / dv->bd, dv->bd, smem, h->stream>>>(a);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaEventRecord(h->ev1, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(results, a.results, S * sizeof(demi_dpor_result), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess && viol && cap_viol) e = cudaMemcpyAsync(viol, a.viol, S * cap_viol * sizeof(demi_dpor_violation), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess && hashes && cap_hashes) e = cudaMemcpyAsync(hashes, a.hashes, S * cap_hashes * sizeof(uint64_t), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  float ms = 0;
  if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, h->ev0, h->ev1);
  if (e != cudaSuccess) return fail(h, DEMI_ERR_CUDA, "demi_dpor_batch: %s", cudaGetErrorString(e));
  h->perf.kernel_ms = ms; h->perf.kernel_launches = 1;
  uint64_t il = 0, del = 0, vi = 0;
  for (size_t s = 0; s < S; s++) { il += results[s].interleavings; del += results[s].deliveries; vi += results[s].violations; }
  h->perf.prefixes = il; h->perf.deliveries = del; h->perf.violations = vi;
  return DEMI_OK;
}

}  // namespace

extern "C" int32_t demi_dpor_batch_ex(demi_handle* h, const demi_ext_event* ext, const uint32_t* ext_offsets, uint32_t n_searches,
                                      const demi_dpor_params* params, const demi_dpor_ex* ex, demi_dpor_result* results,
                                      demi_dpor_violation* viol, uint32_t cap_viol, uint64_t* hashes, uint32_t cap_hashes) {
  if (!h) return DEMI_ERR_INVALID;
  if (!ext || !ext_offsets || !params || !results) return fail(h, DEMI_ERR_INVALID, "demi_dpor_batch: null argument");
  if (n_searches == 0) return DEMI_OK;
  { int32_t mrc = demi_need_model(h); if (mrc != DEMI_OK) return mrc; }
  SeedHost seed;
  const bool have_seed = ex && ex->seed;
  if (have_seed) { int32_t rc = build_seed(h, ex->seed, seed); if (rc != DEMI_OK) return rc; }
  if (ex && ex->caps && !ex->cap_offsets) return fail(h, DEMI_ERR_INVALID, "demi_dpor_batch_ex: caps without cap_offsets");
  return dpor_run(h, ext, ext_offsets, n_searches, params, ex ? ex->flags : 0u, have_seed ? &seed : nullptr,
                  ex ? ex->caps : nullptr, ex ? ex->cap_offsets : nullptr, results, viol, cap_viol, hashes, cap_hashes);
}

extern "C" int32_t demi_dpor_batch(demi_handle* h, const demi_ext_event* ext, const uint32_t* ext_offsets, uint32_t n_searches,
                                   const demi_dpor_params* params, demi_dpor_result* results,
                                   demi_dpor_violation* viol, uint32_t cap_viol, uint64_t* hashes, uint32_t cap_hashes) {
  return demi_dpor_batch_ex(h, ext, ext_offsets, n_searches, params, nullptr, results, viol, cap_viol, hashes, cap_hashes);
}

// ------------------------------------------------------------------------------------------ IncrementalDDMin
namespace {

// ResumableDPOR as DDMin's TestOracle on the handle: every speculative batch is one K3 launch
struct DporDDMinDriver : IncDDMinDriver {
  const demi_dpor_params* P; uint32_t dflags; const SeedHost* seed;
  int32_t run_dpor(const uint64_t* masks, size_t n, const std::vector<int32_t>& caps, const std::vector<uint32_t>& cap_off,
                   demi_dpor_result* res) override {
    std::vector<demi_ext_event> flat;
    std::vector<uint32_t> off(1, 0);
    select(masks, n, flat, off);
    return dpor_run(h, flat.data(), off.data(), (uint32_t)n, P, dflags, seed, caps.data(), cap_off.data(), res, nullptr, 0,
                    nullptr, 0);
  }
};

}  // namespace

extern "C" int32_t demi_incremental_ddmin(demi_handle* h, const demi_ext_event* externals, uint32_t n_externals,
                                          const demi_dpor_params* params, uint32_t flags, const demi_dpor_seed* seed,
                                          int32_t max_max_distance, uint32_t stop_at_size,
                                          uint64_t* mcs_mask, uint32_t mask_words, demi_incddmin_out* out) {
  if (!h) return DEMI_ERR_INVALID;
  if (!externals || !params || !mcs_mask || !out) return fail(h, DEMI_ERR_INVALID, "demi_incremental_ddmin: null argument");
  { int32_t mrc = demi_need_model(h); if (mrc != DEMI_OK) return mrc; }
  if ((uint64_t)mask_words * 64 < n_externals) return fail(h, DEMI_ERR_INVALID, "mask_words too small");
  { int32_t vrc = demi_check_dpor_program(h, "demi_incremental_ddmin", externals, n_externals); if (vrc != DEMI_OK) return vrc; }
  SeedHost sh;
  if (seed) { int32_t rc = build_seed(h, seed, sh); if (rc != DEMI_OK) return rc; }
  DporDDMinDriver d;
  d.h = h; d.looking_for = params->looking_for; d.flags = 0; d.mw = mask_words; d.n_ext = n_externals; d.ext = externals;
  d.P = params; d.dflags = flags; d.seed = seed ? &sh : nullptr;
  return d.minimize(max_max_distance, stop_at_size, mcs_mask, out);
}

// ------------------------------------------------------------------------------------------ IncrementalDDMin, many traces
namespace {

typedef ManyRequest<demi_dpor_result> DporRequest;
// what a request's searches are put through besides their masks: test k's caps are caps[cap_off[k] .. cap_off[k+1])
struct DporPayload { const std::vector<int32_t>* caps; const std::vector<uint32_t>* cap_off; };

// Device bytes the searches of one launch of demi_incremental_ddmin_many may own: the smaller of this and half the
// device memory free when the call starts.  A round's searches go to as many launches as that takes, each holding at
// least one search.
constexpr uint64_t MANY_DPOR_BYTES = 32ull << 30;

// ResumableDPOR on trace `trace` of a demi_incremental_ddmin_many call: its batches join the rendezvous
struct ManyDporDriver : IncDDMinDriver {
  Rendezvous<demi_dpor_result>* R; uint32_t trace;
  const demi_dpor_params* P; uint32_t dflags; const SeedHost* seed; int32_t max_messages;
  int32_t run_dpor(const uint64_t* masks, size_t n, const std::vector<int32_t>& caps, const std::vector<uint32_t>& cap_off,
                   demi_dpor_result* res) override {
    // what dpor_run checks of this trace's launch in demi_incremental_ddmin
    demi_dpor_params Pt = *P;
    Pt.max_messages = max_messages;
    int32_t rc;
    if ((rc = check_max_messages(h, max_messages)) != DEMI_OK || (rc = check_seed(h, Pt, dflags, seed)) != DEMI_OK) return rc;
    const DporPayload pl{&caps, &cap_off};
    DporRequest q;
    q.trace = trace; q.masks = masks; q.n = n; q.payload = &pl;
    R->submit(q);
    if (q.rc != DEMI_OK) return q.rc;
    std::copy(q.res.begin(), q.res.end(), res);
    return DEMI_OK;
  }
};

}  // namespace

extern "C" int32_t demi_incremental_ddmin_many(demi_handle* h, uint32_t n_traces,
                                               const demi_ext_event* externals, const uint32_t* ext_offsets, const uint32_t* n_externals,
                                               const demi_dpor_seed* seeds, const int32_t* max_messages, const uint32_t* looking_for,
                                               const demi_dpor_params* params, uint32_t flags, int32_t max_max_distance,
                                               uint32_t stop_at_size, uint64_t* mcs_masks, uint32_t mask_words,
                                               demi_incddmin_out* out, int32_t* status) {
  if (!h) return DEMI_ERR_INVALID;
  static const char* who = "demi_incremental_ddmin_many";
  if (!n_traces) return DEMI_OK;
  if (!externals || !ext_offsets || !n_externals || !max_messages || !looking_for || !params || !mcs_masks || !out || !status)
    return fail(h, DEMI_ERR_INVALID, "%s: null argument", who);
  { int32_t mrc = demi_need_model(h); if (mrc != DEMI_OK) return mrc; }
  const uint32_t n = n_traces;
  for (uint32_t t = 0; t < n; t++)
    if ((uint64_t)mask_words * 64 < n_externals[t])
      return fail(h, DEMI_ERR_INVALID, "mask_words %u too small for the %u externals of trace %u", mask_words, n_externals[t], t);
  int32_t rc;
  if ((rc = check_shared_params(h, *params)) != DEMI_OK || (rc = check_budget_params(h, *params)) != DEMI_OK) return rc;
  const DporVariant* dv = pick_dv(h->cfg.model);
  if (!dv) return fail(h, DEMI_ERR_INVALID, "no DPOR kernel for model %d", h->cfg.model);
  uint32_t window;
  if ((rc = many_window(h, n, window)) != DEMI_OK) return rc;
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  memset(out, 0, (size_t)n * sizeof(demi_incddmin_out));
  // each trace's program and seed, checked as demi_incremental_ddmin checks them: a trace that fails does so alone
  std::vector<SeedHost> sh(n);
  std::vector<int32_t> pre(n, DEMI_OK);
  std::vector<std::string> pre_msg(n);
  {
    demi_handle eh;
    for (uint32_t t = 0; t < n; t++) {
      int32_t prc = demi_check_dpor_program(&eh, "demi_incremental_ddmin", externals + ext_offsets[t], n_externals[t]);
      if (prc == DEMI_OK && seeds) prc = build_seed(&eh, seeds + t, sh[t]);
      if (prc != DEMI_OK) { pre[t] = prc; pre_msg[t] = eh.err; }
    }
  }
  // the seeds of every trace, uploaded once: the view table, then the nodes, the original indices and the traces
  std::vector<DporSeedView> views(n);
  std::vector<uint4> nodes;
  std::vector<int32_t> orig;
  std::vector<uint32_t> itrace;
  for (uint32_t t = 0; t < n; t++) {
    views[t] = DporSeedView{(uint32_t)nodes.size(), (uint32_t)sh[t].nodes.size(), (uint32_t)itrace.size(),
                            (uint32_t)sh[t].trace.size(), max_messages[t], looking_for[t], {0, 0}};
    nodes.insert(nodes.end(), sh[t].nodes.begin(), sh[t].nodes.end());
    orig.insert(orig.end(), sh[t].orig_index.begin(), sh[t].orig_index.end());
    itrace.insert(itrace.end(), sh[t].trace.begin(), sh[t].trace.end());
  }
  auto al = [](size_t b) { return (b + 15) & ~(size_t)15; };
  const size_t b_views = al(n * sizeof(DporSeedView)), b_nodes = al(nodes.size() * sizeof(uint4)), b_orig = al(orig.size() * sizeof(int32_t));
  DevBuf seed_dev;
  if ((rc = seed_dev.grow(h, b_views + b_nodes + b_orig + al(itrace.size() * sizeof(uint32_t)) + 16)) != DEMI_OK) return rc;
  char* base = seed_dev.get<char>();
  CUDA_TRY(h, cudaMemcpy(base, views.data(), n * sizeof(DporSeedView), cudaMemcpyHostToDevice));
  if (!nodes.empty()) CUDA_TRY(h, cudaMemcpy(base + b_views, nodes.data(), nodes.size() * sizeof(uint4), cudaMemcpyHostToDevice));
  if (!orig.empty()) CUDA_TRY(h, cudaMemcpy(base + b_views + b_nodes, orig.data(), orig.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
  if (!itrace.empty())
    CUDA_TRY(h, cudaMemcpy(base + b_views + b_nodes + b_orig, itrace.data(), itrace.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  const MultiSeeds seeds_dev{(const DporSeedView*)base, (const uint4*)(base + b_views), (const uint32_t*)(base + b_views + b_nodes + b_orig),
                             (const int32_t*)(base + b_views + b_nodes), nullptr};
  size_t free_b = 0, total_b = 0;
  CUDA_TRY(h, cudaMemGetInfo(&free_b, &total_b));
  const uint64_t budget = std::min<uint64_t>(MANY_DPOR_BYTES, free_b / 2);
  const bool arv = (flags & DEMI_DF_ARVIND_ORDERING) != 0;
  demi_perf perf{};
  // the union of a round's requests, in request order, split into launches that fit the budget
  auto serve = [&](std::vector<DporRequest*>& batch) -> int32_t {
    std::vector<uint32_t> tos, off(1, 0), coff(1, 0);
    std::vector<demi_ext_event> flat;
    std::vector<int32_t> caps;
    for (const DporRequest* q : batch) {
      const DporPayload& pl = *(const DporPayload*)q->payload;
      const demi_ext_event* ex = externals + ext_offsets[q->trace];
      for (size_t k = 0; k < q->n; k++) {
        const uint64_t* m = q->masks + k * mask_words;
        for (uint32_t i = 0; i < n_externals[q->trace]; i++) if ((m[i >> 6] >> (i & 63)) & 1ull) flat.push_back(ex[i]);
        off.push_back((uint32_t)flat.size());
        caps.insert(caps.end(), pl.caps->begin() + (*pl.cap_off)[k], pl.caps->begin() + (*pl.cap_off)[k + 1]);
        coff.push_back((uint32_t)caps.size());
        tos.push_back(q->trace);
      }
    }
    const size_t total = tos.size();
    std::vector<demi_dpor_result> res(total);
    for (size_t lo = 0; lo < total;) {
      size_t hi = lo;
      int32_t mm = 0;
      while (hi < total) {
        const int32_t m2 = std::max(mm, max_messages[tos[hi]]);
        if (hi > lo && (hi - lo + 1) * dpor_search_bytes(*params, (uint32_t)m2 + 2, dv->nq, arv, false) > budget) break;
        mm = m2; hi++;
      }
      const uint32_t m = (uint32_t)(hi - lo);
      demi_dpor_params Pl = *params;
      Pl.max_messages = mm;
      std::vector<uint32_t> loff(m + 1), lcoff(m + 1);
      for (uint32_t i = 0; i <= m; i++) { loff[i] = off[lo + i] - off[lo]; lcoff[i] = coff[lo + i] - coff[lo]; }
      MultiSeeds ms = seeds_dev;
      ms.trace_of_search = tos.data() + lo;
      const int32_t lrc = dpor_run(h, flat.data() + off[lo], loff.data(), m, &Pl, flags, nullptr, caps.data() + coff[lo], lcoff.data(),
                                   res.data() + lo, nullptr, 0, nullptr, 0, &ms);
      if (lrc != DEMI_OK) return lrc;
      perf.kernel_launches++; perf.kernel_ms += h->perf.kernel_ms; perf.prefixes += h->perf.prefixes;
      perf.deliveries += h->perf.deliveries; perf.violations += h->perf.violations;
      lo = hi;
    }
    scatter_results(batch, res);
    return DEMI_OK;
  };
  auto drive = [&](uint32_t t, Rendezvous<demi_dpor_result>& R, demi_handle* eh) -> int32_t {
    if (pre[t] != DEMI_OK) { eh->err = pre_msg[t]; return pre[t]; }
    ManyDporDriver d;
    d.R = &R; d.trace = t;
    d.h = eh; d.looking_for = looking_for[t]; d.flags = 0; d.mw = mask_words; d.n_ext = n_externals[t];
    d.ext = externals + ext_offsets[t];
    d.P = params; d.dflags = flags; d.seed = seeds ? &sh[t] : nullptr; d.max_messages = max_messages[t];
    return d.minimize(max_max_distance, stop_at_size, mcs_masks + (size_t)t * mask_words, out + t);
  };
  rc = run_many<demi_dpor_result>(h, who, n, window, drive, serve, status);
  h->perf.kernel_launches = perf.kernel_launches; h->perf.kernel_ms = perf.kernel_ms; h->perf.prefixes = perf.prefixes;
  h->perf.deliveries = perf.deliveries; h->perf.violations = perf.violations;
  for (DevBuf& d : h->dpor_buf) d.reset();             // a round's launches may hold far more than one trace's call needs
  if (rc != DEMI_OK) return rc;
  for (uint32_t t = 0; t < n; t++)
    if (status[t] != DEMI_OK) { h->err = trace_msg(who, t, h->err); break; }
  return DEMI_OK;
}
