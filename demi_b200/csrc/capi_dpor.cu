// capi_dpor.cu — C ABI for batched DPORwHeuristics searches (K3), the edit-distance bounded / resumable
// configuration of RunnerUtils.editDistanceDporDDMin, and IncrementalDDMin on top of it.
#include "dpor_kernel.cuh"
#include "models/model_ir.cuh"
#include "engine.hpp"
#include "ddmin_driver.hpp"

using namespace demi;

typedef void (*dpor_fn)(const DporArgs);
struct DporVariant { int model; int bd; dpor_fn fn; size_t smem; int nq; };
template <class MODEL, int BD>
static DporVariant make_dv() {
  using M = DporMachine<MODEL, BD>;
  return DporVariant{MODEL::ID, BD, dpor_kernel<MODEL, BD>, (size_t)M::WORDS * BD * sizeof(uint32_t), M::NQ};
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

int32_t dpor_run(demi_handle* h, const demi_ext_event* ext, const uint32_t* ext_offsets, uint32_t n_searches,
                 const demi_dpor_params* params, uint32_t flags, const SeedHost* seed,
                 const int32_t* caps, const uint32_t* cap_offsets, demi_dpor_result* results,
                 demi_dpor_violation* viol, uint32_t cap_viol, uint64_t* hashes, uint32_t cap_hashes) {
  const demi_dpor_params& P = *params;
  if (P.node_cap < 2 || P.node_cap > (1u << 20)) return fail(h, DEMI_ERR_INVALID, "node_cap must be in [2, 2^20]");
  if (P.explored_slots < 2 || (P.explored_slots & (P.explored_slots - 1))) return fail(h, DEMI_ERR_INVALID, "explored_slots must be a power of two");
  if (P.max_messages < 0 || P.max_messages > 1022) return fail(h, DEMI_ERR_INVALID, "max_messages must be in [0, 1022] (setMaxMessagesToSchedule)");
  if (!P.heap_cap || !P.max_interleavings) return fail(h, DEMI_ERR_INVALID, "heap_cap / max_interleavings must be positive");
  if (P.max_interleavings >= (1u << 20)) return fail(h, DEMI_ERR_INVALID, "max_interleavings must be below 2^20 (backtrack key packing)");
  if ((flags & DEMI_DF_ARVIND_ORDERING) && !seed) return fail(h, DEMI_ERR_INVALID, "ArvindDistanceOrdering needs the original trace (demi_dpor_seed)");
  if (seed && seed->nodes.size() > P.node_cap) return fail(h, DEMI_ERR_CAPACITY, "node_cap %u is below the seed graph's %zu nodes", P.node_cap, seed->nodes.size());
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
  if (seed) {
    up(a.init_nodes, seed->nodes.data(), n_seed_nodes * sizeof(uint4));
    up(a.init_trace, seed->trace.data(), n_seed_trace * sizeof(uint32_t));
    up(a.orig_index, seed->orig_index.data(), n_seed_nodes * sizeof(int32_t));
  }
  if (e == cudaSuccess && h->cfg.model == DEMI_MODEL_IR) e = ir_bind(h->ir_dev, h->stream);   // this unit's copy of g_ir
  // the race scan's position table goes to shared memory when it leaves room for >= 8 blocks per SM
  size_t smem = dv->smem;
  const size_t scan_bytes = (size_t)a.T1 * dv->bd * sizeof(uint32_t);
  a.scan_in_smem = (dv->smem + scan_bytes <= 27 * 1024) ? 1u : 0u;
  if (a.scan_in_smem) smem += scan_bytes;
  if (e == cudaSuccess) e = cudaFuncSetAttribute(dv->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e == cudaSuccess) e = cudaEventRecord(h->ev0, h->stream);
  if (e == cudaSuccess) {
    dv->fn<<<(n_searches + dv->bd - 1) / dv->bd, dv->bd, smem, h->stream>>>(a);
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

// ResumableDPOR (IncrementalDeltaDebugging.scala:90-122) as DDMin's TestOracle.  subseqToDPOR becomes
// `history`: the caps each subsequence's instance has been tested with by the SEQUENTIAL walk.  A test of mask m
// under the current cap is the outcome of a fresh instance put through history[m] ++ [cap]; evaluating it does not
// touch any state, so the speculative batch may contain tests the walk never asks for.
struct DporDDMinDriver : DDMinDriver {
  const demi_dpor_params* P; uint32_t dflags; const SeedHost* seed;
  int32_t cap = 0;
  std::map<Mask, std::vector<int32_t>> history;
  uint64_t interleavings = 0;

  int32_t evaluate(const uint64_t* masks, size_t n, signed char* out) override {
    std::vector<demi_ext_event> flat;
    std::vector<uint32_t> off(1, 0), coff(1, 0);
    std::vector<int32_t> caps;
    for (size_t k = 0; k < n; k++) {
      const uint64_t* m = masks + k * mw;
      for (uint32_t i = 0; i < n_ext; i++) if ((m[i >> 6] >> (i & 63)) & 1ull) flat.push_back(ext[i]);
      off.push_back((uint32_t)flat.size());
      auto it = history.find(Mask(m, m + mw));
      if (it != history.end()) caps.insert(caps.end(), it->second.begin(), it->second.end());
      caps.push_back(cap);
      coff.push_back((uint32_t)caps.size());
    }
    std::vector<demi_dpor_result> res(n);
    int32_t rc = dpor_run(h, flat.data(), off.data(), (uint32_t)n, P, dflags, seed, caps.data(), coff.data(),
                          res.data(), nullptr, 0, nullptr, 0);
    if (rc != DEMI_OK) return rc;
    for (size_t i = 0; i < n; i++) {
      if (res[i].status) return fail(h, DEMI_ERR_CAPACITY, "demi_incremental_ddmin: a DPOR instance reported status %u", res[i].status);
      out[i] = res[i].violations != 0;
      interleavings += res[i].interleavings;
    }
    return DEMI_OK;
  }
  // the walk called oracle.test(m): the instance has now seen this cap; a repeated test is a new question
  void consumed(const Mask& m) override { history[m].push_back(cap); memo.erase(m); }
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
  memset(out, 0, sizeof(*out));
  DporDDMinDriver d;
  d.h = h; d.looking_for = params->looking_for; d.flags = 0; d.mw = mask_words; d.n_ext = n_externals; d.ext = externals;
  d.P = params; d.dflags = flags; d.seed = seed ? &sh : nullptr;
  Mask cur(mask_words, 0), zero(mask_words, 0);
  for (uint32_t i = 0; i < n_externals; i++) DDMinDriver::setbit(cur, i);
  int32_t dist = 0;                                                              // oracle.setMaxDistance(currentDistance) :53
  while (dist < max_max_distance && DDMinDriver::popcount(cur) > stop_at_size) { // :66
    d.cap = dist;
    d.memo.clear();                                                              // ddmin = new DDMin(oracle, checkUnmodifed=false) :68
    d.original_num_events = DDMinDriver::popcount(cur); d.total_inputs_pruned = 0;
    cur = d.ddmin2(cur, zero);
    if (d.error != DEMI_OK) return d.error;
    out->rounds++;
    dist = dist == 0 ? 2 : dist << 1;                                            // :72
  }
  std::copy(cur.begin(), cur.end(), mcs_mask);
  out->mcs_size = DDMinDriver::popcount(cur);
  out->total_replays = d.total_replays;                                          // mergeStats :33-41
  out->instances = (uint32_t)d.history.size();
  out->tests_executed = d.replays_executed;
  out->batches = d.batches;
  out->interleavings_executed = d.interleavings;
  return DEMI_OK;
}
