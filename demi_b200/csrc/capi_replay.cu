// capi_replay.cu — C ABI for STSSched replay batches (K2) and DDMin.
//
// DDMin (minification/DeltaDebugging.scala:27-109) is sequential by definition:
// every test depends on the outcome of the previous one.  Here the recursion is
// still walked in exactly that order (so the decisions, the MCS and the
// MinimizationStats counters are the sequential ones), but test outcomes come
// from a memo that is filled speculatively: whenever the walk needs a test that
// has not been evaluated, the possible futures of the current ddmin2 frame (and of
// the interference siblings waiting on the recursion stack) are expanded a few
// levels deep and evaluated in ONE kernel launch.
#include <map>
#include <deque>
#include "replay_kernel.cuh"
#include "engine.hpp"
#include "models/model_ir.cuh"

using namespace demi;

namespace {
typedef void (*replay_fn)(const ReplayArgs);
typedef void (*replay_many_fn)(const ReplayArgs, const ReplayTraceView*, const uint4*, uint32_t, ReplayArgs*,
                               const uint32_t* const*);
// K2 per model: the four instantiations of replay_lane_kernel, fn[WILD][REC], and of replay_many_kernel, many[WILD][REC], at the
// model's block size and shared memory.  Every K2 instantiation is in this unit, so that its copy of model_ir.cuh's
// loaded model is the one K2 reads.
struct ReplayVariant { int model; int bd; replay_fn fn[2][2]; replay_many_fn many[2][2]; size_t smem; int n_actors; };
template <class MODEL>
ReplayVariant make_rv() {
  constexpr int BD = replay_block<MODEL>;
  using M = ReplayMachine<MODEL, BD>;     // WORDS does not depend on REC or WILD
  return ReplayVariant{MODEL::ID, BD,
                       {{replay_lane_kernel<MODEL, BD, false, false>, replay_lane_kernel<MODEL, BD, true, false>},
                        {replay_lane_kernel<MODEL, BD, false, true>, replay_lane_kernel<MODEL, BD, true, true>}},
                       {{replay_many_kernel<MODEL, BD, false, false>, replay_many_kernel<MODEL, BD, true, false>},
                        {replay_many_kernel<MODEL, BD, false, true>, replay_many_kernel<MODEL, BD, true, true>}},
                       (size_t)M::WORDS * BD * sizeof(uint32_t), MODEL::N_ACTORS};
}
const ReplayVariant* pick_rv(int model) {
  static const std::vector<ReplayVariant> v = {make_rv<PingPong3>(), make_rv<Raft5>(), make_rv<Bcast32>(), make_rv<IrModel>()};
  for (const ReplayVariant& r : v) if (r.model == model) return &r;
  return nullptr;
}
}  // namespace

ReplayArgs replay_args(const demi_handle* h, const ReplayTraceView& trace, uint32_t looking_for, uint32_t flags) {
  ReplayArgs a{};
  a.model_flags = h->cfg.model_flags; a.blocked_mask = h->cfg.blocked_mask; a.ignore_timers = h->cfg.ignore_timers;
  a.looking_for = looking_for; a.flags = flags;
  a.external_type_mask = demi_ext_type_mask(h);
  bind_trace(a, trace);
  return a;
}

int32_t check_trace(demi_handle* h, const char* who, const demi_event* events, uint32_t n_events,
                    const demi_ext_event* externals, uint32_t n_externals) {
  if (!events || !n_events || !externals || !n_externals)
    return fail(h, DEMI_ERR_INVALID, "%s: empty trace or externals", who);   // assume(!original_trace.isEmpty)
  if (n_externals > 4096) return fail(h, DEMI_ERR_INVALID, "%s: more than 4096 external events", who);
  if (n_events >= (1u << 31)) return fail(h, DEMI_ERR_INVALID, "%s: trace too long", who);
  int32_t vrc = demi_check_events(h, who, events, n_events, 0); if (vrc != DEMI_OK) return vrc;
  return demi_check_externals(h, who, externals, n_externals);   // (rejects HardKill)
}

int32_t trace_tables(demi_handle* h, const char* who, const demi_event* events, uint32_t n_events,
                     const demi_ext_event* externals, uint32_t n_externals, TraceTables& t) {
  const uint32_t ext_mask = demi_ext_type_mask(h);
  // FIFO correspondence of external MsgSends and original Sends (EventTrace.scala:385-386, :419-436)
  t.ordinal.assign(n_events, 0xFFFF);
  std::map<uint32_t, uint16_t> uniq_to_ord;
  uint32_t ord = 0, max_uniq = 0, n_send_events = 0;
  for (uint32_t i = 0; i < n_events; i++) {
    const demi_event& e = events[i];
    if (e.kind < DEMI_EV_MSG_SEND || e.kind > DEMI_EV_QUIESCENCE)
      return fail(h, DEMI_ERR_INVALID, "%s: event %u has unknown kind %u", who, i, e.kind);
    if (e.kind == DEMI_EV_MSG_SEND) {
      n_send_events++;
      if (e.uniq > max_uniq) max_uniq = e.uniq;
      if (demi_type_is_external(ext_mask, e.type)) {
        if (ord >= 0xFFFF) return fail(h, DEMI_ERR_INVALID, "%s: too many external sends", who);
        t.ordinal[i] = (uint16_t)ord; uniq_to_ord[e.uniq] = (uint16_t)ord; ord++;
      }
    }
  }
  for (uint32_t i = 0; i < n_events; i++)
    if (events[i].kind == DEMI_EV_MSG_EVENT) {
      auto it = uniq_to_ord.find(events[i].uniq);
      if (it != uniq_to_ord.end()) t.ordinal[i] = it->second;
      if (events[i].uniq > max_uniq) max_uniq = events[i].uniq;
    }
  t.sidx.clear();
  for (uint32_t i = 0; i < n_externals; i++) if (externals[i].kind == DEMI_EXT_SEND) t.sidx.push_back((uint16_t)i);
  t.n_uniq = max_uniq + 1;
  t.n_send_events = n_send_events;
  return DEMI_OK;
}

ReplayTraceView trace_view(const TraceTables& t, uint32_t n_events, uint32_t n_externals) {
  ReplayTraceView v{};
  v.n_events = n_events; v.n_ext = n_externals; v.n_sends = (uint32_t)t.sidx.size();
  v.n_uniq_words = (t.n_uniq + 31) / 32;
  v.pending_cap = demi_replay_pending_cap(t.n_send_events);
  v.tosend_cap = demi_tosend_cap(v.n_sends);
  v.table_slots = demi_pow2_at_least(2 * v.pending_cap, 256, 1u << 16);
  return v;
}

extern "C" int32_t demi_set_trace(demi_handle* h, const demi_event* events, uint32_t n_events,
                                  const demi_ext_event* externals, uint32_t n_externals) {
  if (!h) return DEMI_ERR_INVALID;
  { int32_t vrc = check_trace(h, "demi_set_trace", events, n_events, externals, n_externals); if (vrc != DEMI_OK) return vrc; }
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  { int32_t mrc = demi_need_model(h); if (mrc != DEMI_OK) return mrc; }
  TraceTables t;
  int32_t rc;
  if ((rc = trace_tables(h, "demi_set_trace", events, n_events, externals, n_externals, t)) != DEMI_OK) return rc;
  const std::vector<uint16_t>& sidx = t.sidx;
  DevBuf ext_dev, ord_dev, sidx_dev, trace_dev;
  if ((rc = ext_dev.upload(h, externals, n_externals * sizeof(demi_ext_event))) != DEMI_OK) return rc;
  if ((rc = ord_dev.upload(h, t.ordinal.data(), n_events * sizeof(uint16_t))) != DEMI_OK) return rc;
  if ((rc = sidx_dev.grow(h, std::max<size_t>(sidx.size(), 1) * sizeof(uint16_t))) != DEMI_OK) return rc;
  if (!sidx.empty())
    CUDA_TRY(h, cudaMemcpy(sidx_dev.get(), sidx.data(), sidx.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
  if ((rc = trace_dev.upload(h, events, n_events * sizeof(demi_event))) != DEMI_OK) return rc;
  if ((rc = h->rp_counters.grow(h, 2 * sizeof(unsigned long long))) != DEMI_OK) return rc;     // allocated once per handle
  h->trace_host.assign(events, events + n_events);
  h->trace_ext_host.assign(externals, externals + n_externals);
  h->conjoined.assign(n_externals, -1);                       // a new EventDag has no conjoined atoms
  h->trace = trace_view(t, n_events, n_externals);
  h->trace.events = trace_dev.get<const uint4>(); h->trace.ev_ordinal = ord_dev.get<const uint16_t>();
  h->trace.ext = ext_dev.get<const uint4>(); h->trace.send_ext_index = sidx_dev.get<const uint16_t>();
  h->trace_dev = std::move(trace_dev); h->trace_ext_dev = std::move(ext_dev);
  h->ev_ordinal_dev = std::move(ord_dev); h->send_ext_index_dev = std::move(sidx_dev);
  return DEMI_OK;
}

extern "C" int32_t demi_conjoin_atoms(demi_handle* h, uint32_t e1, uint32_t e2) {
  if (!h) return DEMI_ERR_INVALID;
  if (h->trace_ext_host.empty()) return fail(h, DEMI_ERR_STATE, "demi_set_trace has not been called");
  const uint32_t n = (uint32_t)h->trace_ext_host.size();
  if (e1 >= n || e2 >= n) return fail(h, DEMI_ERR_INVALID, "No such external event: %u", e1 >= n ? e1 : e2);   // :168-173
  if (e1 == e2) return fail(h, DEMI_ERR_INVALID, "demi_conjoin_atoms: an event cannot be conjoined with itself");
  if (h->conjoined[e1] >= 0 || h->conjoined[e2] >= 0)                          // the asserts at :174-175
    return fail(h, DEMI_ERR_STATE, "demi_conjoin_atoms: external %u is already conjoined", h->conjoined[e1] >= 0 ? e1 : e2);
  h->conjoined[e1] = (int32_t)e2; h->conjoined[e2] = (int32_t)e1;
  return DEMI_OK;
}

namespace {
// How a launch uses the table: hash tables stamped with the launch's generations (exact replays), or the insertion-
// ordered list of the REC variant (a recording) or of the WILD variants
enum class TableUse { GENERATIONS, RECORD, LIST };

cudaError_t replay_ir_bind(const demi_handle* h, cudaStream_t s) {
  return h->cfg.model == DEMI_MODEL_IR ? ir_bind(h->ir_dev, s) : cudaSuccess;
}

// The per-warp scratch of a K2 launch of `warps` warps with a's geometry (table_slots, tosend_cap, n_uniq_words, flags),
// its first generation and its counters, all in a.  Generation stamps: each launch gets a fresh range [gen_base,
// gen_base + tests per thread]; the table is cleared only when it was (re)allocated, its geometry changed, or the
// 16-bit range is exhausted.  A list leaves its entries behind, so the launch after it clears the table
// (rp_gen_next = 0); a single recording clears it first too.  A wildcard list and the recordings of a multi-trace
// launch need no clearing of their own: a test reads only the entries it wrote.
int32_t replay_scratch(demi_handle* h, ReplayArgs& a, uint64_t warps, int n_actors, uint32_t per_thread, TableUse use,
                       cudaStream_t s) {
  int32_t rc;
  const size_t table_bytes = warps * a.table_slots * 32 * sizeof(uint4);
  const bool fresh_table = h->rp_table.bytes() < table_bytes;
  if ((rc = h->rp_table.grow(h, table_bytes)) != DEMI_OK) return rc;
  if ((rc = h->rp_tosend.grow(h, warps * a.tosend_cap * 32 * sizeof(uint32_t))) != DEMI_OK) return rc;
  if (a.flags & DEMI_RF_FILTER_KNOWN_ABSENTS)
    if ((rc = h->rp_pruned.grow(h, warps * (a.n_uniq_words + n_actors) * 32 * sizeof(uint32_t))) != DEMI_OK) return rc;
  if (use == TableUse::LIST) {
    a.gen_base = 1;
  } else {
    const uint64_t geometry = ((uint64_t)a.table_slots << 32) ^ warps;
    if (fresh_table || h->rp_gen_next == 0 || h->rp_table_geometry != geometry || h->rp_gen_next + per_thread >= 0xFFF0u ||
        use == TableUse::RECORD) {
      CUDA_TRY(h, cudaMemsetAsync(h->rp_table.get(), 0, table_bytes, s));
      h->rp_gen_next = 1;
      h->rp_table_geometry = geometry;
    }
    a.gen_base = h->rp_gen_next;
  }
  h->rp_gen_next = use == TableUse::GENERATIONS ? h->rp_gen_next + per_thread : 0;
  CUDA_TRY(h, cudaMemsetAsync(h->rp_counters.get(), 0, 2 * sizeof(unsigned long long), s));
  a.table = h->rp_table.get<uint4>(); a.tosend = h->rp_tosend.get<uint32_t>();
  a.pruned = (a.flags & DEMI_RF_FILTER_KNOWN_ABSENTS) ? h->rp_pruned.get<uint32_t>() : nullptr;
  a.counters = h->rp_counters.get<unsigned long long>();
  return DEMI_OK;
}
}  // namespace

int32_t replay_launch(demi_handle* h, ReplayArgs& a, bool wild, bool record, const ReplayTiles* many, bool timed,
                      cudaStream_t s) {
  const ReplayVariant* rv = pick_rv(h->cfg.model);
  if (!rv) return fail(h, DEMI_ERR_INVALID, "no replay kernel for model %d", h->cfg.model);
  int32_t rc;
  int bps = 0;
  const void* fn = many ? (const void*)rv->many[wild][record] : (const void*)rv->fn[wild][record];
  if ((rc = demi_occupancy(h, fn, rv->bd, rv->smem, &bps)) != DEMI_OK) return rc;
  if (bps < 1) return fail(h, DEMI_ERR_CAPACITY, "replay kernel does not fit on an SM");
  // a block takes a test per thread of the single-trace kernel, a tile per warp of the multi-trace one; a recording
  // runs one test, so one block
  const uint32_t wpb = (uint32_t)rv->bd / 32, per_block = many ? wpb : (uint32_t)rv->bd;
  const uint64_t items = many ? many->n_tiles : a.n_masks;
  uint64_t blocks = std::min<uint64_t>((items + per_block - 1) / per_block, (uint64_t)h->sm_count * bps);
  // a wildcard list holds table_slots uint4 per lane: keep the scratch under 4 GiB
  if (wild) blocks = std::min<uint64_t>(blocks, std::max<uint64_t>(1, (4ull << 30) / ((uint64_t)a.table_slots * 32 * sizeof(uint4)) / wpb));
  const int grid = (int)std::max<uint64_t>(1, blocks);
  const uint64_t warps = (uint64_t)grid * wpb;
  const uint32_t per_thread = (uint32_t)((items + (uint64_t)grid * per_block - 1) / ((uint64_t)grid * per_block)) + 1;
  const TableUse use = wild || (record && many) ? TableUse::LIST : record ? TableUse::RECORD : TableUse::GENERATIONS;
  if ((rc = replay_scratch(h, a, warps, rv->n_actors, per_thread, use, s)) != DEMI_OK) return rc;
  if (many && (rc = h->rp_bound.grow(h, warps * sizeof(ReplayArgs))) != DEMI_OK) return rc;
  CUDA_TRY(h, replay_ir_bind(h, s));
  if (timed) CUDA_TRY(h, cudaEventRecord(h->ev0, s));
  if (many)
    rv->many[wild][record]<<<grid, rv->bd, rv->smem, s>>>(a, many->views, many->tiles, many->n_tiles, h->rp_bound.get<ReplayArgs>(),
                                                          many->modes);
  else rv->fn[wild][record]<<<grid, rv->bd, rv->smem, s>>>(a);
  CUDA_TRY(h, cudaGetLastError());
  if (timed) CUDA_TRY(h, cudaEventRecord(h->ev1, s));
  return DEMI_OK;
}

static int32_t launch_replay(demi_handle* h, const void* masks_dev, const void* skips_dev, uint32_t n_masks, uint32_t mask_words,
                             uint32_t looking_for, uint32_t flags, void* out_dev, void* stream,
                             demi_event* rec_dev, uint32_t rec_cap, uint32_t* rec_count_dev) {
  if (!h) return DEMI_ERR_INVALID;
  if (h->trace_host.empty()) return fail(h, DEMI_ERR_STATE, "demi_set_trace has not been called");
  if (!out_dev) return fail(h, DEMI_ERR_INVALID, "replay: null output buffer");
  const uint32_t n_ext = (uint32_t)h->trace_ext_host.size();
  if (masks_dev && mask_words * 64 < n_ext) return fail(h, DEMI_ERR_INVALID, "mask_words %u too small for %u externals", mask_words, n_ext);
  if (n_masks == 0) return DEMI_OK;
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  ReplayArgs a = replay_args(h, h->trace, looking_for, flags);
  a.masks = (const uint64_t*)masks_dev; a.n_masks = n_masks; a.mask_words = mask_words;
  a.skips = (const uint32_t*)skips_dev;
  a.rec_events = rec_dev; a.rec_cap = rec_cap; a.rec_count = rec_count_dev;
  a.results = (demi_replay_result*)out_dev;
  const int32_t rc = replay_launch(h, a, false, rec_dev != nullptr, nullptr, false, (cudaStream_t)stream);
  if (rc != DEMI_OK) return rc;
  h->perf.kernel_launches = 1;
  h->perf.prefixes = n_masks;
  return DEMI_OK;
}

extern "C" int32_t demi_replay_batch_dev(demi_handle* h, const void* masks_dev, uint32_t n_masks, uint32_t mask_words,
                                         uint32_t looking_for, uint32_t flags, void* out_dev, void* stream) {
  if (!h) return DEMI_ERR_INVALID;
  if (!masks_dev) return fail(h, DEMI_ERR_INVALID, "demi_replay_batch_dev: null buffer");
  return launch_replay(h, masks_dev, nullptr, n_masks, mask_words, looking_for, flags, out_dev, stream, nullptr, 0, nullptr);
}

extern "C" int32_t demi_replay_batch_ex(demi_handle* h, const uint64_t* masks, const uint32_t* skip_events, uint32_t n_tests,
                                        uint32_t mask_words, uint32_t looking_for, uint32_t flags, demi_replay_result* out_host) {
  if (!h) return DEMI_ERR_INVALID;
  if (!out_host) return fail(h, DEMI_ERR_INVALID, "demi_replay_batch_ex: null output");
  if (n_tests == 0) return DEMI_OK;
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  int32_t rc;
  const size_t mbytes = masks ? (size_t)n_tests * mask_words * sizeof(uint64_t) : 0, rbytes = (size_t)n_tests * sizeof(demi_replay_result);
  const size_t sbytes = skip_events ? (size_t)n_tests * sizeof(uint32_t) : 0;
  if ((rc = h->rp_masks.grow(h, std::max<size_t>(mbytes + sbytes, 8))) != DEMI_OK) return rc;
  if ((rc = h->rp_results.grow(h, rbytes)) != DEMI_OK) return rc;
  char* base = h->rp_masks.get<char>();
  if (masks) CUDA_TRY(h, cudaMemcpyAsync(base, masks, mbytes, cudaMemcpyHostToDevice, h->stream));
  if (skip_events) CUDA_TRY(h, cudaMemcpyAsync(base + mbytes, skip_events, sbytes, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaEventRecord(h->ev0, h->stream));
  rc = launch_replay(h, masks ? base : nullptr, skip_events ? base + mbytes : nullptr, n_tests, mask_words, looking_for, flags,
                     h->rp_results.get(), h->stream, nullptr, 0, nullptr);
  if (rc != DEMI_OK) return rc;
  CUDA_TRY(h, cudaEventRecord(h->ev1, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(out_host, h->rp_results.get(), rbytes, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  float ms = 0;
  CUDA_TRY(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  h->perf.kernel_ms = ms; h->perf.h2d_bytes = mbytes + sbytes; h->perf.d2h_bytes = rbytes;
  return DEMI_OK;
}

extern "C" int32_t demi_replay_trace(demi_handle* h, const uint64_t* mask, uint32_t mask_words, uint32_t skip_event,
                                     uint32_t looking_for, uint32_t flags,
                                     demi_event* events, uint32_t cap_events, uint32_t* n_events, demi_replay_result* result) {
  if (!h) return DEMI_ERR_INVALID;
  if (!events || !cap_events || !result) return fail(h, DEMI_ERR_INVALID, "demi_replay_trace: null buffer");
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  DevBuf d_mask, d_skip, d_rec, d_cnt, d_res;
  int32_t rc;
  if ((rc = d_rec.grow(h, (size_t)cap_events * sizeof(demi_event))) != DEMI_OK) return rc;
  if ((rc = d_cnt.grow(h, 4)) != DEMI_OK) return rc;
  if ((rc = d_res.grow(h, sizeof(demi_replay_result))) != DEMI_OK) return rc;
  if ((rc = d_skip.grow(h, 4)) != DEMI_OK) return rc;
  if (mask && (rc = d_mask.grow(h, (size_t)mask_words * 8)) != DEMI_OK) return rc;
  if (mask) CUDA_TRY(h, cudaMemcpyAsync(d_mask.get(), mask, (size_t)mask_words * 8, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(d_skip.get(), &skip_event, 4, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(d_cnt.get(), 0, 4, h->stream));
  if ((rc = launch_replay(h, d_mask.get(), d_skip.get(), 1, mask_words, looking_for, flags, d_res.get(), h->stream,
                          d_rec.get<demi_event>(), cap_events, d_cnt.get<uint32_t>())) != DEMI_OK) return rc;
  uint32_t cnt = 0;
  CUDA_TRY(h, cudaMemcpyAsync(&cnt, d_cnt.get(), 4, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(result, d_res.get(), sizeof(demi_replay_result), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (cnt) CUDA_TRY(h, cudaMemcpy(events, d_rec.get(), (size_t)std::min(cnt, cap_events) * sizeof(demi_event), cudaMemcpyDeviceToHost));
  if (n_events) *n_events = cnt;
  return DEMI_OK;
}

extern "C" int32_t demi_replay_batch(demi_handle* h, const uint64_t* masks, uint32_t n_masks, uint32_t mask_words,
                                     uint32_t looking_for, uint32_t flags, demi_replay_result* out_host) {
  if (!h) return DEMI_ERR_INVALID;
  if (!masks || !out_host) return fail(h, DEMI_ERR_INVALID, "demi_replay_batch: null buffer");
  if (n_masks == 0) return DEMI_OK;
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  int32_t rc;
  const size_t mbytes = (size_t)n_masks * mask_words * sizeof(uint64_t), rbytes = (size_t)n_masks * sizeof(demi_replay_result);
  if ((rc = h->rp_masks.grow(h, mbytes)) != DEMI_OK) return rc;
  if ((rc = h->rp_results.grow(h, rbytes)) != DEMI_OK) return rc;
  CUDA_TRY(h, cudaMemcpyAsync(h->rp_masks.get(), masks, mbytes, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaEventRecord(h->ev0, h->stream));
  rc = demi_replay_batch_dev(h, h->rp_masks.get(), n_masks, mask_words, looking_for, flags, h->rp_results.get(), h->stream);
  if (rc != DEMI_OK) return rc;
  CUDA_TRY(h, cudaEventRecord(h->ev1, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(out_host, h->rp_results.get(), rbytes, cudaMemcpyDeviceToHost, h->stream));
  unsigned long long c[2] = {0, 0};
  CUDA_TRY(h, cudaMemcpyAsync(c, h->rp_counters.get(), sizeof(c), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  float ms = 0;
  CUDA_TRY(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  h->perf.kernel_ms = ms; h->perf.violations = c[0]; h->perf.deliveries = c[1];
  h->perf.h2d_bytes = mbytes; h->perf.d2h_bytes = rbytes + sizeof(c);
  return DEMI_OK;
}

// ---------------------------------------------------------------------- DDMin
#include "ddmin_driver.hpp"

int32_t replay_verdicts(demi_handle* h, const demi_replay_result* res, size_t n, signed char* out) {
  for (size_t i = 0; i < n; i++) {
    if (res[i].status != 0) return fail(h, DEMI_ERR_CAPACITY, "demi_ddmin: a replay reported status %u", (unsigned)res[i].status);
    out[i] = res[i].violation != 0;
  }
  return DEMI_OK;
}

namespace {

// STSSched as DDMin's TestOracle: a batch of masks = one replay launch
struct StsDDMinDriver : DDMinDriver {
  int32_t evaluate(const uint64_t* masks, size_t n, signed char* out) override {   // the slice goes to the kernel as is
    std::vector<demi_replay_result> res(n);
    const int32_t rc = demi_replay_batch(h, masks, (uint32_t)n, mw, looking_for, flags, res.data());
    return rc != DEMI_OK ? rc : replay_verdicts(h, res.data(), n, out);
  }
};

}  // namespace

int32_t ddmin_sts(DDMinDriver& d, int32_t check_unmodified, uint64_t* mcs_mask, uint32_t* iteration_sizes,
                  uint32_t cap_iterations, demi_ddmin_out* out) {
  demi_handle* h = d.h;
  const uint32_t mask_words = d.mw, n_ext = d.n_ext;
  // tests per speculative batch: a launch costs ~3 ms of latency whatever its size (one test walks the whole trace),
  // building a batch ~0.2 us per test on the host; ~6000 tests = five to six levels of the decision tree per launch
  d.wide_cap = getenv("DEMI_DDMIN_WIDE") ? (size_t)atol(getenv("DEMI_DDMIN_WIDE")) : 6000;
  // STSSched ignores WaitQuiescence: drop them from the DAG (RunnerUtils.scala:678-684)
  Mask dag(mask_words, 0), zero(mask_words, 0);
  for (uint32_t i = 0; i < n_ext; i++) if (d.ext[i].kind != DEMI_EXT_WAIT_QUIESCENCE) DDMinDriver::setbit(dag, i);
  if (check_unmodified) {                                                 // DeltaDebugging.scala:41-47
    bool v = d.test(dag, dag, zero);
    if (d.error != DEMI_OK) return d.error;
    if (!v) return fail(h, DEMI_ERR_INVALID, "Unmodified trace does not trigger violation");
  }
  d.original_num_events = DDMinDriver::popcount(dag);
  Mask mcs = d.ddmin2(dag, zero);
  if (d.error != DEMI_OK) return d.error;
  d.iteration_sizes.push_back(d.original_num_events - d.total_inputs_pruned);     // fencepost :60
  // assert(original_num_events - total_inputs_pruned == mcs.length) :58
  if (d.original_num_events - d.total_inputs_pruned != DDMinDriver::popcount(mcs))
    return fail(h, DEMI_ERR_STATE, "demi_ddmin: bookkeeping assertion failed (DeltaDebugging.scala:58)");
  std::copy(mcs.begin(), mcs.end(), mcs_mask);
  // verify_mcs (DeltaDebugging.scala:64-71; RunnerUtils.scala:689-701)
  bool verified = d.test(mcs, mcs, zero);
  if (d.error != DEMI_OK) return d.error;
  out->mcs_size = DDMinDriver::popcount(mcs);
  out->reserved[0] = (uint32_t)d.spec_us; out->reserved[1] = (uint32_t)d.eval_us;    // host microseconds: building batches / evaluating them
  out->total_replays = d.total_replays;
  out->n_iterations = (uint32_t)d.iteration_sizes.size();
  out->replays_executed = d.replays_executed;
  out->batches = d.batches;
  out->verified = verified ? 1u : 0u;
  if (iteration_sizes)
    for (uint32_t i = 0; i < cap_iterations && i < out->n_iterations; i++) iteration_sizes[i] = d.iteration_sizes[i];
  return DEMI_OK;
}

extern "C" int32_t demi_ddmin(demi_handle* h, uint32_t looking_for, uint32_t flags, int32_t check_unmodified,
                              uint64_t* mcs_mask, uint32_t mask_words,
                              uint32_t* iteration_sizes, uint32_t cap_iterations, demi_ddmin_out* out) {
  if (!h) return DEMI_ERR_INVALID;
  if (!mcs_mask || !out) return fail(h, DEMI_ERR_INVALID, "demi_ddmin: null output");
  if (h->trace_host.empty()) return fail(h, DEMI_ERR_STATE, "demi_set_trace has not been called");
  const uint32_t n_ext = (uint32_t)h->trace_ext_host.size();
  if (mask_words * 64 < n_ext) return fail(h, DEMI_ERR_INVALID, "mask_words too small");
  memset(out, 0, sizeof(*out));
  StsDDMinDriver d;
  d.h = h; d.looking_for = looking_for; d.flags = flags; d.mw = mask_words; d.n_ext = n_ext;
  d.ext = h->trace_ext_host.data();
  d.conjoined = &h->conjoined;
  return ddmin_sts(d, check_unmodified, mcs_mask, iteration_sizes, cap_iterations, out);
}
