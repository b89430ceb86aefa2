// capi_wildcard.cu — fungible clocks: WildcardMinimizer (minification/wildcard_minimization/WildcardMinimizer.scala:
// 133-241) with testScheduler = STSSched, ClockClusterizer (ClockClusterizer.scala:39-228) and OneAtATimeIterator
// (:230-290), Aggressiveness.ALL_TIMERS_FIRST_ITR.
//
// WildcardDriver (wildcard_driver.hpp) makes the decisions; here they are served on the handle's single trace: the
// tests a copy of the clusterizer would issue if every test failed are evaluated in one K2 launch (the WILD
// instantiation of replay_lane_kernel) and committed in order up to the first success; the successful one is re-run in
// recording mode for the trace and the ignored-absent ids, which are fed to the real clusterizer before speculating
// again.
#include "replay_kernel.cuh"
#include "engine.hpp"
#include "wildcard_driver.hpp"

using namespace demi;

namespace {
int32_t wc_analyse(demi_handle* h, const char* who, WcTrace& t) {
  if (h->trace_host.empty()) return fail(h, DEMI_ERR_STATE, "demi_set_trace has not been called");
  std::string msg;
  if (!t.build(h->trace_host.data(), (uint32_t)h->trace_host.size(), demi_ext_type_mask(h), h->clock_incr, who, msg))
    return fail(h, DEMI_ERR_INVALID, "%s", msg.c_str());
  return DEMI_OK;
}
}  // namespace

int32_t wc_check_flags(demi_handle* h, const char* who, uint32_t flags) {
  if (flags & DEMI_RF_STRICT) return fail(h, DEMI_ERR_INVALID, "%s: DEMI_RF_STRICT has no wildcard form", who);
  if (flags & ~(DEMI_RF_FILTER_KNOWN_ABSENTS | DEMI_WC_LAST_ONLY)) return fail(h, DEMI_ERR_INVALID, "%s: unknown flags 0x%x", who, flags);
  return DEMI_OK;
}

namespace {

// One launch of n_tests wildcard tests.  Device inputs live in the replay buffers of capi_replay.cu; the list this
// variant leaves in the table means the exact path clears the table before its next launch.
int32_t wc_launch(demi_handle* h, const WcTrace& t, const uint64_t* include_host, uint32_t n_tests, uint32_t looking_for,
                  uint32_t flags, demi_replay_result* out_host,
                  demi_event* rec_host, uint32_t rec_cap, uint32_t* n_rec,
                  uint32_t* ign_host, uint32_t ign_cap, uint32_t* n_ign) {
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  const bool record = rec_host != nullptr;
  cudaStream_t s = h->stream;
  int32_t rc;
  const uint32_t n_ext = (uint32_t)h->trace_ext_host.size();
  ReplayArgs a = replay_args(h, h->trace, looking_for, flags);
  a.pending_cap = demi_wildcard_pending_cap(demi_model_key(h), (uint32_t)t.pos.size(), h->trace.n_sends);
  a.table_slots = a.pending_cap;                        // list storage (the kernel compacts it in place)
  a.masks = nullptr; a.n_masks = n_tests; a.mask_words = std::max<uint32_t>(1, (n_ext + 63) / 64);   // the full MCS
  a.wc_words = t.words;
  std::copy(h->clock_incr, h->clock_incr + 8, a.wc_incr);
  const size_t ev_bytes = t.ev.size() * sizeof(uint32_t), inc_bytes = (size_t)n_tests * t.words * sizeof(uint64_t);
  // staging in rp_masks: include masks | per-event modes | the two REC counters
  const size_t ev_off = (inc_bytes + 15) & ~(size_t)15, cnt_off = (ev_off + ev_bytes + 15) & ~(size_t)15;
  if ((rc = h->rp_masks.grow(h, cnt_off + 16)) != DEMI_OK) return rc;
  if ((rc = h->rp_results.grow(h, (size_t)n_tests * sizeof(demi_replay_result))) != DEMI_OK) return rc;
  char* base = h->rp_masks.get<char>();
  uint32_t* counts = (uint32_t*)(base + cnt_off);
  CUDA_TRY(h, cudaMemcpyAsync(base, include_host, inc_bytes, cudaMemcpyHostToDevice, s));
  CUDA_TRY(h, cudaMemcpyAsync(base + ev_off, t.ev.data(), ev_bytes, cudaMemcpyHostToDevice, s));
  a.wc_include = (const uint64_t*)base; a.wc_ev = (const uint32_t*)(base + ev_off);
  a.results = h->rp_results.get<demi_replay_result>();
  DevBuf d_rec, d_ign;
  if (record) {
    if ((rc = d_rec.grow(h, (size_t)rec_cap * sizeof(demi_event))) != DEMI_OK) return rc;
    if ((rc = d_ign.grow(h, (size_t)std::max<uint32_t>(ign_cap, 1) * sizeof(uint32_t))) != DEMI_OK) return rc;
    CUDA_TRY(h, cudaMemsetAsync(counts, 0, 8, s));
    a.rec_events = d_rec.get<demi_event>(); a.rec_cap = rec_cap; a.rec_count = counts;
    a.wc_ignored = d_ign.get<uint32_t>(); a.wc_ignored_cap = ign_cap; a.wc_ignored_count = counts + 1;
  }
  if ((rc = replay_launch(h, a, true, record, nullptr, true, s)) != DEMI_OK) return rc;
  CUDA_TRY(h, cudaMemcpyAsync(out_host, a.results, (size_t)n_tests * sizeof(demi_replay_result), cudaMemcpyDeviceToHost, s));
  uint32_t c[2] = {0, 0};
  if (record) CUDA_TRY(h, cudaMemcpyAsync(c, counts, sizeof(c), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaStreamSynchronize(s));
  if (record && c[0]) CUDA_TRY(h, cudaMemcpy(rec_host, d_rec.get(), (size_t)std::min(c[0], rec_cap) * sizeof(demi_event), cudaMemcpyDeviceToHost));
  if (record && c[1] && ign_host) CUDA_TRY(h, cudaMemcpy(ign_host, d_ign.get(), (size_t)std::min(c[1], ign_cap) * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  float ms = 0;
  CUDA_TRY(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  h->perf.kernel_ms = ms; h->perf.kernel_launches = 1; h->perf.prefixes = n_tests;
  h->perf.h2d_bytes = inc_bytes + ev_bytes; h->perf.d2h_bytes = (size_t)n_tests * sizeof(demi_replay_result);
  if (record) {
    if (n_rec) *n_rec = c[0];
    if (n_ign) *n_ign = c[1];
    if (c[1] > ign_cap && ign_host) return fail(h, DEMI_ERR_CAPACITY, "wildcard replay: %u ignored deliveries, room for %u", c[1], ign_cap);
  }
  return DEMI_OK;
}

}  // namespace

extern "C" int32_t demi_set_clock_rules(demi_handle* h, const uint32_t* rules, uint32_t n_rules, const uint32_t* increment_types) {
  if (!h) return DEMI_ERR_INVALID;
  if (n_rules && !rules) return fail(h, DEMI_ERR_INVALID, "demi_set_clock_rules: null rules");
  uint32_t table[256] = {};
  for (uint32_t i = 0; i < n_rules; i++) {
    const uint32_t r = rules[i], type = r & 0xFF, word = (r >> 8) & 0xFF, shift = (r >> 16) & 0xFF, bits = r >> 24;
    if (word > 1) return fail(h, DEMI_ERR_INVALID, "demi_set_clock_rules: rule %u reads word %u (p0 or p1 only)", i, word);
    if (shift > 31) return fail(h, DEMI_ERR_INVALID, "demi_set_clock_rules: rule %u shifts by %u", i, shift);
    if (bits < 1 || bits > 32) return fail(h, DEMI_ERR_INVALID, "demi_set_clock_rules: rule %u has %u bits (1..32)", i, bits);
    if (table[type]) return fail(h, DEMI_ERR_INVALID, "demi_set_clock_rules: two rules for type %u", type);
    table[type] = r;
  }
  std::copy(table, table + 256, h->clock_rule);
  for (int w = 0; w < 8; w++) h->clock_incr[w] = increment_types ? increment_types[w] : 0u;
  return DEMI_OK;
}

extern "C" int32_t demi_wildcard_replay_batch(demi_handle* h, const uint64_t* include_masks, uint32_t n_tests,
                                              uint32_t looking_for, uint32_t flags, demi_replay_result* out) {
  if (!h) return DEMI_ERR_INVALID;
  if (!include_masks || !out) return fail(h, DEMI_ERR_INVALID, "demi_wildcard_replay_batch: null buffer");
  int32_t rc;
  if ((rc = wc_check_flags(h, "demi_wildcard_replay_batch", flags)) != DEMI_OK) return rc;
  WcTrace t;
  if ((rc = wc_analyse(h, "demi_wildcard_replay_batch", t)) != DEMI_OK) return rc;
  if (n_tests == 0) return DEMI_OK;
  return wc_launch(h, t, include_masks, n_tests, looking_for, flags, out, nullptr, 0, nullptr, nullptr, 0, nullptr);
}

extern "C" int32_t demi_wildcard_replay_trace(demi_handle* h, const uint64_t* include_mask, uint32_t looking_for, uint32_t flags,
                                              demi_event* events, uint32_t cap_events, uint32_t* n_events,
                                              uint32_t* ignored_positions, uint32_t cap_ignored, uint32_t* n_ignored,
                                              demi_replay_result* result) {
  if (!h) return DEMI_ERR_INVALID;
  if (!include_mask || !events || !cap_events || !result) return fail(h, DEMI_ERR_INVALID, "demi_wildcard_replay_trace: null buffer");
  int32_t rc;
  if ((rc = wc_check_flags(h, "demi_wildcard_replay_trace", flags)) != DEMI_OK) return rc;
  WcTrace t;
  if ((rc = wc_analyse(h, "demi_wildcard_replay_trace", t)) != DEMI_OK) return rc;
  return wc_launch(h, t, include_mask, 1, looking_for, flags, result, events, cap_events, n_events,
                   ignored_positions, ignored_positions ? cap_ignored : 0, n_ignored);
}

extern "C" int32_t demi_wildcard_minimize(demi_handle* h, uint32_t looking_for, uint32_t flags,
                                          demi_event* out_trace, uint32_t cap_events,
                                          uint32_t* internal_sizes, uint32_t cap_sizes, demi_intmin_out* out) {
  if (!h) return DEMI_ERR_INVALID;
  if (!out) return fail(h, DEMI_ERR_INVALID, "demi_wildcard_minimize: null output");
  int32_t rc;
  if ((rc = wc_check_flags(h, "demi_wildcard_minimize", flags)) != DEMI_OK) return rc;
  if (h->trace_host.empty()) return fail(h, DEMI_ERR_STATE, "demi_set_trace has not been called");
  const std::vector<demi_ext_event> ext = h->trace_ext_host;
  WildcardDriver d;
  if (!d.init(h->trace_host.data(), (uint32_t)h->trace_host.size(), demi_ext_type_mask(h), h->clock_rule, h->clock_incr, out))
    return fail(h, d.error, "%s", d.msg.c_str());
  std::vector<demi_event> rec(65536);
  std::vector<uint32_t> ign_pos(d.t.pos.size() + 1);
  for (;;) {
    const std::vector<uint64_t>& cand = d.candidates();
    if (cand.empty()) break;
    std::vector<demi_replay_result> res(d.n_candidates());
    if ((rc = wc_launch(h, d.t, cand.data(), (uint32_t)res.size(), looking_for, flags, res.data(),
                        nullptr, 0, nullptr, nullptr, 0, nullptr)) != DEMI_OK) return rc;
    const uint64_t* mask = nullptr;
    const WildcardDriver::Step step = d.commit(res.data(), &mask);
    if (step == WildcardDriver::FAILED) return fail(h, d.error, "%s", d.msg.c_str());
    if (step == WildcardDriver::DONE) continue;
    uint32_t n_rec = 0, n_ign = 0; demi_replay_result r1;
    if ((rc = wc_launch(h, d.t, mask, 1, looking_for, flags, &r1, rec.data(), (uint32_t)rec.size(), &n_rec,
                        ign_pos.data(), (uint32_t)ign_pos.size(), &n_ign)) != DEMI_OK) return rc;
    if (!d.advance(r1, rec.data(), n_rec, ign_pos.data(), n_ign)) return fail(h, d.error, "%s", d.msg.c_str());
  }
  if ((rc = demi_set_trace(h, d.min_trace.data(), (uint32_t)d.min_trace.size(), ext.data(), (uint32_t)ext.size())) != DEMI_OK) return rc;
  d.finish(out_trace, cap_events, internal_sizes, cap_sizes);
  return DEMI_OK;
}
