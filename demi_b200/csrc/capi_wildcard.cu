// capi_wildcard.cu — fungible clocks: WildcardMinimizer (minification/wildcard_minimization/WildcardMinimizer.scala:
// 133-241) with testScheduler = STSSched, ClockClusterizer (ClockClusterizer.scala:39-228) and OneAtATimeIterator
// (:230-290), Aggressiveness.ALL_TIMERS_FIRST_ITR.
//
// Every test the clusterizer issues is one STSScheduler.test of the SAME base trace (ClockClusterizer keeps
// `originalTrace`), described by which of its deliveries are included; the next test depends on earlier outcomes
// only through the clusterizer's blacklists.  So, as in capi_intmin.cu, the tests a copy of the clusterizer would
// issue if every test failed are evaluated in one K2 launch (the WILD instantiation of replay_lane_kernel) and
// committed in order up to the first success; the successful one is re-run in recording mode for the trace and
// the ignored-absent ids, which are fed to the real clusterizer before speculating again.
#include <set>
#include "replay_kernel.cuh"
#include "engine.hpp"

using namespace demi;

namespace {
inline bool incr_of(const demi_handle* h, uint32_t type) { return (h->clock_incr[type >> 5] >> (type & 31)) & 1u; }
// FingerprintFactory.getLogicalClock as data: false = None
inline bool clock_of(const demi_handle* h, const demi_event& e, uint32_t& clock) {
  const uint32_t r = h->clock_rule[e.type];
  if (!r) return false;
  const uint32_t word = (r >> 8) & 0xFF, shift = (r >> 16) & 0xFF, bits = r >> 24;
  const uint32_t v = (word ? e.p1 : e.p0) >> shift;
  clock = bits >= 32 ? v : (v & ((1u << bits) - 1u));
  return true;
}

// The base trace's deliveries and their match modes (fixed by the trace, the external filter and the clock rules)
struct WcTrace {
  std::vector<uint32_t> ev;          // per event: mode << 16 | delivery ordinal (MsgEvents only)
  std::vector<uint32_t> pos;         // per delivery: trace position
  uint32_t words = 1;
};
int32_t wc_analyse(demi_handle* h, const char* who, WcTrace& t) {
  if (h->trace_host.empty()) return fail(h, DEMI_ERR_STATE, "demi_set_trace has not been called");
  const uint32_t ext_mask = demi_ext_type_mask(h);
  std::set<uint32_t> seen;
  t.ev.assign(h->trace_host.size(), 0);
  for (uint32_t i = 0; i < h->trace_host.size(); i++) {
    const demi_event& e = h->trace_host[i];
    if (e.kind != DEMI_EV_MSG_EVENT) continue;
    if (!seen.insert(e.uniq).second) return fail(h, DEMI_ERR_INVALID, "%s: Uniq id %u names two deliveries of the trace", who, (unsigned)e.uniq);
    const uint32_t d = (uint32_t)t.pos.size();
    if (d > 0xFFFFu) return fail(h, DEMI_ERR_INVALID, "%s: more than 65536 deliveries", who);
    const uint8_t m = demi_type_is_external(ext_mask, e.type) ? WC_EXACT : incr_of(h, e.type) ? WC_CLOCK : WC_CLASS;
    t.ev[i] = ((uint32_t)m << 16) | d;
    t.pos.push_back(i);
  }
  t.words = std::max<uint32_t>(1, ((uint32_t)t.pos.size() + 63) / 64);
  return DEMI_OK;
}
int32_t wc_check_flags(demi_handle* h, const char* who, uint32_t flags) {
  if (flags & DEMI_RF_STRICT) return fail(h, DEMI_ERR_INVALID, "%s: DEMI_RF_STRICT has no wildcard form", who);
  if (flags & ~(DEMI_RF_FILTER_KNOWN_ABSENTS | DEMI_WC_LAST_ONLY)) return fail(h, DEMI_ERR_INVALID, "%s: unknown flags 0x%x", who, flags);
  return DEMI_OK;
}

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

// ---- ClockClusterizer (ClockClusterizer.scala:39-134) with ClockClusterIterator (:138-228) and OneAtATimeIterator
// (:230-290).  The trace's Uniq ids are distinct, so a set of ids is a set of deliveries: flags by delivery ordinal,
// with the ordinals in ascending id order where the Scala sorts ids.  Copyable: speculation runs a copy to the end.
typedef std::vector<uint8_t> Flags;
struct Delivery { uint32_t id; bool incr, has_clock; uint32_t clock; };
struct Clusterizer {
  const std::vector<Delivery>* d = nullptr;     // originalTrace's UniqueMsgEvents, in trace order
  std::vector<uint32_t> by_id;                  // delivery ordinals in ascending Uniq id
  // ClockClusterIterator
  Flags all_ids;                                // allIds (:139-150)
  bool first_cluster_removal = true;            // :154
  int64_t next_clock_to_remove = -1;            // :156
  Flags cblack;                                 // blacklist (:159)
  std::vector<int64_t> clocks;                  // :161
  // OneAtATimeIterator
  Flags t_all, tblack;
  std::vector<uint32_t> to_remove; size_t tr_head = 0;   // toRemove = to_remove[tr_head..]
  bool t_first = true;
  // ClockClusterizer
  Flags current_cluster, current_timers;
  bool trying_first_cluster = true;

  size_t n() const { return d->size(); }
  std::vector<int64_t> compute_remaining_clocks() const {             // :162-173
    const int64_t lowest = clocks.empty() ? 0 : clocks.front();
    std::set<int64_t> s;
    for (size_t j = 0; j < n(); j++) if (!cblack[j] && (*d)[j].has_clock) s.insert((*d)[j].clock);
    std::vector<int64_t> out;
    for (int64_t c : s) if (!(c < lowest)) out.push_back(c);           // sorted.dropWhile(c => c < lowest)
    return out;
  }
  Flags c_current() const {                                           // :176-201
    const int64_t rm = first_cluster_removal ? -1 : next_clock_to_remove;
    Flags out(n(), 0);
    for (size_t j = 0; j < n(); j++) {
      const Delivery& x = (*d)[j];
      if (x.incr) continue;                                           // handled by OneAtATimeIterator
      out[j] = !x.has_clock || !((int64_t)x.clock == rm || cblack[j]);
    }
    return out;
  }
  Flags c_next() {                                                    // :204-215
    if (first_cluster_removal) { Flags r = c_current(); first_cluster_removal = false; return r; }
    next_clock_to_remove = clocks.front();
    Flags r = c_current();
    clocks.erase(clocks.begin());
    return r;
  }
  bool c_has_next() const { return first_cluster_removal || !clocks.empty(); }
  void c_produced(const Flags& prev, const Flags& ign, bool any_ign) {   // :219-225
    for (size_t j = 0; j < n(); j++) if (all_ids[j] && !prev[j]) cblack[j] = 1;
    if (any_ign) {
      for (size_t j = 0; j < n(); j++) if (all_ids[j] && ign[j]) cblack[j] = 1;
      clocks = compute_remaining_clocks();
    }
  }
  Flags t_current() const {                                           // :254-260
    Flags out(n(), 0);
    for (size_t j = 0; j < n(); j++) out[j] = t_all[j] && !tblack[j] && (t_first || j != to_remove[tr_head]);
    return out;
  }
  Flags t_next() {                                                    // :263-273
    Flags r = t_current();
    if (t_first) t_first = false; else tr_head++;
    return r;
  }
  bool t_has_next() const { return t_first || tr_head < to_remove.size(); }
  void t_produced(const Flags& prev, const Flags& ign) {              // :279-282
    for (size_t j = 0; j < n(); j++) if (t_all[j] && (!prev[j] || ign[j])) tblack[j] = 1;
  }
  void t_reset() {                                                    // :284-287: (all -- blacklist).toSeq.sorted
    to_remove.clear(); tr_head = 0;
    for (uint32_t j : by_id) if (t_all[j] && !tblack[j]) to_remove.push_back(j);
    t_first = true;
  }

  void init(const std::vector<Delivery>& dv) {
    d = &dv;
    by_id.resize(dv.size());
    for (size_t j = 0; j < dv.size(); j++) by_id[j] = (uint32_t)j;
    std::sort(by_id.begin(), by_id.end(), [&](uint32_t a, uint32_t b) { return dv[a].id < dv[b].id; });
    all_ids.assign(dv.size(), 0); t_all.assign(dv.size(), 0); cblack.assign(dv.size(), 0); tblack.assign(dv.size(), 0);
    current_timers.assign(dv.size(), 0);
    for (size_t j = 0; j < dv.size(); j++) {
      all_ids[j] = !dv[j].incr && dv[j].has_clock;
      t_all[j] = dv[j].incr;                                          // OneAtATimeIterator.fromTrace (:231-242)
    }
    clocks = compute_remaining_clocks();                              // :174
    for (uint32_t j : by_id) if (t_all[j]) to_remove.push_back(j);   // all.toSeq.sorted: by Uniq id (:249)
    current_cluster = c_next();                                       // ClockClusterizer.scala:57
  }
  // getNextTrace (:73-134) as the include mask over the deliveries; false = None
  bool next(bool violation, const Flags& ign, bool any_ign, std::vector<uint64_t>& mask) {
    if (violation) { t_produced(current_timers, ign); c_produced(current_cluster, ign, any_ign); }
    if (!t_has_next() || (violation && !trying_first_cluster)) {      // ALL_TIMERS_FIRST_ITR
      trying_first_cluster = false;
      if (!c_has_next()) return false;
      t_reset();
      current_cluster = c_next();
    }
    current_timers = t_next();
    mask.assign(std::max<size_t>(1, (n() + 63) / 64), 0);
    for (size_t j = 0; j < n(); j++)
      if (current_timers[j] || current_cluster[j]) mask[j >> 6] |= 1ull << (j & 63);
    return true;
  }
};
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
  WcTrace t;
  if ((rc = wc_analyse(h, "demi_wildcard_minimize", t)) != DEMI_OK) return rc;
  memset(out, 0, sizeof(*out));
  const std::vector<demi_event> base = h->trace_host;
  const std::vector<demi_ext_event> ext = h->trace_ext_host;
  std::vector<Delivery> dv(t.pos.size());
  for (size_t j = 0; j < t.pos.size(); j++) {
    const demi_event& e = base[t.pos[j]];
    dv[j].id = e.uniq; dv[j].incr = incr_of(h, e.type);
    dv[j].has_clock = clock_of(h, e, dv[j].clock);
  }
  auto count_msg_events = [](const std::vector<demi_event>& v) {     // RunnerUtils.countMsgEvents
    uint32_t n = 0; for (const demi_event& e : v) n += e.kind == DEMI_EV_MSG_EVENT; return n;
  };
  Clusterizer cz;
  cz.init(dv);
  const Flags none(dv.size(), 0);
  std::vector<demi_event> min_trace = base, rec(65536);
  std::vector<uint32_t> sizes, ign_pos(t.pos.size() + 1);
  const size_t wide_cap = 8192;                                      // tests per launch (host memory for masks only)
  std::vector<uint64_t> cur;
  bool has = cz.next(false, none, false, cur);                       // doMinimize :193; record_prune_start :195
  while (has) {
    std::vector<std::vector<uint64_t>> cand{cur};
    {
      Clusterizer spec = cz;
      std::vector<uint64_t> m;
      while (cand.size() < wide_cap && spec.next(false, none, false, m)) cand.push_back(m);
    }
    std::vector<uint64_t> flat(cand.size() * t.words);
    for (size_t c = 0; c < cand.size(); c++) std::copy(cand[c].begin(), cand[c].end(), flat.begin() + c * t.words);
    std::vector<demi_replay_result> res(cand.size());
    if ((rc = wc_launch(h, t, flat.data(), (uint32_t)cand.size(), looking_for, flags, res.data(),
                        nullptr, 0, nullptr, nullptr, 0, nullptr)) != DEMI_OK) return rc;
    out->replays_executed += (uint32_t)cand.size();
    out->batches++;
    for (size_t c = 0; c < cand.size(); c++) {
      if (c > 0 && (!cz.next(false, none, false, cur) || cur != cand[c]))
        return fail(h, DEMI_ERR_STATE, "demi_wildcard_minimize: speculation diverged from the clusterizer");
      if (res[c].status) return fail(h, DEMI_ERR_CAPACITY, "demi_wildcard_minimize: a replay reported status %u", (unsigned)res[c].status);
      out->total_replays++;                                           // stats.increment_replays
      sizes.push_back(count_msg_events(min_trace));                   // record_internal_size(countMsgEvents(minTrace)) :210-212
      if (!res[c].violation) {
        if (c + 1 == cand.size()) has = cz.next(false, none, false, cur);
        continue;
      }
      uint32_t n_rec = 0, n_ign = 0; demi_replay_result r1;
      if ((rc = wc_launch(h, t, cand[c].data(), 1, looking_for, flags, &r1, rec.data(), (uint32_t)rec.size(), &n_rec,
                          ign_pos.data(), (uint32_t)ign_pos.size(), &n_ign)) != DEMI_OK) return rc;
      if (r1.status || !r1.violation) return fail(h, DEMI_ERR_STATE, "demi_wildcard_minimize: recorded re-run disagrees with the batch");
      if (n_rec <= min_trace.size()) min_trace.assign(rec.begin(), rec.begin() + n_rec);   // :217-219
      Flags ign(dv.size(), 0);                                        // ignoredAbsentIds (:214-236), as deliveries
      for (uint32_t k = 0; k < n_ign; k++) ign[t.ev[ign_pos[k]] & 0xFFFFu] = 1;
      has = cz.next(true, ign, n_ign > 0, cur);
      break;
    }
  }
  sizes.push_back(count_msg_events(min_trace));                       // record_prune_end; fencepost :180-185
  if ((rc = demi_set_trace(h, min_trace.data(), (uint32_t)min_trace.size(), ext.data(), (uint32_t)ext.size())) != DEMI_OK) return rc;
  out->n_events = (uint32_t)min_trace.size();
  out->deliveries_before = count_msg_events(base);
  out->deliveries_after = count_msg_events(min_trace);
  out->n_internal_sizes = (uint32_t)sizes.size();
  out->unignorable = 0;
  if (out_trace) std::copy(min_trace.begin(), min_trace.begin() + std::min<size_t>(min_trace.size(), cap_events), out_trace);
  if (internal_sizes) for (uint32_t i = 0; i < cap_sizes && i < sizes.size(); i++) internal_sizes[i] = sizes[i];
  return DEMI_OK;
}
