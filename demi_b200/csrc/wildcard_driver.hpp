// wildcard_driver.hpp — WildcardMinimizer (minification/wildcard_minimization/WildcardMinimizer.scala:133-241) with
// testScheduler = STSSched, ClockClusterizer (ClockClusterizer.scala:39-228) and OneAtATimeIterator (:230-290),
// Aggressiveness.ALL_TIMERS_FIRST_ITR, as a step-wise driver that does not replay anything itself.
//
// Every test the clusterizer issues is one STSScheduler.test of the SAME base trace (ClockClusterizer keeps
// `originalTrace`), described by which of its deliveries are included; the next test depends on earlier outcomes only
// through the clusterizer's blacklists.  So the tests a copy of the clusterizer would issue if every test failed are
// independent.  A round of the driver is:
//   candidates()   those include masks (at most WIDE_CAP), empty when the minimization is over;
//   commit(res)    their replays, walked in order up to the first success, whose recorded re-run is needed (RECORD);
//                  DONE when none succeeded (candidates() then says whether more remain);
//   advance(...)   the recorded re-run of that success and the trace positions of the deliveries it ignored: the
//                  recording replaces minTrace when it is no longer, and the real clusterizer takes the outcome.
// The caller decides how replays are run (one trace on the handle, or many traces in shared launches); the decisions,
// counters and the final trace are the sequential ones either way.  Host-only.
#pragma once
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <set>
#include <string>
#include <vector>
#include "../../include/demi_b200.h"
#include "../../include/demi_limits.h"
#include "replay_trace.hpp"

namespace demi {

// The base trace's deliveries and their match modes (fixed by the trace, the external filter and the clock rules)
struct WcTrace {
  std::vector<uint32_t> ev;          // per event: mode << 16 | delivery ordinal (MsgEvents only)
  std::vector<uint32_t> pos;         // per delivery: trace position
  uint32_t words = 1;                // include-mask words: ceil(deliveries / 64), at least 1

  static bool incr_of(const uint32_t* incr, uint32_t type) { return (incr[type >> 5] >> (type & 31)) & 1u; }
  // trace[0, n) under the external type mask and the causesClockIncrement set; false (with msg) when a Uniq id names
  // two deliveries or there are more than 65536 of them
  bool build(const demi_event* trace, uint32_t n, uint32_t ext_mask, const uint32_t* incr, const char* who, std::string& msg) {
    std::set<uint32_t> seen;
    ev.assign(n, 0); pos.clear();
    char buf[160];
    for (uint32_t i = 0; i < n; i++) {
      const demi_event& e = trace[i];
      if (e.kind != DEMI_EV_MSG_EVENT) continue;
      if (!seen.insert(e.uniq).second) {
        snprintf(buf, sizeof(buf), "%s: Uniq id %u names two deliveries of the trace", who, (unsigned)e.uniq);
        msg = buf; return false;
      }
      const uint32_t d = (uint32_t)pos.size();
      if (d > 0xFFFFu) { snprintf(buf, sizeof(buf), "%s: more than 65536 deliveries", who); msg = buf; return false; }
      const uint32_t m = demi_type_is_external(ext_mask, e.type) ? WC_EXACT : incr_of(incr, e.type) ? WC_CLOCK : WC_CLASS;
      ev[i] = (m << 16) | d;
      pos.push_back(i);
    }
    words = std::max<uint32_t>(1, ((uint32_t)pos.size() + 63) / 64);
    return true;
  }
};

struct WildcardDriver {
  typedef std::vector<uint8_t> Flags;
  struct Delivery { uint32_t id; bool incr, has_clock; uint32_t clock; };

  // ---- ClockClusterizer (ClockClusterizer.scala:39-134) with ClockClusterIterator (:138-228) and OneAtATimeIterator
  // (:230-290).  The trace's Uniq ids are distinct, so a set of ids is a set of deliveries: flags by delivery ordinal,
  // with the ordinals in ascending id order where the Scala sorts ids.  Copyable: speculation runs a copy to the end.
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

  enum Step { DONE, RECORD, FAILED };
  static constexpr size_t WIDE_CAP = 8192;   // candidates per round (host memory for masks only)

  WildcardDriver() = default;
  WildcardDriver(const WildcardDriver&) = delete;          // the clusterizer points at `dv`
  WildcardDriver& operator=(const WildcardDriver&) = delete;

  WcTrace t;                               // the base trace's deliveries and match modes
  std::vector<demi_event> base, min_trace; // originalTrace; minTrace
  std::vector<uint64_t> cand;              // the current round's candidates, t.words words each
  std::vector<uint32_t> sizes;             // record_internal_size
  demi_intmin_out* out = nullptr;
  int32_t error = DEMI_OK;                 // FAILED: the code and message the single-trace call returns
  std::string msg;

  size_t n_candidates() const { return cand.size() / t.words; }

  // the verified MCS trace trace[0, n) (copied) under the external type mask and the clock rules (clock_rule: 256
  // packed rules by type, 0 = no clock; incr: the 256-bit causesClockIncrement set).  false (error DEMI_ERR_INVALID,
  // `o` untouched) when the trace cannot be wildcarded; else `o` is zeroed here and filled as the run goes.
  bool init(const demi_event* trace, uint32_t n, uint32_t ext_mask, const uint32_t* clock_rule, const uint32_t* incr,
            demi_intmin_out* o) {
    WcTrace built;
    if (!built.build(trace, n, ext_mask, incr, "demi_wildcard_minimize", msg)) { error = DEMI_ERR_INVALID; return false; }
    init(std::move(built), trace, n, clock_rule, incr, o);
    return true;
  }
  // the same, with the trace's deliveries and modes already built (WcTrace::build under the same mask and set)
  void init(WcTrace&& built, const demi_event* trace, uint32_t n, const uint32_t* clock_rule, const uint32_t* incr,
            demi_intmin_out* o) {
    t = std::move(built);
    out = o;
    memset(out, 0, sizeof(*out));
    base.assign(trace, trace + n);
    min_trace = base;
    dv.resize(t.pos.size());
    for (size_t j = 0; j < t.pos.size(); j++) {
      const demi_event& e = base[t.pos[j]];
      dv[j].id = e.uniq; dv[j].incr = WcTrace::incr_of(incr, e.type);
      dv[j].has_clock = clock_of(clock_rule, e, dv[j].clock);
    }
    last_size = count_msg_events(base);
    out->deliveries_before = last_size;
    cz.init(dv);
    has = cz.next(false, Flags(dv.size(), 0), false, cur);              // doMinimize :193; record_prune_start :195
  }

  // The include masks the clusterizer would issue from here if every test failed: the next one, then a copy's
  const std::vector<uint64_t>& candidates() {
    cand.clear();
    if (!has) return cand;
    cand = cur;
    Clusterizer spec = cz;
    const Flags none(dv.size(), 0);
    std::vector<uint64_t> m;
    while (n_candidates() < WIDE_CAP && spec.next(false, none, false, m)) cand.insert(cand.end(), m.begin(), m.end());
    return cand;
  }

  // res[c] is the replay of candidate c.  RECORD: *mask (t.words words, valid until the next candidates()) is the
  // test whose recorded re-run advance() takes next.
  Step commit(const demi_replay_result* res, const uint64_t** mask) {
    const size_t n = n_candidates();
    out->replays_executed += (uint32_t)n;
    out->batches++;
    const Flags none(dv.size(), 0);
    for (size_t c = 0; c < n; c++) {
      const uint64_t* m = cand.data() + c * t.words;
      if (c > 0 && (!cz.next(false, none, false, cur) || !std::equal(cur.begin(), cur.end(), m)))
        return failed(DEMI_ERR_STATE, "demi_wildcard_minimize: speculation diverged from the clusterizer");
      if (res[c].status) return failed(DEMI_ERR_CAPACITY, "demi_wildcard_minimize: a replay reported status %u", (unsigned)res[c].status);
      out->total_replays++;                                             // stats.increment_replays
      sizes.push_back(last_size);                                       // record_internal_size(countMsgEvents(minTrace)) :210-212
      if (!res[c].violation) {
        if (c + 1 == n) has = cz.next(false, none, false, cur);
        continue;
      }
      *mask = m;
      return RECORD;
    }
    return DONE;
  }

  // r, rec[0, n_rec) and ign_pos[0, n_ign): the recorded re-run of the test commit() returned and the trace positions
  // of the deliveries it ignored.  false (FAILED) when the re-run does not reproduce what the batch found.
  bool advance(const demi_replay_result& r, const demi_event* rec, uint32_t n_rec, const uint32_t* ign_pos, uint32_t n_ign) {
    if (r.status || !r.violation) { failed(DEMI_ERR_STATE, "demi_wildcard_minimize: recorded re-run disagrees with the batch"); return false; }
    if (n_rec <= min_trace.size()) {                                    // :217-219
      min_trace.assign(rec, rec + n_rec);
      last_size = count_msg_events(min_trace);
    }
    Flags ign(dv.size(), 0);                                            // ignoredAbsentIds (:214-236), as deliveries
    for (uint32_t k = 0; k < n_ign; k++) ign[t.ev[ign_pos[k]] & 0xFFFFu] = 1;
    has = cz.next(true, ign, n_ign > 0, cur);
    return true;
  }

  // the outputs of a finished run: the minimized trace (at most cap_events of it) and the sizes (at most cap_sizes),
  // with the final fencepost (record_prune_end, :180-185)
  void finish(demi_event* out_trace, uint32_t cap_events, uint32_t* internal_sizes, uint32_t cap_sizes) {
    sizes.push_back(last_size);
    out->n_events = (uint32_t)min_trace.size();
    out->deliveries_after = last_size;
    out->n_internal_sizes = (uint32_t)sizes.size();
    out->unignorable = 0;
    if (out_trace) std::copy(min_trace.begin(), min_trace.begin() + std::min<size_t>(min_trace.size(), cap_events), out_trace);
    if (internal_sizes) for (uint32_t i = 0; i < cap_sizes && i < sizes.size(); i++) internal_sizes[i] = sizes[i];
  }

  // FingerprintFactory.getLogicalClock as data: false = None
  static bool clock_of(const uint32_t* clock_rule, const demi_event& e, uint32_t& clock) {
    const uint32_t r = clock_rule[e.type];
    if (!r) return false;
    const uint32_t word = (r >> 8) & 0xFF, shift = (r >> 16) & 0xFF, bits = r >> 24;
    const uint32_t v = (word ? e.p1 : e.p0) >> shift;
    clock = bits >= 32 ? v : (v & ((1u << bits) - 1u));
    return true;
  }

 private:
  std::vector<Delivery> dv;
  Clusterizer cz;
  std::vector<uint64_t> cur;               // the clusterizer's next test
  bool has = false;                        // ... when there is one
  uint32_t last_size = 0;                  // countMsgEvents(minTrace)

  static uint32_t count_msg_events(const std::vector<demi_event>& v) {   // RunnerUtils.countMsgEvents
    uint32_t n = 0; for (const demi_event& e : v) n += e.kind == DEMI_EV_MSG_EVENT; return n;
  }
  Step failed(int32_t code, const char* fmt, ...) __attribute__((format(printf, 3, 4))) {
    char buf[256];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    error = code; msg = buf;
    return FAILED;
  }
};

}  // namespace demi
