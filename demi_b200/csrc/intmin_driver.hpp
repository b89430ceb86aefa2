// intmin_driver.hpp — STSSchedMinimizer (minification/internal_minimization/ScheduleCheckers.scala:19-107) with the
// LeftToRightOneAtATime (OneAtATimeRemoval.scala:17-137) or SrcDstFIFORemoval (:139-251) removal strategy, as a
// step-wise driver that does not replay anything itself.
//
// The reference tries ONE delivery at a time: drop it from the last failing trace, ask STSSched whether the violation
// still shows, and on success continue from the trace STSSched recorded.  While removals keep failing, the candidates
// all refer to the same base trace, so they are independent.  A round of the driver is:
//   candidates()   the remaining candidate list of the current base trace, as getNextTrace would produce it if every
//                  test failed; empty when the minimization is over;
//   commit(res)    the replays of those candidates, walked in the strategy's order up to the first success: that
//                  candidate is the delivery to drop, and its recorded re-run is needed; no success ends the run;
//   advance(rec)   the recorded re-run of that removal: it becomes the new base trace, and what it lost is pruned.
// The caller decides how replays are run (one trace on the handle, or many traces in shared launches); the decisions,
// counters and the final trace are the sequential ones either way.  Host-only.
#pragma once
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <tuple>
#include <vector>
#include "../../include/demi_b200.h"
#include "../../include/demi_limits.h"

namespace demi {

struct IntMinDriver {
  typedef std::tuple<uint32_t, uint32_t, uint32_t, uint32_t, uint32_t> Key;   // (snd, rcv, type, p0, p1) == (snd, rcv, fingerprint)
  typedef std::map<Key, uint32_t> MultiSet;
  static Key key_of(const demi_event& e) { return Key(e.src, e.dst, e.type, e.p0, e.p1); }
  static uint32_t count_of(const MultiSet& m, const Key& k) { auto it = m.find(k); return it == m.end() ? 0u : it->second; }

  // RemovalStrategy state.  Copyable: the candidates the strategy would produce if every test failed are obtained
  // from a copy, the real object then replays the same calls as results are committed.
  struct Strategy {
    typedef std::tuple<uint32_t, uint32_t, uint32_t> Fp;               // (type, p0, p1)
    bool fifo = false;
    MultiSet tried;                                                    // triedIgnoring (:20)
    std::map<std::pair<uint32_t, uint32_t>, std::vector<Fp>> src_dst;  // srcDstToMessages (:150)
    std::map<std::pair<uint32_t, uint32_t>, int> cur_idx;              // srcDstToCurrentIdx (:168)
    bool have_prev = false; std::pair<uint32_t, uint32_t> prev;        // previouslyChosenSrcDst (:162)
    const std::vector<demi_event>* verified = nullptr;

    void init_fifo(const std::vector<demi_event>& v) {                 // :152-159
      fifo = true; verified = &v;
      for (const demi_event& e : v)
        if (e.kind == DEMI_EV_MSG_EVENT && e.src < DEMI_MAX_ACTORS) src_dst[{e.src, e.dst}].push_back(Fp(e.type, e.p0, e.p1));
    }
    bool choice(const demi_event& e) {                                 // choiceFilter :178-203 (LeftToRight: true, :131-137)
      if (!fifo) return true;
      if (e.src < DEMI_MAX_ACTORS) {
        auto it = src_dst.find({e.src, e.dst});
        if (it != src_dst.end()) {
          int idx = ++cur_idx[{e.src, e.dst}];
          if (idx == (int)it->second.size() - 1) {
            it->second.pop_back();
            if (it->second.empty()) src_dst.erase(it);
            have_prev = true; prev = {e.src, e.dst};
            return true;
          }
        }
      }
      have_prev = false;
      return e.src >= DEMI_MAX_ACTORS;                                 // "deadLetters": a timer
    }
    // getNextTrace (:57-124; SrcDstFIFORemoval's prologue :209-249): index of the delivery to drop, or -1
    int next(const std::vector<demi_event>& trace, const MultiSet& pruned, bool triggered) {
      if (fifo) {
        if (!triggered && have_prev) src_dst.erase(prev);              // "this src,dst is done"
        if (triggered) {
          src_dst.clear();
          MultiSet copy = pruned;
          for (size_t i = verified->size(); i-- > 0;) {
            const demi_event& e = (*verified)[i];
            if (e.kind != DEMI_EV_MSG_EVENT || e.src >= DEMI_MAX_ACTORS) continue;
            auto it = copy.find(key_of(e));
            if (it != copy.end() && it->second) { it->second--; continue; }
            auto& vec = src_dst[{e.src, e.dst}];
            vec.insert(vec.begin(), Fp(e.type, e.p0, e.p1));
          }
        }
        cur_idx.clear();
        for (auto& kv : src_dst) cur_idx[kv.first] = -1;
      }
      MultiSet keys = pruned;                                          // keysThisIteration ++= alreadyRemoved
      for (uint32_t i = 0; i < trace.size(); i++) {
        if (trace[i].kind != DEMI_EV_MSG_EVENT) continue;
        const Key k = key_of(trace[i]);
        const uint32_t c = ++keys[k];
        if (c > count_of(tried, k) && choice(trace[i])) { tried[k]++; return (int)i; }
      }
      return -1;
    }
  };

  // what commit() found
  enum Step { DONE, RECORD, FAILED };

  IntMinDriver() = default;
  IntMinDriver(const IntMinDriver&) = delete;              // the strategy points at `verified`
  IntMinDriver& operator=(const IntMinDriver&) = delete;

  std::vector<demi_event> verified, cur;   // the verified MCS trace; lastFailingTrace
  std::vector<uint32_t> cand;              // the current round's candidate list (trace positions to skip)
  std::vector<uint32_t> sizes;             // record_internal_size
  demi_intmin_out* out = nullptr;
  int32_t error = DEMI_OK;                 // FAILED: the code and message the single-trace call returns
  std::string msg;

  // the verified MCS trace trace[0, n) (copied); `out` is zeroed here and filled as the run goes
  void init(const demi_event* trace, uint32_t n, uint32_t ext_type_mask, bool fifo, demi_intmin_out* o) {
    out = o;
    memset(out, 0, sizeof(*out));
    verified.assign(trace, trace + n);
    cur = verified;
    if (fifo) strat.init_fifo(verified);
    // OneAtATimeStrategy.init (:27-48): external deliveries are never ignored
    for (const demi_event& e : cur)
      if (e.kind == DEMI_EV_MSG_EVENT && demi_type_is_external(ext_type_mask, e.type)) strat.tried[key_of(e)]++;
    for (auto& kv : strat.tried) out->unignorable += kv.second;
    last_size = 0;
    for (const demi_event& e : cur) last_size += e.kind == DEMI_EV_MSG_EVENT;
    out->deliveries_before = last_size;
  }

  // The candidate list getNextTrace would produce on the current base trace if every test failed (:57-124)
  const std::vector<uint32_t>& candidates() {
    cand.clear();
    Strategy spec = strat;
    bool t = triggered;
    for (;;) {
      const int found = spec.next(cur, pruned, t);
      if (found < 0) break;
      cand.push_back((uint32_t)found);
      t = false;
    }
    return cand;
  }

  // res[c] is the replay of cand[c].  RECORD: *skip is the delivery whose removal reproduced the violation, and
  // advance() takes its recorded re-run next.  DONE: every remaining candidate was tried and failed.
  Step commit(const demi_replay_result* res, uint32_t* skip) {
    out->replays_executed += (uint32_t)cand.size();
    out->batches++;
    for (size_t c = 0; c < cand.size(); c++) {
      if (res[c].status) return failed(DEMI_ERR_CAPACITY, "demi_internal_minimize: a replay reported status %u", (unsigned)res[c].status);
      out->total_replays++;                                           // stats.increment_replays
      const int chosen = strat.next(cur, pruned, triggered);          // the real strategy takes the same step
      if (chosen != (int)cand[c]) return failed(DEMI_ERR_STATE, "demi_internal_minimize: speculation diverged from the strategy");
      triggered = res[c].violation != 0;
      if (!res[c].violation) { sizes.push_back(last_size); continue; }   // "Ignoring didn't work."
      *skip = cand[c];
      return RECORD;
    }
    return DONE;
  }

  // r and rec[0, n_rec): the recorded re-run of the removal commit() returned.  On success the trace STSSched recorded
  // becomes lastFailingTrace (:57-91); false (FAILED) when the re-run does not reproduce what the batch found.
  bool advance(const demi_replay_result& r, const demi_event* rec, uint32_t n_rec) {
    if (r.status || !r.violation) { failed(DEMI_ERR_STATE, "demi_internal_minimize: recorded re-run disagrees with the batch"); return false; }
    MultiSet prior, fresh;
    for (const demi_event& e : cur) if (e.kind == DEMI_EV_MSG_EVENT) prior[key_of(e)]++;
    uint32_t new_size = 0;
    for (uint32_t i = 0; i < n_rec; i++) if (rec[i].kind == DEMI_EV_MSG_EVENT) { fresh[key_of(rec[i])]++; new_size++; }
    for (auto& kv : prior) {                                          // MultiSet.setDifference (schedulers/Util.scala:93-106)
      const uint32_t c2 = count_of(fresh, kv.first);
      if (kv.second > c2) pruned[kv.first] += kv.second - c2;
    }
    cur.assign(rec, rec + n_rec);
    last_size = new_size;
    sizes.push_back(last_size);
    return true;
  }

  // the outputs of a finished run: the minimized trace (at most cap_events of it) and the sizes (at most cap_sizes)
  void finish(demi_event* out_trace, uint32_t cap_events, uint32_t* internal_sizes, uint32_t cap_sizes) {
    out->n_events = (uint32_t)cur.size();
    out->deliveries_after = last_size;
    out->n_internal_sizes = (uint32_t)sizes.size();
    if (out_trace) std::copy(cur.begin(), cur.begin() + std::min<size_t>(cur.size(), cap_events), out_trace);
    if (internal_sizes) for (uint32_t i = 0; i < cap_sizes && i < sizes.size(); i++) internal_sizes[i] = sizes[i];
  }

 private:
  Strategy strat;
  MultiSet pruned;
  bool triggered = false;                  // violationTriggered (ScheduleCheckers.scala:48)
  uint32_t last_size = 0;

  Step failed(int32_t code, const char* fmt, ...) __attribute__((format(printf, 3, 4))) {
    char buf[256];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    error = code; msg = buf;
    return FAILED;
  }
};

}  // namespace demi
