// incddmin_driver.hpp — IncrementalDDMin(ResumableDPOR) (minification/IncrementalDeltaDebugging.scala:20-122) as a
// DDMin driver (ddmin_driver.hpp) that does not run any DPOR search itself.
//
// ResumableDPOR keeps one DPORwHeuristics instance per external subsequence (subseqToDPOR).  Here that state is
// `history`: the caps each subsequence's instance has been tested with by the SEQUENTIAL walk.  A test of mask m under
// the current cap is the outcome of a fresh instance put through history[m] ++ [cap]; evaluating it does not touch any
// state, so the speculative batch may contain tests the walk never asks for, and the driver's speculation depends only
// on its own memo.  The caller supplies run_dpor(): one launch on the handle (demi_incremental_ddmin), many traces'
// instances in shared launches (demi_incremental_ddmin_many), or the CPU oracle (the host tests).  Host-only.
#pragma once
#include <map>
#include <vector>
#include "ddmin_driver.hpp"

namespace demi {

struct IncDDMinDriver : DDMinDriver {
  int32_t cap = 0;
  std::map<Mask, std::vector<int32_t>> history;
  uint64_t interleavings = 0;

  // n DPOR instances: instance k runs the externals masks[k] selects (mw words each) and is put through the caps
  // caps[cap_off[k] .. cap_off[k+1]) in order, one DPORwHeuristics.test each; res[k] is its record, accumulated over
  // its tests as demi_dpor_batch_ex accumulates it.
  virtual int32_t run_dpor(const uint64_t* masks, size_t n, const std::vector<int32_t>& caps,
                           const std::vector<uint32_t>& cap_off, demi_dpor_result* res) = 0;

  // the externals mask k selects, appended to `flat`, with their end offset in `off`
  void select(const uint64_t* masks, size_t n, std::vector<demi_ext_event>& flat, std::vector<uint32_t>& off) const {
    for (size_t k = 0; k < n; k++) {
      const uint64_t* m = masks + k * mw;
      for (uint32_t i = 0; i < n_ext; i++) if ((m[i >> 6] >> (i & 63)) & 1ull) flat.push_back(ext[i]);
      off.push_back((uint32_t)flat.size());
    }
  }

  int32_t evaluate(const uint64_t* masks, size_t n, signed char* out) override {
    std::vector<uint32_t> coff(1, 0);
    std::vector<int32_t> caps;
    for (size_t k = 0; k < n; k++) {
      const uint64_t* m = masks + k * mw;
      auto it = history.find(Mask(m, m + mw));
      if (it != history.end()) caps.insert(caps.end(), it->second.begin(), it->second.end());
      caps.push_back(cap);
      coff.push_back((uint32_t)caps.size());
    }
    std::vector<demi_dpor_result> res(n);
    const int32_t rc = run_dpor(masks, n, caps, coff, res.data());
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

  // IncrementalDDMin.minimize (:49-77) over every external: the distance cap doubles 0, 2, 4, ... while it is below
  // max_max_distance and the MCS is larger than stop_at_size.  On DEMI_OK, mcs_mask (mw words) and out are filled.
  int32_t minimize(int32_t max_max_distance, uint32_t stop_at_size, uint64_t* mcs_mask, demi_incddmin_out* out) {
    memset(out, 0, sizeof(*out));
    Mask cur(mw, 0), zero(mw, 0);
    for (uint32_t i = 0; i < n_ext; i++) setbit(cur, i);
    int32_t dist = 0;                                                              // oracle.setMaxDistance(currentDistance) :53
    while (dist < max_max_distance && popcount(cur) > stop_at_size) {              // :66
      cap = dist;
      memo.clear();                                                                // ddmin = new DDMin(oracle, checkUnmodifed=false) :68
      original_num_events = popcount(cur); total_inputs_pruned = 0;
      cur = ddmin2(cur, zero);
      if (error != DEMI_OK) return error;
      out->rounds++;
      dist = dist == 0 ? 2 : dist << 1;                                            // :72
    }
    std::copy(cur.begin(), cur.end(), mcs_mask);
    out->mcs_size = popcount(cur);
    out->total_replays = total_replays;                                            // mergeStats :33-41
    out->instances = (uint32_t)history.size();
    out->tests_executed = replays_executed;
    out->batches = batches;
    out->interleavings_executed = interleavings;
    return DEMI_OK;
  }
};

}  // namespace demi
