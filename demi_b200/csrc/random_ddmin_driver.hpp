// random_ddmin_driver.hpp — RunnerUtils.randomDDMin (RunnerUtils.scala:601-623) as a DDMin driver (ddmin_driver.hpp)
// that runs no test itself: DDMin over the whole program with RandomScheduler.test as the TestOracle, then verify_mcs.
//
// A test of mask m is N executions of m's subsequence; its record (demi_random_test_result) is a function of the
// subsequence, N and the parameters alone, so a speculative batch may hold tests the sequential walk never consumes.
// The caller supplies run_tests(): one launch sequence on the handle (demi_random_ddmin), many traces' tests in shared
// launches (demi_random_ddmin_many), or the CPU oracle (the host tests).  Host-only.
#pragma once
#include <map>
#include <vector>
#include "ddmin_driver.hpp"

namespace demi {

struct RandomDDMinDriver : DDMinDriver {
  std::map<Mask, demi_random_test_result> records;
  std::vector<uint32_t> consumed_runs;      // executions_run of each test the sequential walk consumed, in order
  uint64_t executions_executed = 0;

  // n tests: res[k] is the record of masks[k] (mw words each); *executed = the executions of those tests that ran
  virtual int32_t run_tests(const uint64_t* masks, size_t n, demi_random_test_result* res, uint64_t* executed) = 0;

  int32_t evaluate(const uint64_t* masks, size_t n, signed char* out) override {
    std::vector<demi_random_test_result> res(n);
    uint64_t executed = 0;
    int32_t rc = run_tests(masks, n, res.data(), &executed);
    if (rc != DEMI_OK) return rc;
    executions_executed += executed;
    for (size_t i = 0; i < n; i++) {
      records[Mask(masks + i * mw, masks + (i + 1) * mw)] = res[i];
      out[i] = res[i].status == 0 && res[i].first_hit >= 0;
    }
    return DEMI_OK;
  }
  // a test's status fails the call only here, where the sequential walk uses its result
  void consumed(const Mask& m) override {
    const demi_random_test_result& r = records.at(m);
    if (r.status) { error = fail(h, DEMI_ERR_CAPACITY, "demi_random_ddmin: a test execution reported status %u", (unsigned)r.status); return; }
    consumed_runs.push_back(r.executions_run);
  }

  // Tests per speculative batch, sized by executions per launch: about 2^20 executions (a few milliseconds of the lane
  // engine on raft5-sized programs, so the launch latency is amortised), and never more than the 6000 tests of the
  // replay path (beyond that the host's batch building costs more than the launch).  DEMI_DDMIN_WIDE overrides it.
  void set_width(uint64_t n_prefixes) {
    wide_cap = std::max<size_t>(16, std::min<size_t>(6000, ((size_t)1 << 20) / n_prefixes));
    if (getenv("DEMI_DDMIN_WIDE")) wide_cap = (size_t)atol(getenv("DEMI_DDMIN_WIDE"));
  }

  // DDMin.minimize over the n_ext externals at `ext` (mw, looking_for and h set by the caller), then verify_mcs.  On
  // DEMI_OK, mcs_mask (mw words), iteration_sizes / iteration_keys (at most cap entries) and out are filled.
  int32_t minimize(bool check_unmodified, uint64_t* mcs_mask, uint32_t* iteration_sizes, uint64_t* iteration_keys, uint32_t cap,
                   demi_random_ddmin_out* out) {
    memset(out, 0, sizeof(*out));
    // DDMin.minimize's dag is the whole program, WaitQuiescence included (UnmodifiedEventDag, Minimizer.scala:15-20)
    Mask dag(mw, 0), zero(mw, 0);
    for (uint32_t i = 0; i < n_ext; i++) setbit(dag, i);
    if (check_unmodified) {                                                 // DeltaDebugging.scala:41-47
      bool v = test(dag, dag, zero);
      if (error != DEMI_OK) return error;
      if (!v) return fail(h, DEMI_ERR_INVALID, "Unmodified trace does not trigger violation");
      consumed_runs.clear();                                                // _stats.reset() (:48)
    }
    original_num_events = n_ext;
    Mask mcs = ddmin2(dag, zero);
    if (error != DEMI_OK) return error;
    DDMinDriver::iteration_sizes.push_back(original_num_events - total_inputs_pruned);     // fencepost :60
    if (original_num_events - total_inputs_pruned != popcount(mcs))
      return fail(h, DEMI_ERR_STATE, "demi_random_ddmin: bookkeeping assertion failed (DeltaDebugging.scala:58)");
    const uint32_t tests = (uint32_t)consumed_runs.size();
    std::vector<uint64_t> keys;
    uint64_t total = 0;
    for (uint32_t r : consumed_runs) { total += r; keys.push_back(total); }
    keys.push_back(total);                                                  // the fencepost's key
    out->mcs_size = popcount(mcs);
    bool verified = true;                                                   // nothing pruned: the original trace stands
    out->mcs_first_hit = -1;
    if (out->mcs_size < n_ext) {                                            // verify_mcs (RunnerUtils.scala:612-620)
      // the MCS's own test alone: taken from the tests already run, else evaluated by itself (no speculation below it)
      auto it = records.find(mcs);
      if (it == records.end()) {
        signed char v;
        int32_t rc = evaluate(mcs.data(), 1, &v);
        if (rc != DEMI_OK) return rc;
        replays_executed++;
        it = records.find(mcs);
      }
      const demi_random_test_result& r = it->second;
      if (r.status) return fail(h, DEMI_ERR_CAPACITY, "demi_random_ddmin: the MCS's test reported status %u", (unsigned)r.status);
      verified = r.first_hit >= 0;
      out->mcs_first_hit = r.first_hit;
    }
    std::copy(mcs.begin(), mcs.end(), mcs_mask);
    out->tests = tests;
    out->total_replays = total;
    out->n_iterations = (uint32_t)DDMinDriver::iteration_sizes.size();
    out->executions_executed = executions_executed;
    out->tests_evaluated = replays_executed;
    out->batches = batches;
    out->verified = verified ? 1u : 0u;
    for (uint32_t i = 0; i < cap && i < out->n_iterations; i++) {
      if (iteration_sizes) iteration_sizes[i] = DDMinDriver::iteration_sizes[i];
      if (iteration_keys) iteration_keys[i] = keys[i];
    }
    return DEMI_OK;
  }
};

}  // namespace demi
