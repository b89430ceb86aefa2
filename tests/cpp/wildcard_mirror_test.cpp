// C++ host mirror (include/demi_b200.hpp) of the fungible-clock stage: fuzz -> DDMin -> internal minimization ->
// WildcardMinimizer (BackTrackStrategy and LastOnlyStrategy) -> strict replay of the result.  Without a CUDA device:
// the arguments outside the accelerated path are refused first, then the no-fallback contract.
#include <cstdio>
#include "demi_b200.hpp"

using namespace demi;

#define CHECK(c) do { if (!(c)) { std::printf("CHECK failed: %s (line %d)\n", #c, __LINE__); return 1; } } while (0)

int main() {
  SchedulerConfig cfg;
  cfg.model = DEMI_MODEL_RAFT5;
  cfg.model_flags = 1;
  ExternalEvents prog;
  for (int a = 0; a < 5; a++) prog.push_back(Start((uint8_t)a));
  for (int a = 0; a < 5; a++) prog.push_back(Send((uint8_t)a, 1, 0x1F));
  for (int k = 0; k < 6; k++) prog.push_back(Send((uint8_t)(k % 5), 2, 1 + k));
  prog.push_back(WaitQuiescence());
  bool threw = false;
  try { WildcardMinimizer(cfg, prog, EventTrace(), 1, raft5_clock_rules(), BackTrackStrategy(), TestScheduler::DPORwHeuristics); }
  catch (const std::invalid_argument&) { threw = true; }
  CHECK(threw);
  threw = false;
  try { WildcardMinimizer(cfg, prog, EventTrace(), 1, raft5_clock_rules(), BackTrackStrategy(), TestScheduler::STSSched,
                          ClusteringStrategy::ClockClusterizer, /*skipClockClusters=*/true); }
  catch (const std::invalid_argument&) { threw = true; }
  CHECK(threw);
  if (demi_device_count() == 0) {
    try { WildcardMinimizer w(cfg, prog, EventTrace(), 1, raft5_clock_rules()); std::printf("expected an exception\n"); return 1; }
    catch (const Error& e) { CHECK(e.code == DEMI_ERR_NO_DEVICE); std::printf("no device: %s\nOK (no-fallback contract)\n", e.what()); return 0; }
  }
  RandomScheduler sched(cfg, /*max_executions=*/4000, /*invariant_check_interval=*/5, /*seed=*/1);
  sched.setMaxMessages(50);
  auto found = sched.explore(prog);
  CHECK(found.has_value());
  ViolationFingerprint fp = found->second;
  STSScheduler sts(cfg, found->first, prog);
  DDMin ddmin(sts, /*checkUnmodifed=*/true);
  ExternalEvents mcs = ddmin.minimize(fp);
  auto verified = ddmin.verify_mcs(mcs, fp);
  if (!verified) { mcs.assign(prog.begin(), prog.end() - 1); verified = sts.test(mcs, fp); }
  CHECK(verified.has_value());
  STSSchedMinimizer im(mcs, *verified, fp, SrcDstFIFORemoval(), cfg);
  EventTrace itrace = im.minimize().second;
  for (int last = 0; last < 2; last++) {
    WildcardMinimizer wm = last ? WildcardMinimizer(cfg, mcs, itrace, fp, raft5_clock_rules(), LastOnlyStrategy())
                                : WildcardMinimizer(cfg, mcs, itrace, fp, raft5_clock_rules(), BackTrackStrategy());
    auto res = wm.minimize();
    std::printf("wildcard minimization (%s): %u -> %u deliveries in %u replays (%u executed, %u batches)\n",
                last ? "LastOnly" : "BackTrack", wm.last.deliveries_before, wm.last.deliveries_after,
                res.first.total_replays_ref(), wm.last.replays_executed, wm.last.batches);
    CHECK(wm.last.deliveries_after <= wm.last.deliveries_before && res.second.size() == wm.last.n_events);
    CHECK(res.first.internal_size.size() == wm.last.n_internal_sizes && res.first.total_replays_ref() == wm.last.total_replays);
    CHECK(res.first.stats.back().name == "(FungibleClockMinimizer,STSSched)");
    ReplayScheduler final_check(cfg, res.second, mcs);
    CHECK(final_check.replay(fp).violation == fp);
  }
  std::printf("OK\n");
  return 0;
}
