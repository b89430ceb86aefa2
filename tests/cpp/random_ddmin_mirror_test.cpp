// C++ host mirror (include/demi_b200.hpp) of DDMin with a RandomScheduler as the TestOracle: demi::randomDDMin on a
// violation RandomScheduler.explore finds in a pingpong3 program with HardKill, against demi_random_ddmin called
// directly, and DDMin(RandomScheduler).minimize against randomDDMin.  Prints "mcs <indices> total <total_replays>
// verified <0|1> events <verified trace length>", which the Python side compares with demi_b200.randomDDMin.
// Without a CUDA device: the no-fallback contract.
#include <cstdio>
#include "demi_b200.hpp"

using namespace demi;

#define CHECK(c) do { if (!(c)) { std::printf("CHECK failed: %s (line %d)\n", #c, __LINE__); return 1; } } while (0)

int main() {
  SchedulerConfig cfg;
  cfg.model = DEMI_MODEL_PINGPONG3;
  cfg.model_flags = 1 | (2 << 8);                     // a violation once actor 0 has seen 2 pongs
  ExternalEvents prog;
  for (int a = 0; a < 3; a++) prog.push_back(Start((uint8_t)a));
  for (uint32_t k = 0; k < 6; k++) prog.push_back(Send((uint8_t)(k % 3), 1, k));
  prog.push_back(WaitQuiescence());
  prog.push_back(HardKill(1));
  prog.push_back(Send(0, 1, 50));
  prog.push_back(Send(2, 1, 51));
  prog.push_back(WaitQuiescence());
  if (demi_device_count() == 0) {
    try { RandomScheduler s(cfg); std::printf("expected an exception\n"); return 1; }
    catch (const Error& e) { CHECK(e.code == DEMI_ERR_NO_DEVICE); std::printf("no device: %s\nOK (no-fallback contract)\n", e.what()); return 0; }
  }
  RandomScheduler explorer(cfg, 64, 0, 7);
  auto found = explorer.explore(prog);
  CHECK(found.has_value());
  const EventTrace trace = found->first;
  const ViolationFingerprint violation = found->second;
  RandomDDMinResult r = randomDDMin(cfg, trace, prog, violation, 16, 7);
  CHECK(r.violation == violation && !r.mcs.empty() && r.mcs.size() < prog.size());
  CHECK(r.verified.has_value() == (r.out.verified != 0));
  CHECK(r.stats.inner().total_replays == r.out.total_replays);
  // the C ABI called directly gives the same MCS and counters
  Engine e(cfg);
  e.check(demi_set_externals(e.handle(), prog.data(), (uint32_t)prog.size()));
  demi_fuzz_params p{7, 16, (int32_t)trace.size(), 0, violation, 0};
  std::vector<uint64_t> mcs(1, 0), keys(256);
  std::vector<uint32_t> sizes(256);
  demi_random_ddmin_out out{};
  e.check(demi_random_ddmin(e.handle(), &p, 0, mcs.data(), 1, sizes.data(), keys.data(), 256, &out));
  CHECK(events_of(prog, mcs).size() == r.mcs.size() && mask_of(prog, r.mcs) == mcs);
  CHECK(out.total_replays == r.out.total_replays && out.n_iterations == r.out.n_iterations && out.verified == r.out.verified);
  // the keyed series: each iteration size sits at the running sum of executions
  uint32_t at_fencepost = 0;
  for (auto& kv : r.stats.inner().iterationSize) at_fencepost = kv.first;
  CHECK(at_fencepost == out.total_replays);
  // DDMin(RandomScheduler).minimize is the same minimization
  RandomScheduler oracle(cfg, 16, 0, 7);
  oracle.setMaxMessages((int32_t)trace.size());
  DDMin ddmin(oracle);
  CHECK(ddmin.minimize(violation, prog).size() == r.mcs.size());
  std::printf("mcs");
  for (size_t i = 0; i < prog.size(); i++) if ((mcs[i >> 6] >> (i & 63)) & 1ull) std::printf(" %zu", i);
  std::printf(" total %llu verified %u events %zu\nOK\n", (unsigned long long)out.total_replays, out.verified,
              r.verified ? r.verified->size() : (size_t)0);
  return 0;
}
