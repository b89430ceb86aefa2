// The C++ mirror's Engine::fuzz_traces_many (include/demi_b200.hpp) on raft5 programs of mixed lengths, one with a
// HardKill and one that demi_set_externals rejects: every trace's status, EventTrace, record and DepTracker tree equal
// demi_set_externals + demi_fuzz_trace on a second handle, and with masks demi_set_externals + demi_random_test_trace.
// Prints "N traces OK" at the end.
#include <cstdio>
#include <cstring>
#include "demi_b200.hpp"

using namespace demi;

#define CHECK(c) do { if (!(c)) { std::printf("FAILED: %s (line %d)\n", #c, __LINE__); return 1; } } while (0)

static ExternalEvents raft5(int cmds, bool hard_kill) {
  ExternalEvents prog;
  for (int a = 0; a < 5; a++) prog.push_back(Start((uint8_t)a));
  for (int a = 0; a < 5; a++) prog.push_back(Send((uint8_t)a, 1, 0x1F));   // BOOT, membership bitmask
  prog.push_back(WaitQuiescence());
  for (int k = 0; k < cmds; k++) prog.push_back(Send((uint8_t)(k % 5), 2, 10 + k));   // CLIENT_CMD
  if (hard_kill) { prog.push_back(WaitQuiescence()); prog.push_back(HardKill(1)); prog.push_back(Send(2, 2, 40)); }
  prog.push_back(WaitQuiescence());
  return prog;
}

int main() {
  SchedulerConfig cfg; cfg.model = DEMI_MODEL_RAFT5; cfg.model_flags = 1;
  Engine eng(cfg), ref(cfg);
  std::vector<ExternalEvents> progs;
  std::vector<int64_t> seeds; std::vector<int32_t> maxm; std::vector<ViolationFingerprint> looking;
  for (int t = 0; t < 10; t++) {
    progs.push_back(raft5(1 + t % 4, t == 7));
    seeds.push_back(100 + 7 * t); maxm.push_back(40 + 5 * (t % 3)); looking.push_back(t % 2);
  }
  progs[4].push_back(WaitQuiescence());                                     // adjacent WaitQuiescence: rejected
  const std::vector<Engine::RecordedExecution> got = eng.fuzz_traces_many(progs, seeds, maxm, looking, 5, {}, true, 1024, 1024);
  std::vector<std::vector<uint64_t>> masks;
  for (size_t t = 0; t < progs.size(); t++) {
    std::vector<uint64_t> m(1, (1ull << progs[t].size()) - 1);
    if (t % 2) m[0] &= ~(1ull << 11);                                      // drop the first CLIENT_CMD
    masks.push_back(m);
  }
  const std::vector<Engine::RecordedExecution> sub = eng.fuzz_traces_many(progs, seeds, maxm, looking, 5, masks, false, 1024);
  for (size_t t = 0; t < progs.size(); t++) {
    const int32_t rc = demi_set_externals(ref.handle(), progs[t].data(), (uint32_t)progs[t].size());
    CHECK(got[t].status == rc && sub[t].status == rc);
    if (rc != DEMI_OK) { CHECK(t == 4 && got[t].trace.empty()); continue; }
    demi_fuzz_params p{seeds[t], 1, maxm[t], 5, looking[t], 0};
    std::vector<demi_event> ev(1024); std::vector<uint16_t> par(1024); uint32_t n = 0, nn = 0; demi_fuzz_result r{};
    ref.check(demi_fuzz_trace(ref.handle(), &p, seeds[t], ev.data(), 1024, &n, par.data(), 1024, &nn, &r));
    CHECK(n == got[t].trace.size() && !std::memcmp(ev.data(), got[t].trace.data(), n * sizeof(demi_event)));
    CHECK(nn == got[t].depGraph.size() && !std::memcmp(par.data(), got[t].depGraph.data(), nn * sizeof(uint16_t)));
    CHECK(!std::memcmp(&r, &got[t].result, sizeof(r)));
    ref.check(demi_random_test_trace(ref.handle(), masks[t].data(), 1, &p, seeds[t], ev.data(), 1024, &n, &r));
    CHECK(n == sub[t].trace.size() && !std::memcmp(ev.data(), sub[t].trace.data(), n * sizeof(demi_event)));
    CHECK(!std::memcmp(&r, &sub[t].result, sizeof(r)) && sub[t].depGraph.empty());
  }
  std::printf("%zu traces OK\n", progs.size());
  return 0;
}
