// The C++ mirror's many-trace calls (Engine::fuzz_traces, set_traces, replay_batch_many, ddmin_many) on the raft5
// headline program: every record equals the single-trace calls' (demi_fuzz_trace, demi_set_trace + demi_replay_batch,
// DDMin over STSScheduler).  Prints "OK" at the end.
#include <cstdio>
#include <cstring>
#include "demi_b200.hpp"

using namespace demi;

#define CHECK(c) do { if (!(c)) { std::printf("FAILED: %s (line %d)\n", #c, __LINE__); return 1; } } while (0)

int main() {
  SchedulerConfig cfg; cfg.model = DEMI_MODEL_RAFT5; cfg.model_flags = 1;
  Engine eng(cfg);
  ExternalEvents prog;
  for (int a = 0; a < 5; a++) prog.push_back(Start((uint8_t)a));
  for (int a = 0; a < 5; a++) prog.push_back(Send((uint8_t)a, 1, 0x1F));   // BOOT, membership bitmask
  prog.push_back(WaitQuiescence());
  eng.check(demi_set_externals(eng.handle(), prog.data(), (uint32_t)prog.size()));
  demi_fuzz_params p{1, 4000, 50, 5, 0, 0};
  std::vector<demi_fuzz_result> res(4000);
  eng.check(demi_fuzz_batch(eng.handle(), &p, res.data()));
  std::vector<uint32_t> hits;
  std::vector<ViolationFingerprint> codes;
  for (uint32_t i = 0; i < res.size() && hits.size() < 24; i++)
    if (res[i].violation && !res[i].status) { hits.push_back(i); codes.push_back(res[i].violation); }
  CHECK(hits.size() == 24);
  const std::vector<EventTrace> traces = eng.fuzz_traces(1, hits, 50, 5);
  for (size_t i = 0; i < hits.size(); i++) {
    std::vector<demi_event> ev(1024); uint32_t n = 0; demi_fuzz_result r{};
    eng.check(demi_fuzz_trace(eng.handle(), &p, 1 + hits[i], ev.data(), 1024, &n, nullptr, 0, nullptr, &r));
    CHECK(n == traces[i].size() && !std::memcmp(ev.data(), traces[i].data(), n * sizeof(demi_event)));
  }
  eng.set_traces(traces, {prog});
  const uint32_t mw = eng.set_mask_words();
  std::vector<uint32_t> tr; std::vector<uint64_t> masks;
  for (uint32_t k = 0; k < 8 * traces.size(); k++) { tr.push_back(k % traces.size()); masks.push_back((0x9E3779B97F4A7C15ull * (k + 1)) >> 53); }
  const std::vector<demi_replay_result> many = eng.replay_batch_many(tr, masks, codes);
  const std::vector<Engine::DDMinManyResult> dd = eng.ddmin_many(codes);
  for (size_t t = 0; t < traces.size(); t++) {
    eng.check(demi_set_trace(eng.handle(), traces[t].data(), (uint32_t)traces[t].size(), prog.data(), (uint32_t)prog.size()));
    for (size_t k = 0; k < tr.size(); k++) {
      if (tr[k] != t) continue;
      demi_replay_result one{};
      eng.check(demi_replay_batch(eng.handle(), &masks[k], 1, mw, codes[t], 0, &one));
      CHECK(!std::memcmp(&one, &many[k], sizeof(one)));
    }
    std::vector<uint64_t> mcs(mw); std::vector<uint32_t> iters(256); demi_ddmin_out out{};
    eng.check(demi_ddmin(eng.handle(), codes[t], 0, 1, mcs.data(), mw, iters.data(), 256, &out));
    CHECK(dd[t].status == DEMI_OK && dd[t].out.mcs_size == out.mcs_size && dd[t].out.total_replays == out.total_replays);
    CHECK(dd[t].out.replays_executed == out.replays_executed && dd[t].out.batches == out.batches && dd[t].out.verified == out.verified);
    const ExternalEvents want = events_of(prog, mcs);
    CHECK(dd[t].mcs.size() == want.size());
    for (size_t i = 0; i < want.size(); i++) CHECK(dd[t].mcs[i].id == want[i].id);
    CHECK(dd[t].iteration_sizes == std::vector<uint32_t>(iters.begin(), iters.begin() + out.n_iterations));
  }
  std::printf("%zu traces OK\n", traces.size());
  return 0;
}
