// The C++ mirror's Engine::wildcard_minimize_many on the raft5 headline program with raft5's clock rules, after DDMin,
// the recorded verify_mcs and internal minimization: every minimized trace, its sizes and its record equal
// demi_set_trace + demi_wildcard_minimize, for both ambiguity resolutions.  Prints "OK" at the end.
#include <cstdio>
#include <cstring>
#include "demi_b200.hpp"

using namespace demi;

#define CHECK(c) do { if (!(c)) { std::printf("FAILED: %s (line %d)\n", #c, __LINE__); return 1; } } while (0)

int main() {
  SchedulerConfig cfg; cfg.model = DEMI_MODEL_RAFT5; cfg.model_flags = 1;
  Engine eng(cfg);
  // raft5's FingerprintFactory: the term is p0 & 0xFF of RequestVote, VoteReply, AppendEntries and AppendReply; an
  // ElectionTick increments the clock
  const uint32_t rules[4] = {DEMI_CLOCK_RULE(4, 0, 0, 8), DEMI_CLOCK_RULE(5, 0, 0, 8), DEMI_CLOCK_RULE(7, 0, 0, 8),
                             DEMI_CLOCK_RULE(8, 0, 0, 8)};
  const uint32_t incr[8] = {1u << 3, 0, 0, 0, 0, 0, 0, 0};
  eng.check(demi_set_clock_rules(eng.handle(), rules, 4, incr));
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
  eng.set_traces(traces, {prog});
  const uint32_t mw = eng.set_mask_words();
  const std::vector<Engine::DDMinManyResult> dd = eng.ddmin_many(codes);
  std::vector<uint32_t> tr; std::vector<uint64_t> masks;
  for (uint32_t t = 0; t < traces.size(); t++) {
    CHECK(dd[t].status == DEMI_OK);
    tr.push_back(t);
    const std::vector<uint64_t> m = mask_of(prog, dd[t].mcs);
    masks.insert(masks.end(), m.begin(), m.end());
  }
  const std::vector<Engine::RecordedReplay> rec = eng.replay_traces_many(tr, masks, {}, codes);
  std::vector<EventTrace> verified(traces.size());
  std::vector<ExternalEvents> mcs(traces.size());
  for (size_t t = 0; t < traces.size(); t++) {
    CHECK(rec[t].result.status == 0);
    verified[t] = rec[t].trace;
    mcs[t] = dd[t].mcs;
  }
  eng.set_traces(verified, mcs);
  const std::vector<Engine::IntMinManyResult> im = eng.internal_minimize_many(codes, DEMI_IM_SRC_DST_FIFO);
  std::vector<EventTrace> base(traces.size());
  for (size_t t = 0; t < traces.size(); t++) { CHECK(im[t].status == DEMI_OK); base[t] = im[t].trace; }
  eng.set_traces(base, mcs);
  size_t shrunk = 0;
  for (uint32_t flags : {0u, (uint32_t)DEMI_WC_LAST_ONLY}) {
    const std::vector<Engine::IntMinManyResult> wc = eng.wildcard_minimize_many(codes, flags);
    for (size_t t = 0; t < traces.size(); t++) {
      eng.check(demi_set_trace(eng.handle(), base[t].data(), (uint32_t)base[t].size(), mcs[t].data(), (uint32_t)mcs[t].size()));
      std::vector<demi_event> ev(4096); std::vector<uint32_t> sizes(1024); demi_intmin_out out{};
      const int32_t rc = demi_wildcard_minimize(eng.handle(), codes[t], flags, ev.data(), 4096, sizes.data(), 1024, &out);
      CHECK(wc[t].status == rc);
      if (rc != DEMI_OK) continue;
      CHECK(!std::memcmp(&out, &wc[t].out, sizeof(out)));
      CHECK(wc[t].trace.size() == out.n_events && !std::memcmp(ev.data(), wc[t].trace.data(), out.n_events * sizeof(demi_event)));
      CHECK(wc[t].internal_sizes == std::vector<uint32_t>(sizes.begin(), sizes.begin() + out.n_internal_sizes));
      shrunk += out.deliveries_after < out.deliveries_before;
    }
  }
  CHECK(shrunk > 0);
  std::printf("%zu traces OK\n", traces.size());
  return 0;
}
