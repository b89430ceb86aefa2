// C++ host mirror (include/demi_b200.hpp) of fuzzing campaigns: demi::fuzz (RunnerUtils.fuzz) against a host loop built
// from the per-program calls (demi_fuzzer_generate, demi_set_externals, demi_fuzz_batch one execution at a time), with a
// predicate, a spent budget, strict replay and provenance.  Prints "found <execution> <violation>" for the default
// call, which the Python side compares with demi_b200.fuzz.  Without a CUDA device: the no-fallback contract.
#include <cstdio>
#include "demi_b200.hpp"

using namespace demi;

#define CHECK(c) do { if (!(c)) { std::printf("CHECK failed: %s (line %d)\n", #c, __LINE__); return 1; } } while (0)

// the first execution < budget whose record violates and passes `accept`: (execution, violation), or (-1, 0)
static std::pair<int64_t, uint32_t> host_loop(const SchedulerConfig& cfg, const demi_fuzzer_config& fz, const ExternalEvents& prefix,
                                              uint64_t budget, const std::function<bool(uint32_t)>& accept) {
  Engine eng(cfg);
  ExternalEvents prog(prefix.size() + fz.num_events + 1);
  for (uint64_t k = 0; k < budget; k++) {
    uint32_t n = 0;
    eng.check(demi_fuzzer_generate(&fz, PROGRAM_SEED_OFFSET + (int64_t)k, prefix.data(), (uint32_t)prefix.size(), nullptr, 0,
                                   prog.data(), (uint32_t)prog.size(), &n));
    eng.check(demi_set_externals(eng.handle(), prog.data(), n));
    demi_fuzz_params p{(int64_t)k, 1, 50, 5, 0, 0};
    demi_fuzz_result r{};
    eng.check(demi_fuzz_batch(eng.handle(), &p, &r));
    if (!r.status && r.violation && accept(r.violation)) return {(int64_t)k, r.violation};
  }
  return {-1, 0};
}

int main() {
  SchedulerConfig cfg;
  cfg.model = DEMI_MODEL_RAFT5;
  cfg.model_flags = 3;
  ExternalEvents prefix;
  for (int a = 0; a < 5; a++) prefix.push_back(Start((uint8_t)a));
  for (int a = 0; a < 5; a++) prefix.push_back(Send((uint8_t)a, 1, 0x1F));
  prefix.push_back(WaitQuiescence());
  const demi_fuzzer_config fz{0.01, 0.3, 0.1, 0.1, 0.1, 40, 2};      // FuzzerWeights' defaults, CLIENT_CMD
  if (demi_device_count() == 0) {
    try { fuzz(fz, prefix, {}, cfg); std::printf("expected an exception\n"); return 1; }
    catch (const Error& e) { CHECK(e.code == DEMI_ERR_NO_DEVICE); std::printf("no device: %s\nOK (no-fallback contract)\n", e.what()); return 0; }
  }
  auto any = [](uint32_t) { return true; };
  auto first = fuzz(fz, prefix, {}, cfg, false, 5, 50, false, nullptr, 2000, 0, std::nullopt, nullptr, 17);
  CHECK(first.has_value());
  std::printf("found %llu %u\n", (unsigned long long)first->execution, first->violation);
  auto want = host_loop(cfg, fz, prefix, 2000, any);
  CHECK(want.first == (int64_t)first->execution && want.second == first->violation);
  CHECK(first->initialTrace.size() >= 1 && first->initialTrace[0] == 0);
  // a predicate that rejects the first violation code: the next matching execution
  const uint32_t v0 = first->violation;
  auto other_pred = [v0](uint32_t v) { return v != v0; };
  auto other = fuzz(fz, prefix, {}, cfg, false, 5, 50, false, other_pred, 5000);
  auto want2 = host_loop(cfg, fz, prefix, 5000, other_pred);
  if (want2.first < 0) CHECK(!other.has_value());
  else CHECK(other.has_value() && (int64_t)other->execution == want2.first && other->violation == want2.second && other->violation != v0);
  // a spent budget
  CHECK(!fuzz(fz, prefix, {}, cfg, false, 5, 50, false, nullptr, first->execution).has_value());
  // strict replay and provenance: the same execution; `filtered` is what ProvenanceTracker keeps of its trace
  auto prov = fuzz(fz, prefix, {}, cfg, /*validate_replay=*/true, 5, 50, /*computeProvenance=*/true, nullptr, 2000);
  CHECK(prov.has_value() && prov->execution == first->execution && prov->trace.size() == first->trace.size());
  uint32_t deliveries = 0;
  for (const demi_event& e : prov->trace) deliveries += e.kind == DEMI_EV_MSG_EVENT;
  CHECK(!prov->filtered.empty() && prov->filtered.size() <= deliveries);
  for (const demi_event& e : prov->filtered) CHECK(e.kind == DEMI_EV_MSG_EVENT);
  std::printf("filtered %zu of %u deliveries\nOK\n", prov->filtered.size(), deliveries);
  return 0;
}
