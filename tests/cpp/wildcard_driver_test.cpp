// WildcardDriver (demi_b200/csrc/wildcard_driver.hpp) on the host, with the CPU oracle's wildcard STSSched replay
// (oracle_wildcard_replay) as both the evaluator of candidate include masks and the recorder of the successful one.
// Many drivers run in lock-step rounds as demi_wildcard_minimize_many runs them: every driver's candidates, then every
// evaluation, every commit, every recording, every advance.  Each trace's outcome must equal oracle_wildcard_minimize's,
// for both ambiguity resolutions, with and without filterKnownAbsents, and in every grouping of the traces.
//
// Input (argv[1]): little-endian uint32 words: n_cases, then per case model, model_flags, looking_for, n_blob_bytes,
// the blob (padded to words), n_ext, n_ext x 4 words, n_events, n_events x 4 words, n_rules, the rules, the 8 words of
// the causesClockIncrement set.  Prints "OK" at the end.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
extern "C" {
#include "../../oracle/sts.h"
void oracle_wildcard_replay(const demi_config* cfg, const demi_event* ev, uint32_t n_ev, const demi_ext_event* ext, uint32_t n_ext,
                            const uint64_t* include, const uint32_t* incr, uint32_t looking_for, uint32_t flags,
                            demi_replay_result* out, demi_event* rec, uint32_t cap_rec, uint32_t* n_rec,
                            uint32_t* ignored, uint32_t cap_ignored, uint32_t* n_ignored);
int oracle_wildcard_minimize(const demi_config* cfg, const demi_event* verified, uint32_t n_verified,
                             const demi_ext_event* mcs_ext, uint32_t n_ext, const uint32_t* rule, const uint32_t* incr,
                             uint32_t looking_for, uint32_t flags,
                             demi_event* out_trace, uint32_t cap_out, uint32_t* n_out,
                             uint32_t* total_replays, uint32_t* internal_sizes, uint32_t cap_sizes, uint32_t* n_sizes);
int oracle_load_model(const void* blob, size_t size);
uint32_t oracle_ir_external_mask(void);
}
#include "../../demi_b200/csrc/wildcard_driver.hpp"

struct Case {
  demi_config cfg{}; uint32_t code = 0; std::vector<uint32_t> blob; std::vector<demi_ext_event> ext; std::vector<demi_event> ev;
  uint32_t rule[256] = {}; uint32_t incr[8] = {};
};
// one trace's outcome: status (0 or the driver's error), the trace, the sizes, the replays the oracle also counts
struct Outcome {
  int32_t status = 0; std::vector<demi_event> trace; std::vector<uint32_t> sizes; uint32_t total = 0;
  bool operator==(const Outcome& o) const {
    return status == o.status && sizes == o.sizes && total == o.total && trace.size() == o.trace.size() &&
           !memcmp(trace.data(), o.trace.data(), trace.size() * sizeof(demi_event));
  }
};

static uint32_t ext_mask(const Case& c) { return c.cfg.model == 100 ? oracle_ir_external_mask() : demi_external_type_mask(c.cfg.model); }

// one wildcard STSScheduler.test of the case's base trace: result, recording, ignored trace positions
static demi_replay_result replay(const Case& c, const uint64_t* include, uint32_t flags, std::vector<demi_event>& rec,
                                 std::vector<uint32_t>& ign) {
  demi_replay_result r{};
  uint32_t n = 0, ni = 0;
  rec.resize(65536); ign.resize(c.ev.size() + 1);
  oracle_wildcard_replay(&c.cfg, c.ev.data(), (uint32_t)c.ev.size(), c.ext.data(), (uint32_t)c.ext.size(), include, c.incr,
                         c.code, flags, &r, rec.data(), (uint32_t)rec.size(), &n, ign.data(), (uint32_t)ign.size(), &ni);
  rec.resize(n); ign.resize(ni);
  return r;
}

static Outcome solo(const Case& c, uint32_t flags) {
  Outcome o;
  std::vector<demi_event> out(65536); std::vector<uint32_t> sizes(65536);
  uint32_t n_out = 0, n_sizes = 0;
  o.status = oracle_wildcard_minimize(&c.cfg, c.ev.data(), (uint32_t)c.ev.size(), c.ext.data(), (uint32_t)c.ext.size(), c.rule,
                                      c.incr, c.code, flags, out.data(), (uint32_t)out.size(), &n_out, &o.total, sizes.data(),
                                      (uint32_t)sizes.size(), &n_sizes) ? -1 : 0;
  o.trace.assign(out.begin(), out.begin() + n_out);
  o.sizes.assign(sizes.begin(), sizes.begin() + n_sizes);
  return o;
}

// the drivers of cases[idx[..]] in lock-step rounds
static std::vector<Outcome> lock_step(const std::vector<Case>& cases, const std::vector<size_t>& idx, uint32_t flags) {
  const size_t n = idx.size();
  std::vector<demi::WildcardDriver> d(n);
  std::vector<demi_intmin_out> out(n);
  std::vector<Outcome> o(n);
  std::vector<char> live(n, 1);
  for (size_t k = 0; k < n; k++) {
    const Case& c = cases[idx[k]];
    if (!d[k].init(c.ev.data(), (uint32_t)c.ev.size(), ext_mask(c), c.rule, c.incr, &out[k])) { o[k].status = -1; live[k] = 0; }
  }
  std::vector<demi_event> rec; std::vector<uint32_t> ign;
  for (;;) {
    std::vector<std::vector<demi_replay_result>> res(n);
    bool any = false;
    for (size_t k = 0; k < n; k++)
      if (live[k]) { if (d[k].candidates().empty()) live[k] = 0; else any = true; }
    if (!any) break;
    for (size_t k = 0; k < n; k++)
      if (live[k])
        for (size_t c = 0; c < d[k].n_candidates(); c++)
          res[k].push_back(replay(cases[idx[k]], d[k].cand.data() + c * d[k].t.words, flags, rec, ign));
    std::vector<const uint64_t*> mask(n, nullptr);
    for (size_t k = 0; k < n; k++) {
      if (!live[k]) continue;
      const demi::WildcardDriver::Step step = d[k].commit(res[k].data(), &mask[k]);
      if (step == demi::WildcardDriver::FAILED) { o[k].status = -1; live[k] = 0; mask[k] = nullptr; }
      else if (step == demi::WildcardDriver::DONE) mask[k] = nullptr;
    }
    for (size_t k = 0; k < n; k++) {
      if (!mask[k]) continue;
      const demi_replay_result r = replay(cases[idx[k]], mask[k], flags, rec, ign);
      if (!d[k].advance(r, rec.data(), (uint32_t)rec.size(), ign.data(), (uint32_t)ign.size())) { o[k].status = -1; live[k] = 0; }
    }
  }
  for (size_t k = 0; k < n; k++) {
    if (o[k].status) continue;
    std::vector<demi_event> tr(65536); std::vector<uint32_t> sizes(65536);
    d[k].finish(tr.data(), (uint32_t)tr.size(), sizes.data(), (uint32_t)sizes.size());
    o[k].trace.assign(tr.begin(), tr.begin() + out[k].n_events);
    o[k].sizes.assign(sizes.begin(), sizes.begin() + out[k].n_internal_sizes);
    o[k].total = out[k].total_replays;
  }
  return o;
}

int main(int argc, char** argv) {
  if (argc < 2) { std::printf("usage: wildcard_driver_test cases.bin\n"); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) { std::printf("cannot open %s\n", argv[1]); return 2; }
  auto word = [&]() { uint32_t w = 0; if (fread(&w, 4, 1, f) != 1) { std::printf("short input\n"); exit(2); } return w; };
  std::vector<Case> cases(word());
  for (Case& c : cases) {
    c.cfg.model = (int32_t)word(); c.cfg.model_flags = word(); c.code = word();
    c.blob.resize((word() + 3) / 4);
    for (uint32_t& w : c.blob) w = word();
    c.ext.resize(word());
    for (demi_ext_event& e : c.ext) { uint32_t w[4] = {word(), word(), word(), word()}; memcpy(&e, w, 16); }
    c.ev.resize(word());
    for (demi_event& e : c.ev) { uint32_t w[4] = {word(), word(), word(), word()}; memcpy(&e, w, 16); }
    for (uint32_t k = word(); k > 0; k--) { const uint32_t r = word(); c.rule[r & 0xFF] = r; }
    for (uint32_t& w : c.incr) w = word();
  }
  fclose(f);
  // cases of one model (and blob) run together: the oracle holds one loaded model at a time
  size_t checked = 0, shrunk = 0;
  for (size_t lo = 0; lo < cases.size();) {
    size_t hi = lo;
    while (hi < cases.size() && cases[hi].cfg.model == cases[lo].cfg.model && cases[hi].blob == cases[lo].blob) hi++;
    if (!cases[lo].blob.empty() && oracle_load_model(cases[lo].blob.data(), cases[lo].blob.size() * 4) != 0) {
      std::printf("FAILED: model load\n"); return 1;
    }
    for (uint32_t flags : {0u, (uint32_t)DEMI_WC_LAST_ONLY, (uint32_t)DEMI_RF_FILTER_KNOWN_ABSENTS,
                           (uint32_t)(DEMI_WC_LAST_ONLY | DEMI_RF_FILTER_KNOWN_ABSENTS)}) {
      std::vector<Outcome> want;
      for (size_t i = lo; i < hi; i++) {
        want.push_back(solo(cases[i], flags));
        shrunk += want.back().trace.size() < cases[i].ev.size();
      }
      // groupings: all together, each alone, every other one in reverse order
      std::vector<std::vector<size_t>> groups(1);
      for (size_t i = lo; i < hi; i++) { groups[0].push_back(i); groups.push_back({i}); }
      groups.emplace_back();
      for (size_t i = hi; i-- > lo;) if ((i - lo) % 2 == 0) groups.back().push_back(i);
      for (const std::vector<size_t>& g : groups) {
        const std::vector<Outcome> got = lock_step(cases, g, flags);
        for (size_t k = 0; k < g.size(); k++) {
          if (!(got[k] == want[g[k] - lo])) {
            std::printf("FAILED: case %zu (model %d), flags 0x%x, group of %zu\n", g[k], cases[g[k]].cfg.model, flags, g.size());
            return 1;
          }
          checked++;
        }
      }
    }
    lo = hi;
  }
  std::printf("%zu cases, %zu shrunk, %zu outcomes OK\n", cases.size(), shrunk, checked);
  return shrunk ? 0 : 1;
}
