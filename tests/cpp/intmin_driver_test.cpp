// IntMinDriver (demi_b200/csrc/intmin_driver.hpp) on the host, with the CPU oracle's STSSched replay
// (oracle_sts_replay_trace, with a skipped event) as both the evaluator of candidate removals and the recorder of the
// successful one.  Many drivers run in lock-step rounds as demi_internal_minimize_many runs them: every driver's
// candidates, then every evaluation, every commit, every recording, every advance.  Each trace's outcome must equal
// oracle_internal_minimize's, for both removal strategies and in every grouping of the traces.
//
// Input (argv[1]): little-endian uint32 words: n_cases, then per case model, model_flags, looking_for, n_blob_bytes,
// the blob (padded to words), n_ext, n_ext x 4 words, n_events, n_events x 4 words.  Prints "OK" at the end.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
extern "C" {
#include "../../oracle/sts.h"
int oracle_sts_replay_trace(const demi_config* cfg, const demi_replay_input* in, const uint64_t* mask, uint32_t looking_for,
                            uint32_t flags, uint32_t skip_event, demi_replay_result* out,
                            demi_event* rec, uint32_t cap_rec, uint32_t* n_rec);
int oracle_internal_minimize(const demi_config* cfg, const demi_event* verified, uint32_t n_verified,
                             const demi_ext_event* mcs_ext, uint32_t n_ext, uint32_t looking_for, uint32_t flags_in,
                             demi_event* out_trace, uint32_t cap_out, uint32_t* n_out,
                             uint32_t* total_replays, uint32_t* internal_sizes, uint32_t cap_sizes, uint32_t* n_sizes,
                             uint32_t* unignorable);
int oracle_load_model(const void* blob, size_t size);
uint32_t oracle_ir_external_mask(void);
}
#include "../../demi_b200/csrc/intmin_driver.hpp"

struct Case { demi_config cfg{}; uint32_t code = 0; std::vector<uint32_t> blob; std::vector<demi_ext_event> ext; std::vector<demi_event> ev; };
// one trace's outcome: status (0 or the driver's error), the trace, the sizes, the counters the oracle also reports
struct Outcome {
  int32_t status = 0; std::vector<demi_event> trace; std::vector<uint32_t> sizes; uint32_t total = 0, unig = 0;
  bool operator==(const Outcome& o) const {
    return status == o.status && sizes == o.sizes && total == o.total && unig == o.unig && trace.size() == o.trace.size() &&
           !memcmp(trace.data(), o.trace.data(), trace.size() * sizeof(demi_event));
  }
};

static uint32_t ext_mask(const Case& c) { return c.cfg.model == 100 ? oracle_ir_external_mask() : demi_external_type_mask(c.cfg.model); }

// STSScheduler(trace).test(full externals) leaving out trace event `skip`, recording into rec
static demi_replay_result replay(const Case& c, const std::vector<demi_event>& trace, uint32_t flags, uint32_t skip,
                                 std::vector<demi_event>& rec) {
  demi_replay_input in;
  uint32_t n_send_ev = 0, n_ext_sends = 0;
  for (const demi_event& e : trace) n_send_ev += e.kind == DEMI_EV_MSG_SEND;
  for (const demi_ext_event& e : c.ext) n_ext_sends += e.kind == DEMI_EXT_SEND;
  in.events = trace.data(); in.n_events = (uint32_t)trace.size(); in.externals = c.ext.data(); in.n_externals = (uint32_t)c.ext.size();
  in.external_type_mask = ext_mask(c);
  in.pending_cap = demi_replay_pending_cap(n_send_ev); in.tosend_cap = demi_tosend_cap(n_ext_sends);
  std::vector<uint64_t> full((c.ext.size() + 63) / 64 + 1, 0);
  for (size_t i = 0; i < c.ext.size(); i++) full[i >> 6] |= 1ull << (i & 63);
  demi_replay_result r{};
  uint32_t n = 0;
  rec.resize(65536);
  oracle_sts_replay_trace(&c.cfg, &in, full.data(), c.code, flags, skip, &r, rec.data(), (uint32_t)rec.size(), &n);
  rec.resize(n);
  return r;
}

static Outcome solo(const Case& c, uint32_t flags) {
  Outcome o;
  std::vector<demi_event> out(65536); std::vector<uint32_t> sizes(65536);
  uint32_t n_out = 0, n_sizes = 0;
  o.status = oracle_internal_minimize(&c.cfg, c.ev.data(), (uint32_t)c.ev.size(), c.ext.data(), (uint32_t)c.ext.size(), c.code,
                                      flags, out.data(), (uint32_t)out.size(), &n_out, &o.total, sizes.data(),
                                      (uint32_t)sizes.size(), &n_sizes, &o.unig) ? -1 : 0;
  o.trace.assign(out.begin(), out.begin() + n_out);
  o.sizes.assign(sizes.begin(), sizes.begin() + n_sizes);
  return o;
}

// the drivers of cases[idx[..]] in lock-step rounds
static std::vector<Outcome> lock_step(const std::vector<Case>& cases, const std::vector<size_t>& idx, uint32_t flags) {
  const size_t n = idx.size();
  const uint32_t rflags = flags & ~DEMI_IM_SRC_DST_FIFO;
  std::vector<demi::IntMinDriver> d(n);
  std::vector<demi_intmin_out> out(n);
  std::vector<Outcome> o(n);
  std::vector<char> live(n, 1);
  for (size_t k = 0; k < n; k++) {
    const Case& c = cases[idx[k]];
    d[k].init(c.ev.data(), (uint32_t)c.ev.size(), ext_mask(c), (flags & DEMI_IM_SRC_DST_FIFO) != 0, &out[k]);
  }
  std::vector<demi_event> rec;
  for (;;) {
    std::vector<std::vector<demi_replay_result>> res(n);
    bool any = false;
    for (size_t k = 0; k < n; k++)
      if (live[k]) { if (d[k].candidates().empty()) live[k] = 0; else any = true; }
    if (!any) break;
    for (size_t k = 0; k < n; k++)
      if (live[k]) for (uint32_t s : d[k].cand) res[k].push_back(replay(cases[idx[k]], d[k].cur, rflags, s, rec));
    std::vector<uint32_t> skip(n, 0);
    std::vector<char> record(n, 0);
    for (size_t k = 0; k < n; k++) {
      if (!live[k]) continue;
      const demi::IntMinDriver::Step step = d[k].commit(res[k].data(), &skip[k]);
      if (step == demi::IntMinDriver::FAILED) { o[k].status = -1; live[k] = 0; }
      else if (step == demi::IntMinDriver::DONE) live[k] = 0;
      else record[k] = 1;
    }
    for (size_t k = 0; k < n; k++) {
      if (!record[k]) continue;
      const demi_replay_result r = replay(cases[idx[k]], d[k].cur, rflags, skip[k], rec);
      if (!d[k].advance(r, rec.data(), (uint32_t)rec.size())) { o[k].status = -1; live[k] = 0; }
    }
  }
  for (size_t k = 0; k < n; k++) {
    if (o[k].status) continue;
    std::vector<demi_event> tr(65536); std::vector<uint32_t> sizes(65536);
    d[k].finish(tr.data(), (uint32_t)tr.size(), sizes.data(), (uint32_t)sizes.size());
    o[k].trace.assign(tr.begin(), tr.begin() + out[k].n_events);
    o[k].sizes.assign(sizes.begin(), sizes.begin() + out[k].n_internal_sizes);
    o[k].total = out[k].total_replays; o[k].unig = out[k].unignorable;
  }
  return o;
}

int main(int argc, char** argv) {
  if (argc < 2) { std::printf("usage: intmin_driver_test cases.bin\n"); return 2; }
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
  }
  fclose(f);
  // cases of one model (and blob) run together: the oracle holds one loaded model at a time
  size_t checked = 0;
  for (size_t lo = 0; lo < cases.size();) {
    size_t hi = lo;
    while (hi < cases.size() && cases[hi].cfg.model == cases[lo].cfg.model && cases[hi].blob == cases[lo].blob) hi++;
    if (!cases[lo].blob.empty() && oracle_load_model(cases[lo].blob.data(), cases[lo].blob.size() * 4) != 0) {
      std::printf("FAILED: model load\n"); return 1;
    }
    for (uint32_t flags : {0u, (uint32_t)DEMI_IM_SRC_DST_FIFO, (uint32_t)DEMI_RF_FILTER_KNOWN_ABSENTS}) {
      std::vector<Outcome> want;
      for (size_t i = lo; i < hi; i++) want.push_back(solo(cases[i], flags));
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
  std::printf("%zu cases, %zu outcomes OK\n", cases.size(), checked);
  return 0;
}
