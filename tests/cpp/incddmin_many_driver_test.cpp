// IncDDMinDriver (demi_b200/csrc/incddmin_driver.hpp) host-only, as demi_incremental_ddmin_many runs it: many drivers
// on threads at once behind the shared rendezvous (many_rendezvous.hpp), every round's requests served together by the
// CPU oracle's DPOR instances (oracle_dpor_open / oracle_dpor_test / oracle_dpor_close).  Each test of a request is a
// fresh instance put through its cap history, which is what the device evaluates.  Built with AddressSanitizer.  Each
// trace's MCS, total_replays, rounds and instances must equal oracle_incremental_ddmin's, and all of its counters must
// equal those of its driver run alone, for every window.
//
// Input (argv[1]): little-endian uint32 words: n_cases, then per case model, model_flags, looking_for, max_messages,
// max_interleavings, n_blob_bytes, the blob (padded to words), n_ext, n_ext x 4 words, n_nodes, n_nodes x 4 words (the
// seed graph), n_trace, n_trace words (the seed trace).  Consecutive cases with the same model and blob form a group,
// minimised in one rendezvous.  Prints "OK" at the end.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
extern "C" {
#include "../../oracle/dpor.h"
int oracle_incremental_ddmin(const demi_config* cfg, const demi_ext_event* ext, uint32_t n_ext,
                             const demi_dpor_params* P, const oracle_dpor_opts* opts,
                             int32_t max_max_distance, uint32_t stop_at_size, uint32_t cap_instances,
                             uint64_t* mcs, uint32_t mw, uint32_t* total_replays, uint32_t* rounds,
                             uint64_t* total_interleavings, uint32_t* n_instances, uint32_t* mcs_sizes, uint32_t cap_sizes);
int oracle_load_model(const void* blob, size_t size);
}
#include "../../demi_b200/csrc/incddmin_driver.hpp"
#include "../../demi_b200/csrc/many_rendezvous.hpp"

thread_local std::string g_create_error;

using namespace demi;

constexpr int32_t MAX_MAX_DISTANCE = 16;
constexpr uint32_t STOP_AT_SIZE = 1;
constexpr uint32_t FLAGS = DEMI_DF_ARVIND_ORDERING | DEMI_DF_PRIORITIZE_PENDING;   // oracle_incremental_ddmin's configuration

struct Case {
  demi_config cfg{}; uint32_t code = 0, maxm = 0, budget = 0;
  std::vector<uint32_t> blob; uint32_t blob_bytes = 0;
  std::vector<demi_ext_event> ext; std::vector<uint32_t> nodes, trace;
  uint32_t mw() const { return (uint32_t)(ext.size() + 63) / 64 ? (uint32_t)(ext.size() + 63) / 64 : 1u; }
  demi_dpor_params params() const { return demi_dpor_params{(int32_t)maxm, -1, budget, code, 1u, 4096u, 1u << 16, 1u << 17}; }
  oracle_dpor_opts opts() const {
    return oracle_dpor_opts{nodes.data(), (uint32_t)nodes.size() / 4, trace.data(), (uint32_t)trace.size(), 1u, 1u};
  }
};

// One DPOR instance over `ext`, put through `caps` in order; its record accumulated as demi_dpor_batch_ex accumulates it
static demi_dpor_result instance(const Case& c, const std::vector<demi_ext_event>& ext, const int32_t* caps, uint32_t n_caps) {
  const demi_dpor_params P = c.params();
  const oracle_dpor_opts o = c.opts();
  void* s = oracle_dpor_open(&c.cfg, ext.data(), (uint32_t)ext.size(), &P, &o);
  demi_dpor_result acc{};
  if (!s) { acc.status = 0xFFFF; return acc; }
  for (uint32_t i = 0; i < n_caps; i++) {
    demi_dpor_result r{};
    oracle_dpor_test(s, caps[i], &r, nullptr, 0, nullptr, 0);
    acc.interleavings += r.interleavings;
    acc.violations = r.violations;
    if (r.status) acc.status = r.status;
  }
  oracle_dpor_close(s);
  return acc;
}

// the instances of n tests of case c: test k runs the externals mask k selects through caps[cap_off[k] .. cap_off[k+1])
static void run_tests(const Case& c, const IncDDMinDriver& d, const uint64_t* masks, size_t n, const std::vector<int32_t>& caps,
                      const std::vector<uint32_t>& cap_off, demi_dpor_result* res) {
  for (size_t k = 0; k < n; k++) {
    std::vector<demi_ext_event> flat;
    std::vector<uint32_t> off;
    d.select(masks + k * d.mw, 1, flat, off);
    res[k] = instance(c, flat, caps.data() + cap_off[k], cap_off[k + 1] - cap_off[k]);
  }
}

struct SoloDriver : IncDDMinDriver {
  const Case* c;
  int32_t run_dpor(const uint64_t* masks, size_t n, const std::vector<int32_t>& caps, const std::vector<uint32_t>& cap_off,
                   demi_dpor_result* res) override {
    run_tests(*c, *this, masks, n, caps, cap_off, res);
    return DEMI_OK;
  }
};

struct DporPayload { const std::vector<int32_t>* caps; const std::vector<uint32_t>* cap_off; };

struct ManyDriver : IncDDMinDriver {
  Rendezvous<demi_dpor_result>* R; uint32_t trace;
  int32_t run_dpor(const uint64_t* masks, size_t n, const std::vector<int32_t>& caps, const std::vector<uint32_t>& cap_off,
                   demi_dpor_result* res) override {
    const DporPayload pl{&caps, &cap_off};
    ManyRequest<demi_dpor_result> q;
    q.trace = trace; q.masks = masks; q.n = n; q.payload = &pl;
    R->submit(q);
    if (q.rc != DEMI_OK) return q.rc;
    std::copy(q.res.begin(), q.res.end(), res);
    return DEMI_OK;
  }
};

template <class D> static void setup(D& d, demi_handle* h, const Case& c) {
  d.h = h; d.looking_for = c.code; d.flags = 0; d.mw = c.mw(); d.n_ext = (uint32_t)c.ext.size(); d.ext = c.ext.data();
}

struct Outcome {
  int32_t status = 0; std::vector<uint64_t> mcs; demi_incddmin_out out{};
  bool operator==(const Outcome& o) const { return status == o.status && mcs == o.mcs && !memcmp(&out, &o.out, sizeof(out)); }
};

static Outcome solo(const Case& c) {
  demi_handle eh;
  SoloDriver d;
  setup(d, &eh, c);
  d.c = &c;
  Outcome r;
  r.mcs.assign(c.mw(), 0);
  r.status = d.minimize(MAX_MAX_DISTANCE, STOP_AT_SIZE, r.mcs.data(), &r.out);
  return r;
}

static std::vector<Outcome> many(const std::vector<Case>& cs, size_t lo, size_t hi, uint32_t window) {
  const uint32_t n = (uint32_t)(hi - lo);
  std::vector<Outcome> r(n);
  std::vector<int32_t> status(n, -1);
  auto drive = [&](uint32_t t, Rendezvous<demi_dpor_result>& R, demi_handle* eh) -> int32_t {
    ManyDriver d;
    setup(d, eh, cs[lo + t]);
    d.R = &R; d.trace = t;
    r[t].mcs.assign(cs[lo + t].mw(), 0);
    return d.minimize(MAX_MAX_DISTANCE, STOP_AT_SIZE, r[t].mcs.data(), &r[t].out);
  };
  auto serve = [&](std::vector<ManyRequest<demi_dpor_result>*>& batch) -> int32_t {
    for (ManyRequest<demi_dpor_result>* q : batch) {
      const Case& c = cs[lo + q->trace];
      const DporPayload& pl = *(const DporPayload*)q->payload;
      SoloDriver shape;                    // select() needs the trace's externals and mask width
      setup(shape, nullptr, c);
      q->res.resize(q->n);
      run_tests(c, shape, q->masks, q->n, *pl.caps, *pl.cap_off, q->res.data());
    }
    return DEMI_OK;
  };
  demi_handle h;
  const int32_t rc = run_many<demi_dpor_result>(&h, "incddmin_many_driver_test", n, window, drive, serve, status.data());
  for (uint32_t t = 0; t < n; t++) r[t].status = rc != DEMI_OK ? rc : status[t];
  return r;
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<uint32_t> w;
  uint32_t x;
  while (fread(&x, 4, 1, f) == 1) w.push_back(x);
  fclose(f);
  size_t p = 0;
  auto take = [&](void* dst, size_t words) { memcpy(dst, &w[p], words * 4); p += words; };
  std::vector<Case> cs(w[p++]);
  for (Case& c : cs) {
    c.cfg.model = (int32_t)w[p++]; c.cfg.model_flags = w[p++]; c.code = w[p++]; c.maxm = w[p++]; c.budget = w[p++];
    c.blob_bytes = w[p++];
    c.blob.resize((c.blob_bytes + 3) / 4); take(c.blob.data(), c.blob.size());
    c.ext.resize(w[p++]); take(c.ext.data(), c.ext.size() * 4);
    c.nodes.resize(w[p++] * 4); take(c.nodes.data(), c.nodes.size());
    c.trace.resize(w[p++]); take(c.trace.data(), c.trace.size());
  }
  size_t checked = 0;
  for (size_t lo = 0; lo < cs.size();) {
    size_t hi = lo + 1;
    while (hi < cs.size() && cs[hi].cfg.model == cs[lo].cfg.model && cs[hi].blob == cs[lo].blob) hi++;
    if (cs[lo].blob_bytes && oracle_load_model(cs[lo].blob.data(), cs[lo].blob_bytes) != 0) { std::printf("FAILED: load_model\n"); return 1; }
    std::vector<Outcome> alone;
    for (size_t i = lo; i < hi; i++) {
      const Case& c = cs[i];
      alone.push_back(solo(c));
      const demi_dpor_params P = c.params();
      const oracle_dpor_opts o = c.opts();
      std::vector<uint64_t> mcs(c.mw(), 0);
      uint32_t total = 0, rounds = 0, inst = 0;
      uint64_t il = 0;
      const int rc = oracle_incremental_ddmin(&c.cfg, c.ext.data(), (uint32_t)c.ext.size(), &P, &o, MAX_MAX_DISTANCE, STOP_AT_SIZE,
                                              4096, mcs.data(), c.mw(), &total, &rounds, &il, &inst, nullptr, 0);
      const Outcome& a = alone.back();
      if (rc != 0 || a.status != DEMI_OK || a.mcs != mcs || a.out.total_replays != total || a.out.rounds != rounds ||
          a.out.instances != inst) {
        std::printf("FAILED: case %zu alone differs from oracle_incremental_ddmin (rc %d status %d)\n", i, rc, a.status);
        return 1;
      }
    }
    for (uint32_t window : {1u, 7u, 512u}) {
      const std::vector<Outcome> got = many(cs, lo, hi, window);
      for (size_t i = lo; i < hi; i++)
        if (!(got[i - lo] == alone[i - lo])) {
          std::printf("FAILED: case %zu window %u differs from its solo run\n", i, window);
          return 1;
        }
    }
    checked += hi - lo;
    lo = hi;
  }
  std::printf("%zu cases\nOK\n", checked);
  return 0;
}
