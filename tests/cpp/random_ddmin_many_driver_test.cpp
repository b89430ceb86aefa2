// RandomDDMinDriver (demi_b200/csrc/random_ddmin_driver.hpp) host-only, as demi_random_ddmin_many runs it: many
// drivers on threads at once behind the shared rendezvous (many_rendezvous.hpp), every round's requests served together
// by the CPU oracle's random-oracle tests (oracle_random_test_batch, one test per call, each under its trace's own
// program and parameters).  Built with AddressSanitizer.  Each trace's MCS, iteration sizes and keys, tests,
// total_replays and verified must equal oracle_random_ddmin's, and its whole demi_random_ddmin_out must equal that of
// its driver run alone, for every window.
//
// Input (argv[1]): little-endian uint32 words: n_cases, then per case model, model_flags, n_execs, seed (low, high),
// max_messages, interval, looking_for, check_unmodified, n_blob_bytes, the blob (padded to words), n_ext, n_ext x 4
// words.  Consecutive cases with the same model and blob form a group, minimised in one rendezvous.  Prints "OK" at
// the end.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "../../include/demi_b200.h"
extern "C" {
int oracle_random_test_batch(const demi_config* cfg, const demi_ext_event* ext, uint32_t n_ext, const uint64_t* masks,
                             uint32_t n_tests, uint32_t mw, const demi_fuzz_params* p, demi_random_test_result* out, int threads);
int oracle_random_ddmin(const demi_config* cfg, const demi_ext_event* ext, uint32_t n_ext, const demi_fuzz_params* p,
                        int check_unmodified, uint64_t* mcs, uint32_t mw, uint64_t* test_log, demi_random_test_result* recs,
                        uint32_t cap_log, uint32_t* n_tests, uint32_t* iter_sizes, uint64_t* iter_keys, uint32_t cap_iter,
                        uint32_t* n_iter, uint64_t* total_replays, int* verified);
int oracle_load_model(const void* blob, size_t size);
}
#include "../../demi_b200/csrc/random_ddmin_driver.hpp"
#include "../../demi_b200/csrc/many_rendezvous.hpp"

thread_local std::string g_create_error;

using namespace demi;

constexpr uint32_t CAP = 4096;

struct Case {
  demi_config cfg{}; demi_fuzz_params p{}; uint32_t check_unmodified = 0;
  std::vector<uint32_t> blob; uint32_t blob_bytes = 0;
  std::vector<demi_ext_event> ext;
  uint32_t mw() const { return ext.size() ? (uint32_t)(ext.size() + 63) / 64 : 1u; }
};

// the records of n tests of case c; every execution the oracle runs counts as one that ran
static void run_tests(const Case& c, const uint64_t* masks, size_t n, demi_random_test_result* res, uint64_t* executed) {
  oracle_random_test_batch(&c.cfg, c.ext.data(), (uint32_t)c.ext.size(), masks, (uint32_t)n, c.mw(), &c.p, res, 1);
  *executed = 0;
  for (size_t k = 0; k < n; k++) *executed += res[k].executions_run;
}

struct SoloDriver : RandomDDMinDriver {
  const Case* c;
  int32_t run_tests(const uint64_t* masks, size_t n, demi_random_test_result* res, uint64_t* executed) override {
    ::run_tests(*c, masks, n, res, executed);
    return DEMI_OK;
  }
};

struct Rec { demi_random_test_result rec; uint32_t ran; };

struct ManyDriver : RandomDDMinDriver {
  Rendezvous<Rec>* R; uint32_t trace;
  int32_t run_tests(const uint64_t* masks, size_t n, demi_random_test_result* res, uint64_t* executed) override {
    ManyRequest<Rec> q;
    q.trace = trace; q.masks = masks; q.n = n;
    R->submit(q);
    if (q.rc != DEMI_OK) return q.rc;
    *executed = 0;
    for (size_t k = 0; k < n; k++) { res[k] = q.res[k].rec; *executed += q.res[k].ran; }
    return DEMI_OK;
  }
};

template <class D> static void setup(D& d, demi_handle* h, const Case& c) {
  d.h = h; d.looking_for = c.p.looking_for; d.flags = 0; d.mw = c.mw(); d.n_ext = (uint32_t)c.ext.size(); d.ext = c.ext.data();
  d.set_width(c.p.n_prefixes);
}

struct Outcome {
  int32_t status = 0; std::vector<uint64_t> mcs; std::vector<uint32_t> sizes; std::vector<uint64_t> keys;
  demi_random_ddmin_out out{};
  bool operator==(const Outcome& o) const {
    return status == o.status && mcs == o.mcs && sizes == o.sizes && keys == o.keys && !memcmp(&out, &o.out, sizeof(out));
  }
};

static int32_t minimize(RandomDDMinDriver& d, const Case& c, Outcome& r) {
  r.mcs.assign(c.mw(), 0); r.sizes.assign(CAP, 0); r.keys.assign(CAP, 0);
  r.status = d.minimize(c.check_unmodified != 0, r.mcs.data(), r.sizes.data(), r.keys.data(), CAP, &r.out);
  r.sizes.resize(std::min(r.out.n_iterations, CAP)); r.keys.resize(std::min(r.out.n_iterations, CAP));
  return r.status;
}

static Outcome solo(const Case& c) {
  demi_handle eh;
  SoloDriver d;
  setup(d, &eh, c);
  d.c = &c;
  Outcome r;
  minimize(d, c, r);
  return r;
}

static std::vector<Outcome> many(const std::vector<Case>& cs, size_t lo, size_t hi, uint32_t window) {
  const uint32_t n = (uint32_t)(hi - lo);
  std::vector<Outcome> r(n);
  std::vector<int32_t> status(n, -1);
  auto drive = [&](uint32_t t, Rendezvous<Rec>& R, demi_handle* eh) -> int32_t {
    ManyDriver d;
    setup(d, eh, cs[lo + t]);
    d.R = &R; d.trace = t;
    return minimize(d, cs[lo + t], r[t]);
  };
  auto serve = [&](std::vector<ManyRequest<Rec>*>& batch) -> int32_t {
    for (ManyRequest<Rec>* q : batch) {
      std::vector<demi_random_test_result> res(q->n);
      uint64_t executed;
      q->res.resize(q->n);
      for (size_t k = 0; k < q->n; k++) {          // one test at a time: each test's own count of executions
        run_tests(cs[lo + q->trace], q->masks + k * cs[lo + q->trace].mw(), 1, &res[k], &executed);
        q->res[k] = Rec{res[k], (uint32_t)executed};
      }
    }
    return DEMI_OK;
  };
  demi_handle h;
  const int32_t rc = run_many<Rec>(&h, "random_ddmin_many_driver_test", n, window, drive, serve, status.data());
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
    c.cfg.model = (int32_t)w[p++]; c.cfg.model_flags = w[p++];
    c.p.n_prefixes = w[p++];
    const uint64_t lo = w[p++], hi = w[p++];
    c.p.seed_base = (int64_t)(lo | (hi << 32));
    c.p.max_messages = (int32_t)w[p++]; c.p.invariant_check_interval = (int32_t)w[p++]; c.p.looking_for = w[p++];
    c.check_unmodified = w[p++];
    c.blob_bytes = w[p++];
    c.blob.resize((c.blob_bytes + 3) / 4); take(c.blob.data(), c.blob.size());
    c.ext.resize(w[p++]); take(c.ext.data(), c.ext.size() * 4);
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
      std::vector<uint64_t> mcs(c.mw(), 0), keys(CAP, 0);
      std::vector<uint32_t> sizes(CAP, 0);
      uint32_t n_tests = 0, n_iter = 0;
      uint64_t total = 0;
      int verified = 0;
      const int rc = oracle_random_ddmin(&c.cfg, c.ext.data(), (uint32_t)c.ext.size(), &c.p, (int)c.check_unmodified, mcs.data(),
                                         c.mw(), nullptr, nullptr, CAP, &n_tests, sizes.data(), keys.data(), CAP, &n_iter, &total,
                                         &verified);
      sizes.resize(n_iter); keys.resize(n_iter);
      const Outcome& a = alone.back();
      if (rc != 0 || a.status != DEMI_OK || a.mcs != mcs || a.sizes != sizes || a.keys != keys || a.out.tests != n_tests ||
          a.out.total_replays != total || a.out.verified != (uint32_t)verified || a.out.n_iterations != n_iter) {
        std::printf("FAILED: case %zu alone differs from oracle_random_ddmin (rc %d status %d)\n", i, rc, a.status);
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
