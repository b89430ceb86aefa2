/*
 * ORACLE — test infrastructure only (see machine.h header).  PARITY UNPINNED
 * against a running reference; pinned by derivable KATs only.
 *
 * DDMin with RandomScheduler as the TestOracle (RunnerUtils.randomDDMin, RunnerUtils.scala:601-623).  This file
 * includes ddmin.c so that the minimizer is the same DDMin restatement as the STSSched one; a test is N executions of
 * the machine of machine.c.  It replaces ddmin.c in the random-oracle build of the oracle (random_ddmin.mk,
 * liboracle_random_ddmin.so).
 */
#include "ddmin.c"
#include <pthread.h>

typedef struct {
  int32_t  first_hit;         /* lowest j with status 0 and a violation, -1 = none              */
  uint32_t executions_run;    /* first_hit + 1, or N                                            */
  uint32_t violation;
  uint16_t status;            /* first nonzero status among executions 0..executions_run-1      */
  uint16_t reserved;
} oracle_random_rec;

/* RandomScheduler.test(subsequence) (RandomScheduler.scala:597-612) over explore (:234-272): execution j runs
 * FullyRandom(seed_base + j), j < N = p->n_prefixes, and explore returns at the first execution that finds the
 * violation.  The subsequence is the program's events the mask keeps, as written. */
static void random_test(const demi_config* cfg, const demi_ext_event* ext, uint32_t n_ext, const uint64_t* mask,
                        const demi_fuzz_params* p, demi_ext_event* buf, om_machine* scratch, oracle_random_rec* out) {
  uint32_t n = 0;
  for (uint32_t i = 0; i < n_ext; i++) if (bit(mask, i)) buf[n++] = ext[i];
  memset(out, 0, sizeof(*out));
  out->first_hit = -1;
  out->executions_run = (uint32_t)p->n_prefixes;
  for (uint32_t j = 0; j < (uint32_t)p->n_prefixes; j++) {
    demi_fuzz_result r;
    oracle_run_prefix(cfg, buf, n, p, jr_seed_at(p->seed_base, j), &r, NULL, 0, NULL, 0, scratch);
    if (r.status && !out->status) out->status = r.status;
    if (!r.status && r.violation) { out->first_hit = (int32_t)j; out->executions_run = j + 1; out->violation = r.violation; return; }
  }
}

typedef struct {
  const demi_config* cfg; const demi_ext_event* ext; uint32_t n_ext; const uint64_t* masks; uint32_t mw;
  const demi_fuzz_params* p; oracle_random_rec* out; uint32_t lo, hi;
} rt_job;
static void* rt_worker(void* a) {
  rt_job* j = (rt_job*)a;
  om_machine* m = (om_machine*)malloc(sizeof(om_machine));
  demi_ext_event* buf = (demi_ext_event*)malloc(sizeof(demi_ext_event) * (j->n_ext + 1));
  for (uint32_t t = j->lo; t < j->hi; t++) random_test(j->cfg, j->ext, j->n_ext, j->masks + (size_t)t * j->mw, j->p, buf, m, &j->out[t]);
  free(buf); free(m);
  return NULL;
}
/* n_tests tests over `threads` host threads (static block partition) */
int oracle_random_test_batch(const demi_config* cfg, const demi_ext_event* ext, uint32_t n_ext, const uint64_t* masks,
                             uint32_t n_tests, uint32_t mw, const demi_fuzz_params* p, oracle_random_rec* out, int threads) {
  if (threads < 1) threads = 1;
  if ((uint32_t)threads > n_tests) threads = n_tests ? (int)n_tests : 1;
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)threads);
  rt_job* jobs = (rt_job*)malloc(sizeof(rt_job) * (size_t)threads);
  for (int k = 0; k < threads; k++) {
    rt_job jb = { cfg, ext, n_ext, masks, mw, p, out, (uint32_t)((uint64_t)n_tests * k / threads),
                  (uint32_t)((uint64_t)n_tests * (k + 1) / threads) };
    jobs[k] = jb;
    pthread_create(&th[k], NULL, rt_worker, &jobs[k]);
  }
  for (int k = 0; k < threads; k++) pthread_join(th[k], NULL);
  free(th); free(jobs);
  return 0;
}

typedef struct {
  const demi_config* cfg; const demi_ext_event* ext; uint32_t n_ext; const demi_fuzz_params* p;
  demi_ext_event* buf; om_machine* scratch;
  int skip;                                               /* the unmodified check: not counted (_stats.reset(), :48) */
  oracle_random_rec* recs; uint64_t* keys; uint32_t cap, n_tests; uint64_t total;
  int error;
} rdd_ctx;
static int rdd_test(void* ctx, const uint64_t* mask) {
  rdd_ctx* c = (rdd_ctx*)ctx;
  oracle_random_rec r;
  random_test(c->cfg, c->ext, c->n_ext, mask, c->p, c->buf, c->scratch, &r);
  if (r.status) c->error = 1;
  if (c->skip) { c->skip = 0; } else {
    c->total += r.executions_run;
    if (c->n_tests < c->cap) { if (c->recs) c->recs[c->n_tests] = r; if (c->keys) c->keys[c->n_tests] = c->total; }
    c->n_tests++;
  }
  return r.status == 0 && r.first_hit >= 0;
}

/* DDMin.minimize over the whole program (WaitQuiescence included) with RandomScheduler.test as the oracle, then
 * verify_mcs when the MCS is shorter than the program.  test_log / recs: the tests of the sequential walk, in order
 * (the check_unmodified test excluded), at most min(cap_log, cap_iter) of them; iter_sizes[i] is keyed by iter_keys[i], the running sum of executions_run
 * (MinimizationStats.total_replays counts executions).  Returns 0, -1 on "Unmodified trace does not trigger
 * violation", -2 on malformed atoms, -3 on too many events, -4 when a test the walk consumed reported a status. */
int oracle_random_ddmin(const demi_config* cfg, const demi_ext_event* ext, uint32_t n_ext, const demi_fuzz_params* p,
                        int check_unmodified, uint64_t* mcs, uint32_t mw, uint64_t* test_log, oracle_random_rec* recs,
                        uint32_t cap_log, uint32_t* n_tests, uint32_t* iter_sizes, uint64_t* iter_keys, uint32_t cap_iter,
                        uint32_t* n_iter, uint64_t* total_replays, int* verified) {
  if (mw > MW_MAX || (uint64_t)mw * 64 < n_ext) return -3;
  rdd_ctx c; memset(&c, 0, sizeof(c));
  c.cfg = cfg; c.ext = ext; c.n_ext = n_ext; c.p = p;
  c.buf = (demi_ext_event*)malloc(sizeof(demi_ext_event) * (n_ext + 1));
  c.scratch = (om_machine*)malloc(sizeof(om_machine));
  c.skip = check_unmodified; c.recs = recs; c.keys = iter_keys; c.cap = cap_iter < cap_log ? cap_iter : cap_log;
  ddmin_t d; memset(&d, 0, sizeof(d));
  d.ext = ext; d.n_ext = n_ext; d.mw = mw; d.test = rdd_test; d.ctx = &c;
  d.iter_sizes = iter_sizes; d.cap_iter = cap_iter; d.test_log = test_log; d.cap_log = cap_log;
  uint64_t dag[MW_MAX];
  memset(dag, 0, sizeof(dag));
  for (uint32_t i = 0; i < n_ext; i++) setbit(dag, i);
  int rc = ddmin_minimize(&d, dag, check_unmodified, mcs);
  if (rc == 0 && c.error) rc = -4;
  if (iter_keys && c.n_tests < cap_iter) iter_keys[c.n_tests] = c.total;     /* the fencepost's key */
  if (n_tests) *n_tests = c.n_tests;
  if (n_iter) *n_iter = d.n_iter;
  if (total_replays) *total_replays = c.total;
  if (verified) {
    *verified = 0;
    if (rc == 0) {
      if (popcount_mask(mcs, mw) < n_ext) {                              /* verify_mcs (RunnerUtils.scala:612-620) */
        oracle_random_rec r;
        random_test(cfg, ext, n_ext, mcs, p, c.buf, c.scratch, &r);
        if (r.status) rc = -4;
        *verified = r.status == 0 && r.first_hit >= 0;
      } else {
        *verified = 1;                                                   /* nothing pruned: the original trace stands */
      }
    }
  }
  free(c.buf); free(c.scratch);
  return rc;
}
