/*
 * ORACLE — test infrastructure only (see machine.h header).
 *
 * Batch driver (the CPU baseline: RunnerUtils.fuzz's loop of independent
 * RandomScheduler executions, RunnerUtils.scala:75-91, one per seed) and small
 * known-answer entry points used by tests/test_oracle_kat.py.
 */
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include "machine.h"

typedef struct {
  const demi_config* cfg; const demi_ext_event* ext; uint32_t n_ext;
  const demi_fuzz_params* p; demi_fuzz_result* out; uint64_t lo, hi;
} fuzz_job;

static void* fuzz_worker(void* arg) {
  fuzz_job* j = (fuzz_job*)arg;
  om_machine* m = (om_machine*)malloc(sizeof(om_machine));
  for (uint64_t i = j->lo; i < j->hi; i++)
    oracle_run_prefix(j->cfg, j->ext, j->n_ext, j->p, jr_seed_at(j->p->seed_base, i),
                      &j->out[i], 0, 0, 0, 0, m);
  free(m);
  return 0;
}

int oracle_fuzz_batch(const demi_config* cfg, const demi_ext_event* ext, uint32_t n_ext,
                      const demi_fuzz_params* p, demi_fuzz_result* out, int threads) {
  if (!oracle_get_model(cfg->model)) return DEMI_ERR_INVALID;
  if (threads < 1) threads = 1;
  if (threads > 256) threads = 256;
  pthread_t tid[256];
  fuzz_job jobs[256];
  uint64_t n = p->n_prefixes, per = (n + (uint64_t)threads - 1) / (uint64_t)threads;
  int started = 0;
  for (int t = 0; t < threads; t++) {
    uint64_t lo = per * (uint64_t)t, hi = lo + per;
    if (lo >= n) break;
    if (hi > n) hi = n;
    jobs[t].cfg = cfg; jobs[t].ext = ext; jobs[t].n_ext = n_ext; jobs[t].p = p; jobs[t].out = out;
    jobs[t].lo = lo; jobs[t].hi = hi;
    pthread_create(&tid[t], 0, fuzz_worker, &jobs[t]);
    started++;
  }
  for (int t = 0; t < started; t++) pthread_join(tid[t], 0);
  return DEMI_OK;
}

/* Single-prefix recording run (for EventTrace / dep-tree parity). */
int oracle_fuzz_trace(const demi_config* cfg, const demi_ext_event* ext, uint32_t n_ext,
                      const demi_fuzz_params* p, int64_t seed,
                      demi_event* events, uint32_t cap_events, uint32_t* n_events,
                      uint16_t* dep_parent, uint32_t cap_nodes, uint32_t* n_nodes,
                      demi_fuzz_result* result) {
  if (!oracle_get_model(cfg->model)) return DEMI_ERR_INVALID;
  demi_fuzz_result r;
  om_machine* m = (om_machine*)malloc(sizeof(om_machine));
  if (!m) return DEMI_ERR_INVALID;
  oracle_run_prefix(cfg, ext, n_ext, p, seed, &r, events, cap_events, dep_parent, cap_nodes, m);
  if (n_events) *n_events = r.status ? r.n_events : m->n_events;   /* the whole trace: r.n_events saturates at 65535 */
  free(m);
  if (n_nodes) *n_nodes = r.n_nodes;
  if (result) *result = r;
  return r.status ? DEMI_ERR_CAPACITY : DEMI_OK;
}

/* ------------------------------------------------------------------- KATs */
uint64_t oracle_jr_rejections;
uint64_t oracle_jrandom_rejections(void) { return __atomic_load_n(&oracle_jr_rejections, __ATOMIC_RELAXED); }
void oracle_jrandom_reset_rejections(void) { __atomic_store_n(&oracle_jr_rejections, 0, __ATOMIC_RELAXED); }


/* java.util.Random: out[i] = nextInt() if bound <= 0 else nextInt(bound) */
void oracle_kat_jrandom(int64_t seed, int32_t bound, int32_t n, int32_t* out) {
  jrandom r; jr_seed(&r, seed);
  for (int i = 0; i < n; i++) out[i] = bound > 0 ? jr_next_int_bound(&r, bound) : jr_next_int(&r);
}

/* RandomizedHashSet script.  ops[i]: >=0 -> insert element with tag ops[i]
 * (tag stored in p0, receiver = tag & 31); -1 -> removeRandomElement;
 * -2 -> find_non_blocked_message with blocked_mask; -(1000+k) -> remove the
 * element at array index k (RandomizedHashSet.remove).  After the script,
 * `arr_out` receives the tags in array order, `removed_out` the tags returned by
 * the remove ops in order (-1 for None).  Returns the final array length. */
int oracle_kat_hashset(int64_t seed, uint32_t blocked_mask, const int32_t* ops, int32_t n_ops,
                       int32_t* arr_out, int32_t* removed_out, int32_t* n_removed) {
  om_machine* m = (om_machine*)calloc(1, sizeof(om_machine));
  m->pending_cap = OM_MAX_PENDING;
  m->blocked_mask = blocked_mask;
  jr_seed(&m->rng, seed);
  int nr = 0;
  for (int i = 0; i < n_ops; i++) {
    int32_t op = ops[i];
    if (op >= 0) {
      om_pending e; memset(&e, 0, sizeof(e));
      e.msg.dst = (uint8_t)(op & 31); e.msg.p0 = (uint32_t)op;
      om_pending_insert(m, &e);
    } else if (op == -1) {
      om_pending e = om_pending_remove_random(m);
      removed_out[nr++] = (int32_t)e.msg.p0;
    } else if (op == -2) {
      om_pending e;
      removed_out[nr++] = om_find_non_blocked(m, &e) ? (int32_t)e.msg.p0 : -1;
    } else if (op <= -1000) {
      uint32_t k = (uint32_t)(-op - 1000);
      om_pending v = m->pending[k];
      m->pending[k] = m->pending[m->n_pending - 1];
      m->n_pending--;
      removed_out[nr++] = (int32_t)v.msg.p0;
    }
  }
  int len = (int)m->n_pending;
  for (int i = 0; i < len; i++) arr_out[i] = (int32_t)m->pending[i].msg.p0;
  *n_removed = nr;
  free(m);
  return len;
}

size_t oracle_sizeof_machine(void) { return sizeof(om_machine); }
