/*
 * ORACLE — test infrastructure only (see machine.h header).
 *
 * The seeded Fuzzer (fuzzing/Fuzzer.scala:24-194) restated in C from the Scala source, and the CPU campaign: the
 * loop of RunnerUtils.fuzz (RunnerUtils.scala:75-91) as written, a new `fuzzer.generateFuzzTest()` per execution,
 * then one RandomScheduler execution of it.  Execution i draws its program with seed program_seed_base + i (the
 * Fuzzer, Fuzzer.scala:67-68, and its three RandomizedHashSets, Util.scala:110-115, all take it in place of the wall
 * clock) and runs under FullyRandom(seed_base + i).  Independent of the engine's fuzzer_gen.cuh: its own check is
 * the Python restatement in demi_b200/fuzzer.py.
 */
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include "machine.h"

/* RandomizedHashSet[T] (Util.scala:110-185): an ArrayBuffer plus its own Random */
typedef struct { uint32_t* arr; uint32_t len; jrandom rand; } rhs;

static void rhs_init(rhs* s, uint32_t* storage, int64_t seed) { s->arr = storage; s->len = 0; jr_seed(&s->rand, seed); }
static void rhs_insert(rhs* s, uint32_t v) { s->arr[s->len++] = v; }
/* removeRandomElement (:171-176): remove(arr(rand.nextInt(arr.length))), remove = swap the last element in (:146-163) */
static uint32_t rhs_remove_random(rhs* s) {
  int32_t i = jr_next_int_bound(&s->rand, (int32_t)s->len);
  uint32_t v = s->arr[i];
  s->arr[i] = s->arr[s->len - 1];
  s->len--;
  return v;
}
/* getRandomElement (:178-183).  On an empty set the reference throws (nextInt(0)); nextInt(0) as restated draws
 * index 0, which still holds the element removed last — the engine's defined behaviour, kept here. */
static uint32_t rhs_get_random(rhs* s) { return s->arr[jr_next_int_bound(&s->rand, (int32_t)s->len)]; }

/* java.util.Random.nextDouble */
static double jr_next_double(jrandom* r) {
  int64_t hi = (int64_t)jr_next(r, 26), lo = (int64_t)jr_next(r, 27);
  return (double)((hi << 27) + lo) * (1.0 / (double)(1LL << 53));
}

enum { GEN_NONE = 0, GEN_KILL, GEN_SEND, GEN_PARTITION, GEN_UNPARTITION, GEN_WAIT };

typedef struct {
  const demi_fuzzer_config* cfg;
  jrandom rand;
  rhs alive, partitioned, unpartitioned;
  uint32_t counter;      /* ClientCommandGenerator's running counter: a fresh generator per program */
  uint32_t next_id;      /* UniqueExternalEvent ids: every event object the generator creates takes the next one */
} fz_state;

/* FuzzerWeights.getNextEventType (Fuzzer.scala:43-57): allWeights = kill, send, partition, unpartition */
static int next_event_type(const demi_fuzzer_config* c, double r) {
  const double w[4] = {c->kill, c->send, c->partition, c->unpartition};
  const int t[4] = {GEN_KILL, GEN_SEND, GEN_PARTITION, GEN_UNPARTITION};
  double total = c->kill + c->send + c->partition + c->unpartition + c->wait_quiescence;
  double scaled = r * total, current = 0.0;
  for (int k = 0; k < 4; k++) {
    current = current + w[k];
    if (scaled < current) return t[k];
  }
  return GEN_WAIT;
}

static demi_ext_event new_event(fz_state* f, uint8_t kind, uint32_t a, uint32_t b, uint32_t type, uint32_t p0) {
  demi_ext_event e;
  memset(&e, 0, sizeof(e));
  e.kind = kind; e.a = (uint8_t)a; e.b = (uint8_t)b; e.type = (uint8_t)type; e.p0 = p0;
  e.id = ++f->next_id;
  return e;
}

/* generateNextEvent (Fuzzer.scala:84-121); returns 0 for None */
static int generate_next_event(fz_state* f, demi_ext_event* out) {
  for (;;) {
    switch (next_event_type(f->cfg, jr_next_double(&f->rand))) {
      case GEN_KILL:
        if (f->alive.len == 0) return 0;
        *out = new_event(f, DEMI_EXT_KILL, rhs_remove_random(&f->alive), 0, 0, 0);
        return 1;
      case GEN_SEND: {
        uint32_t dst = rhs_get_random(&f->alive);
        f->counter++;
        *out = new_event(f, DEMI_EXT_SEND, dst, 0, f->cfg->send_type, f->counter);
        return 1;
      }
      case GEN_PARTITION: {
        if (f->unpartitioned.len == 0) continue;                 /* "Try again..." */
        uint32_t pair = rhs_remove_random(&f->unpartitioned);
        rhs_insert(&f->partitioned, pair);
        *out = new_event(f, DEMI_EXT_PARTITION, pair >> 16, pair & 0xFFFF, 0, 0);
        return 1;
      }
      case GEN_UNPARTITION: {
        if (f->partitioned.len == 0) continue;
        uint32_t pair = rhs_remove_random(&f->partitioned);
        rhs_insert(&f->unpartitioned, pair);
        *out = new_event(f, DEMI_EXT_UNPARTITION, pair >> 16, pair & 0xFFFF, 0, 0);
        return 1;
      }
      default:
        *out = new_event(f, DEMI_EXT_WAIT_QUIESCENCE, 0, 0, 0, 0);
        return 1;
    }
  }
}

/* generateFuzzTest (Fuzzer.scala:123-174) after reset (:176-193).  `out` has room for n_prefix + num_events +
 * n_postfix + 1 events; returns the program's length. */
uint32_t oracle_fuzzer_generate(const demi_fuzzer_config* cfg, int64_t seed, const demi_ext_event* prefix, uint32_t n_prefix,
                                const demi_ext_event* postfix, uint32_t n_postfix, demi_ext_event* out) {
  uint32_t nodes[256], n_nodes = 0;
  for (uint32_t i = 0; i < n_prefix; i++)
    if (prefix[i].kind == DEMI_EXT_START && n_nodes < 256) nodes[n_nodes++] = prefix[i].a;
  const uint32_t pairs = n_nodes * (n_nodes > 0 ? n_nodes - 1 : 0) / 2;
  uint32_t* store = (uint32_t*)malloc(sizeof(uint32_t) * (n_nodes + 2 * pairs + 1));
  fz_state f;
  f.cfg = cfg; f.counter = 0; f.next_id = 0;
  for (uint32_t i = 0; i < n_prefix; i++) if (prefix[i].id > f.next_id) f.next_id = prefix[i].id;
  for (uint32_t i = 0; i < n_postfix; i++) if (postfix[i].id > f.next_id) f.next_id = postfix[i].id;
  jr_seed(&f.rand, seed);
  rhs_init(&f.alive, store, seed);
  for (uint32_t i = 0; i < n_nodes; i++) rhs_insert(&f.alive, nodes[i]);
  rhs_init(&f.partitioned, store + n_nodes, seed);
  rhs_init(&f.unpartitioned, store + n_nodes + pairs, seed);
  for (uint32_t i = 0; i < n_nodes; i++)
    for (uint32_t j = i + 1; j < n_nodes; j++) rhs_insert(&f.unpartitioned, (nodes[i] << 16) | nodes[j]);
  uint32_t len = 0;
  memcpy(out, prefix, sizeof(demi_ext_event) * n_prefix);
  len = n_prefix;
  int just_wq = len > 0 && out[len - 1].kind == DEMI_EXT_WAIT_QUIESCENCE;
  for (uint32_t i = 0; i < cfg->num_events; i++) {
    demi_ext_event ev;
    int some = generate_next_event(&f, &ev);
    while (some && ev.kind == DEMI_EXT_WAIT_QUIESCENCE && just_wq) some = generate_next_event(&f, &ev);
    if (!some) { free(store); return len; }                      /* no postfix, no final WaitQuiescence */
    just_wq = ev.kind == DEMI_EXT_WAIT_QUIESCENCE;
    out[len++] = ev;
  }
  memcpy(out + len, postfix, sizeof(demi_ext_event) * n_postfix);
  len += n_postfix;
  if (len > 0 && out[len - 1].kind != DEMI_EXT_WAIT_QUIESCENCE) out[len++] = new_event(&f, DEMI_EXT_WAIT_QUIESCENCE, 0, 0, 0, 0);
  free(store);
  return len;
}

typedef struct {
  const demi_config* cfg; const demi_fuzzer_config* fz;
  const demi_ext_event* prefix; uint32_t n_prefix; const demi_ext_event* postfix; uint32_t n_postfix;
  const demi_fuzz_params* p; int64_t program_seed_base; demi_fuzz_result* out; uint64_t lo, hi;
} campaign_job;

static void* campaign_worker(void* arg) {
  campaign_job* j = (campaign_job*)arg;
  om_machine* m = (om_machine*)malloc(sizeof(om_machine));
  demi_ext_event* prog = (demi_ext_event*)malloc(sizeof(demi_ext_event) * (j->n_prefix + j->fz->num_events + j->n_postfix + 1));
  for (uint64_t i = j->lo; i < j->hi; i++) {
    uint32_t n = oracle_fuzzer_generate(j->fz, jr_seed_at(j->program_seed_base, i), j->prefix, j->n_prefix, j->postfix, j->n_postfix, prog);
    oracle_run_prefix(j->cfg, prog, n, j->p, jr_seed_at(j->p->seed_base, i), &j->out[i], 0, 0, 0, 0, m);
  }
  free(prog);
  free(m);
  return 0;
}

/* p->n_prefixes executions on `threads` threads, split like oracle_fuzz_batch */
int oracle_fuzz_campaign(const demi_config* cfg, const demi_fuzzer_config* fz, const demi_ext_event* prefix, uint32_t n_prefix,
                         const demi_ext_event* postfix, uint32_t n_postfix, const demi_fuzz_params* p, int64_t program_seed_base,
                         demi_fuzz_result* out, int threads) {
  if (!oracle_get_model(cfg->model)) return DEMI_ERR_INVALID;
  if (threads < 1) threads = 1;
  if (threads > 256) threads = 256;
  pthread_t tid[256];
  campaign_job jobs[256];
  uint64_t n = p->n_prefixes, per = (n + (uint64_t)threads - 1) / (uint64_t)threads;
  int started = 0;
  for (int t = 0; t < threads; t++) {
    uint64_t lo = per * (uint64_t)t, hi = lo + per;
    if (lo >= n) break;
    if (hi > n) hi = n;
    campaign_job* j = &jobs[t];
    j->cfg = cfg; j->fz = fz; j->prefix = prefix; j->n_prefix = n_prefix; j->postfix = postfix; j->n_postfix = n_postfix;
    j->p = p; j->program_seed_base = program_seed_base; j->out = out; j->lo = lo; j->hi = hi;
    pthread_create(&tid[t], 0, campaign_worker, j);
    started++;
  }
  for (int t = 0; t < started; t++) pthread_join(tid[t], 0);
  return DEMI_OK;
}
