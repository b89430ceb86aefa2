/*
 * ORACLE — test infrastructure only (see machine.h header).  PARITY UNPINNED
 * against a running reference; pinned by derivable KATs only.
 *
 * Fungible clocks, strictly sequential: WildcardMinimizer.minimize / doMinimize
 * (minification/wildcard_minimization/WildcardMinimizer.scala:133-241) with
 * testScheduler = STSSched and ClockClusterizer (ClockClusterizer.scala:39-134),
 * ClockClusterIterator (:138-228), OneAtATimeIterator (:230-290),
 * Aggressiveness.ALL_TIMERS_FIRST_ITR.  FingerprintFactory.getLogicalClock and
 * causesClockIncrement are the packed rules of demi_set_clock_rules (demi_b200.h).
 */
#include <stdlib.h>
#include <string.h>
#include "machine.h"
#include "sts_wildcard.h"
uint32_t oracle_ir_external_mask(void);
int oracle_model_key(int model);

#define WC_IDS 65536
typedef struct {
  /* originalTrace's UniqueMsgEvents in trace order */
  uint32_t n; uint16_t* id; uint8_t* incr; uint8_t* has_clock; uint32_t* clock;
  /* ClockClusterIterator */
  uint8_t all_ids[WC_IDS], cblack[WC_IDS];
  int first_cluster_removal; int64_t next_clock_to_remove;
  int64_t* clocks; uint32_t n_clocks;
  /* OneAtATimeIterator */
  uint8_t t_all[WC_IDS], tblack[WC_IDS];
  uint16_t* to_remove; uint32_t n_to_remove; int t_first;
  /* ClockClusterizer */
  uint8_t cur_cluster[WC_IDS], cur_timers[WC_IDS];
  int trying_first_cluster;
} wc_clusterizer;

static int cmp_i64(const void* a, const void* b) { int64_t x = *(const int64_t*)a, y = *(const int64_t*)b; return x < y ? -1 : x > y; }

static void compute_remaining_clocks(wc_clusterizer* c) {          /* :162-173 */
  const int64_t lowest = c->n_clocks ? c->clocks[0] : 0;
  int64_t* v = (int64_t*)malloc(sizeof(int64_t) * (c->n + 1));
  uint32_t k = 0;
  for (uint32_t j = 0; j < c->n; j++) if (!c->cblack[c->id[j]] && c->has_clock[j]) v[k++] = c->clock[j];
  qsort(v, k, sizeof(int64_t), cmp_i64);
  uint32_t m = 0;
  for (uint32_t j = 0; j < k; j++) {
    if (m && v[m - 1] == v[j]) continue;                           /* .toSet */
    v[m++] = v[j];
  }
  uint32_t s = 0;
  while (s < m && v[s] < lowest) s++;                              /* dropWhile(c => c < lowest) */
  free(c->clocks);
  c->clocks = (int64_t*)malloc(sizeof(int64_t) * (m - s + 1));
  memcpy(c->clocks, v + s, sizeof(int64_t) * (m - s));
  c->n_clocks = m - s;
  free(v);
}
static void cluster_current(const wc_clusterizer* c, uint8_t* out) {   /* :176-201 */
  const int64_t rm = c->first_cluster_removal ? -1 : c->next_clock_to_remove;
  memset(out, 0, WC_IDS);
  for (uint32_t j = 0; j < c->n; j++) {
    if (c->incr[j]) continue;                                      /* handled by OneAtATimeIterator */
    if (!c->has_clock[j]) { out[c->id[j]] = 1; continue; }
    if ((int64_t)c->clock[j] == rm || c->cblack[c->id[j]]) continue;
    out[c->id[j]] = 1;
  }
}
static void cluster_next(wc_clusterizer* c, uint8_t* out) {         /* :204-215 */
  if (c->first_cluster_removal) { cluster_current(c, out); c->first_cluster_removal = 0; return; }
  c->next_clock_to_remove = c->clocks[0];
  cluster_current(c, out);
  memmove(c->clocks, c->clocks + 1, sizeof(int64_t) * (c->n_clocks - 1));
  c->n_clocks--;
}
static int cluster_has_next(const wc_clusterizer* c) { return c->first_cluster_removal || c->n_clocks; }
static void cluster_produced(wc_clusterizer* c, const uint8_t* prev, const uint8_t* ign, int any_ign) {   /* :219-225 */
  for (uint32_t j = 0; j < c->n; j++) {
    const uint16_t id = c->id[j];
    if (c->all_ids[id] && !prev[id]) c->cblack[id] = 1;
  }
  if (any_ign) {
    for (uint32_t j = 0; j < c->n; j++) if (c->all_ids[c->id[j]] && ign[c->id[j]]) c->cblack[c->id[j]] = 1;
    compute_remaining_clocks(c);
  }
}
static void timers_current(const wc_clusterizer* c, uint8_t* out) {   /* :254-260 */
  memset(out, 0, WC_IDS);
  for (uint32_t j = 0; j < c->n; j++) {
    const uint16_t id = c->id[j];
    if (!c->t_all[id] || c->tblack[id]) continue;
    if (!c->t_first && id == c->to_remove[0]) continue;
    out[id] = 1;
  }
}
static void timers_next(wc_clusterizer* c, uint8_t* out) {           /* :263-273 */
  timers_current(c, out);
  if (c->t_first) c->t_first = 0;
  else { memmove(c->to_remove, c->to_remove + 1, sizeof(uint16_t) * (c->n_to_remove - 1)); c->n_to_remove--; }
}
static void timers_reset(wc_clusterizer* c) {                        /* :284-287: (all -- blacklist).toSeq.sorted */
  c->n_to_remove = 0;
  for (uint32_t id = 0; id < WC_IDS; id++) if (c->t_all[id] && !c->tblack[id]) c->to_remove[c->n_to_remove++] = (uint16_t)id;
  c->t_first = 1;
}

static wc_clusterizer* clusterizer_new(const demi_event* ev, uint32_t n_ev, const uint32_t* rule, const uint32_t* incr) {
  wc_clusterizer* c = (wc_clusterizer*)calloc(1, sizeof(wc_clusterizer));
  c->id = (uint16_t*)malloc(sizeof(uint16_t) * (n_ev + 1)); c->incr = (uint8_t*)malloc(n_ev + 1);
  c->has_clock = (uint8_t*)malloc(n_ev + 1); c->clock = (uint32_t*)malloc(sizeof(uint32_t) * (n_ev + 1));
  c->to_remove = (uint16_t*)malloc(sizeof(uint16_t) * (n_ev + 1));
  for (uint32_t i = 0; i < n_ev; i++) {
    const demi_event* e = &ev[i];
    if (e->kind != DEMI_EV_MSG_EVENT) continue;
    const uint32_t j = c->n++;
    c->id[j] = e->uniq;
    c->incr[j] = (uint8_t)((incr[e->type >> 5] >> (e->type & 31)) & 1u);
    const uint32_t r = rule[e->type];                              /* getLogicalClock */
    c->has_clock[j] = r != 0;
    if (r) {
      const uint32_t word = (r >> 8) & 0xFF, shift = (r >> 16) & 0xFF, bits = r >> 24;
      const uint32_t v = (word ? e->p1 : e->p0) >> shift;
      c->clock[j] = bits >= 32 ? v : (v & ((1u << bits) - 1u));
    }
    if (!c->incr[j] && c->has_clock[j]) c->all_ids[e->uniq] = 1;  /* allIds :139-150 */
    if (c->incr[j]) c->t_all[e->uniq] = 1;                         /* OneAtATimeIterator.fromTrace :231-242 */
  }
  c->first_cluster_removal = 1; c->next_clock_to_remove = -1;
  compute_remaining_clocks(c);                                     /* clocks = computeRemainingClocks :174 */
  c->n_to_remove = 0;
  for (uint32_t id = 0; id < WC_IDS; id++) if (c->t_all[id]) c->to_remove[c->n_to_remove++] = (uint16_t)id;   /* all.toSeq.sorted */
  c->t_first = 1;
  cluster_next(c, c->cur_cluster);                                 /* currentCluster = clusterIterator.next :57 */
  c->trying_first_cluster = 1;
  return c;
}
static void clusterizer_free(wc_clusterizer* c) {
  free(c->id); free(c->incr); free(c->has_clock); free(c->clock); free(c->to_remove); free(c->clocks); free(c);
}
/* getNextTrace (:73-134) as the include mask over the deliveries; 0 = None */
static int clusterizer_next(wc_clusterizer* c, int violation, const uint8_t* ign, int any_ign, uint64_t* mask) {
  if (violation) {
    for (uint32_t j = 0; j < c->n; j++) {                          /* timerIterator.producedViolation :279-282 */
      const uint16_t id = c->id[j];
      if (c->t_all[id] && (!c->cur_timers[id] || ign[id])) c->tblack[id] = 1;
    }
    cluster_produced(c, c->cur_cluster, ign, any_ign);
  }
  if (!(c->t_first || c->n_to_remove) || (violation && !c->trying_first_cluster)) {
    c->trying_first_cluster = 0;
    if (!cluster_has_next(c)) return 0;
    timers_reset(c);
    cluster_next(c, c->cur_cluster);
  }
  timers_next(c, c->cur_timers);
  memset(mask, 0, sizeof(uint64_t) * ((c->n + 63) / 64 + 1));
  for (uint32_t j = 0; j < c->n; j++)
    if (c->cur_timers[c->id[j]] || c->cur_cluster[c->id[j]]) mask[j >> 6] |= 1ull << (j & 63);
  return 1;
}

static void wc_input(const demi_config* cfg, const demi_event* ev, uint32_t n_ev, const demi_ext_event* ext, uint32_t n_ext,
                     demi_replay_input* in) {
  uint32_t n_deliv = 0, n_ext_sends = 0;
  for (uint32_t i = 0; i < n_ev; i++) n_deliv += ev[i].kind == DEMI_EV_MSG_EVENT;
  for (uint32_t i = 0; i < n_ext; i++) n_ext_sends += ext[i].kind == DEMI_EXT_SEND;
  in->events = ev; in->n_events = n_ev; in->externals = ext; in->n_externals = n_ext;
  in->external_type_mask = cfg->model == 100 ? oracle_ir_external_mask() : demi_external_type_mask(cfg->model);
  in->pending_cap = demi_wildcard_pending_cap(oracle_model_key(cfg->model), n_deliv, n_ext_sends);
  in->tosend_cap = demi_tosend_cap(n_ext_sends);
}

/* one wildcard STSScheduler.test with the shared capacity rules */
void oracle_wildcard_replay(const demi_config* cfg, const demi_event* ev, uint32_t n_ev, const demi_ext_event* ext, uint32_t n_ext,
                            const uint64_t* include, const uint32_t* incr, uint32_t looking_for, uint32_t flags,
                            demi_replay_result* out, demi_event* rec, uint32_t cap_rec, uint32_t* n_rec,
                            uint32_t* ignored, uint32_t cap_ignored, uint32_t* n_ignored) {
  demi_replay_input in;
  wc_input(cfg, ev, n_ev, ext, n_ext, &in);
  oracle_sts_replay_wild(cfg, &in, include, incr, looking_for, flags, out, rec, cap_rec, n_rec, ignored, cap_ignored, n_ignored);
}

/* The include masks getNextTrace(false, {}) yields from a fresh clusterizer, i.e. the tests issued if every test
 * fails; returns how many (at most cap). */
uint32_t oracle_wildcard_cluster_sequence(const demi_event* ev, uint32_t n_ev, const uint32_t* rule, const uint32_t* incr,
                                          const uint8_t* outcomes, uint32_t n_outcomes, const uint16_t* ign_ids,
                                          const uint32_t* ign_counts, uint64_t* masks, uint32_t mask_words, uint32_t cap) {
  /* outcomes[k] / ign_ids: the result of test k (violation, and then ign_counts[k] ids); tests beyond n_outcomes fail */
  wc_clusterizer* c = clusterizer_new(ev, n_ev, rule, incr);
  uint8_t* ign = (uint8_t*)calloc(WC_IDS, 1);
  uint64_t* m = (uint64_t*)malloc(sizeof(uint64_t) * ((c->n + 63) / 64 + 1));
  uint32_t k = 0, off = 0;
  int v = 0, any = 0;
  while (k < cap && clusterizer_next(c, v, ign, any, m)) {
    memcpy(masks + (size_t)k * mask_words, m, sizeof(uint64_t) * mask_words);
    memset(ign, 0, WC_IDS); any = 0;
    v = k < n_outcomes ? outcomes[k] : 0;
    const uint32_t ni = k < n_outcomes ? ign_counts[k] : 0;
    for (uint32_t q = 0; q < ni; q++) { ign[ign_ids[off + q]] = 1; any = 1; }
    off += ni;
    k++;
  }
  free(ign); free(m); clusterizer_free(c);
  return k;
}

int oracle_wildcard_minimize(const demi_config* cfg, const demi_event* verified, uint32_t n_verified,
                             const demi_ext_event* mcs_ext, uint32_t n_ext, const uint32_t* rule, const uint32_t* incr,
                             uint32_t looking_for, uint32_t flags,
                             demi_event* out_trace, uint32_t cap_out, uint32_t* n_out,
                             uint32_t* total_replays, uint32_t* internal_sizes, uint32_t cap_sizes, uint32_t* n_sizes) {
  wc_clusterizer* c = clusterizer_new(verified, n_verified, rule, incr);
  demi_event* min_trace = (demi_event*)malloc(sizeof(demi_event) * (n_verified + 1));
  memcpy(min_trace, verified, sizeof(demi_event) * n_verified);
  uint32_t n_min = n_verified;
  demi_event* rec = (demi_event*)malloc(sizeof(demi_event) * 65536);
  uint32_t* ign_pos = (uint32_t*)malloc(sizeof(uint32_t) * (n_verified + 1));
  uint8_t* ign = (uint8_t*)calloc(WC_IDS, 1);
  uint64_t* mask = (uint64_t*)malloc(sizeof(uint64_t) * ((c->n + 63) / 64 + 1));
  uint32_t replays = 0, ns = 0;
  int rc = 0;
  int has = clusterizer_next(c, 0, ign, 0, mask);                 /* doMinimize :193 */
  while (has) {
    demi_replay_result r; uint32_t n_rec = 0, n_ign = 0;
    oracle_wildcard_replay(cfg, verified, n_verified, mcs_ext, n_ext, mask, incr, looking_for, flags, &r,
                           rec, 65536, &n_rec, ign_pos, n_verified + 1, &n_ign);
    replays++;                                                     /* stats.increment_replays */
    if (r.status) { rc = -1; break; }
    uint32_t cnt = 0;
    for (uint32_t i = 0; i < n_min; i++) cnt += min_trace[i].kind == DEMI_EV_MSG_EVENT;
    if (internal_sizes && ns < cap_sizes) internal_sizes[ns] = cnt;   /* record_internal_size :210-212 */
    ns++;
    memset(ign, 0, WC_IDS);
    int any = 0;
    if (r.violation) {
      if (n_rec <= n_min) {                                        /* ret.get.size <= minTrace.size :217-219 */
        min_trace = (demi_event*)realloc(min_trace, sizeof(demi_event) * (n_rec + 1));
        memcpy(min_trace, rec, sizeof(demi_event) * n_rec);
        n_min = n_rec;
      }
      for (uint32_t q = 0; q < n_ign; q++) { ign[verified[ign_pos[q]].uniq] = 1; any = 1; }   /* ignoredAbsentIds :232-235 */
    }
    has = clusterizer_next(c, r.violation != 0, ign, any, mask);
  }
  if (!rc) {
    uint32_t cnt = 0;
    for (uint32_t i = 0; i < n_min; i++) cnt += min_trace[i].kind == DEMI_EV_MSG_EVENT;
    if (internal_sizes && ns < cap_sizes) internal_sizes[ns] = cnt;   /* fencepost :183-184 */
    ns++;
  }
  if (n_out) *n_out = n_min;
  if (out_trace) memcpy(out_trace, min_trace, sizeof(demi_event) * (n_min < cap_out ? n_min : cap_out));
  if (total_replays) *total_replays = replays;
  if (n_sizes) *n_sizes = ns;
  free(min_trace); free(rec); free(ign_pos); free(ign); free(mask); clusterizer_free(c);
  return rc;
}
