/*
 * ORACLE — test infrastructure only (see machine.h header).  PARITY UNPINNED
 * against a running reference; pinned by derivable KATs and, for width = 1, by
 * sequence equality with the sequential restatement in dpor.c.
 *
 * Frontier ("wide") DPOR: the CPU restatement of demi_dpor_frontier
 * (include/demi_b200.h).  Same algorithmic content as dpor.c — DPORwHeuristics
 * (schedulers/DPORwHeuristics.scala): schedule_new_message :421-648,
 * event_produced/getMessage :773-847, dpor :1020-1185 (isCoEnabeled :1091-1110,
 * analyze_dep :1043-1077, getCommonPrefix :994-1018, getNext :1142-1162),
 * DefaultBacktrackOrdering (BacktrackOrdering.scala:58-69), ExploredTacker
 * (AuxilaryTypes.scala:209-246) — with `width` backtrack points dequeued per
 * round and, for n_ranks > 1, the deterministic steal protocol the engine runs
 * over NCCL, simulated here rank by rank in one process.
 *
 * Everything is written sequentially and literally (linear scans, memmove
 * queues, a sorted array as the backtrack queue); the engine's data structures
 * are different, the observable results must be identical.
 */
#include <stdlib.h>
#include <string.h>
#include "machine.h"
#include "dpor.h"
#include "dpor_frontier.h"
int oracle_model_key(int model);

typedef struct { uint64_t ord, pk; } fkey;                          /* queue entry: order key, explored-set key of (later, earlier) */
typedef struct { uint64_t id; demi_msg msg; uint16_t ppos; } fpend;  /* a pending message and the position that created it */

typedef struct {
  /* explored ordered pairs.  The table is private and grows, so it never fills; `e_cap` (explored_slots) is the
   * engine's table, and a round after which n_E·2 ≥ e_cap ends the search with DEMI_DS_EXPLORED_OVF */
  uint64_t* E; uint64_t e_slots, n_E, e_cap; int no_history;   /* trackHistory = false (:86): the set stays empty */
  uint64_t* log; uint64_t n_log, cap_log, log_alloc;       /* pair keys marked since the last exchange (shared with the other ranks there) */
  /* trace store */
  demi_frontier_entry* tr; uint32_t* tr_len; uint32_t* tr_branch; uint32_t n_slots, cap_slots, T1;
  /* backtrack queue, ascending ord; pool_top = points enqueued + received so far, bounded by pool_cap (the arena) */
  fkey* pool; uint64_t n_pool, cap_pool, pool_top;
  demi_frontier_result R;
  demi_dpor_violation* viol; uint32_t cap_viol;
  uint64_t* hashes; uint64_t cap_hashes, n_hashes;
  uint32_t round_first_slot, round_n;                                /* the traces executed in the current round */
  /* the counters after the current round's getNext: a round that ends in a capacity status goes back to them */
  demi_frontier_result snap; uint32_t snap_slots; uint64_t snap_hashes, snap_E;
  int explored_fixed;                                                /* R.explored_pairs was set by a failed round */
} frank;

typedef struct {
  om_machine m;
  const demi_frontier_params* F;
  const demi_ext_event* ext; uint32_t n_ext;
  fpend* pend; uint32_t n_pend, cap_pend;
  uint32_t isolated;
  uint64_t parent_id; uint32_t cur_pos;
  demi_frontier_entry* cur; uint32_t cur_len;
  int32_t nsched;
  int status;
} fexec;

static __thread fexec* g_fx = 0;
int oracle_in_frontier_mode(void) { return g_fx != 0; }

/* --------------------------------------------------------- explored set */
static int e_has(const frank* r, uint64_t key) {
  if (r->no_history) return 0;
  uint64_t s = demi_fr_explored_slot(key, r->e_slots);
  while (r->E[s]) { if (r->E[s] == key) return 1; s = (s + 1) & (r->e_slots - 1); }
  return 0;
}
static void e_place(uint64_t* E, uint64_t slots, uint64_t key) {
  uint64_t s = demi_fr_explored_slot(key, slots);
  while (E[s]) s = (s + 1) & (slots - 1);
  E[s] = key;
}
static void e_add(frank* r, uint64_t key) {
  if (r->no_history) return;
  uint64_t s = demi_fr_explored_slot(key, r->e_slots);
  while (r->E[s]) { if (r->E[s] == key) return; s = (s + 1) & (r->e_slots - 1); }
  r->E[s] = key; r->n_E++;
  if (r->n_E * 2 >= r->e_slots) {                                         /* keep the private table at most half full */
    uint64_t* E2 = (uint64_t*)calloc(r->e_slots * 2, 8);
    for (uint64_t i = 0; i < r->e_slots; i++) if (r->E[i]) e_place(E2, r->e_slots * 2, r->E[i]);
    free(r->E); r->E = E2; r->e_slots *= 2;
  }
  if (r->log) {                                                           /* its capacity is checked after the round */
    if (r->n_log == r->log_alloc) { r->log_alloc *= 2; r->log = (uint64_t*)realloc(r->log, 8 * r->log_alloc); }
    r->log[r->n_log++] = key;
  }
}

/* --------------------------------------------- DPORwHeuristics.event_produced */
static int qorder(const fexec* x, const demi_msg* c) {                  /* canonical order of pendingEvents.find (:454-456) */
  return (int)((c->src == DEMI_DEADLETTERS ? (uint32_t)x->m.model->n_actors : c->src) * DEMI_MAX_ACTORS + c->dst);
}
static void f_event_produced(fexec* x, const demi_msg* msg) {           /* :803-847 after the cancelled-timer drop */
  om_machine* m = &x->m;
  if (x->status) return;
  for (uint32_t i = 0; i < m->n_cancelled; i++) {
    om_timer_key* k = &m->cancelled[i];
    if (k->dst == msg->dst && k->type == msg->type && k->p0 == msg->p0 && k->p1 == msg->p1) {
      for (uint32_t j = i; j + 1 < m->n_cancelled; j++) m->cancelled[j] = m->cancelled[j + 1];
      m->n_cancelled--;
      return;
    }
  }
  if (x->n_pend >= x->cap_pend) { x->status = DEMI_DS_QUEUE_OVF; return; }
  fpend* p = &x->pend[x->n_pend++];
  p->msg = *msg; p->msg.flags = 0;
  /* getMessage (:773-801): same parent + same (snd, rcv, fingerprint) = same Unique */
  p->id = demi_fr_child_id(x->parent_id, (uint32_t)msg->src | ((uint32_t)msg->dst << 8) | ((uint32_t)msg->type << 16), msg->p0, msg->p1);
  p->ppos = (uint16_t)x->cur_pos;
}
void front_om_send(om_machine* m, int src, int dst, uint8_t type, uint32_t p0, uint32_t p1) {
  (void)m;
  demi_msg msg; msg.src = (uint8_t)src; msg.dst = (uint8_t)dst; msg.type = type; msg.flags = 0; msg.p0 = p0; msg.p1 = p1;
  f_event_produced(g_fx, &msg);
}
void front_queue_overflow(void) { if (!g_fx->status) g_fx->status = DEMI_DS_QUEUE_OVF; }
/* enqueue_timer = enqueue_message, whatever ignoreTimers says (see dpor.c's dpor_timer_send) */
static void f_timer_send(fexec* x, int rcv, uint8_t type, uint32_t p0, uint32_t p1) {
  demi_msg t; t.src = DEMI_DEADLETTERS; t.dst = (uint8_t)rcv; t.type = type; t.flags = 0; t.p0 = p0; t.p1 = p1;
  f_event_produced(x, &t);
}
static int f_reg_find(const om_machine* m, int dst, uint8_t type, uint32_t p0, uint32_t p1) {
  for (uint32_t i = 0; i < m->n_registry; i++)
    if (m->registry[i].dst == dst && m->registry[i].type == type && m->registry[i].p0 == p0 && m->registry[i].p1 == p1) return (int)i;
  return -1;
}
void front_om_schedule(om_machine* m, int self, uint8_t type, uint32_t p0, uint32_t p1, int repeating) {
  fexec* x = g_fx;
  if (x->status) return;
  if (f_reg_find(m, self, type, p0, p1) >= 0) return;                     /* "Non-unique timer" */
  if (repeating) {
    if (m->n_registry >= DEMI_TIMERSET_CAP) { x->status = DEMI_DS_QUEUE_OVF; return; }
    om_timer_key* k = &m->registry[m->n_registry++];
    k->dst = (uint8_t)self; k->type = type; k->p0 = p0; k->p1 = p1;
  }
  f_timer_send(x, self, type, p0, p1);
}
void front_om_cancel(om_machine* m, int self, uint8_t type, uint32_t p0, uint32_t p1) {   /* notify_timer_cancel :961-985 */
  fexec* x = g_fx;
  if (x->status) return;
  int have = 0;
  for (uint32_t i = 0; i < m->n_cancelled; i++)
    if (m->cancelled[i].dst == self && m->cancelled[i].type == type && m->cancelled[i].p0 == p0 && m->cancelled[i].p1 == p1) have = 1;
  if (!have) {
    if (m->n_cancelled >= DEMI_TIMERSET_CAP) { x->status = DEMI_DS_QUEUE_OVF; return; }
    om_timer_key* k = &m->cancelled[m->n_cancelled++];
    k->dst = (uint8_t)self; k->type = type; k->p0 = p0; k->p1 = p1;
  }
  int ri = f_reg_find(m, self, type, p0, p1);
  if (ri >= 0) { for (uint32_t j = (uint32_t)ri; j + 1 < m->n_registry; j++) m->registry[j] = m->registry[j + 1]; m->n_registry--; }
  for (uint32_t i = 0; i < x->n_pend; i++) {
    const demi_msg* c = &x->pend[i].msg;
    if (c->src == DEMI_DEADLETTERS && c->dst == self && c->type == type && c->p0 == p0 && c->p1 == p1) {
      memmove(&x->pend[i], &x->pend[i + 1], sizeof(fpend) * (x->n_pend - i - 1));
      x->n_pend--;
      return;
    }
  }
}

/* One interleaving.  `kt`/`li`/`branch`/`ei`: the backtrack point (kt = NULL: no nextTrace, the first execution).
 * nextTrace = kt[1..branch] ++ (kt[branch+1..li] minus every entry whose id is kt[ei].id)   (:1060-1063, :1180) */
static uint32_t f_execute(fexec* x, const demi_frontier_entry* kt, uint32_t branch, uint32_t li, uint32_t ei, uint64_t* sched_hash) {
  om_machine* m = &x->m;
  memset(m->states, 0, sizeof(m->states));
  m->model->init(m->states, m->model_flags);
  m->n_registry = m->n_cancelled = 0;
  x->n_pend = 0;
  x->isolated = m->model->n_actors >= 32 ? 0xFFFFFFFFu : ((1u << m->model->n_actors) - 1u);
  x->cur_len = 0;
  memset(&x->cur[0], 0, sizeof(x->cur[0]));
  x->cur[0].id = DEMI_FR_ROOT_ID; x->cur[0].src = x->cur[0].dst = 0xFF; x->cur_len = 1;   /* currentTrace += root :343 */
  x->parent_id = DEMI_FR_ROOT_ID; x->cur_pos = 0;
  x->nsched = 0;
  uint64_t sh = 0;
  for (uint32_t i = 0; i < x->n_ext && !x->status; i++) {                  /* runExternal :684-721 */
    if (x->ext[i].kind == DEMI_EXT_START) x->isolated &= ~(1u << x->ext[i].a);
    else if (x->ext[i].kind == DEMI_EXT_SEND) {
      demi_msg s; s.src = DEMI_DEADLETTERS; s.dst = x->ext[i].a; s.type = x->ext[i].type; s.flags = 0; s.p0 = x->ext[i].p0; s.p1 = x->ext[i].p1;
      f_event_produced(x, &s);
    }
  }
  uint32_t np = 1;                                                          /* cursor in nextTrace (position in kt) */
  const uint64_t skip_id = kt ? kt[ei].id : 0;
  while (!x->status) {
    /* schedule_new_message :421-648 */
    x->nsched++;
    if (x->nsched > x->F->max_messages) break;                              /* :583-586 */
    int pick = -1;
    if (kt) {
      while (np <= li && np > branch && kt[np].id == skip_id) np++;         /* replayThis filters `earlier` out */
      if (np <= li) {
        const demi_frontier_entry* want = &kt[np++];                        /* getMatchingMessage :516-524 */
        if (!((m->blocked_mask >> want->dst) & 1u))
          for (uint32_t i = 0; i < x->n_pend; i++) if (x->pend[i].id == want->id) { pick = (int)i; break; }
      }
    }
    if (pick < 0) {                                                         /* getPendingEvent :452-472 (canonical order) */
      int best = 0x7FFFFFFF;
      for (uint32_t i = 0; i < x->n_pend; i++) {
        const demi_msg* c = &x->pend[i].msg;
        if ((m->blocked_mask >> c->dst) & 1u) continue;
        int q = qorder(x, c);
        if (q < best) { best = q; pick = (int)i; }
      }
    }
    if (pick < 0) break;
    fpend p = x->pend[pick];
    memmove(&x->pend[pick], &x->pend[pick + 1], sizeof(fpend) * (x->n_pend - (uint32_t)pick - 1));
    x->n_pend--;
    int snd_iso = p.msg.src < DEMI_MAX_ACTORS && ((x->isolated >> p.msg.src) & 1u);
    if (snd_iso || ((x->isolated >> p.msg.dst) & 1u)) continue;             /* discarded :626-635 */
    demi_frontier_entry* e = &x->cur[x->cur_len];
    memset(e, 0, sizeof(*e));
    e->id = p.id; e->src = p.msg.src; e->dst = p.msg.dst; e->type = p.msg.type; e->parent_pos = p.ppos;
    sh += demi_event_term((uint32_t)p.msg.src | ((uint32_t)p.msg.dst << 8) | ((uint32_t)p.msg.type << 16), p.msg.p0, p.msg.p1, x->cur_len, 0, 0);
    x->cur_pos = x->cur_len++;                                              /* :636-637 */
    x->parent_id = p.id;
    /* Instrumenter.dispatch_new_message: re-arm a repeating timer, then receive() */
    if (f_reg_find(m, p.msg.dst, p.msg.type, p.msg.p0, p.msg.p1) >= 0) f_timer_send(x, p.msg.dst, p.msg.type, p.msg.p0, p.msg.p1);
    if (x->status) break;
    m->model->receive(m, p.msg.dst, &m->states[p.msg.dst * m->model->state_words], &p.msg);
  }
  *sched_hash = sh;
  if (x->status) return 0;
  uint32_t v = m->model->invariant(m->states, m->model_flags);              /* checkInvariant :394-418 */
  if (x->F->looking_for) v = (v == x->F->looking_for) ? v : 0;
  return v;
}

/* ------------------------------------------------------------ rank state */
/* `add` ascending; merge.  pool_cap bounds the arena (every point enqueued or received over the search), not the live
 * queue: DEMI_DS_HEAP_OVF when these `n` would take the total past it.  The live queue never exceeds the arena. */
static int pool_insert_sorted(frank* r, const fkey* add, uint64_t n) {
  if (r->pool_top + n > r->cap_pool) { r->R.status = DEMI_DS_HEAP_OVF; return 0; }
  uint64_t i = r->n_pool, j = n, k = r->n_pool + n;
  while (j > 0) {
    if (i > 0 && r->pool[i - 1].ord > add[j - 1].ord) r->pool[--k] = r->pool[--i];
    else r->pool[--k] = add[--j];
  }
  r->n_pool += n; r->pool_top += n;
  return 1;
}
/* the counters after getNext, before the round executes */
static void round_snapshot(frank* r) {
  r->snap = r->R; r->snap_slots = r->n_slots; r->snap_hashes = r->n_hashes; r->snap_E = r->n_E;
}
/* a round that ends in a capacity status adds nothing to the executed work: interleavings, deliveries, violations,
 * races, keys_enqueued, rounds, trace slots and hashes go back to the last completed round; keys_dropped, pool_left
 * and explored_pairs keep the failed round's getNext */
static void round_fail(frank* r, uint32_t status) {
  r->R = r->snap; r->n_slots = r->snap_slots; r->n_hashes = r->snap_hashes;
  r->R.explored_pairs = r->snap_E; r->explored_fixed = 1;
  r->R.status = status;
  r->round_n = 0;
}
static int fkey_cmp(const void* a, const void* b) {
  const fkey* x = (const fkey*)a; const fkey* y = (const fkey*)b;
  return x->ord < y->ord ? -1 : x->ord > y->ord ? 1 : 0;
}

/* the race scan of one trace slot (dpor() :1122-1139) for later positions beyond its branch point.
 * pass 0: mark (earlier, later) explored (:1071-1073); pass 1: enqueue (later, earlier) unless explored. */
static void f_scan(frank* r, uint32_t slot, int pass, fkey* out, uint64_t* n_out) {
  const demi_frontier_entry* t = r->tr + (size_t)slot * r->T1;
  const uint32_t n = r->tr_len[slot], b = r->tr_branch[slot];
  uint16_t fp[DEMI_FR_MAX_POS + 1], pp[DEMI_FR_MAX_POS + 1];
  for (uint32_t i = 0; i < n; i++) {                                        /* first position of the same Unique (indexWhere :1058) */
    fp[i] = (uint16_t)i;
    for (uint32_t j = 1; j < i; j++) if (t[j].id == t[i].id) { fp[i] = (uint16_t)j; break; }
  }
  for (uint32_t i = 0; i < n; i++) pp[i] = i ? fp[t[i].parent_pos] : 0;
  for (uint32_t li = b + 1; li < n; li++)
    for (uint32_t ei = 1; ei < li; ei++) {
      if (t[ei].dst != t[li].dst) continue;                                 /* isCoEnabeled :1096 */
      const uint32_t lfp = fp[li], efp = fp[ei];
      uint32_t a = lfp;
      while (a > efp) a = pp[a];                                            /* laterN.pathTo(earlierN) :1104 */
      if (a == efp) continue;
      uint32_t c = efp; a = lfp;                                            /* getCommonPrefix(...).last :994-1018 */
      while (a != c) { if (a > c) a = pp[a]; else c = pp[c]; }
      if (pass == 0) { e_add(r, demi_fr_pair_key(t[ei].id, t[li].id)); r->R.races++; continue; }
      const uint64_t pk = demi_fr_pair_key(t[li].id, t[ei].id);
      if (e_has(r, pk)) continue;                                           /* would be dropped when dequeued (:1156-1160) */
      out[*n_out].ord = demi_fr_ord(a, slot, li, ei); out[*n_out].pk = pk; (*n_out)++;
    }
}

/* one round on one rank: dequeue up to `quota` unexplored points, execute (the scan follows); returns the points run */
static uint32_t f_round(frank* r, fexec* x, uint32_t quota, fkey* scratch) {
  /* getNext (:1142-1162), `quota` times without an intervening scan */
  uint64_t taken = 0; uint32_t n_sel = 0;
  fkey* sel = scratch;                                                      /* the selected points, queue order */
  while (taken < r->n_pool && n_sel < quota) {
    const fkey k = r->pool[taken++];
    if (e_has(r, k.pk)) { r->R.keys_dropped++; continue; }
    e_add(r, k.pk);                                                         /* :1169-1171 */
    sel[n_sel++] = k;
  }
  memmove(r->pool, r->pool + taken, sizeof(fkey) * (r->n_pool - taken));
  r->n_pool -= taken;
  r->round_first_slot = r->n_slots; r->round_n = 0;
  if (!n_sel) { r->R.rounds++; return 0; }
  round_snapshot(r);
  /* the whole round needs its trace slots before any point runs */
  if ((uint64_t)r->n_slots + n_sel > r->cap_slots) { round_fail(r, DEMI_DS_TRACE_OVF); return n_sel; }
  for (uint32_t s = 0; s < n_sel; s++) {
    const uint32_t kslot = demi_fr_ord_slot(sel[s].ord), branch = demi_fr_ord_branch(sel[s].ord);
    const uint32_t li = demi_fr_ord_later(sel[s].ord), ei = demi_fr_ord_earlier(sel[s].ord);
    const uint32_t slot = r->n_slots++;
    x->cur = r->tr + (size_t)slot * r->T1;
    uint64_t sh;
    uint32_t v = f_execute(x, r->tr + (size_t)kslot * r->T1, branch, li, ei, &sh);
    if (x->status) { round_fail(r, (uint32_t)x->status); return n_sel; }
    r->tr_len[slot] = x->cur_len; r->tr_branch[slot] = branch;
    r->round_n++;
    if (r->hashes && r->n_hashes < r->cap_hashes) r->hashes[r->n_hashes] = sh;
    r->n_hashes++;
    r->R.interleavings++; r->R.deliveries += x->cur_len - 1;
    if (v) {
      if (r->viol && r->R.violations < r->cap_viol) {
        demi_dpor_violation* o = &r->viol[r->R.violations];
        o->schedule_hash = sh; o->interleaving = (uint32_t)(r->n_hashes - 1); o->length = (uint16_t)(x->cur_len - 1); o->code = (uint16_t)v;
      }
      r->R.violations++;
    }
  }
  r->R.rounds++;
  return n_sel;
}
/* the scan of the round's traces and the enqueue; the explored table's and the arena's capacities are decided here,
 * for the whole round (cap_scratch holds any round: at most rcap < T1²/2 points per trace) */
static void f_scan_round(frank* r, fkey* scratch, uint64_t cap_scratch) {
  for (uint32_t s = 0; s < r->round_n; s++) f_scan(r, r->round_first_slot + s, 0, 0, 0);
  uint64_t n_new = 0;
  for (uint32_t s = 0; s < r->round_n; s++) {
    if (n_new + (uint64_t)r->T1 * r->T1 > cap_scratch) { round_fail(r, DEMI_DS_HEAP_OVF); return; }
    f_scan(r, r->round_first_slot + s, 1, scratch, &n_new);
  }
  if (r->n_E * 2 >= r->e_cap || (r->log && r->n_log > r->cap_log)) { round_fail(r, DEMI_DS_EXPLORED_OVF); return; }
  if (r->pool_top + n_new > r->cap_pool) { round_fail(r, DEMI_DS_HEAP_OVF); return; }
  qsort(scratch, n_new, sizeof(fkey), fkey_cmp);                            /* already ascending per slot; slots ascending per branch */
  r->R.keys_enqueued += n_new;
  pool_insert_sorted(r, scratch, n_new);
  r->round_n = 0;
}

int oracle_dpor_frontier(const demi_config* cfg, const demi_ext_event* ext, uint32_t n_ext,
                         const demi_frontier_params* F, uint32_t n_ranks, demi_frontier_result* results,
                         demi_dpor_violation* viol, uint32_t cap_viol, uint64_t* hashes, uint64_t cap_hashes) {
  const oracle_model* model = oracle_get_model(cfg->model);
  if (!model || !n_ranks || n_ranks > 64) return DEMI_ERR_INVALID;
  if (F->max_messages < 1 || F->max_messages > 1000 || !F->width) return DEMI_ERR_INVALID;
  if (F->explored_slots & (F->explored_slots - 1)) return DEMI_ERR_INVALID;
  uint32_t n_sends = 0;
  for (uint32_t i = 0; i < n_ext; i++) {
    if (ext[i].kind != DEMI_EXT_START && ext[i].kind != DEMI_EXT_SEND) return DEMI_ERR_INVALID;   /* :710 */
    if (ext[i].kind == DEMI_EXT_SEND) n_sends++;
  }
  const uint32_t T1 = (uint32_t)F->max_messages + 2;
  const uint32_t S = F->rounds_per_exchange ? F->rounds_per_exchange : 1;
  frank* R = (frank*)calloc(n_ranks, sizeof(frank));
  fexec* x = (fexec*)calloc(1, sizeof(fexec));
  x->m.model = model; x->m.model_flags = cfg->model_flags; x->m.blocked_mask = cfg->blocked_mask;
  x->F = F; x->ext = ext; x->n_ext = n_ext;
  x->cap_pend = demi_fr_pool_entries(oracle_model_key(cfg->model), F->max_messages, n_sends);
  x->pend = (fpend*)malloc(sizeof(fpend) * x->cap_pend);
  const uint64_t cap_scratch = (uint64_t)F->width * T1 * T1 / 2 + (uint64_t)T1 * T1 + F->width + 16;
  fkey* scratch = (fkey*)malloc(sizeof(fkey) * cap_scratch);
  fkey* sbuf = (fkey*)malloc(sizeof(fkey) * (2 * (size_t)F->steal_max + 2));
  for (uint32_t q = 0; q < n_ranks; q++) {
    frank* r = &R[q];
    r->no_history = (F->flags & DEMI_FR_NO_HISTORY) != 0;
    r->e_cap = F->explored_slots; r->e_slots = r->no_history ? 1 : 1024; r->E = (uint64_t*)calloc(r->e_slots, 8);
    if (n_ranks > 1 && !r->no_history) {
      r->cap_log = F->explored_slots / 2 < (1ull << 22) ? F->explored_slots / 2 : (1ull << 22);
      r->log_alloc = 1024; r->log = (uint64_t*)malloc(8 * r->log_alloc);
    }
    r->T1 = T1; r->cap_slots = F->trace_cap;
    r->tr = (demi_frontier_entry*)malloc(sizeof(demi_frontier_entry) * (size_t)r->cap_slots * T1);
    r->tr_len = (uint32_t*)calloc(r->cap_slots, 4); r->tr_branch = (uint32_t*)calloc(r->cap_slots, 4);
    r->cap_pool = F->pool_cap; r->pool = (fkey*)malloc(sizeof(fkey) * r->cap_pool);
    r->viol = viol ? viol + (size_t)q * cap_viol : 0; r->cap_viol = cap_viol;
    r->hashes = hashes ? hashes + (size_t)q * cap_hashes : 0; r->cap_hashes = cap_hashes;
  }
  g_fx = x;
  uint64_t executed = 0; int any_status = 0, found = 0, exhausted = 0, budget = 0;
  /* the first execution: no nextTrace (:1219-1221 with an empty backtrack set), on rank 0 */
  {
    frank* r = &R[0];
    round_snapshot(r);
    if (F->max_interleavings < 1) {}
    else if (r->cap_slots < 1) round_fail(r, DEMI_DS_TRACE_OVF);
    else {
      x->cur = r->tr; uint64_t sh;
      uint32_t v = f_execute(x, 0, 0, 0, 0, &sh);
      if (x->status) round_fail(r, (uint32_t)x->status);
      else {
        r->tr_len[0] = x->cur_len; r->tr_branch[0] = 0; r->n_slots = 1;
        r->round_first_slot = 0; r->round_n = 1;
        if (r->hashes && r->cap_hashes) r->hashes[0] = sh;
        r->n_hashes = 1; r->R.interleavings = 1; r->R.deliveries = x->cur_len - 1; r->R.rounds = 1;
        if (v) {
          if (r->viol && cap_viol) { r->viol[0].schedule_hash = sh; r->viol[0].interleaving = 0; r->viol[0].length = (uint16_t)(x->cur_len - 1); r->viol[0].code = (uint16_t)v; }
          r->R.violations = 1;
        }
        f_scan_round(r, scratch, cap_scratch);
      }
    }
  }
  for (;;) {
    /* ---- exchange point: what every rank learns from the all-gather */
    executed = 0; any_status = 0; found = 0; uint64_t total_pool = 0;
    for (uint32_t q = 0; q < n_ranks; q++) { executed += R[q].R.interleavings; any_status |= R[q].R.status != 0; found |= R[q].R.violations != 0; total_pool += R[q].n_pool; }
    if (any_status) break;
    if (F->stop_if_found && found) break;                                   /* :1147 */
    if (executed >= F->max_interleavings) { budget = 1; break; }
    if (!total_pool) { exhausted = 1; break; }
    /* ---- the pair keys every rank marked since the last exchange become known to all ranks (a set union) */
    if (n_ranks > 1 && R[0].log) {
      int log_ovf = 0;                                                      /* a log past its capacity fails every rank */
      for (uint32_t q = 0; q < n_ranks; q++) log_ovf |= R[q].n_log > R[q].cap_log;
      if (log_ovf) { for (uint32_t q = 0; q < n_ranks; q++) R[q].R.status = DEMI_DS_EXPLORED_OVF; any_status = 1; break; }
      for (uint32_t q = 0; q < n_ranks; q++) R[q].R.bytes_sent += R[q].n_log * 8ull * (n_ranks - 1);
      for (uint32_t rcv = 0; rcv < n_ranks; rcv++)
        for (uint32_t src = 0; src < n_ranks; src++) {
          if (src == rcv) continue;
          uint64_t* keep = R[rcv].log; R[rcv].log = 0;                 /* learned keys are not shared again */
          for (uint64_t i = 0; i < R[src].n_log; i++) e_add(&R[rcv], R[src].log[i]);
          R[rcv].log = keep;
        }
      for (uint32_t q = 0; q < n_ranks; q++) R[q].n_log = 0;
      any_status = 0;
      for (uint32_t q = 0; q < n_ranks; q++) any_status |= R[q].R.status != 0;
      if (any_status) break;
    }
    /* ---- steal plan: ranks that cannot fill their next S rounds take from ranks that can spare */
    if (n_ranks > 1) {
      const uint64_t need = (uint64_t)S * F->width;
      for (uint32_t q = 0; q < n_ranks; q++) R[q].R.exchanges++;
      /* target queue length: enough for the next S rounds, or an equal share when there is less than that */
      const uint64_t share = (total_pool + n_ranks - 1) / n_ranks;
      const uint64_t target = need < share ? need : share;
      uint64_t have[64], give[64];
      for (uint32_t q = 0; q < n_ranks; q++) { have[q] = R[q].n_pool; give[q] = have[q] > target ? have[q] - target : 0; }
      for (uint32_t rcv = 0; rcv < n_ranks; rcv++) {
        uint64_t want = have[rcv] < target ? target - have[rcv] : 0;
        for (uint32_t don = 0; don < n_ranks && want; don++) {
          if (don == rcv || !give[don]) continue;
          uint64_t m = want < give[don] ? want : give[don];
          if (m > F->steal_max) m = F->steal_max;
          if (!m) continue;
          give[don] -= m; want -= m;
          /* the donor hands over the LAST m points of its queue (shallowest branch), queue order kept; points whose
           * pair is explored on the donor are dropped, the others are marked explored there (someone runs them) */
          frank* d = &R[don]; frank* r = &R[rcv];
          fkey* moved = sbuf; uint64_t n_moved = 0;
          const uint64_t lo = d->n_pool - m;
          for (uint64_t i = lo; i < d->n_pool; i++) {
            if (e_has(d, d->pool[i].pk)) { d->R.keys_dropped++; continue; }
            e_add(d, d->pool[i].pk);
            moved[n_moved++] = d->pool[i];
          }
          d->n_pool = lo;
          d->R.records_sent += n_moved; d->R.bytes_sent += 16ull * (T1 + 2) * n_moved;   /* fixed-stride records on the wire */
          /* a receiver takes a donor's batch whole or, when its trace slots or its arena cannot hold it, not at all
           * (and no later batch) */
          if (r->R.status || !n_moved) continue;
          if ((uint64_t)r->n_slots + n_moved > r->cap_slots) { r->R.status = DEMI_DS_TRACE_OVF; continue; }
          if (r->pool_top + n_moved > r->cap_pool) { r->R.status = DEMI_DS_HEAP_OVF; continue; }
          /* each record = the point + its trace prefix [0..later]; the receiver stores the prefix in a new slot */
          for (uint64_t i = 0; i < n_moved; i++) {
            const uint32_t kslot = demi_fr_ord_slot(moved[i].ord), li = demi_fr_ord_later(moved[i].ord);
            const uint32_t slot = r->n_slots++;
            memcpy(r->tr + (size_t)slot * T1, d->tr + (size_t)kslot * T1, sizeof(demi_frontier_entry) * (li + 1));
            r->tr_len[slot] = li + 1; r->tr_branch[slot] = li;            /* nothing left to scan on an imported prefix */
            fkey k; k.pk = moved[i].pk;
            k.ord = demi_fr_ord(demi_fr_ord_branch(moved[i].ord), slot, li, demi_fr_ord_earlier(moved[i].ord));
            sbuf[F->steal_max + i] = k;
          }
          r->R.records_received += n_moved;
          fkey* in = sbuf + F->steal_max;
          qsort(in, n_moved, sizeof(fkey), fkey_cmp);
          pool_insert_sorted(r, in, n_moved);
        }
      }
      any_status = 0;
      for (uint32_t q = 0; q < n_ranks; q++) any_status |= R[q].R.status != 0;
      if (any_status) break;
    }
    /* ---- S rounds per rank.  What is left of the budget goes to the ranks in rank order, each taking what its queue
     * (as every rank knows it after the exchange) could use in S rounds — so the budget follows the work */
    uint64_t left = F->max_interleavings - executed;
    for (uint32_t q = 0; q < n_ranks; q++) {
      frank* r = &R[q];
      uint64_t cap = (uint64_t)S * F->width;
      if (cap > r->n_pool) cap = r->n_pool;
      uint64_t allow = cap < left ? cap : left;
      left -= allow;
      for (uint32_t s = 0; s < S && allow && r->n_pool && !r->R.status; s++) {
        uint32_t quota = allow < F->width ? (uint32_t)allow : F->width;
        const uint32_t n_run = f_round(r, x, quota, scratch);
        allow -= n_run;
        if (n_run && !r->R.status) f_scan_round(r, scratch, cap_scratch);
        if (F->stop_if_found && r->R.violations) break;
      }
    }
  }
  g_fx = 0;
  for (uint32_t q = 0; q < n_ranks; q++) {
    frank* r = &R[q];
    if (!r->explored_fixed) r->R.explored_pairs = r->n_E;
    r->R.pool_left = r->n_pool; r->R.trace_slots = r->n_slots;
    r->R.exhausted = (uint32_t)exhausted; r->R.budget_exhausted = (uint32_t)budget;
    results[q] = r->R;
    free(r->log); free(r->E); free(r->tr); free(r->tr_len); free(r->tr_branch); free(r->pool);
  }
  free(scratch); free(sbuf); free(x->pend); free(x); free(R);
  return any_status ? DEMI_ERR_CAPACITY : DEMI_OK;
}
