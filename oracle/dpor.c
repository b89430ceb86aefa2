/*
 * ORACLE — test infrastructure only (see machine.h header).  PARITY UNPINNED
 * against a running reference; pinned by derivable KATs only.
 *
 * DPORwHeuristics (schedulers/DPORwHeuristics.scala) restated, sequential:
 *   schedule_new_message :421-648, event_produced/getMessage :773-847,
 *   notify_quiescence :855-942, dpor :1020-1185 (isCoEnabeled :1091-1110,
 *   analyze_dep :1043-1077, getCommonPrefix :994-1018, getNext :1142-1162),
 *   test/run/runExternal :1193-1242, :723-762, :684-721,
 *   DefaultBacktrackOrdering (BacktrackOrdering.scala:58-69),
 *   ExploredTacker (AuxilaryTypes.scala:209-246).
 *
 * Scope: externals are Start and Send only (DPORwHeuristicsUtil.convertToDPORTrace
 * with ignoreQuiescence=true, :1279-1303; runExternal throws on anything else,
 * :710); checkpointing off (so the invariant is checked at the end of each
 * interleaving only, :559-571, :877-901).
 * Canonical orders where the reference depends on scala-library internals that
 * are not in the tree (SURVEY §8c): the divergent choice (`pendingEvents.find`,
 * :454-456, HashMap iteration order) takes the non-empty (snd,rcv) queue with
 * the lowest snd*256+rcv; equal-priority backtrack keys (PriorityQueue tie
 * order, :170, :1154) are served first-in first-out.
 * A search that finds a violation and is resumed by calling test() again
 * (:1219-1221) continues exactly as if it had not stopped; `stop_if_found`
 * selects between the two.
 *
 * oracle_dpor_open / oracle_dpor_test / oracle_dpor_close keep one DPORwHeuristics
 * instance alive across test() calls, which is what ResumableDPOR
 * (IncrementalDeltaDebugging.scala:90-122) relies on, and add the configuration of
 * RunnerUtils.editDistanceDporDDMin (RunnerUtils.scala:822-835): setInitialDepGraph
 * / setInitialTrace (:210-217), prioritizePendingUponDivergence (:65-68, :542-555),
 * ArvindDistanceOrdering (BacktrackOrdering.scala:99-173) and setMaxDistance
 * (:128-134, :1145-1146).  With a distance cap the enqueue-time explored filter is
 * off, because getNext inspects the head of the queue before it filters (:1144-1160).
 */
#include <stdlib.h>
#include <string.h>
#include "machine.h"
#include "dpor.h"

#define DQ_CAP 256           /* per (snd,rcv) FIFO capacity */
#define DP_MAX_T 1024

typedef struct { demi_msg msg; uint32_t parent; uint16_t depth; } dnode;
typedef struct { uint32_t branch, seq, e1, e2, trace_ref, later_i, dist, earlier_i; } bkey;

typedef struct {
  om_machine m;                         /* actor states, registry/cancelled sets, model hooks */
  const demi_dpor_params* P;
  /* persistent dependency graph (a tree, SURVEY A.4) */
  dnode* nodes; uint32_t n_nodes, cap_nodes;
  /* explored ordered pairs */
  uint64_t* explored; uint32_t explored_slots, n_explored;
  /* backtrack heap */
  bkey* heap; uint32_t n_heap, cap_heap, seq;
  /* traces of finished interleavings */
  uint32_t* traces; uint32_t* trace_len; uint32_t n_traces, cap_traces, T1;
  /* per-interleaving */
  uint32_t queues[(DEMI_MAX_ACTORS + 1) * DEMI_MAX_ACTORS][DQ_CAP];
  uint16_t qlen[(DEMI_MAX_ACTORS + 1) * DEMI_MAX_ACTORS];
  uint32_t isolated;
  uint32_t parent_event, current_depth;
  uint32_t cur_trace[DP_MAX_T]; uint32_t cur_len;
  uint32_t next_trace[DP_MAX_T]; uint32_t next_len, next_pos;
  const uint32_t* next_rd;                                 /* the nextTrace followed: next_trace or the initial trace */
  int32_t nsched;
  int status;
  /* instance state that survives test() calls */
  demi_dpor_params params;
  demi_ext_event* ext; uint32_t n_ext;
  oracle_dpor_opts opts;
  int32_t* orig_index;                  /* ArvindDistanceOrdering.originalIndices: node -> index in originalTrace, -1 absent */
  int started, found;                   /* found: shortestTraceSoFar != null */
  int32_t max_distance;                 /* stop_at_distance; < 0: should_cap_distance = false */
  uint32_t* path;                       /* scratch for arvindDistance */
} dpor_t;

static __thread dpor_t* g_dpor = 0;
int oracle_in_dpor_mode(void) { return g_dpor != 0; }

static uint32_t qindex(const dpor_t* d, uint32_t src, uint32_t dst) {
  uint32_t s = src == DEMI_DEADLETTERS ? (uint32_t)d->m.model->n_actors : src;
  return s * DEMI_MAX_ACTORS + dst;
}

/* DPORwHeuristics.getMessage (:773-801): reuse the child of parentEvent with equal
 * (snd, rcv, fingerprint) in the PERSISTENT graph, else a new Unique. */
static uint32_t dpor_get_message(dpor_t* d, const demi_msg* msg) {
  for (uint32_t i = 1; i < d->n_nodes; i++) {
    const dnode* n = &d->nodes[i];
    if (n->parent == d->parent_event && n->msg.src == msg->src && n->msg.dst == msg->dst &&
        n->msg.type == msg->type && n->msg.p0 == msg->p0 && n->msg.p1 == msg->p1) return i;
  }
  if (d->n_nodes >= d->cap_nodes) { d->status = DEMI_DS_NODE_OVF; return 0; }
  uint32_t id = d->n_nodes++;
  d->nodes[id].msg = *msg; d->nodes[id].msg.flags = 0;
  d->nodes[id].parent = d->parent_event;
  d->nodes[id].depth = (uint16_t)(d->nodes[d->parent_event].depth + 1);
  return id;
}

/* DPORwHeuristics.event_produced (:803-847) after Instrumenter.aroundDispatch's
 * cancelled-timer drop (Instrumenter.scala:1090-1096) */
static void dpor_event_produced(dpor_t* d, const demi_msg* msg) {
  om_machine* m = &d->m;
  if (d->status) return;
  for (uint32_t i = 0; i < m->n_cancelled; i++) {
    om_timer_key* k = &m->cancelled[i];
    if (k->dst == msg->dst && k->type == msg->type && k->p0 == msg->p0 && k->p1 == msg->p1) {
      for (uint32_t j = i; j + 1 < m->n_cancelled; j++) m->cancelled[j] = m->cancelled[j + 1];
      m->n_cancelled--;
      return;
    }
  }
  uint32_t id = dpor_get_message(d, msg);
  if (d->status) return;
  /* depth-bound gate :832 */
  if (d->P->depth_bound < 0 || (int32_t)d->current_depth < d->P->depth_bound) {
    uint32_t q = qindex(d, msg->src, msg->dst);
    if (d->qlen[q] >= DQ_CAP) { d->status = DEMI_DS_QUEUE_OVF; return; }
    d->queues[q][d->qlen[q]++] = id;
  }
}

void dpor_om_send(om_machine* m, int src, int dst, uint8_t type, uint32_t p0, uint32_t p1) {
  (void)m;
  demi_msg msg; msg.src = (uint8_t)src; msg.dst = (uint8_t)dst; msg.type = type; msg.flags = 0; msg.p0 = p0; msg.p1 = p1;
  dpor_event_produced(g_dpor, &msg);
}
void dpor_queue_overflow(void) { if (!g_dpor->status) g_dpor->status = DEMI_DS_QUEUE_OVF; }
/* Scheduler.enqueue_timer default = enqueue_message: the timer message is sent at
 * once (Scheduler.scala:73; DPORwHeuristics.scala:946-955).  SchedulerConfig.ignoreTimers
 * is not read here: the reference reads it only in ExternalEventInjector.handle_timer
 * (ExternalEventInjector.scala:283-285), which DPORwHeuristics never calls. */
static void dpor_timer_send(dpor_t* d, int rcv, uint8_t type, uint32_t p0, uint32_t p1) {
  demi_msg t; t.src = DEMI_DEADLETTERS; t.dst = (uint8_t)rcv; t.type = type; t.flags = 0; t.p0 = p0; t.p1 = p1;
  dpor_event_produced(d, &t);
}
static int reg_find(const om_machine* m, int dst, uint8_t type, uint32_t p0, uint32_t p1) {
  for (uint32_t i = 0; i < m->n_registry; i++)
    if (m->registry[i].dst == dst && m->registry[i].type == type && m->registry[i].p0 == p0 && m->registry[i].p1 == p1) return (int)i;
  return -1;
}
void dpor_om_schedule(om_machine* m, int self, uint8_t type, uint32_t p0, uint32_t p1, int repeating) {
  dpor_t* d = g_dpor;
  if (d->status) return;
  if (reg_find(m, self, type, p0, p1) >= 0) return;                       /* "Non-unique timer" */
  if (repeating) {
    if (m->n_registry >= DEMI_TIMERSET_CAP) { d->status = DEMI_DS_QUEUE_OVF; return; }
    om_timer_key* k = &m->registry[m->n_registry++];
    k->dst = (uint8_t)self; k->type = type; k->p0 = p0; k->p1 = p1;
  }
  dpor_timer_send(d, self, type, p0, p1);
}
/* DPORwHeuristics.notify_timer_cancel (:961-985) */
void dpor_om_cancel(om_machine* m, int self, uint8_t type, uint32_t p0, uint32_t p1) {
  dpor_t* d = g_dpor;
  if (d->status) return;
  int have = 0;
  for (uint32_t i = 0; i < m->n_cancelled; i++)
    if (m->cancelled[i].dst == self && m->cancelled[i].type == type && m->cancelled[i].p0 == p0 && m->cancelled[i].p1 == p1) have = 1;
  if (!have) {
    if (m->n_cancelled >= DEMI_TIMERSET_CAP) { d->status = DEMI_DS_QUEUE_OVF; return; }
    om_timer_key* k = &m->cancelled[m->n_cancelled++];
    k->dst = (uint8_t)self; k->type = type; k->p0 = p0; k->p1 = p1;
  }
  int ri = reg_find(m, self, type, p0, p1);
  if (ri >= 0) { for (uint32_t j = (uint32_t)ri; j + 1 < m->n_registry; j++) m->registry[j] = m->registry[j + 1]; m->n_registry--; }
  uint32_t q = qindex(d, DEMI_DEADLETTERS, (uint32_t)self);
  for (uint32_t i = 0; i < d->qlen[q]; i++) {
    const demi_msg* c = &d->nodes[d->queues[q][i]].msg;
    if (c->type == type && c->p0 == p0 && c->p1 == p1) {
      for (uint32_t j = i; j + 1 < d->qlen[q]; j++) d->queues[q][j] = d->queues[q][j + 1];
      d->qlen[q]--;
      return;
    }
  }
}

/* ------------------------------------------------------------- explored set */
static int explored_has(const dpor_t* d, uint32_t a, uint32_t b) {
  uint64_t key = ((uint64_t)a << 32) | b;
  uint32_t s = (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 40) & (d->explored_slots - 1);
  while (d->explored[s] != ~0ull) { if (d->explored[s] == key) return 1; s = (s + 1) & (d->explored_slots - 1); }
  return 0;
}
static void explored_add(dpor_t* d, uint32_t a, uint32_t b) {
  uint64_t key = ((uint64_t)a << 32) | b;
  uint32_t s = (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 40) & (d->explored_slots - 1);
  while (d->explored[s] != ~0ull) { if (d->explored[s] == key) return; s = (s + 1) & (d->explored_slots - 1); }
  if (d->n_explored * 2 >= d->explored_slots) { d->status = DEMI_DS_EXPLORED_OVF; return; }
  d->explored[s] = key; d->n_explored++;
}

/* ------------------------------------------------------------------- heap */
static int key_before(const bkey* a, const bkey* b) {    /* a is served before b */
  /* ArvindDistanceOrdering.getOrdered (BacktrackOrdering.scala:153-163): the LARGER distance compares
   * higher and PriorityQueue serves the maximum; `dist` is 0 for DefaultBacktrackOrdering */
  if (a->dist != b->dist) return a->dist > b->dist;
  if (a->branch != b->branch) return a->branch > b->branch;   /* deeper first (DefaultBacktrackOrdering) */
  /* canonical order among ties: first-in first-out.  Keys are enqueued in (interleaving, later position,
   * earlier position) order, so that triple is the sequence number; a key that a resumed test() enqueues a
   * second time (:1219-1220) sorts next to its first copy, which no explored schedule can observe */
  if (a->trace_ref != b->trace_ref) return a->trace_ref < b->trace_ref;
  if (a->later_i != b->later_i) return a->later_i < b->later_i;
  if (a->earlier_i != b->earlier_i) return a->earlier_i < b->earlier_i;
  return a->seq < b->seq;
}
static void heap_push(dpor_t* d, bkey k) {
  if (d->n_heap >= d->cap_heap) { d->status = DEMI_DS_HEAP_OVF; return; }
  uint32_t i = d->n_heap++;
  d->heap[i] = k;
  while (i > 0) { uint32_t p = (i - 1) / 2; if (!key_before(&d->heap[i], &d->heap[p])) break;
    bkey t = d->heap[i]; d->heap[i] = d->heap[p]; d->heap[p] = t; i = p; }
}
static bkey heap_pop(dpor_t* d) {
  bkey top = d->heap[0];
  d->heap[0] = d->heap[--d->n_heap];
  uint32_t i = 0;
  for (;;) {
    uint32_t l = 2 * i + 1, r = l + 1, b = i;
    if (l < d->n_heap && key_before(&d->heap[l], &d->heap[b])) b = l;
    if (r < d->n_heap && key_before(&d->heap[r], &d->heap[b])) b = r;
    if (b == i) break;
    bkey t = d->heap[i]; d->heap[i] = d->heap[b]; d->heap[b] = t; i = b;
  }
  return top;
}

/* ------------------------------------------------ one interleaving (run) */
static void set_parent(dpor_t* d, uint32_t node) {          /* setParentEvent :278-282 */
  d->parent_event = node;
  d->current_depth = (uint32_t)d->nodes[node].depth + 1;
}

/* returns node id or 0 for None */
static uint32_t dpor_schedule(dpor_t* d) {
  const uint32_t nq = (uint32_t)(d->m.model->n_actors + 1) * DEMI_MAX_ACTORS;
  for (;;) {
    if (d->status) return 0;
    d->nsched++;                                            /* :583-586 */
    if (d->P->max_messages >= 0 && d->nsched > d->P->max_messages) return 0;
    uint32_t pick = 0;
    /* getMatchingMessage :474-537 via getNextTraceMessage :363-372 (id 0 entries skipped); with
     * prioritizePendingUponDivergence, getNextMatchingMessage (:542-555) keeps popping nextTrace until an
     * expected message is pending */
    do {
      while (d->next_pos < d->next_len && d->next_rd[d->next_pos] == 0) d->next_pos++;
      if (d->next_pos >= d->next_len) break;
      uint32_t want = d->next_rd[d->next_pos++];
      const demi_msg* c = &d->nodes[want].msg;
      if (!((d->m.blocked_mask >> c->dst) & 1u)) {
        uint32_t q = qindex(d, c->src, c->dst);
        for (uint32_t i = 0; i < d->qlen[q]; i++)
          if (d->queues[q][i] == want) {                    /* equivalentTo: same receiver and id :440-445 */
            for (uint32_t j = i; j + 1 < d->qlen[q]; j++) d->queues[q][j] = d->queues[q][j + 1];
            d->qlen[q]--;
            pick = want;
            break;
          }
      }
    } while (!pick && d->opts.prioritize_pending);
    if (!pick) {                                            /* divergent: getPendingEvent :452-472 */
      for (uint32_t q = 0; q < nq; q++) {
        uint32_t dst = q % DEMI_MAX_ACTORS;
        if (!d->qlen[q] || ((d->m.blocked_mask >> dst) & 1u)) continue;
        pick = d->queues[q][0];
        for (uint32_t j = 0; j + 1 < d->qlen[q]; j++) d->queues[q][j] = d->queues[q][j + 1];
        d->qlen[q]--;
        break;
      }
    }
    if (!pick) return 0;
    const demi_msg* c = &d->nodes[pick].msg;
    int snd_iso = c->src < DEMI_MAX_ACTORS && ((d->isolated >> c->src) & 1u);
    if (snd_iso || ((d->isolated >> c->dst) & 1u)) continue;   /* discarded :626-635 */
    if (d->cur_len >= DP_MAX_T) { d->status = DEMI_DS_TRACE_OVF; return 0; }
    d->cur_trace[d->cur_len++] = pick;                       /* :636-637 */
    set_parent(d, pick);
    return pick;
  }
}

static uint32_t dpor_run_interleaving(dpor_t* d, const demi_ext_event* ext, uint32_t n_ext) {
  om_machine* m = &d->m;
  memset(m->states, 0, sizeof(m->states));
  m->model->init(m->states, m->model_flags);
  m->n_registry = m->n_cancelled = 0;
  memset(d->qlen, 0, sizeof(d->qlen));
  d->isolated = m->model->n_actors >= 32 ? 0xFFFFFFFFu : ((1u << m->model->n_actors) - 1u);
  d->cur_len = 0; d->cur_trace[d->cur_len++] = 0;            /* currentTrace += root :343 */
  set_parent(d, 0);
  d->nsched = 0;
  /* runExternal :684-721 */
  for (uint32_t i = 0; i < n_ext && !d->status; i++) {
    if (ext[i].kind == DEMI_EXT_START) d->isolated &= ~(1u << ext[i].a);
    else if (ext[i].kind == DEMI_EXT_SEND) {
      demi_msg s; s.src = DEMI_DEADLETTERS; s.dst = ext[i].a; s.type = ext[i].type; s.flags = 0; s.p0 = ext[i].p0; s.p1 = ext[i].p1;
      dpor_event_produced(d, &s);
    }
  }
  uint32_t pick;
  while (!d->status && (pick = dpor_schedule(d)) != 0) {
    demi_msg msg = d->nodes[pick].msg;
    /* Instrumenter.dispatch_new_message: re-arm a repeating timer, then receive() */
    if (reg_find(m, msg.dst, msg.type, msg.p0, msg.p1) >= 0) dpor_timer_send(d, msg.dst, msg.type, msg.p0, msg.p1);
    if (d->status) break;
    m->model->receive(m, msg.dst, &m->states[msg.dst * m->model->state_words], &msg);
  }
  if (d->status) return 0;
  uint32_t v = m->model->invariant(m->states, m->model_flags);   /* checkInvariant :394-418 */
  if (d->P->looking_for) v = (v == d->P->looking_for) ? v : 0;
  return v;
}

static int is_ancestor(const dpor_t* d, uint32_t anc, uint32_t node) {   /* laterN.pathTo(earlierN) :1104 */
  while (d->nodes[node].depth > d->nodes[anc].depth) node = d->nodes[node].parent;
  return node == anc;
}
static uint32_t lca(const dpor_t* d, uint32_t a, uint32_t b) {           /* getCommonPrefix(...).last :994-1018 */
  while (d->nodes[a].depth > d->nodes[b].depth) a = d->nodes[a].parent;
  while (d->nodes[b].depth > d->nodes[a].depth) b = d->nodes[b].parent;
  while (a != b) { a = d->nodes[a].parent; b = d->nodes[b].parent; }
  return a;
}

/* the delivered-message sequence of a trace, id-independent */
static uint64_t schedule_hash(const dpor_t* d, const uint32_t* tr, uint32_t len) {
  uint64_t h = 0;
  for (uint32_t i = 1; i < len; i++) {
    const demi_msg* c = &d->nodes[tr[i]].msg;
    h += demi_event_term((uint32_t)c->src | ((uint32_t)c->dst << 8) | ((uint32_t)c->type << 16), c->p0, c->p1, i, 0, 0);
  }
  return h;
}

/* ArvindDistanceOrdering.arvindDistance (BacktrackOrdering.scala:119-146): path = the dependency path root..e1
 * (getCommonPrefix(e1, e1)) ++ replayThis ++ [e1, e2]; +1 per event that is not in the original trace, +1 per
 * earlier path element that the original trace orders after it */
uint32_t oracle_arvind_distance_of(const int32_t* oi, uint32_t n) {
  uint32_t dist = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (oi[i] < 0) { dist++; continue; }                      /* "Not in original" :133-135 */
    for (uint32_t j = 0; j < i; j++) if (oi[j] >= 0 && oi[j] > oi[i]) dist++;   /* "Reordered" :137-142 */
  }
  return dist;
}
static uint32_t arvind_distance(dpor_t* d, const bkey* k) {
  uint32_t n = 0, depth = d->nodes[k->e1].depth;
  uint32_t* path = d->path;
  for (uint32_t v = k->e1, i = depth + 1; i-- > 0; v = d->nodes[v].parent) path[i] = v;
  n = depth + 1;
  const uint32_t* kt = d->traces + (size_t)k->trace_ref * d->T1;
  for (uint32_t i = k->branch + 1; i <= k->later_i; i++) if (kt[i] != k->e2) path[n++] = kt[i];
  path[n++] = k->e1; path[n++] = k->e2;
  int32_t* oi = (int32_t*)path;
  for (uint32_t i = 0; i < n; i++) oi[i] = path[i] < d->opts.n_init_nodes ? d->orig_index[path[i]] : -1;
  return oracle_arvind_distance_of(oi, n);
}

/* dpor(trace) :1020-1185: race scan over the last trace (index k in d->traces), then getNext.  Returns 1 and
 * fills next_trace, or 0 for None. */
static int dpor_analyse(dpor_t* d, uint32_t k, demi_dpor_result* out) {
  const demi_dpor_params* P = &d->params;
  const uint32_t* tr = d->traces + (size_t)k * d->T1; const uint32_t n = d->trace_len[k];
  const int capped = d->max_distance >= 0;
  for (uint32_t li = 1; li < n && !d->status; li++)
    for (uint32_t ei = 1; ei < li && !d->status; ei++) {
      uint32_t later = tr[li], earlier = tr[ei];
      if (d->nodes[later].msg.dst != d->nodes[earlier].msg.dst) continue;       /* isCoEnabeled :1096 */
      if (is_ancestor(d, earlier, later)) continue;                              /* :1104-1107 */
      uint32_t l = lca(d, earlier, later);
      uint32_t branch = 0;
      while (branch < n && tr[branch] != l) branch++;                            /* indexWhere :1058 */
      explored_add(d, earlier, later);                                           /* :1071-1073 */
      out->races++;
      if (!capped && explored_has(d, later, earlier)) continue;   /* would be skipped when popped (:1156-1160) */
      bkey key = { branch, d->seq++, later, earlier, k, li, 0, ei };
      if (d->opts.arvind) key.dist = arvind_distance(d, &key);
      heap_push(d, key);                                                         /* :1134 */
    }
  if (d->status) return 0;
  /* getNext :1142-1162 */
  bkey key;
  for (;;) {
    if (!d->n_heap) { out->exhausted = 1; return 0; }
    if (capped && (int32_t)(d->opts.arvind ? d->heap[0].dist : 0u) >= d->max_distance) return 0;   /* :1145-1146 */
    if (P->stop_if_found && d->found) return 0;                                  /* :1147 */
    key = heap_pop(d);
    if (!explored_has(d, key.e1, key.e2)) break;
  }
  explored_add(d, key.e1, key.e2);                                               /* :1169-1171 */
  if (d->status) return 0;
  /* nextTrace = trace.take(maxIndex+1) ++ replayThis (:1180); replayThis =
   * keyTrace.drop(branchI+1).dropRight(size-laterI-1).filter(_.id != earlier.id) (:1060-1063) */
  d->next_len = 0; d->next_pos = 0; d->next_rd = d->next_trace;
  for (uint32_t i = 0; i <= key.branch && i < n; i++) d->next_trace[d->next_len++] = tr[i];
  const uint32_t* kt = d->traces + (size_t)key.trace_ref * d->T1;
  for (uint32_t i = key.branch + 1; i <= key.later_i; i++)
    if (kt[i] != key.e2) d->next_trace[d->next_len++] = kt[i];
  return 1;
}

void* oracle_dpor_open(const demi_config* cfg, const demi_ext_event* ext, uint32_t n_ext,
                       const demi_dpor_params* P, const oracle_dpor_opts* opts) {
  const oracle_model* model = oracle_get_model(cfg->model);
  if (!model) return 0;
  for (uint32_t i = 0; i < n_ext; i++)
    if (ext[i].kind != DEMI_EXT_START && ext[i].kind != DEMI_EXT_SEND) return 0;  /* "unsuported external event" :710 */
  if (P->max_messages + 2 > DP_MAX_T) return 0;
  dpor_t* d = (dpor_t*)calloc(1, sizeof(dpor_t));
  d->params = *P; d->P = &d->params;
  d->ext = (demi_ext_event*)malloc(sizeof(demi_ext_event) * (n_ext + 1)); memcpy(d->ext, ext, sizeof(demi_ext_event) * n_ext); d->n_ext = n_ext;
  if (opts) d->opts = *opts;
  d->m.model = model; d->m.model_flags = cfg->model_flags; d->m.blocked_mask = cfg->blocked_mask;
  d->cap_nodes = P->node_cap; d->nodes = (dnode*)calloc(d->cap_nodes, sizeof(dnode)); d->n_nodes = 1;
  d->explored_slots = P->explored_slots; d->explored = (uint64_t*)malloc(8ull * d->explored_slots);
  memset(d->explored, 0xFF, 8ull * d->explored_slots);
  d->cap_heap = P->heap_cap; d->heap = (bkey*)malloc(sizeof(bkey) * d->cap_heap);
  d->T1 = (uint32_t)P->max_messages + 2;
  d->cap_traces = P->max_interleavings + 1;
  d->traces = (uint32_t*)malloc(4ull * d->cap_traces * d->T1);
  d->trace_len = (uint32_t*)malloc(4ull * d->cap_traces);
  d->path = (uint32_t*)malloc(4ull * (d->cap_nodes + 2 * DP_MAX_T + 4));
  d->max_distance = -1;
  /* setInitialDepGraph (:214-217): the instance starts from the recorded execution's graph */
  if (d->opts.n_init_nodes) {
    if (d->opts.n_init_nodes > d->cap_nodes) { d->status = DEMI_DS_NODE_OVF; return d; }
    d->orig_index = (int32_t*)malloc(4ull * d->opts.n_init_nodes);
    for (uint32_t i = 0; i < d->opts.n_init_nodes; i++) {
      const uint32_t* w = d->opts.init_nodes + 4 * (size_t)i;
      d->nodes[i].msg.src = (uint8_t)(w[0] & 0xFF); d->nodes[i].msg.dst = (uint8_t)((w[0] >> 8) & 0xFF);
      d->nodes[i].msg.type = (uint8_t)((w[0] >> 16) & 0xFF); d->nodes[i].msg.flags = 0;
      d->nodes[i].msg.p0 = w[1]; d->nodes[i].msg.p1 = w[2];
      d->nodes[i].parent = i ? w[3] : 0;
      d->nodes[i].depth = i ? (uint16_t)(d->nodes[w[3]].depth + 1) : 0;
      d->orig_index[i] = -1;
    }
    d->n_nodes = d->opts.n_init_nodes;
    /* ArvindDistanceOrdering.init (BacktrackOrdering.scala:110-116): later occurrences overwrite */
    for (uint32_t i = 0; i < d->opts.n_init_trace; i++)
      if (d->opts.init_trace[i] < d->opts.n_init_nodes) d->orig_index[d->opts.init_trace[i]] = (int32_t)i;
  }
  return d;
}

void oracle_dpor_close(void* s) {
  dpor_t* d = (dpor_t*)s;
  if (!d) return;
  free(d->nodes); free(d->explored); free(d->heap); free(d->traces); free(d->trace_len); free(d->ext);
  free(d->orig_index); free(d->path); free(d);
}

/* One DPORwHeuristics.test (:1193-1242) on a live instance.  max_distance < 0: no setMaxDistance.
 * Returns DEMI_OK / DEMI_ERR_CAPACITY; out->violations > 0 <=> Some(trace). */
int oracle_dpor_test(void* s, int32_t max_distance, demi_dpor_result* out,
                     demi_dpor_violation* viol, uint32_t cap_viol, uint64_t* interleaving_hashes, uint32_t cap_hashes) {
  dpor_t* d = (dpor_t*)s;
  const demi_dpor_params* P = &d->params;
  memset(out, 0, sizeof(*out));
  uint32_t n_viol = 0;
  d->max_distance = max_distance;
  g_dpor = d;
  if (d->status) goto finish;
  if (P->stop_if_found && d->found) { n_viol = 1; goto finish; }                 /* "Already have shortestTrace!" :1197-1201 */
  if (d->n_traces >= P->max_interleavings) { out->budget_exhausted = 1; goto finish; }   /* engine budget, not in the reference */
  /* initialTrace :1219-1221 */
  d->next_len = d->next_pos = 0;
  if (d->started && d->n_heap) {
    if (!dpor_analyse(d, d->n_traces - 1, out)) d->next_len = 0;                 /* None: run() clears nextTrace :757-759 */
  } else if (d->opts.n_init_trace) {
    d->next_rd = d->opts.init_trace; d->next_len = d->opts.n_init_trace;      /* followed whole, however long */
  }
  d->started = 1;
  out->exhausted = 0;
  while (!d->status) {
    uint32_t v = dpor_run_interleaving(d, d->ext, d->n_ext);
    if (d->status) break;
    uint32_t k = d->n_traces++;
    memcpy(d->traces + (size_t)k * d->T1, d->cur_trace, 4ull * d->cur_len);
    d->trace_len[k] = d->cur_len;
    uint64_t sh = schedule_hash(d, d->cur_trace, d->cur_len);
    if (interleaving_hashes && out->interleavings < cap_hashes) interleaving_hashes[out->interleavings] = sh;
    out->interleavings++;
    out->deliveries += d->cur_len - 1;
    if (v) {
      if (viol && n_viol < cap_viol) { viol[n_viol].schedule_hash = sh; viol[n_viol].interleaving = k; viol[n_viol].length = d->cur_len - 1; viol[n_viol].code = v; }
      n_viol++;
      d->found = 1;                                                              /* checkInvariant :404-410 */
      if (P->stop_if_found) break;                                              /* test() returns Some(trace) :1236-1238 */
    }
    if (d->n_traces >= P->max_interleavings) { out->budget_exhausted = 1; break; }
    if (!dpor_analyse(d, k, out)) break;
  }
finish:
  g_dpor = 0;
  out->violations = n_viol;
  out->n_nodes = d->n_nodes; out->n_explored = d->n_explored; out->heap_left = d->n_heap;
  out->status = (uint32_t)d->status;
  return d->status ? DEMI_ERR_CAPACITY : DEMI_OK;
}

int oracle_dpor_search(const demi_config* cfg, const demi_ext_event* ext, uint32_t n_ext,
                       const demi_dpor_params* P, demi_dpor_result* out,
                       demi_dpor_violation* viol, uint32_t cap_viol, uint64_t* interleaving_hashes, uint32_t cap_hashes) {
  memset(out, 0, sizeof(*out));
  void* s = oracle_dpor_open(cfg, ext, n_ext, P, 0);
  if (!s) return DEMI_ERR_INVALID;
  int rc = oracle_dpor_test(s, -1, out, viol, cap_viol, interleaving_hashes, cap_hashes);
  oracle_dpor_close(s);
  return rc;
}
