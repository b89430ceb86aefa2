/*
 * ORACLE — test infrastructure only (see machine.h header).  PARITY UNPINNED
 * against a running reference; pinned by derivable KATs only.
 *
 * STSScheduler.test with WildCardMatch deliveries, on top of the STSSched
 * restatement of sts.c: this file includes sts.c so that it runs on the same
 * machine (its pending set, recording and model callbacks) without changing it.
 * It replaces sts.c in the wildcard build of the oracle (wildcard.mk,
 * liboracle_wildcard.so).
 */
#include "sts.c"
#include "sts_wildcard.h"

/* ------------------------------------------------------- wildcard replay
 * STSScheduler.test of the trace ClockClusterizer.getNextTrace builds (wildcard_minimization/ClockClusterizer.scala:
 * 100-133): an external delivery stays exact; an included delivery of a causesClockIncrement type becomes the
 * "CausesClockIncrement" WildCardMatch, any other included one a class (type) WildCardMatch; a delivery that is not
 * included is left out.  `include` has one bit per MsgEvent of the trace, in trace order; `incr` is the 256-bit
 * type set.  Recording is always on inside (into a private buffer when the caller passes none), so the pending
 * array keeps insertion order, which is Uniq order. */
static int wc_selects(int clock_mode, const uint32_t* incr, uint8_t want_type, const demi_msg* q) {
  if (clock_mode) return (int)((incr[q->type >> 5] >> (q->type & 31)) & 1u);     /* fingerprinter.causesClockIncrement */
  return q->type == want_type;                                                   /* ClassTag(msg.getClass) == classTag */
}
/* messagePending for a WildCardMatch (:381-403): the selector over all pending (snd, rcv) messages */
static int wc_pending(const om_machine* m, int snd, int rcv, int clock_mode, const uint32_t* incr, uint8_t type) {
  for (uint32_t i = 0; i < m->n_pending; i++) {
    const demi_msg* q = &m->pending[i].msg;
    if (q->src == snd && q->dst == rcv && wc_selects(clock_mode, incr, type, q)) return 1;
  }
  return 0;
}
/* schedule_new_message for a WildCardMatch (:696-708): the fingerprint queues of (snd, rcv) sorted by the Uniq id of
 * their head, the selector applied to the heads (BackTrackStrategy: first match; LastOnlyStrategy: last match; the
 * clock-increment selector: indexWhere, i.e. first).  Returns the pending index of the chosen queue's head. */
static int wc_pick(const om_machine* m, int snd, int rcv, int clock_mode, int last, const uint32_t* incr, uint8_t type) {
  int chosen = -1;
  for (uint32_t i = 0; i < m->n_pending; i++) {
    const demi_msg* q = &m->pending[i].msg;
    if (q->src != snd || q->dst != rcv) continue;
    int head = 1;                                                   /* no older pending message with this fingerprint */
    for (uint32_t j = 0; j < i && head; j++) {
      const demi_msg* r = &m->pending[j].msg;
      if (r->src == q->src && r->dst == q->dst && r->type == q->type && r->p0 == q->p0 && r->p1 == q->p1) head = 0;
    }
    if (!head || !wc_selects(clock_mode, incr, type, q)) continue;
    chosen = (int)i;
    if (clock_mode || !last) break;
  }
  return chosen;
}

void oracle_sts_replay_wild(const demi_config* cfg, const demi_replay_input* in, const uint64_t* include,
                            const uint32_t* incr, uint32_t looking_for, uint32_t flags, demi_replay_result* out,
                            demi_event* rec, uint32_t cap_rec, uint32_t* n_rec,
                            uint32_t* ignored, uint32_t cap_ignored, uint32_t* n_ignored) {
  sts_machine* S = (sts_machine*)malloc(sizeof(sts_machine));
  demi_event* own = rec ? 0 : (demi_event*)malloc(sizeof(demi_event) * 65536);
  g_rec = rec ? rec : own; g_rec_cap = rec ? cap_rec : 65536; g_rec_n = 0; g_rec_uniq = 0; g_rec_ovf = 0;
  om_machine* m = &S->m;
  const oracle_model* model = oracle_get_model(cfg->model);
  memset(out, 0, sizeof(*out));
  const uint32_t n = in->n_events;
  uint8_t* keep = (uint8_t*)malloc(n + 1);
  const uint32_t mw = (in->n_externals + 63) / 64 + 1;               /* the full external sequence (the MCS) */
  uint64_t* full = (uint64_t*)malloc(sizeof(uint64_t) * mw);
  memset(full, 0xFF, sizeof(uint64_t) * mw);
  oracle_sts_project(in, full, (flags & DEMI_RF_FILTER_KNOWN_ABSENTS) != 0, keep);
  free(full);
  /* per MsgEvent: 0 exact, 1 class wildcard, 2 clock-increment wildcard; dropped deliveries leave `keep` */
  uint8_t* mode = (uint8_t*)calloc(n + 1, 1);
  uint32_t d = 0;
  for (uint32_t i = 0; i < n; i++) {
    const demi_event* e = &in->events[i];
    if (e->kind != DEMI_EV_MSG_EVENT) continue;
    const int inc = (int)((include[d >> 6] >> (d & 63)) & 1ull);
    d++;
    if (demi_type_is_external(in->external_type_mask, e->type)) continue;          /* EventTypes.isExternal: exact */
    if (!inc) { keep[i] = 0; continue; }
    mode[i] = ((incr[e->type >> 5] >> (e->type & 31)) & 1u) ? 2 : 1;
  }
  const int last = (flags & DEMI_WC_LAST_ONLY) != 0;
  uint32_t n_ign = 0;

  m->model = model; m->model_flags = cfg->model_flags; m->blocked_mask = cfg->blocked_mask;
  m->ignore_timers = cfg->ignore_timers; m->looking_for = looking_for;
  m->pending_cap = in->pending_cap; m->tosend_cap = in->tosend_cap;
  memset(m->states, 0, sizeof(m->states));
  model->init(m->states, cfg->model_flags);
  m->inaccessible = model->n_actors >= 32 ? 0xFFFFFFFFu : ((1u << model->n_actors) - 1u);
  m->killed = 0; memset(m->partitioned, 0, sizeof(m->partitioned));
  m->n_pending = m->max_pending = m->n_tosend = 0;
  m->n_registry = m->n_cancelled = m->n_just = m->n_resend = 0;
  m->status = 0; m->violation = 0;
  S->delivered = S->ignored = 0; S->rhash = 0;
  g_sts_mode = 1;

  uint32_t idx = 0;
  for (;;) {
    sts_flush(m);                                                   /* schedule_new_message :655 */
    int found = 0;
    while (idx < n && !m->status) {                                 /* advanceReplay (:405-559) */
      const demi_event* e = &in->events[idx];
      if (keep[idx]) {
        switch (e->kind) {
          case DEMI_EV_SPAWN:
            rec_push(DEMI_EV_SPAWN, e->src, e->dst, 0, 0, 0, 0);
            m->inaccessible &= ~(1u << e->dst); m->killed &= ~(1u << e->dst); break;
          case DEMI_EV_KILL:
            rec_push(DEMI_EV_KILL, e->src, e->dst, 0, 0, 0, 0);
            m->killed |= 1u << e->dst; m->inaccessible |= 1u << e->dst; break;
          case DEMI_EV_PARTITION: rec_push(DEMI_EV_PARTITION, e->src, e->dst, 0, 0, 0, 0); m->partitioned[e->src] |= 1u << e->dst; break;
          case DEMI_EV_UNPARTITION: rec_push(DEMI_EV_UNPARTITION, e->src, e->dst, 0, 0, 0, 0); m->partitioned[e->src] &= ~(1u << e->dst); break;
          case DEMI_EV_QUIESCENCE: case DEMI_EV_BEGIN_WAIT_QUIESCENCE:
            rec_push(e->kind, e->src, e->dst, 0, 0, 0, 0); break;
          case DEMI_EV_MSG_SEND:
            if (demi_type_is_external(in->external_type_mask, e->type)) {
              demi_msg s; s.src = DEMI_DEADLETTERS; s.dst = e->dst; s.type = e->type; s.flags = DEMI_MF_EXTERNAL;
              s.p0 = e->p0; s.p1 = e->p1;
              sts_tosend_push(m, &s);
            }
            break;
          case DEMI_EV_MSG_EVENT: {
            sts_flush(m);                                           /* messagePending :381-403 */
            const int pend = mode[idx] ? wc_pending(m, e->src, e->dst, mode[idx] == 2, incr, e->type)
                                       : sts_find(m, e->src, e->dst, e->type, e->p0, e->p1) >= 0;
            if (pend && !((m->blocked_mask >> e->dst) & 1u)) found = 1;
            else {                                                  /* "Ignoring message" :528-529; ignoreAbsentCallback */
              S->ignored++;
              if (ignored && n_ign < cap_ignored) ignored[n_ign] = idx;
              n_ign++;
            }
            break;
          }
          default: break;
        }
      }
      if (found) break;
      idx++;
    }
    if (m->status) break;
    sts_flush(m);                                                   /* :682 */
    if (idx >= n) break;
    const demi_event* e = &in->events[idx];
    const int pi = mode[idx] ? wc_pick(m, e->src, e->dst, mode[idx] == 2, last, incr, e->type)
                             : sts_find(m, e->src, e->dst, e->type, e->p0, e->p1);
    const demi_msg msg = m->pending[pi].msg;                        /* the selected message, its own type and payload */
    rec_push(DEMI_EV_MSG_EVENT, msg.src, msg.dst, msg.type, msg.p0, msg.p1, m->pending[pi].uniq);   /* appendMsgEvent :749 */
    sts_remove_at(m, (uint32_t)pi);
    idx++;
    S->rhash += demi_event_term((uint32_t)msg.src | ((uint32_t)msg.dst << 8) | ((uint32_t)msg.type << 16),
                                msg.p0, msg.p1, S->delivered, 0, 0);
    S->delivered++;
    if (key_find(m->registry, m->n_registry, msg.dst, msg.type, msg.p0, msg.p1) >= 0)
      sts_handle_timer(m, msg.dst, msg.type, msg.p0, msg.p1);
    if (m->status) break;
    demi_msg dm = msg; dm.flags = 0;
    model->receive(m, msg.dst, &m->states[msg.dst * model->state_words], &dm);
    if (m->status) break;
  }
  g_sts_mode = 0;

  if (m->status) { out->status = m->status; }
  else {
    uint32_t v = model->invariant(m->states, m->model_flags);       /* :283-289 */
    out->violation = (looking_for ? (v == looking_for ? v : 0) : v);
    out->delivered = (uint16_t)S->delivered;
    out->ignored = (uint16_t)S->ignored;
    uint64_t sh = 0;
    uint32_t nw = (uint32_t)(model->n_actors * model->state_words);
    for (uint32_t i = 0; i < nw; i++) sh += demi_state_term(m->states[i], i);
    out->state_hash = sh + S->rhash;
  }
  if (n_rec) *n_rec = rec ? g_rec_n : 0;
  if (n_ignored) *n_ignored = n_ign;
  if (rec && g_rec_ovf && !out->status) out->status = DEMI_PS_EVENT_OVF;
  g_rec = 0;
  free(keep); free(mode); free(own); free(S);
}
