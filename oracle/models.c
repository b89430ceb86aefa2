/*
 * ORACLE — test infrastructure only (see machine.h header).
 *
 * Built-in actor models.  In the reference the "state-transition functor" is
 * the application's own Akka receive() (Instrumenter.scala:913-1017 hands the
 * envelope to ActorCell.receiveMessage, WeaveActor.aj:90-108); the Raft
 * application DEMi was evaluated on (akka-raft) lives in another repository
 * (README.md:12,27-28) and is NOT under /root/reference.  These models are
 * therefore *models of* such applications, specified in DESIGN.md §3 and
 * implemented twice, independently: here (scalar C) and in
 * demi_b200/csrc/models/ (warp-cooperative CUDA).  PARITY UNPINNED against
 * akka-raft; bit-exact parity is between this file and the CUDA models.
 */
#include <string.h>
#include "machine.h"

/* ============================================================= pingpong3 */
/* BASELINE.json configs[0]: 3-actor ping-pong.  Ping(k) to X => X sends
 * Pong(k) to (X+1)%3.   state: w0 = pings received, w1 = pongs received. */
enum { PP_PING = 1, PP_PONG = 2 };

static void pp_init(uint32_t* st, uint32_t flags) { (void)st; (void)flags; }
static void pp_receive(om_machine* m, int self, uint32_t* st, const demi_msg* msg) {
  if (msg->type == PP_PING) {
    st[0]++;
    om_send(m, self, (self + 1) % 3, PP_PONG, msg->p0, 0);
  } else if (msg->type == PP_PONG) {
    st[1]++;
  }
}
/* flags bit0: test hook — "violation 7" once actor 0 has received >= (flags>>8) pongs */
static uint32_t pp_invariant(const uint32_t* st, uint32_t flags) {
  if ((flags & 1u) && st[1] >= (flags >> 8)) return 7;
  return 0;
}

/* ViolationFingerprint.affectedNodes (TestOracle.scala:9-18): the actors the violation was observed on */
static uint32_t pp_affected(const uint32_t* st, uint32_t flags, uint32_t code) {
  (void)st; (void)flags;
  return code == 7 ? 1u : 0u;
}

/* ================================================================= raft5 */
/* 5-node Raft (Ongaro & Ousterhout, "In Search of an Understandable Consensus
 * Algorithm", Figure 2), tick-driven timers, log capacity 8, one entry per
 * AppendEntries.  State = 10 words, byte layout: */
enum { R_ROLE = 0, R_TERM = 1, R_VOTED = 2, R_VOTES = 3, R_LOGLEN = 4, R_COMMIT = 5, R_HEARD = 6,
       R_PAD = 7, R_LOGTERM = 8, R_LOGVAL = 16, R_NEXT = 24, R_MATCH = 29, R_STATE_BYTES = 40 };
enum { ROLE_INIT = 0, ROLE_FOLLOWER = 1, ROLE_CANDIDATE = 2, ROLE_LEADER = 3 };
enum { RM_BOOT = 1, RM_CLIENT_CMD = 2, RM_ELECTION_TICK = 3, RM_REQUEST_VOTE = 4, RM_VOTE_REPLY = 5,
       RM_HEARTBEAT_TICK = 6, RM_APPEND_ENTRIES = 7, RM_APPEND_REPLY = 8 };
#define RAFT_N 5
#define RAFT_LOG_CAP 8
#define RAFT_NONE 0xFF
#define RAFT_BUG_DOUBLE_VOTE 0x1u   /* grants a vote even if already voted this term */
#define RAFT_BUG_STALE_COMMIT 0x2u  /* leader commits entries of older terms by counting replicas */

static void raft_init(uint32_t* st, uint32_t flags) {
  (void)flags;
  for (int a = 0; a < RAFT_N; a++) {
    uint8_t* s = (uint8_t*)&st[a * 10];
    memset(s, 0, R_STATE_BYTES);
    s[R_VOTED] = RAFT_NONE;
  }
}
static void raft_step_down(om_machine* m, int self, uint8_t* s, uint8_t t) {
  if (s[R_ROLE] == ROLE_LEADER) om_cancel_timer(m, self, RM_HEARTBEAT_TICK, 0, 0);
  if (t > s[R_TERM]) { s[R_TERM] = t; s[R_VOTED] = RAFT_NONE; }
  s[R_ROLE] = ROLE_FOLLOWER;
  s[R_VOTES] = 0;
}
static void raft_send_append(om_machine* m, int self, const uint8_t* s, int j) {
  uint32_t prev = s[R_NEXT + j];
  uint32_t pt = prev ? s[R_LOGTERM + prev - 1] : 0;
  uint32_t has = prev < s[R_LOGLEN];
  uint32_t et = has ? s[R_LOGTERM + prev] : 0, ev = has ? s[R_LOGVAL + prev] : 0;
  om_send(m, self, j, RM_APPEND_ENTRIES,
          (uint32_t)s[R_TERM] | (prev << 8) | (pt << 16) | ((uint32_t)s[R_COMMIT] << 24),
          has | (et << 8) | (ev << 16));
}
/* DESIGN.md §3, raft5 R1: a reply to a non-actor (deadLetters, the sender of an external message) is not issued */
static void raft_reply(om_machine* m, int self, int src, uint8_t type, uint32_t p0) {
  if (src >= RAFT_N) return;
  om_send(m, self, src, type, p0, 0);
}
static void raft_receive(om_machine* m, int self, uint32_t* stw, const demi_msg* msg) {
  uint8_t* s = (uint8_t*)stw;
  uint32_t flags = m->model_flags;
  uint32_t last_idx = s[R_LOGLEN];
  uint32_t last_term = last_idx ? s[R_LOGTERM + last_idx - 1] : 0;
  switch (msg->type) {
    case RM_BOOT:
      if (s[R_ROLE] == ROLE_INIT) {
        s[R_ROLE] = ROLE_FOLLOWER;
        om_schedule_repeating(m, self, RM_ELECTION_TICK, 0, 0);
      }
      break;
    case RM_CLIENT_CMD:
      if (s[R_ROLE] == ROLE_LEADER && s[R_LOGLEN] < RAFT_LOG_CAP) {
        s[R_LOGTERM + s[R_LOGLEN]] = s[R_TERM];
        s[R_LOGVAL + s[R_LOGLEN]] = (uint8_t)(msg->p0 & 0x7F);
        s[R_LOGLEN]++;
      }
      break;
    case RM_ELECTION_TICK:
      if (s[R_ROLE] == ROLE_INIT || s[R_ROLE] == ROLE_LEADER) break;
      if (s[R_HEARD]) { s[R_HEARD] = 0; break; }
      if (s[R_TERM] == 255) break;
      s[R_TERM]++;
      s[R_ROLE] = ROLE_CANDIDATE;
      s[R_VOTED] = (uint8_t)self;
      s[R_VOTES] = (uint8_t)(1u << self);
      for (int j = 0; j < RAFT_N; j++)
        if (j != self)
          om_send(m, self, j, RM_REQUEST_VOTE, (uint32_t)s[R_TERM] | (last_idx << 8) | (last_term << 16), 0);
      break;
    case RM_REQUEST_VOTE: {
      if (s[R_ROLE] == ROLE_INIT) break;
      int c = msg->src;
      uint8_t t = (uint8_t)(msg->p0 & 0xFF);
      uint32_t li = (msg->p0 >> 8) & 0xFF, lt = (msg->p0 >> 16) & 0xFF;
      if (t > s[R_TERM]) raft_step_down(m, self, s, t);
      int up_to_date = lt > last_term || (lt == last_term && li >= last_idx);
      int can_vote = (s[R_VOTED] == RAFT_NONE || s[R_VOTED] == c) || (flags & RAFT_BUG_DOUBLE_VOTE);
      uint32_t grant = (t == s[R_TERM] && can_vote && up_to_date) ? 1u : 0u;
      if (grant) { s[R_VOTED] = (uint8_t)c; s[R_HEARD] = 1; }
      raft_reply(m, self, c, RM_VOTE_REPLY, (uint32_t)s[R_TERM] | (grant << 8));
      break;
    }
    case RM_VOTE_REPLY: {
      if (s[R_ROLE] == ROLE_INIT) break;
      uint8_t t = (uint8_t)(msg->p0 & 0xFF);
      uint32_t g = (msg->p0 >> 8) & 1u;
      if (t > s[R_TERM]) { raft_step_down(m, self, s, t); break; }
      if (msg->src >= RAFT_N) break;                  /* DESIGN.md §3, raft5 R2: no vote from a non-actor */
      if (s[R_ROLE] == ROLE_CANDIDATE && t == s[R_TERM] && g) {
        s[R_VOTES] |= (uint8_t)(1u << msg->src);
        if (__builtin_popcount(s[R_VOTES]) >= 3) {
          s[R_ROLE] = ROLE_LEADER;
          for (int j = 0; j < RAFT_N; j++) { s[R_NEXT + j] = s[R_LOGLEN]; s[R_MATCH + j] = 0; }
          if (s[R_LOGLEN] < RAFT_LOG_CAP) {       /* leader no-op entry */
            s[R_LOGTERM + s[R_LOGLEN]] = s[R_TERM];
            s[R_LOGVAL + s[R_LOGLEN]] = (uint8_t)(0x80 | self);
            s[R_LOGLEN]++;
          }
          for (int j = 0; j < RAFT_N; j++) if (j != self) raft_send_append(m, self, s, j);
          om_schedule_repeating(m, self, RM_HEARTBEAT_TICK, 0, 0);
        }
      }
      break;
    }
    case RM_HEARTBEAT_TICK:
      if (s[R_ROLE] == ROLE_LEADER)
        for (int j = 0; j < RAFT_N; j++) if (j != self) raft_send_append(m, self, s, j);
      break;
    case RM_APPEND_ENTRIES: {
      if (s[R_ROLE] == ROLE_INIT) break;
      int l = msg->src;
      uint8_t t = (uint8_t)(msg->p0 & 0xFF);
      uint32_t prev = (msg->p0 >> 8) & 0xFF, pt = (msg->p0 >> 16) & 0xFF, lc = (msg->p0 >> 24) & 0xFF;
      uint32_t has = msg->p1 & 1u, et = (msg->p1 >> 8) & 0xFF, ev = (msg->p1 >> 16) & 0xFF;
      if (t < s[R_TERM]) { raft_reply(m, self, l, RM_APPEND_REPLY, (uint32_t)s[R_TERM]); break; }
      if (t > s[R_TERM] || s[R_ROLE] != ROLE_FOLLOWER) raft_step_down(m, self, s, t);
      s[R_HEARD] = 1;
      int ok = prev <= s[R_LOGLEN] && (prev == 0 || s[R_LOGTERM + prev - 1] == pt);
      if (!ok) { raft_reply(m, self, l, RM_APPEND_REPLY, (uint32_t)s[R_TERM]); break; }
      uint32_t mi = prev;
      if (has) {
        if (s[R_LOGLEN] > prev && s[R_LOGTERM + prev] != et) {      /* conflict: truncate */
          for (uint32_t k = prev; k < RAFT_LOG_CAP; k++) { s[R_LOGTERM + k] = 0; s[R_LOGVAL + k] = 0; }
          s[R_LOGLEN] = (uint8_t)prev;
        }
        if (s[R_LOGLEN] == prev && prev < RAFT_LOG_CAP) {
          s[R_LOGTERM + prev] = (uint8_t)et; s[R_LOGVAL + prev] = (uint8_t)ev;
          s[R_LOGLEN] = (uint8_t)(prev + 1);
        }
        if (s[R_LOGLEN] > prev) mi = prev + 1;
      }
      uint32_t nc = lc < mi ? lc : mi;
      if (nc > s[R_COMMIT]) s[R_COMMIT] = (uint8_t)nc;
      raft_reply(m, self, l, RM_APPEND_REPLY, (uint32_t)s[R_TERM] | (1u << 8) | (mi << 16));
      break;
    }
    case RM_APPEND_REPLY: {
      if (s[R_ROLE] == ROLE_INIT) break;
      int j = msg->src;
      uint8_t t = (uint8_t)(msg->p0 & 0xFF);
      uint32_t ok = (msg->p0 >> 8) & 1u, mi = (msg->p0 >> 16) & 0xFF;
      if (t > s[R_TERM]) { raft_step_down(m, self, s, t); break; }
      if (s[R_ROLE] != ROLE_LEADER || t != s[R_TERM]) break;
      if (j >= RAFT_N) break;                         /* DESIGN.md §3, raft5 R2: nothing indexed by a non-actor */
      if (ok) {
        if (mi > s[R_MATCH + j]) s[R_MATCH + j] = (uint8_t)mi;
        if (mi > s[R_NEXT + j]) s[R_NEXT + j] = (uint8_t)mi;
        for (uint32_t idx = s[R_LOGLEN]; idx > s[R_COMMIT]; idx--) {
          if (s[R_LOGTERM + idx - 1] != s[R_TERM] && !(flags & RAFT_BUG_STALE_COMMIT)) continue;
          int cnt = 1;
          for (int k = 0; k < RAFT_N; k++) if (k != self && s[R_MATCH + k] >= idx) cnt++;
          if (cnt >= 3) { s[R_COMMIT] = (uint8_t)idx; break; }
        }
      } else if (s[R_NEXT + j] > 0) {
        s[R_NEXT + j]--;
      }
      break;
    }
    default: break;
  }
}
/* code 1: election safety (two leaders in one term);
 * code 2: state-machine safety (committed prefixes disagree). */
static uint32_t raft_invariant(const uint32_t* st, uint32_t flags) {
  (void)flags;
  for (int i = 0; i < RAFT_N; i++)
    for (int j = i + 1; j < RAFT_N; j++) {
      const uint8_t* a = (const uint8_t*)&st[i * 10];
      const uint8_t* b = (const uint8_t*)&st[j * 10];
      if (a[R_ROLE] == ROLE_LEADER && b[R_ROLE] == ROLE_LEADER && a[R_TERM] == b[R_TERM]) return 1;
    }
  for (int i = 0; i < RAFT_N; i++)
    for (int j = i + 1; j < RAFT_N; j++) {
      const uint8_t* a = (const uint8_t*)&st[i * 10];
      const uint8_t* b = (const uint8_t*)&st[j * 10];
      uint32_t c = a[R_COMMIT] < b[R_COMMIT] ? a[R_COMMIT] : b[R_COMMIT];
      for (uint32_t k = 0; k < c; k++)
        if (a[R_LOGTERM + k] != b[R_LOGTERM + k] || a[R_LOGVAL + k] != b[R_LOGVAL + k]) return 2;
    }
  return 0;
}

/* the first pair, in (i, j) order, that witnesses `code` */
static uint32_t raft_affected(const uint32_t* st, uint32_t flags, uint32_t code) {
  (void)flags;
  for (int i = 0; i < RAFT_N; i++)
    for (int j = i + 1; j < RAFT_N; j++) {
      const uint8_t* a = (const uint8_t*)&st[i * 10];
      const uint8_t* b = (const uint8_t*)&st[j * 10];
      if (code == 1 && a[R_ROLE] == ROLE_LEADER && b[R_ROLE] == ROLE_LEADER && a[R_TERM] == b[R_TERM])
        return (1u << i) | (1u << j);
      if (code == 2) {
        uint32_t c = a[R_COMMIT] < b[R_COMMIT] ? a[R_COMMIT] : b[R_COMMIT];
        for (uint32_t k = 0; k < c; k++)
          if (a[R_LOGTERM + k] != b[R_LOGTERM + k] || a[R_LOGVAL + k] != b[R_LOGVAL + k]) return (1u << i) | (1u << j);
      }
    }
  return 0;
}

/* =============================================================== bcast32 */
/* BASELINE.json configs[4]: 32-actor broadcast storm.  Flood(ttl) => count++,
 * remember the largest ttl seen, re-broadcast Flood(ttl-1) to all 31 peers
 * while ttl > 0.   state: w0 = count, w1 = max ttl seen + 1. */
enum { BC_FLOOD = 1, BC_INJECT = 2 };   /* INJECT: the external seed message, handled like FLOOD */
static void bc_init(uint32_t* st, uint32_t flags) { (void)st; (void)flags; }
static void bc_receive(om_machine* m, int self, uint32_t* st, const demi_msg* msg) {
  if (msg->type != BC_FLOOD && msg->type != BC_INJECT) return;
  st[0]++;
  if (msg->p0 + 1 > st[1]) st[1] = msg->p0 + 1;
  if (msg->p0 > 0)
    for (int j = 0; j < 32; j++)
      if (j != self) om_send(m, self, j, BC_FLOOD, msg->p0 - 1, 0);
}
/* violation 3 once some actor has received >= flags floods (flags != 0) */
static uint32_t bc_invariant(const uint32_t* st, uint32_t flags) {
  if (!flags) return 0;
  for (int a = 0; a < 32; a++) if (st[a * 2] >= flags) return 3;
  return 0;
}

static uint32_t bc_affected(const uint32_t* st, uint32_t flags, uint32_t code) {
  if (code != 3 || !flags) return 0;
  for (int a = 0; a < 32; a++) if (st[a * 2] >= flags) return 1u << a;
  return 0;
}

static const oracle_model MODELS[] = {
  { DEMI_MODEL_PINGPONG3, 3, 2, pp_init, pp_receive, pp_invariant, pp_affected },
  { DEMI_MODEL_RAFT5, 5, 10, raft_init, raft_receive, raft_invariant, raft_affected },
  { DEMI_MODEL_BCAST32, 32, 2, bc_init, bc_receive, bc_invariant, bc_affected },
};
extern const oracle_model ORACLE_IR_MODEL;      /* model_ir.c: a model loaded with oracle_load_model */
int oracle_ir_loaded(void);
const oracle_model* oracle_get_model(int id) {
  if (id == ORACLE_IR_MODEL.id) return oracle_ir_loaded() ? &ORACLE_IR_MODEL : 0;
  for (unsigned i = 0; i < sizeof(MODELS) / sizeof(MODELS[0]); i++)
    if (MODELS[i].id == id) return &MODELS[i];
  return 0;
}
