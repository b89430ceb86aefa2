// replay_kernel.cuh — K2: batched STSScheduler.test (schedulers/STSScheduler.scala:
// 199-310).  One THREAD owns one test, i.e. one external-event subsequence
// (a bitmask over EventTrace.original_externals); the 32 lanes of a warp walk
// the SAME recorded trace in lock-step, so every lane handles the same event at
// the same time and the actor transition that runs for an expected delivery is
// the same message type in all lanes (near-zero divergence).
//
// Per event i (uniform) each lane evaluates, fused in one pass:
//   subsequenceIntersection (EventTrace.scala:290-380)      -> keep / drop
//   filterSends             (EventTrace.scala:382-452)      -> keep / drop
//   filterKnownAbsentInternals (EventTrace.scala:458-534)   -> keep / drop (optional)
// and, for kept events, the STSSched step: advanceReplay (:405-559),
// schedule_new_message (:643-776), event_produced (:561-623).
//
// Data layout: the trace + side tables are shared by the whole batch and stay
// L2/L1 resident (24 KB for 2000 events).  Per test: actor states / outbox /
// partition rows thread-interleaved in shared memory; the pending multiset
// ((snd,rcv) -> fingerprint -> FIFO of indistinguishable entries,
// STSScheduler.scala:112-114) is an open-addressing hash table of
// {hdr,p0,p1,generation|count} in HBM, interleaved per warp.
#pragma once
#include "actor_step.cuh"
#include "replay_trace.hpp"

namespace demi {

struct ReplayArgs {
  uint32_t model_flags, blocked_mask;
  int32_t  ignore_timers;
  uint32_t looking_for, flags;
  // trace (shared by all tests)
  const uint4* events; uint32_t n_events;        // demi_event records
  const uint16_t* ev_ordinal;                    // per event: FIFO ordinal of the external Send it belongs to, 0xFFFF if none
  const uint4* ext; uint32_t n_ext;              // demi_ext_event records (original_externals)
  const uint16_t* send_ext_index; uint32_t n_sends;   // j-th original Send -> its index in ext
  uint32_t external_type_mask;
  uint32_t n_uniq_words;                         // words of the per-test pruned-send bitset
  // tests
  const uint64_t* masks; uint32_t n_masks, mask_words;   // masks == nullptr: every test uses the full subsequence
  const uint32_t* skips;                                   // optional: test i also drops trace event skips[i]
  demi_replay_result* results;
  // recording (single-test launches of the REC variant): the EventTrace STSScheduler.test returns
  demi_event* rec_events; uint32_t rec_cap; uint32_t* rec_count;
  // capacities
  uint32_t pending_cap, tosend_cap, table_slots; // table_slots: power of two >= 2*pending_cap
  uint32_t gen_base;                             // first hash-table generation this launch may use (1..0xFFFE)
  // per-warp scratch in HBM
  uint4*    table;      // [warps][table_slots][32]
  uint32_t* tosend;     // [warps][tosend_cap][32]
  uint32_t* pruned;     // [warps][n_uniq_words + N][32]  (only with DEMI_RF_FILTER_KNOWN_ABSENTS)
  unsigned long long* counters;   // [0] reproduced, [1] delivered
  // wildcard replay (WILD instantiations only; the others ignore these): per trace event, for MsgEvents,
  // mode << 16 | delivery ordinal; include masks over deliveries; the causesClockIncrement type set; the
  // trace positions of ignored deliveries (REC launches: one list, or with ROWS a row of wc_ignored_cap per test)
  const uint32_t* wc_ev; const uint64_t* wc_include; uint32_t wc_words;
  uint32_t wc_incr[8];
  uint32_t* wc_ignored; uint32_t wc_ignored_cap; uint32_t* wc_ignored_count;
};

// a's trace: the host binds the single trace (demi_set_trace), replay_many_kernel each tile's trace of a set
__host__ __device__ __forceinline__ void bind_trace(ReplayArgs& a, const ReplayTraceView& v) {
  a.events = v.events; a.n_events = v.n_events; a.ev_ordinal = v.ev_ordinal;
  a.ext = v.ext; a.n_ext = v.n_ext; a.send_ext_index = v.send_ext_index; a.n_sends = v.n_sends;
  a.n_uniq_words = v.n_uniq_words; a.pending_cap = v.pending_cap; a.tosend_cap = v.tosend_cap;
  a.table_slots = v.table_slots;
}

// K2's block size per model: a test's actor states are thread-interleaved in shared memory, so the models of more than
// eight actors (bcast32, a loaded model) run half the threads per block
template <class MODEL> constexpr int replay_block = MODEL::N_ACTORS <= 8 ? 256 : 128;

// WILD: ClockClusterizer's wildcarded trace (capi_wildcard.cu).  The pending set is the insertion-ordered list of
// the REC variant (Uniq order = list order), compacted in place when taken entries dominate it.
// ROWS (with REC): many recordings in one launch; test idx records into row idx of rec_events (rec_cap events each)
// and its count into rec_count[idx]; with WILD also the trace positions of its ignored deliveries into row idx of
// wc_ignored (wc_ignored_cap each) and their count into wc_ignored_count[idx].  The row pointers are members of the
// machines that record rows only, so the other instantiations keep their layout (a loaded model's machine lives in the
// stack frame).
template <bool ROWS, bool WILD> struct RecRow { uint4* rec_row; };
template <> struct RecRow<true, true> { uint4* rec_row; uint32_t* ign_row; };
template <bool WILD> struct RecRow<false, WILD> {};
template <class MODEL, int BD, bool REC = false, bool WILD = false, bool ROWS = false>
struct ReplayMachine : TimerTable<MODEL>, RecRow<ROWS, WILD> {
  using Model = MODEL;
  static constexpr int BLOCK = BD;
  static constexpr bool LIST = REC || WILD;
  static constexpr int N = MODEL::N_ACTORS;
  static constexpr int SW = MODEL::STATE_WORDS;
  static constexpr int OB = MODEL::REPLAY_OUTBOX;
  static constexpr bool DIRECT = model_replay_direct<MODEL>::value;
  static constexpr int OBW = DIRECT ? 0 : OB * 3;      // the outbox is staged in shared memory only when it can overflow
  static constexpr uint32_t UNSUPPORTED = DEMI_RS_UNSUPPORTED, QUEUE_OVF = DEMI_PS_QUEUE_OVF;
  static constexpr int WORDS = N * SW + OBW + N;

  uint32_t* smw;
  const ReplayArgs* A;
  uint4* table; uint32_t* tosend; uint32_t* pruned;
  const uint64_t* mask;

  uint32_t gen;                      // hash-table generation of this test
  uint32_t n_pending, n_tosend;
  typename TimerTable<MODEL>::mask_t registry, cancelled;      // timer-slot bitmasks
  uint32_t inaccessible, killed;
  uint32_t status;
  uint32_t delivered, ignored;
  uint64_t rhash;
  // projection state
  uint32_t rem_cursor;               // next candidate index into ext for `remaining.head`
  uint32_t alive;                    // filterKnownAbsentInternals: actorToAlive

  __device__ __forceinline__ uint32_t& part_row(uint32_t a) { return smw[(N * SW + OBW + a) * BD]; }
  __device__ __forceinline__ LaneState actor(uint32_t a) { return LaneState{smw + a * SW * BD, BD}; }
  // externals are consulted in (nearly) increasing index order: keep the current 64-bit word of the mask in registers
  uint32_t mword_idx; uint64_t mword;
  __device__ __forceinline__ bool in_mask(uint32_t i) {
    if (!mask) return true;
    const uint32_t w = i >> 6;
    if (w != mword_idx) { mword_idx = w; mword = __ldg(mask + w); }
    return (mword >> (i & 63)) & 1ull;
  }
  // ---- recording (REC): trace + Uniq ids; the pending set becomes an insertion-ordered list so that
  // equal messages leave oldest-first (Queue.dequeue, STSScheduler.scala:729) and Uniq ids pair up
  uint32_t n_rec, n_uniq, n_list;
  __device__ __forceinline__ void rec_push(uint32_t kind, uint32_t src, uint32_t dst, uint32_t type,
                                           uint32_t p0, uint32_t p1, uint32_t uniq) {
    if (!REC) return;
    if (n_rec >= A->rec_cap) { status = DEMI_PS_EVENT_OVF; return; }
    uint4* row;                      // ROWS: this test's row (A is the warp's, the row the lane's own)
    if constexpr (ROWS) row = this->rec_row; else row = reinterpret_cast<uint4*>(A->rec_events);
    row[n_rec++] = make_uint4(kind | (src << 8) | (dst << 16) | (type << 24), p0, p1, uniq);
  }

  // ---- pending multiset
  __device__ __forceinline__ uint32_t hash_key(uint32_t hdr, uint32_t p0, uint32_t p1) const {
    return demi_fmix32((hdr * 0x9E3779B1u) ^ (p0 * 0x85EBCA77u) ^ (p1 * 0xC2B2AE3Du)) & (A->table_slots - 1);
  }
  // returns slot index of the key (live in this generation) or of the first free slot; found tells which
  __device__ __forceinline__ uint32_t probe(uint32_t hdr, uint32_t p0, uint32_t p1, bool& found, uint32_t& count) {
    uint32_t s = hash_key(hdr, p0, p1);
    for (uint32_t tries = 0;; tries++) {
      if (tries >= A->table_slots) { status = DEMI_RS_UNSUPPORTED; found = false; count = 0; return s; }
      uint4 q = table[(size_t)s * 32];
      if ((q.w >> 16) != gen) { found = false; count = 0; return s; }
      if (q.x == hdr && q.y == p0 && q.z == p1) { found = true; count = q.w & 0xFFFFu; return s; }
      s = (s + 1) & (A->table_slots - 1);
    }
  }
  // ---- WILD: list entries before list_lo are all taken; list_compact squeezes the taken entries out, order kept
  uint32_t list_lo;
  __device__ __forceinline__ void list_compact() {
    uint32_t j = 0;
    for (uint32_t i = list_lo; i < n_list; i++) {
      uint4 q = table[(size_t)i * 32];
      if (q.w & 0x80000000u) table[(size_t)(j++) * 32] = q;
    }
    n_list = j; list_lo = 0;
  }
  __device__ __forceinline__ void list_take(uint32_t i, uint4 q) {
    table[(size_t)i * 32] = make_uint4(q.x, q.y, q.z, q.w & 0x7FFFFFFFu);
    n_pending--;
    if (WILD && i == list_lo)
      while (list_lo < n_list && !(table[(size_t)list_lo * 32].w & 0x80000000u)) list_lo++;
  }
  __device__ __forceinline__ bool wc_incr(uint32_t type) const { return (A->wc_incr[type >> 5] >> (type & 31)) & 1u; }
  // The pending message a wildcard delivery from snd to rcv takes (STSScheduler.messagePending :381-403 and
  // schedule_new_message :696-708): list position, or -1 when none matches.  The fingerprint queues of (snd, rcv)
  // in the order of their head's Uniq id are the list's live entries of (snd, rcv) that no older live entry shares
  // a fingerprint with.  The oldest matching message heads the first matching queue (BackTrackStrategy,
  // ClockClusterizer.scala:107-112 for the clock-increment selector); LastOnlyStrategy takes the newest such head.
  __device__ __forceinline__ int wild_pick(uint32_t snd, uint32_t rcv, uint32_t mode, uint32_t type, bool last) {
    const uint32_t pair = snd | (rcv << 8);
    int pick = -1;
    // Last: the payloads of the queue heads met so far (a class selector matches one header, so the payload is the
    // fingerprint); past HEADS of them an entry is checked against every older entry instead
    constexpr uint32_t HEADS = 8;
    uint32_t seen_p0[HEADS], seen_p1[HEADS], n_seen = 0;
    for (uint32_t i = list_lo; i < n_list; i++) {
      const uint4 q = table[(size_t)i * 32];
      if (!(q.w & 0x80000000u) || (q.x & 0xFFFFu) != pair) continue;
      const uint32_t t = (q.x >> 16) & 0xFF;
      if (!(mode == WC_CLOCK ? wc_incr(t) : t == type)) continue;
      if (mode == WC_CLOCK || !last) return (int)i;
      bool head = true;
      for (uint32_t k = 0; k < n_seen && k < HEADS && head; k++) head = !(seen_p0[k] == q.y && seen_p1[k] == q.z);
      for (uint32_t j = list_lo; head && n_seen > HEADS && j < i; j++) {
        const uint4 r = table[(size_t)j * 32];
        head = !((r.w & 0x80000000u) && r.x == q.x && r.y == q.y && r.z == q.z);
      }
      if (head) {
        pick = (int)i;
        if (n_seen < HEADS) { seen_p0[n_seen] = q.y; seen_p1[n_seen] = q.z; }
        n_seen++;
      }
    }
    return pick;
  }

  __device__ __forceinline__ void pending_add(uint32_t hdr, uint32_t p0, uint32_t p1, uint32_t uniq = 0) {
    if (n_pending >= A->pending_cap) { status = DEMI_PS_PENDING_OVF; return; }
    if (LIST) {
      // n_pending < pending_cap <= table_slots, so compacting a full list frees a slot; compacting once dead entries
      // outnumber live ones keeps every scan short (amortised O(1) per operation)
      if (WILD && (n_list >= A->table_slots || n_list - list_lo >= 2 * n_pending + 32)) list_compact();
      if (n_list >= A->table_slots) { status = DEMI_RS_UNSUPPORTED; return; }
      table[(size_t)n_list * 32] = make_uint4(hdr, p0, p1, uniq | 0x80000000u);
      n_list++; n_pending++;
      return;
    }
    bool found; uint32_t count;
    uint32_t s = probe(hdr, p0, p1, found, count);
    if (status) return;
    table[(size_t)s * 32] = make_uint4(hdr, p0, p1, (gen << 16) | (count + 1));
    n_pending++;
  }
  __device__ __forceinline__ bool pending_take(uint32_t hdr, uint32_t p0, uint32_t p1, uint32_t* uniq_out = nullptr) {
    if (LIST) {
      for (uint32_t i = WILD ? list_lo : 0; i < n_list; i++) {
        uint4 q = table[(size_t)i * 32];
        if ((q.w & 0x80000000u) && q.x == hdr && q.y == p0 && q.z == p1) {
          if (uniq_out) *uniq_out = q.w & 0xFFFFu;
          list_take(i, q);
          return true;
        }
      }
      return false;
    }
    bool found; uint32_t count;
    uint32_t s = probe(hdr, p0, p1, found, count);
    if (!found || count == 0) return false;
    table[(size_t)s * 32] = make_uint4(hdr, p0, p1, (gen << 16) | (count - 1));
    n_pending--;
    return true;
  }
  __device__ __forceinline__ bool pending_has(uint32_t hdr, uint32_t p0, uint32_t p1) {
    bool found; uint32_t count;
    probe(hdr, p0, p1, found, count);
    return found && count > 0;
  }

  __device__ __forceinline__ bool crosses_partition(uint32_t snd, uint32_t rcv) {
    bool snd_actor = snd < DEMI_MAX_ACTORS;
    if (snd == rcv && !((killed >> snd) & 1u)) return false;
    if (snd_actor) {
      if ((part_row(snd) >> rcv) & 1u) return true;
      if ((part_row(rcv) >> snd) & 1u) return true;
    }
    if ((inaccessible >> rcv) & 1u) return true;
    if (snd_actor && ((inaccessible >> snd) & 1u)) return true;
    return false;
  }

  // STSScheduler.event_produced (STSScheduler.scala:561-623) after the cancelled-timer drop
  __device__ __forceinline__ void event_produced(uint32_t src, uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1,
                                                 bool external = false) {
    if (status) return;
    if (timer_dropped(*this, dst, type, p0, p1)) return;
    uint32_t uniq = 0;
    if (LIST) {
      uniq = ++n_uniq & 0xFFFFu;                                    // Uniq(...) :570, 16-bit (DESIGN.md §2); appendMsgSend :620-622
      rec_push(DEMI_EV_MSG_SEND, (!external && src == DEMI_DEADLETTERS) ? DEMI_TIMER_SND : src, dst, type, p0, p1, uniq);
    }
    if (!external && crosses_partition(src, dst)) return;
    pending_add(make_hdr(src, dst, type, 0), p0, p1, uniq);
  }
  __device__ __forceinline__ void tosend_push(uint32_t code) {
    if (n_tosend >= A->tosend_cap) { status = DEMI_PS_QUEUE_OVF; return; }
    tosend[(size_t)n_tosend * 32] = code;
    n_tosend++;
  }
  // ExternalEventInjector.send_external_messages: codes are (1<<31 | event index) for
  // externals re-sent from the trace, else a timer slot
  __device__ __forceinline__ void flush() {
    for (uint32_t i = 0; i < n_tosend && !status; i++) {
      uint32_t code = tosend[(size_t)i * 32];
      if (code & 0x80000000u) {
        uint4 e = __ldg(A->events + (code & 0x7FFFFFFFu));
        event_produced(DEMI_DEADLETTERS, (e.x >> 16) & 0xFF, e.x >> 24, e.y, e.z, true);
      } else {
        uint32_t dst, type, p0, p1;
        timer_msg(*this, code, dst, type, p0, p1);
        event_produced(DEMI_DEADLETTERS, dst, type, p0, p1, false);
      }
    }
    n_tosend = 0;
    timer_flushed(*this);
  }
  // ExternalEventInjector.handle_timer: into messagesToSend unless ignoreTimers (STSScheduler.enqueue_timer :870)
  __device__ __forceinline__ void enqueue_timer(uint32_t slot) {
    if (A->ignore_timers) return;
    timer_queued(*this, slot);
    tosend_push(slot);
  }
  // the cancelled timer's pending copy (STSScheduler.notify_timer_cancel :846-868)
  __device__ __forceinline__ void cancel_pending(uint32_t self, uint32_t slot, uint32_t type, uint32_t p0, uint32_t p1) {
    for (uint32_t i = 0; i < n_tosend; i++)
      if (tosend[(size_t)i * 32] == slot) {                         // order-preserving removal
        for (uint32_t j = i; j + 1 < n_tosend; j++) tosend[(size_t)j * 32] = tosend[(size_t)(j + 1) * 32];
        n_tosend--;
        return;
      }
    pending_take(make_hdr(DEMI_DEADLETTERS, self, type, 0), p0, p1);
  }

  __device__ __forceinline__ void deliver(uint32_t src, uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) {
    rhash += demi_event_term(src | (dst << 8) | (type << 16), p0, p1, delivered, 0, 0);
    delivered++;
    timer_rearm(*this, dst, type, p0, p1);
    if (status) return;
    actor_receive<DIRECT>(*this, src, dst, type, p0, p1);
    flush();     // schedule_new_message begins with send_external_messages (:655)
  }

  // WILD + REC: the trace positions of ignored deliveries, from which WildcardMinimizer takes ignoredAbsentIds
  // (WildcardMinimizer.scala:197-235)
  const uint64_t* wc_inc; uint32_t n_ign;
  __device__ __forceinline__ void note_ignored(uint32_t i) {
    if (!(WILD && REC)) return;
    if constexpr (ROWS && WILD) { if (n_ign < A->wc_ignored_cap) this->ign_row[n_ign] = i; }
    else if (A->wc_ignored && n_ign < A->wc_ignored_cap) A->wc_ignored[n_ign] = i;
    n_ign++;
  }

  __device__ __forceinline__ void run(uint32_t test_idx, uint32_t generation, demi_replay_result& out) {
    mask = A->masks ? A->masks + (size_t)test_idx * A->mask_words : nullptr;
    mword_idx = 0xFFFFFFFFu; mword = 0;
    const uint32_t skip = A->skips ? A->skips[test_idx] : 0xFFFFFFFFu;
    n_rec = n_uniq = n_list = 0;       // the list is rebuilt from its first entry: nothing of a previous test is read
    if constexpr (ROWS) this->rec_row = reinterpret_cast<uint4*>(A->rec_events) + (size_t)test_idx * A->rec_cap;
    if constexpr (ROWS && WILD) this->ign_row = A->wc_ignored + (size_t)test_idx * A->wc_ignored_cap;
    if constexpr (WILD) { wc_inc = A->wc_include + (size_t)test_idx * A->wc_words; list_lo = 0; n_ign = 0; }
    gen = generation;
    actor_init(*this);
    for (uint32_t a = 0; a < N; a++) part_row(a) = 0;
    n_pending = n_tosend = 0; registry = cancelled = 0; timer_reset(*this);
    inaccessible = (N >= 32) ? 0xFFFFFFFFu : ((1u << N) - 1u);
    killed = 0; status = 0; delivered = ignored = 0; rhash = 0;
    rem_cursor = 0; alive = 0;
    const bool fka = (A->flags & DEMI_RF_FILTER_KNOWN_ABSENTS) != 0;
    const bool strict = (A->flags & DEMI_RF_STRICT) != 0;
    // filterKnownAbsentInternals: prunedMessageSends bitset, then N rows of actorsToPartitioned flags
    if (fka) for (uint32_t w = 0; w < A->n_uniq_words + N; w++) pruned[(size_t)w * 32] = 0;
#define PF_ROW(a) pruned[(size_t)(A->n_uniq_words + (a)) * 32]
    bool diverged = false;
    const uint32_t n_ev = A->n_events;

    // the walk is one dependent chain per test; the next event and its ordinal are fetched a step ahead so that their
    // L2 latency overlaps the current event's work
    uint4 e_next = n_ev ? __ldg(A->events) : make_uint4(0, 0, 0, 0);
    uint32_t ord_next = n_ev ? __ldg(A->ev_ordinal) : 0xFFFFu;
    for (uint32_t i = 0; i < n_ev && !status && !diverged; i++) {
      const uint4 e = e_next;
      const uint32_t ord_cur = ord_next;
      if (i + 1 < n_ev) { e_next = __ldg(A->events + i + 1); ord_next = __ldg(A->ev_ordinal + i + 1); }
      const uint32_t kind = e.x & 0xFF, src = (e.x >> 8) & 0xFF, dst = (e.x >> 16) & 0xFF, type = e.x >> 24;
      const uint32_t uniq = e.w & 0xFFFF;
      const bool is_msg = kind == DEMI_EV_MSG_SEND || kind == DEMI_EV_MSG_EVENT;
      bool k = false;
      // ---- pass 1: subsequenceIntersection (EventTrace.scala:307-374)
      if (is_msg || kind == DEMI_EV_QUIESCENCE || kind == DEMI_EV_BEGIN_WAIT_QUIESCENCE) {
        k = true;
      } else {
        // advance to `remaining.head`: next external in the subsequence that is not a Send
        while (rem_cursor < A->n_ext) {
          uint32_t xk = __ldg(A->ext + rem_cursor).x & 0xFF;
          if (xk != DEMI_EXT_SEND && in_mask(rem_cursor)) break;
          rem_cursor++;
        }
        if (rem_cursor < A->n_ext) {
          uint32_t hx = __ldg(A->ext + rem_cursor).x;
          uint32_t hk = hx & 0xFF, ha = (hx >> 8) & 0xFF, hb = (hx >> 16) & 0xFF;
          if (kind == DEMI_EV_KILL) k = (hk == DEMI_EXT_KILL && ha == dst);
          else if (kind == DEMI_EV_SPAWN) k = (hk == DEMI_EXT_START && ha == dst);
          else if (kind == DEMI_EV_PARTITION) k = (hk == DEMI_EXT_PARTITION && ha == src && hb == dst);
          else if (kind == DEMI_EV_UNPARTITION) k = (hk == DEMI_EXT_UNPARTITION && ha == src && hb == dst);
          if (k) rem_cursor++;
        }   // remaining.isEmpty: external-type events are dropped (:308-314)
      }
      // ---- pass 2: filterSends (EventTrace.scala:425-446), FIFO-ordinal form
      if (k && is_msg) {
        const uint32_t ord = ord_cur;
        if (ord < A->n_sends && !in_mask(__ldg(A->send_ext_index + ord))) k = false;
      }
      // ---- pass 3: filterKnownAbsentInternals (EventTrace.scala:501-532), as written
      if (k && fka) {
        if (kind == DEMI_EV_MSG_SEND) {
          bool snd_alive = src >= DEMI_MAX_ACTORS || ((alive >> src) & 1u);
          bool parted = src < DEMI_MAX_ACTORS && ((PF_ROW(src) >> dst) & 1u);
          if (!(snd_alive && !parted)) { k = false; pruned[(size_t)(uniq >> 5) * 32] |= 1u << (uniq & 31); }
        } else if (kind == DEMI_EV_MSG_EVENT) {
          bool rcv_alive = (alive >> dst) & 1u;
          bool parted = src < DEMI_MAX_ACTORS && ((PF_ROW(src) >> dst) & 1u);
          bool ps = (pruned[(size_t)(uniq >> 5) * 32] >> (uniq & 31)) & 1u;
          if (!(rcv_alive && !parted && !ps)) k = false;
        } else if (kind == DEMI_EV_SPAWN) alive |= 1u << dst;
        else if (kind == DEMI_EV_KILL) alive &= ~(1u << dst);
        else if (kind == DEMI_EV_PARTITION) PF_ROW(src) &= ~(1u << dst);
        else if (kind == DEMI_EV_UNPARTITION) PF_ROW(src) |= 1u << dst;
      }
      if (!k || i == skip) continue;
      uint32_t wmode = WC_EXACT;
      if constexpr (WILD) {
        if (kind == DEMI_EV_MSG_EVENT) {                             // ClockClusterizer.getNextTrace (:101-126)
          const uint32_t w = __ldg(A->wc_ev + i), d = w & 0xFFFFu;
          wmode = w >> 16;
          if (wmode != WC_EXACT && !((__ldg(wc_inc + (d >> 6)) >> (d & 63)) & 1ull)) continue;
        }
      }
      // ---- STSSched: advanceReplay (:405-559)
      switch (kind) {
        case DEMI_EV_SPAWN: rec_push(kind, src, dst, 0, 0, 0, 0); inaccessible &= ~(1u << dst); killed &= ~(1u << dst); break;
        case DEMI_EV_KILL: rec_push(kind, src, dst, 0, 0, 0, 0); killed |= 1u << dst; inaccessible |= 1u << dst; break;
        case DEMI_EV_PARTITION: rec_push(kind, src, dst, 0, 0, 0, 0); part_row(src) |= 1u << dst; break;
        case DEMI_EV_UNPARTITION: rec_push(kind, src, dst, 0, 0, 0, 0); part_row(src) &= ~(1u << dst); break;
        case DEMI_EV_QUIESCENCE: case DEMI_EV_BEGIN_WAIT_QUIESCENCE: rec_push(kind, src, dst, 0, 0, 0, 0); break;
        case DEMI_EV_MSG_SEND:
          if (demi_type_is_external(A->external_type_mask, type)) tosend_push(0x80000000u | i);   // enqueue_message :469-470
          break;
        case DEMI_EV_MSG_EVENT: {
          flush();                                                   // messagePending :381-403
          if (status) break;
          if constexpr (WILD) {
            if (wmode != WC_EXACT) {                                 // WildCardMatch: deliver the selected pending message
              const int at = ((A->blocked_mask >> (dst & 31)) & 1u) ? -1
                             : wild_pick(src, dst, wmode, type, (A->flags & DEMI_WC_LAST_ONLY) != 0);
              if (at >= 0) {
                const uint4 q = table[(size_t)at * 32];
                const uint32_t qt = (q.x >> 16) & 0xFF;
                list_take((uint32_t)at, q);
                rec_push(DEMI_EV_MSG_EVENT, src, dst, qt, q.y, q.z, q.w & 0xFFFFu);
                deliver(src, dst, qt, q.y, q.z);
              } else { ignored++; note_ignored(i); }
              break;
            }
          }
          uint32_t hdr = make_hdr(src, dst, type, 0);
          uint32_t duniq = 0;
          bool enabled = !((A->blocked_mask >> (dst & 31)) & 1u) && pending_take(hdr, e.y, e.z, &duniq);
          if (enabled) { rec_push(DEMI_EV_MSG_EVENT, src, dst, type, e.y, e.z, duniq); deliver(src, dst, type, e.y, e.z); }   // :696-772
          else if (strict) diverged = true;                          // ReplayScheduler: ReplayException
          else { ignored++; note_ignored(i); }                       // "Ignoring message" :528-529
          break;
        }
        default: break;
      }
    }
#undef PF_ROW
    if (!status && !diverged) flush();                               // :682 before trace_finished
    out.violation = 0; out.delivered = 0; out.ignored = 0; out.state_hash = 0;
    if (REC && A->rec_count) A->rec_count[ROWS ? test_idx : 0] = n_rec;
    if (WILD && REC && A->wc_ignored_count) A->wc_ignored_count[ROWS ? test_idx : 0] = n_ign;
    if (status) { out.status = (uint16_t)status; return; }
    if (diverged) { out.status = DEMI_RS_DIVERGED; out.delivered = (uint16_t)delivered; return; }
    uint32_t v = MODEL::invariant(LaneAll<SW>{smw, BD}, A->model_flags);      // :283-289
    out.violation = (uint16_t)(A->looking_for ? (v == A->looking_for ? v : 0u) : v);
    out.status = 0;
    out.delivered = (uint16_t)delivered; out.ignored = (uint16_t)ignored;
    uint64_t sh = 0;
    for (uint32_t i = 0; i < N * SW; i++) sh += demi_state_term(smw[i * BD], i);
    out.state_hash = sh + rhash;
  }

  // ---- the per-thread skeleton of K2's kernels.  This thread's shared memory and its lane of warp gwarp's scratch,
  // laid out by `scratch`'s geometry; A is what the tests read.
  __device__ __forceinline__ void bind(uint32_t* smem, const ReplayArgs* a, const ReplayArgs& scratch, uint64_t gwarp,
                                       uint32_t lane) {
    smw = smem;
    A = a;
    table = scratch.table + gwarp * (uint64_t)scratch.table_slots * 32 + lane;
    tosend = scratch.tosend + gwarp * (uint64_t)scratch.tosend_cap * 32 + lane;
    pruned = scratch.pruned ? scratch.pruned + gwarp * (uint64_t)(scratch.n_uniq_words + N) * 32 + lane : nullptr;
  }
  // The next test's generation.  Generations continue across launches (the host hands out disjoint ranges), so the
  // table needs no clearing between launches; on wrap-around this thread clears its own slots.
  __device__ __forceinline__ void next_generation(uint32_t& generation, const ReplayArgs& scratch) {
    generation++;
    if (generation >= 0xFFFFu) {
      for (uint32_t s = 0; s < scratch.table_slots; s++) table[(size_t)s * 32] = make_uint4(0, 0, 0, 0);
      generation = 1;
    }
  }
  // runs test idx, stores its result to launch.results[idx] in one 16-byte store and counts it
  template <class IDX>
  __device__ __forceinline__ void run_store(IDX idx, uint32_t generation, const ReplayArgs& launch,
                                            unsigned long long& repro, unsigned long long& deliv) {
    demi_replay_result r;
    run((uint32_t)idx, generation, r);
    reinterpret_cast<uint4*>(launch.results + idx)[0] =
        make_uint4((uint32_t)r.violation | ((uint32_t)r.status << 16), (uint32_t)r.delivered | ((uint32_t)r.ignored << 16),
                   (uint32_t)r.state_hash, (uint32_t)(r.state_hash >> 32));
    repro += (r.status == 0 && r.violation) ? 1u : 0u;
    deliv += r.delivered;
  }
};

// adds a warp's counts to the launch's counters: [0] reproduced, [1] delivered
__device__ __forceinline__ void replay_count(const ReplayArgs& args, unsigned long long& repro, unsigned long long& deliv,
                                             uint32_t lane) {
  for (int o = 16; o > 0; o >>= 1) {
    repro += __shfl_xor_sync(FULL_MASK, repro, o);
    deliv += __shfl_xor_sync(FULL_MASK, deliv, o);
  }
  if (lane == 0 && args.counters && (repro | deliv)) {
    atomicAdd(args.counters, repro);
    atomicAdd(args.counters + 1, deliv);
  }
}

template <class MODEL, int BD, bool REC = false, bool WILD = false>
__global__ void __launch_bounds__(BD, (model_replay_direct<MODEL>::value && MODEL::N_ACTORS <= 8) ? 1024 / BD : 1)
replay_lane_kernel(const __grid_constant__ ReplayArgs args) {
  using M = ReplayMachine<MODEL, BD, REC, WILD>;
  extern __shared__ __align__(16) uint32_t lane_smem[];
  const uint32_t tid = threadIdx.x;
  const uint64_t gthread = (uint64_t)blockIdx.x * BD + tid;
  const uint64_t total = (uint64_t)gridDim.x * BD;
  const uint32_t lane = tid & 31;

  M m;
  m.bind(lane_smem + tid, &args, args, gthread >> 5, lane);
  unsigned long long my_repro = 0, my_deliv = 0;
  uint32_t generation = args.gen_base - 1;
  for (uint64_t idx = gthread; idx < args.n_masks; idx += total) {
    m.next_generation(generation, args);
    m.run_store(idx, generation, args, my_repro, my_deliv);
  }
  replay_count(args, my_repro, my_deliv, lane);
}

// K2 over many traces.  A tile {trace, first test, tests (<= 32), looking_for} belongs to one warp, so the trace stays
// warp-uniform and the lanes walk it in lock-step as in replay_lane_kernel; warps take tiles grid-stride.  `args`
// carries what the tiles share (flags, masks, results) and the scratch geometry, which is the largest of the launch's
// traces; each tile binds its trace's view into the warp's copy of it, bound[warp] in global memory.  The copy is in
// neither registers (they would come out of the per-event loop's) nor shared memory (a block's copies would cost raft5
// one of its four resident blocks per SM); its fields are read through L1.
// REC: every test records the EventTrace STSScheduler.test returns into its own row (ROWS above): the row is a
// member of the lane's machine, set from its test index, so the warp's copy of the arguments stays shared.
// WILD: ClockClusterizer's tests over each tile's trace.  A tile also binds its trace's mode table, modes[trace]; test
// idx reads its include mask at wc_include + idx * wc_words, the launch's stride.  With REC each test also writes its
// ignored deliveries into its own row.
template <class MODEL, int BD, bool REC = false, bool WILD = false>
__global__ void __launch_bounds__(BD, (model_replay_direct<MODEL>::value && MODEL::N_ACTORS <= 8) ? 1024 / BD : 1)
replay_many_kernel(const __grid_constant__ ReplayArgs args, const ReplayTraceView* __restrict__ views,
                   const uint4* __restrict__ tiles, uint32_t n_tiles, ReplayArgs* bound,
                   const uint32_t* const* __restrict__ modes) {
  using M = ReplayMachine<MODEL, BD, REC, WILD, REC>;
  extern __shared__ __align__(16) uint32_t lane_smem[];
  const uint32_t tid = threadIdx.x;
  const uint64_t gwarp = ((uint64_t)blockIdx.x * BD + tid) >> 5;
  const uint64_t total_warps = (uint64_t)gridDim.x * (BD / 32);
  const uint32_t lane = tid & 31;

  ReplayArgs& la = bound[gwarp];
  if (lane == 0) la = args;
  __syncwarp();
  M m;
  m.bind(lane_smem + tid, &la, args, gwarp, lane);
  unsigned long long my_repro = 0, my_deliv = 0;
  uint32_t generation = args.gen_base - 1;
  for (uint64_t t = gwarp; t < n_tiles; t += total_warps) {
    const uint4 tile = tiles[t];
    __syncwarp();                                  // every lane is done with the previous tile's trace
    if (lane == 0) {
      bind_trace(la, views[tile.x]); la.looking_for = tile.w;
      if constexpr (WILD) la.wc_ev = modes[tile.x];
    }
    __syncwarp();
    if (lane >= tile.z) continue;
    m.next_generation(generation, args);
    const uint32_t idx = tile.y + lane;
    m.run_store(idx, generation, args, my_repro, my_deliv);
  }
  replay_count(args, my_repro, my_deliv, lane);
}

}  // namespace demi
