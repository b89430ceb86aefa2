// lane_kernel.cuh — K1-lane: the high-throughput random-fuzz kernel.  One
// THREAD owns one schedule prefix (one RandomScheduler execution, reference:
// schedulers/RandomScheduler.scala:234-272, :352-485); a warp advances 32
// prefixes in lock-step.  Same semantics as machine.cuh, restated for a scalar
// owner:
//
//   registers      java.util.Random state, counters, network masks, and the
//                  timer sets as BITMASKS over the model's finite timer universe
//                  (justScheduledTimers / timerToCancellable / timersCancelled-
//                  ThisStep), messagesToSend and timersToResend as byte queues
//   shared memory  actor states, the receive() outbox and partition rows,
//                  thread-interleaved (word w of thread t at [w*BD + t]: every
//                  access is bank-conflict free whatever each lane indexes)
//   HBM / L1 / L2  the pending-message array (RandomizedHashSet.arr), 16-byte
//                  entries (8-byte in the steady raft5 kernel's ROW8 flavour),
//                  LPCAP contiguous ones per thread (entry i of thread t at
//                  [t*LPCAP + i])
//
// Exactness: every structure here is a bounded, duplicate-free restatement.
// Whenever an execution could leave that regime (a capacity would overflow, or
// the DepTracker child-reuse rule (DepTracker.scala:94-108) could fire) the
// thread stops and appends the prefix index to the defer list; the general
// warp engine (fuzz_kernel.cuh) then re-runs exactly those prefixes.  A
// prefix that completes here has, by construction, the same result as in the
// general engine.
#pragma once
#include "machine.cuh"
#include "models/models.cuh"
#include "lane_steady.hpp"
#include <type_traits>

namespace demi {

#ifndef DEMI_K1_PEND_HINT
#define DEMI_K1_PEND_HINT 1      // pending array accessed with an L2 evict_last policy
#endif
#ifndef DEMI_K1_RESULT_CS
#define DEMI_K1_RESULT_CS 1      // result records written with streaming (evict-first) stores
#endif
#ifndef DEMI_K1_DIRECT_OUTBOX
#define DEMI_K1_DIRECT_OUTBOX 1  // models with LANE_SENDS_DISTINCT: receive()'s operations are applied as they are issued
#endif
#ifndef DEMI_K1_LPCAP_RAFT5
#define DEMI_K1_LPCAP_RAFT5 96
#endif
#ifndef DEMI_K1_PHASE_CLOCK
#define DEMI_K1_PHASE_CLOCK 0    // profiling builds only (tools/profile_lane_phases.py): per-phase clock64() sums
#endif

constexpr uint32_t LANE_DEFER = 0xFFFFu;      // internal status: hand over to the warp engine

// The phase clock.  Lane 0 of each warp keeps, per phase of an execution step, the clock64() cycles from the phase's
// entry to the next phase's entry, the active lanes at the entry (__popc(__activemask())) and the number of entries.
// The warp adds them to demi_k1_phase_sums when it finishes; demi_k1_phase_read (capi.cu) copies them out.  Lanes
// that diverge from lane 0 are seen only through lane 0's waits, so the figures say what the warp pays per phase.
enum LanePhase : uint32_t { LP_FLUSH, LP_PICK, LP_RECEIVE, LP_SEND, LP_CANCEL, LP_SCHEDULE, LP_INVARIANT, LP_TAIL, LP_COUNT };
#if DEMI_K1_PHASE_CLOCK
static __device__ unsigned long long demi_k1_phase_sums[LP_COUNT * 3];     // [phase][cycles, lanes, entries]
#endif
struct LanePhaseClock {
#if DEMI_K1_PHASE_CLOCK
  unsigned long long cyc[LP_COUNT], lanes[LP_COUNT], n[LP_COUNT], t0;
  uint32_t cur;
  __device__ __forceinline__ void start() {
    for (int p = 0; p < LP_COUNT; p++) cyc[p] = lanes[p] = n[p] = 0;
    cur = LP_TAIL; t0 = clock64();
  }
  __device__ __forceinline__ void enter(uint32_t p) {
    const uint32_t act = __activemask();
    if ((threadIdx.x & 31u) == 0) {
      const unsigned long long now = clock64();
      cyc[cur] += now - t0; t0 = now; cur = p;
      lanes[p] += __popc(act); n[p]++;
    }
  }
  __device__ __forceinline__ void finish() {
    enter(LP_TAIL);
    if ((threadIdx.x & 31u) == 0)
      for (int p = 0; p < LP_COUNT; p++) {
        atomicAdd(&demi_k1_phase_sums[p * 3 + 0], cyc[p]);
        atomicAdd(&demi_k1_phase_sums[p * 3 + 1], lanes[p]);
        atomicAdd(&demi_k1_phase_sums[p * 3 + 2], n[p]);
      }
  }
#else
  __device__ __forceinline__ void start() {}
  __device__ __forceinline__ void enter(uint32_t) {}
  __device__ __forceinline__ void finish() {}
#endif
};

// The pending arrays are the only data this kernel re-reads from global memory; the result records are written once.
// An L2 evict_last policy on the former (and evict-first stores for the latter) keeps the arrays cache-resident, so
// that their stores are not written back to DRAM between a prefix's steps.  Every access to the arrays goes
// through these two volatile asm statements (which keep their program order), and nothing else aliases the arrays,
// so no "memory" clobber is needed.
__device__ __forceinline__ uint64_t l2_evict_last_policy() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint4 ld_l2_hint(const uint4* p, uint64_t pol) {
#if DEMI_K1_PEND_HINT
  uint4 v;
  asm volatile("ld.global.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(pol));
  return v;
#else
  (void)pol; return *p;
#endif
}
__device__ __forceinline__ void st_l2_hint(uint4* p, uint4 v, uint64_t pol) {
#if DEMI_K1_PEND_HINT
  asm volatile("st.global.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol));
#else
  (void)pol; *p = v;
#endif
}
// 8-byte rows (the steady raft5 kernel's ROW8 flavour, lane_steady.hpp) under the same policy
__device__ __forceinline__ uint2 ld_l2_hint(const uint2* p, uint64_t pol) {
#if DEMI_K1_PEND_HINT
  uint2 v;
  asm volatile("ld.global.L2::cache_hint.v2.u32 {%0,%1}, [%2], %3;" : "=r"(v.x), "=r"(v.y) : "l"(p), "l"(pol));
  return v;
#else
  (void)pol; return *p;
#endif
}
__device__ __forceinline__ void st_l2_hint(uint2* p, uint2 v, uint64_t pol) {
#if DEMI_K1_PEND_HINT
  asm volatile("st.global.L2::cache_hint.v2.u32 [%0], {%1,%2}, %3;" :: "l"(p), "r"(v.x), "r"(v.y), "l"(pol));
#else
  (void)pol; *p = v;
#endif
}
constexpr int LANE_TOSEND_CAP = 16;
constexpr int LANE_RESEND_CAP = 8;

// One actor's state, thread-interleaved in shared memory.
struct LaneState {
  uint32_t* base;      // &smem[word0 * BD + tid]
  uint32_t bd;
  __device__ __forceinline__ uint8_t& operator[](uint32_t i) const {
    return reinterpret_cast<uint8_t*>(base + (i >> 2) * bd)[i & 3];
  }
  __device__ __forceinline__ uint8_t& b(uint32_t i) const { return (*this)[i]; }
  __device__ __forceinline__ uint32_t& w(uint32_t i) const { return base[i * bd]; }
};
template <int SW>
struct LaneAll {
  uint32_t* base; uint32_t bd;
  __device__ __forceinline__ LaneState actor(uint32_t a) const { return LaneState{base + a * SW * bd, bd}; }
};

// receive()'s outbox, thread-interleaved in shared memory (3 words per op).
template <int CAP>
struct LaneOutbox {
  uint32_t* base; uint32_t bd;
  uint32_t n, self;
  bool overflow;
  __device__ __forceinline__ void push(uint32_t op, uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) {
    if (n >= CAP) { overflow = true; return; }
    base[(n * 3 + 0) * bd] = op | (dst << 8) | (type << 16);
    base[(n * 3 + 1) * bd] = p0;
    base[(n * 3 + 2) * bd] = p1;
    n++;
  }
  __device__ __forceinline__ bool reserve(uint32_t) { return true; }     // drain() reserves each staged send
  __device__ __forceinline__ void send(uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) { push(OP_SEND, dst, type, p0, p1); }
  __device__ __forceinline__ void schedule_once(uint32_t type, uint32_t p0, uint32_t p1) { push(OP_SCHED_ONCE, self, type, p0, p1); }
  __device__ __forceinline__ void schedule_repeating(uint32_t type, uint32_t p0, uint32_t p1) { push(OP_SCHED_REPEAT, self, type, p0, p1); }
  __device__ __forceinline__ void cancel_timer(uint32_t type, uint32_t p0, uint32_t p1) { push(OP_CANCEL, self, type, p0, p1); }
};

// small FIFO of bytes in four 32-bit registers: entry i is byte (i & 3) of w[i >> 2], and the bytes at and above n
// are zero.  Every operation is a few byte permutes (PRMT), funnel shifts or bitwise ops on the words; none loops over
// the entries.
struct ByteQueue16 {
  uint32_t w[4]; uint32_t n;
  __device__ __forceinline__ void clear() { w[0] = w[1] = w[2] = w[3] = 0; n = 0; }
  // Word k takes byte b at bit 8n - 32k: a clamping funnel shift of b gives 0 wherever that is not in 0..24 (a
  // "negative" amount wraps to a large one).  Caller checks n < 16.
  __device__ __forceinline__ void push(uint32_t b) {
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) w[k] |= __funnelshift_lc(0u, b, n * 8u - 32u * k);
    n++;
  }
  // An empty queue takes the `len` bytes of hi:lo (those at and above len zero) as its entries.
  __device__ __forceinline__ void assign(uint32_t lo, uint32_t hi, uint32_t len) { w[0] = lo; w[1] = hi; n = len; }
  // Removes and returns entry 0: the queue shifts down one byte, and the zero bytes above n shift in behind it.
  // Caller checks n > 0.
  __device__ __forceinline__ uint32_t pop() {
    const uint32_t b = w[0] & 0xFFu;
    w[0] = __funnelshift_r(w[0], w[1], 8);
    w[1] = __funnelshift_r(w[1], w[2], 8);
    w[2] = __funnelshift_r(w[2], w[3], 8);
    w[3] >>= 8;
    n--;
    return b;
  }
  // The index of the first entry equal to b (b < 0x80), or a value >= n when there is none.  All 16 bytes are compared
  // at once (a SIMD byte compare per word, its byte masks gathered into one bit per entry); the zero bytes above n
  // can match only b = 0, and only after every entry that does.
  __device__ __forceinline__ uint32_t find(uint32_t b) const {
    const uint32_t pat = b * 0x01010101u;
    uint32_t bits = 0x10000u;
#pragma unroll
    for (uint32_t k = 0; k < 4; k++)
      bits |= (((__vcmpeq4(w[k], pat) & 0x80808080u) * 0x00204081u) >> 28) << (4 * k);
    return __ffs(bits) - 1u;
  }
  // Order preserving: every entry above i moves down one byte.  Word k is permuted with the word above it (byte 0 of
  // w[k+1] is byte 4 of the pair); it keeps its `keep` bytes below i and takes the next byte for each one above:
  // selector 0x3210 for keep = 4 (a word below i's), 0x4321 for keep = 0 (a word above it).
  __device__ __forceinline__ void remove_at(uint32_t i) {
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int keep = min(max((int)i - 4 * k, 0), 4);
      const uint32_t sel = 0x4321u - (0x1111u >> (16 - 4 * keep));
      w[k] = __byte_perm(w[k], k < 3 ? w[k + 1] : 0u, sel);
    }
    n--;
  }
};

// receive()'s view when its operations are applied as they are issued (`dst ! msg` is synchronous in the reference,
// Instrumenter.scala:1098-1108): no staging in shared memory.  Only for models whose receive() cannot produce two equal
// sends (MODEL::LANE_SENDS_DISTINCT), because the duplicate-send screen needs the whole outbox.  The model reserves
// its sends before it issues them: reserve(k), then k sends.
template <class M>
struct LaneDirectOutbox {
  M* m; uint32_t self;
  __device__ __forceinline__ bool reserve(uint32_t k) { return m->reserve_sends(self, k); }
  __device__ __forceinline__ void send(uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) { m->actor_send_produced(self, dst, type, p0, p1); }
  __device__ __forceinline__ void schedule_once(uint32_t type, uint32_t p0, uint32_t p1) { m->schedule_timer(OP_SCHED_ONCE, self, type, p0, p1); }
  __device__ __forceinline__ void schedule_repeating(uint32_t type, uint32_t p0, uint32_t p1) { m->schedule_timer(OP_SCHED_REPEAT, self, type, p0, p1); }
  __device__ __forceinline__ void cancel_timer(uint32_t type, uint32_t p0, uint32_t p1) { m->cancel_timer(self, type, p0, p1); }
};
template <class M>
__device__ __forceinline__ void receive_phase(LaneDirectOutbox<M>& o, uint32_t rp) {
  o.m->clk.enter(rp == RP_CANCEL ? LP_CANCEL : rp == RP_SEND ? LP_SEND : LP_SCHEDULE);
}

// REC: the execution's EventTrace and DepTracker parents are written out (provenance batches, demi_fuzz_provenance)
// STEADY: every execution starts from the launch's pre-delivery snapshot (lane_steady.hpp) and nothing external
// happens after it.  The host has checked lane_steady_eligible, so this instantiation carries no code for externals,
// partitions, isolated or killed actors, ignoreTimers, a violation filter or the node capacity, and tests the
// pending array against one bound (A->pending_cap, which the host has clamped to LPCAP).  Every rule is the generic
// one with those cases compiled out.
// ROW8 (STEADY raft5 only): the pending rows are 8 bytes in the layout of lane_steady.hpp, which the host has proven
// holds every row of the launch (lane_row8_eligible).  A row is packed where it is stored and unpacked where it is
// read, so the rest of the machine and the model see the 16-byte form.
template <class MODEL, int BD, int LPCAP, bool REC = false, bool STEADY = false, bool ROW8 = false>
struct LaneMachine {
  static_assert(!(STEADY && REC), "recording launches run the generic instantiation");
  static_assert(!ROW8 || (STEADY && MODEL::ID == DEMI_MODEL_RAFT5), "the 8-byte layout and its proof are the steady raft5 machine's");
  static constexpr int N = MODEL::N_ACTORS;
  static constexpr int SW = MODEL::STATE_WORDS;
  static constexpr int OB = MODEL::LANE_OUTBOX;
  // the outbox is staged in shared memory only when receive()'s operations are not applied as they are issued
  static constexpr bool DIRECT = DEMI_K1_DIRECT_OUTBOX && MODEL::LANE_SENDS_DISTINCT;
  static constexpr int OBW = DIRECT ? 0 : OB * 3;
  static constexpr uint32_t CT = MODEL::LANE_CANCEL_TYPE;            // 0: receive() cancels no timer
  static constexpr int TW = CT ? (N + 1) / 2 : 0;
  static_assert(CT == 0 || LPCAP < 0xFF, "tcopy keeps a pending index in one byte, 0xFF meaning unknown");
  static constexpr int PW = STEADY ? 0 : N;               // partition rows: none when the program has no partition
  static constexpr int WORDS = N * SW + OBW + PW + TW;     // states + outbox + partition rows + cancellable timer copies

  uint32_t* smw;             // &smem[tid]; word w at smw[w*BD]
  using Row = typename std::conditional<ROW8, uint2, uint4>::type;
  Row* pend;                 // entry i at pend[i]
  uint4* rec_ev; uint16_t* rec_par;   // REC: this execution's EventTrace slot and parent array
  uint64_t pol;              // L2 cache policy of the pending array
  const KernelArgs* A;

  JRandom rng;
  uint32_t n_pending, max_pending;
  ByteQueue16 tosend;        // byte: timer slot, or 0x80|k for the k-th external Send
  uint64_t resend; uint32_t n_resend;
  uint32_t just, registry, cancelled;            // bit per timer slot
  uint32_t root_timers, window_timers;           // duplicate guards for the child-reuse rule
  // Every send takes the next Unique id and the next DepTracker node together (no child is reused in this engine), so
  // the two are equal and one counter serves both: a send's word 3 is node | node << 16.
  uint32_t n_nodes, parent_event, n_events;
  int32_t nsched, nmod;
  uint32_t ext_idx, ext_send_idx;
  uint32_t violation, status;
  uint32_t inaccessible, killed;
  uint64_t thash;
  // the sends of one receive(), set up by reserve_sends: no partition or isolation in effect, and the linear part of
  // the trace hash term of the next send with its dst, type, p0 and p1 words left out
  bool sends_open;
  uint64_t send_lin;
  LanePhaseClock clk;        // empty unless DEMI_K1_PHASE_CLOCK

  __device__ __forceinline__ uint32_t& part_row(uint32_t a) { return smw[(N * SW + OBW + a) * BD]; }
  // Where the timer message of type CT (the one timer receive() cancels) of each actor is in the pending array, so that
  // Cancellable.cancel need not scan for it: 16 bits per actor (actor a in half a & 1 of word a >> 1), the low byte the
  // number of its copies in the array, the high byte the index of the copy when there is exactly one and it is known
  // (0xFF otherwise: after 2 -> 1 it is not).  Only timer_produced inserts timer messages (an external with a timer's
  // key defers) and every removal goes through pending_remove_at, so these are exact.  Other timers are not tracked:
  // the check on each removal is one compare of the header's flags and type.
  __device__ __forceinline__ uint32_t& tcopy_word(uint32_t a) { return smw[(N * SW + OBW + PW + (a >> 1)) * BD]; }
  __device__ __forceinline__ uint32_t tcopy(uint32_t a) { return (tcopy_word(a) >> ((a & 1u) * 16)) & 0xFFFFu; }
  __device__ __forceinline__ void tcopy_set(uint32_t a, uint32_t e) {
    uint32_t& w = tcopy_word(a);
    const uint32_t sh = (a & 1u) * 16;
    w = (w & ~(0xFFFFu << sh)) | (e << sh);
  }
  __device__ __forceinline__ static bool cancellable_timer(uint32_t hdr) { return (hdr >> 16) == ((DEMI_MF_TIMER << 8) | CT); }
  __device__ __forceinline__ LaneState actor(uint32_t a) { return LaneState{smw + a * SW * BD, BD}; }

  __device__ __forceinline__ void defer() { status = LANE_DEFER; }

  // EventTrace.+= (EventTrace.scala:88-110); w3 = uniq | node << 16.  Here uniq == node < node_cap <= 65535, so the
  // 16-bit Uniq wrap (DESIGN.md §2) is never reached: an execution with more ids is one with identical Sends, which
  // only the warp engine runs.
  __device__ __forceinline__ void record_event(uint32_t kind, uint32_t src, uint32_t dst, uint32_t type,
                                               uint32_t p0, uint32_t p1, uint32_t w3, uint32_t parent) {
    uint32_t w0 = kind | (src << 8) | (dst << 16) | (type << 24);
    thash += demi_event_term(w0, p0, p1, w3, n_events, parent);
    record_rest(w0, p0, p1, w3, parent);
  }
  // the provenance copy of the element, and its position
  __device__ __forceinline__ void record_rest(uint32_t w0, uint32_t p0, uint32_t p1, uint32_t w3, uint32_t parent) {
    if (REC) {
      if (n_events >= A->rec_cap) { defer(); return; }
      rec_ev[n_events] = make_uint4(w0, p0, p1, w3);
      const uint32_t node = w3 >> 16;
      if ((w0 & 0xFF) == DEMI_EV_MSG_SEND && node < A->rec_parent_cap) rec_par[node] = (uint16_t)parent;   // DepTracker edge
    }
    n_events++;
  }

  // RandomizedHashSet.insert (schedulers/Util.scala:126-136).  max_pending is brought up to date before each removal
  // and at the end of the execution, the only points where the set can be at a maximum.
  __device__ __forceinline__ static Row row_pack(const uint4& e) {
    if constexpr (ROW8) {
      static_assert(MODEL::N_ACTORS == (int)LANE_ROW8_ACTORS && MODEL::LOG_CAP < 16, "lane_steady.hpp's proof is about this model");
      const uint64_t r = lane_row8_pack(e.x, e.y, e.z, e.w & 0xFFFFu);
      return make_uint2((uint32_t)r, (uint32_t)(r >> 32));
    } else {
      return e;
    }
  }
  __device__ __forceinline__ static uint4 row_unpack(const Row& q) {
    if constexpr (ROW8) {
      const uint64_t r = q.x | (uint64_t)q.y << 32;
      // no flags in the header: nothing reads them but row_cancellable, which reads the row
      return make_uint4(lane_row8_sdt(r), lane_row8_p0(r), lane_row8_p1(r), lane_row8_node(r) * 0x10001u);
    } else {
      return q;
    }
  }
  // whether a stored row is a copy of the cancellable timer (type CT), and its receiver
  __device__ __forceinline__ static bool row_cancellable(const Row& q) {
    if constexpr (ROW8) return lane_row8_timer_of(q.x | (uint64_t)q.y << 32, CT);
    else return cancellable_timer(q.x);
  }
  __device__ __forceinline__ static uint32_t row_dst(const Row& q) {
    if constexpr (ROW8) return lane_row8_dst(q.x | (uint64_t)q.y << 32);
    else return hdr_dst(q.x);
  }
  __device__ __forceinline__ uint4 row_load(uint32_t i) { return row_unpack(ld_l2_hint(pend + i, pol)); }

  __device__ __forceinline__ bool pending_full(uint32_t k) const {
    if constexpr (STEADY) return n_pending + k > A->pending_cap;
    return n_pending + k > A->pending_cap || n_pending + k > LPCAP;
  }
  __device__ __forceinline__ void pending_push(uint4 e) {          // the caller has checked pending_full
    st_l2_hint(pend + n_pending, row_pack(e), pol);
    n_pending++;
  }
  __device__ __forceinline__ void pending_insert(uint4 e) {
    if (pending_full(1)) { defer(); return; }
    pending_push(e);
  }
  // RandomizedHashSet.remove (schedulers/Util.scala:146-163)
  __device__ __forceinline__ uint4 pending_remove_at(uint32_t i) {
    if (n_pending > max_pending) max_pending = n_pending;
    const Row vr = ld_l2_hint(pend + i, pol);
    const Row last = ld_l2_hint(pend + (n_pending - 1), pol);
    st_l2_hint(pend + i, last, pol);
    n_pending--;
    const uint4 v = row_unpack(vr);
    if constexpr (CT != 0) {
      // in place on the actor's half of the word: the count is at least 1 here, and indices stay below LPCAP < 0xFF
      if (row_cancellable(vr)) {                         // one copy fewer, its index no longer known
        const uint32_t a = row_dst(vr), sh = (a & 1u) * 16;
        tcopy_word(a) = (tcopy_word(a) - (1u << sh)) | (0xFF00u << sh);
      }
      if (row_cancellable(last)) {                       // moved from index n_pending to i
        const uint32_t a = row_dst(last), sh = (a & 1u) * 16 + 8;
        uint32_t& w = tcopy_word(a);
        if (((w >> sh) & 0xFFu) == n_pending) w ^= (n_pending ^ i) << sh;
      }
    }
    return v;
  }

  // EventOrchestrator.crosses_partition (EventOrchestrator.scala:345-351)
  __device__ __forceinline__ bool network_open() {           // everyone started, no one isolated
    if constexpr (STEADY) return true;
    return !(inaccessible | killed) && !A->has_partitions;
  }
  __device__ __forceinline__ bool crosses_partition(uint32_t snd, uint32_t rcv) {
    return !network_open() && crosses_partition_closed(snd, rcv);
  }
  __device__ __forceinline__ bool crosses_partition_closed(uint32_t snd, uint32_t rcv) {
    bool snd_actor = snd < DEMI_MAX_ACTORS;
    if (snd == rcv && !((killed >> snd) & 1u)) return false;
    if (A->has_partitions && snd_actor) {
      if ((part_row(snd) >> rcv) & 1u) return true;
      if ((part_row(rcv) >> snd) & 1u) return true;
    }
    if ((inaccessible >> rcv) & 1u) return true;
    if (snd_actor && ((inaccessible >> snd) & 1u)) return true;
    return false;
  }

  // RandomScheduler.event_produced (RandomScheduler.scala:274-321) after
  // Instrumenter.aroundDispatch's cancelled-timer drop (Instrumenter.scala:1090-1096).
  // DepTracker.getMessage (DepTracker.scala:82-109): in the regime this engine
  // accepts no child is ever reused, so the Unique id is simply the next one.
  // The sends of receive() itself (sender an actor, no flags): the external / timer branches do not apply.
  //
  // reserve_sends(self, k) is called once before the next k of them: it checks the node and pending capacities for
  // all k and defers if they do not fit, so that actor_send_produced applies each send with no further check.  With
  // exactly k sends inserted this defers exactly when the per-send checks would have; a send that crosses a partition
  // or hits a cancelled timer is not inserted, so there the reservation may be conservative (deferring is always
  // exact: the general engine re-runs the prefix).  Only REC's trace capacity is still checked per event.
  __device__ __forceinline__ bool reserve_sends(uint32_t self, uint32_t k) {
    if (status) return false;
    if ((!STEADY && n_nodes + k > A->node_cap) || pending_full(k)) { defer(); return false; }
    sends_open = network_open();
    // demi_event_term of the first send, dst / type / payload terms left out: word 0 = kind | self << 8, word 3 =
    // node | node << 16 (node <= 0xFFFE, as n_nodes + k <= node_cap <= 0xFFFF), sequence n_events
    send_lin = demi_hash6_lin(DEMI_EV_MSG_SEND | (self << 8), 0, 0, n_nodes * 0x10001u, n_events, parent_event);
    return true;
  }
  __device__ __forceinline__ void actor_send_produced(uint32_t self, uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) {
    if (REC && status) return;
    if (cancelled) {
      const int slot = MODEL::timer_slot(dst, type, p0, p1);
      if (slot >= 0 && ((cancelled >> slot) & 1u)) { cancelled &= ~(1u << slot); return; }
    }
    const uint32_t w3 = n_nodes++ * 0x10001u;
    if (STEADY || sends_open || !crosses_partition_closed(self, dst)) pending_push(make_uint4(make_hdr(self, dst, type, 0), p0, p1, w3));
    // the hash term of this send: word 0 adds dst << 16 | type << 24 to the reserved kind | self << 8, and the next
    // send's word 3 and sequence number are one node (0x10001) and one event further on
    const uint32_t w0_tail = (dst << 16) | (type << 24);
    thash += demi_hash6_fin(send_lin + (uint64_t)w0_tail * DEMI_HASH6_KA + (uint64_t)p0 * DEMI_HASH6_KB +
                            (uint64_t)p1 * DEMI_HASH6_KC);
    send_lin += 0x10001ull * DEMI_HASH6_KD + DEMI_HASH6_KE;
    record_rest(DEMI_EV_MSG_SEND | (self << 8) | w0_tail, p0, p1, w3, parent_event);
  }
  // A timer message flushed from messagesToSend (sender deadLetters, recorded as "Timer"); `slot` is its key.
  __device__ __forceinline__ void timer_produced(uint32_t slot) {
    const uint32_t bit = 1u << slot;
    if (cancelled & bit) { cancelled &= ~bit; return; }
    if (!STEADY && n_nodes >= A->node_cap) { defer(); return; }
    // two equal timer sends under one parent would share a Unique: defer those.  (STEADY: a timer is flushed only
    // after a delivery, whose node is the parent.)
    if (!STEADY && parent_event == 0) { if (root_timers & bit) { defer(); return; } root_timers |= bit; }
    else { if (window_timers & bit) { defer(); return; } window_timers |= bit; }
    const uint32_t w3 = n_nodes++ * 0x10001u;
    uint32_t dst, type, p0, p1;
    MODEL::slot_msg(slot, dst, type, p0, p1);
    if (!crosses_partition(DEMI_DEADLETTERS, dst)) {
      pending_insert(make_uint4(make_hdr(DEMI_DEADLETTERS, dst, type, DEMI_MF_TIMER), p0, p1, w3));
      if (status) return;
      if constexpr (CT != 0)
        if (type == CT) {
          const uint32_t n = tcopy(dst) & 0xFFu;
          tcopy_set(dst, n == 0 ? (1u | (n_pending - 1) << 8) : ((n + 1) | 0xFF00u));
        }
    }
    record_event(DEMI_EV_MSG_SEND, DEMI_TIMER_SND, dst, type, p0, p1, w3, parent_event);
  }
  // An external Send flushed from messagesToSend (`hdr` carries DEMI_MF_EXTERNAL).
  __device__ __forceinline__ void external_produced(uint32_t hdr, uint32_t p0, uint32_t p1) {
    const uint32_t dst = hdr_dst(hdr), type = hdr_type(hdr);
    const int slot = MODEL::timer_slot(dst, type, p0, p1);
    if (slot >= 0) {
      if ((cancelled >> slot) & 1u) { cancelled &= ~(1u << slot); return; }
      defer(); return;                          // an external that equals a timer key could share its Unique
    }
    if (n_nodes >= A->node_cap) { defer(); return; }
    parent_event = 0;                           // reportNewlyEnabledExternal (DepTracker.scala:119-122)
    const uint32_t w3 = n_nodes++ * 0x10001u;   // (identical external Sends are screened on the host)
    pending_insert(make_uint4(hdr, p0, p1, w3));
    if (status) return;
    record_event(DEMI_EV_MSG_SEND, hdr_src(hdr), dst, type, p0, p1, w3, 0u);
  }

  // RandomScheduler.enqueue_timer (RandomScheduler.scala:549-559) of a slot whose justScheduledTimers bit is set
  __device__ __forceinline__ void resend_push(uint32_t slot) {
    if (n_resend >= LANE_RESEND_CAP) { defer(); return; }
    resend |= (uint64_t)slot << (n_resend * 8);
    n_resend++;
  }
  // scheduler.scheduleOnce / schedule (Instrumenter.scala:1126-1190), then RandomScheduler.enqueue_timer ->
  // ExternalEventInjector.handle_timer (ExternalEventInjector.scala:282-297).  This is the only place a single timer
  // enters messagesToSend.
  __device__ __forceinline__ void schedule_timer(uint32_t kind, uint32_t self, uint32_t type, uint32_t p0, uint32_t p1) {
    if (status) return;
    const int s2 = MODEL::timer_slot(self, type, p0, p1);
    if (s2 < 0) { defer(); return; }
    if ((registry >> s2) & 1u) return;                        // "Non-unique timer" (Instrumenter.scala:1154-1157)
    if (kind == OP_SCHED_REPEAT) {
      if (__popc(registry) >= DEMI_TIMERSET_CAP) { defer(); return; }
      registry |= 1u << s2;
    }
    if ((just >> s2) & 1u) { resend_push((uint32_t)s2); return; }
    if (!STEADY && A->ignore_timers) return;
    if (tosend.n >= LANE_TOSEND_CAP || (!STEADY && tosend.n >= A->tosend_cap)) { defer(); return; }
    tosend.push((uint32_t)s2);
  }
  // First the ops receive() left in the outbox (`n_ops`, sender `self`), in program order; then, if `do_flush`,
  // ExternalEventInjector.send_external_messages (ExternalEventInjector.scala:306-365).  Two loops, so that the
  // lanes of a warp reconverge between the phases and their flush items are processed together.
  __device__ __forceinline__ void drain(uint32_t n_ops, uint32_t self, bool do_flush) {
    if constexpr (!DIRECT) {
      uint32_t* ob = smw + N * SW * BD;
#pragma unroll 1
      for (uint32_t i = 0; i < n_ops && !status; i++) {
        const uint32_t w0 = ob[(i * 3) * BD], p0 = ob[(i * 3 + 1) * BD], p1 = ob[(i * 3 + 2) * BD];
        const uint32_t kind = w0 & 0xFF, odst = (w0 >> 8) & 0xFF, otype = (w0 >> 16) & 0xFF;
        if (kind == OP_SEND) { if (reserve_sends(self, 1)) actor_send_produced(self, odst, otype, p0, p1); continue; }
        if (kind == OP_CANCEL) { cancel_timer(odst, otype, p0, p1); continue; }
        schedule_timer(kind, odst, otype, p0, p1);
      }
    }
    if (status || !do_flush) return;
    // in order from the front; a flush that runs to the end leaves the queue empty (a deferred prefix's queue is
    // never read again)
#pragma unroll 1
    while (tosend.n != 0 && !status) {
      const uint32_t b = tosend.pop();
      if (!STEADY && (b & 0x80u)) {
        const uint4 raw = __ldg(reinterpret_cast<const uint4*>(A->ext_sends) + (b & 0x7Fu));
        external_produced(raw.x, raw.y, raw.z);
      } else {
        timer_produced(b);
      }
    }
  }

  // Cancellable.cancel(): Instrumenter.cancelTimer (Instrumenter.scala:159-168) ->
  // RandomScheduler.notify_timer_cancel (RandomScheduler.scala:525-534)
  __device__ __forceinline__ void cancel_timer(uint32_t self, uint32_t type, uint32_t p0, uint32_t p1) {
    if (status) return;
    int slot = MODEL::timer_slot(self, type, p0, p1);
    if (slot < 0) { defer(); return; }
    uint32_t bit = 1u << slot;
    if (!(cancelled & bit) && __popc(cancelled) >= DEMI_TIMERSET_CAP) { defer(); return; }
    cancelled |= bit;
    registry &= ~bit;
    const uint32_t at = tosend.find((uint32_t)slot);  // handle_timer_cancel (ExternalEventInjector.scala:601-610)
    if (at < tosend.n) { tosend.remove_at(at); return; }
    // FullyRandom.remove (RandomScheduler.scala:653-664): first match in array order.  The only entries that match are
    // the slot's timer messages: for the tracked type CT, with none pending there is nothing to remove, and a single
    // copy at a known index is the first match.  Otherwise the array is scanned, four entries fetched per step so that
    // their latencies overlap (this scan was 6 % of the kernel's stall samples when it fetched one).
    if constexpr (CT != 0)
      if (type == CT) {
        const uint32_t e = tcopy(self);
        if ((e & 0xFFu) == 0) return;
        if ((e >> 8) != 0xFFu) { pending_remove_at(e >> 8); return; }
      }
    const uint32_t want = make_hdr(DEMI_DEADLETTERS, self, type, 0);
#pragma unroll 1
    for (uint32_t i = 0; i < n_pending; i += 4) {
      uint4 q[4];
#pragma unroll
      for (uint32_t k = 0; k < 4; k++) q[k] = (i + k < n_pending) ? row_load(i + k) : make_uint4(0, 0, 0, 0);
#pragma unroll
      for (uint32_t k = 0; k < 4; k++)
        if ((q[k].x & 0x00FFFFFFu) == want && q[k].y == p0 && q[k].z == p1) { pending_remove_at(i + k); return; }
    }
  }

  __device__ __forceinline__ uint32_t check_invariant() {
    uint32_t v = MODEL::invariant(LaneAll<SW>{smw, BD}, A->model_flags);
    if (STEADY || !A->looking_for) return v;                    // violationMatches (RandomScheduler.scala:138-154)
    return (v && v == A->looking_for) ? A->looking_for : 0u;
  }

  // EventOrchestrator.inject_until_quiescence (EventOrchestrator.scala:132-189)
  __device__ __forceinline__ void inject_until_quiescence() {
    bool loop = true;
    while (loop && ext_idx < A->n_ext && !status) {
      uint4 raw = __ldg(reinterpret_cast<const uint4*>(A->ext) + ext_idx);
      uint32_t kind = raw.x & 0xFF, a = (raw.x >> 8) & 0xFF, b = (raw.x >> 16) & 0xFF;
      uint32_t ek = 0, es = DEMI_DEADLETTERS, ed = a;          // the EventTrace element this external leaves
      switch (kind) {
        case DEMI_EXT_START:
          ek = DEMI_EV_SPAWN;
          inaccessible &= ~(1u << a); killed &= ~(1u << a);
          break;
        case DEMI_EXT_KILL:
          ek = DEMI_EV_KILL;
          killed |= 1u << a; inaccessible |= 1u << a;
          break;
        case DEMI_EXT_SEND:
          if (tosend.n >= LANE_TOSEND_CAP || ext_send_idx >= 0x80u) { defer(); break; }
          tosend.push(0x80u | ext_send_idx);
          ext_send_idx++;
          break;
        case DEMI_EXT_PARTITION:
          ek = DEMI_EV_PARTITION; es = a; ed = b;
          part_row(a) |= 1u << b;
          break;
        case DEMI_EXT_UNPARTITION:
          ek = DEMI_EV_UNPARTITION; es = a; ed = b;
          part_row(a) &= ~(1u << b);
          break;
        case DEMI_EXT_WAIT_QUIESCENCE:
          ek = DEMI_EV_BEGIN_WAIT_QUIESCENCE; ed = DEMI_DEADLETTERS;
          loop = false;
          break;
        default: break;
      }
      if (ek) record_event(ek, es, ed, 0, 0, 0, 0, 0);
      ext_idx++;
    }
  }

  // RandomScheduler.schedule_new_message (RandomScheduler.scala:352-485); blockedActors is empty here
  // the stop conditions at the top of schedule_new_message (:354-401); they read
  // only counters and actor states, so they are evaluated before the previous
  // delivery's outbox is drained (drain() then flushes only if we go on)
  __device__ __forceinline__ bool may_continue() {
    if (status | violation) return false;
    if (nsched > A->max_messages) { if (!STEADY) ext_idx = A->n_ext; return false; }
    if (A->interval > 0 && nmod == 0 && nsched != 0) {
      violation = check_invariant();
      if (violation) return false;
    }
    return true;
  }
  __device__ __forceinline__ bool pick_next(uint4& pick) {
    if (status) return false;
    if (n_pending == 0) return false;
    return pick_at(rng.next_int(n_pending), pick);              // Util.scala:171-176
  }
  // The pick of pending index i: what pick_next does once it has drawn i.  lane_tree_kernel picks each i in turn.
  __device__ __forceinline__ bool pick_at(uint32_t i, uint4& pick) {
    pick = pending_remove_at(i);
    nsched++;
    if (nsched == 0x7FFFFFFF) nsched = 1;
    if (++nmod == A->interval) nmod = 0;
    uint32_t src = hdr_src(pick.x), dst = hdr_dst(pick.x), type = hdr_type(pick.x);
    record_event(DEMI_EV_MSG_EVENT, src, dst, type, pick.y, pick.z, pick.w, 0);
    parent_event = pick.w >> 16;                                // reportNewlyDelivered (DepTracker.scala:132-135)
    window_timers = 0;
    // updateRepeatingTimer :405-421
    const int slot = MODEL::timer_slot(dst, type, pick.y, pick.z);
    if (slot >= 0 && ((registry >> slot) & 1u)) {
      just |= 1u << slot;
      // Instrumenter.dispatch_new_message's re-arm of the repeating timer (Instrumenter.scala:1008-1016), applied
      // here, before receive() as there: its enqueue_timer finds the just-set bit, so the slot goes to resend
      resend_push((uint32_t)slot);
    } else {
      // handle_timer of each re-send entry, in order.  messagesToSend is empty here: run() flushed it to the end just
      // before this pick (a flush that defers ends the execution), so the list becomes the whole queue, and its at most
      // LANE_RESEND_CAP entries always fit.
      if (STEADY || !A->ignore_timers) tosend.assign((uint32_t)resend, (uint32_t)(resend >> 32), n_resend);
      resend = 0; n_resend = 0;
      just = 0;
    }
    return !status;
  }

  // Instrumenter.dispatch_new_message (Instrumenter.scala:913-1017); pick_next has re-armed a repeating timer
  // returns the number of outbox ops receive() produced (applied by drain())
  __device__ __forceinline__ uint32_t dispatch_new_message(const uint4& pick) {
    uint32_t src = hdr_src(pick.x), dst = hdr_dst(pick.x), type = hdr_type(pick.x);
    if constexpr (DIRECT) {
      LaneDirectOutbox<LaneMachine> direct{this, dst};
      MODEL::receive(direct, dst, actor(dst), src, type, pick.y, pick.z, A->model_flags);
      return 0;
    }
    LaneOutbox<OB> ob;
    ob.base = smw + N * SW * BD; ob.bd = BD; ob.n = 0; ob.self = dst; ob.overflow = false;
    MODEL::receive(ob, dst, actor(dst), src, type, pick.y, pick.z, A->model_flags);
    if (ob.overflow) { defer(); return 0; }
    // equal sends out of one receive() would share a Unique (child reuse): defer.  A 64-bit filter over the
    // (op, dst, type) words settles the common case — all headers distinct — in one pass; only a filter hit
    // (a real duplicate, or a 1-in-64 collision) pays for the pairwise comparison.
    if (MODEL::LANE_SENDS_DISTINCT) return ob.n;                    // one send per receiver: nothing can be equal
    uint64_t seen = 0; bool maybe = false;
    for (uint32_t i = 0; i < ob.n; i++) {
      const uint64_t bit = 1ull << ((ob.base[(i * 3) * BD] * 0x9E3779B1u) >> 26);
      maybe |= (seen & bit) != 0;
      seen |= bit;
    }
    if (maybe)
    for (uint32_t i = 1; i < ob.n; i++) {
      const uint32_t wi = ob.base[(i * 3) * BD];
      for (uint32_t j = 0; j < i; j++)
        if (wi == ob.base[(j * 3) * BD] && (wi & 0xFF) == OP_SEND &&
            ob.base[(i * 3 + 1) * BD] == ob.base[(j * 3 + 1) * BD] && ob.base[(i * 3 + 2) * BD] == ob.base[(j * 3 + 2) * BD]) {
          defer(); return 0;
        }
    }
    return ob.n;
  }

  __device__ __forceinline__ void reset(int64_t seed) {
    rng.seed(seed);
#pragma unroll 1
    for (uint32_t i = 0; i < N * SW; i++) smw[i * BD] = MODEL::init_word(i, A->model_flags);
    if constexpr (!STEADY)
      for (uint32_t a = 0; a < N; a++) part_row(a) = 0;
    if constexpr (TW > 0)
      for (uint32_t w = 0; w < (uint32_t)TW; w++) smw[(N * SW + OBW + PW + w) * BD] = 0;
    n_pending = max_pending = 0;
    tosend.clear(); resend = 0; n_resend = 0;
    just = registry = cancelled = root_timers = window_timers = 0;
    n_nodes = 1; parent_event = 0; n_events = 0;
    nsched = 0; nmod = 0; ext_idx = 0; ext_send_idx = 0;
    violation = status = 0;
    inaccessible = (N >= 32) ? 0xFFFFFFFFu : ((1u << N) - 1u);
    killed = 0; thash = 0;
  }

  // An execution up to its first pick: the externals up to the first WaitQuiescence and the flush of their Sends.
  // It draws no random number, so it is the same for every seed; lane_snapshot_kernel runs it once per program.
  __device__ __forceinline__ void first_flush() {
    inject_until_quiescence();
    const bool go = may_continue();
    drain(0, 0, go);
  }
  // A node record of the tree (lane_steady.hpp): the header, the state and timer-copy words, then the pending rows.
  static constexpr uint32_t NODE_WORDS = lane_node_words(N * SW + TW);
  static constexpr uint32_t NODE_ROWS_AT = NODE_WORDS - LANE_NODE_ROWS * 4;
  __device__ __forceinline__ uint32_t& machine_word(uint32_t i) {      // i < N * SW: a state word, else a timer copy
    return smw[(i < (uint32_t)(N * SW) ? i : i + OBW + PW) * BD];
  }
  // Stores the machine as a node without children.  pend may already be the record's rows (lane_tree_kernel).
  __device__ __forceinline__ void store_node(uint32_t* r) {
    r[LN_CHILD] = LANE_NODE_LEAF; r[LN_N_PENDING] = n_pending; r[LN_NSCHED] = (uint32_t)nsched; r[LN_VIOLATION] = violation;
    r[LN_NMOD] = (uint32_t)nmod; r[LN_MAX_PENDING] = max_pending; r[LN_N_NODES] = n_nodes; r[LN_N_EVENTS] = n_events;
    r[LN_PARENT_EVENT] = parent_event; r[LN_REGISTRY] = registry; r[LN_CANCELLED] = cancelled; r[LN_JUST] = just;
    r[LN_WINDOW_TIMERS] = window_timers; r[LN_N_RESEND] = n_resend;
    r[LN_RESEND_LO] = (uint32_t)resend; r[LN_RESEND_HI] = (uint32_t)(resend >> 32);
    r[LN_THASH_LO] = (uint32_t)thash; r[LN_THASH_HI] = (uint32_t)(thash >> 32);
    for (uint32_t i = 0; i < (uint32_t)(N * SW + TW); i++) r[LANE_NODE_HEAD + i] = machine_word(i);
    uint4* rows = reinterpret_cast<uint4*>(r + NODE_ROWS_AT);
    if ((void*)rows != (void*)pend)
      for (uint32_t i = 0; i < n_pending; i++) rows[i] = row_load(i);
  }
  // The steady machine becomes the one stored in record r (status 0): every register and shared word the rest of an
  // execution reads.  tosend is empty at a stored pick point, or never read again when the execution stops there.
  __device__ __forceinline__ void load_node(const uint32_t* r) {
    static_assert(STEADY, "a node is the steady machine");
    const uint4* q = reinterpret_cast<const uint4*>(r);
    const uint4 h0 = __ldg(q), h1 = __ldg(q + 1), h2 = __ldg(q + 2), h3 = __ldg(q + 3), h4 = __ldg(q + 4);
    n_pending = h0.y; nsched = (int32_t)h0.z; violation = h0.w;
    nmod = (int32_t)h1.x; max_pending = h1.y; n_nodes = h1.z; n_events = h1.w;
    parent_event = h2.x; registry = h2.y; cancelled = h2.z; just = h2.w;
    window_timers = h3.x; n_resend = h3.y; resend = h3.z | (uint64_t)h3.w << 32;
    thash = h4.x | (uint64_t)h4.y << 32;
    status = 0;
    tosend.clear();
#pragma unroll 1
    for (uint32_t i = 0; i < (uint32_t)(N * SW + TW); i++) machine_word(i) = __ldg(r + LANE_NODE_HEAD + i);
    const uint4* rows = reinterpret_cast<const uint4*>(r + NODE_ROWS_AT);
#pragma unroll 1
    for (uint32_t i = 0; i < n_pending; i++) st_l2_hint(pend + i, row_pack(__ldg(rows + i)), pol);
  }
  // STEADY: the machine after the execution's first picks.  Each level of the tree draws the index pick_next would
  // draw; the walk stops at a node without children, or before a child that is not stored, and leaves the generator
  // as it is before the draw that the delivery loop then makes again.  The loop re-enters at its top, where
  // may_continue() repeats a pure check (or stops the execution, as it did when the node was stored) and drain()
  // finds tosend empty.
  __device__ __forceinline__ void restore() {
    const uint32_t* tree = reinterpret_cast<const uint32_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&A->lane_snap->tree)));
    const uint32_t* at = tree;
    uint4 h = __ldg(reinterpret_cast<const uint4*>(at));
#pragma unroll 1
    while (h.x != LANE_NODE_LEAF) {
      JRandom r = rng;
      const uint32_t* c = tree + (size_t)(h.x + r.next_int(h.y)) * NODE_WORDS;
      const uint4 hc = __ldg(reinterpret_cast<const uint4*>(c));
      if (hc.y == LANE_NODE_ABSENT) break;
      rng = r; at = c; h = hc;
    }
    load_node(at);
  }

  // The deliveries of an execution, segment by segment.  STEADY has one segment and starts it at the top of the
  // delivery loop: with nothing scheduled and tosend empty, may_continue() and drain() do nothing before the first pick.
  __device__ __forceinline__ void deliver() {
    uint32_t n_ops = 0, self = 0;          // outbox of the delivery that has not been drained yet
    for (;;) {
      if constexpr (!STEADY) inject_until_quiescence();
      for (;;) {
        clk.enter(LP_INVARIANT);
        const bool go = may_continue();
        clk.enter(LP_FLUSH);
        drain(n_ops, self, go);            // previous receive()'s sends, then (if going on) the flush
        n_ops = 0;
        uint4 pick;
        clk.enter(LP_PICK);
        if (!go || !pick_next(pick)) break;
        self = hdr_dst(pick.x);
        clk.enter(LP_RECEIVE);
        n_ops = dispatch_new_message(pick);
        if (status) break;
      }
      clk.enter(LP_TAIL);
      if constexpr (STEADY) break;
      if (status | violation) break;
      if (ext_idx < A->n_ext) {
        record_event(DEMI_EV_QUIESCENCE, DEMI_DEADLETTERS, DEMI_DEADLETTERS, 0, 0, 0, 0, 0);
        continue;
      }
      break;
    }
  }
  // The final invariant check and the result record.
  __device__ __forceinline__ void finish(demi_fuzz_result& out) {
    if (!status && nsched <= A->max_messages && !violation) violation = check_invariant();
    if (n_pending > max_pending) max_pending = n_pending;
    out.status = (uint16_t)status;
    if (!status) {
      uint64_t sh = 0;
#pragma unroll 1
      for (uint32_t i = 0; i < N * SW; i++) sh += demi_state_term(smw[i * BD], i);
      if (A->fuzz_flags & DEMI_FF_HASH_PENDING)
#pragma unroll 1
        for (uint32_t i = 0; i < n_pending; i++) {
          const uint4 q = row_load(i);
          sh += demi_pending_term(q.x & 0x00FFFFFFu, q.y, q.z);
        }
      out.violation = violation; out.steps = (uint32_t)nsched;
      out.state_hash = sh; out.trace_hash = thash;
      out.n_nodes = (uint16_t)n_nodes;
      out.n_events = (uint16_t)(n_events > 65535u ? 65535u : n_events);
      out.max_pending = (uint16_t)max_pending;
    }
  }

  __device__ __forceinline__ void run(int64_t seed, demi_fuzz_result& out) {
    clk.enter(LP_TAIL);
    if constexpr (STEADY) { rng.seed(seed); restore(); }
    else reset(seed);
    deliver();
    finish(out);
  }
};

// The pre-delivery snapshot of the launch's program (lane_steady.hpp): one thread runs reset() and first_flush() of
// the generic machine with the physical limits in place of a batch's capacities (a batch compares the recorded
// counts with its own), LANE_SNAP_CAP pending rows (a program that enables more defers, and is not snapshotted),
// and stores the machine, both as the snapshot's scalars (what the host decides on) and as the root record of the
// tree, which follows the snapshot.  Launched when the program is set, not per batch.
template <class MODEL>
__global__ void lane_snapshot_kernel(const __grid_constant__ KernelArgs args, LaneSnapshot* out) {
  using M = LaneMachine<MODEL, 1, (int)LANE_SNAP_CAP>;
  static_assert(M::NODE_WORDS == LaneMachine<MODEL, 1, 1, false, true>::NODE_WORDS, "one record layout per model");
  __shared__ uint32_t smem[M::WORDS];
  M m;
  m.smw = smem;
  m.pend = reinterpret_cast<uint4*>(out->pend);
  m.A = &args;
  m.pol = l2_evict_last_policy();
  m.rec_ev = nullptr; m.rec_par = nullptr;
  m.reset(0);
  m.first_flush();
  out->thash = m.thash;
  out->n_pending = m.n_pending; out->n_nodes = m.n_nodes; out->n_events = m.n_events; out->parent_event = m.parent_event;
  out->root_timers = m.root_timers; out->registry = m.registry; out->cancelled = m.cancelled; out->tosend_n = m.tosend.n;
  out->ext_idx = m.ext_idx; out->ext_send_idx = m.ext_send_idx; out->inaccessible = m.inaccessible; out->killed = m.killed;
  out->status = m.status;
  m.store_node(reinterpret_cast<uint32_t*>(out + 1));
}

// One level of the tree: thread c builds child c of the level, the machine after its parent picks pending index
// kids[c].y, delivers it and reaches its next pick point (the top of the delivery loop: may_continue() and the flush),
// exactly as the steady kernel does.  The launch's pending bound is lowered to the record's rows: an execution that
// would exceed them defers here and is not stored, like every deferred one, so the walk stops at its parent and the
// steady kernel runs that delivery itself.  The first child of each parent links the parent to its children.
constexpr int LANE_TREE_BD = 32;
template <class MODEL, int LPCAP>
__global__ void __launch_bounds__(LANE_TREE_BD)
lane_tree_kernel(const __grid_constant__ KernelArgs args, uint32_t* tree, const uint2* kids, uint32_t first, uint32_t n) {
  using M = LaneMachine<MODEL, LANE_TREE_BD, LPCAP, false, true>;
  __shared__ uint32_t smem[M::WORDS * LANE_TREE_BD];
  const uint32_t c = blockIdx.x * LANE_TREE_BD + threadIdx.x;
  if (c >= n) return;
  const uint2 k = kids[c];
  uint32_t* r = tree + (size_t)(first + c) * M::NODE_WORDS;
  M m;
  m.smw = smem + threadIdx.x;
  m.pend = reinterpret_cast<uint4*>(r + M::NODE_ROWS_AT);
  m.A = &args;
  m.pol = l2_evict_last_policy();
  m.rec_ev = nullptr; m.rec_par = nullptr;
  m.clk.start();
  m.rng.seed(0);
  m.load_node(tree + (size_t)k.x * M::NODE_WORDS);
  uint4 pick;
  if (m.pick_at(k.y, pick)) {
    const uint32_t n_ops = m.dispatch_new_message(pick);
    if (!m.status) {
      const bool go = m.may_continue();
      m.drain(n_ops, hdr_dst(pick.x), go);
    }
  }
  if (m.status) r[LN_N_PENDING] = LANE_NODE_ABSENT;
  else m.store_node(r);
  if (k.y == 0) tree[(size_t)k.x * M::NODE_WORDS + LN_CHILD] = first + c;
}

#ifndef DEMI_K1_MIN_BLOCKS
#define DEMI_K1_MIN_BLOCKS 3
#endif
// REC launches walk a work list (`index_list`): slot `it` of the list owns rec_events[it*rec_cap ..), rec_parent[it*cap ..),
// rec_counts[it*4 ..) and results[it]; a deferred slot is handed to the general engine by POSITION (ovf_list holds `it`).
// PROG (campaigns; with TESTS random-oracle tests, see fuzz_kernel): prefix idx runs its program of the arena in `args.prog_*`; the 0x80 | k entries
// of messagesToSend resolve through that program's Send table.  A deferred prefix keeps its index, so the PROG
// instantiation of the warp engine re-runs it on the same program.
template <class MODEL, int BD, int LPCAP, bool REC = false, bool PROG = false, bool TESTS = false, bool STEADY = false,
          bool PARAMS = false, bool ROW8 = false>
__global__ void __launch_bounds__(BD, DEMI_K1_MIN_BLOCKS)
fuzz_lane_kernel(const __grid_constant__ KernelArgs args) {
  static_assert(!(PROG && REC), "a campaign execution is recorded through demi_fuzz_trace on its program");
  static_assert(PROG || !TESTS, "random-oracle tests bind their programs as campaigns do");
  static_assert(!STEADY || !(REC || PROG), "a steady launch runs one fixed program, unrecorded");
  static_assert(TESTS || !PARAMS, "per-program parameters are those of random-oracle tests");
  using M = LaneMachine<MODEL, BD, LPCAP, REC, STEADY, ROW8>;
  extern __shared__ __align__(16) uint32_t lane_smem[];
  const uint32_t tid = threadIdx.x;
  const uint64_t gthread = (uint64_t)blockIdx.x * BD + tid;
  const uint64_t total = (uint64_t)gridDim.x * BD;

  M m;
  m.smw = lane_smem + tid;
  m.pend = reinterpret_cast<typename M::Row*>(args.lane_pend) + gthread * (uint64_t)LPCAP;     // LPCAP rows per thread
  KernelArgs la;
  if constexpr (PROG) { la = args; m.A = &la; } else m.A = &args;
  m.pol = l2_evict_last_policy();
  m.rec_ev = nullptr; m.rec_par = nullptr;
  m.clk.start();

  const uint64_t count = (REC && args.index_list) ? (uint64_t)(*args.index_count) : args.n_prefixes;
  unsigned long long my_steps = 0;
  uint32_t my_viol = 0, my_defer = 0;      // at most one per prefix of this thread
  for (uint64_t it = gthread; it < count; it += total) {
    const uint64_t idx = (REC && args.index_list) ? (uint64_t)args.index_list[it] : it;
    if (REC) {
      m.rec_ev = reinterpret_cast<uint4*>(args.rec_events + it * (uint64_t)args.rec_cap);
      m.rec_par = args.rec_parent + it * (uint64_t)args.rec_parent_cap;
      m.rec_par[0] = 0;
    }
    demi_fuzz_result r;
    if constexpr (TESTS) {
      uint64_t prog; int64_t seed;
      if (prog_test_bind<PARAMS>(la, args, idx, true, prog, seed)) {
        m.run(seed, r);
        prog_note_hit(args, idx, prog, r);
      } else {
        r = demi_fuzz_result{};
        r.status = PS_SKIPPED;
      }
    } else {
      if constexpr (PROG) prog_bind(la, args, idx, true);
      m.run(seed_at(args.seed_base, idx), r);
    }
    if (r.status == LANE_DEFER) {
      uint32_t pos = atomicAdd(args.ovf_count, 1u);
      args.ovf_list[pos] = (uint32_t)(REC ? it : idx);
      my_defer++;
    } else {
      // written once, never re-read here: streaming stores, so that the records do not push the pending arrays out of L2
      uint4* dst = reinterpret_cast<uint4*>(args.results + (REC ? it : idx));
      const uint4 r0 = make_uint4(r.violation, r.steps, (uint32_t)r.state_hash, (uint32_t)(r.state_hash >> 32));
      const uint4 r1 = make_uint4((uint32_t)r.trace_hash, (uint32_t)(r.trace_hash >> 32), (uint32_t)r.n_nodes | ((uint32_t)r.n_events << 16),
                                  (uint32_t)r.max_pending | ((uint32_t)r.status << 16));
#if DEMI_K1_RESULT_CS
      __stcs(dst, r0); __stcs(dst + 1, r1);
#else
      dst[0] = r0; dst[1] = r1;
#endif
      if (REC) {
        uint32_t aff = 0;
        if (r.status == 0 && r.violation) {      // ViolationFingerprint.affectedNodes of the violation the execution stopped on
          uint32_t st[M::N * M::SW];
          for (uint32_t i = 0; i < (uint32_t)(M::N * M::SW); i++) st[i] = m.smw[i * BD];
          aff = MODEL::affected(st, args.model_flags, r.violation);
        }
        reinterpret_cast<uint4*>(args.rec_counts)[it] = make_uint4(m.n_events, m.n_nodes, aff, r.violation);
      }
      my_steps += r.steps;
      my_viol += r.violation ? 1u : 0u;
    }
  }
  m.clk.finish();
  // warp-aggregate the summary counters
  for (int o = 16; o > 0; o >>= 1) {
    my_steps += __shfl_xor_sync(FULL_MASK, my_steps, o);
    my_viol += __shfl_xor_sync(FULL_MASK, my_viol, o);
    my_defer += __shfl_xor_sync(FULL_MASK, my_defer, o);
  }
  if ((tid & 31) == 0 && args.sum_steps && (my_steps | my_viol | my_defer)) {
    atomicAdd(args.sum_steps, my_steps);
    atomicAdd(args.n_violations, (unsigned long long)my_viol);
    if (my_defer) atomicAdd(args.sum_steps + 2, (unsigned long long)my_defer);      // [2]: prefixes handed to the general engine
  }
}

}  // namespace demi
