// machine.cuh — the warp-cooperative "DEMi machine": one RandomScheduler
// execution (reference: schedulers/RandomScheduler.scala:234-272, :352-485)
// owned by one warp.
//
// Layout (per warp):
//   shared memory : pending-message array (RandomizedHashSet.arr, Util.scala:112)
//                   as uint4 {hdr,p0,p1,uniq|node<<16}, actor states, the
//                   messagesToSend queue, the receive() outbox
//   registers     : java.util.Random state, counters, network masks (uniform);
//                   timer sets, partition rows, recent dep-tree nodes and the
//                   "delivered" bitmap are LANE-DISTRIBUTED (lane i holds entry
//                   i; membership tests are one compare + ballot)
//   global scratch: the DepTracker node table (only re-read when a parent can
//                   have older children), optional EventTrace recording
//
// Control flow is warp-uniform.  The actor's receive() runs on lane 0 only and
// emits its sends / timer operations into an outbox that the whole warp then
// applies in program order (the reference delivers `!` synchronously and in
// program order, Instrumenter.scala:1098-1108).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "../../include/demi_b200.h"
#include "../../include/demi_limits.h"

namespace demi {

constexpr unsigned FULL_MASK = 0xffffffffu;
constexpr uint32_t FIFO_PAIRS = 1056;      // (32 actors + deadLetters... pair code = src*32+dst) rounded up
constexpr uint32_t FIFO_NIL = 0xFFFFu;
constexpr int OUTBOX_CAP = 40;

enum OutOp : uint32_t { OP_SEND = 0, OP_SCHED_ONCE = 1, OP_SCHED_REPEAT = 2, OP_CANCEL = 3 };

__device__ __forceinline__ uint32_t make_hdr(uint32_t src, uint32_t dst, uint32_t type, uint32_t flags) {
  return src | (dst << 8) | (type << 16) | (flags << 24);
}
__device__ __forceinline__ uint32_t hdr_src(uint32_t h) { return h & 0xFF; }
__device__ __forceinline__ uint32_t hdr_dst(uint32_t h) { return (h >> 8) & 0xFF; }
__device__ __forceinline__ uint32_t hdr_type(uint32_t h) { return (h >> 16) & 0xFF; }
__device__ __forceinline__ uint32_t hdr_flags(uint32_t h) { return h >> 24; }
// timer key: (receiver, message) with the message == (type,p0,p1)
__device__ __forceinline__ uint32_t timer_key(uint32_t dst, uint32_t type) { return dst | (type << 8); }

// What receive() sees: a scalar, single-lane view.
struct Outbox {
  uint4* ops;        // shared memory, OUTBOX_CAP entries
  uint32_t n;
  uint32_t self;
  bool overflow;
  __device__ __forceinline__ void push(uint32_t op, uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) {
    if (n >= OUTBOX_CAP) { overflow = true; return; }
    ops[n++] = make_uint4(op | (dst << 8) | (type << 16), p0, p1, 0u);
  }
  // the next `k` operations are sends (models.cuh Raft5): nothing to prepare here
  __device__ __forceinline__ bool reserve(uint32_t) { return true; }
  // `dst ! msg`
  __device__ __forceinline__ void send(uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) { push(OP_SEND, dst, type, p0, p1); }
  // context.system.scheduler.scheduleOnce(_, self, msg)
  __device__ __forceinline__ void schedule_once(uint32_t type, uint32_t p0, uint32_t p1) { push(OP_SCHED_ONCE, self, type, p0, p1); }
  // context.system.scheduler.schedule(_, _, self, msg)
  __device__ __forceinline__ void schedule_repeating(uint32_t type, uint32_t p0, uint32_t p1) { push(OP_SCHED_REPEAT, self, type, p0, p1); }
  // cancellable.cancel()
  __device__ __forceinline__ void cancel_timer(uint32_t type, uint32_t p0, uint32_t p1) { push(OP_CANCEL, self, type, p0, p1); }
};

// State accessor of one actor over contiguous (shared) memory: warp engine.
struct ContigState {
  uint32_t* p;
  __device__ __forceinline__ uint8_t& operator[](uint32_t i) const { return reinterpret_cast<uint8_t*>(p)[i]; }
  __device__ __forceinline__ uint8_t& b(uint32_t i) const { return reinterpret_cast<uint8_t*>(p)[i]; }
  __device__ __forceinline__ uint32_t& w(uint32_t i) const { return p[i]; }
};

// Lane-distributed small ordered set of (receiver,msg) keys; lane i holds entry i.
struct LaneSet {
  uint32_t key, p0, p1;   // this lane's entry
  uint32_t n;             // warp-uniform count
  __device__ __forceinline__ void clear() { n = 0; }
  __device__ __forceinline__ int find(uint32_t lane, uint32_t k, uint32_t a, uint32_t b) const {
    unsigned m = __ballot_sync(FULL_MASK, lane < n && key == k && p0 == a && p1 == b);
    return m ? (__ffs(m) - 1) : -1;
  }
  // returns false on overflow
  __device__ __forceinline__ bool push(uint32_t lane, uint32_t k, uint32_t a, uint32_t b) {
    if (n >= DEMI_TIMERSET_CAP) return false;
    if (lane == n) { key = k; p0 = a; p1 = b; }
    n++;
    return true;
  }
  __device__ __forceinline__ void remove_at(uint32_t lane, uint32_t i) {
    uint32_t k2 = __shfl_down_sync(FULL_MASK, key, 1);
    uint32_t a2 = __shfl_down_sync(FULL_MASK, p0, 1);
    uint32_t b2 = __shfl_down_sync(FULL_MASK, p1, 1);
    if (lane >= i) { key = k2; p0 = a2; p1 = b2; }
    n--;
  }
  // warp-uniform read of entry i
  __device__ __forceinline__ void get(uint32_t i, uint32_t& k, uint32_t& a, uint32_t& b) const {
    k = __shfl_sync(FULL_MASK, key, i); a = __shfl_sync(FULL_MASK, p0, i); b = __shfl_sync(FULL_MASK, p1, i);
  }
};

// java.util.Random (Java SE spec; seeded at schedulers/Util.scala:115, drawn at :172)
struct JRandom {
  uint64_t s;
  __device__ __forceinline__ void seed(int64_t v) { s = ((uint64_t)v ^ 0x5DEECE66Dull) & ((1ull << 48) - 1); }
  __device__ __forceinline__ uint32_t next31() {
    s = (s * 0x5DEECE66Dull + 0xBull) & ((1ull << 48) - 1);
    return (uint32_t)(s >> 17);
  }
  __device__ __forceinline__ uint32_t next_int(uint32_t bound) {   // bound > 0
    uint32_t r = next31();
    uint32_t m = bound - 1;
    if ((bound & m) == 0) return (uint32_t)(((uint64_t)bound * (uint64_t)r) >> 31);
    uint32_t u = r;
    // java: while (u - (r = u % bound) + m < 0) in int32 arithmetic
    while ((int32_t)(u - (r = u % bound) + m) < 0) u = next31();
    return r;
  }
};
// The seed of execution `off` of a batch that starts at `base`.  Java's long addition wraps, and only the low 48 bits
// reach the generator, so the sum is taken in uint64_t: int64_t addition would be undefined past INT64_MAX.
__host__ __device__ __forceinline__ int64_t seed_at(int64_t base, uint64_t off) { return (int64_t)((uint64_t)base + off); }

struct LaneSnapshot;
struct KernelArgs {
  // configuration
  uint32_t model_flags;
  uint32_t blocked_mask;
  int32_t  ignore_timers;
  int32_t  max_messages;      // already mapped: <0 -> INT_MAX
  int32_t  interval;
  uint32_t looking_for;
  int64_t  seed_base;
  uint64_t n_prefixes;
  uint32_t fuzz_flags;        // DEMI_FF_*
  int32_t  strategy;          // DEMI_RS_* (SrcDstFIFO needs a PEND_GLOBAL variant)
  uint16_t* fifo_scratch;     // [total_warps][PCAP/2 + 3*FIFO_PAIRS] u16: next[], head[], tail[], pairs[]
  // external-event program
  const demi_ext_event* ext;
  uint32_t n_ext;
  // capacities of this launch
  uint32_t node_cap;          // dep-tree nodes per warp in `node_scratch` (spec: demi_node_cap)
  uint32_t pending_cap;       // spec capacity (demi_pending_cap) <= physical PCAP
  uint32_t tosend_cap;        // spec capacity (demi_tosend_cap)  <= physical TCAP
  // outputs
  demi_fuzz_result* results;
  // tiering: if `index_list` != null the launch handles prefixes index_list[0..*index_count)
  const uint32_t* index_list;
  const uint32_t* index_count;
  // recording launches only: if `pos_list` != null, handle just the work-list POSITIONS pos_list[0..*pos_count)
  const uint32_t* pos_list;
  const uint32_t* pos_count;
  // prefixes that overflowed THIS tier are appended here (may be null => final tier)
  uint32_t* ovf_list;
  uint32_t* ovf_count;
  // scratch
  uint4*    node_scratch;     // [total_warps][node_cap]
  uint4*    pend_scratch;     // [total_warps][pending_cap] when the pending set lives in HBM
  // recording launches: slot `it` (the position in the launch's work list) owns rec_events[it*rec_cap ..),
  // rec_counts[it*4 ..) = {n_events, n_nodes, affectedNodes, violation} and rec_parent[it*rec_parent_cap ..)
  union {
    demi_event* rec_events;
    // the TESTS + PARAMS kernels (demi_random_test_batch_many), which never record: test p's {seed_base lo, hi, max_messages
    // as the caller gave it, looking_for}.  In the recording slot, so that the struct stays as it was.
    const uint4* prog_params;
  };
  uint32_t rec_cap; uint32_t* rec_counts; uint16_t* rec_parent; uint32_t rec_parent_cap;
  // summary counters
  unsigned long long* sum_steps; unsigned long long* n_violations;
  // lane engine (lane_kernel.cuh)
  union {
    uint4*  lane_pend;        // [total_warps][LPCAP][32] pending entries
    // the many-program recording kernels (demi_fuzz_traces_many), warp engine only: execution idx's {seed lo, hi,
    // max_messages as the caller gave it, looking_for}, as `prog_params`.  In the lane engine's slot, which a warp-engine
    // launch never reads, so that the struct stays as it was.
    const uint4* rec_params;
  };
  union {
    const uint4* ext_sends;   // the program's Send events as {hdr|EXTERNAL, p0, p1, 0}, in order
    // STEADY launches inject nothing and have no Send table: they read the program's pre-delivery snapshot
    // (lane_steady.hpp) through the same slot, so that the struct, and with it every other kernel, stays as it was
    const LaneSnapshot* lane_snap;
  };
  uint32_t  has_partitions;   // program contains Partition/UnPartition events
  // FullyRandom's userDefinedFilter as rules (demi_set_user_filter): {src_mask, dst_mask, type_mask, flags}
  uint4     filter[DEMI_MAX_FILTER_RULES]; uint32_t n_filter;
  // campaign launches (the PROG kernels): execution idx runs program idx of the arena, under that program's own
  // capacities (demi_pending_cap / demi_tosend_cap / demi_node_cap of its Sends).  Appended last, so that the
  // parameter offsets of the other kernels stay where they were.
  const demi_ext_event* prog_ext;      // [n][prog_stride] events
  const uint2* prog_hdr;               // [n] {length, number of Sends}
  const uint4* prog_sends;             // [n][prog_send_stride] the Sends as in `ext_sends` (lane engine)
  uint32_t prog_stride, prog_send_stride;
  int32_t  prog_model_key;             // the `model` argument of the capacity rules
  int32_t  prog_max_messages;          // max_messages as the caller gave it (the capacity rules read it unmapped)
  uint32_t prog_lane_pcap;             // lane engine: defer beyond this many pending messages (0 = no extra limit)
  // random-oracle tests (demi_random_test_batch, the TESTS kernels): execution idx runs program idx / prog_execs under
  // seed_base + idx % prog_execs; prog_first_hit[program] is the lowest execution index with a hit so far (atomicMin,
  // 0xFFFFFFFF = none), and an execution whose index is above it is skipped (PS_SKIPPED)
  uint32_t prog_execs;
  uint32_t* prog_first_hit;
};
// the record status of an execution skipped because its program already has a hit at a lower index (never leaves
// the device: the per-test reduction reads it)
constexpr uint16_t PS_SKIPPED = 0xFFFEu;
// The program view of a campaign execution: `la` is the executing thread's copy of the launch arguments, and
// `max_messages` the program's, unmapped.
__device__ __forceinline__ void prog_bind(KernelArgs& la, const KernelArgs& args, uint64_t idx, bool lane, int32_t max_messages) {
  const uint2 h = args.prog_hdr[idx];
  la.ext = args.prog_ext + idx * (uint64_t)args.prog_stride;
  la.n_ext = h.x;
  la.pending_cap = demi_pending_cap(args.prog_model_key, max_messages, h.y);
  if (lane && args.prog_lane_pcap && args.prog_lane_pcap < la.pending_cap) la.pending_cap = args.prog_lane_pcap;
  la.tosend_cap = demi_tosend_cap(h.y);
  la.node_cap = demi_node_cap(demi_pending_cap(args.prog_model_key, max_messages, h.y));
  la.ext_sends = args.prog_sends + idx * (uint64_t)args.prog_send_stride;
}
__device__ __forceinline__ void prog_bind(KernelArgs& la, const KernelArgs& args, uint64_t idx, bool lane) {
  prog_bind(la, args, idx, lane, args.prog_max_messages);
}
// A program's own parameters q = {seed base lo, hi, max_messages as the caller gave it, looking_for}: execution j of it
// runs under seed base + j; binds max_messages (mapped as plan_launch maps it) and looking_for, and returns max_messages
// unmapped, which the capacity rules read.
__device__ __forceinline__ int32_t prog_params_bind(KernelArgs& la, const uint4 q, uint32_t j, int64_t& seed) {
  seed = seed_at((int64_t)(((uint64_t)q.y << 32) | q.x), j);
  const int32_t max_messages = (int32_t)q.z;
  la.max_messages = max_messages < 0 ? 0x7FFFFFFF : max_messages;
  la.looking_for = q.w;
  return max_messages;
}
// A random-oracle test execution (the TESTS kernels): execution idx is execution j = idx % prog_execs of program
// prog = idx / prog_execs, under seed_base + j.  Binds the program on every path (so that the copy stays in
// registers) and returns false if the execution is skipped.  `lane`: one thread per execution (else a warp, kept
// uniform).  PARAMS: the program's seed base, max_messages and looking_for come from prog_params[prog].
template <bool PARAMS = false>
__device__ __forceinline__ bool prog_test_bind(KernelArgs& la, const KernelArgs& args, uint64_t idx, bool lane, uint64_t& prog,
                                               int64_t& seed) {
  const uint32_t p = (uint32_t)idx / args.prog_execs, j = (uint32_t)idx - p * args.prog_execs;
  prog = p;
  int32_t max_messages = args.prog_max_messages;
  if constexpr (PARAMS) {
    max_messages = prog_params_bind(la, args.prog_params[p], j, seed);
  } else {
    seed = seed_at(args.seed_base, j);
  }
  uint32_t fh = *(volatile const uint32_t*)(args.prog_first_hit + p);
  if (!lane) fh = __shfl_sync(FULL_MASK, fh, 0);
  prog_bind(la, args, p, lane, max_messages);
  return j <= fh;
}
// after a TESTS execution: a hit lowers its program's first_hit (the caller writes from one thread per execution)
__device__ __forceinline__ void prog_note_hit(const KernelArgs& args, uint64_t idx, uint64_t prog, const demi_fuzz_result& r) {
  if (r.status == 0 && r.violation)
    atomicMin(args.prog_first_hit + prog, (uint32_t)idx - (uint32_t)prog * args.prog_execs);
}

// -----------------------------------------------------------------------------
// The machine.  MODEL supplies: N_ACTORS, STATE_WORDS, init_state(), receive(),
// invariant_lane().  PCAP/TCAP: pending / messagesToSend capacities.
// PEND_GLOBAL: pending array lives in HBM scratch instead of shared memory.
template <class MODEL, int PCAP, int TCAP, bool PEND_GLOBAL, bool RECORD>
struct Machine {
  static constexpr int N = MODEL::N_ACTORS;
  static constexpr int SW = MODEL::STATE_WORDS;

  // ---- per-warp shared memory view
  struct Smem {
    uint4 pend[PEND_GLOBAL ? 1 : PCAP];
    uint4 tosend[TCAP];
    uint4 outbox[OUTBOX_CAP];
    uint32_t states[N * SW];
  };

  Smem* sm;
  uint4* pend_g;            // PEND_GLOBAL
  uint4* nodes_g;           // dep-tree node table {hdr,p0,p1,parent}
  demi_event* rec_ev;       // RECORD: this execution's EventTrace slot
  const KernelArgs* A;
  uint32_t lane;

  // ---- warp-uniform registers
  JRandom rng;
  uint32_t n_pending, max_pending, n_tosend;
  uint32_t n_nodes, parent_event, recent_base, n_recent;
  bool scan_full;
  uint32_t n_events, n_uniq;
  int32_t nsched, nmod;
  uint32_t ext_idx;
  uint32_t violation, status;
  uint32_t inaccessible, killed;
  uint32_t dead, blocked;     // hard-killed actors (receiverIsAlive false); Instrumenter.blockedActors of this execution
  uint64_t thash;
  // ---- SrcDstFIFO (RandomScheduler.scala:702-909); only in PEND_GLOBAL variants.  The lower half of the
  // pending array is timersAndExternals (:712), the upper half the entry pool of the per-pair FIFO lists
  // srcDstToMessages (:706); srcDsts (:704) is `f_pairs`.
  static constexpr uint32_t HALF = PCAP / 2;
  JRandom rng_pairs;
  uint32_t n_pairs, n_queued, fifo_free;
  uint16_t *f_next, *f_head, *f_tail, *f_pairs;
  __device__ __forceinline__ bool fifo_mode() const { return PEND_GLOBAL && A->strategy == DEMI_RS_SRC_DST_FIFO; }
  __device__ __forceinline__ uint32_t ld16(const uint16_t* p) const { return (uint32_t)__ldcg(p); }

  // ---- lane-distributed registers
  LaneSet just, resend, registry, cancelled;
  uint32_t part_row;        // lane a: EventOrchestrator.partitioned row of actor a
  uint32_t r_hdr, r_p0, r_p1, r_parent;   // lane i: i-th node created since the last delivery
  uint32_t delivered_bits;  // lane w: bit b set <=> node 32w+b has been delivered before

  // ------------------------------------------------------------- pending array
  __device__ __forceinline__ uint4 pend_load(uint32_t i) const {
    if (PEND_GLOBAL) return __ldcg(&pend_g[i]);
    return sm->pend[i];
  }
  __device__ __forceinline__ void pend_store(uint32_t i, uint4 v) {
    if (PEND_GLOBAL) __stcg(&pend_g[i], v); else sm->pend[i] = v;
  }

  // EventTrace.+= / appendMsgSend / appendMsgEvent (EventTrace.scala:88-110)
  __device__ __forceinline__ void record_event(uint32_t kind, uint32_t src, uint32_t dst, uint32_t type,
                                               uint32_t p0, uint32_t p1, uint32_t uniq, uint32_t node,
                                               uint32_t parent) {
    uint32_t w0 = kind | (src << 8) | (dst << 16) | (type << 24);
    uint32_t w3 = uniq | (node << 16);
    thash += demi_event_term(w0, p0, p1, w3, n_events, parent);
    if (RECORD) {
      if (n_events >= A->rec_cap) { status = DEMI_PS_EVENT_OVF; return; }
      if (lane == 0) reinterpret_cast<uint4*>(rec_ev)[n_events] = make_uint4(w0, p0, p1, w3);
    }
    n_events++;
  }

  // RandomizedHashSet.insert: append (schedulers/Util.scala:126-136)
  // SrcDstFIFO.+= (RandomScheduler.scala:786-805)
  __device__ __forceinline__ void fifo_insert(uint4 e) {
    if (n_pending + n_queued >= A->pending_cap) { status = DEMI_PS_PENDING_OVF; return; }
    if (hdr_src(e.x) == DEMI_DEADLETTERS) {
      if (n_pending >= HALF) { status = DEMI_PS_PENDING_OVF; return; }
      if (lane == 0) pend_store(n_pending, e);
      n_pending++;
    } else {
      if (n_queued >= HALF) { status = DEMI_PS_PENDING_OVF; return; }
      const uint32_t pair = hdr_src(e.x) * 32u + hdr_dst(e.x);
      const uint32_t slot = fifo_free;
      fifo_free = ld16(f_next + slot);
      const uint32_t head = ld16(f_head + pair), tail = ld16(f_tail + pair);
      __syncwarp();
      if (lane == 0) {
        pend_store(HALF + slot, e);
        __stcg(f_next + slot, (uint16_t)FIFO_NIL);
        if (head == FIFO_NIL) { __stcg(f_pairs + n_pairs, (uint16_t)pair); __stcg(f_head + pair, (uint16_t)slot); }
        else __stcg(f_next + tail, (uint16_t)slot);
        __stcg(f_tail + pair, (uint16_t)slot);
      }
      if (head == FIFO_NIL) n_pairs++;
      n_queued++;
      __syncwarp();
    }
    if (n_pending + n_queued > max_pending) max_pending = n_pending + n_queued;
  }
  __device__ __forceinline__ void pending_insert(uint4 e) {
    if (fifo_mode()) { fifo_insert(e); return; }
    if (n_pending >= A->pending_cap) { status = DEMI_PS_PENDING_OVF; return; }
    if (lane == 0) pend_store(n_pending, e);
    n_pending++;
    if (n_pending > max_pending) max_pending = n_pending;
  }
  // RandomizedHashSet.remove: A[i] = A[last]; shrink (schedulers/Util.scala:146-163).
  // Caller must have made prior stores visible (__syncwarp).
  __device__ __forceinline__ uint4 pending_remove_at(uint32_t i) {
    uint4 v = pend_load(i);
    uint4 last = pend_load(n_pending - 1);
    __syncwarp();
    if (lane == 0) pend_store(i, last);
    n_pending--;
    __syncwarp();
    return v;
  }

  // DepTracker.getMessage + addNodeAndEdge (DepTracker.scala:82-116): reuse the
  // lowest-id child of parentEvent with equal (snd,rcv,fingerprint), else
  // allocate the next Unique.
  __device__ __forceinline__ uint32_t dep_report_newly_enabled(uint32_t hdr_noflags, uint32_t p0, uint32_t p1) {
    int found = -1;
    if (scan_full) {
      __syncwarp();
      for (uint32_t base = 1; base < n_nodes && found < 0; base += 32) {
        uint32_t i = base + lane;
        bool hit = false;
        if (i < n_nodes) {
          uint4 nd = __ldcg(&nodes_g[i]);
          hit = nd.w == parent_event && nd.x == hdr_noflags && nd.y == p0 && nd.z == p1;
        }
        unsigned m = __ballot_sync(FULL_MASK, hit);
        if (m) found = (int)(base + __ffs(m) - 1);
      }
    } else {
      unsigned m = __ballot_sync(FULL_MASK, lane < n_recent && r_parent == parent_event &&
                                            r_hdr == hdr_noflags && r_p0 == p0 && r_p1 == p1);
      if (m) found = (int)(recent_base + __ffs(m) - 1);
    }
    if (found >= 0) return (uint32_t)found;
    if (n_nodes >= A->node_cap) { status = DEMI_PS_NODE_OVF; return 0; }
    uint32_t id = n_nodes++;
    if (lane == 0) __stcg(&nodes_g[id], make_uint4(hdr_noflags, p0, p1, parent_event));
    if (n_recent < 32) {
      if (lane == n_recent) { r_hdr = hdr_noflags; r_p0 = p0; r_p1 = p1; r_parent = parent_event; }
      n_recent++;
    } else {
      scan_full = true;   // window exhausted: fall back to the table for the rest of this step
    }
    return id;
  }

  // EventOrchestrator.crosses_partition (EventOrchestrator.scala:345-351)
  __device__ __forceinline__ bool crosses_partition(uint32_t snd, uint32_t rcv) const {
    bool snd_actor = snd < DEMI_MAX_ACTORS;
    if (snd == rcv && !((killed >> snd) & 1u)) return false;
    uint32_t row_s = __shfl_sync(FULL_MASK, part_row, snd & 31);
    uint32_t row_r = __shfl_sync(FULL_MASK, part_row, rcv & 31);
    if (snd_actor && ((row_s >> rcv) & 1u)) return true;
    if (snd_actor && ((row_r >> snd) & 1u)) return true;
    if ((inaccessible >> rcv) & 1u) return true;
    if (snd_actor && ((inaccessible >> snd) & 1u)) return true;
    return false;
  }

  // RandomScheduler.event_produced(cell, envelope) (RandomScheduler.scala:274-321),
  // preceded by Instrumenter.aroundDispatch's cancelled-timer drop
  // (Instrumenter.scala:1090-1096).
  __device__ __forceinline__ void event_produced(uint32_t hdr, uint32_t p0, uint32_t p1) {
    if (status) return;
    uint32_t src = hdr_src(hdr), dst = hdr_dst(hdr), type = hdr_type(hdr), flags = hdr_flags(hdr);
    if (cancelled.n) {
      int ci = cancelled.find(lane, timer_key(dst, type), p0, p1);
      if (ci >= 0) { cancelled.remove_at(lane, (uint32_t)ci); return; }
    }
    // Uniq(...) :283.  Ids are 16-bit and wrap modulo 2^16 (DESIGN.md §2), as the oracle and demi_event have them;
    // unmasked, bit 16 would land in the node field of the pending entry and of the trace word.
    uint32_t uniq = ++n_uniq & 0xFFFFu;
    uint32_t hdr_nf = hdr & 0x00FFFFFFu;
    bool is_timer = false;
    uint32_t node;
    if (flags & DEMI_MF_EXTERNAL) {
      // ExternalMessage :298-307 -> reportNewlyEnabledExternal (DepTracker.scala:119-122)
      parent_event = 0;
      scan_full = true;
      node = dep_report_newly_enabled(hdr_nf, p0, p1);
      if (status) return;
      pending_insert(make_uint4(hdr, p0, p1, uniq | (node << 16)));
    } else {
      // InternalMessage :287-297
      is_timer = (src == DEMI_DEADLETTERS);
      node = dep_report_newly_enabled(hdr_nf, p0, p1);
      if (status) return;
      if (!crosses_partition(src, dst)) pending_insert(make_uint4(hdr, p0, p1, uniq | (node << 16)));
    }
    // :319-320; a reused node keeps its original parent
    // (its parent was equal to parentEvent, that is what the lookup matched on)
    record_event(DEMI_EV_MSG_SEND, is_timer ? DEMI_TIMER_SND : src, dst, type, p0, p1, uniq, node, parent_event);
  }

  __device__ __forceinline__ void tosend_push(uint32_t hdr, uint32_t p0, uint32_t p1) {
    if (n_tosend >= A->tosend_cap) { status = DEMI_PS_QUEUE_OVF; return; }
    if (lane == 0) sm->tosend[n_tosend] = make_uint4(hdr, p0, p1, 0u);
    n_tosend++;
  }
  // ExternalEventInjector.handle_timer (ExternalEventInjector.scala:282-297)
  __device__ __forceinline__ void handle_timer(uint32_t rcv, uint32_t type, uint32_t p0, uint32_t p1) {
    if (A->ignore_timers) return;
    tosend_push(make_hdr(DEMI_DEADLETTERS, rcv, type, DEMI_MF_TIMER), p0, p1);
  }
  // RandomScheduler.enqueue_timer (RandomScheduler.scala:549-559)
  __device__ __forceinline__ void enqueue_timer(uint32_t rcv, uint32_t type, uint32_t p0, uint32_t p1) {
    if (just.n && just.find(lane, timer_key(rcv, type), p0, p1) >= 0) {
      if (!resend.push(lane, timer_key(rcv, type), p0, p1)) status = DEMI_PS_QUEUE_OVF;
      return;
    }
    handle_timer(rcv, type, p0, p1);
  }
  // ExternalEventInjector.send_external_messages (ExternalEventInjector.scala:306-365)
  __device__ __forceinline__ void send_external_messages() {
    if (!n_tosend) return;
    __syncwarp();
    for (uint32_t i = 0; i < n_tosend && !status; i++) {
      uint4 q = sm->tosend[i];
      if ((dead >> hdr_dst(q.x)) & 1u) continue;     // "Dropping message to non-existent receiver" (ExternalEventInjector.scala:343-346)
      event_produced(q.x, q.y, q.z);
    }
    n_tosend = 0;
    __syncwarp();
  }

  // Cancellable.cancel(): Instrumenter.cancelTimer (Instrumenter.scala:159-168) ->
  // RandomScheduler.notify_timer_cancel (RandomScheduler.scala:525-534)
  __device__ __forceinline__ void cancel_timer(uint32_t self, uint32_t type, uint32_t p0, uint32_t p1) {
    uint32_t k = timer_key(self, type);
    if (cancelled.find(lane, k, p0, p1) < 0)
      if (!cancelled.push(lane, k, p0, p1)) { status = DEMI_PS_QUEUE_OVF; return; }
    int ri = registry.find(lane, k, p0, p1);
    if (ri >= 0) registry.remove_at(lane, (uint32_t)ri);
    __syncwarp();
    // handle_timer_cancel: first match in messagesToSend (ExternalEventInjector.scala:601-610)
    int hit = -1;
    for (uint32_t base = 0; base < n_tosend && hit < 0; base += 32) {
      uint32_t i = base + lane;
      bool h = false;
      if (i < n_tosend) {
        uint4 q = sm->tosend[i];
        h = hdr_dst(q.x) == self && hdr_type(q.x) == type && q.y == p0 && q.z == p1;
      }
      unsigned m = __ballot_sync(FULL_MASK, h);
      if (m) hit = (int)(base + __ffs(m) - 1);
    }
    if (hit >= 0) {
      // order-preserving removal (Queue.dequeueFirst)
      for (uint32_t base = (uint32_t)hit; base + 1 < n_tosend; base += 32) {
        uint32_t i = base + lane;
        uint4 q = make_uint4(0, 0, 0, 0);
        if (i + 1 < n_tosend) q = sm->tosend[i + 1];
        __syncwarp();
        if (i + 1 < n_tosend) sm->tosend[i] = q;
        __syncwarp();
      }
      n_tosend--;
      return;
    }
    // FullyRandom.remove("deadLetters", rcv, msg): first match in arr order (RandomScheduler.scala:653-664)
    hit = -1;
    for (uint32_t base = 0; base < n_pending && hit < 0; base += 32) {
      uint32_t i = base + lane;
      bool h = false;
      if (i < n_pending) {
        uint4 q = pend_load(i);
        h = hdr_src(q.x) == DEMI_DEADLETTERS && hdr_dst(q.x) == self && hdr_type(q.x) == type &&
            q.y == p0 && q.z == p1;
      }
      unsigned m = __ballot_sync(FULL_MASK, h);
      if (m) hit = (int)(base + __ffs(m) - 1);
    }
    if (hit >= 0) pending_remove_at((uint32_t)hit);
  }

  // TestOracle.Invariant over the actor states + RandomScheduler.violationMatches (:138-154)
  __device__ __forceinline__ uint32_t check_invariant() {
    __syncwarp();
    uint32_t code = MODEL::invariant_lane(sm->states, A->model_flags, lane);
    // min non-zero code over lanes
    uint32_t c = code ? code : 0xFFFFFFFFu;
    c = __reduce_min_sync(FULL_MASK, c);
    uint32_t v = (c == 0xFFFFFFFFu) ? 0u : c;
    if (!A->looking_for) return v;
    return (v && v == A->looking_for) ? A->looking_for : 0u;
  }

  // EventOrchestrator.trigger_hard_kill (EventOrchestrator.scala:243-310) in the model world (include/demi_b200.h)
  __device__ void hard_kill(uint32_t a) {
    record_event(DEMI_EV_HARD_KILL, DEMI_DEADLETTERS, a, 0, 0, 0, 0, 0, 0);
    if (fifo_mode()) { status = DEMI_PS_QUEUE_OVF; return; }
    // scheduler.actorTerminated(name) -> FullyRandom.removeAll (RandomScheduler.scala:686-696): every element of the
    // array as it was when the loop started is visited once, in position order, and a match is swap-removed at its
    // CURRENT index.  Pass 1 lists the Uniq ids of the matches in position order (in the free top of the array).
    // That needs n_pending + matches <= 2 * pending_cap entries, so plan_launch sends every program with a HardKill to
    // the HBM variants (PCAP = 16384 >= 2 * 8192); the PENDING_OVF below is never reached there.  Pass 2 removes, for
    // each listed id, the first entry carrying it; after the 16-bit wrap that can be an entry of another receiver, as
    // in the oracle (DESIGN.md §2).
    __syncwarp();
    const uint32_t n0 = n_pending, TOP = (uint32_t)PCAP;
    uint32_t r = 0;
    for (uint32_t base = 0; base < n0; base += 32) {
      const uint32_t i = base + lane;
      uint4 q = make_uint4(0, 0, 0, 0);
      const bool hit = i < n0 && hdr_dst((q = pend_load(i)).x) == a;
      const unsigned m = __ballot_sync(FULL_MASK, hit);
      if (n0 + r + __popc(m) > TOP) { status = DEMI_PS_PENDING_OVF; return; }
      __syncwarp();
      if (hit) pend_store(TOP - 1 - (r + __popc(m & ((1u << lane) - 1u))), make_uint4(q.w & 0xFFFFu, 0, 0, 0));
      r += __popc(m);
      __syncwarp();
    }
    for (uint32_t k = 0; k < r; k++) {
      const uint32_t u = pend_load(TOP - 1 - k).x;
      int at = -1;
      for (uint32_t base = 0; base < n_pending && at < 0; base += 32) {
        const uint32_t i = base + lane;
        const bool hit = i < n_pending && (pend_load(i).w & 0xFFFFu) == u;
        const unsigned m = __ballot_sync(FULL_MASK, hit);
        if (m) at = (int)(base + __ffs(m) - 1);
      }
      if (at >= 0) pending_remove_at((uint32_t)at);
    }
    blocked &= ~(1u << a);                                      // blockedActors - name :280
    for (uint32_t i = 0; i < registry.n;) {                     // removeCancellable for its timers :281-287
      uint32_t k, p0, p1; registry.get(i, k, p0, p1);
      if ((k & 0xFFu) == a) registry.remove_at(lane, i); else i++;
    }
    killed |= 1u << a; inaccessible |= 1u << a; dead |= 1u << a;
    // the stopped instance is gone: a later Start(name) is a fresh actor
    for (uint32_t w = lane; w < (uint32_t)SW; w += 32) sm->states[a * SW + w] = MODEL::init_word(a * SW + w, A->model_flags);
    __syncwarp();
  }

  // EventOrchestrator.inject_until_quiescence (EventOrchestrator.scala:132-189)
  __device__ __forceinline__ void inject_until_quiescence() {
    bool loop = true;
    while (loop && ext_idx < A->n_ext && !status) {
      uint4 raw = __ldg(reinterpret_cast<const uint4*>(A->ext) + ext_idx);
      uint32_t kind = raw.x & 0xFF, a = (raw.x >> 8) & 0xFF, b = (raw.x >> 16) & 0xFF, type = raw.x >> 24;
      switch (kind) {
        case DEMI_EXT_START:                 // trigger_start :219-231
          record_event(DEMI_EV_SPAWN, DEMI_DEADLETTERS, a, 0, 0, 0, 0, 0, 0);
          inaccessible &= ~(1u << a); killed &= ~(1u << a); dead &= ~(1u << a);
          break;
        case DEMI_EXT_HARD_KILL: hard_kill(a); break;
        case DEMI_EXT_KILL:                  // trigger_kill :233-241
          record_event(DEMI_EV_KILL, DEMI_DEADLETTERS, a, 0, 0, 0, 0, 0, 0);
          killed |= 1u << a; inaccessible |= 1u << a;
          break;
        case DEMI_EXT_SEND:                  // :160-161 -> enqueue_message
          tosend_push(make_hdr(DEMI_DEADLETTERS, a, type, DEMI_MF_EXTERNAL), raw.y, raw.z);
          break;
        case DEMI_EXT_PARTITION:             // trigger_partition :314-322
          record_event(DEMI_EV_PARTITION, a, b, 0, 0, 0, 0, 0, 0);
          if (lane == a) part_row |= 1u << b;
          break;
        case DEMI_EXT_UNPARTITION:           // trigger_unpartition :324-332 (ordered pair only)
          record_event(DEMI_EV_UNPARTITION, a, b, 0, 0, 0, 0, 0, 0);
          if (lane == a) part_row &= ~(1u << b);
          break;
        case DEMI_EXT_WAIT_QUIESCENCE:       // :182-184
          record_event(DEMI_EV_BEGIN_WAIT_QUIESCENCE, DEMI_DEADLETTERS, DEMI_DEADLETTERS, 0, 0, 0, 0, 0, 0);
          loop = false;
          break;
        default: break;
      }
      ext_idx++;
    }
  }

  // Util.find_non_blocked_message (schedulers/Util.scala:470-489) over
  // RandomizedHashSet.removeRandomElement (:171-176).  Rejected draws are
  // stashed at the top of the array and re-appended in draw order.
  // entries [top - nb, top), written downward in draw order, go back behind the live entries in draw order
  __device__ __forceinline__ void reappend_stash(uint32_t top, uint32_t nb) {
    const uint32_t lo = top - nb;
    for (uint32_t base = 0; base < nb / 2; base += 32) {          // reverse in place ...
      uint32_t i = base + lane;
      uint4 x = make_uint4(0, 0, 0, 0), y = x;
      if (i < nb / 2) { x = pend_load(lo + i); y = pend_load(top - 1 - i); }
      __syncwarp();
      if (i < nb / 2) { pend_store(lo + i, y); pend_store(top - 1 - i, x); }
      __syncwarp();
    }
    if (lo != n_pending) {                                         // ... then slide down
      for (uint32_t base = 0; base < nb; base += 32) {
        uint32_t i = base + lane;
        uint4 x = make_uint4(0, 0, 0, 0);
        if (i < nb) x = pend_load(lo + i);
        __syncwarp();
        if (i < nb) pend_store(n_pending + i, x);
        __syncwarp();
      }
    }
    n_pending += nb;
  }
  // !userDefinedFilter(snd, rcv, msg), the filter given as rules (demi_set_user_filter)
  __device__ __forceinline__ bool filter_rejects(uint32_t hdr) const {
    const uint32_t src = hdr_src(hdr), dst = hdr_dst(hdr), type = hdr_type(hdr);
    for (uint32_t i = 0; i < A->n_filter; i++) {
      const uint4 r = A->filter[i];
      const bool src_ok = src < DEMI_MAX_ACTORS ? ((r.x >> src) & 1u) : (r.w & DEMI_FRULE_DEADLETTERS);
      if (src_ok && ((r.y >> dst) & 1u) && ((r.z >> (type & 31)) & 1u)) return true;
    }
    return false;
  }
  // FullyRandom.removeRandomElement (RandomScheduler.scala:666-684), as written: redraw while the filter rejects and
  // more than one element is left; the rejected draws go back after the loop.  [.., top) is free stash space.
  __device__ __forceinline__ uint4 draw(uint32_t top) {
    uint32_t idx = rng.next_int(n_pending);
    uint4 e = pending_remove_at(idx);
    if (!A->n_filter) return e;
    uint32_t nr = 0;
    while (n_pending > 1 && filter_rejects(e.x)) {
      if (lane == 0) pend_store(top - 1 - nr, e);
      nr++;
      __syncwarp();
      idx = rng.next_int(n_pending);
      e = pending_remove_at(idx);
    }
    if (nr) reappend_stash(top, nr);
    return e;
  }
  // Util.find_non_blocked_message (schedulers/Util.scala:470-489) over the strategy's removeRandomElement.
  // Rejected draws are stashed at the top of the array and re-appended in draw order.
  __device__ __forceinline__ bool find_non_blocked(uint4& out) {
    if (n_pending == 0) return false;
    __syncwarp();
    const uint32_t blocked_mask = blocked;
    const uint32_t TOP = fifo_mode() ? HALF : (uint32_t)PCAP;      // the stash lives at the top of the array in use
    uint32_t nb = 0;
    uint4 e = draw(TOP);
    bool got = true;
    while ((blocked_mask >> (hdr_dst(e.x) & 31)) & 1u) {
      if (lane == 0) pend_store(TOP - 1 - nb, e);
      nb++;
      __syncwarp();
      if (n_pending == 0) { got = false; break; }
      e = draw(TOP - nb);
    }
    if (nb) reappend_stash(TOP, nb);
    out = e;
    return got;
  }

  // SrcDstFIFO.getNonBlockedMessage (RandomScheduler.scala:716-756) + dequeue (:758-768)
  __device__ __forceinline__ bool fifo_get_non_blocked(uint4& out) {
    const uint32_t blocked_mask = blocked;
    bool any = false;
    __syncwarp();
    for (uint32_t base = 0; base < n_pairs && !any; base += 32) {
      uint32_t i = base + lane;
      bool ok = i < n_pairs && !((blocked_mask >> (ld16(f_pairs + i) & 31u)) & 1u);
      any = __any_sync(FULL_MASK, ok);
    }
    if (!any) return find_non_blocked(out);                                     // only timers left :717-728
    if (rng_pairs.next_int(n_pending + n_queued) < n_pending)                    // :732
      if (find_non_blocked(out)) return true;
    uint32_t idx = rng_pairs.next_int(n_pairs);                                  // :750-753
    while ((blocked_mask >> (ld16(f_pairs + idx) & 31u)) & 1u) idx = rng_pairs.next_int(n_pairs);
    const uint32_t pair = ld16(f_pairs + idx);
    const uint32_t slot = ld16(f_head + pair);
    out = pend_load(HALF + slot);
    const uint32_t nxt = ld16(f_next + slot);
    __syncwarp();
    if (lane == 0) { __stcg(f_head + pair, (uint16_t)nxt); __stcg(f_next + slot, (uint16_t)fifo_free); }
    fifo_free = slot;
    if (nxt == FIFO_NIL) {                                                       // srcDsts.remove(idx): order preserving
      for (uint32_t base = idx; base + 1 < n_pairs; base += 32) {
        uint32_t i = base + lane;
        uint32_t v = 0;
        if (i + 1 < n_pairs) v = ld16(f_pairs + i + 1);
        __syncwarp();
        if (i + 1 < n_pairs) __stcg(f_pairs + i, (uint16_t)v);
        __syncwarp();
      }
      n_pairs--;
    }
    n_queued--;
    __syncwarp();
    return true;
  }

  // RandomScheduler.schedule_new_message (RandomScheduler.scala:352-485)
  __device__ __forceinline__ bool schedule_new_message(uint4& pick) {
    if (status | violation) return false;                        // :354-360
    if (nsched > A->max_messages) { ext_idx = A->n_ext; return false; }   // :369-373 finish_early
    if (A->interval > 0 && nmod == 0 && nsched != 0) {           // :376-401 (no checkpointing)
      violation = check_invariant();
      if (violation) return false;
    }
    send_external_messages();                                    // :424
    if (status) return false;
    if (fifo_mode()) { if (!fifo_get_non_blocked(pick)) return false; }   // :446-449
    else if (!find_non_blocked(pick)) return false;              // :451-457
    nsched++;                                                    // :462
    if (nsched == 0x7FFFFFFF) nsched = 1;
    if (++nmod == A->interval) nmod = 0;
    uint32_t src = hdr_src(pick.x), dst = hdr_dst(pick.x), type = hdr_type(pick.x);
    uint32_t uniq = pick.w & 0xFFFF, node = pick.w >> 16;
    record_event(DEMI_EV_MSG_EVENT, src, dst, type, pick.y, pick.z, uniq, node, 0);   // :467
    // depTracker.reportNewlyDelivered :468 (DepTracker.scala:132-135)
    parent_event = node;
    recent_base = n_nodes; n_recent = 0;
    {
      uint32_t w = __shfl_sync(FULL_MASK, delivered_bits, (node >> 5) & 31);
      scan_full = (node >= 1024u) || ((w >> (node & 31)) & 1u);
      if (node < 1024u && lane == (node >> 5)) delivered_bits |= 1u << (node & 31);
    }
    // updateRepeatingTimer :405-421
    uint32_t k = timer_key(dst, type);
    if (registry.n && registry.find(lane, k, pick.y, pick.z) >= 0) {
      if (just.find(lane, k, pick.y, pick.z) < 0)
        if (!just.push(lane, k, pick.y, pick.z)) status = DEMI_PS_QUEUE_OVF;
    } else {
      for (uint32_t i = 0; i < resend.n; i++) {
        uint32_t rk, ra, rb;
        resend.get(i, rk, ra, rb);
        handle_timer(rk & 0xFF, rk >> 8, ra, rb);
      }
      resend.clear();
      just.clear();
    }
    return !status;
  }

  __device__ __noinline__ void receive_scalar(Outbox& ob, uint32_t self, uint32_t src, uint32_t type,
                                              uint32_t p0, uint32_t p1) {
    ContigState st{&sm->states[self * SW]};
    MODEL::receive(ob, self, st, src, type, p0, p1, A->model_flags);
  }

  // Instrumenter.dispatch_new_message (Instrumenter.scala:913-1017)
  __device__ __forceinline__ void dispatch_new_message(const uint4& pick) {
    uint32_t src = hdr_src(pick.x), dst = hdr_dst(pick.x), type = hdr_type(pick.x);
    // repeating timer re-armed right after the hand-off (:1008-1016)
    if (registry.n && registry.find(lane, timer_key(dst, type), pick.y, pick.z) >= 0)
      enqueue_timer(dst, type, pick.y, pick.z);
    if (status) return;
    // the actor's receive(): lane 0, scalar
    uint32_t n_ops = 0;
    __syncwarp();
    if (lane == 0) {
      Outbox ob; ob.ops = sm->outbox; ob.n = 0; ob.self = dst; ob.overflow = false;
      receive_scalar(ob, dst, src, type, pick.y, pick.z);
      n_ops = ob.overflow ? 0xFFFFFFFFu : ob.n;
    }
    n_ops = __shfl_sync(FULL_MASK, n_ops, 0);
    __syncwarp();
    if (n_ops == 0xFFFFFFFFu) { status = DEMI_PS_QUEUE_OVF; return; }
    for (uint32_t i = 0; i < n_ops && !status; i++) {
      uint4 op = sm->outbox[i];
      uint32_t kind = op.x & 0xFF, odst = (op.x >> 8) & 0xFF, otype = (op.x >> 16) & 0xFF;
      if (kind == OP_SEND) {
        // `!` -> Instrumenter.tell -> aroundDispatch -> event_produced (Instrumenter.scala:1098-1108)
        event_produced(make_hdr(dst, odst, otype, 0), op.y, op.z);
      } else if (kind == OP_CANCEL) {
        cancel_timer(odst, otype, op.y, op.z);
      } else {
        // registerCancellable -> handleTick -> enqueue_timer (Instrumenter.scala:1145-1200)
        uint32_t k = timer_key(odst, otype);
        if (registry.n && registry.find(lane, k, op.y, op.z) >= 0) continue;   // "Non-unique timer" :1154-1157
        if (kind == OP_SCHED_REPEAT)
          if (!registry.push(lane, k, op.y, op.z)) { status = DEMI_PS_QUEUE_OVF; break; }
        enqueue_timer(odst, otype, op.y, op.z);
      }
    }
  }

  __device__ __forceinline__ void reset(int64_t seed) {
    rng.seed(seed);
    for (uint32_t i = lane; i < N * SW; i += 32) sm->states[i] = MODEL::init_word(i, A->model_flags);
    n_pending = max_pending = n_tosend = 0;
    n_nodes = 1; parent_event = 0; recent_base = 1; n_recent = 0; scan_full = true;
    n_events = n_uniq = 0; nsched = 0; nmod = 0; ext_idx = 0;
    violation = status = 0;
    // populateActorSystem: every actor starts isolated (ExternalEventInjector.scala:371-378)
    inaccessible = (N >= 32) ? 0xFFFFFFFFu : ((1u << N) - 1u);
    killed = 0; thash = 0; dead = 0; blocked = A->blocked_mask;
    just.clear(); resend.clear(); registry.clear(); cancelled.clear();
    part_row = 0; delivered_bits = 0;
    r_hdr = r_p0 = r_p1 = r_parent = 0;
    n_pairs = n_queued = fifo_free = 0;
    if (fifo_mode()) {
      rng_pairs.seed(seed);                                       // SrcDstFIFO.rand (:705), see demi_b200.h
      for (uint32_t i = lane; i < FIFO_PAIRS; i += 32) { __stcg(f_head + i, (uint16_t)FIFO_NIL); __stcg(f_tail + i, (uint16_t)FIFO_NIL); }
      for (uint32_t i = lane; i < HALF; i += 32) __stcg(f_next + i, (uint16_t)(i + 1 < HALF ? i + 1 : FIFO_NIL));
    }
    if (lane == 0) __stcg(&nodes_g[0], make_uint4(0, 0, 0, 0));   // DepTracker.root (DepTracker.scala:15-17)
    __syncwarp();
  }

  // One RandomScheduler.explore execution (RandomScheduler.scala:234-272):
  // execute_trace -> advanceTrace (ExternalEventInjector.scala:382-441), the
  // Instrumenter loop (Instrumenter.scala:1113-1140, :794-815), notify_quiescence
  // (RandomScheduler.scala:487-500), handle_quiescence (ExternalEventInjector.scala:541-580).
  __device__ __forceinline__ void run(int64_t seed, demi_fuzz_result& out) {
    reset(seed);
    for (;;) {
      inject_until_quiescence();
      uint4 pick;
      while (schedule_new_message(pick)) {
        dispatch_new_message(pick);
        if (status) break;
      }
      if (status | violation) break;
      if (ext_idx < A->n_ext) {
        record_event(DEMI_EV_QUIESCENCE, DEMI_DEADLETTERS, DEMI_DEADLETTERS, 0, 0, 0, 0, 0, 0);
        continue;
      }
      break;
    }
    // explore(): checkIfBugFound only if messagesScheduledSoFar <= maxMessages (:255-262, :156-180)
    if (!status && nsched <= A->max_messages && !violation) violation = check_invariant();

    if (status) {
      out.violation = 0; out.steps = 0; out.state_hash = 0; out.trace_hash = 0;
      out.n_nodes = 0; out.n_events = 0; out.max_pending = 0; out.status = (uint16_t)status;
    } else {
      __syncwarp();
      uint64_t sh = 0;
      for (uint32_t i = lane; i < N * SW; i += 32) sh += demi_state_term(sm->states[i], i);
      if (A->fuzz_flags & DEMI_FF_HASH_PENDING)
        for (uint32_t i = lane; i < n_pending; i += 32) {
          uint4 q = pend_load(i);
          sh += demi_pending_term(q.x & 0x00FFFFFFu, q.y, q.z);
        }
      if ((A->fuzz_flags & DEMI_FF_HASH_PENDING) && fifo_mode())
        for (uint32_t pi = 0; pi < n_pairs; pi++)
          for (uint32_t sl = ld16(f_head + ld16(f_pairs + pi)); sl != FIFO_NIL; sl = ld16(f_next + sl)) {
            uint4 q = pend_load(HALF + sl);
            if (lane == 0) sh += demi_pending_term(q.x & 0x00FFFFFFu, q.y, q.z);
          }
      for (int o = 16; o > 0; o >>= 1) sh += __shfl_xor_sync(FULL_MASK, sh, o);
      out.violation = violation; out.steps = (uint32_t)nsched;
      out.state_hash = sh; out.trace_hash = thash;
      out.n_nodes = (uint16_t)n_nodes;
      out.n_events = (uint16_t)(n_events > 65535u ? 65535u : n_events);
      out.max_pending = (uint16_t)max_pending; out.status = 0;
    }
  }
};

}  // namespace demi
