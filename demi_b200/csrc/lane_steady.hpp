// lane_steady.hpp — the lane engine's pre-delivery snapshot and the rule that decides whether a launch may start
// from it.  Plain C++ (no CUDA types), so that the rule can be unit-tested on the host.
//
// java.util.Random is first consulted when RandomScheduler picks the first message, so everything an execution does
// before that pick (the externals up to the first WaitQuiescence and the flush of their Sends) is the same for every
// seed of a program.  lane_snapshot_kernel (lane_kernel.cuh) runs that part once, on the generic LaneMachine, and
// stores the machine here; the STEADY instantiation of the lane kernel starts every execution from the copy.
//
// It goes further: java.util.Random only picks an index into the pending array, and the machine is deterministic
// given those indices, so the machine after the first d picks depends on those d indices alone.  The tree of every
// such machine up to a depth d (lane_tree_extend decides d) is built once per program and launch key, and a steady
// execution draws its first d indices exactly as pick_next would, walks the tree, and starts at the node it reaches.
#pragma once
#include <stdint.h>

namespace demi {

constexpr uint32_t LANE_SNAP_CAP = 16;        // pending entries a snapshot holds; a program that enables more is not snapshotted

struct alignas(16) LaneSnapshot {
  uint32_t pend[LANE_SNAP_CAP][4];            // the pending array (16-byte entries) at the first pick
  uint64_t thash;
  uint32_t n_pending, n_nodes, n_events, parent_event;
  uint32_t root_timers, registry, cancelled, tosend_n;
  uint32_t ext_idx, ext_send_idx, inaccessible, killed;
  uint32_t status;                            // 0, or LANE_DEFER: the lane engine cannot run the program's first segment
  uint32_t depth;                             // levels of the tree below its root (the host sets both when it builds it)
  uint64_t tree;                              // device address of the tree's node records, the root first
};
static_assert(sizeof(LaneSnapshot) % 16 == 0, "the snapshot is copied as 16-byte words");

// What a batch launch contributes to the decision.  pending_cap is the bound the lane kernel will test (the launch's
// pending capacity, the test limit DEMI_LANE_PENDING_CAP and the kernel's physical rows, whichever is least).
struct LaneSteadyLaunch {
  uint32_t n_ext;                 // events of the program
  bool partitions;                // it has a Partition or UnPartition
  bool ignore_timers;
  uint32_t looking_for;
  int32_t max_messages;           // mapped: a negative maxMessages is INT_MAX
  uint32_t pending_cap, node_cap, tosend_cap;
  uint32_t lane_tosend_cap;       // LANE_TOSEND_CAP
  uint32_t ops_per_delivery;      // MODEL::LANE_OUTBOX: the most operations (sends, schedules, cancels) one receive() issues
};

// DepTracker nodes an execution can have created after `deliveries` deliveries from a snapshot with n_nodes: every
// send of receive() takes one, and so does every timer message flushed from messagesToSend.  In the steady state an
// entry reaches messagesToSend (directly or through timersToResend) only from a schedule operation of receive() or
// from the one re-arm of a repeating timer in pick_next, so a delivery accounts for at most ops_per_delivery + 1
// nodes however the timers bunch up in single flushes.
inline uint64_t lane_steady_node_bound(uint32_t n_nodes, uint64_t deliveries, uint32_t ops_per_delivery) {
  return (uint64_t)n_nodes + deliveries * ((uint64_t)ops_per_delivery + 1u);
}

// True when every execution of the launch may start from `s` and run the STEADY instantiation, which has no code for
// externals, partitions, isolated actors, ignoreTimers, a violation filter or the node capacity:
//  - the first segment ran in the lane engine (status 0) and fits the launch's pending capacity;
//  - it was the only segment: no external is left, so nothing is injected (no Kill, Partition, Send) ever again;
//  - every actor is started and none is isolated, and the program has no partition, so no send is ever dropped;
//  - no timer state exists yet (nothing was delivered), messagesToSend is empty;
//  - the node capacity cannot be reached within max_messages + 1 deliveries (may_continue stops an execution when
//    nsched > max_messages, so that many happen), and the launch's messagesToSend capacity is not below the queue's.
// A node of the tree is the whole steady LaneMachine at the point where pick_next draws: after may_continue() and the
// flush, the point the snapshot captures at depth 0.  A record is LANE_NODE_HEAD header words (LaneNodeWord), the
// actor state words and the cancellable-timer copies (padded to 16 bytes), then LANE_NODE_ROWS pending rows.  The
// children of a node are contiguous: child i (the machine after picking pending index i) is record `child + i`.
enum LaneNodeWord : uint32_t {
  LN_CHILD, LN_N_PENDING, LN_NSCHED, LN_VIOLATION,     // the first 16 bytes: all a walk reads
  LN_NMOD, LN_MAX_PENDING, LN_N_NODES, LN_N_EVENTS, LN_PARENT_EVENT,
  LN_REGISTRY, LN_CANCELLED, LN_JUST, LN_WINDOW_TIMERS, LN_N_RESEND, LN_RESEND_LO, LN_RESEND_HI, LN_THASH_LO, LN_THASH_HI,
  LANE_NODE_HEAD = 20
};
constexpr uint32_t LANE_NODE_LEAF = 0xFFFFFFFFu;     // LN_CHILD of a node without children
constexpr uint32_t LANE_NODE_ABSENT = 0xFFFFFFFFu;   // LN_N_PENDING of a child that is not stored: its execution deferred
                                                     // or would have exceeded the rows; the walk stops at its parent
constexpr uint32_t LANE_NODE_ROWS = 32;
static_assert(LANE_SNAP_CAP <= LANE_NODE_ROWS, "the root holds the snapshot's rows");
constexpr uint32_t LANE_TREE_MAX_DEPTH = 8;
#ifndef DEMI_K1_TREE_BUDGET
#define DEMI_K1_TREE_BUDGET (4u << 20)
#endif
constexpr uint64_t LANE_TREE_BUDGET = DEMI_K1_TREE_BUDGET;   // bytes of node records (DESIGN §10.1: why this many)

// words of one record of a machine with `machine_words` state and timer-copy words
constexpr uint32_t lane_node_words(uint32_t machine_words) {
  return LANE_NODE_HEAD + ((machine_words + 3u) & ~3u) + LANE_NODE_ROWS * 4u;
}
// Whether the tree, `depth` levels below its root and `nodes` records in all, gets the next level of `children`
// records: the deepest tree, at most LANE_TREE_MAX_DEPTH levels, whose records fit LANE_TREE_BUDGET.
inline bool lane_tree_extend(uint32_t depth, uint64_t nodes, uint64_t children, uint32_t node_bytes) {
  return depth < LANE_TREE_MAX_DEPTH && children > 0 && (nodes + children) * node_bytes <= LANE_TREE_BUDGET;
}
// A stored node (not LANE_NODE_ABSENT) gets children when its execution goes on to a pick: no violation found, no more
// than max_messages delivered (may_continue), and a message pending.  A deferred execution is never stored.
inline bool lane_node_expands(uint32_t n_pending, int32_t nsched, uint32_t violation, int32_t max_messages) {
  return n_pending != LANE_NODE_ABSENT && n_pending > 0 && violation == 0 && nsched <= max_messages;
}
// What a tree depends on besides the program: every input of its first deliveries.  maxMessages is compared with
// nsched <= LANE_TREE_MAX_DEPTH only, so every larger value builds the same tree.
struct LaneTreeKey {
  uint32_t model_flags; int32_t interval, max_messages; uint32_t pending_cap;
  bool operator==(const LaneTreeKey& o) const {
    return model_flags == o.model_flags && interval == o.interval && max_messages == o.max_messages && pending_cap == o.pending_cap;
  }
};
inline LaneTreeKey lane_tree_key(uint32_t model_flags, int32_t interval, int32_t max_messages, uint32_t pending_cap) {
  const int32_t m = max_messages > (int32_t)LANE_TREE_MAX_DEPTH ? (int32_t)LANE_TREE_MAX_DEPTH + 1 : max_messages;
  return LaneTreeKey{model_flags, interval, m, pending_cap};
}

inline bool lane_steady_eligible(const LaneSnapshot& s, const LaneSteadyLaunch& l) {
  if (s.status != 0 || s.ext_idx != l.n_ext || l.partitions) return false;
  if ((s.inaccessible | s.killed) != 0) return false;
  if ((s.root_timers | s.registry | s.cancelled | s.tosend_n | s.parent_event) != 0) return false;
  if (l.ignore_timers || l.looking_for != 0) return false;
  if (s.n_pending > l.pending_cap || s.n_pending > LANE_SNAP_CAP) return false;
  if (l.tosend_cap < l.lane_tosend_cap) return false;
  if (l.max_messages < 0) return false;
  return lane_steady_node_bound(s.n_nodes, (uint64_t)l.max_messages + 1u, l.ops_per_delivery) <= l.node_cap;
}

// ---------------------------------------------------------------------------------------------- 8-byte raft5 rows
// The steady raft5 lane kernel's ROW8 flavour keeps each pending row (header, p0, p1, DepTracker node) in 64 bits
// instead of 128, which halves the rows' L2 footprint.  raft5's payloads leave fixed bits of p0 and p1 zero, and the
// header and the node go into those bits, so a row is packed with a few ORs and unpacked with two ANDs and a few bit
// extracts, and no row is range-tested on the device: lane_row8_eligible proves on the host, once per launch, that
// every row a steady execution can create has its payload zero there.  The two 32-bit words:
//   lo = p0 (bits 12..15 and 28..31 zero)  | type << 12 | (node >> 8) << 28
//   hi = p1 (bits 1..7 and 24..31 zero)    | src code << 1 | dst << 4 | (node & 0xFF) << 24
// so p0's byte 1 and byte 3 and p1's byte 0 hold 4, 4 and 1 bits, p1's byte 3 none, and the node 12 bits.  The src code
// is the actor (0..4), or 5 + flags for a message from deadLetters (flags 0, EXTERNAL or TIMER): an actor's sends
// carry no flags.  Word 3 of a row is node | node << 16 (Uniq equals node in the lane engine), so one field holds both.
//
// Why raft5's payloads fit (Raft5::receive, models.cuh), given that the snapshot's rows do (checked below): every p0
// byte 0, byte 2 and p1 byte 1 and 2 is a term, a log term, a log value or a log index, each one state byte.  p0 byte 1
// is RequestVote's lastIndex (LOGLEN <= LOG_CAP), a grant or ok bit, or AppendEntries' prev, which is NEXT[j]: NEXT
// is only set to LOGLEN, lowered by one, or raised to the matchIndex of an AppendReply from an actor (DESIGN §3 raft5
// R2: never from deadLetters, so never from an external Send), which is at most LOG_CAP.  p0 byte 3 is AppendEntries'
// commit index, at most LOG_CAP (COMMIT is the minimum of a leaderCommit and a matchIndex <= LOG_CAP, or the highest of
// at most LOG_CAP log entries).  p1 byte 0 is AppendEntries' has-entry bit.  Every other byte a receive() sends is zero,
// and timers have p0 = p1 = 0.
#if defined(__CUDACC__)
#define LANE_ROW8_HD __host__ __device__ __forceinline__
#else
#define LANE_ROW8_HD inline
#endif
constexpr uint32_t LANE_ROW8_ACTORS = 5;            // Raft5::N_ACTORS
constexpr uint32_t LANE_ROW8_NODE_BITS = 12;
constexpr uint32_t LANE_ROW8_P0 = 0x0FFF0FFFu, LANE_ROW8_P1 = 0x00FFFF01u;     // the payload bits of lo and hi

// lo | hi << 32; the caller knows that p0 and p1 have no bit outside LANE_ROW8_P0 / LANE_ROW8_P1 and node < 2^12
LANE_ROW8_HD uint64_t lane_row8_pack(uint32_t hdr, uint32_t p0, uint32_t p1, uint32_t node) {
  const uint32_t src = hdr & 0xFFu, code = src < LANE_ROW8_ACTORS ? src : 5u + (hdr >> 24);
  const uint32_t lo = p0 | ((hdr >> 16) & 0xFu) << 12 | (node >> 8) << 28;
  const uint32_t hi = p1 | (code & 7u) << 1 | ((hdr >> 8) & 7u) << 4 | node << 24;
  return (uint64_t)lo | (uint64_t)hi << 32;
}
// src, dst and type of a packed row, as make_hdr places them, without the flags: all the steady machine reads of a
// header, except whether the row is a timer message of a given type, which lane_row8_timer_of reads from the row
LANE_ROW8_HD uint32_t lane_row8_sdt(uint64_t r) {
  const uint32_t lo = (uint32_t)r, hi = (uint32_t)(r >> 32), code = (hi >> 1) & 7u;
  return (code < LANE_ROW8_ACTORS ? code : 0xFFu) | ((hi >> 4) & 7u) << 8 | ((lo >> 12) & 0xFu) << 16;
}
LANE_ROW8_HD uint32_t lane_row8_dst(uint64_t r) { return (uint32_t)(r >> 36) & 7u; }
// a timer message (from deadLetters, flagged TIMER: src code 7) of `type`
LANE_ROW8_HD bool lane_row8_timer_of(uint64_t r, uint32_t type) {
  return (((uint32_t)(r >> 32) & 0xEu) | ((uint32_t)r & 0xF000u)) == (0xEu | type << 12);
}
// the whole header (src, dst, type and flags as make_hdr builds them)
LANE_ROW8_HD uint32_t lane_row8_hdr(uint64_t r) {
  const uint32_t code = (uint32_t)(r >> 33) & 7u;
  return lane_row8_sdt(r) | (code < LANE_ROW8_ACTORS ? 0u : (code - 5u) << 24);
}
LANE_ROW8_HD uint32_t lane_row8_p0(uint64_t r) { return (uint32_t)r & LANE_ROW8_P0; }
LANE_ROW8_HD uint32_t lane_row8_p1(uint64_t r) { return (uint32_t)(r >> 32) & LANE_ROW8_P1; }
LANE_ROW8_HD uint32_t lane_row8_node(uint64_t r) { return (uint32_t)(r >> 56) | ((uint32_t)r >> 28) << 8; }

// Whether the layout holds a row exactly.
LANE_ROW8_HD bool lane_row8_fits(uint32_t hdr, uint32_t p0, uint32_t p1) {
  if ((p0 & ~LANE_ROW8_P0) | (p1 & ~LANE_ROW8_P1)) return false;
  const uint64_t r = lane_row8_pack(hdr, p0, p1, 0);
  return lane_row8_hdr(r) == hdr;
}

// True when a steady raft5 launch (lane_steady_eligible holds) may run the ROW8 flavour: every row of the snapshot
// fits the layout, and every DepTracker node the execution can create is below 2^12 (lane_steady_node_bound over
// max_messages + 1 deliveries, as in lane_steady_eligible).  The snapshot's rows are the only ones not made by
// Raft5::receive or a timer: they hold the program's external Sends, whose payloads are whatever the program gave them.
inline bool lane_row8_eligible(const LaneSnapshot& s, int32_t max_messages, uint32_t ops_per_delivery) {
  if (max_messages < 0 || s.n_pending > LANE_SNAP_CAP) return false;
  for (uint32_t i = 0; i < s.n_pending; i++)
    if (!lane_row8_fits(s.pend[i][0], s.pend[i][1], s.pend[i][2])) return false;
  return lane_steady_node_bound(s.n_nodes, (uint64_t)max_messages + 1u, ops_per_delivery) <= (1ull << LANE_ROW8_NODE_BITS);
}

}  // namespace demi
