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

}  // namespace demi
