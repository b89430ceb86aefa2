// lane_steady.hpp — the lane engine's pre-delivery snapshot and the rule that decides whether a launch may start
// from it.  Plain C++ (no CUDA types), so that the rule can be unit-tested on the host.
//
// java.util.Random is first consulted when RandomScheduler picks the first message, so everything an execution does
// before that pick (the externals up to the first WaitQuiescence and the flush of their Sends) is the same for every
// seed of a program.  lane_snapshot_kernel (lane_kernel.cuh) runs that part once, on the generic LaneMachine, and
// stores the machine here; the STEADY instantiation of the lane kernel starts every execution from the copy.
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
  uint32_t reserved[3];
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
