// The host side of the lane engine's steady instantiation (demi_b200/csrc/lane_steady.hpp): which launches may start
// from a program's pre-delivery snapshot.  No device is needed: the rule is plain C++ over the snapshot's scalars.
#include <climits>
#include <cstdio>
#include "lane_steady.hpp"
#include "demi_limits.h"

using namespace demi;

static int failures = 0;
#define EXPECT(cond) do { if (!(cond)) { printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); failures++; } } while (0)

// the snapshot of raft5_program(): five Starts, five BOOTs, WaitQuiescence
static LaneSnapshot bench_snapshot() {
  LaneSnapshot s{};
  s.n_pending = 5; s.n_nodes = 6; s.n_events = 11; s.ext_idx = 11; s.ext_send_idx = 5;
  return s;
}
// the benchmark's batch: raft5, maxMessages 50
static LaneSteadyLaunch bench_launch(int32_t max_messages = 50) {
  LaneSteadyLaunch l{};
  l.n_ext = 11; l.max_messages = max_messages;
  const uint32_t pcap = demi_pending_cap(2, max_messages, 5);
  l.pending_cap = pcap < 96 ? pcap : 96; l.node_cap = demi_node_cap(pcap); l.tosend_cap = demi_tosend_cap(5);
  l.lane_tosend_cap = 16; l.ops_per_delivery = 6;
  return l;
}

int main() {
  EXPECT(sizeof(LaneSnapshot) == LANE_SNAP_CAP * 16 + 80);
  EXPECT(lane_steady_eligible(bench_snapshot(), bench_launch()));
  EXPECT(bench_launch().node_cap == 576);
  EXPECT(lane_steady_node_bound(6, 51, 6) == 363);

  // each condition alone
  { LaneSnapshot s = bench_snapshot(); s.status = 0xFFFF; EXPECT(!lane_steady_eligible(s, bench_launch())); }
  { LaneSnapshot s = bench_snapshot(); s.ext_idx = 10; EXPECT(!lane_steady_eligible(s, bench_launch())); }      // a second segment
  { LaneSnapshot s = bench_snapshot(); s.killed = 8; EXPECT(!lane_steady_eligible(s, bench_launch())); }
  { LaneSnapshot s = bench_snapshot(); s.inaccessible = 16; EXPECT(!lane_steady_eligible(s, bench_launch())); }
  { LaneSnapshot s = bench_snapshot(); s.tosend_n = 1; EXPECT(!lane_steady_eligible(s, bench_launch())); }
  { LaneSnapshot s = bench_snapshot(); s.root_timers = 1; EXPECT(!lane_steady_eligible(s, bench_launch())); }
  { LaneSnapshot s = bench_snapshot(); s.registry = 1; EXPECT(!lane_steady_eligible(s, bench_launch())); }
  { LaneSnapshot s = bench_snapshot(); s.cancelled = 1; EXPECT(!lane_steady_eligible(s, bench_launch())); }
  { LaneSteadyLaunch l = bench_launch(); l.partitions = true; EXPECT(!lane_steady_eligible(bench_snapshot(), l)); }
  { LaneSteadyLaunch l = bench_launch(); l.ignore_timers = true; EXPECT(!lane_steady_eligible(bench_snapshot(), l)); }
  { LaneSteadyLaunch l = bench_launch(); l.looking_for = 1; EXPECT(!lane_steady_eligible(bench_snapshot(), l)); }
  { LaneSteadyLaunch l = bench_launch(); l.tosend_cap = 15; EXPECT(!lane_steady_eligible(bench_snapshot(), l)); }

  // the pending capacity: the snapshot must fit the launch's bound and the struct's rows
  { LaneSteadyLaunch l = bench_launch(); l.pending_cap = 5; EXPECT(lane_steady_eligible(bench_snapshot(), l));
    l.pending_cap = 4; EXPECT(!lane_steady_eligible(bench_snapshot(), l)); }
  { LaneSnapshot s = bench_snapshot(); s.n_pending = LANE_SNAP_CAP; s.n_nodes = 17; EXPECT(lane_steady_eligible(s, bench_launch()));
    s.n_pending = LANE_SNAP_CAP + 1; EXPECT(!lane_steady_eligible(s, bench_launch())); }

  // the node capacity at its exact edge (demi_node_cap's largest value, 16448), and no overflow at unbounded depth
  EXPECT(bench_launch(2347).node_cap == 16448 && bench_launch(2348).node_cap == 16448);
  EXPECT(lane_steady_eligible(bench_snapshot(), bench_launch(2347)));
  EXPECT(!lane_steady_eligible(bench_snapshot(), bench_launch(2348)));
  { LaneSteadyLaunch l = bench_launch(); l.node_cap = 363; EXPECT(lane_steady_eligible(bench_snapshot(), l));
    l.node_cap = 362; EXPECT(!lane_steady_eligible(bench_snapshot(), l)); }
  { LaneSteadyLaunch l = bench_launch(); l.max_messages = INT_MAX; l.node_cap = 65535; EXPECT(!lane_steady_eligible(bench_snapshot(), l));
    l.ops_per_delivery = 0xFFFFFFFFu; EXPECT(!lane_steady_eligible(bench_snapshot(), l)); }
  { LaneSteadyLaunch l = bench_launch(); l.max_messages = 0; EXPECT(lane_steady_eligible(bench_snapshot(), l)); }

  if (failures) return 1;
  printf("OK\n");
  return 0;
}
