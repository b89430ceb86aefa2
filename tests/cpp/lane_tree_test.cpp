// The host side of the steady lane kernel's tree (demi_b200/csrc/lane_steady.hpp): the record layout, the depth rule,
// which nodes get children and the key.  No device is needed: all of it is plain C++.
#include <cstdio>
#include "lane_steady.hpp"

using namespace demi;

static int failures = 0;
#define EXPECT(cond) do { if (!(cond)) { printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); failures++; } } while (0)

int main() {
  // records are whole 16-byte words, rows last; the walk reads the first 16 bytes
  EXPECT(lane_node_words(53) == 20 + 56 + 128);           // raft5: 50 state words, 3 timer copies
  EXPECT(lane_node_words(6) == 20 + 8 + 128);             // pingpong3
  EXPECT(lane_node_words(64) % 4 == 0 && lane_node_words(1) % 4 == 0);
  EXPECT(LN_VIOLATION < 4 && LN_CHILD < 4 && LN_N_PENDING < 4 && LN_NSCHED < 4 && LN_THASH_HI < LANE_NODE_HEAD);
  EXPECT(sizeof(LaneSnapshot) == LANE_SNAP_CAP * 16 + 80);

  // the depth rule: the next level is built while the whole tree fits the budget, up to the depth cap
  const uint32_t nb = lane_node_words(53) * 4;
  const uint64_t fit = LANE_TREE_BUDGET / nb;
  EXPECT(lane_tree_extend(0, 1, 5, nb));
  EXPECT(lane_tree_extend(3, fit - 10, 10, nb));
  EXPECT(!lane_tree_extend(3, fit - 10, 11, nb));
  EXPECT(!lane_tree_extend(0, 1, 0, nb));                  // no child to build
  EXPECT(!lane_tree_extend(LANE_TREE_MAX_DEPTH, 1, 1, nb));
  EXPECT(lane_tree_extend(LANE_TREE_MAX_DEPTH - 1, 1, 1, nb));
  // the benchmark's tree (raft5, 1 + 5 + 25 + 140 + 960 records to depth 4) fits
  EXPECT(lane_tree_extend(3, 1 + 5 + 25 + 140, 960, nb));

  // which stored nodes get children
  EXPECT(lane_node_expands(5, 0, 0, 50));
  EXPECT(!lane_node_expands(0, 3, 0, 50));                 // nothing pending
  EXPECT(!lane_node_expands(LANE_NODE_ABSENT, 3, 0, 50));  // not stored
  EXPECT(!lane_node_expands(5, 3, 1, 50));                 // a violation ended the execution
  EXPECT(lane_node_expands(5, 3, 0, 3) && !lane_node_expands(5, 4, 0, 3));   // may_continue: nsched > maxMessages

  // the key: maxMessages beyond the depth cap builds the same tree, and everything else tells trees apart
  EXPECT(lane_tree_key(1, 5, 50, 96) == lane_tree_key(1, 5, 0x7FFFFFFF, 96));
  EXPECT(lane_tree_key(1, 5, LANE_TREE_MAX_DEPTH + 1, 96) == lane_tree_key(1, 5, 50, 96));
  EXPECT(!(lane_tree_key(1, 5, LANE_TREE_MAX_DEPTH, 96) == lane_tree_key(1, 5, 50, 96)));
  EXPECT(!(lane_tree_key(1, 5, 3, 96) == lane_tree_key(1, 5, 4, 96)));
  EXPECT(!(lane_tree_key(0, 5, 50, 96) == lane_tree_key(1, 5, 50, 96)));
  EXPECT(!(lane_tree_key(1, 1, 50, 96) == lane_tree_key(1, 5, 50, 96)));
  EXPECT(!(lane_tree_key(1, 5, 50, 24) == lane_tree_key(1, 5, 50, 96)));

  if (failures) { printf("%d FAILED\n", failures); return 1; }
  printf("OK\n");
  return 0;
}
