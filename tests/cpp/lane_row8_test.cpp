// The 8-byte pending rows of the steady raft5 lane kernel (demi_b200/csrc/lane_steady.hpp): the layout holds every row
// raft5's receive() and its timers can create, and the per-launch rule admits a launch exactly when the snapshot's rows
// fit and every DepTracker node stays below 2^12.  No device is needed: the layout and the rule are plain C++.
#include <cstdio>
#include <initializer_list>
#include "lane_steady.hpp"

using namespace demi;

static int failures = 0;
#define EXPECT(cond) do { if (!(cond)) { printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); failures++; } } while (0)

enum { BOOT = 1, CLIENT_CMD = 2, ELECTION_TICK = 3, REQUEST_VOTE = 4, VOTE_REPLY = 5, HEARTBEAT_TICK = 6,
       APPEND_ENTRIES = 7, APPEND_REPLY = 8 };                 // Raft5's message types (models.cuh)
static uint32_t hdr(uint32_t src, uint32_t dst, uint32_t type, uint32_t flags) {
  return src | dst << 8 | type << 16 | flags << 24;
}
static bool round_trip(uint32_t h, uint32_t p0, uint32_t p1, uint32_t node) {
  const uint64_t r = lane_row8_pack(h, p0, p1, node);
  return lane_row8_hdr(r) == h && lane_row8_p0(r) == p0 && lane_row8_p1(r) == p1 && lane_row8_node(r) == node;
}

// the snapshot of raft5_program(client_cmds): five BOOTs (membership 0x1F), then the client commands 1 + i to i % 5
static LaneSnapshot snapshot(uint32_t client_cmds = 0) {
  LaneSnapshot s{};
  s.n_pending = 5 + client_cmds; s.n_nodes = 6 + client_cmds;
  for (uint32_t i = 0; i < s.n_pending; i++) {
    const bool boot = i < 5;
    s.pend[i][0] = hdr(0xFF, boot ? i : (i - 5) % 5, boot ? BOOT : CLIENT_CMD, 1);
    s.pend[i][1] = boot ? 0x1F : 1 + (i - 5);
    s.pend[i][3] = (i + 1) * 0x10001u;
  }
  return s;
}

int main() {
  // every row raft5 creates: a term, log term or log value is one byte; indices are at most LOG_CAP = 8, and
  // AppendEntries' prev (NEXT) at most 15; flags are none for an actor's sends
  uint32_t checked = 0;
  for (uint32_t src = 0; src < 5; src++)
    for (uint32_t dst = 0; dst < 5; dst++)
      for (uint32_t t = 0; t < 256; t += 17) {
        for (uint32_t b = 0; b < 256; b += 15) {
          for (uint32_t i = 0; i <= 8; i++) {
            EXPECT(round_trip(hdr(src, dst, REQUEST_VOTE, 0), t | i << 8 | b << 16, 0, 363));
            EXPECT(round_trip(hdr(src, dst, APPEND_REPLY, 0), t | 1u << 8 | i << 16, 0, 4095));
            checked += 2;
          }
          for (uint32_t prev = 0; prev < 16; prev++)
            for (uint32_t commit = 0; commit <= 8; commit++) {
              EXPECT(round_trip(hdr(src, dst, APPEND_ENTRIES, 0), t | prev << 8 | b << 16 | commit << 24,
                                1u | (255u - b) << 8 | b << 16, prev * 250u + commit));
              EXPECT(round_trip(hdr(src, dst, APPEND_ENTRIES, 0), t | prev << 8 | b << 16 | commit << 24, 0, 7));
              checked += 2;
            }
        }
        EXPECT(round_trip(hdr(src, dst, VOTE_REPLY, 0), t | 1u << 8, 0, 100));
        EXPECT(round_trip(hdr(src, dst, VOTE_REPLY, 0), t, 0, 0));
        EXPECT(round_trip(hdr(src, dst, APPEND_REPLY, 0), t, 0, 4000));
        checked += 3;
      }
  for (uint32_t dst = 0; dst < 5; dst++) {
    EXPECT(round_trip(hdr(0xFF, dst, ELECTION_TICK, 2), 0, 0, 42));      // timers: deadLetters, flagged TIMER
    EXPECT(round_trip(hdr(0xFF, dst, HEARTBEAT_TICK, 2), 0, 0, 4095));
    EXPECT(round_trip(hdr(0xFF, dst, BOOT, 1), 0x1F, 0, 1));             // external Sends: deadLetters, flagged EXTERNAL
    EXPECT(round_trip(hdr(0xFF, dst, CLIENT_CMD, 1), 0x7F, 0, 2));
    EXPECT(round_trip(hdr(0xFF, dst, CLIENT_CMD, 0), 3, 0, 2));          // deadLetters without flags
  }
  EXPECT(checked > 100000);
  // the header alone, and what pending_remove_at reads of a row
  EXPECT(lane_row8_hdr(lane_row8_pack(hdr(0xFF, 3, HEARTBEAT_TICK, 2), 0, 0, 17)) == hdr(0xFF, 3, HEARTBEAT_TICK, 2));
  for (uint32_t dst = 0; dst < 5; dst++)
    for (uint32_t type = 1; type <= 8; type++)
      for (uint32_t src : {0u, 4u, 0xFFu})
        for (uint32_t flags : {0u, 1u, 2u}) {
          if (src < 5 && flags) continue;
          const uint64_t r = lane_row8_pack(hdr(src, dst, type, flags), 0x0FFF0FFFu, 0xFFFF01u, 4095);
          EXPECT(lane_row8_sdt(r) == hdr(src, dst, type, 0));
          EXPECT(lane_row8_dst(r) == dst);
          EXPECT(lane_row8_timer_of(r, HEARTBEAT_TICK) == (src == 0xFF && flags == 2 && type == HEARTBEAT_TICK));
        }

  // what the layout cannot hold
  EXPECT(!lane_row8_fits(hdr(0xFF, 0, CLIENT_CMD, 3), 0, 0));            // both flags
  EXPECT(!lane_row8_fits(hdr(0, 0, VOTE_REPLY, 1), 0, 0));               // an actor's row with a flag
  EXPECT(!lane_row8_fits(hdr(7, 0, VOTE_REPLY, 0), 0, 0));               // a sender that is neither an actor nor deadLetters
  EXPECT(!lane_row8_fits(hdr(0xFE, 0, VOTE_REPLY, 0), 0, 0));
  EXPECT(!lane_row8_fits(hdr(0, 8, VOTE_REPLY, 0), 0, 0));               // dst in 3 bits
  EXPECT(!lane_row8_fits(hdr(0, 0, 16, 0), 0, 0));                       // type in 4 bits
  EXPECT(!lane_row8_fits(hdr(0xFF, 0, CLIENT_CMD, 1), 16u << 8, 0));     // p0 byte 1 in 4 bits
  EXPECT(!lane_row8_fits(hdr(0xFF, 0, CLIENT_CMD, 1), 16u << 24, 0));    // p0 byte 3 in 4 bits
  EXPECT(!lane_row8_fits(hdr(0xFF, 0, CLIENT_CMD, 1), 0, 2));            // p1 byte 0 in 1 bit
  EXPECT(!lane_row8_fits(hdr(0xFF, 0, CLIENT_CMD, 1), 0, 1u << 24));     // p1 byte 3 is zero
  EXPECT(lane_row8_fits(hdr(0xFF, 0, CLIENT_CMD, 1), 0x0FFF0FFFu, 0xFFFF01u));

  // the rule: the benchmark's launch (maxMessages 50: nodes below 6 + 51 * 7 = 363)
  EXPECT(lane_row8_eligible(snapshot(), 50, 6));
  EXPECT(lane_row8_eligible(snapshot(11), 50, 6));
  EXPECT(!lane_row8_eligible(snapshot(), -1, 6));
  // its edge: 6 + 584 * 7 = 4094 nodes fit 12 bits, 6 + 585 * 7 = 4101 do not
  EXPECT(lane_steady_node_bound(6, 584, 6) == 4094);
  EXPECT(lane_row8_eligible(snapshot(), 583, 6));
  EXPECT(!lane_row8_eligible(snapshot(), 584, 6));
  // a snapshot row the layout cannot hold: a client command of 16 << 8
  { LaneSnapshot s = snapshot(1); s.pend[5][1] = 16u << 8; EXPECT(!lane_row8_eligible(s, 50, 6)); }
  { LaneSnapshot s = snapshot(1); s.pend[5][1] = 15u << 8; EXPECT(lane_row8_eligible(s, 50, 6)); }
  // external protocol messages: their payloads are checked field by field (a deadLetters AppendReply never moves NEXT,
  // so its matchIndex is only a byte)
  { LaneSnapshot s = snapshot(1); s.pend[5][0] = hdr(0xFF, 0, APPEND_REPLY, 1); s.pend[5][1] = 3u | 1u << 8 | 200u << 16;
    EXPECT(lane_row8_eligible(s, 50, 6)); }
  { LaneSnapshot s = snapshot(1); s.pend[5][0] = hdr(0xFF, 0, APPEND_ENTRIES, 1); s.pend[5][1] = 3u | 15u << 8 | 8u << 24;
    s.pend[5][2] = 1u | 3u << 8 | 9u << 16; EXPECT(lane_row8_eligible(s, 50, 6)); }
  { LaneSnapshot s = snapshot(1); s.pend[5][0] = hdr(0xFF, 0, APPEND_ENTRIES, 1); s.pend[5][1] = 3u | 16u << 8;
    EXPECT(!lane_row8_eligible(s, 50, 6)); }
  { LaneSnapshot s = snapshot(1); s.pend[5][0] = hdr(0xFF, 0, VOTE_REPLY, 1); s.pend[5][1] = 3u | 1u << 8; s.pend[5][2] = 2;
    EXPECT(!lane_row8_eligible(s, 50, 6)); }

  if (failures) { printf("%d failures\n", failures); return 1; }
  printf("OK\n");
  return 0;
}
