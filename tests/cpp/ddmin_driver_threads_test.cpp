// DDMinDriver (demi_b200/csrc/ddmin_driver.hpp) host-only, as demi_ddmin_many runs it: many drivers on threads at once,
// each over a synthetic monotone oracle (a test fails iff its mask holds all of the trace's culprit set K).  Built with
// AddressSanitizer, so a driver that touches freed memory fails the run; every driver's MCS and counters must equal its
// solo run.  Prints "OK" at the end.
#include <cstdio>
#include <thread>
#include <vector>
#include "../../demi_b200/csrc/ddmin_driver.hpp"

thread_local std::string g_create_error;

using namespace demi;

struct SupersetDriver : DDMinDriver {
  Mask K;
  int32_t evaluate(const uint64_t* masks, size_t n, signed char* out) override {
    for (size_t i = 0; i < n; i++) {
      bool all = true;
      for (uint32_t w = 0; w < mw; w++) all = all && (masks[i * mw + w] & K[w]) == K[w];
      out[i] = all;
    }
    return DEMI_OK;
  }
};

struct Run { Mask mcs; uint32_t total, batches, executed; std::vector<uint32_t> sizes; };

static Run run(uint32_t seed, size_t wide) {
  // a program of 40..120 externals: Sends, Start/Kill pairs, Partition/UnPartition pairs
  uint32_t x = seed * 2654435761u + 1;
  auto rnd = [&]() { x ^= x << 13; x ^= x >> 17; x ^= x << 5; return x; };
  const uint32_t n = 40 + rnd() % 81;
  std::vector<demi_ext_event> ext;
  for (uint32_t i = 0; ext.size() < n; i++) {
    const uint32_t r = rnd() % 10;
    if (r == 0 && ext.size() + 2 <= n) { ext.push_back({DEMI_EXT_START, (uint8_t)(rnd() % 5), 0, 0, 0, 0, 0}); ext.push_back({DEMI_EXT_KILL, ext.back().a, 0, 0, 0, 0, 0}); }
    else if (r == 1 && ext.size() + 2 <= n) { ext.push_back({DEMI_EXT_PARTITION, 0, 1, 0, 0, 0, 0}); ext.push_back({DEMI_EXT_UNPARTITION, 0, 1, 0, 0, 0, 0}); }
    else ext.push_back({DEMI_EXT_SEND, (uint8_t)(rnd() % 5), 0, 1, i, 0, 0});
  }
  demi_handle eh;
  SupersetDriver d;
  d.h = &eh; d.mw = (n + 63) / 64; d.n_ext = n; d.ext = ext.data(); d.wide_cap = wide;
  d.K.assign(d.mw, 0);
  for (int k = 0; k < 3; k++) { const uint32_t i = rnd() % n; if (ext[i].kind == DEMI_EXT_SEND) DDMinDriver::setbit(d.K, i); }
  Mask dag(d.mw, 0), zero(d.mw, 0);
  for (uint32_t i = 0; i < n; i++) DDMinDriver::setbit(dag, i);
  d.original_num_events = n;
  Run r;
  r.mcs = d.ddmin2(dag, zero);
  r.total = d.total_replays; r.batches = d.batches; r.executed = d.replays_executed; r.sizes = d.iteration_sizes;
  return r;
}

int main() {
  const uint32_t N = 256;
  for (size_t wide : {(size_t)0, (size_t)64, (size_t)6000}) {
    std::vector<Run> solo(N), many(N);
    for (uint32_t s = 0; s < N; s++) solo[s] = run(s, wide);
    std::vector<std::thread> th;
    for (uint32_t k = 0; k < 32; k++)
      th.emplace_back([&, k]() { for (uint32_t s = k; s < N; s += 32) many[s] = run(s, wide); });
    for (std::thread& t : th) t.join();
    for (uint32_t s = 0; s < N; s++)
      if (solo[s].mcs != many[s].mcs || solo[s].total != many[s].total || solo[s].batches != many[s].batches ||
          solo[s].executed != many[s].executed || solo[s].sizes != many[s].sizes) {
        std::printf("FAILED: seed %u wide %zu\n", s, wide);
        return 1;
      }
  }
  std::printf("OK\n");
  return 0;
}
