// fuzzer_gen.cuh — Fuzzer.generateFuzzTest (fuzzing/Fuzzer.scala:123-174) with generateNextEvent (:84-121),
// FuzzerWeights (:24-58) and reset (:176-193), seeded.  One definition for the host entry point demi_fuzzer_generate
// (capi_experiment.cu) and the campaign's generator kernel fuzzer_gen_kernel (capi.cu): one thread draws one program.
// The reference seeds the fuzzer and its three RandomizedHashSets from the wall clock; all four take `seed` here.
#pragma once
#include "../../include/demi_b200.h"
#include "../../include/demi_limits.h"

namespace demi {

// java.util.Random (Java SE specification); scala.util.Random delegates to it (Fuzzer.scala:68)
struct FzJavaRandom {
  uint64_t s;
  DEMI_HD void seed(int64_t v) { s = ((uint64_t)v ^ 0x5DEECE66Dull) & ((1ull << 48) - 1); }
  DEMI_HD int32_t next(int bits) { s = (s * 0x5DEECE66Dull + 0xBull) & ((1ull << 48) - 1); return (int32_t)(int64_t)(s >> (48 - bits)); }
  DEMI_HD int32_t next_int(int32_t bound) {
    int32_t r = next(31), m = bound - 1;
    if ((bound & m) == 0) return (int32_t)(((int64_t)bound * (int64_t)r) >> 31);
    // Java's `u - (r = u % bound) + m < 0` wraps in int; here in uint32_t, where the wrap is defined
    for (int32_t u = r; (int32_t)((uint32_t)u - (uint32_t)(r = u % bound) + (uint32_t)m) < 0; u = next(31)) {}
    return r;
  }
  DEMI_HD double next_double() { return (double)(((int64_t)next(26) << 27) + next(27)) * (1.0 / (double)(1ll << 53)); }
};

// RandomizedHashSet (schedulers/Util.scala:110-185) over a caller-owned array
template <class T>
struct FzSet {
  T* arr; uint32_t n; FzJavaRandom rand;
  DEMI_HD void init(T* a, int64_t seed) { arr = a; n = 0; rand.seed(seed); }
  DEMI_HD void insert(T v) { arr[n++] = v; }
  DEMI_HD bool empty() const { return n == 0; }
  DEMI_HD T remove_random() { const int32_t i = rand.next_int((int32_t)n); const T v = arr[i]; arr[i] = arr[n - 1]; n--; return v; }
  DEMI_HD T get_random() { return arr[rand.next_int((int32_t)n)]; }
};

// Room a program needs: the prefix, num_events generated events, the postfix and the closing WaitQuiescence.
DEMI_HD uint64_t fuzzer_program_room(const demi_fuzzer_config& cfg, uint32_t n_prefix, uint32_t n_postfix) {
  return (uint64_t)n_prefix + cfg.num_events + n_postfix + 1u;
}
// Scratch of the three sets: `alive` holds one entry per Start of the prefix, `pairs` two runs of
// starts*(starts-1)/2 entries (currentlyPartitioned, currentlyUnpartitioned).
DEMI_HD uint32_t fuzzer_pair_room(uint32_t starts) { return starts * (starts - 1u) / 2u; }

// Writes the program to out[0 .. return value) (out has fuzzer_program_room entries) and its number of Sends to
// *n_sends.  The message counter of message_gen starts at 1 in every program.
DEMI_HD uint32_t fuzzer_generate(const demi_fuzzer_config& cfg, int64_t seed,
                                 const demi_ext_event* prefix, uint32_t n_prefix,
                                 const demi_ext_event* postfix, uint32_t n_postfix,
                                 uint8_t* alive_buf, uint16_t* pair_buf, demi_ext_event* out, uint32_t* n_sends) {
  const double w_kill = cfg.kill, w_send = cfg.send, w_part = cfg.partition, w_unpart = cfg.unpartition;   // allWeights (:40)
  const double total = cfg.kill + cfg.send + cfg.partition + cfg.unpartition + cfg.wait_quiescence;
  uint32_t next_id = 0, starts = 0, len = 0, sends = 0;
  for (uint32_t i = 0; i < n_prefix; i++) {
    const demi_ext_event e = prefix[i];
    if (e.kind == DEMI_EXT_START) alive_buf[starts++] = e.a;        // `nodes`, in prefix order
    if (e.kind == DEMI_EXT_SEND) sends++;
    if (e.id > next_id) next_id = e.id;
    out[len++] = e;
  }
  for (uint32_t i = 0; i < n_postfix; i++) if (postfix[i].id > next_id) next_id = postfix[i].id;
  FzJavaRandom rand; rand.seed(seed);
  FzSet<uint8_t> alive; FzSet<uint16_t> partitioned, unpartitioned;
  const uint32_t np = fuzzer_pair_room(starts);
  alive.init(alive_buf, seed); alive.n = starts;                    // the Starts were written in insertion order
  partitioned.init(pair_buf, seed); unpartitioned.init(pair_buf + np, seed);
  for (uint32_t i = 0; i < starts; i++)
    for (uint32_t j = i + 1; j < starts; j++) unpartitioned.insert((uint16_t)(alive_buf[i] | (alive_buf[j] << 8)));
  uint32_t counter = 0;
  bool just_wq = len > 0 && out[len - 1].kind == DEMI_EXT_WAIT_QUIESCENCE;
  bool ran_out = false;
  for (uint32_t i = 0; i < cfg.num_events; i++) {
    demi_ext_event ev{};
    // generateNextEvent; kind 0 = "no more events" (Kill with nobody alive, :92-95)
    for (;;) {
      ev = demi_ext_event{};
      const double scaled = rand.next_double() * total;
      uint32_t kind = 0;
      double cur = w_kill;
      if (scaled < cur) {
        if (alive.empty()) break;
        kind = DEMI_EXT_KILL; ev.a = alive.remove_random();
      } else if (scaled < (cur += w_send)) {
        // With everyone killed the reference's getRandomElement throws (nextInt(0)); here nextInt(0) draws index 0,
        // which still holds the actor killed last.
        kind = DEMI_EXT_SEND; ev.a = alive.get_random(); ev.type = (uint8_t)cfg.send_type; ev.p0 = ++counter;
      } else if (scaled < (cur += w_part)) {
        if (unpartitioned.empty()) continue;                          // "Try again..."
        const uint16_t p = unpartitioned.remove_random(); partitioned.insert(p);
        kind = DEMI_EXT_PARTITION; ev.a = (uint8_t)(p & 0xFF); ev.b = (uint8_t)(p >> 8);
      } else if (scaled < (cur += w_unpart)) {
        if (partitioned.empty()) continue;
        const uint16_t p = partitioned.remove_random(); unpartitioned.insert(p);
        kind = DEMI_EXT_UNPARTITION; ev.a = (uint8_t)(p & 0xFF); ev.b = (uint8_t)(p >> 8);
      } else {
        kind = DEMI_EXT_WAIT_QUIESCENCE;
      }
      ev.id = ++next_id;                                              // a rejected WaitQuiescence used up its id too
      if (kind == DEMI_EXT_WAIT_QUIESCENCE && just_wq) continue;       // no two WaitQuiescence in a row
      ev.kind = (uint8_t)kind;
      break;
    }
    if (!ev.kind) { ran_out = true; break; }
    just_wq = ev.kind == DEMI_EXT_WAIT_QUIESCENCE;
    if (ev.kind == DEMI_EXT_SEND) sends++;
    out[len++] = ev;
  }
  if (!ran_out) {
    for (uint32_t i = 0; i < n_postfix; i++) { out[len++] = postfix[i]; if (postfix[i].kind == DEMI_EXT_SEND) sends++; }
    if (len > 0 && out[len - 1].kind != DEMI_EXT_WAIT_QUIESCENCE) {
      demi_ext_event wq{}; wq.kind = DEMI_EXT_WAIT_QUIESCENCE; wq.id = ++next_id;
      out[len++] = wq;
    }
  }
  *n_sends = sends;
  return len;
}

}  // namespace demi
