// demi_b200.hpp — C++ host-side mirror of DEMi's scheduler plugin surface over the C ABI
// (include/demi_b200.h).  Header-only; link with -ldemi_b200.
//
// The reference's host is Scala; this image has no JVM toolchain, so the compiled-language host
// layer that sits above the C ABI is C++ here (the JNI/Scala binding a DEMi maintainer would add is
// in jni/).  Class and method names, argument meaning and error behaviour follow the reference:
//
//   SchedulerConfig      src/main/scala/verification/SchedulerConfig.scala:9-37
//   RandomScheduler      schedulers/RandomScheduler.scala:41 (explore :234, test :597, setMaxMessages :55,
//                        setInvariant :521)
//   STSScheduler         schedulers/STSScheduler.scala:84 (test :199)
//   ReplayScheduler      schedulers/ReplayScheduler.scala:71 (replay; ReplayException :128-130)
//   DDMin                minification/DeltaDebugging.scala:7 (minimize :27, verify_mcs :64)
//   STSSchedMinimizer    minification/internal_minimization/ScheduleCheckers.scala:19 (minimize :34)
//   WildcardMinimizer    minification/wildcard_minimization/WildcardMinimizer.scala:47 (minimize :133)
//   DPORwHeuristics      schedulers/DPORwHeuristics.scala:77 (test :1193, setMaxMessagesToSchedule :123,
//                        setDepthBound :116)
//   MinimizationStats    minification/Minimizer.scala:30-237 (the counters DDMin / the minimizers drive)
//
// Reference exceptions map to C++ ones: IllegalArgumentException -> std::invalid_argument,
// IllegalStateException -> std::logic_error, ReplayException -> demi::ReplayException, anything the
// engine reports -> demi::Error (code + demi_last_error text).  There is no CPU fallback: without a
// CUDA device the constructors throw demi::Error(DEMI_ERR_NO_DEVICE).
#pragma once
#include <algorithm>
#include <cstdint>
#include <functional>
#include <map>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>
#include "demi_b200.h"

namespace demi {

struct Error : std::runtime_error {
  int32_t code;
  Error(int32_t c, const std::string& what) : std::runtime_error(what), code(c) {}
};
struct ReplayException : std::runtime_error { using std::runtime_error::runtime_error; };

typedef uint32_t ViolationFingerprint;          // the model's violation code; 0 = "any" where optional
typedef std::vector<demi_ext_event> ExternalEvents;
typedef std::vector<demi_event> EventTrace;

// ---- external events (ExternalEvents.scala:62-91) with stable ids (UniqueExternalEvent._id)
inline uint32_t next_external_id() { static uint32_t id = 0; return ++id; }            // IDGenerator
inline demi_ext_event Start(uint8_t name) { return {DEMI_EXT_START, name, 0, 0, 0, 0, next_external_id()}; }
inline demi_ext_event Kill(uint8_t name) { return {DEMI_EXT_KILL, name, 0, 0, 0, 0, next_external_id()}; }
inline demi_ext_event HardKill(uint8_t name) { return {DEMI_EXT_HARD_KILL, name, 0, 0, 0, 0, next_external_id()}; }
inline demi_ext_event Send(uint8_t name, uint8_t type, uint32_t p0 = 0, uint32_t p1 = 0) {
  return {DEMI_EXT_SEND, name, 0, type, p0, p1, next_external_id()};
}
inline demi_ext_event WaitQuiescence() { return {DEMI_EXT_WAIT_QUIESCENCE, 0, 0, 0, 0, 0, next_external_id()}; }
inline demi_ext_event Partition(uint8_t a, uint8_t b) { return {DEMI_EXT_PARTITION, a, b, 0, 0, 0, next_external_id()}; }
inline demi_ext_event UnPartition(uint8_t a, uint8_t b) { return {DEMI_EXT_UNPARTITION, a, b, 0, 0, 0, next_external_id()}; }

struct SchedulerConfig {
  int32_t model = DEMI_MODEL_RAFT5;
  uint32_t model_flags = 0;
  int32_t device = 0;
  bool ignoreTimers = false;
  bool filterKnownAbsents = false;
  uint32_t blocked_mask = 0;
  int32_t strategy = DEMI_RS_FULLY_RANDOM;      // RandomizationStrategy: FullyRandom | SrcDstFIFO
};

// MinimizationStats (minification/Minimizer.scala:30-237) with the reference's shape: one InnerStats per
// <strategy, oracle> pair, the maps keyed by the replay number, and toJson() with the keys of minimization_stats.json.
struct MinimizationStats {
  struct InnerStats {
    std::string name;
    uint32_t total_replays = 0;
    std::map<uint32_t, uint32_t> iterationSize, internalIterationSize, maxDistance;
    std::map<std::string, double> stats;
    explicit InnerStats(const std::string& n) : name(n) { reset(); }
    void reset() {                                                       // :125-157 (total_replays is not reset, as written)
      iterationSize.clear(); internalIterationSize.clear(); maxDistance.clear(); stats.clear();
      for (const char* k : {"prune_duration_seconds", "prune_start_epoch", "prune_end_epoch", "replay_duration_seconds",
                            "replay_end_epoch", "replay_start_epoch", "original_duration_seconds"}) stats[k] = -1.0;
      for (const char* k : {"total_inputs", "total_events", "initial_verification_runs_needed", "minimized_deliveries",
                            "minimized_externals", "minimized_timers"}) stats[k] = 0.0;
    }
    static std::string map_json(const std::map<uint32_t, uint32_t>& m) {
      std::string o = "{"; bool first = true;
      for (auto& kv : m) { o += (first ? "\"" : ", \"") + std::to_string(kv.first) + "\": " + std::to_string(kv.second); first = false; }
      return o + "}";
    }
    std::string toJson() const {                                          // :207-217
      std::string o = "{\"name\": \"" + name + "\", \"iteration_size\": " + map_json(iterationSize) +
                      ", \"internal_iteration_size\": " + map_json(internalIterationSize) + ", \"total_replays\": " +
                      std::to_string(total_replays) + ", \"maxDistance\": " + map_json(maxDistance);
      for (auto& kv : stats) o += ", \"" + kv.first + "\": " + std::to_string(kv.second);
      return o + "}";
    }
  };
  std::string minimization_strategy, test_oracle;
  std::vector<InnerStats> stats;
  void updateStrategy(const std::string& strategy, const std::string& oracle) {   // :41-47
    minimization_strategy = strategy; test_oracle = oracle;
    stats.emplace_back("(" + strategy + "," + oracle + ")");
  }
  InnerStats& inner() { if (stats.empty()) updateStrategy(minimization_strategy, test_oracle); return stats.back(); }
  void reset() { inner().reset(); }
  void increment_replays(uint32_t n = 1) { inner().total_replays += n; }
  void record_iteration_size(uint32_t n) { inner().iterationSize[inner().total_replays] = n; iteration_size.push_back(n); }
  void record_internal_size(uint32_t n) { inner().internalIterationSize[inner().total_replays] = n; internal_size.push_back(n); }
  void record_distance_increase(uint32_t d) { inner().maxDistance[d] = inner().total_replays; }
  void recordDeliveryStats(uint32_t deliveries, uint32_t externals, uint32_t timers) {
    inner().stats["minimized_deliveries"] = deliveries; inner().stats["minimized_externals"] = externals; inner().stats["minimized_timers"] = timers;
  }
  std::string toJson() const {                                            // :98-100
    std::string o = "["; bool first = true;
    for (auto& s : stats) { o += (first ? "" : ", ") + s.toJson(); first = false; }
    return o + "]";
  }
  // the engine returns a minimization's whole record_*_size series; kept in recording order beside the maps
  std::vector<uint32_t> iteration_size, internal_size;
  uint32_t& total_replays_ref() { return inner().total_replays; }
  // one record per test keyed by the replay number, the fencepost record on the last replay number again
  void record_series(const uint32_t* sizes, size_t n, bool internal) {
    InnerStats& in = inner();
    const uint32_t base = in.total_replays;
    for (size_t i = 0; i < n; i++) {
      const uint32_t key = base + (uint32_t)std::min(i + 1, n > 1 ? n - 1 : (size_t)1);
      (internal ? in.internalIterationSize : in.iterationSize)[key] = sizes[i];
      (internal ? internal_size : iteration_size).push_back(sizes[i]);
    }
  }
};

// One demi_handle.
class Engine {
 public:
  explicit Engine(const SchedulerConfig& c) : cfg(c) {
    demi_config dc{};
    dc.device = c.device; dc.model = c.model; dc.model_flags = c.model_flags; dc.blocked_mask = c.blocked_mask;
    dc.ignore_timers = c.ignoreTimers ? 1 : 0; dc.strategy = c.strategy;
    int32_t rc = demi_create(&dc, &h);
    if (rc != DEMI_OK) throw Error(rc, demi_last_error(nullptr));
  }
  ~Engine() { demi_destroy(h); }
  Engine(const Engine&) = delete;
  Engine& operator=(const Engine&) = delete;
  void check(int32_t rc) const {
    if (rc == DEMI_OK) return;
    std::string msg = demi_last_error(h);
    if (rc == DEMI_ERR_INVALID) throw std::invalid_argument(msg);
    if (rc == DEMI_ERR_STATE) throw std::logic_error(msg);
    throw Error(rc, msg);
  }
  demi_handle* handle() const { return h; }
  // an application model as data (demi_model_ir.h) for SchedulerConfig.model == 100; actor / message names as in the blob
  void load_model(const std::vector<uint32_t>& blob) { check(demi_load_model(h, blob.data(), blob.size() * sizeof(uint32_t))); }
  int32_t actor_index(const std::string& name) const { return demi_actor_index(h, name.c_str()); }
  std::string actor_name(int32_t idx) const { const char* n = demi_actor_name(h, idx); return n ? n : ""; }
  // FullyRandom's userDefinedFilter (RandomScheduler.scala:666-684) as rules; an empty list removes it
  void set_user_filter(const std::vector<demi_filter_rule>& rules) { check(demi_set_user_filter(h, rules.data(), (uint32_t)rules.size())); }
  // UnmodifiedEventDag.conjoinAtoms (minification/Util.scala:167-178): DDMin treats the two externals as one atom
  void conjoin_atoms(uint32_t i1, uint32_t i2) { check(demi_conjoin_atoms(h, i1, i2)); }      // indices into the trace's externals
  demi_perf stats() const { demi_perf p{}; demi_stats(h, &p); return p; }
  int32_t lane_kernel() const { return demi_lane_kernel(h); }      // DEMI_LANE_*: what the last fuzz launch ran
  // ---- campaigns: a new Fuzzer program per execution (RunnerUtils.fuzz's loop, RunnerUtils.scala:75-91)
  // demi_set_fuzzer: new Fuzzer(num_events, weights, message_gen, prefix, postfix) (Fuzzer.scala:61-82)
  void set_fuzzer(const demi_fuzzer_config& c, const ExternalEvents& prefix, const ExternalEvents& postfix = {}) {
    check(demi_set_fuzzer(h, &c, prefix.data(), (uint32_t)prefix.size(), postfix.empty() ? nullptr : postfix.data(),
                          (uint32_t)postfix.size()));
    fz_cfg = c; fz_prefix = prefix; fz_postfix = postfix;
  }
  // the program the campaign execution with this program seed runs (demi_fuzzer_generate)
  ExternalEvents fuzzer_program(int64_t program_seed) const {
    ExternalEvents out(fz_prefix.size() + fz_cfg.num_events + fz_postfix.size() + 1);
    uint32_t n = 0;
    check(demi_fuzzer_generate(&fz_cfg, program_seed, fz_prefix.data(), (uint32_t)fz_prefix.size(),
                               fz_postfix.empty() ? nullptr : fz_postfix.data(), (uint32_t)fz_postfix.size(), out.data(),
                               (uint32_t)out.size(), &n));
    out.resize(n);
    return out;
  }
  // demi_fuzz_campaign: record i = program fuzzer_program(program_seed_base + i) under FullyRandom(seed_base + i)
  std::vector<demi_fuzz_result> fuzz_campaign(int64_t seed_base, uint64_t n, int32_t max_messages, int32_t interval,
                                              int64_t program_seed_base, uint32_t looking_for = 0) {
    demi_fuzz_params p{seed_base, n, max_messages, interval, looking_for, 0};
    std::vector<demi_fuzz_result> out(n);
    check(demi_fuzz_campaign(h, &p, program_seed_base, out.data()));
    return out;
  }
  // ---- many traces: recording, replay and DDMin with their tests in shared launches
  // demi_fuzz_traces: the EventTraces of executions seed_base + prefix_index[i] of the program (demi_set_externals)
  std::vector<EventTrace> fuzz_traces(int64_t seed_base, const std::vector<uint32_t>& prefix_index, int32_t max_messages,
                                      int32_t interval, uint32_t looking_for = 0, uint32_t cap_events = 4096) {
    demi_fuzz_params p{seed_base, prefix_index.size(), max_messages, interval, looking_for, 0};
    std::vector<demi_event> ev(prefix_index.size() * (size_t)cap_events);
    std::vector<uint32_t> n(prefix_index.size());
    check(demi_fuzz_traces(h, &p, prefix_index.data(), (uint32_t)prefix_index.size(), ev.data(), cap_events, n.data(), nullptr));
    std::vector<EventTrace> out(n.size());
    for (size_t i = 0; i < n.size(); i++) out[i].assign(ev.begin() + i * cap_events, ev.begin() + i * cap_events + n[i]);
    return out;
  }
  // demi_fuzz_traces_tree: fuzz_traces plus each execution's DepTracker tree (fuzz_trace's dep_parent for that seed)
  std::vector<std::pair<EventTrace, std::vector<uint16_t>>> fuzz_traces_tree(int64_t seed_base, const std::vector<uint32_t>& prefix_index,
                                                                            int32_t max_messages, int32_t interval, uint32_t looking_for = 0,
                                                                            uint32_t cap_events = 4096, uint32_t cap_nodes = 4096) {
    demi_fuzz_params p{seed_base, prefix_index.size(), max_messages, interval, looking_for, 0};
    const size_t n = prefix_index.size();
    std::vector<demi_event> ev(n * (size_t)cap_events);
    std::vector<uint16_t> par(n * (size_t)cap_nodes);
    std::vector<uint32_t> ne(n), nn(n);
    check(demi_fuzz_traces_tree(h, &p, prefix_index.data(), (uint32_t)n, ev.data(), cap_events, ne.data(), par.data(), cap_nodes,
                                nn.data(), nullptr));
    std::vector<std::pair<EventTrace, std::vector<uint16_t>>> out(n);
    for (size_t i = 0; i < n; i++) {
      out[i].first.assign(ev.begin() + i * cap_events, ev.begin() + i * cap_events + ne[i]);
      out[i].second.assign(par.begin() + i * cap_nodes, par.begin() + i * cap_nodes + std::min(nn[i], cap_nodes));
    }
    return out;
  }
  // demi_set_traces: trace i with externals[i] (or one program shared by all when externals has one entry)
  void set_traces(const std::vector<EventTrace>& traces, const std::vector<ExternalEvents>& externals) {
    const bool shared = externals.size() == 1;
    std::vector<demi_event> ev; std::vector<demi_ext_event> ex;
    std::vector<uint32_t> eo, ne, xo, nx;
    for (size_t i = 0; i < traces.size(); i++) {
      eo.push_back((uint32_t)ev.size()); ne.push_back((uint32_t)traces[i].size());
      ev.insert(ev.end(), traces[i].begin(), traces[i].end());
      const ExternalEvents& x = externals.at(shared ? 0 : i);
      xo.push_back(shared ? 0u : (uint32_t)ex.size()); nx.push_back((uint32_t)x.size());
      if (!shared || i == 0) ex.insert(ex.end(), x.begin(), x.end());
    }
    check(demi_set_traces(h, (uint32_t)traces.size(), ev.data(), eo.data(), ne.data(), ex.data(), xo.data(), nx.data()));
    set_ext.clear();
    for (size_t i = 0; i < traces.size(); i++) set_ext.push_back(externals.at(shared ? 0 : i));
  }
  uint32_t set_mask_words() const {
    size_t m = 1;
    for (const ExternalEvents& x : set_ext) m = std::max(m, x.size());
    return (uint32_t)((m + 63) / 64);
  }
  // demi_replay_batch_many: masks[i] (set_mask_words() words) on trace trace_of_test[i]
  std::vector<demi_replay_result> replay_batch_many(const std::vector<uint32_t>& trace_of_test, const std::vector<uint64_t>& masks,
                                                    const std::vector<ViolationFingerprint>& looking_for, uint32_t flags = 0) {
    std::vector<demi_replay_result> out(trace_of_test.size());
    check(demi_replay_batch_many(h, trace_of_test.data(), masks.data(), (uint32_t)trace_of_test.size(), set_mask_words(),
                                 looking_for.data(), flags, out.data()));
    return out;
  }
  // demi_ddmin_many: per trace of the set, its MCS (WaitQuiescence dropped) and the DDMin record, or the error code
  struct DDMinManyResult { ExternalEvents mcs; demi_ddmin_out out; int32_t status; std::vector<uint32_t> iteration_sizes; };
  std::vector<DDMinManyResult> ddmin_many(const std::vector<ViolationFingerprint>& looking_for, uint32_t flags = 0,
                                          bool checkUnmodifed = true, uint32_t cap_iterations = 256) {
    const size_t n = set_ext.size();
    const uint32_t mw = set_mask_words();
    std::vector<uint64_t> mcs(n * mw);
    std::vector<uint32_t> iters(n * cap_iterations);
    std::vector<demi_ddmin_out> out(n);
    std::vector<int32_t> status(n);
    check(demi_ddmin_many(h, looking_for.data(), flags, checkUnmodifed ? 1 : 0, mcs.data(), mw, iters.data(), cap_iterations,
                          out.data(), status.data()));
    std::vector<DDMinManyResult> r(n);
    for (size_t t = 0; t < n; t++) {
      r[t].out = out[t]; r[t].status = status[t];
      if (status[t] != DEMI_OK) continue;
      for (size_t i = 0; i < set_ext[t].size(); i++) if ((mcs[t * mw + (i >> 6)] >> (i & 63)) & 1ull) r[t].mcs.push_back(set_ext[t][i]);
      r[t].iteration_sizes.assign(iters.begin() + t * cap_iterations, iters.begin() + t * cap_iterations + std::min(out[t].n_iterations, cap_iterations));
    }
    return r;
  }
  // demi_replay_traces_many: the EventTrace of test i (trace trace_of_test[i], masks[i] of set_mask_words() words or the
  // full externals when masks is empty, trace event skip_events[i] left out or none when skip_events is empty)
  struct RecordedReplay { EventTrace trace; demi_replay_result result; };
  std::vector<RecordedReplay> replay_traces_many(const std::vector<uint32_t>& trace_of_test, const std::vector<uint64_t>& masks,
                                                 const std::vector<uint32_t>& skip_events,
                                                 const std::vector<ViolationFingerprint>& looking_for, uint32_t flags = 0,
                                                 uint32_t cap_events = 4096) {
    const size_t n = trace_of_test.size();
    std::vector<demi_event> ev(n * (size_t)cap_events);
    std::vector<uint32_t> ne(n);
    std::vector<demi_replay_result> res(n);
    check(demi_replay_traces_many(h, trace_of_test.data(), masks.empty() ? nullptr : masks.data(),
                                  skip_events.empty() ? nullptr : skip_events.data(), (uint32_t)n, set_mask_words(),
                                  looking_for.data(), flags, ev.data(), cap_events, ne.data(), res.data()));
    std::vector<RecordedReplay> r(n);
    for (size_t i = 0; i < n; i++) {
      r[i].result = res[i];
      r[i].trace.assign(ev.begin() + i * cap_events, ev.begin() + i * cap_events + std::min(ne[i], cap_events));
    }
    return r;
  }
  // demi_internal_minimize_many: per trace of the set (a verified MCS trace), its minimized trace and record, or the
  // error code
  struct IntMinManyResult { EventTrace trace; std::vector<uint32_t> internal_sizes; demi_intmin_out out; int32_t status; };
  std::vector<IntMinManyResult> internal_minimize_many(const std::vector<ViolationFingerprint>& looking_for, uint32_t flags = 0,
                                                       uint32_t cap_events = 4096, uint32_t cap_sizes = 1024) {
    const size_t n = set_ext.size();
    std::vector<demi_event> ev(n * (size_t)cap_events);
    std::vector<uint32_t> sizes(n * (size_t)cap_sizes);
    std::vector<demi_intmin_out> out(n);
    std::vector<int32_t> status(n);
    check(demi_internal_minimize_many(h, looking_for.data(), flags, ev.data(), cap_events, sizes.data(), cap_sizes, out.data(),
                                      status.data()));
    std::vector<IntMinManyResult> r(n);
    for (size_t t = 0; t < n; t++) {
      r[t].out = out[t]; r[t].status = status[t];
      if (status[t] != DEMI_OK) continue;
      r[t].trace.assign(ev.begin() + t * cap_events, ev.begin() + t * cap_events + std::min(out[t].n_events, cap_events));
      r[t].internal_sizes.assign(sizes.begin() + t * cap_sizes, sizes.begin() + t * cap_sizes + std::min(out[t].n_internal_sizes, cap_sizes));
    }
    return r;
  }
  // demi_wildcard_minimize_many: per trace of the set (a verified MCS trace), its wildcard-minimized trace and record
  // under the handle's clock rules, or the error code
  std::vector<IntMinManyResult> wildcard_minimize_many(const std::vector<ViolationFingerprint>& looking_for, uint32_t flags = 0,
                                                       uint32_t cap_events = 4096, uint32_t cap_sizes = 1024) {
    const size_t n = set_ext.size();
    std::vector<demi_event> ev(n * (size_t)cap_events);
    std::vector<uint32_t> sizes(n * (size_t)cap_sizes);
    std::vector<demi_intmin_out> out(n);
    std::vector<int32_t> status(n);
    check(demi_wildcard_minimize_many(h, looking_for.data(), flags, ev.data(), cap_events, sizes.data(), cap_sizes, out.data(),
                                      status.data()));
    std::vector<IntMinManyResult> r(n);
    for (size_t t = 0; t < n; t++) {
      r[t].out = out[t]; r[t].status = status[t];
      if (status[t] != DEMI_OK) continue;
      r[t].trace.assign(ev.begin() + t * cap_events, ev.begin() + t * cap_events + std::min(out[t].n_events, cap_events));
      r[t].internal_sizes.assign(sizes.begin() + t * cap_sizes, sizes.begin() + t * cap_sizes + std::min(out[t].n_internal_sizes, cap_sizes));
    }
    return r;
  }
  // demi_random_ddmin_many: randomDDMin on every program t (RandomScheduler.test with N = max_executions), with its own
  // seed, setMaxMessages and violation; per trace its MCS mask, keyed iteration sizes and record, or the error code
  struct RandomDDMinManyResult {
    std::vector<uint64_t> mcs_mask; std::vector<uint32_t> iteration_sizes; std::vector<uint64_t> iteration_keys;
    demi_random_ddmin_out out{}; int32_t status = DEMI_OK;
  };
  std::vector<RandomDDMinManyResult> random_ddmin_many(const std::vector<ExternalEvents>& programs, const std::vector<int64_t>& seeds,
                                                       const std::vector<int32_t>& max_messages,
                                                       const std::vector<ViolationFingerprint>& looking_for, uint32_t max_executions,
                                                       int32_t interval = 0, bool check_unmodified = false,
                                                       uint32_t cap_iterations = 1024) {
    const size_t n = programs.size();
    const FlatPrograms fp = flatten(programs);
    const size_t words = fp.words;
    const demi_fuzz_params p{0, max_executions, -1, interval, 0, 0};
    std::vector<uint64_t> mcs(n * words), keys(n * (size_t)cap_iterations);
    std::vector<uint32_t> sizes(n * (size_t)cap_iterations);
    std::vector<demi_random_ddmin_out> out(n);
    std::vector<int32_t> status(n);
    check(demi_random_ddmin_many(h, (uint32_t)n, fp.ev.data(), fp.off.data(), fp.cnt.data(), seeds.data(), max_messages.data(),
                                 looking_for.data(), &p, check_unmodified ? 1 : 0, mcs.data(), (uint32_t)words, sizes.data(),
                                 keys.data(), cap_iterations, out.data(), status.data()));
    std::vector<RandomDDMinManyResult> r(n);
    for (size_t t = 0; t < n; t++) {
      r[t].out = out[t]; r[t].status = status[t];
      if (status[t] != DEMI_OK) continue;
      const size_t k = std::min(out[t].n_iterations, cap_iterations);
      r[t].mcs_mask.assign(mcs.begin() + t * words, mcs.begin() + (t + 1) * words);
      r[t].iteration_sizes.assign(sizes.begin() + t * cap_iterations, sizes.begin() + t * cap_iterations + k);
      r[t].iteration_keys.assign(keys.begin() + t * cap_iterations, keys.begin() + t * cap_iterations + k);
    }
    return r;
  }
  // demi_fuzz_traces_many: execution seeds[t] of programs[t] (of the subsequence masks[t] keeps of it, when masks is
  // not empty), with its own setMaxMessages and violation; per trace its EventTrace, DepTracker tree (with_trees),
  // record, or the error code
  struct RecordedExecution { EventTrace trace; std::vector<uint16_t> depGraph; demi_fuzz_result result{}; int32_t status = DEMI_OK; };
  std::vector<RecordedExecution> fuzz_traces_many(const std::vector<ExternalEvents>& programs, const std::vector<int64_t>& seeds,
                                                  const std::vector<int32_t>& max_messages,
                                                  const std::vector<ViolationFingerprint>& looking_for, int32_t interval,
                                                  const std::vector<std::vector<uint64_t>>& masks = {}, bool with_trees = false,
                                                  uint32_t cap_events = 4096, uint32_t cap_nodes = 4096) {
    const size_t n = programs.size();
    const FlatPrograms fp = flatten(programs);
    const size_t words = fp.words;
    std::vector<uint64_t> mk;
    if (!masks.empty())
      for (size_t t = 0; t < n; t++) {
        std::vector<uint64_t> row = masks.at(t);
        row.resize(words, 0);
        mk.insert(mk.end(), row.begin(), row.end());
      }
    const demi_fuzz_params p{0, 0, -1, interval, 0, 0};
    std::vector<demi_event> ev(n * (size_t)cap_events);
    std::vector<uint16_t> par(with_trees ? n * (size_t)cap_nodes : 0);
    std::vector<uint32_t> ne(n), nn(n);
    std::vector<demi_fuzz_result> res(n);
    std::vector<int32_t> status(n);
    check(demi_fuzz_traces_many(h, (uint32_t)n, fp.ev.data(), fp.off.data(), fp.cnt.data(), mk.empty() ? nullptr : mk.data(),
                                (uint32_t)words, seeds.data(), max_messages.data(), looking_for.data(), &p, ev.data(), cap_events,
                                ne.data(), with_trees ? par.data() : nullptr, cap_nodes, nn.data(), res.data(), status.data()));
    std::vector<RecordedExecution> r(n);
    for (size_t t = 0; t < n; t++) {
      r[t].result = res[t]; r[t].status = status[t];
      if (status[t] != DEMI_OK) continue;
      r[t].trace.assign(ev.begin() + t * cap_events, ev.begin() + t * cap_events + std::min(ne[t], cap_events));
      if (with_trees) r[t].depGraph.assign(par.begin() + t * cap_nodes, par.begin() + t * cap_nodes + std::min(nn[t], cap_nodes));
    }
    return r;
  }
  const SchedulerConfig cfg;
 private:
  // programs one after the other (one empty event at least, so that the pointer is valid), where each starts, its
  // length, and the mask words of the longest
  struct FlatPrograms { ExternalEvents ev; std::vector<uint32_t> off, cnt; size_t words = 1; };
  static FlatPrograms flatten(const std::vector<ExternalEvents>& programs) {
    FlatPrograms f;
    for (const ExternalEvents& p : programs) {
      f.off.push_back((uint32_t)f.ev.size()); f.cnt.push_back((uint32_t)p.size());
      f.ev.insert(f.ev.end(), p.begin(), p.end());
      f.words = std::max<size_t>(f.words, (p.size() + 63) / 64);
    }
    if (f.ev.empty()) f.ev.resize(1);
    return f;
  }
  demi_handle* h = nullptr;
  std::vector<ExternalEvents> set_ext;         // the externals of each trace of the set (demi_set_traces)
  demi_fuzzer_config fz_cfg{};
  ExternalEvents fz_prefix, fz_postfix;
};

inline std::vector<uint64_t> mask_of(const ExternalEvents& all, const ExternalEvents& subseq) {
  std::vector<uint64_t> m((all.size() + 63) / 64 ? (all.size() + 63) / 64 : 1, 0);
  for (const demi_ext_event& s : subseq)
    for (size_t i = 0; i < all.size(); i++)
      if (all[i].id == s.id) { m[i >> 6] |= 1ull << (i & 63); break; }
  return m;
}
inline ExternalEvents events_of(const ExternalEvents& all, const std::vector<uint64_t>& mask) {
  ExternalEvents out;
  for (size_t i = 0; i < all.size(); i++) if ((mask[i >> 6] >> (i & 63)) & 1ull) out.push_back(all[i]);
  return out;
}

class RandomScheduler {
 public:
  RandomScheduler(const SchedulerConfig& cfg, uint32_t max_executions = 1, int32_t invariant_check_interval = 0,
                  int64_t seed = 0, std::shared_ptr<Engine> e = nullptr)
      : engine(e ? e : std::make_shared<Engine>(cfg)), max_executions(max_executions),
        invariant_check_interval(invariant_check_interval), seed(seed) {}
  std::string getName() const { return "RandomScheduler"; }
  void setMaxMessages(int32_t n) { maxMessages = n; }
  void setInvariant(bool have) { have_invariant = have; }          // models carry their invariant
  // Some((trace, fingerprint)) of the first violating execution, else nullopt (RandomScheduler.scala:234-272)
  std::optional<std::pair<EventTrace, ViolationFingerprint>> explore(const ExternalEvents& trace,
                                                                     ViolationFingerprint lookingFor = 0) {
    if (!have_invariant) throw std::invalid_argument("Must invoke setInvariant before test()");   // :244-246
    engine->check(demi_set_externals(engine->handle(), trace.data(), (uint32_t)trace.size()));
    demi_fuzz_params p{seed, max_executions, maxMessages, invariant_check_interval, lookingFor, 0};
    results.assign(max_executions, demi_fuzz_result{});
    engine->check(demi_fuzz_batch(engine->handle(), &p, results.data()));
    if (stats) stats->increment_replays(max_executions);
    for (uint32_t i = 0; i < max_executions; i++) {
      if (results[i].status) throw Error(DEMI_ERR_CAPACITY, "a prefix overflowed an engine structure");
      if (!results[i].violation) continue;
      EventTrace ev(65536);
      uint32_t n_ev = 0, n_nodes = 0;
      demi_fuzz_result r{};
      depGraph.assign(65536, 0);
      engine->check(demi_fuzz_trace(engine->handle(), &p, seed + i, ev.data(), (uint32_t)ev.size(), &n_ev,
                                    depGraph.data(), (uint32_t)depGraph.size(), &n_nodes, &r));
      ev.resize(n_ev); depGraph.resize(n_nodes);
      // ViolationFingerprint.affectedNodes of the execution found (TestOracle.scala:9-18)
      uint32_t which = i; uint64_t keep[32]; demi_provenance_out po{};
      if (maxMessages >= 0 && maxMessages + 2 <= 32 * 64) {
        engine->check(demi_fuzz_provenance(engine->handle(), &p, &which, 1, keep, 32, &po, nullptr));
        affectedNodes = po.affected_mask;
      }
      return std::make_pair(ev, r.violation);
    }
    return std::nullopt;
  }
  // TestOracle.test: Some(trace) iff the violation was reproduced (RandomScheduler.scala:597-612)
  std::optional<EventTrace> test(const ExternalEvents& events, ViolationFingerprint fp, MinimizationStats* s = nullptr) {
    stats = s;
    auto r = explore(events, fp);
    if (!r) return std::nullopt;
    return r->first;
  }
  std::shared_ptr<Engine> engine;
  std::vector<demi_fuzz_result> results;
  std::vector<uint16_t> depGraph;      // depTracker.getGraph of the violating execution, as parent pointers
  uint32_t affectedNodes = 0;          // ... and its fingerprint's affectedNodes
  // the test parameters DDMin uses when this scheduler is its oracle: N = max_executions, execution j under seed + j
  demi_fuzz_params test_params(ViolationFingerprint fp) const {
    return demi_fuzz_params{seed, max_executions, maxMessages, invariant_check_interval, fp, 0};
  }
  int64_t getSeed() const { return seed; }
  int32_t getInvariantCheckInterval() const { return invariant_check_interval; }
 private:
  uint32_t max_executions; int32_t invariant_check_interval; int64_t seed;
  int32_t maxMessages = -1;                                           // Int.MaxValue (:54)
  bool have_invariant = true;
  MinimizationStats* stats = nullptr;
};

class STSScheduler {
 public:
  STSScheduler(const SchedulerConfig& cfg, const EventTrace& original_trace, const ExternalEvents& original_externals,
               bool allowPeek = false, std::shared_ptr<Engine> e = nullptr)
      : engine(e ? e : std::make_shared<Engine>(cfg)), original_trace(original_trace), original_externals(original_externals),
        flags(cfg.filterKnownAbsents ? DEMI_RF_FILTER_KNOWN_ABSENTS : 0) {
    if (allowPeek) throw std::invalid_argument("STSSched with Peek is outside the accelerated path");
    if (original_trace.empty()) throw std::invalid_argument("original_trace must not be empty");     // assume(:203)
    engine->check(demi_set_trace(engine->handle(), original_trace.data(), (uint32_t)original_trace.size(),
                                 original_externals.data(), (uint32_t)original_externals.size()));
  }
  std::string getName() const { return "STSSchedNoPeek"; }
  uint32_t mask_words() const { return (uint32_t)((original_externals.size() + 63) / 64 ? (original_externals.size() + 63) / 64 : 1); }
  // Some(recorded trace) iff the violation was reproduced (STSScheduler.scala:199-310)
  std::optional<EventTrace> test(const ExternalEvents& subseq, ViolationFingerprint fp, MinimizationStats* stats = nullptr) {
    if (stats) stats->increment_replays();
    std::vector<uint64_t> m = mask_of(original_externals, subseq);
    EventTrace ev(65536);
    uint32_t n = 0; demi_replay_result r{};
    engine->check(demi_replay_trace(engine->handle(), m.data(), mask_words(), 0xFFFFFFFFu, fp, flags, ev.data(),
                                    (uint32_t)ev.size(), &n, &r));
    if (r.status) throw Error(DEMI_ERR_CAPACITY, "replay reported a capacity status");
    if (!r.violation) return std::nullopt;
    ev.resize(n);
    return ev;
  }
  std::vector<demi_replay_result> test_batch(const std::vector<std::vector<uint64_t>>& masks, ViolationFingerprint fp) {
    std::vector<uint64_t> flat;
    for (auto& m : masks) flat.insert(flat.end(), m.begin(), m.end());
    std::vector<demi_replay_result> out(masks.size());
    engine->check(demi_replay_batch(engine->handle(), flat.data(), (uint32_t)masks.size(), mask_words(), fp, flags, out.data()));
    return out;
  }
  std::shared_ptr<Engine> engine;
  const EventTrace original_trace;
  const ExternalEvents original_externals;
  const uint32_t flags;
};

class ReplayScheduler : public STSScheduler {
 public:
  using STSScheduler::STSScheduler;
  // strict replay of the recorded trace; throws ReplayException on divergence (ReplayScheduler.scala:71-140)
  demi_replay_result replay(ViolationFingerprint fp = 0) {
    std::vector<uint64_t> m = mask_of(original_externals, original_externals);
    demi_replay_result r{};
    engine->check(demi_replay_batch(engine->handle(), m.data(), 1, mask_words(), fp, flags | DEMI_RF_STRICT, &r));
    if (r.status == DEMI_RS_DIVERGED) throw ReplayException("Expected event not pending after " + std::to_string(r.delivered) + " deliveries");
    if (r.status) throw Error(DEMI_ERR_CAPACITY, "replay reported a capacity status");
    return r;
  }
};

class DDMin {
 public:
  DDMin(STSScheduler& oracle, bool checkUnmodifed = false, MinimizationStats* stats = nullptr)
      : _stats(stats ? stats : &own), oracle(&oracle), checkUnmodifed(checkUnmodifed) {}
  // RunnerUtils.randomDDMin's DDMin (RunnerUtils.scala:601-623): a RandomScheduler as the TestOracle
  DDMin(RandomScheduler& oracle, bool checkUnmodifed = false, MinimizationStats* stats = nullptr)
      : _stats(stats ? stats : &own), random(&oracle), checkUnmodifed(checkUnmodifed) {}
  // the MCS (WaitQuiescence dropped, RunnerUtils.scala:678-684); throws std::invalid_argument
  // ("Unmodified trace does not trigger violation") like DeltaDebugging.scala:41-47
  ExternalEvents minimize(ViolationFingerprint fp) {
    if (!oracle) throw std::invalid_argument("DDMin over a RandomScheduler minimizes the events it is given");
    std::vector<uint64_t> mcs(oracle->mask_words(), 0);
    std::vector<uint32_t> iters(1 << 16);
    oracle->engine->check(demi_ddmin(oracle->engine->handle(), fp, oracle->flags, checkUnmodifed ? 1 : 0, mcs.data(),
                                     oracle->mask_words(), iters.data(), (uint32_t)iters.size(), &last));
    _stats->iteration_size.clear();
    _stats->record_series(iters.data(), last.n_iterations, false);
    _stats->total_replays_ref() = last.total_replays;
    return events_of(oracle->original_externals, mcs);
  }
  // over a RandomScheduler: the whole program `events`, WaitQuiescence included (demi_random_ddmin).  MinimizationStats
  // counts executions: each iteration size is keyed by the running sum of the executions the tests ran.
  ExternalEvents minimize(ViolationFingerprint fp, const ExternalEvents& events) {
    if (!random) return minimize(fp);
    Engine& e = *random->engine;
    e.check(demi_set_externals(e.handle(), events.data(), (uint32_t)events.size()));
    const uint32_t mw = events.size() ? (uint32_t)((events.size() + 63) / 64) : 1u;
    std::vector<uint64_t> mcs(mw, 0), keys(1 << 16);
    std::vector<uint32_t> sizes(1 << 16);
    const demi_fuzz_params p = random->test_params(fp);
    e.check(demi_random_ddmin(e.handle(), &p, checkUnmodifed ? 1 : 0, mcs.data(), mw, sizes.data(), keys.data(),
                              (uint32_t)sizes.size(), &last_random));
    _stats->updateStrategy("DDMin", random->getName());
    const uint32_t base = _stats->total_replays_ref();
    const uint32_t n = std::min<uint32_t>(last_random.n_iterations, (uint32_t)sizes.size());
    for (uint32_t i = 0; i < n; i++) {
      _stats->total_replays_ref() = base + (uint32_t)keys[i];
      _stats->record_iteration_size(sizes[i]);
    }
    _stats->total_replays_ref() = base + (uint32_t)last_random.total_replays;
    return events_of(events, mcs);
  }
  std::optional<EventTrace> verify_mcs(const ExternalEvents& mcs, ViolationFingerprint fp) {
    if (random) return random->test(mcs, fp);
    return oracle->test(mcs, fp);
  }
  demi_ddmin_out last{};
  demi_random_ddmin_out last_random{};
  MinimizationStats* _stats;
 private:
  STSScheduler* oracle = nullptr;
  RandomScheduler* random = nullptr;
  bool checkUnmodifed; MinimizationStats own;
};

// RunnerUtils.randomDDMin (RunnerUtils.scala:601-623) on a recorded experiment: DDMin(RandomScheduler(cfg,
// max_executions, seed), checkUnmodifed = false) with setMaxMessages(trace.size).  Returns (MCS, stats, verified trace,
// violation); the verified trace is the EventTrace of the MCS's first violating execution (nullopt when it does not
// reproduce), or `trace` itself when nothing was pruned.  Execution j of every test runs FullyRandom(seed + j).
struct RandomDDMinResult {
  ExternalEvents mcs; MinimizationStats stats; std::optional<EventTrace> verified; ViolationFingerprint violation;
  demi_random_ddmin_out out;
};
inline RandomDDMinResult randomDDMin(const SchedulerConfig& cfg, const EventTrace& trace, const ExternalEvents& externals,
                                     ViolationFingerprint violation, uint32_t max_executions = 1, int64_t seed = 0,
                                     std::shared_ptr<Engine> engine = nullptr) {
  RandomScheduler sched(cfg, max_executions, 0, seed, engine);
  sched.setMaxMessages((int32_t)trace.size());
  RandomDDMinResult r;
  DDMin ddmin(sched, false, &r.stats);
  r.mcs = ddmin.minimize(violation, externals);
  r.out = ddmin.last_random;
  r.violation = violation;
  if (r.mcs.size() >= externals.size()) { r.verified = trace; return r; }
  if (!r.out.verified) return r;
  const std::vector<uint64_t> m = mask_of(externals, r.mcs);
  const demi_fuzz_params p = sched.test_params(violation);
  EventTrace ev(65536);
  uint32_t n = 0; demi_fuzz_result res{};
  sched.engine->check(demi_random_test_trace(sched.engine->handle(), m.data(), (uint32_t)m.size(), &p,
                                             seed + r.out.mcs_first_hit, ev.data(), (uint32_t)ev.size(), &n, &res));
  ev.resize(n);
  r.verified = ev;
  return r;
}

struct LeftToRightOneAtATime {};       // RemovalStrategy (OneAtATimeRemoval.scala:131-137)
struct SrcDstFIFORemoval {};           // RemovalStrategy (OneAtATimeRemoval.scala:139-251)

class STSSchedMinimizer {
 public:
  STSSchedMinimizer(const ExternalEvents& mcs, const EventTrace& verified_mcs, ViolationFingerprint violation,
                    LeftToRightOneAtATime, const SchedulerConfig& cfg, std::shared_ptr<Engine> e = nullptr)
      : engine(e ? e : std::make_shared<Engine>(cfg)), mcs(mcs), verified_mcs(verified_mcs), violation(violation),
        flags(cfg.filterKnownAbsents ? DEMI_RF_FILTER_KNOWN_ABSENTS : 0) {}
  STSSchedMinimizer(const ExternalEvents& mcs, const EventTrace& verified_mcs, ViolationFingerprint violation,
                    SrcDstFIFORemoval, const SchedulerConfig& cfg, std::shared_ptr<Engine> e = nullptr)
      : engine(e ? e : std::make_shared<Engine>(cfg)), mcs(mcs), verified_mcs(verified_mcs), violation(violation),
        flags((cfg.filterKnownAbsents ? DEMI_RF_FILTER_KNOWN_ABSENTS : 0) | DEMI_IM_SRC_DST_FIFO) {}
  std::pair<MinimizationStats, EventTrace> minimize() {
    engine->check(demi_set_trace(engine->handle(), verified_mcs.data(), (uint32_t)verified_mcs.size(), mcs.data(), (uint32_t)mcs.size()));
    EventTrace out(65536); std::vector<uint32_t> sizes(65536);
    engine->check(demi_internal_minimize(engine->handle(), violation, flags, out.data(), (uint32_t)out.size(), sizes.data(),
                                         (uint32_t)sizes.size(), &last));
    out.resize(last.n_events);
    MinimizationStats s;
    s.total_replays_ref() = last.total_replays;
    s.internal_size.clear();
    s.record_series(sizes.data(), last.n_internal_sizes, true);
    return {s, out};
  }
  demi_intmin_out last{};
 private:
  std::shared_ptr<Engine> engine; ExternalEvents mcs; EventTrace verified_mcs; ViolationFingerprint violation; uint32_t flags;
};

// ---- fungible clocks (minification/wildcard_minimization/)
// FingerprintFactory.getLogicalClock / causesClockIncrement as data (demi_set_clock_rules): packed rules + the
// clock-incrementing message types.
struct ClockRules { std::vector<uint32_t> rules; std::vector<uint32_t> increment_types; };
// raft5: the term is p0 & 0xFF of RequestVote, VoteReply, AppendEntries and AppendReply; ElectionTick increments it
// (the hint at ClockClusterizer.scala:24-27).
inline ClockRules raft5_clock_rules() {
  return ClockRules{{DEMI_CLOCK_RULE(4, 0, 0, 8), DEMI_CLOCK_RULE(5, 0, 0, 8), DEMI_CLOCK_RULE(7, 0, 0, 8),
                     DEMI_CLOCK_RULE(8, 0, 0, 8)}, {3}};
}
struct BackTrackStrategy {};           // AmbiguityResolutionStrategy (AmbiguityResolutionStrategies.scala:44-75)
struct LastOnlyStrategy {};            // (:109-117)
enum class TestScheduler { STSSched, DPORwHeuristics };                                   // WildcardMinimizer.scala:21-27
enum class ClusteringStrategy { ClockClusterizer, SingletonClusterizer, ClockThenSingleton };   // :31-36

// WildcardMinimizer(schedulerConfig, mcs, trace, violation, ...) (WildcardMinimizer.scala:47-241) with
// testScheduler = STSSched and ClockClusterizer: runTheGamut's WildcardsNoBackTracks / WildcardsLastOnly
// (RunnerUtils.scala:413-440).  The other test schedulers and clusterizers, and skipClockClusters, are outside the
// accelerated path and throw std::invalid_argument.
class WildcardMinimizer {
 public:
  template <class Strategy = BackTrackStrategy>
  WildcardMinimizer(const SchedulerConfig& cfg, const ExternalEvents& mcs, const EventTrace& trace, ViolationFingerprint violation,
                    ClockRules rules, Strategy = Strategy(), TestScheduler ts = TestScheduler::STSSched,
                    ClusteringStrategy cs = ClusteringStrategy::ClockClusterizer, bool skipClockClusters = false,
                    std::shared_ptr<Engine> e = nullptr)
      : mcs(mcs), trace(trace), violation(violation), rules(std::move(rules)),
        flags((cfg.filterKnownAbsents ? DEMI_RF_FILTER_KNOWN_ABSENTS : 0) |
              (std::is_same<Strategy, LastOnlyStrategy>::value ? DEMI_WC_LAST_ONLY : 0)) {
    static_assert(std::is_same<Strategy, BackTrackStrategy>::value || std::is_same<Strategy, LastOnlyStrategy>::value,
                  "BackTrackStrategy and LastOnlyStrategy are the accelerated resolution strategies");
    if (ts != TestScheduler::STSSched) throw std::invalid_argument("DPORwHeuristics as the test scheduler is outside the accelerated path");
    if (cs != ClusteringStrategy::ClockClusterizer) throw std::invalid_argument("only ClockClusterizer is on the accelerated path");
    if (skipClockClusters) throw std::invalid_argument("skipClockClusters is outside the accelerated path");
    engine = e ? e : std::make_shared<Engine>(cfg);
  }
  std::pair<MinimizationStats, EventTrace> minimize() {
    engine->check(demi_set_trace(engine->handle(), trace.data(), (uint32_t)trace.size(), mcs.data(), (uint32_t)mcs.size()));
    uint32_t incr[8] = {};
    for (uint32_t t : rules.increment_types) incr[(t & 0xFF) >> 5] |= 1u << (t & 31);
    engine->check(demi_set_clock_rules(engine->handle(), rules.rules.data(), (uint32_t)rules.rules.size(), incr));
    EventTrace out(65536); std::vector<uint32_t> sizes(65536);
    engine->check(demi_wildcard_minimize(engine->handle(), violation, flags, out.data(), (uint32_t)out.size(), sizes.data(),
                                         (uint32_t)sizes.size(), &last));
    out.resize(last.n_events);
    MinimizationStats s;
    s.updateStrategy("FungibleClockMinimizer", "STSSched");                   // WildcardMinimizer.scala:141
    s.record_series(sizes.data(), last.n_internal_sizes, true);               // :210-212 and the fencepost :184
    s.total_replays_ref() = last.total_replays;
    return {s, out};
  }
  demi_intmin_out last{};
 private:
  std::shared_ptr<Engine> engine; ExternalEvents mcs; EventTrace trace; ViolationFingerprint violation; ClockRules rules;
  uint32_t flags;
};

// ProvenanceTracker(trace, depGraph) (schedulers/Util.scala:267-376): `trace` is the recorded EventTrace of an
// execution, `dep_parent` its DepTracker tree, both as returned by demi_fuzz_trace.
class ProvenanceTracker {
 public:
  ProvenanceTracker(std::shared_ptr<Engine> e, EventTrace trace, std::vector<uint16_t> dep_parent)
      : engine(std::move(e)), trace(std::move(trace)), dep_parent(std::move(dep_parent)) {}
  // pruneConcurrentEvents(violation): the deliveries of `trace` (by index into it) that stay; the root event,
  // which the reference filters out afterwards (EventTrace.intersection, EventTrace.scala:127-131), is not listed
  std::vector<uint32_t> pruneConcurrentEvents(uint32_t affectedNodes) {
    std::vector<uint32_t> delivery_index;
    for (uint32_t i = 0; i < trace.size(); i++) if (trace[i].kind == DEMI_EV_MSG_EVENT) delivery_index.push_back(i);
    const uint32_t words = (uint32_t)((delivery_index.size() + 1 + 63) / 64);
    std::vector<uint64_t> keep(words, 0);
    engine->check(demi_provenance(engine->handle(), trace.data(), (uint32_t)trace.size(), dep_parent.data(),
                                  (uint32_t)dep_parent.size(), affectedNodes, keep.data(), words, &last));
    if (last.status == DEMI_PV_CYCLE) throw std::runtime_error("happens-before relation is cyclic");   // Util.scala:506
    if (last.status) throw Error(DEMI_ERR_CAPACITY, "provenance: trace does not fit");
    std::vector<uint32_t> kept;
    for (uint32_t t = 1; t <= delivery_index.size(); t++)
      if ((keep[t >> 6] >> (t & 63)) & 1ull) kept.push_back(delivery_index[t - 1]);
    return kept;
  }
  demi_provenance_out last{};
 private:
  std::shared_ptr<Engine> engine;
  EventTrace trace;
  std::vector<uint16_t> dep_parent;
};

// RunnerUtils.fuzz (RunnerUtils.scala:62-147), the mirror of demi_b200.fuzz (schedulers.py), with the same deviations:
// it stops after max_executions (nullopt), execution i draws its program with seed program_seed_base + i (default
// seed_base + 2^32, so that the Fuzzer's and FullyRandom's java.util.Random streams differ) and runs under
// FullyRandom(seed_base + i), and an execution that overflows an engine capacity is passed over.  As written:
// executions stop at their first violation of any kind, the predicate filters on the host, the first accepted
// execution in index order is re-generated and recorded (demi_fuzz_trace); with validate_replay it must replay
// strictly and end in a violation (replayer.violationAtEnd non-empty, :106-109), else the loop goes on; with
// computeProvenance `filtered` holds the deliveries ProvenanceTracker keeps.
struct FuzzFound {
  EventTrace trace;
  ViolationFingerprint violation = 0;
  std::vector<uint16_t> depGraph;          // DepTracker tree as parent pointers
  std::vector<uint16_t> initialTrace;      // DepTracker.getInitialTrace: the root, then each delivery's node
  EventTrace filtered;                     // computeProvenance: the deliveries that stay
  ExternalEvents externals;                // the program (fuzzTest)
  uint64_t execution = 0;
};
constexpr int64_t PROGRAM_SEED_OFFSET = 1ll << 32;
inline std::optional<FuzzFound> fuzz(const demi_fuzzer_config& fuzzer, const ExternalEvents& prefix, const ExternalEvents& postfix,
                                     const SchedulerConfig& cfg, bool validate_replay = false, int32_t invariant_check_interval = 30,
                                     std::optional<int32_t> maxMessages = std::nullopt, bool computeProvenance = false,
                                     std::function<bool(ViolationFingerprint)> violationWereLookingFor = nullptr,
                                     uint64_t max_executions = 100000, int64_t seed_base = 0,
                                     std::optional<int64_t> program_seed_base = std::nullopt,
                                     std::shared_ptr<Engine> e = nullptr, uint64_t chunk = 1u << 16) {
  if (computeProvenance && !maxMessages)
    throw std::invalid_argument("computeProvenance needs maxMessages (the pruning mask covers maxMessages + 2 deliveries)");
  std::shared_ptr<Engine> eng = e ? e : std::make_shared<Engine>(cfg);
  eng->set_fuzzer(fuzzer, prefix, postfix);
  const int64_t pbase = program_seed_base ? *program_seed_base : seed_base + PROGRAM_SEED_OFFSET;
  const int32_t mm = maxMessages ? *maxMessages : -1;
  for (uint64_t done = 0; done < max_executions;) {
    const uint64_t n = std::min(chunk, max_executions - done);
    const std::vector<demi_fuzz_result> res =
        eng->fuzz_campaign(seed_base + (int64_t)done, n, mm, invariant_check_interval, pbase + (int64_t)done);
    for (uint64_t i = 0; i < n; i++) {
      if (res[i].status || !res[i].violation) continue;
      const ViolationFingerprint v = res[i].violation;
      if (violationWereLookingFor && !violationWereLookingFor(v)) continue;
      const uint64_t k = done + i;
      FuzzFound f;
      f.externals = eng->fuzzer_program(pbase + (int64_t)k);
      f.execution = k; f.violation = v;
      eng->check(demi_set_externals(eng->handle(), f.externals.data(), (uint32_t)f.externals.size()));
      demi_fuzz_params p{seed_base + (int64_t)k, 1, mm, invariant_check_interval, 0, 0};
      f.trace.resize(65536); f.depGraph.resize(65536);
      uint32_t n_ev = 0, n_nodes = 0; demi_fuzz_result r{};
      eng->check(demi_fuzz_trace(eng->handle(), &p, seed_base + (int64_t)k, f.trace.data(), (uint32_t)f.trace.size(), &n_ev,
                                 f.depGraph.data(), (uint32_t)f.depGraph.size(), &n_nodes, &r));
      f.trace.resize(n_ev); f.depGraph.resize(n_nodes);
      if (validate_replay) {
        bool deterministic = true;
        try {
          ReplayScheduler replayer(cfg, f.trace, f.externals, false, eng);
          deterministic = replayer.replay(0).violation != 0;
        } catch (const ReplayException&) { deterministic = false; }
        if (!deterministic) continue;
      }
      f.initialTrace.push_back(0);
      for (const demi_event& x : f.trace) if (x.kind == DEMI_EV_MSG_EVENT) f.initialTrace.push_back(x.node);
      if (computeProvenance) {
        eng->check(demi_set_externals(eng->handle(), f.externals.data(), (uint32_t)f.externals.size()));
        const uint32_t words = (uint32_t)((mm + 2 + 63) / 64), which = 0;
        std::vector<uint64_t> keep(words);
        demi_provenance_out po{};
        eng->check(demi_fuzz_provenance(eng->handle(), &p, &which, 1, keep.data(), words, &po, nullptr));
        ProvenanceTracker pt(eng, f.trace, f.depGraph);
        for (uint32_t idx : pt.pruneConcurrentEvents(po.affected_mask)) f.filtered.push_back(f.trace[idx]);
      }
      return f;
    }
    done += n;
  }
  return std::nullopt;
}

class DPORwHeuristics {
 public:
  DPORwHeuristics(const SchedulerConfig& cfg, int32_t depth_bound = -1, bool stopIfViolationFound = true,
                  uint32_t max_interleavings = 1000, std::shared_ptr<Engine> e = nullptr)
      : engine(e ? e : std::make_shared<Engine>(cfg)), depth_bound(depth_bound), stop(stopIfViolationFound), budget(max_interleavings) {}
  std::string getName() const { return "DPORwHeuristics"; }
  void setMaxMessagesToSchedule(int32_t n) { max_messages = n; }
  void setDepthBound(int32_t d) { depth_bound = d; }
  // the first violating interleaving, or nullopt (DPORwHeuristics.scala:1193-1242)
  std::optional<demi_dpor_violation> test(const ExternalEvents& events, ViolationFingerprint fp, MinimizationStats* stats = nullptr) {
    if (max_messages < 0) throw std::invalid_argument("setMaxMessagesToSchedule is required");
    ExternalEvents prog;                                              // convertToDPORTrace (:1279-1303)
    for (const demi_ext_event& e : events) if (e.kind == DEMI_EXT_START || e.kind == DEMI_EXT_SEND) prog.push_back(e);
    uint32_t offs[2] = {0, (uint32_t)prog.size()};
    demi_dpor_params P{max_messages, depth_bound, budget, fp, stop ? 1u : 0u, 4096, 1u << 16, 1u << 15};
    demi_dpor_violation v[8]{};
    engine->check(demi_dpor_batch(engine->handle(), prog.data(), offs, 1, &P, &last, v, 8, nullptr, 0));
    if (stats) stats->increment_replays(last.interleavings);
    if (last.status) throw Error(DEMI_ERR_CAPACITY, "DPOR search reported a capacity status");
    if (!last.violations) return std::nullopt;
    return v[0];
  }
  demi_dpor_result last{};
 private:
  std::shared_ptr<Engine> engine; int32_t depth_bound; bool stop; uint32_t budget; int32_t max_messages = -1;
};

// ResumableDPOR (minification/IncrementalDeltaDebugging.scala:90-122) in RunnerUtils.editDistanceDporDDMin's
// configuration (RunnerUtils.scala:822-835): every instance starts from the recorded execution's dependency graph
// and trace, orders backtrack points by ArvindDistanceOrdering and prioritises pending messages on divergence.
// An instance's state is a function of the caps it has been tested with; that list is what is kept per subsequence.
class ResumableDPOR {
 public:
  ResumableDPOR(const SchedulerConfig& cfg, EventTrace trace, std::vector<uint16_t> depGraph, int32_t max_messages,
                uint32_t max_interleavings = 1000, std::shared_ptr<Engine> e = nullptr,
                uint32_t flags = DEMI_DF_ARVIND_ORDERING | DEMI_DF_PRIORITIZE_PENDING)
      : engine(e ? e : std::make_shared<Engine>(cfg)), trace(std::move(trace)), depGraph(std::move(depGraph)),
        max_messages(max_messages), budget(max_interleavings), flags(flags) {}
  std::string getName() const { return "DPOR"; }
  void setMaxDistance(int32_t d) { currentMaxDistance = d; }
  demi_dpor_seed seed() const { return demi_dpor_seed{trace.data(), (uint32_t)trace.size(), depGraph.data(), (uint32_t)depGraph.size()}; }
  demi_dpor_params params(ViolationFingerprint fp) const { return demi_dpor_params{max_messages, -1, budget, fp, 1u, 4096, 1u << 16, 1u << 16}; }
  // Some(trace) <=> true (:102-121)
  bool test(const ExternalEvents& events, ViolationFingerprint fp, MinimizationStats* stats = nullptr) {
    ExternalEvents prog; std::vector<uint32_t> key;
    for (const demi_ext_event& e : events) if (e.kind == DEMI_EXT_START || e.kind == DEMI_EXT_SEND) { prog.push_back(e); key.push_back(e.id); }
    std::vector<int32_t>& caps = subseqToDPOR[key];
    caps.push_back(currentMaxDistance);
    const uint32_t offs[2] = {0, (uint32_t)prog.size()}, coffs[2] = {0, (uint32_t)caps.size()};
    const demi_dpor_seed sd = seed();
    const demi_dpor_params P = params(fp);
    const demi_dpor_ex ex{flags, &sd, caps.data(), coffs};
    engine->check(demi_dpor_batch_ex(engine->handle(), prog.data(), offs, 1, &P, &ex, &last, nullptr, 0, nullptr, 0));
    if (last.status) throw Error(DEMI_ERR_CAPACITY, "DPOR instance reported a capacity status");
    if (stats) stats->increment_replays();
    return last.violations != 0;
  }
  std::shared_ptr<Engine> engine;
  demi_dpor_result last{};
  uint32_t flags_value() const { return flags; }
 private:
  EventTrace trace; std::vector<uint16_t> depGraph; int32_t max_messages; uint32_t budget, flags;
  int32_t currentMaxDistance = 0;
  std::map<std::vector<uint32_t>, std::vector<int32_t>> subseqToDPOR;
};

// IncrementalDDMin(oracle, maxMaxDistance, stopAtSize) (minification/IncrementalDeltaDebugging.scala:20-88)
class IncrementalDDMin {
 public:
  IncrementalDDMin(ResumableDPOR& oracle, int32_t maxMaxDistance = 256, uint32_t stopAtSize = 1, MinimizationStats* stats = nullptr)
      : oracle(oracle), maxMaxDistance(maxMaxDistance), stopAtSize(stopAtSize), stats(stats) {}
  ExternalEvents minimize(const ExternalEvents& events, ViolationFingerprint fp) {
    ExternalEvents prog;
    for (const demi_ext_event& e : events) if (e.kind == DEMI_EXT_START || e.kind == DEMI_EXT_SEND) prog.push_back(e);
    std::vector<uint64_t> mcs((prog.size() + 63) / 64 ? (prog.size() + 63) / 64 : 1, 0);
    const demi_dpor_seed sd = oracle.seed();
    const demi_dpor_params P = oracle.params(fp);
    oracle.engine->check(demi_incremental_ddmin(oracle.engine->handle(), prog.data(), (uint32_t)prog.size(), &P, oracle.flags_value(),
                                                &sd, maxMaxDistance, stopAtSize, mcs.data(), (uint32_t)mcs.size(), &last));
    if (stats) stats->increment_replays(last.total_replays);
    return events_of(prog, mcs);
  }
  // minimize() on many violating executions in one call (demi_incremental_ddmin_many): execution t is programs[t] recorded
  // as traces[t] with DepTracker tree trees[t] and setMaxMessagesToSchedule max_messages[t]; the oracle's engine, budget
  // and flags apply to every one.  status[t] is its return code (a failed execution's MCS is empty), outs[t] its counters.
  std::vector<ExternalEvents> minimize_many(const std::vector<ExternalEvents>& programs, const std::vector<EventTrace>& traces,
                                            const std::vector<std::vector<uint16_t>>& trees, const std::vector<int32_t>& max_messages,
                                            ViolationFingerprint fp, std::vector<int32_t>* status = nullptr,
                                            std::vector<demi_incddmin_out>* outs = nullptr) {
    const size_t n = programs.size();
    ExternalEvents flat; std::vector<uint32_t> off, cnt, lf(n, fp);
    std::vector<demi_dpor_seed> seeds(n);
    size_t words = 1;
    for (size_t t = 0; t < n; t++) {
      off.push_back((uint32_t)flat.size());
      uint32_t k = 0;
      for (const demi_ext_event& e : programs[t]) if (e.kind == DEMI_EXT_START || e.kind == DEMI_EXT_SEND) { flat.push_back(e); k++; }
      cnt.push_back(k);
      words = std::max<size_t>(words, (k + 63) / 64);
      seeds[t] = demi_dpor_seed{traces[t].data(), (uint32_t)traces[t].size(), trees[t].data(), (uint32_t)trees[t].size()};
    }
    const demi_dpor_params P = oracle.params(fp);
    std::vector<uint64_t> mcs(n * words, 0);
    std::vector<demi_incddmin_out> out(n);
    std::vector<int32_t> st(n);
    oracle.engine->check(demi_incremental_ddmin_many(oracle.engine->handle(), (uint32_t)n, flat.data(), off.data(), cnt.data(),
                                                     seeds.data(), max_messages.data(), lf.data(), &P, oracle.flags_value(),
                                                     maxMaxDistance, stopAtSize, mcs.data(), (uint32_t)words, out.data(), st.data()));
    std::vector<ExternalEvents> res(n);
    for (size_t t = 0; t < n; t++) {
      if (st[t] != DEMI_OK) continue;
      if (stats) stats->increment_replays(out[t].total_replays);
      ExternalEvents prog(flat.begin() + off[t], flat.begin() + off[t] + cnt[t]);
      res[t] = events_of(prog, std::vector<uint64_t>(mcs.begin() + t * words, mcs.begin() + (t + 1) * words));
    }
    if (status) *status = st;
    if (outs) *outs = out;
    return res;
  }
  bool verify_mcs(const ExternalEvents& mcs, ViolationFingerprint fp) { return oracle.test(mcs, fp); }
  demi_incddmin_out last{};
 private:
  ResumableDPOR& oracle; int32_t maxMaxDistance; uint32_t stopAtSize; MinimizationStats* stats;
};

// Fuzzer (Fuzzer.scala:24-194): seeded generation of external-event programs.
struct FuzzerWeights { double kill = 0.01, send = 0.3, wait_quiescence = 0.1, partition = 0.1, unpartition = 0.1; };
class Fuzzer {
 public:
  Fuzzer(uint32_t num_events, FuzzerWeights w, uint32_t send_type, ExternalEvents prefix = {}, ExternalEvents postfix = {})
      : num_events(num_events), weights(w), send_type(send_type), prefix(std::move(prefix)), postfix(std::move(postfix)) {}
  ExternalEvents generateFuzzTest(int64_t seed) const {
    demi_fuzzer_config c{weights.kill, weights.send, weights.wait_quiescence, weights.partition, weights.unpartition, num_events, send_type};
    ExternalEvents out(prefix.size() + postfix.size() + 2 * (size_t)num_events + 8);
    uint32_t n = 0;
    int32_t rc = demi_fuzzer_generate(&c, seed, prefix.data(), (uint32_t)prefix.size(), postfix.data(), (uint32_t)postfix.size(),
                                      out.data(), (uint32_t)out.size(), &n);
    if (rc != DEMI_OK) throw Error(rc, demi_last_error(nullptr));
    out.resize(n);
    return out;
  }
 private:
  uint32_t num_events; FuzzerWeights weights; uint32_t send_type; ExternalEvents prefix, postfix;
};

// The flat experiment directory that replaces ExperimentSerializer / ExperimentDeserializer (Serialization.scala:57-254).
struct Experiment {
  int32_t model = 0; uint32_t model_flags = 0; ViolationFingerprint violation = 0;
  ExternalEvents externals; EventTrace trace; std::vector<uint16_t> dep_parent; std::vector<uint64_t> mcs_mask;
  void save(const std::string& dir) const {
    demi_experiment e{};
    e.model = model; e.model_flags = model_flags; e.violation = violation;
    e.externals = const_cast<demi_ext_event*>(externals.data()); e.n_externals = (uint32_t)externals.size();
    e.events = const_cast<demi_event*>(trace.data()); e.n_events = (uint32_t)trace.size();
    e.dep_parent = const_cast<uint16_t*>(dep_parent.data()); e.n_nodes = (uint32_t)dep_parent.size();
    e.mcs_mask = const_cast<uint64_t*>(mcs_mask.data()); e.mask_words = (uint32_t)mcs_mask.size();
    int32_t rc = demi_experiment_save(dir.c_str(), &e);
    if (rc != DEMI_OK) throw Error(rc, demi_last_error(nullptr));
  }
  static Experiment load(const std::string& dir) {
    Experiment x;
    demi_experiment e{};
    int32_t rc = demi_experiment_load(dir.c_str(), &e);                 // counts first
    if (rc != DEMI_OK && rc != DEMI_ERR_CAPACITY) throw Error(rc, demi_last_error(nullptr));
    x.externals.resize(e.n_externals); x.trace.resize(e.n_events); x.dep_parent.resize(e.n_nodes); x.mcs_mask.resize(e.mask_words);
    e.externals = x.externals.data(); e.cap_externals = e.n_externals; e.events = x.trace.data(); e.cap_events = e.n_events;
    e.dep_parent = x.dep_parent.data(); e.cap_nodes = e.n_nodes; e.mcs_mask = x.mcs_mask.data(); e.cap_mask_words = e.mask_words;
    rc = demi_experiment_load(dir.c_str(), &e);
    if (rc != DEMI_OK) throw Error(rc, demi_last_error(nullptr));
    x.model = e.model; x.model_flags = e.model_flags; x.violation = e.violation;
    return x;
  }
};

// ONE DPORwHeuristics.test as a frontier of backtrack points (demi_dpor_frontier); with several devices the frontier is
// sharded and rebalanced by the library's NCCL steal rounds (demi_create_multi + demi_dpor_frontier_multi).
class FrontierDPOR {
 public:
  explicit FrontierDPOR(const SchedulerConfig& cfg, std::vector<int32_t> devices = {}) {
    if (devices.empty()) devices.push_back(cfg.device);
    demi_config dc{};
    dc.device = devices[0]; dc.model = cfg.model; dc.model_flags = cfg.model_flags; dc.blocked_mask = cfg.blocked_mask;
    dc.ignore_timers = cfg.ignoreTimers ? 1 : 0; dc.strategy = cfg.strategy;
    hs.resize(devices.size(), nullptr);
    int32_t rc = devices.size() == 1 ? demi_create(&dc, &hs[0]) : demi_create_multi(&dc, devices.data(), (int32_t)devices.size(), hs.data());
    if (rc != DEMI_OK) throw Error(rc, demi_last_error(nullptr));
  }
  ~FrontierDPOR() { for (demi_handle* h : hs) demi_destroy(h); }
  FrontierDPOR(const FrontierDPOR&) = delete;
  FrontierDPOR& operator=(const FrontierDPOR&) = delete;
  demi_frontier_params params{/*max_messages*/100, 0, 0, /*width*/16384, /*max_interleavings*/1u << 20, /*explored_slots*/1u << 22,
                              /*pool_cap*/1u << 22, /*trace_cap (0: max_interleavings + slack)*/0, /*rounds_per_exchange*/4, /*steal_max*/4096, 0};
  void setMaxMessagesToSchedule(int32_t n) { params.max_messages = n; }
  void trackHistory(bool on) { params.flags = on ? (params.flags & ~DEMI_FR_NO_HISTORY) : (params.flags | DEMI_FR_NO_HISTORY); }
  // returns the violating interleavings found (all ranks); `results[r]` holds rank r's counters
  std::vector<demi_dpor_violation> test(const ExternalEvents& events, ViolationFingerprint fp, uint32_t cap_viol = 4096) {
    params.looking_for = fp;
    if (!params.trace_cap) params.trace_cap = (uint32_t)std::min<uint64_t>(params.max_interleavings + 8ull * params.steal_max + 16, (1u << 28) - 1);
    const size_t n = hs.size();
    results.assign(n, demi_frontier_result{});
    std::vector<demi_dpor_violation> viol(n * cap_viol);
    int32_t rc = n == 1 ? demi_dpor_frontier(hs[0], events.data(), (uint32_t)events.size(), &params, &results[0], viol.data(), cap_viol, nullptr, 0)
                        : demi_dpor_frontier_multi(hs.data(), (int32_t)n, events.data(), (uint32_t)events.size(), &params, results.data(),
                                                   viol.data(), cap_viol, nullptr, 0);
    if (rc != DEMI_OK) { std::string msg = demi_last_error(hs[0]); if (rc == DEMI_ERR_INVALID) throw std::invalid_argument(msg); throw Error(rc, msg); }
    std::vector<demi_dpor_violation> out;
    for (size_t r = 0; r < n; r++) {
      const uint64_t k = std::min<uint64_t>(results[r].violations, cap_viol);
      out.insert(out.end(), viol.begin() + r * cap_viol, viol.begin() + r * cap_viol + k);
    }
    return out;
  }
  uint64_t interleavings() const { uint64_t t = 0; for (auto& r : results) t += r.interleavings; return t; }
  std::vector<demi_frontier_result> results;
 private:
  std::vector<demi_handle*> hs;
};

}  // namespace demi
