// engine.hpp — the handle behind the C ABI, shared by capi.cu and capi_replay.cu.
#pragma once
#include <climits>
#include <cstdlib>
#include <cstdio>
#include <cstdarg>
#include <cstring>
#include <string>
#include <vector>
#include <map>
#include <algorithm>
#include <cuda_runtime.h>
#include "../../include/demi_b200.h"
#include "../../include/demi_limits.h"
#include "../../include/demi_model_ir.h"
#include "lane_steady.hpp"
#include "replay_trace.hpp"

extern thread_local std::string g_create_error;

struct demi_handle;
struct FrComm;                                     // the communicator (capi_frontier.cu)
struct FrCache;                                    // K3F's buffers and queue directory, kept between calls (capi_frontier.cu)
// A device allocation with one owner, which frees it: moved, never copied.  Every device buffer of the library is one.
class DevBuf {
 public:
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : p_(o.p_), bytes_(o.bytes_) { o.p_ = nullptr; o.bytes_ = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { reset(); std::swap(p_, o.p_); std::swap(bytes_, o.bytes_); }
    return *this;
  }
  ~DevBuf() { reset(); }
  void reset() { if (p_) cudaFree(p_); p_ = nullptr; bytes_ = 0; }
  // At least `bytes`: the buffer is kept when it is big enough, else freed and allocated anew.  On failure it is empty
  // and the call returns DEMI_ERR_CUDA through fail().
  int32_t grow(demi_handle* h, size_t bytes);
  // grow(bytes), then a synchronous copy of host `src`
  int32_t upload(demi_handle* h, const void* src, size_t bytes);
  template <class T = void> T* get() const { return (T*)p_; }
  size_t bytes() const { return bytes_; }
 private:
  void* p_ = nullptr; size_t bytes_ = 0;
};

struct DedupScratch { DevBuf keys, keep, counts; };

// What the fuzz launches need to know about an external program: its Sends (for a Fuzzer, those of its largest
// program), whether it has a HardKill or a Partition / UnPartition, and whether no two of its Sends are equal (two
// equal Sends would share a DepTracker Unique under the root).
struct ProgramInfo { uint32_t sends = 0; bool hard_kill = false, partitions = false, sends_distinct = true; };

struct demi_handle {
  DedupScratch dedup;
  demi_config cfg{};
  std::string err;
  int sm_count = 0;
  // external program
  std::vector<demi_ext_event> ext_host;
  DevBuf ext_dev;                                  // demi_ext_event[ext_host.size()]
  ProgramInfo ext_info;
  // device buffers
  DevBuf results_dev;                              // demi_fuzz_result
  DevBuf node_scratch, pend_scratch;               // uint4
  DevBuf counters_dev;                             // unsigned long long: [0]=sum_steps [1]=n_violations
  // lane engine
  DevBuf ext_sends_dev, lane_pend;                 // uint4
  DevBuf ovf_list, ovf_count;                      // uint32_t
  DevBuf fifo_scratch;                             // uint16_t
  int use_lane_engine = 1;
  uint32_t lane_pending_cap = 0;      // DEMI_LANE_PENDING_CAP (tests): the lane engine defers beyond this many pending messages
  DevBuf lane_snap_dev;                            // demi::LaneSnapshot of ext_host (demi_set_externals takes it)
  demi::LaneSnapshot lane_snap{};                  // its host copy: what launch_plan decides on
  int32_t lane_kernel = DEMI_LANE_NONE;            // the lane instantiation the last fuzz launch ran (demi_lane_kernel)
  // the tree of the steady instantiation (lane_steady.hpp): node records, built for ext_host under lane_tree_key
  DevBuf lane_tree, lane_tree_kids;                // uint32_t records; uint2 (parent, pending index) of a level's children
  bool lane_tree_built = false;
  demi::LaneTreeKey lane_tree_key{};
  int32_t lane_tree_depth = -1;                    // the depth the last fuzz launch walked (-1: not the steady one)
  int32_t lane_row_bytes = 0;                      // bytes per pending row of its lane kernel (0: none ran)
  DevBuf prov_scratch;
  std::vector<DevBuf> dpor_buf;                    // K3 per-search structures, one per entry of dpor_run's table (capi_dpor.cu)
  cudaStream_t stream = nullptr, copy_stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  demi_perf perf{};
  // ---- STSSched replay / DDMin (capi_replay.cu)
  std::vector<demi_event> trace_host;
  std::vector<demi_ext_event> trace_ext_host;
  std::vector<int32_t> conjoined;          // UnmodifiedEventDag._conjoinedAtoms over trace_ext_host (demi_conjoin_atoms)
  DevBuf trace_dev, trace_ext_dev;                 // trace_host, trace_ext_host
  DevBuf ev_ordinal_dev, send_ext_index_dev;       // uint16_t
  demi::ReplayTraceView trace{};                   // the trace as K2 reads it: its counts, capacities and the buffers above
  DevBuf rp_table; uint32_t rp_gen_next = 0; uint64_t rp_table_geometry = 0;
  DevBuf rp_tosend, rp_pruned, rp_masks, rp_results;
  DevBuf rp_counters;                              // unsigned long long[2]
  DevBuf rp_bound;                                 // demi::ReplayArgs per warp of a multi-trace K2 launch
  DevBuf rp_rec;                                   // a multi-trace recording launch's rows (demi_event), then counts
  // ---- the trace set (demi_set_traces, capi_replay_many.cu): independent of the single trace above
  struct TraceSet {
    uint32_t n = 0;
    std::vector<std::vector<demi_ext_event>> ext;      // per trace: its externals (DDMin's atoms)
    DevBuf events, ordinal, externals, send_index;   // every trace's records, one after the other
    std::vector<demi::ReplayTraceView> view;         // per trace: its view of the buffers above
    DevBuf views;                                    // view, on the device
  } set;
  // ---- communicator (capi_frontier.cu): NCCL inside the library
  FrComm* comm = nullptr;
  FrCache* frontier = nullptr;
  // ---- a model loaded with demi_load_model (model == DEMI_MODEL_IR)
  bool ir_loaded = false;
  DevBuf ir_blob_dev;                              // the blob's header and programs (ir_dev points into it)
  demi_ir_device ir_dev{};
  uint32_t ir_ext_mask = 0, ir_fanout = 0, ir_n_actors = 0, ir_n_types = 0;
  std::vector<std::string> names;      // actor names, then message-type names
  // ---- FullyRandom's userDefinedFilter as rules (demi_set_user_filter); HardKill in the external program
  std::vector<demi_filter_rule> filter;
  // ---- FingerprintFactory.getLogicalClock / causesClockIncrement as data (demi_set_clock_rules, capi_wildcard.cu):
  // per type the packed rule (0 = no clock; a valid rule has bits >= 1, so it is never 0) and the incrementing set
  uint32_t clock_rule[256] = {};
  uint32_t clock_incr[8] = {};
  // ---- the Fuzzer of demi_fuzz_campaign (demi_set_fuzzer) and the arena its generator kernel writes
  bool has_fuzzer = false;
  demi_fuzzer_config fuzzer{};
  uint32_t fz_n_prefix = 0, fz_n_postfix = 0;
  DevBuf fz_fixed_dev;                                    // demi_ext_event: prefix | postfix
  ProgramInfo fz_info;                                    // sends: prefix + postfix + num_events
  DevBuf fz_arena;
  // ---- launch bookkeeping
  std::map<const void*, int> occupancy;          // kernel -> resident blocks per SM (asked once per handle)
  DevBuf trace_rec;                              // demi_fuzz_trace's records (stage_records, one slot); only grows
};
// K2, STSSched replay (capi_replay.cu): the ReplayArgs fields that follow from the handle's configuration and `trace`;
// the rest are zero
namespace demi { struct ReplayArgs; }
demi::ReplayArgs replay_args(const demi_handle* h, const demi::ReplayTraceView& trace, uint32_t looking_for, uint32_t flags);
// the multi-trace kernel's own arguments: the set's views, the launch's tiles and, for WILD, each trace's mode table
// (capi_replay_many.cu)
struct ReplayTiles { const demi::ReplayTraceView* views; const uint4* tiles; uint32_t n_tiles; const uint32_t* const* modes; };
// Every K2 launch: the WILD or exact, REC or batch single-trace kernel, or with `many` the same four of the multi-trace
// kernel, on a's tests; the grid, the per-warp scratch, the generation range and the counters, the loaded model's binding.  `timed`
// records h->ev0 and h->ev1 around the kernel alone.
int32_t replay_launch(demi_handle* h, demi::ReplayArgs& a, bool wild, bool record, const ReplayTiles* many, bool timed,
                      cudaStream_t s);
// what demi_set_trace checks of a trace before it builds its side tables; `who` leads every message
int32_t check_trace(demi_handle* h, const char* who, const demi_event* events, uint32_t n_events,
                    const demi_ext_event* externals, uint32_t n_externals);
// the side tables of a trace K2 reads: per event the FIFO ordinal of its external Send, the index of each Send among
// the externals, the Uniq-id bound and the number of MsgSends
struct TraceTables { std::vector<uint16_t> ordinal, sidx; uint32_t n_uniq = 0, n_send_events = 0; };
int32_t trace_tables(demi_handle* h, const char* who, const demi_event* events, uint32_t n_events,
                     const demi_ext_event* externals, uint32_t n_externals, TraceTables& t);
// the counts and capacities of a trace's view (its buffers are the caller's)
demi::ReplayTraceView trace_view(const TraceTables& t, uint32_t n_events, uint32_t n_externals);
// the flags a wildcard replay accepts (capi_wildcard.cu): DEMI_RF_FILTER_KNOWN_ABSENTS and DEMI_WC_LAST_ONLY
int32_t wc_check_flags(demi_handle* h, const char* who, uint32_t flags);
// DDMin's verdicts on n replays: out[i] = "replay i reproduced the violation"; a replay that reported a status fails
int32_t replay_verdicts(demi_handle* h, const demi_replay_result* res, size_t n, signed char* out);
// demi_ddmin's walk over a driver whose oracle, trace and flags are set: check_unmodified, ddmin2, verify_mcs, outputs
namespace demi { struct DDMinDriver; }
int32_t ddmin_sts(demi::DDMinDriver& d, int32_t check_unmodified, uint64_t* mcs_mask, uint32_t* iteration_sizes,
                  uint32_t cap_iterations, demi_ddmin_out* out);
void demi_comm_free(demi_handle* h);
void demi_frontier_free(demi_handle* h);

inline int32_t fail(demi_handle* h, int32_t code, const char* fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
  if (h) h->err = buf; else g_create_error = buf;
  return code;
}
#define CUDA_TRY(h, expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) \
  return fail((h), DEMI_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)


// ---- validation of caller-supplied records (JNI hands over JVM buffers): every actor index, node id and parent
// pointer is range-checked before any host table or kernel indexes with it.
inline int demi_model_actors(const demi_handle* h) {
  const int model = h->cfg.model;
  if (model == DEMI_MODEL_IR) return (int)h->ir_n_actors;
  return model == DEMI_MODEL_PINGPONG3 ? 3 : model == DEMI_MODEL_RAFT5 ? 5 : 32;
}
// the `model` argument of the capacity rules in demi_limits.h (a loaded model carries its fan-out in the key)
inline int demi_model_key(const demi_handle* h) { return h->cfg.model == DEMI_MODEL_IR ? (DEMI_MODEL_IR | (int)(h->ir_fanout << 8)) : h->cfg.model; }
inline uint32_t demi_ext_type_mask(const demi_handle* h) { return h->cfg.model == DEMI_MODEL_IR ? h->ir_ext_mask : demi_external_type_mask(h->cfg.model); }
inline int32_t demi_need_model(demi_handle* h) {
  if (h->cfg.model == DEMI_MODEL_IR && !h->ir_loaded) return fail(h, DEMI_ERR_STATE, "demi_load_model has not been called");
  return DEMI_OK;
}
// External event ev[i] of a program `who` was handed: a kind it accepts (HardKill only with `hard_kill`: RandomScheduler
// fuzzing has it, replay and DPOR do not), actors of the model, and with `single_wait` no WaitQuiescence right after
// another (MessageTypes.sanityCheckTrace, ExternalEvents.scala:138-149).  `where` names the part of the program, or is "".
inline int32_t demi_check_external(demi_handle* h, const char* who, const char* where, const demi_ext_event* ev, uint32_t i,
                                   bool hard_kill, bool single_wait) {
  const demi_ext_event& e = ev[i];
  const uint32_t na = (uint32_t)demi_model_actors(h);
  if (e.kind < DEMI_EXT_START || e.kind > (hard_kill ? DEMI_EXT_HARD_KILL : DEMI_EXT_UNPARTITION))
    return fail(h, DEMI_ERR_INVALID, "%s: %sevent %u has kind %u, which this entry point does not accept", who, where, i, (unsigned)e.kind);
  const bool needs_a = e.kind != DEMI_EXT_WAIT_QUIESCENCE;
  const bool needs_b = e.kind == DEMI_EXT_PARTITION || e.kind == DEMI_EXT_UNPARTITION;
  if ((needs_a && e.a >= na) || (needs_b && e.b >= na)) return fail(h, DEMI_ERR_INVALID, "%s: %sevent %u names an unknown actor", who, where, i);
  if (single_wait && e.kind == DEMI_EXT_WAIT_QUIESCENCE && i > 0 && ev[i - 1].kind == DEMI_EXT_WAIT_QUIESCENCE)
    return fail(h, DEMI_ERR_INVALID, "%s: consecutive WaitQuiescence at %sevent %u", who, where, i);
  return DEMI_OK;
}
// a program to replay: no HardKill, consecutive WaitQuiescence allowed
inline int32_t demi_check_externals(demi_handle* h, const char* who, const demi_ext_event* ev, uint32_t n) {
  for (uint32_t i = 0; i < n; i++) {
    const int32_t rc = demi_check_external(h, who, "", ev, i, false, false);
    if (rc != DEMI_OK) return rc;
  }
  return DEMI_OK;
}
// a program for DPOR: Start and Send only ("unsuported external event", DPORwHeuristics.scala:710), actors of the model
inline int32_t demi_check_dpor_program(demi_handle* h, const char* who, const demi_ext_event* ev, uint32_t n) {
  const uint32_t na = (uint32_t)demi_model_actors(h);
  for (uint32_t i = 0; i < n; i++) {
    if (ev[i].kind != DEMI_EXT_START && ev[i].kind != DEMI_EXT_SEND)
      return fail(h, DEMI_ERR_INVALID, "%s: external %u: DPOR accepts Start and Send only", who, i);
    if (ev[i].a >= na) return fail(h, DEMI_ERR_INVALID, "%s: external %u names an unknown actor", who, i);
  }
  return DEMI_OK;
}
// n_nodes == 0: node ids are not checked (traces recorded by STSScheduler carry node = 0)
// max_actors == 0: the handle's model decides; else an explicit bound (provenance pruning works on any <= 32 actors)
inline int32_t demi_check_events(demi_handle* h, const char* who, const demi_event* ev, uint32_t n, uint32_t n_nodes,
                                 uint32_t max_actors = 0) {
  const uint32_t na = max_actors ? max_actors : (uint32_t)demi_model_actors(h);
  for (uint32_t i = 0; i < n; i++) {
    const demi_event& e = ev[i];
    bool ok = true;
    switch (e.kind) {
      case DEMI_EV_MSG_SEND:  ok = (e.src < na || e.src == DEMI_DEADLETTERS || e.src == DEMI_TIMER_SND) && e.dst < na; break;
      case DEMI_EV_MSG_EVENT: ok = (e.src < na || e.src == DEMI_DEADLETTERS || e.src == DEMI_TIMER_SND) && e.dst < na; break;
      case DEMI_EV_SPAWN: case DEMI_EV_KILL: ok = e.dst < na; break;
      case DEMI_EV_PARTITION: case DEMI_EV_UNPARTITION: ok = e.src < na && e.dst < na; break;
      case DEMI_EV_BEGIN_WAIT_QUIESCENCE: case DEMI_EV_QUIESCENCE: break;
      default: return fail(h, DEMI_ERR_INVALID, "%s: event %u has unknown kind %u", who, i, (unsigned)e.kind);
    }
    if (!ok) return fail(h, DEMI_ERR_INVALID, "%s: event %u names an unknown actor (src %u, dst %u)", who, i, (unsigned)e.src, (unsigned)e.dst);
    if (n_nodes && (e.kind == DEMI_EV_MSG_SEND || e.kind == DEMI_EV_MSG_EVENT) && e.node >= n_nodes)
      return fail(h, DEMI_ERR_INVALID, "%s: event %u names node %u outside the tree of %u", who, i, (unsigned)e.node, n_nodes);
  }
  return DEMI_OK;
}
inline int32_t demi_check_parents(demi_handle* h, const char* who, const uint16_t* dep_parent, uint32_t n_nodes) {
  for (uint32_t v = 1; v < n_nodes; v++)
    if (dep_parent[v] >= v) return fail(h, DEMI_ERR_INVALID, "%s: node %u has parent %u (a parent is created before its children)", who, v, (unsigned)dep_parent[v]);
  return DEMI_OK;
}

// DEMI_TEST_ALLOC_LIMIT=n (tests): an allocation of more than n bytes fails as a full device would, without asking the
// driver.  It is read only when a buffer is about to be allocated, so a test can set it around one call.
inline int32_t DevBuf::grow(demi_handle* h, size_t bytes) {
  if (bytes_ >= bytes) return DEMI_OK;
  reset();
  const char* limit = getenv("DEMI_TEST_ALLOC_LIMIT");
  const cudaError_t e = limit && *limit && bytes > strtoull(limit, nullptr, 10) ? cudaErrorMemoryAllocation : cudaMalloc(&p_, bytes);
  if (e != cudaSuccess) { p_ = nullptr; return fail(h, DEMI_ERR_CUDA, "cudaMalloc of %zu bytes: %s", bytes, cudaGetErrorString(e)); }
  bytes_ = bytes;
  return DEMI_OK;
}
inline int32_t DevBuf::upload(demi_handle* h, const void* src, size_t bytes) {
  const int32_t rc = grow(h, bytes);
  if (rc != DEMI_OK) return rc;
  CUDA_TRY(h, cudaMemcpy(p_, src, bytes, cudaMemcpyHostToDevice));
  return DEMI_OK;
}

// Resident blocks per SM of kernel `fn` at `block` threads and `smem` bytes of dynamic shared memory (which it is
// allowed first).  Both are fixed per device, so they are asked once per handle; the cache is keyed on the kernel
// alone, so `smem` must be fixed per kernel too.
inline int32_t demi_occupancy(demi_handle* h, const void* fn, int block, size_t smem, int* blocks_per_sm) {
  auto it = h->occupancy.find(fn);
  if (it != h->occupancy.end()) { *blocks_per_sm = it->second; return DEMI_OK; }
  CUDA_TRY(h, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CUDA_TRY(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, fn, block, smem));
  h->occupancy[fn] = *blocks_per_sm;
  return DEMI_OK;
}
