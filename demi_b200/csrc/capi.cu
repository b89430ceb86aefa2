// capi.cu — the C ABI (include/demi_b200.h) over the CUDA engine.
// No CPU fallback: every compute entry point needs a CUDA device.
#include <climits>
#include <cmath>
#include <cstddef>
#include <cstdlib>
#include <cstdio>
#include <cstdarg>
#include <cstring>
#include <string>
#include <vector>
#include <algorithm>
#include <cuda_runtime.h>
#include "fuzz_kernel.cuh"
#include "provenance_kernel.cuh"
#include "lane_kernel.cuh"
#include "models/model_ir.cuh"
#include "fuzzer_gen.cuh"

using namespace demi;

#include "engine.hpp"

thread_local std::string g_create_error;

// ------------------------------------------------------------ kernel table
constexpr int WARPS = 4;
typedef void (*kernel_fn)(const KernelArgs);
// What a fuzz launch runs: a batch of prefixes over the handle's program, the recording of chosen prefixes
// (provenance, traces), a campaign's generated programs (PROG), random-oracle tests over subsequences (PROG + TESTS),
// or random-oracle tests of many traces, each with its own parameters (PROG + TESTS + PARAMS).  Both engines have one
// instantiation per mode, except the recording of many programs' executions, each with its own parameters
// (PROG + RECORD + PARAMS), which the warp engine alone runs.
enum LaunchMode { LM_BATCH, LM_RECORD, LM_PROGRAM, LM_TESTS, LM_TEST_PARAMS, LM_RECORD_PARAMS, LM_COUNT };
struct Variant {
  int model; uint32_t pcap, tcap; bool pend_global;
  size_t smem_per_warp;
  kernel_fn fn[LM_COUNT];        // a recording variant has LM_RECORD and LM_RECORD_PARAMS, the others every other mode
};
template <class MODEL, int PCAP, int TCAP, bool PG, bool REC>
static Variant make_variant() {
  using M = Machine<MODEL, PCAP, TCAP, PG, REC>;
  Variant v{MODEL::ID, (uint32_t)PCAP, (uint32_t)TCAP, PG, sizeof(typename M::Smem),
            {fuzz_kernel<MODEL, PCAP, TCAP, PG, REC, WARPS>, nullptr,
             REC ? nullptr : fuzz_kernel<MODEL, PCAP, TCAP, PG, REC, WARPS, !REC>,
             REC ? nullptr : fuzz_kernel<MODEL, PCAP, TCAP, PG, REC, WARPS, !REC, !REC>,
             REC ? nullptr : fuzz_kernel<MODEL, PCAP, TCAP, PG, REC, WARPS, !REC, !REC, !REC>,
             REC ? fuzz_kernel<MODEL, PCAP, TCAP, PG, REC, WARPS, REC, false, REC> : nullptr}};
  if (REC) std::swap(v.fn[LM_BATCH], v.fn[LM_RECORD]);
  return v;
}
static const std::vector<Variant>& variants() {
  static const std::vector<Variant> v = {
    make_variant<PingPong3, 128, 128, false, false>(),
    make_variant<PingPong3, 16384, 1024, true, false>(),
    make_variant<PingPong3, 16384, 1024, true, true>(),
    make_variant<Raft5, 256, 32, false, false>(),
    make_variant<Raft5, 512, 32, false, false>(),
    make_variant<Raft5, 256, 32, false, true>(),          // recording, shared-memory pending set (provenance batches)
    make_variant<Raft5, 16384, 1024, true, false>(),
    make_variant<Raft5, 16384, 1024, true, true>(),
    make_variant<Bcast32, 16384, 32, true, false>(),
    make_variant<Bcast32, 16384, 1024, true, false>(),
    make_variant<Bcast32, 16384, 1024, true, true>(),
    make_variant<IrModel, 128, 128, false, false>(),      // a model loaded with demi_load_model
    make_variant<IrModel, 16384, 1024, true, false>(),
    make_variant<IrModel, 16384, 1024, true, true>(),
  };
  return v;
}
static const Variant* pick_variant(int model, LaunchMode mode, uint32_t pcap, uint32_t tcap, bool need_global) {
  for (const Variant& v : variants())
    if (v.model == model && v.fn[mode] && v.pcap >= pcap && v.tcap >= tcap && (v.pend_global || !need_global)) return &v;
  return nullptr;
}

// lane-engine table
// `steady`: the LM_BATCH instantiation that starts from the program's tree (`snapshot` takes its root, `tree` builds
// one level, of records `node_bytes` long); `ops` is the model's operations per receive(), which the node-capacity
// proof of lane_steady_eligible counts with.  `row8`: the steady instantiation with 8-byte pending rows, for the model
// whose rows lane_row8_eligible can prove fit them (raft5), else null.
typedef void (*snapshot_fn)(const KernelArgs, LaneSnapshot*);
typedef void (*tree_fn)(const KernelArgs, uint32_t*, const uint2*, uint32_t, uint32_t);
struct LaneVariant {
  int model; int bd; uint32_t lpcap; size_t smem_per_block; kernel_fn fn[LM_COUNT];
  kernel_fn steady; size_t steady_smem; snapshot_fn snapshot; tree_fn tree; uint32_t node_bytes; uint32_t ops;
  kernel_fn row8;
};
template <class MODEL, int BD, int LPCAP, bool ROW8 = false>
static LaneVariant make_lane_variant() {
  using M = LaneMachine<MODEL, BD, LPCAP>;
  using S = LaneMachine<MODEL, BD, LPCAP, false, true>;
  return LaneVariant{MODEL::ID, BD, (uint32_t)LPCAP, (size_t)M::WORDS * BD * sizeof(uint32_t),
                     {fuzz_lane_kernel<MODEL, BD, LPCAP>, fuzz_lane_kernel<MODEL, BD, LPCAP, true>,
                      fuzz_lane_kernel<MODEL, BD, LPCAP, false, true>, fuzz_lane_kernel<MODEL, BD, LPCAP, false, true, true>,
                      fuzz_lane_kernel<MODEL, BD, LPCAP, false, true, true, false, true>},
                     fuzz_lane_kernel<MODEL, BD, LPCAP, false, false, false, true>, (size_t)S::WORDS * BD * sizeof(uint32_t),
                     lane_snapshot_kernel<MODEL>, lane_tree_kernel<MODEL, LPCAP>, S::NODE_WORDS * 4u, (uint32_t)MODEL::LANE_OUTBOX,
                     ROW8 ? fuzz_lane_kernel<MODEL, BD, LPCAP, false, false, false, true, false, ROW8> : nullptr};
}
#ifndef DEMI_K1_BD_RAFT5
#define DEMI_K1_BD_RAFT5 256
#endif
static const LaneVariant* lane_variant_of(int model) {
  static const std::vector<LaneVariant> v = {
    make_lane_variant<Raft5, DEMI_K1_BD_RAFT5, DEMI_K1_LPCAP_RAFT5, true>(),
    make_lane_variant<PingPong3, 256, 128>(),
    make_lane_variant<Bcast32, 128, 8192>(),
  };
  for (const LaneVariant& lv : v) if (lv.model == model) return &lv;
  return nullptr;
}

// ---------------------------------------------------------------- lifecycle
#ifndef DEMI_BUILD_ID
#define DEMI_BUILD_ID "unknown"
#endif
#ifndef DEMI_K1_ID
#define DEMI_K1_ID "unknown"
#endif
extern "C" const char* demi_version(void) { return "demi_b200 0.2 (sm_90a) build " DEMI_BUILD_ID " k1 " DEMI_K1_ID; }

extern "C" const char* demi_last_error(const demi_handle* h) {
  return h ? h->err.c_str() : g_create_error.c_str();
}

#if DEMI_K1_PHASE_CLOCK
// The lane engine's phase sums ([phase][cycles, active lanes, entries], LanePhase order) of every launch since the
// last reset; only a library built with DEMI_K1_PHASE_CLOCK has this symbol.
extern "C" int32_t demi_k1_phase_read(unsigned long long* out, int32_t reset) {
  if (cudaDeviceSynchronize() != cudaSuccess) return DEMI_ERR_CUDA;
  if (out && cudaMemcpyFromSymbol(out, demi_k1_phase_sums, sizeof(demi_k1_phase_sums)) != cudaSuccess) return DEMI_ERR_CUDA;
  if (reset) {
    static const unsigned long long zero[LP_COUNT * 3] = {};
    if (cudaMemcpyToSymbol(demi_k1_phase_sums, zero, sizeof(zero)) != cudaSuccess) return DEMI_ERR_CUDA;
  }
  return LP_COUNT;
}
#endif

extern "C" int32_t demi_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

extern "C" int32_t demi_create(const demi_config* cfg, demi_handle** out) {
  if (!cfg || !out) return fail(nullptr, DEMI_ERR_INVALID, "demi_create: null argument");
  *out = nullptr;
  if (cfg->model != DEMI_MODEL_PINGPONG3 && cfg->model != DEMI_MODEL_RAFT5 && cfg->model != DEMI_MODEL_BCAST32 &&
      cfg->model != DEMI_MODEL_IR)
    return fail(nullptr, DEMI_ERR_INVALID, "demi_create: unknown model %d", cfg->model);
  if (cfg->strategy != DEMI_RS_FULLY_RANDOM && cfg->strategy != DEMI_RS_SRC_DST_FIFO)
    return fail(nullptr, DEMI_ERR_INVALID, "demi_create: unknown randomization strategy %d", cfg->strategy);
  int n = demi_device_count();
  if (n <= 0) return fail(nullptr, DEMI_ERR_NO_DEVICE, "demi_create: no CUDA device (this engine has no CPU fallback)");
  if (cfg->device < 0 || cfg->device >= n)
    return fail(nullptr, DEMI_ERR_INVALID, "demi_create: device %d out of range (%d devices)", cfg->device, n);
  demi_handle* h = new demi_handle();
  h->cfg = *cfg;
  cudaError_t e = cudaSetDevice(cfg->device);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&h->sm_count, cudaDevAttrMultiProcessorCount, cfg->device);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreate(&h->ev0);
  if (e == cudaSuccess) e = cudaEventCreate(&h->ev1);
  if (getenv("DEMI_DISABLE_LANE_ENGINE")) h->use_lane_engine = 0;
  if (const char* e = getenv("DEMI_LANE_PENDING_CAP")) h->lane_pending_cap = (uint32_t)atoi(e);   // tests: make the lane engine defer early
  int32_t rc = e == cudaSuccess ? DEMI_OK : fail(nullptr, DEMI_ERR_CUDA, "demi_create: %s", cudaGetErrorString(e));
  // no handle yet: a failure goes to demi_last_error(NULL)
  if (rc == DEMI_OK) rc = h->counters_dev.grow(nullptr, 4 * sizeof(unsigned long long));
  if (rc == DEMI_OK) rc = h->ovf_count.grow(nullptr, sizeof(uint32_t));
  if (rc != DEMI_OK) {
    demi_destroy(h);                       // frees whatever was created before the failure
    return rc;
  }
  *out = h;
  return DEMI_OK;
}

extern "C" void demi_destroy(demi_handle* h) {
  if (!h) return;
  cudaSetDevice(h->cfg.device);
  demi_frontier_free(h);
  demi_comm_free(h);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->stream) cudaStreamDestroy(h->stream);
  if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
  delete h;                                // its device buffers free themselves
}

// demi_load_model: validate, keep the name table on the host, put programs + initial states on the device
extern "C" int32_t demi_load_model(demi_handle* h, const void* model_blob, size_t size) {
  if (!h) return DEMI_ERR_INVALID;
  if (h->cfg.model != DEMI_MODEL_IR) return fail(h, DEMI_ERR_STATE, "demi_load_model: the handle was created for built-in model %d", h->cfg.model);
  const uint32_t* w = (const uint32_t*)model_blob;
  if (!w || size < DEMI_IR_HEADER_WORDS * 4 || w[0] != DEMI_IR_MAGIC) return fail(h, DEMI_ERR_INVALID, "demi_load_model: not a model blob");
  if (w[1] != DEMI_IR_VERSION) return fail(h, DEMI_ERR_INVALID, "demi_load_model: version %u, this library reads %u", w[1], DEMI_IR_VERSION);
  const uint32_t na = w[2], sw = w[3], nt = w[4], rl = w[5], il = w[6], nb = w[9];
  if (na < 1 || na > DEMI_IR_ACTORS || sw < 1 || sw > DEMI_IR_STATE_WORDS || rl > DEMI_IR_MAX_CODE || il > DEMI_IR_MAX_CODE || w[8] > DEMI_IR_OUTBOX || nt > 256)
    return fail(h, DEMI_ERR_INVALID, "demi_load_model: %u actors x %u words, %u + %u instructions, fan-out %u exceed the limits of demi_model_ir.h", na, sw, rl, il, w[8]);
  const size_t words = (size_t)DEMI_IR_HEADER_WORDS + rl + il + (size_t)na * sw;
  if (size < words * 4 + nb) return fail(h, DEMI_ERR_INVALID, "demi_load_model: blob truncated (%zu of %zu bytes)", size, words * 4 + nb);
  // every operand is a register number < 16 by construction; jump targets and opcodes are checked here
  for (int prog = 0; prog < 2; prog++) {
    const uint32_t* code = w + DEMI_IR_HEADER_WORDS + (prog ? rl : 0); const uint32_t len = prog ? il : rl;
    for (uint32_t pc = 0; pc < len; pc++) {
      const uint32_t op = code[pc] & 0xFF;
      if (op > DEMI_IR_RET) return fail(h, DEMI_ERR_INVALID, "demi_load_model: unknown opcode %u at %u", op, pc);
      if (op == DEMI_IR_LDI || (op >= DEMI_IR_JMP && op <= DEMI_IR_JGE)) {
        if (pc + 1 >= len) return fail(h, DEMI_ERR_INVALID, "demi_load_model: instruction at %u lacks its immediate", pc);
        if (op != DEMI_IR_LDI && code[pc + 1] > len) return fail(h, DEMI_ERR_INVALID, "demi_load_model: jump at %u leaves the program", pc);
        pc++;
      }
    }
  }
  std::vector<std::string> names;
  const char* nm = (const char*)(w + words); size_t off = 0;
  while (off < nb && names.size() < (size_t)na + nt) { const size_t l = strnlen(nm + off, nb - off); names.emplace_back(nm + off, l); off += l + 1; }
  if (names.size() != (size_t)na + nt) return fail(h, DEMI_ERR_INVALID, "demi_load_model: %zu names for %u actors + %u message types", names.size(), na, nt);
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  DevBuf blob;
  const int32_t rc = blob.upload(h, w, words * 4);
  if (rc != DEMI_OK) return rc;
  h->ir_blob_dev = std::move(blob);
  h->ir_dev.recv = h->ir_blob_dev.get<uint32_t>() + DEMI_IR_HEADER_WORDS; h->ir_dev.inv = h->ir_dev.recv + rl; h->ir_dev.init = h->ir_dev.inv + il;
  h->ir_dev.recv_len = rl; h->ir_dev.inv_len = il; h->ir_dev.n_actors = na; h->ir_dev.state_words = sw;
  h->ir_ext_mask = w[7]; h->ir_fanout = w[8]; h->ir_n_actors = na; h->ir_n_types = nt;
  h->names = std::move(names);
  h->ir_loaded = true;
  return DEMI_OK;
}
extern "C" int32_t demi_actor_index(const demi_handle* h, const char* name) {
  if (!h || !name) return -1;
  const int na = demi_model_actors(h);
  if (h->cfg.model == DEMI_MODEL_IR) { for (int i = 0; i < na; i++) if (h->names[i] == name) return i; return -1; }
  char* end = nullptr; const long v = strtol(name, &end, 10);
  return (*name && !*end && v >= 0 && v < na) ? (int32_t)v : -1;
}
extern "C" const char* demi_actor_name(const demi_handle* h, uint32_t index) {
  if (!h || (int)index >= demi_model_actors(h)) return nullptr;
  if (h->cfg.model == DEMI_MODEL_IR) return h->names[index].c_str();
  static const char* digits[32] = {"0","1","2","3","4","5","6","7","8","9","10","11","12","13","14","15","16","17","18","19","20",
                                   "21","22","23","24","25","26","27","28","29","30","31"};
  return digits[index];
}

// A Send external in the form the lane engine reads from its Send table (LaneMachine::external_produced decodes it,
// lane_kernel.cuh:452): a message from deadLetters, flagged external.
__host__ __device__ inline uint4 lane_send(const demi_ext_event& e) {
  return make_uint4(DEMI_DEADLETTERS | ((uint32_t)e.a << 8) | ((uint32_t)e.type << 16) | ((uint32_t)DEMI_MF_EXTERNAL << 24),
                    e.p0, e.p1, 0u);
}

// Adds event e of a program to *info; `sends` collects the program's Sends in the lane engine's form.
static void describe_event(ProgramInfo* info, std::vector<uint4>* sends, const demi_ext_event& e) {
  if (e.kind == DEMI_EXT_PARTITION || e.kind == DEMI_EXT_UNPARTITION) info->partitions = true;
  if (e.kind == DEMI_EXT_HARD_KILL) info->hard_kill = true;
  if (e.kind != DEMI_EXT_SEND) return;
  const uint4 m = lane_send(e);
  for (const uint4& o : *sends) if (o.x == m.x && o.y == m.y && o.z == m.z) info->sends_distinct = false;
  sends->push_back(m);
  info->sends++;
}

extern "C" int32_t demi_set_externals(demi_handle* h, const demi_ext_event* ev, uint32_t n) {
  if (!h) return DEMI_ERR_INVALID;
  if (!ev && n) return fail(h, DEMI_ERR_INVALID, "demi_set_externals: null events");
  { int32_t mrc = demi_need_model(h); if (mrc != DEMI_OK) return mrc; }
  ProgramInfo info;
  std::vector<uint4> sv;                 // the lane engine's Send table
  for (uint32_t i = 0; i < n; i++) {
    const int32_t rc = demi_check_external(h, "demi_set_externals", "", ev, i, true, true);
    if (rc != DEMI_OK) return rc;
    describe_event(&info, &sv, ev[i]);
  }
  // the program the handle has: everything below would compute what it holds, the tree included
  if (n && n == h->ext_host.size() && memcmp(ev, h->ext_host.data(), n * sizeof(demi_ext_event)) == 0) return DEMI_OK;
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  DevBuf ext_dev, sends_dev, snap_dev;
  LaneSnapshot snap{};
  snap.status = LANE_DEFER;                // no lane engine for the model: no snapshot
  int32_t rc;
  if (n && (rc = ext_dev.upload(h, ev, n * sizeof(demi_ext_event))) != DEMI_OK) return rc;
  if (!sv.empty() && (rc = sends_dev.upload(h, sv.data(), sv.size() * sizeof(uint4))) != DEMI_OK) return rc;
  if (const LaneVariant* lv = lane_variant_of(h->cfg.model)) {
    // The program's pre-delivery snapshot, under the physical limits: a batch compares its counts with its own
    // capacities (launch_plan).  It depends on the program and the model alone (no actor has received anything, and
    // the snapshot holds no actor state, so neither model_flags nor ignoreTimers shows in it), hence it is taken here
    // and not per batch.
    const size_t snap_bytes = sizeof(LaneSnapshot) + lv->node_bytes;      // the snapshot, then the tree's root
    if ((rc = snap_dev.grow(h, snap_bytes)) != DEMI_OK) return rc;
    KernelArgs a{};
    a.ext = ext_dev.get<demi_ext_event>(); a.n_ext = n;
    a.ext_sends = sends_dev.get<uint4>();
    a.has_partitions = info.partitions ? 1u : 0u;
    a.model_flags = h->cfg.model_flags;
    a.max_messages = INT_MAX;
    a.node_cap = 65535u; a.pending_cap = 0xFFFFu; a.tosend_cap = 0xFFFFu;
    CUDA_TRY(h, cudaMemsetAsync(snap_dev.get(), 0, snap_bytes, h->stream));
    lv->snapshot<<<1, 1, 0, h->stream>>>(a, snap_dev.get<LaneSnapshot>());
    CUDA_TRY(h, cudaGetLastError());
    CUDA_TRY(h, cudaMemcpyAsync(&snap, snap_dev.get(), sizeof(LaneSnapshot), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  h->ext_host.assign(ev, ev + n);
  h->ext_info = info;
  h->ext_dev = std::move(ext_dev);
  h->ext_sends_dev = std::move(sends_dev);
  h->lane_snap_dev = std::move(snap_dev);
  h->lane_snap = snap;
  h->lane_tree_built = false;
  return DEMI_OK;
}

extern "C" int32_t demi_set_user_filter(demi_handle* h, const demi_filter_rule* rules, uint32_t n) {
  if (!h) return DEMI_ERR_INVALID;
  if (n > DEMI_MAX_FILTER_RULES || (!rules && n)) return fail(h, DEMI_ERR_INVALID, "demi_set_user_filter: at most %d rules", DEMI_MAX_FILTER_RULES);
  h->filter.assign(rules, rules + n);
  return DEMI_OK;
}

// The lane engine for a launch over a program `prog` describes (for a campaign, the Fuzzer's; a random-oracle test
// decides on the base program, and each of its subsequences meets every condition the base program meets)
static const LaneVariant* pick_lane_variant(const demi_handle* h, const ProgramInfo& prog) {
  if (!h->use_lane_engine || h->cfg.blocked_mask || !prog.sends_distinct || h->cfg.strategy != DEMI_RS_FULLY_RANDOM ||
      prog.hard_kill || !h->filter.empty()) return nullptr;          // actor termination and user filters: the general engine
  return lane_variant_of(h->cfg.model);
}

// ------------------------------------------------------------------- launch
struct LaunchPlan { const Variant* v; LaunchMode mode; const ProgramInfo* prog; int grid; size_t smem; KernelArgs args; };

// The variant (in *v, when v is given) that a launch of `mode` over a program `prog` describes runs on under h's
// configuration, at pending capacity pcap and tosend capacity tcap.  Its two refusals, in this order, go to `to` (h, or
// a trace's own handle): no variant fits, or SrcDstFIFO with a HardKill or a user filter.
static int32_t check_variant(const demi_handle* h, demi_handle* to, LaunchMode mode, const ProgramInfo& prog, uint32_t pcap,
                             uint32_t tcap, const Variant** v) {
  const bool fifo = h->cfg.strategy == DEMI_RS_SRC_DST_FIFO;          // SrcDstFIFO lives in the HBM-pending variants
  // so does every program with a HardKill: Machine::hard_kill needs room for n_pending + matches <= 2 * pcap entries,
  // which only the HBM variants (PCAP = 16384 >= 2 * 8192) have.  A random-oracle test decides on the base program.
  const Variant* pv = pick_variant(h->cfg.model, mode, pcap, tcap, fifo || prog.hard_kill);
  if (!pv) return fail(to, DEMI_ERR_CAPACITY, "no kernel variant for pending_cap=%u tosend_cap=%u", pcap, tcap);
  if (fifo && (prog.hard_kill || !h->filter.empty()))
    return fail(to, DEMI_ERR_INVALID, "HardKill and userDefinedFilter are offered for FullyRandom only");
  if (v) *v = pv;
  return DEMI_OK;
}

// A launch of `mode` over the program (ext, n_ext) that `prog` describes.  A campaign has no one program: `prog` is
// its Fuzzer's, sized for the largest program, and each execution binds its own events.  Nor has a launch of many
// traces' tests: `prog` joins its base programs, and `pcap_at_least` is the largest of their pending capacities,
// each under its own max_messages.
static int32_t plan_launch(demi_handle* h, const demi_fuzz_params* p, LaunchMode mode, const ProgramInfo& prog,
                           const demi_ext_event* ext, uint32_t n_ext, LaunchPlan* plan, uint32_t pcap_at_least = 0) {
  if (!p) return fail(h, DEMI_ERR_INVALID, "null params");
  if (mode == LM_PROGRAM && !h->has_fuzzer) return fail(h, DEMI_ERR_STATE, "demi_set_fuzzer has not been called");
  if (mode != LM_PROGRAM && mode != LM_TEST_PARAMS && mode != LM_RECORD_PARAMS && h->ext_host.empty())
    return fail(h, DEMI_ERR_STATE, "demi_set_externals has not been called");
  if (p->n_prefixes > 0xFFFFFFFFull) return fail(h, DEMI_ERR_INVALID, "n_prefixes > 2^32-1 per call");
  { int32_t mrc = demi_need_model(h); if (mrc != DEMI_OK) return mrc; }
  const uint32_t pcap = std::max(pcap_at_least, demi_pending_cap(demi_model_key(h), p->max_messages, prog.sends));
  const uint32_t tcap = demi_tosend_cap(prog.sends);
  const Variant* v;
  int32_t rc;
  if ((rc = check_variant(h, h, mode, prog, pcap, tcap, &v)) != DEMI_OK) return rc;
  const size_t smem = v->smem_per_warp * WARPS;
  int blocks_per_sm = 0;
  if ((rc = demi_occupancy(h, (const void*)v->fn[mode], WARPS * 32, smem, &blocks_per_sm)) != DEMI_OK) return rc;
  if (blocks_per_sm < 1) return fail(h, DEMI_ERR_CAPACITY, "kernel variant does not fit on an SM (smem %zu)", smem);
  uint64_t want = (p->n_prefixes + WARPS - 1) / WARPS;
  uint64_t full = (uint64_t)h->sm_count * (uint64_t)blocks_per_sm;
  int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>(want, full));
  const uint64_t total_warps = (uint64_t)grid * WARPS;
  const uint32_t node_cap = demi_node_cap(pcap);

  if ((rc = h->node_scratch.grow(h, total_warps * node_cap * sizeof(uint4))) != DEMI_OK) return rc;
  if (v->pend_global)
    if ((rc = h->pend_scratch.grow(h, total_warps * (uint64_t)v->pcap * sizeof(uint4))) != DEMI_OK) return rc;

  KernelArgs a{};
  a.model_flags = h->cfg.model_flags;
  a.blocked_mask = h->cfg.blocked_mask;
  a.ignore_timers = h->cfg.ignore_timers;
  a.max_messages = p->max_messages < 0 ? INT_MAX : p->max_messages;   // maxMessages = Int.MaxValue (RandomScheduler.scala:54)
  a.interval = p->invariant_check_interval;
  a.looking_for = p->looking_for;
  a.seed_base = p->seed_base;
  a.n_prefixes = p->n_prefixes;
  a.fuzz_flags = p->flags;
  a.strategy = h->cfg.strategy;
  if (h->cfg.strategy == DEMI_RS_SRC_DST_FIFO) {
    if ((rc = h->fifo_scratch.grow(h, total_warps * (uint64_t)(v->pcap / 2 + 3 * FIFO_PAIRS) * sizeof(uint16_t))) != DEMI_OK) return rc;
    a.fifo_scratch = h->fifo_scratch.get<uint16_t>();
  }
  a.n_filter = (uint32_t)h->filter.size();
  for (uint32_t i = 0; i < a.n_filter; i++) a.filter[i] = make_uint4(h->filter[i].src_mask, h->filter[i].dst_mask, h->filter[i].type_mask, h->filter[i].flags);
  a.ext = ext;
  a.n_ext = n_ext;
  a.node_cap = node_cap;
  a.pending_cap = pcap;
  a.tosend_cap = tcap;
  a.node_scratch = h->node_scratch.get<uint4>();
  a.pend_scratch = h->pend_scratch.get<uint4>();
  a.sum_steps = h->counters_dev.get<unsigned long long>();
  a.n_violations = a.sum_steps + 1;
  plan->v = v; plan->mode = mode; plan->prog = &prog; plan->grid = grid; plan->smem = smem; plan->args = a;
  return DEMI_OK;
}

// The tree of the handle's program for a steady launch with arguments `la` (lane_steady.hpp), kept on the handle and
// built again only when the program or the key changes.  Level by level: the host reads the new level's first 16
// bytes per record, decides with lane_tree_extend whether the next level is built, and lists its children; one thread
// builds each.  The root is the record the snapshot kernel stored after the snapshot.
static int32_t lane_tree(demi_handle* h, const LaneVariant* lv, const KernelArgs& la, cudaStream_t s) {
  const LaneTreeKey key = lane_tree_key(la.model_flags, la.interval, la.max_messages, la.pending_cap);
  if (h->lane_tree_built && h->lane_tree_key == key) return DEMI_OK;
  h->lane_tree_built = false;
  const size_t nb = lv->node_bytes;
  int32_t rc;
  if ((rc = h->lane_tree.grow(h, std::max<size_t>(LANE_TREE_BUDGET, nb))) != DEMI_OK) return rc;
  uint8_t* tree = h->lane_tree.get<uint8_t>();
  CUDA_TRY(h, cudaMemcpyAsync(tree, h->lane_snap_dev.get<uint8_t>() + sizeof(LaneSnapshot), nb, cudaMemcpyDeviceToDevice, s));
  KernelArgs ba = la;
  ba.pending_cap = std::min(la.pending_cap, LANE_NODE_ROWS);
  uint64_t lo = 0, hi = 1;                           // the deepest level's records
  uint32_t depth = 0;
  std::vector<uint4> head;
  std::vector<uint2> kids;
  for (;;) {
    head.resize(hi - lo);
    CUDA_TRY(h, cudaMemcpy2DAsync(head.data(), sizeof(uint4), tree + lo * nb, nb, sizeof(uint4), hi - lo, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(h, cudaStreamSynchronize(s));
    kids.clear();
    for (uint64_t j = 0; j < hi - lo; j++)
      if (lane_node_expands(head[j].y, (int32_t)head[j].z, head[j].w, la.max_messages))
        for (uint32_t i = 0; i < head[j].y; i++) kids.push_back(make_uint2((uint32_t)(lo + j), i));
    if (!lane_tree_extend(depth, hi, kids.size(), (uint32_t)nb)) break;
    if ((rc = h->lane_tree_kids.grow(h, kids.size() * sizeof(uint2))) != DEMI_OK) return rc;
    CUDA_TRY(h, cudaMemcpyAsync(h->lane_tree_kids.get(), kids.data(), kids.size() * sizeof(uint2), cudaMemcpyHostToDevice, s));
    const uint32_t n = (uint32_t)kids.size();
    lv->tree<<<(n + LANE_TREE_BD - 1) / LANE_TREE_BD, LANE_TREE_BD, 0, s>>>(ba, reinterpret_cast<uint32_t*>(tree),
                                                                         h->lane_tree_kids.get<uint2>(), (uint32_t)hi, n);
    CUDA_TRY(h, cudaGetLastError());
    lo = hi; hi += n; depth++;
  }
  h->lane_snap.depth = depth;
  h->lane_snap.tree = (uint64_t)(uintptr_t)tree;
  CUDA_TRY(h, cudaMemcpyAsync(h->lane_snap_dev.get<uint8_t>() + offsetof(LaneSnapshot, depth), &h->lane_snap.depth,
                              sizeof(LaneSnapshot) - offsetof(LaneSnapshot, depth), cudaMemcpyHostToDevice, s));
  CUDA_TRY(h, cudaStreamSynchronize(s));
  h->lane_tree_key = key;
  h->lane_tree_built = true;
  return DEMI_OK;
}

// The lane engine over the plan's `n_items` work items when one applies, then the warp engine on the items it deferred
// (on every item otherwise).  Counts both launches.
static int32_t launch_plan(demi_handle* h, LaunchPlan& plan, uint64_t n_items, cudaStream_t s) {
  KernelArgs& a = plan.args;
  h->lane_kernel = DEMI_LANE_NONE;
  h->lane_row_bytes = 0;
  h->lane_tree_depth = -1;
  if (const LaneVariant* lv = pick_lane_variant(h, *plan.prog)) {
    const uint32_t lane_pcap = std::min(h->lane_pending_cap ? std::min(a.pending_cap, h->lane_pending_cap) : a.pending_cap, lv->lpcap);
    // A batch over the handle's program starts every execution from the program's snapshot when the rule of
    // lane_steady.hpp allows it; every other launch runs the generic instantiation.
    bool steady = false;
    if (plan.mode == LM_BATCH && plan.prog == &h->ext_info) {
      LaneSteadyLaunch l{};
      l.n_ext = a.n_ext; l.partitions = plan.prog->partitions; l.ignore_timers = a.ignore_timers != 0;
      l.looking_for = a.looking_for; l.max_messages = a.max_messages;
      l.pending_cap = lane_pcap; l.node_cap = a.node_cap; l.tosend_cap = a.tosend_cap;
      l.lane_tosend_cap = LANE_TOSEND_CAP; l.ops_per_delivery = lv->ops;
      steady = lane_steady_eligible(h->lane_snap, l);
    }
    // ... and with 8-byte pending rows when the launch's rows provably fit them
    const bool row8 = steady && lv->row8 && lane_row8_eligible(h->lane_snap, a.max_messages, lv->ops);
    const kernel_fn lfn = row8 ? lv->row8 : steady ? lv->steady : lv->fn[plan.mode];
    const size_t lsmem = steady ? lv->steady_smem : lv->smem_per_block;
    int32_t rc;
    int bps = 0;
    if ((rc = demi_occupancy(h, (const void*)lfn, lv->bd, lsmem, &bps)) != DEMI_OK) return rc;
    if (bps < 1) return fail(h, DEMI_ERR_CAPACITY, "lane kernel does not fit on an SM");
    uint64_t want = (n_items + lv->bd - 1) / lv->bd;
    int lgrid = (int)std::max<uint64_t>(1, std::min<uint64_t>(want, (uint64_t)h->sm_count * bps));
    const uint64_t lwarps = (uint64_t)lgrid * (lv->bd / 32);
    if ((rc = h->lane_pend.grow(h, lwarps * lv->lpcap * 32 * sizeof(uint4))) != DEMI_OK) return rc;
    if ((rc = h->ovf_list.grow(h, std::max<size_t>(n_items * sizeof(uint32_t), 64))) != DEMI_OK) return rc;
    CUDA_TRY(h, cudaMemsetAsync(h->ovf_count.get(), 0, sizeof(uint32_t), s));
    KernelArgs la = a;
    la.lane_pend = h->lane_pend.get<uint4>();
    // a campaign and a launch of many traces' tests bind each program's table
    la.ext_sends = plan.mode == LM_PROGRAM || plan.mode == LM_TEST_PARAMS ? nullptr : h->ext_sends_dev.get<uint4>();
    la.has_partitions = plan.prog->partitions ? 1u : 0u;
    la.prog_lane_pcap = h->lane_pending_cap;
    la.ovf_list = h->ovf_list.get<uint32_t>(); la.ovf_count = h->ovf_count.get<uint32_t>();
    if (h->lane_pending_cap) la.pending_cap = std::min(la.pending_cap, h->lane_pending_cap);     // deferring is always exact
    if (steady) {
      la.pending_cap = lane_pcap;                    // one bound, rows included
      la.lane_snap = h->lane_snap_dev.get<LaneSnapshot>();
      if ((rc = lane_tree(h, lv, la, s)) != DEMI_OK) return rc;
    }
    lfn<<<lgrid, lv->bd, lsmem, s>>>(la);
    CUDA_TRY(h, cudaGetLastError());
    h->lane_kernel = steady ? DEMI_LANE_STEADY : DEMI_LANE_GENERIC;
    h->lane_row_bytes = row8 ? 8 : 16;
    h->lane_tree_depth = steady ? (int32_t)h->lane_snap.depth : -1;
    h->perf.kernel_launches++;
    // what the lane engine could not prove exact: a recording launch numbers its outputs by work-list position
    if (plan.mode == LM_RECORD) { a.pos_list = la.ovf_list; a.pos_count = la.ovf_count; }
    else { a.index_list = la.ovf_list; a.index_count = la.ovf_count; }
  }
  if (h->cfg.model == DEMI_MODEL_IR) CUDA_TRY(h, ir_bind(h->ir_dev, s));
  plan.v->fn[plan.mode]<<<plan.grid, WARPS * 32, plan.smem, s>>>(a);
  CUDA_TRY(h, cudaGetLastError());
  h->perf.kernel_launches++;
  return DEMI_OK;
}

// A new batch: its counters and counts start from zero (an empty batch, too, reports its own); demi_fuzz_summary_dev,
// or the host path once it syncs, fills the rest.
static int32_t reset_batch(demi_handle* h, cudaStream_t s) {
  CUDA_TRY(h, cudaMemsetAsync(h->counters_dev.get(), 0, 4 * sizeof(unsigned long long), s));
  h->perf.kernel_launches = 0;
  h->perf.prefixes = 0;
  h->perf.deliveries = 0;
  h->perf.violations = 0;
  h->perf.deferred = 0;
  return DEMI_OK;
}

// demi_perf's counts from the engines' counters: deliveries, violations, and prefixes deferred to the warp engine
static void read_counters(demi_handle* h, const unsigned long long* c) {
  h->perf.deliveries = c[0];
  h->perf.violations = c[1];
  h->perf.deferred = (uint32_t)std::min<unsigned long long>(c[2], 0xFFFFFFFFull);
}

static int32_t launch_fuzz(demi_handle* h, const demi_fuzz_params* p, void* out_dev, void* stream, bool reset_counters) {
  if (!h) return DEMI_ERR_INVALID;
  if (!out_dev) return fail(h, DEMI_ERR_INVALID, "demi_fuzz_batch_dev: null output");
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  LaunchPlan plan;
  int32_t rc = plan_launch(h, p, LM_BATCH, h->ext_info, h->ext_dev.get<demi_ext_event>(), (uint32_t)h->ext_host.size(), &plan);
  if (rc != DEMI_OK) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  if (reset_counters && (rc = reset_batch(h, s)) != DEMI_OK) return rc;
  if (p->n_prefixes == 0) return DEMI_OK;
  plan.args.results = (demi_fuzz_result*)out_dev;
  if ((rc = launch_plan(h, plan, p->n_prefixes, s)) != DEMI_OK) return rc;
  h->perf.prefixes += p->n_prefixes;
  return DEMI_OK;
}

extern "C" int32_t demi_fuzz_batch_dev(demi_handle* h, const demi_fuzz_params* p, void* out_dev, void* stream) {
  return launch_fuzz(h, p, out_dev, stream, true);
}

// Runs n records in chunks of `per` through launch(off, m, dst, first_chunk) on h->stream; chunk i's records travel to
// the host on the copy stream while chunk i+1 is being explored.  Fills demi_perf (kernel_ms spans every launch).
template <class Launch>
static int32_t run_pipelined(demi_handle* h, const char* who, uint64_t n, uint64_t per, demi_fuzz_result* out_host, Launch launch) {
  const size_t bytes = (size_t)n * sizeof(demi_fuzz_result);
  int32_t rc = h->results_dev.grow(h, std::max<size_t>(bytes, 32));
  if (rc != DEMI_OK) return rc;
  demi_fuzz_result* results = h->results_dev.get<demi_fuzz_result>();
  CUDA_TRY(h, cudaEventRecord(h->ev0, h->stream));
  if (n == 0) { rc = launch(0, 0, results, true); if (rc != DEMI_OK) return rc; }
  std::vector<cudaEvent_t> evs;
  for (uint64_t off = 0; off < n; off += per) {
    const uint64_t m = std::min<uint64_t>(per, n - off);
    rc = launch(off, m, results + off, off == 0);
    if (rc != DEMI_OK) break;
    cudaEvent_t ev;
    cudaError_t ce = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    if (ce == cudaSuccess) {
      evs.push_back(ev);
      ce = cudaEventRecord(ev, h->stream);
      if (ce == cudaSuccess) ce = cudaStreamWaitEvent(h->copy_stream, ev, 0);
      if (ce == cudaSuccess) ce = cudaMemcpyAsync(out_host + off, results + off, m * sizeof(demi_fuzz_result),
                                                  cudaMemcpyDeviceToHost, h->copy_stream);
    }
    if (ce != cudaSuccess) { rc = fail(h, DEMI_ERR_CUDA, "%s: %s", who, cudaGetErrorString(ce)); break; }   // events freed below
  }
  cudaError_t e = cudaEventRecord(h->ev1, h->stream);
  unsigned long long cnt[3] = {0, 0, 0};
  if (e == cudaSuccess) e = cudaMemcpyAsync(cnt, h->counters_dev.get(), sizeof(cnt), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->copy_stream);
  for (cudaEvent_t ev : evs) cudaEventDestroy(ev);
  if (rc != DEMI_OK) return rc;
  if (e != cudaSuccess) return fail(h, DEMI_ERR_CUDA, "%s: %s", who, cudaGetErrorString(e));
  float ms = 0;
  CUDA_TRY(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  h->perf.kernel_ms = ms;
  read_counters(h, cnt);
  h->perf.d2h_bytes = bytes + sizeof(cnt);
  h->perf.h2d_bytes = 0;
  return DEMI_OK;
}

extern "C" int32_t demi_fuzz_batch(demi_handle* h, const demi_fuzz_params* p, demi_fuzz_result* out_host) {
  if (!h) return DEMI_ERR_INVALID;
  if (!out_host) return fail(h, DEMI_ERR_INVALID, "demi_fuzz_batch: null output");
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  if (!p) return fail(h, DEMI_ERR_INVALID, "null params");
  const uint64_t CHUNK = 2u << 20;
  const uint64_t n = p->n_prefixes;
  const uint64_t n_chunks = n <= 2 * CHUNK ? 1 : (n + CHUNK - 1) / CHUNK;
  const uint64_t per = n_chunks ? (n + n_chunks - 1) / n_chunks : 0;
  return run_pipelined(h, "demi_fuzz_batch", n, per, out_host, [&](uint64_t off, uint64_t m, demi_fuzz_result* dst, bool first) {
    demi_fuzz_params q = *p;
    q.seed_base = seed_at(p->seed_base, off);
    q.n_prefixes = m;
    return launch_fuzz(h, &q, dst, h->stream, first);
  });
}

// Counts from the last *_dev batch launched on `stream` (waits for it).
extern "C" int32_t demi_fuzz_summary_dev(demi_handle* h, const void* /*results_dev*/, uint64_t /*n*/,
                                         void* stream, uint64_t* n_violations, uint64_t* sum_steps) {
  if (!h) return DEMI_ERR_INVALID;
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  unsigned long long c[3] = {0, 0, 0};
  CUDA_TRY(h, cudaMemcpyAsync(c, h->counters_dev.get(), sizeof(c), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  CUDA_TRY(h, cudaStreamSynchronize((cudaStream_t)stream));
  if (sum_steps) *sum_steps = c[0];
  if (n_violations) *n_violations = c[1];
  read_counters(h, c);
  return DEMI_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Recording: the records both engines write in an LM_RECORD launch (KernelArgs::rec_*) and the provenance kernel
// reads.  Slot i owns events[i*rec_cap ..), parents[i*par_cap ..), counts[i*4 ..) = {n_events, n_nodes, affectedNodes,
// violation} and results[i]; with a work list it runs execution seed_base + list[i], else seed_base + i.
struct Records {
  demi_event* events; uint16_t* parents; uint32_t* counts; demi_fuzz_result* results;
  unsigned char* extra; uint32_t rec_cap, par_cap;      // extra: the caller's bytes per slot, after the records
};

static size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

// Slots per recording launch, so that what stage_records lays out (`extra` per slot included) stays within ~4 GB
static uint32_t record_chunk(uint32_t rec_cap, uint32_t par_cap, size_t extra) {
  const size_t per_slot = (size_t)rec_cap * sizeof(demi_event) + (size_t)par_cap * 2 + 16 + sizeof(demi_fuzz_result) + 4;
  return (uint32_t)std::max<size_t>(1, ((size_t)4 << 30) / (per_slot + extra));
}

// Lays out the records of n slots in `buf`, grown to fit, each region 16-byte aligned: events | parents | counts |
// results | work list | its length | `extra` bytes per slot.  par_cap 0 records no parents (the warp engine alone
// allows it).  With a work list (`list`, n host entries) the list is uploaded, counts and results start cleared and
// the launch leaves the handle's counters alone.  Binds plan->args when a plan is given.
static int32_t stage_records(demi_handle* h, LaunchPlan* plan, uint32_t n, const uint32_t* list, uint32_t rec_cap,
                             uint32_t par_cap, size_t extra, DevBuf& buf, Records* r, cudaStream_t s) {
  const size_t b_ev = (size_t)n * rec_cap * sizeof(demi_event), b_par = align16((size_t)n * par_cap * 2), b_cnt = (size_t)n * 16,
               b_res = (size_t)n * sizeof(demi_fuzz_result), b_list = align16((size_t)n * 4);
  const int32_t rc = buf.grow(h, b_ev + b_par + b_cnt + b_res + b_list + 16 + (size_t)n * extra);
  if (rc != DEMI_OK) return rc;
  unsigned char* p = buf.get<unsigned char>();
  r->events = (demi_event*)p;          p += b_ev;
  r->parents = (uint16_t*)p;           p += b_par;
  r->counts = (uint32_t*)p;            p += b_cnt;
  r->results = (demi_fuzz_result*)p;   p += b_res;
  uint32_t* d_list = (uint32_t*)p;     p += b_list;
  uint32_t* d_len = (uint32_t*)p;      p += 16;
  r->extra = p; r->rec_cap = rec_cap; r->par_cap = par_cap;
  if (list) {
    CUDA_TRY(h, cudaMemcpyAsync(d_list, list, (size_t)n * 4, cudaMemcpyHostToDevice, s));
    CUDA_TRY(h, cudaMemcpyAsync(d_len, &n, 4, cudaMemcpyHostToDevice, s));
    CUDA_TRY(h, cudaMemsetAsync(r->counts, 0, b_cnt, s));
    CUDA_TRY(h, cudaMemsetAsync(r->results, 0xFF, b_res, s));
  }
  if (plan) {
    KernelArgs& a = plan->args;
    a.results = r->results; a.rec_counts = r->counts;
    a.rec_events = r->events; a.rec_cap = rec_cap;
    a.rec_parent = par_cap ? r->parents : nullptr; a.rec_parent_cap = par_cap;
    if (list) { a.index_list = d_list; a.index_count = d_len; a.sum_steps = nullptr; a.n_violations = nullptr; }
  }
  return DEMI_OK;
}

// demi_fuzz_trace over the program (ext, n_ext) that `prog` describes: one prefix, recorded by the warp engine
static int32_t fuzz_trace(demi_handle* h, const demi_fuzz_params* p, int64_t seed, demi_event* events, uint32_t cap_events,
                          uint32_t* n_events, uint16_t* dep_parent, uint32_t cap_nodes, uint32_t* n_nodes, demi_fuzz_result* result,
                          const demi_ext_event* ext, uint32_t n_ext, const ProgramInfo& prog) {
  if (!p) return fail(h, DEMI_ERR_INVALID, "null params");
  if (!events || !cap_events) return fail(h, DEMI_ERR_INVALID, "demi_fuzz_trace: events buffer required");
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  demi_fuzz_params q = *p;
  q.seed_base = seed; q.n_prefixes = 1;
  LaunchPlan plan;
  int32_t rc = plan_launch(h, &q, LM_RECORD, prog, ext, n_ext, &plan);
  if (rc != DEMI_OK) return rc;
  Records rec;
  if ((rc = stage_records(h, &plan, 1, nullptr, cap_events, dep_parent ? cap_nodes : 0, 0, h->trace_rec, &rec, h->stream)) != DEMI_OK) return rc;
  CUDA_TRY(h, cudaMemsetAsync(h->counters_dev.get(), 0, 4 * sizeof(unsigned long long), h->stream));
  if (h->cfg.model == DEMI_MODEL_IR) CUDA_TRY(h, ir_bind(h->ir_dev, h->stream));
  plan.v->fn[LM_RECORD]<<<1, WARPS * 32, plan.smem, h->stream>>>(plan.args);
  cudaError_t e = cudaGetLastError();
  struct { uint32_t counts[4]; demi_fuzz_result r; } got{};          // one slot's counts and result lie side by side
  if (e == cudaSuccess) e = cudaMemcpyAsync(&got, rec.counts, sizeof(got), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e == cudaSuccess && got.r.status == 0) {
    e = cudaMemcpy(events, rec.events, (size_t)std::min(got.counts[0], cap_events) * sizeof(demi_event), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && dep_parent)
      e = cudaMemcpy(dep_parent, rec.parents, (size_t)std::min(got.counts[1], cap_nodes) * sizeof(uint16_t), cudaMemcpyDeviceToHost);
  }
  if (e != cudaSuccess) return fail(h, DEMI_ERR_CUDA, "demi_fuzz_trace: %s", cudaGetErrorString(e));
  if (n_events) *n_events = got.counts[0];
  if (n_nodes) *n_nodes = got.counts[1];
  if (result) *result = got.r;
  if (got.r.status) return fail(h, DEMI_ERR_CAPACITY, "demi_fuzz_trace: prefix status %u", (unsigned)got.r.status);
  return DEMI_OK;
}

extern "C" int32_t demi_fuzz_trace(demi_handle* h, const demi_fuzz_params* p, int64_t seed,
                                   demi_event* events, uint32_t cap_events, uint32_t* n_events,
                                   uint16_t* dep_parent, uint32_t cap_nodes, uint32_t* n_nodes,
                                   demi_fuzz_result* result) {
  if (!h) return DEMI_ERR_INVALID;
  return fuzz_trace(h, p, seed, events, cap_events, n_events, dep_parent, cap_nodes, n_nodes, result, h->ext_dev.get<demi_ext_event>(),
                    (uint32_t)h->ext_host.size(), h->ext_info);
}

// ---------------------------------------------------------------------------------------------------------
// Provenance pruning (ProvenanceTracker, schedulers/Util.scala:267-376)
static size_t prune_bytes(uint32_t mask_words) { return (size_t)mask_words * 8 + sizeof(demi_provenance_out); }

// Prunes n staged records into their `extra` bytes, prune_bytes(mask_words) per slot: keep masks | outputs (a record with
// a status is skipped unless r.results is null).  Queues their copies to the host, the results' when `results` is given;
// `timed` records h->ev1 after the kernel.
static int32_t prune_records(demi_handle* h, const Records& r, uint32_t n, uint32_t mask_words, uint64_t* keep_masks,
                             demi_provenance_out* out, demi_fuzz_result* results, bool timed, cudaStream_t s) {
  constexpr int PW = 4;
  ProvArgs a{};
  a.events = r.events; a.ev_stride = r.rec_cap;
  a.parent = r.parents; a.par_stride = r.par_cap;
  a.counts = r.counts; a.results = r.results;
  a.keep = (uint64_t*)r.extra; a.mask_words = mask_words;
  a.out = (demi_provenance_out*)(r.extra + (size_t)n * mask_words * 8); a.n = n;
  a.t_cap = mask_words * 64;
  a.scratch_stride = a.t_cap + 3 * a.par_stride;
  const uint64_t want = ((uint64_t)n + PW - 1) / PW;
  const int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>(want, (uint64_t)h->sm_count * 8));
  int32_t rc = h->prov_scratch.grow(h, (uint64_t)grid * PW * a.scratch_stride * sizeof(uint32_t));
  if (rc != DEMI_OK) return rc;
  a.scratch = h->prov_scratch.get<uint32_t>();
  provenance_kernel<PW><<<grid, PW * 32, 0, s>>>(a);
  CUDA_TRY(h, cudaGetLastError());
  h->perf.kernel_launches++;
  if (timed) CUDA_TRY(h, cudaEventRecord(h->ev1, s));
  CUDA_TRY(h, cudaMemcpyAsync(keep_masks, a.keep, (size_t)n * mask_words * 8, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaMemcpyAsync(out, a.out, (size_t)n * sizeof(demi_provenance_out), cudaMemcpyDeviceToHost, s));
  if (results) CUDA_TRY(h, cudaMemcpyAsync(results, r.results, (size_t)n * sizeof(demi_fuzz_result), cudaMemcpyDeviceToHost, s));
  return DEMI_OK;
}

extern "C" int32_t demi_provenance(demi_handle* h, const demi_event* events, uint32_t n_events,
                                   const uint16_t* dep_parent, uint32_t n_nodes, uint32_t affected_mask,
                                   uint64_t* keep_mask, uint32_t mask_words, demi_provenance_out* out) {
  if (!h) return DEMI_ERR_INVALID;
  if (!events || !dep_parent || !keep_mask || !out || !mask_words || !n_nodes)
    return fail(h, DEMI_ERR_INVALID, "demi_provenance: events, dep_parent, keep_mask and out are required");
  if (n_nodes > 65536) return fail(h, DEMI_ERR_INVALID, "demi_provenance: node ids are 16-bit");
  { int32_t vrc = demi_check_events(h, "demi_provenance", events, n_events, n_nodes, DEMI_MAX_ACTORS); if (vrc != DEMI_OK) return vrc;
    vrc = demi_check_parents(h, "demi_provenance", dep_parent, n_nodes); if (vrc != DEMI_OK) return vrc; }
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  // the caller's trace as the record of one slot: its events, its parents and the counts a recording would have
  DevBuf tmp;
  Records rec;
  int32_t rc = stage_records(h, nullptr, 1, nullptr, std::max(n_events, 1u), n_nodes, prune_bytes(mask_words), tmp, &rec, h->stream);
  if (rc != DEMI_OK) return rc;
  rec.results = nullptr;                   // no result record: nothing is skipped
  const uint32_t counts[4] = {n_events, n_nodes, affected_mask, 0};
  CUDA_TRY(h, cudaMemcpyAsync(rec.events, events, (size_t)n_events * sizeof(demi_event), cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(rec.parents, dep_parent, (size_t)n_nodes * 2, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(rec.counts, counts, sizeof(counts), cudaMemcpyHostToDevice, h->stream));
  if ((rc = prune_records(h, rec, 1, mask_words, keep_mask, out, nullptr, false, h->stream)) != DEMI_OK) return rc;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return DEMI_OK;
}

extern "C" int32_t demi_fuzz_provenance(demi_handle* h, const demi_fuzz_params* p, const uint32_t* prefix_index, uint32_t n,
                                        uint64_t* keep_masks, uint32_t mask_words, demi_provenance_out* out,
                                        demi_fuzz_result* results) {
  if (!h) return DEMI_ERR_INVALID;
  if (!p) return fail(h, DEMI_ERR_INVALID, "null params");
  if (!n) return DEMI_OK;
  if (!prefix_index || !keep_masks || !out || !mask_words)
    return fail(h, DEMI_ERR_INVALID, "demi_fuzz_provenance: prefix_index, keep_masks and out are required");
  if (p->max_messages < 0 || (uint64_t)p->max_messages + 2 > (uint64_t)mask_words * 64)
    return fail(h, DEMI_ERR_INVALID, "demi_fuzz_provenance: mask_words*64 must cover max_messages + 2 positions");
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  demi_fuzz_params q = *p;
  q.n_prefixes = n;
  LaunchPlan plan;
  int32_t rc = plan_launch(h, &q, LM_RECORD, h->ext_info, h->ext_dev.get<demi_ext_event>(), (uint32_t)h->ext_host.size(), &plan);
  if (rc != DEMI_OK) return rc;
  // an execution records at most one MsgSend + one MsgEvent per message, plus the external markers
  const uint32_t node_cap = plan.args.node_cap;
  const uint32_t ev_cap = 2 * node_cap + 2 * plan.args.n_ext + 16;
  const size_t extra = prune_bytes(mask_words);
  const uint32_t chunk = record_chunk(ev_cap, node_cap, extra);
  cudaStream_t s = h->stream;
  DevBuf buf;
  float ms_all = 0.f;
  h->perf.kernel_launches = 0;
  for (uint32_t off = 0; off < n; off += chunk) {
    const uint32_t m = std::min(chunk, n - off);
    q.n_prefixes = m;                      // a chunk of a larger request plans its own grid
    if (m < n && (rc = plan_launch(h, &q, LM_RECORD, h->ext_info, h->ext_dev.get<demi_ext_event>(), (uint32_t)h->ext_host.size(), &plan)))
      return rc;
    Records rec;
    if ((rc = stage_records(h, &plan, m, prefix_index + off, ev_cap, node_cap, extra, buf, &rec, s)) != DEMI_OK) return rc;
    CUDA_TRY(h, cudaEventRecord(h->ev0, s));
    // the lane engine records every execution it can prove exact; the slots it defers go to the general engine
    if ((rc = launch_plan(h, plan, m, s)) != DEMI_OK) return rc;
    if ((rc = prune_records(h, rec, m, mask_words, keep_masks + (size_t)off * mask_words, out + off, results ? results + off : nullptr,
                            true, s)) != DEMI_OK) return rc;
    CUDA_TRY(h, cudaStreamSynchronize(s));
    float ms = 0.f;
    CUDA_TRY(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
    ms_all += ms;
  }
  h->perf.prefixes = n;
  h->perf.kernel_ms = ms_all;
  return DEMI_OK;
}

// The EventTraces of executions seed_base + prefix_index[i], recorded as demi_fuzz_provenance records them (the lane
// engine first, the slots it defers on the general engine): the events of execution i go to events + i*cap_events, its
// count to n_events[i] and its record to results[i] (may be NULL).  With dep_parent, its DepTracker tree goes to
// dep_parent + i*cap_nodes and its node count to n_nodes[i]; without, one parent entry per slot is staged and the tree
// is not returned.
static int32_t fuzz_traces(demi_handle* h, const char* who, const demi_fuzz_params* p, const uint32_t* prefix_index, uint32_t n,
                           demi_event* events, uint32_t cap_events, uint32_t* n_events, uint16_t* dep_parent, uint32_t cap_nodes,
                           uint32_t* n_nodes, demi_fuzz_result* results) {
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  const uint32_t par_cap = dep_parent ? cap_nodes : 1;
  const uint32_t chunk = record_chunk(cap_events, par_cap, 0);
  cudaStream_t s = h->stream;
  DevBuf buf;
  int32_t rc;
  float ms_all = 0.f;
  int64_t bad = -1;
  uint32_t bad_status = 0;
  std::vector<demi_fuzz_result> res;
  std::vector<uint32_t> cnt;
  h->perf.kernel_launches = 0;
  for (uint32_t off = 0; off < n; off += chunk) {
    const uint32_t m = std::min(chunk, n - off);
    demi_fuzz_params q = *p;
    q.n_prefixes = m;
    LaunchPlan plan;
    if ((rc = plan_launch(h, &q, LM_RECORD, h->ext_info, h->ext_dev.get<demi_ext_event>(), (uint32_t)h->ext_host.size(), &plan)) != DEMI_OK)
      return rc;
    Records rec;
    if ((rc = stage_records(h, &plan, m, prefix_index + off, cap_events, par_cap, 0, buf, &rec, s)) != DEMI_OK) return rc;
    CUDA_TRY(h, cudaEventRecord(h->ev0, s));
    if ((rc = launch_plan(h, plan, m, s)) != DEMI_OK) return rc;
    CUDA_TRY(h, cudaEventRecord(h->ev1, s));
    res.resize(m); cnt.resize((size_t)m * 4);
    CUDA_TRY(h, cudaMemcpyAsync(cnt.data(), rec.counts, cnt.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(h, cudaMemcpyAsync(res.data(), rec.results, res.size() * sizeof(demi_fuzz_result), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(h, cudaStreamSynchronize(s));
    float ms = 0.f;
    CUDA_TRY(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
    ms_all += ms;
    // the events (and parents) travel as rows as wide as the longest successful recording; a failing execution's
    // partial recording is zeroed first, so that it returns no events
    uint32_t width = 0, pwidth = 0;
    for (uint32_t i = 0; i < m; i++) {
      n_events[off + i] = cnt[(size_t)i * 4];
      if (n_nodes) n_nodes[off + i] = cnt[(size_t)i * 4 + 1];
      if (results) results[off + i] = res[i];
      if (res[i].status) {
        if (bad < 0) { bad = off + i; bad_status = res[i].status; }
        CUDA_TRY(h, cudaMemsetAsync(rec.events + (size_t)i * cap_events, 0, (size_t)cap_events * sizeof(demi_event), s));
        if (dep_parent) CUDA_TRY(h, cudaMemsetAsync(rec.parents + (size_t)i * par_cap, 0, (size_t)par_cap * sizeof(uint16_t), s));
      } else {
        width = std::max(width, std::min(cnt[(size_t)i * 4], cap_events));
        pwidth = std::max(pwidth, std::min(cnt[(size_t)i * 4 + 1], par_cap));
      }
    }
    if (width) {
      const size_t pitch = (size_t)cap_events * sizeof(demi_event);
      CUDA_TRY(h, cudaMemcpy2DAsync(events + (size_t)off * cap_events, pitch, rec.events, pitch, (size_t)width * sizeof(demi_event), m,
                                    cudaMemcpyDeviceToHost, s));
    }
    if (dep_parent && pwidth) {
      const size_t pitch = (size_t)par_cap * sizeof(uint16_t);
      CUDA_TRY(h, cudaMemcpy2DAsync(dep_parent + (size_t)off * par_cap, pitch, rec.parents, pitch, (size_t)pwidth * sizeof(uint16_t), m,
                                    cudaMemcpyDeviceToHost, s));
    }
    if (width || (dep_parent && pwidth)) CUDA_TRY(h, cudaStreamSynchronize(s));
  }
  h->perf.prefixes = n;
  h->perf.kernel_ms = ms_all;
  // as demi_fuzz_trace fails for that seed; every record is filled all the same
  if (bad >= 0)
    return fail(h, DEMI_ERR_CAPACITY, "%s: execution %lld (prefix %u) status %u", who, (long long)bad, prefix_index[bad], bad_status);
  return DEMI_OK;
}

extern "C" int32_t demi_fuzz_traces(demi_handle* h, const demi_fuzz_params* p, const uint32_t* prefix_index, uint32_t n,
                                    demi_event* events, uint32_t cap_events, uint32_t* n_events, demi_fuzz_result* results) {
  if (!h) return DEMI_ERR_INVALID;
  if (!p) return fail(h, DEMI_ERR_INVALID, "null params");
  if (!n) return DEMI_OK;
  if (!prefix_index || !events || !cap_events || !n_events)
    return fail(h, DEMI_ERR_INVALID, "demi_fuzz_traces: prefix_index, events, cap_events and n_events are required");
  return fuzz_traces(h, "demi_fuzz_traces", p, prefix_index, n, events, cap_events, n_events, nullptr, 0, nullptr, results);
}

extern "C" int32_t demi_fuzz_traces_tree(demi_handle* h, const demi_fuzz_params* p, const uint32_t* prefix_index, uint32_t n,
                                         demi_event* events, uint32_t cap_events, uint32_t* n_events,
                                         uint16_t* dep_parent, uint32_t cap_nodes, uint32_t* n_nodes, demi_fuzz_result* results) {
  if (!h) return DEMI_ERR_INVALID;
  if (!p) return fail(h, DEMI_ERR_INVALID, "null params");
  if (!n) return DEMI_OK;
  if (!prefix_index || !events || !cap_events || !n_events || !dep_parent || !cap_nodes || !n_nodes)
    return fail(h, DEMI_ERR_INVALID,
                "demi_fuzz_traces_tree: prefix_index, events, cap_events, n_events, dep_parent, cap_nodes and n_nodes are required");
  return fuzz_traces(h, "demi_fuzz_traces_tree", p, prefix_index, n, events, cap_events, n_events, dep_parent, cap_nodes, n_nodes,
                     results);
}

// ---------------------------------------------------------------------------------------------------------
// Campaigns: RunnerUtils.fuzz's loop (RunnerUtils.scala:75-91) with a fresh Fuzzer program per execution.
// Execution i runs program fuzzer_generate(program_seed_base + i) under FullyRandom(seed_base + i).

// the message-type ids a model defines (send_type must be one of them)
static uint32_t model_type_count(const demi_handle* h) {
  switch (h->cfg.model) {
    case DEMI_MODEL_PINGPONG3: return 3;
    case DEMI_MODEL_RAFT5: return 9;
    case DEMI_MODEL_BCAST32: return 3;
    default: return h->ir_n_types;
  }
}

// new Fuzzer(num_events, weights, message_gen, prefix, postfix) (Fuzzer.scala:61-82): checked once here for what
// would make one of its programs fail demi_set_externals, so that every generated program is a valid one.
extern "C" int32_t demi_set_fuzzer(demi_handle* h, const demi_fuzzer_config* cfg, const demi_ext_event* prefix, uint32_t n_prefix,
                                   const demi_ext_event* postfix, uint32_t n_postfix) {
  if (!h) return DEMI_ERR_INVALID;
  if (!cfg || (!prefix && n_prefix) || (!postfix && n_postfix)) return fail(h, DEMI_ERR_INVALID, "demi_set_fuzzer: null argument");
  { int32_t mrc = demi_need_model(h); if (mrc != DEMI_OK) return mrc; }
  uint32_t starts = 0;
  ProgramInfo info;
  std::vector<uint4> sv;
  for (int part = 0; part < 2; part++) {
    const demi_ext_event* ev = part ? postfix : prefix;
    const uint32_t n = part ? n_postfix : n_prefix;
    for (uint32_t i = 0; i < n; i++) {
      const demi_ext_event& e = ev[i];
      const int32_t rc = demi_check_external(h, "demi_set_fuzzer", part ? "postfix " : "prefix ", ev, i, true, true);
      if (rc != DEMI_OK) return rc;
      if (!part && e.kind == DEMI_EXT_START) starts++;
      describe_event(&info, &sv, e);
      // the lane engine's screen (demi_set_externals): no two Sends of a program may be equal.  A generated Send is
      // (alive actor, send_type, p0 = counter in 1..num_events, p1 = 0); a fixed Send that could equal one screens
      // the campaign out, whichever actor the generated one picks.
      if (e.kind == DEMI_EXT_SEND && cfg->send > 0.0 && e.type == cfg->send_type && e.p1 == 0 && e.p0 >= 1 && e.p0 <= cfg->num_events)
        info.sends_distinct = false;
    }
  }
  if (!starts) return fail(h, DEMI_ERR_INVALID, "demi_set_fuzzer: the prefix has no Start (the Fuzzer's actors are the prefix's Starts, Fuzzer.scala:60)");
  if (starts > DEMI_MAX_ACTORS) return fail(h, DEMI_ERR_INVALID, "demi_set_fuzzer: %u Starts in the prefix, at most %d", starts, DEMI_MAX_ACTORS);
  if (n_postfix && postfix[0].kind == DEMI_EXT_WAIT_QUIESCENCE)
    return fail(h, DEMI_ERR_INVALID, "demi_set_fuzzer: the postfix begins with WaitQuiescence (it may follow a generated one)");
  if (cfg->send_type >= model_type_count(h))
    return fail(h, DEMI_ERR_INVALID, "demi_set_fuzzer: send_type %u is not a message type of the model", cfg->send_type);
  const double w[5] = {cfg->kill, cfg->send, cfg->wait_quiescence, cfg->partition, cfg->unpartition};
  double total = 0.0;
  for (double x : w) {
    if (!std::isfinite(x) || x < 0.0) return fail(h, DEMI_ERR_INVALID, "demi_set_fuzzer: weights must be finite and >= 0");
    total += x;
  }
  if (!(total > 0.0)) return fail(h, DEMI_ERR_INVALID, "demi_set_fuzzer: the weights add up to 0");
  if (cfg->num_events > DEMI_FUZZER_MAX_EVENTS)
    return fail(h, DEMI_ERR_INVALID, "demi_set_fuzzer: num_events %u, at most %d", cfg->num_events, DEMI_FUZZER_MAX_EVENTS);
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  std::vector<demi_ext_event> fixed(prefix, prefix + n_prefix);
  if (n_postfix) fixed.insert(fixed.end(), postfix, postfix + n_postfix);
  DevBuf fixed_dev;                      // n_prefix >= 1: the prefix has a Start
  const int32_t rc = fixed_dev.upload(h, fixed.data(), fixed.size() * sizeof(demi_ext_event));
  if (rc != DEMI_OK) return rc;
  h->fz_fixed_dev = std::move(fixed_dev);
  h->fuzzer = *cfg; h->fz_n_prefix = n_prefix; h->fz_n_postfix = n_postfix;
  info.sends += cfg->num_events;                 // the largest program's
  info.partitions |= cfg->partition > 0.0;
  h->fz_info = info;
  h->has_fuzzer = true;
  return DEMI_OK;
}

// One thread per program: program i of the chunk goes to events[i * stride ..), its {length, Sends} to hdr[i] and its
// Sends, in the lane engine's form, to sends[i * send_stride ..).  The three sets live in local memory.
__global__ void __launch_bounds__(128)
fuzzer_gen_kernel(const demi_fuzzer_config cfg, int64_t seed_base, uint64_t n, const demi_ext_event* fixed, uint32_t n_prefix,
                  uint32_t n_postfix, demi_ext_event* events, uint32_t stride, uint2* hdr, uint4* sends, uint32_t send_stride) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t alive[DEMI_MAX_ACTORS];
  uint16_t pairs[2 * (DEMI_MAX_ACTORS * (DEMI_MAX_ACTORS - 1) / 2)];
  demi_ext_event* out = events + i * stride;
  uint32_t n_sends = 0;
  const uint32_t len = demi::fuzzer_generate(cfg, seed_at(seed_base, i), fixed, n_prefix, fixed + n_prefix, n_postfix, alive, pairs,
                                             out, &n_sends);
  hdr[i] = make_uint2(len, n_sends);
  uint4* st = sends + i * send_stride;
  for (uint32_t j = 0, k = 0; j < len; j++) {
    const demi_ext_event e = out[j];
    if (e.kind == DEMI_EXT_SEND) st[k++] = lane_send(e);
  }
}

// The arena in h->fz_arena of `n` programs, as the PROG engines read them: program i's events at ev[i * stride ..),
// hdr[i] = {length, Sends}, its lane-form Sends at sends[i * send_stride ..); then `extra` bytes for the caller at *rest.
struct ProgramArena { demi_ext_event* ev; uint2* hdr; uint4* sends; uint32_t stride, send_stride; };
static int32_t carve_programs(demi_handle* h, uint64_t n, uint32_t stride, uint32_t send_stride, size_t extra, ProgramArena* pa,
                              unsigned char** rest = nullptr) {
  const size_t b_ev = (size_t)n * stride * sizeof(demi_ext_event), b_hdr = ((size_t)n * sizeof(uint2) + 15) & ~(size_t)15,
               b_snd = (size_t)n * send_stride * sizeof(uint4);
  int32_t rc = h->fz_arena.grow(h, b_ev + b_hdr + b_snd + extra);
  if (rc != DEMI_OK) return rc;
  unsigned char* a0 = h->fz_arena.get<unsigned char>();
  *pa = ProgramArena{(demi_ext_event*)a0, (uint2*)(a0 + b_ev), (uint4*)(a0 + b_ev + b_hdr), stride, send_stride};
  if (rest) *rest = a0 + b_ev + b_hdr + b_snd;
  return DEMI_OK;
}
static void bind_programs(const demi_handle* h, KernelArgs& a, const ProgramArena& pa, int32_t max_messages) {
  a.prog_ext = pa.ev; a.prog_hdr = pa.hdr; a.prog_sends = pa.sends;
  a.prog_stride = pa.stride; a.prog_send_stride = pa.send_stride;
  a.prog_model_key = demi_model_key(h);
  a.prog_max_messages = max_messages;
}

// programs per launch: the arena of one chunk stays under 512 MB
static uint64_t campaign_chunk(const demi_handle* h, uint32_t* stride, uint32_t* send_stride) {
  *stride = (uint32_t)demi::fuzzer_program_room(h->fuzzer, h->fz_n_prefix, h->fz_n_postfix);
  *send_stride = std::max(h->fz_info.sends, 1u);
  const uint64_t per = (uint64_t)*stride * sizeof(demi_ext_event) + sizeof(uint2) + (uint64_t)*send_stride * sizeof(uint4);
  return std::max<uint64_t>(1, std::min<uint64_t>(2u << 20, ((uint64_t)512 << 20) / per));
}

// One chunk (n_prefixes <= campaign_chunk): generate its programs, then the lane engine, then the warp engine on what
// the lane engine deferred (or on all of them).
static int32_t launch_campaign(demi_handle* h, const demi_fuzz_params* p, int64_t program_seed_base, void* out_dev, cudaStream_t s,
                               bool reset_counters) {
  LaunchPlan plan;
  int32_t rc = plan_launch(h, p, LM_PROGRAM, h->fz_info, nullptr, 0, &plan);
  if (rc != DEMI_OK) return rc;
  const uint64_t n = p->n_prefixes;
  if (reset_counters && (rc = reset_batch(h, s)) != DEMI_OK) return rc;
  if (n == 0) return DEMI_OK;
  uint32_t stride, send_stride;
  campaign_chunk(h, &stride, &send_stride);
  ProgramArena pa;
  if ((rc = carve_programs(h, n, stride, send_stride, 0, &pa)) != DEMI_OK) return rc;
  fuzzer_gen_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(h->fuzzer, program_seed_base, n, h->fz_fixed_dev.get<demi_ext_event>(), h->fz_n_prefix,
                                                                 h->fz_n_postfix, pa.ev, stride, pa.hdr, pa.sends, send_stride);
  CUDA_TRY(h, cudaGetLastError());
  h->perf.kernel_launches++;
  plan.args.results = (demi_fuzz_result*)out_dev;
  bind_programs(h, plan.args, pa, p->max_messages);
  if ((rc = launch_plan(h, plan, n, s)) != DEMI_OK) return rc;
  h->perf.prefixes += n;
  return DEMI_OK;
}

// What the campaign entry points need before the first chunk: campaign_chunk reads the Fuzzer, and the call-wide
// n_prefixes limit of demi_fuzz_batch_dev (plan_launch only sees one chunk here).
static int32_t check_campaign(demi_handle* h, const demi_fuzz_params* p) {
  if (!p) return fail(h, DEMI_ERR_INVALID, "null params");
  if (!h->has_fuzzer) return fail(h, DEMI_ERR_STATE, "demi_set_fuzzer has not been called");
  if (p->n_prefixes > 0xFFFFFFFFull) return fail(h, DEMI_ERR_INVALID, "n_prefixes > 2^32-1 per call");
  return DEMI_OK;
}

// RunnerUtils.fuzz's loop (RunnerUtils.scala:75-91): `fuzzer.generateFuzzTest()` then `RandomScheduler.explore`, once
// per execution, with results left in HBM.  No sync; demi_fuzz_summary_dev reads the counts.
extern "C" int32_t demi_fuzz_campaign_dev(demi_handle* h, const demi_fuzz_params* p, int64_t program_seed_base, void* out_dev,
                                          void* stream) {
  if (!h) return DEMI_ERR_INVALID;
  if (!out_dev) return fail(h, DEMI_ERR_INVALID, "demi_fuzz_campaign_dev: null output");
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  int32_t rc = check_campaign(h, p);
  if (rc != DEMI_OK) return rc;
  uint32_t stride, send_stride;
  const uint64_t chunk = campaign_chunk(h, &stride, &send_stride), n = p->n_prefixes;
  if (n == 0) return launch_campaign(h, p, program_seed_base, out_dev, (cudaStream_t)stream, true);
  for (uint64_t off = 0; off < n; off += chunk) {
    demi_fuzz_params q = *p;
    q.seed_base = seed_at(p->seed_base, off);
    q.n_prefixes = std::min(chunk, n - off);
    rc = launch_campaign(h, &q, seed_at(program_seed_base, off), (demi_fuzz_result*)out_dev + off, (cudaStream_t)stream, off == 0);
    if (rc != DEMI_OK) return rc;
  }
  return DEMI_OK;
}

// Same, records to the host, pipelined as demi_fuzz_batch.
extern "C" int32_t demi_fuzz_campaign(demi_handle* h, const demi_fuzz_params* p, int64_t program_seed_base, demi_fuzz_result* out_host) {
  if (!h) return DEMI_ERR_INVALID;
  if (!out_host) return fail(h, DEMI_ERR_INVALID, "demi_fuzz_campaign: null output");
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  int32_t rc = check_campaign(h, p);
  if (rc != DEMI_OK) return rc;
  uint32_t stride, send_stride;
  const uint64_t chunk = campaign_chunk(h, &stride, &send_stride);
  return run_pipelined(h, "demi_fuzz_campaign", p->n_prefixes, chunk, out_host, [&](uint64_t off, uint64_t m, demi_fuzz_result* dst, bool first) {
    demi_fuzz_params q = *p;
    q.seed_base = seed_at(p->seed_base, off);
    q.n_prefixes = m;
    return launch_campaign(h, &q, seed_at(program_seed_base, off), dst, h->stream, first);
  });
}

// ---------------------------------------------------------------------------------------------------------
// Random-oracle tests: RandomScheduler.test(subsequence) (RandomScheduler.scala:597-612) for T masks over the handle's
// program, N executions each, T x N executions per launch through the PROG engines.

// One warp per test: the subsequence of the base program that the test's mask keeps, compacted (ballot + prefix sum)
// into the arena layout of the campaigns: events[t * stride ..), hdr[t] = {length, Sends}, the lane-form Sends at
// sends[t * send_stride ..).
__device__ __forceinline__ void subseq_warp(const demi_ext_event* base, uint32_t n_ext, const uint64_t* mask, uint64_t t, uint32_t lane,
                                            demi_ext_event* events, uint32_t stride, uint2* hdr, uint4* sends, uint32_t send_stride) {
  const uint32_t below = (1u << lane) - 1u;
  uint32_t len = 0, ns = 0;
  for (uint32_t b = 0; b < n_ext; b += 32) {
    const uint32_t i = b + lane;
    const bool in = i < n_ext && ((mask[i >> 6] >> (i & 63)) & 1ull);
    demi_ext_event e{};
    if (in) e = base[i];
    const bool send = in && e.kind == DEMI_EXT_SEND;
    const uint32_t m = __ballot_sync(FULL_MASK, in), ms = __ballot_sync(FULL_MASK, send);
    if (in) events[t * stride + len + __popc(m & below)] = e;
    if (send) sends[t * send_stride + ns + __popc(ms & below)] = lane_send(e);
    len += __popc(m); ns += __popc(ms);
  }
  if (lane == 0) hdr[t] = make_uint2(len, ns);
}
__global__ void __launch_bounds__(128)
random_subseq_kernel(const demi_ext_event* base, uint32_t n_ext, const uint64_t* masks, uint32_t mask_words, uint32_t n_tests,
                     demi_ext_event* events, uint32_t stride, uint2* hdr, uint4* sends, uint32_t send_stride) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (t >= n_tests) return;
  subseq_warp(base, n_ext, masks + t * mask_words, t, lane, events, stride, hdr, sends, send_stride);
}
// The same over many base programs: test t keeps bits of program trace_of_test[t], which is
// progs[prog_tab[trace].x ..), prog_tab[trace].y events long.
__global__ void __launch_bounds__(128)
random_subseq_many_kernel(const demi_ext_event* progs, const uint2* prog_tab, const uint32_t* trace_of_test, const uint64_t* masks,
                          uint32_t mask_words, uint32_t n_tests, demi_ext_event* events, uint32_t stride, uint2* hdr, uint4* sends,
                          uint32_t send_stride) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (t >= n_tests) return;
  const uint2 pt = prog_tab[trace_of_test[t]];
  subseq_warp(progs + pt.x, pt.y, masks + t * mask_words, t, lane, events, stride, hdr, sends, send_stride);
}

// One warp per test over its N execution records: the test record, and the executions that ran (not skipped), summed
// into *executed and, with PER_TEST, also written per test to ran[t].
template <bool PER_TEST>
__global__ void __launch_bounds__(128)
random_test_reduce_kernel(const demi_fuzz_result* res, uint32_t n_tests, uint32_t n_execs, demi_random_test_result* out,
                          unsigned long long* executed, uint32_t* ran_of_test) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (t >= n_tests) return;
  int32_t first = -1;
  uint32_t status = 0, violation = 0, ran = 0;
  for (uint32_t b = 0; b < n_execs; b += 32) {
    const uint32_t j = b + lane;
    uint32_t st = PS_SKIPPED, v = 0;
    if (j < n_execs) { const demi_fuzz_result& r = res[t * n_execs + j]; st = r.status; v = r.violation; }
    const uint32_t hit = __ballot_sync(FULL_MASK, st == 0 && v != 0);
    const uint32_t bad = __ballot_sync(FULL_MASK, st != 0 && st != PS_SKIPPED);
    ran += __popc(__ballot_sync(FULL_MASK, st != PS_SKIPPED));
    if (first < 0) {
      const uint32_t upto = hit ? (((hit & (0u - hit)) - 1u) | (hit & (0u - hit))) : FULL_MASK;   // lanes up to the first hit
      const uint32_t first_bad = bad & upto;
      const uint32_t sb = __shfl_sync(FULL_MASK, st, first_bad ? __ffs(first_bad) - 1 : 0);
      if (!status && first_bad) status = sb;
      const uint32_t vh = __shfl_sync(FULL_MASK, v, hit ? __ffs(hit) - 1 : 0);
      if (hit) { first = (int32_t)(b + __ffs(hit) - 1); violation = vh; }
    }
  }
  if (lane == 0) {
    out[t] = demi_random_test_result{first, first >= 0 ? (uint32_t)first + 1 : n_execs, violation, (uint16_t)status, 0};
    atomicAdd(executed, (unsigned long long)ran);
    if constexpr (PER_TEST) ran_of_test[t] = ran;
  }
}

// tests per launch: at most RANDOM_EXECS_PER_LAUNCH executions (their records are 32 B each, 128 MB) and an arena of
// at most 512 MB
static constexpr uint64_t RANDOM_EXECS_PER_LAUNCH = 1u << 22;

static int32_t check_random(demi_handle* h, const char* who, uint32_t mask_words, const demi_fuzz_params* p) {
  if (!p) return fail(h, DEMI_ERR_INVALID, "%s: null params", who);
  if (h->ext_host.empty()) return fail(h, DEMI_ERR_STATE, "demi_set_externals has not been called");
  if (p->n_prefixes == 0 || p->n_prefixes > RANDOM_EXECS_PER_LAUNCH)
    return fail(h, DEMI_ERR_INVALID, "%s: N = n_prefixes must be in 1..%llu", who, (unsigned long long)RANDOM_EXECS_PER_LAUNCH);
  if ((uint64_t)mask_words * 64 < h->ext_host.size()) return fail(h, DEMI_ERR_INVALID, "%s: mask_words too small", who);
  return DEMI_OK;
}

// the tests of one call, in launches of `per` tests; *executed = executions that ran
static int32_t random_tests(demi_handle* h, const uint64_t* masks, uint32_t n_tests, uint32_t mask_words, const demi_fuzz_params* p,
                            demi_random_test_result* out, uint64_t* executed) {
  const uint32_t N = (uint32_t)p->n_prefixes, n_ext = (uint32_t)h->ext_host.size();
  const uint32_t stride = std::max(n_ext, 1u), send_stride = std::max(h->ext_info.sends, 1u);
  const uint64_t per_test = (uint64_t)stride * sizeof(demi_ext_event) + sizeof(uint2) + (uint64_t)send_stride * sizeof(uint4) +
                            (uint64_t)mask_words * 8 + sizeof(demi_random_test_result) + 4;
  const uint64_t per = std::max<uint64_t>(1, std::min<uint64_t>(RANDOM_EXECS_PER_LAUNCH / N, ((uint64_t)512 << 20) / per_test));
  const uint64_t cap_tests = std::min<uint64_t>(per, n_tests);
  // arena: the programs | masks | first_hit | test records | counter
  const size_t b_mask = ((size_t)cap_tests * mask_words * 8 + 15) & ~(size_t)15, b_fh = ((size_t)cap_tests * 4 + 15) & ~(size_t)15,
               b_out = ((size_t)cap_tests * sizeof(demi_random_test_result) + 15) & ~(size_t)15;
  ProgramArena pa;
  unsigned char* rest;
  int32_t rc = carve_programs(h, cap_tests, stride, send_stride, b_mask + b_fh + b_out + 16, &pa, &rest);
  if (rc != DEMI_OK) return rc;
  if ((rc = h->results_dev.grow(h, std::max<size_t>((size_t)cap_tests * N * sizeof(demi_fuzz_result), 32))) != DEMI_OK) return rc;
  demi_fuzz_result* results = h->results_dev.get<demi_fuzz_result>();
  const demi_ext_event* ext = h->ext_dev.get<demi_ext_event>();
  uint64_t* mdev = (uint64_t*)rest;
  uint32_t* first_hit = (uint32_t*)(rest + b_mask);
  demi_random_test_result* odev = (demi_random_test_result*)(rest + b_mask + b_fh);
  unsigned long long* cnt = (unsigned long long*)(rest + b_mask + b_fh + b_out);
  cudaStream_t s = h->stream;
  CUDA_TRY(h, cudaMemsetAsync(cnt, 0, sizeof(unsigned long long), s));
  CUDA_TRY(h, cudaMemsetAsync(h->counters_dev.get(), 0, 4 * sizeof(unsigned long long), s));
  CUDA_TRY(h, cudaEventRecord(h->ev0, s));
  h->perf.kernel_launches = 0;
  for (uint64_t off = 0; off < n_tests; off += per) {
    const uint32_t m = (uint32_t)std::min<uint64_t>(per, n_tests - off);
    demi_fuzz_params q = *p;
    q.n_prefixes = (uint64_t)m * N;
    LaunchPlan plan;
    if ((rc = plan_launch(h, &q, LM_TESTS, h->ext_info, ext, n_ext, &plan)) != DEMI_OK) return rc;
    CUDA_TRY(h, cudaMemcpyAsync(mdev, masks + off * mask_words, (size_t)m * mask_words * 8, cudaMemcpyHostToDevice, s));
    CUDA_TRY(h, cudaMemsetAsync(first_hit, 0xFF, (size_t)m * 4, s));
    random_subseq_kernel<<<(unsigned)(((uint64_t)m * 32 + 127) / 128), 128, 0, s>>>(ext, n_ext, mdev, mask_words, m, pa.ev, stride,
                                                                                     pa.hdr, pa.sends, send_stride);
    CUDA_TRY(h, cudaGetLastError());
    h->perf.kernel_launches++;
    KernelArgs& a = plan.args;
    a.results = results;
    bind_programs(h, a, pa, p->max_messages);
    a.prog_execs = N;
    a.prog_first_hit = first_hit;
    if ((rc = launch_plan(h, plan, q.n_prefixes, s)) != DEMI_OK) return rc;
    random_test_reduce_kernel<false><<<(unsigned)(((uint64_t)m * 32 + 127) / 128), 128, 0, s>>>(results, m, N, odev, cnt, nullptr);
    CUDA_TRY(h, cudaGetLastError());
    h->perf.kernel_launches++;
    CUDA_TRY(h, cudaMemcpyAsync(out + off, odev, (size_t)m * sizeof(demi_random_test_result), cudaMemcpyDeviceToHost, s));
  }
  unsigned long long c[4] = {0, 0, 0, 0}, ran = 0;
  CUDA_TRY(h, cudaEventRecord(h->ev1, s));
  CUDA_TRY(h, cudaMemcpyAsync(c, h->counters_dev.get(), sizeof(c), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaMemcpyAsync(&ran, cnt, sizeof(ran), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaStreamSynchronize(s));
  float ms = 0;
  CUDA_TRY(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  h->perf.kernel_ms = ms;
  h->perf.prefixes = ran;
  read_counters(h, c);
  h->perf.h2d_bytes = (uint64_t)n_tests * mask_words * 8;
  h->perf.d2h_bytes = (uint64_t)n_tests * sizeof(demi_random_test_result);
  *executed = ran;
  return DEMI_OK;
}

extern "C" int32_t demi_random_test_batch(demi_handle* h, const uint64_t* masks, uint32_t n_tests, uint32_t mask_words,
                                          const demi_fuzz_params* p, demi_random_test_result* out) {
  if (!h) return DEMI_ERR_INVALID;
  int32_t rc = check_random(h, "demi_random_test_batch", mask_words, p);
  if (rc != DEMI_OK) return rc;
  if (n_tests && (!masks || !out)) return fail(h, DEMI_ERR_INVALID, "demi_random_test_batch: null masks or output");
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  uint64_t executed = 0;
  if (!n_tests) { h->perf.prefixes = 0; return DEMI_OK; }
  return random_tests(h, masks, n_tests, mask_words, p, out, &executed);
}

// demi_fuzz_trace over the subsequence of the handle's program that `mask` keeps
extern "C" int32_t demi_random_test_trace(demi_handle* h, const uint64_t* mask, uint32_t mask_words, const demi_fuzz_params* p,
                                          int64_t seed, demi_event* events, uint32_t cap_events, uint32_t* n_events,
                                          demi_fuzz_result* result) {
  if (!h) return DEMI_ERR_INVALID;
  if (!p || !mask) return fail(h, DEMI_ERR_INVALID, "demi_random_test_trace: null argument");
  if (h->ext_host.empty()) return fail(h, DEMI_ERR_STATE, "demi_set_externals has not been called");
  if ((uint64_t)mask_words * 64 < h->ext_host.size()) return fail(h, DEMI_ERR_INVALID, "demi_random_test_trace: mask_words too small");
  std::vector<demi_ext_event> sub;
  ProgramInfo info;
  std::vector<uint4> sv;
  for (size_t i = 0; i < h->ext_host.size(); i++)
    if ((mask[i >> 6] >> (i & 63)) & 1ull) {
      sub.push_back(h->ext_host[i]);
      describe_event(&info, &sv, sub.back());
    }
  if (sub.empty()) return fail(h, DEMI_ERR_INVALID, "demi_random_test_trace: the mask keeps no event");
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  DevBuf dev;
  const int32_t rc = dev.upload(h, sub.data(), sub.size() * sizeof(demi_ext_event));
  if (rc != DEMI_OK) return rc;
  return fuzz_trace(h, p, seed, events, cap_events, n_events, nullptr, 0, nullptr, result, dev.get<demi_ext_event>(), (uint32_t)sub.size(), info);
}

#include "random_ddmin_driver.hpp"
#include "many_rendezvous.hpp"
namespace {

// the handle's program: a speculative batch of masks = one demi_random_test_batch
struct HandleRandomDriver : RandomDDMinDriver {
  demi_fuzz_params p{};
  int32_t run_tests(const uint64_t* masks, size_t n, demi_random_test_result* res, uint64_t* executed) override {
    return random_tests(h, masks, (uint32_t)n, mw, &p, res, executed);
  }
};

}  // namespace

extern "C" int32_t demi_random_ddmin(demi_handle* h, const demi_fuzz_params* p, int32_t check_unmodified, uint64_t* mcs_mask,
                                     uint32_t mask_words, uint32_t* iteration_sizes, uint64_t* iteration_keys, uint32_t cap,
                                     demi_random_ddmin_out* out) {
  if (!h) return DEMI_ERR_INVALID;
  if (!mcs_mask || !out) return fail(h, DEMI_ERR_INVALID, "demi_random_ddmin: null output");
  int32_t rc = check_random(h, "demi_random_ddmin", mask_words, p);
  if (rc != DEMI_OK) return rc;
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  HandleRandomDriver d;
  d.h = h; d.p = *p; d.looking_for = p->looking_for; d.mw = mask_words; d.n_ext = (uint32_t)h->ext_host.size();
  d.ext = h->ext_host.data();
  d.set_width(p->n_prefixes);
  return d.minimize(check_unmodified != 0, mcs_mask, iteration_sizes, iteration_keys, cap, out);
}

// ---------------------------------------------------------------------------------------------------------
// Many programs in one call: random-oracle tests, randomDDMin and recorded executions over many traces, each trace
// with its own program, seed base, max_messages and looking_for.  The work of every trace shares launches of the
// PROG + PARAMS instantiations, packed by launch_many.
namespace {

// What a launch reads of the program of a trace (or of the subsequences its items keep): at most `len` events, the
// pending capacity under the trace's max_messages, and what describe_event finds in it
struct ManyProgram { uint32_t len = 0, pcap = 0; ProgramInfo info; };

// A call's traces: their programs (the caller's externals, uploaded once), what each program's launches need, and what
// a trace fails with before any launch.
struct ProgramSet {
  const demi_handle* h = nullptr;              // the call's handle: the configuration every trace runs under
  uint32_t mask_words = 0;
  const int64_t* seed_base = nullptr; const int32_t* max_messages = nullptr; const uint32_t* looking_for = nullptr;
  demi_fuzz_params p{};                        // N, interval and flags
  std::vector<ManyProgram> prog;               // each trace's whole program
  std::vector<int32_t> pre; std::vector<std::string> pre_msg;
  DevBuf dev;                                  // the externals, then uint2 {offset, length} per trace
  const demi_ext_event* progs = nullptr; const uint2* tab = nullptr;
};

// The checks demi_set_externals and demi_random_test_batch make of trace t's program before a launch; the call-wide
// ones (N, mask_words) are the caller's.  The programs and their table are uploaded once.
int32_t program_set(demi_handle* h, uint32_t n, const demi_ext_event* externals, const uint32_t* ext_offsets, const uint32_t* n_externals,
                    const int64_t* seed_base, const int32_t* max_messages, const uint32_t* looking_for, const demi_fuzz_params* p,
                    ProgramSet& ps) {
  ps.h = h; ps.seed_base = seed_base; ps.max_messages = max_messages; ps.looking_for = looking_for;
  ps.p = *p;
  ps.prog.assign(n, ManyProgram{}); ps.pre.assign(n, DEMI_OK); ps.pre_msg.assign(n, std::string());
  uint64_t span = 0;
  std::vector<uint2> tab(n);
  demi_handle eh;
  for (uint32_t t = 0; t < n; t++) {
    const demi_ext_event* ev = externals + ext_offsets[t];
    ManyProgram& pg = ps.prog[t];
    std::vector<uint4> sv;
    int32_t rc = DEMI_OK;
    eh.err.clear();
    eh.cfg = h->cfg; eh.ir_n_actors = h->ir_n_actors;            // demi_model_actors reads these
    for (uint32_t i = 0; i < n_externals[t] && rc == DEMI_OK; i++) {
      rc = demi_check_external(&eh, "demi_set_externals", "", ev, i, true, true);
      if (rc == DEMI_OK) describe_event(&pg.info, &sv, ev[i]);
    }
    if (rc == DEMI_OK && !n_externals[t]) rc = fail(&eh, DEMI_ERR_STATE, "demi_set_externals has not been called");
    if (rc != DEMI_OK) { ps.pre[t] = rc; ps.pre_msg[t] = eh.err; continue; }
    pg.len = n_externals[t];
    pg.pcap = demi_pending_cap(demi_model_key(h), max_messages[t], pg.info.sends);   // demi_random_test_batch's
    tab[t] = make_uint2(ext_offsets[t], n_externals[t]);
    span = std::max<uint64_t>(span, (uint64_t)ext_offsets[t] + n_externals[t]);
  }
  const size_t b_ev = ((size_t)span * sizeof(demi_ext_event) + 15) & ~(size_t)15;
  int32_t rc = ps.dev.grow(h, b_ev + (size_t)n * sizeof(uint2));
  if (rc != DEMI_OK) return rc;
  if (span) CUDA_TRY(h, cudaMemcpy(ps.dev.get(), externals, (size_t)span * sizeof(demi_ext_event), cudaMemcpyHostToDevice));
  CUDA_TRY(h, cudaMemcpy(ps.dev.get<char>() + b_ev, tab.data(), (size_t)n * sizeof(uint2), cudaMemcpyHostToDevice));
  ps.progs = ps.dev.get<demi_ext_event>(); ps.tab = (const uint2*)(ps.dev.get<char>() + b_ev);
  return DEMI_OK;
}

// A unit of work of a many-program launch: a test or an execution over the subsequence of trace `trace`'s program that
// `mask` keeps.  Only items of the same key share a launch.
struct ManyItem { uint32_t trace, key; const uint64_t* mask; };

// One launch of launch_many, for its caller to finish: the plan with the programs bound, the items' parameter table on
// the device, the caller's bytes, and the launch's m items (indices into the call's list).
struct ManyLaunch { LaunchPlan& plan; const uint4* params; unsigned char* extra; const uint32_t* item; uint32_t m; };

// Launches `items` (masks of mw words) over the programs of `ps` in launches of `mode`, `execs` executions per item;
// progs[t] describes what the items of trace t keep.  The items go out grouped by key, in increasing key order, each
// group cut greedily into launches of at most `cap` items and an arena of at most 512 MB, whose program stride is the
// launch's longest program and which counts `extra` bytes of the caller's per item.  Per launch: the arena, laid out
// programs | masks | parameters {seed lo, seed hi, max_messages, looking_for} | trace ids | the caller's 16 + m * extra
// bytes; a plan with the launch's merged ProgramInfo and largest pending capacity (each item binds its own
// max_messages); random_subseq_many_kernel; then run(ManyLaunch&), which binds what its mode needs and launches.
template <class Run>
int32_t launch_many(demi_handle* h, const ProgramSet& ps, LaunchMode mode, uint32_t execs, const ManyProgram* progs,
                    const std::vector<ManyItem>& items, uint32_t mw, uint64_t cap, size_t extra, Run run) {
  std::vector<uint32_t> order(items.size());
  for (uint32_t i = 0; i < order.size(); i++) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return items[a].key < items[b].key; });
  cudaStream_t s = h->stream;
  std::vector<uint64_t> hm;
  std::vector<uint4> hp;
  std::vector<uint32_t> ht;
  for (size_t lo = 0; lo < order.size();) {
    uint32_t stride = 1, send_stride = 1, pcap = 0;
    ProgramInfo li;
    size_t hi = lo;
    for (; hi < order.size() && hi - lo < cap && items[order[hi]].key == items[order[lo]].key; hi++) {
      const ManyProgram& pg = progs[items[order[hi]].trace];
      const uint32_t st = std::max(stride, pg.len), ss = std::max(send_stride, pg.info.sends);
      const uint64_t per = (uint64_t)st * sizeof(demi_ext_event) + sizeof(uint2) + (uint64_t)ss * sizeof(uint4) + (uint64_t)mw * 8 +
                           sizeof(uint4) + 4 + extra;
      if (hi > lo && (hi - lo + 1) * per > ((uint64_t)512 << 20)) break;
      stride = st; send_stride = ss;
      pcap = std::max(pcap, pg.pcap);
      li.sends = std::max(li.sends, pg.info.sends);
      li.hard_kill |= pg.info.hard_kill; li.partitions |= pg.info.partitions;
      li.sends_distinct &= pg.info.sends_distinct;
    }
    const uint32_t m = (uint32_t)(hi - lo);
    auto al = [](size_t b) { return (b + 15) & ~(size_t)15; };
    const size_t b_mask = al((size_t)m * mw * 8), b_par = al((size_t)m * sizeof(uint4)), b_tr = al((size_t)m * 4);
    ProgramArena pa;
    unsigned char* rest;
    int32_t rc = carve_programs(h, m, stride, send_stride, b_mask + b_par + b_tr + 16 + (size_t)m * extra, &pa, &rest);
    if (rc != DEMI_OK) return rc;
    uint64_t* mdev = (uint64_t*)rest;
    uint4* pdev = (uint4*)(rest + b_mask);
    uint32_t* tdev = (uint32_t*)(rest + b_mask + b_par);
    hm.resize((size_t)m * mw); hp.resize(m); ht.resize(m);
    for (uint32_t k = 0; k < m; k++) {
      const ManyItem& it = items[order[lo + k]];
      std::copy(it.mask, it.mask + mw, hm.begin() + (size_t)k * mw);
      const uint64_t sb = (uint64_t)ps.seed_base[it.trace];
      hp[k] = make_uint4((uint32_t)sb, (uint32_t)(sb >> 32), (uint32_t)ps.max_messages[it.trace], ps.looking_for[it.trace]);
      ht[k] = it.trace;
    }
    CUDA_TRY(h, cudaMemcpyAsync(mdev, hm.data(), hm.size() * 8, cudaMemcpyHostToDevice, s));
    CUDA_TRY(h, cudaMemcpyAsync(pdev, hp.data(), hp.size() * sizeof(uint4), cudaMemcpyHostToDevice, s));
    CUDA_TRY(h, cudaMemcpyAsync(tdev, ht.data(), ht.size() * 4, cudaMemcpyHostToDevice, s));
    demi_fuzz_params q = ps.p;
    q.n_prefixes = (uint64_t)m * execs;
    q.max_messages = -1;                   // each item binds its own (prog_params_bind); pcap covers them all
    q.looking_for = 0; q.seed_base = 0;
    LaunchPlan plan;
    if ((rc = plan_launch(h, &q, mode, li, nullptr, 0, &plan, pcap)) != DEMI_OK) return rc;
    bind_programs(h, plan.args, pa, -1);
    random_subseq_many_kernel<<<(unsigned)(((uint64_t)m * 32 + 127) / 128), 128, 0, s>>>(ps.progs, ps.tab, tdev, mdev, mw, m, pa.ev,
                                                                                        stride, pa.hdr, pa.sends, send_stride);
    CUDA_TRY(h, cudaGetLastError());
    h->perf.kernel_launches++;
    ManyLaunch L{plan, pdev, rest + b_mask + b_par + b_tr, order.data() + lo, m};
    if ((rc = run(L)) != DEMI_OK) return rc;
    lo = hi;
  }
  return DEMI_OK;
}

// A test's record and the executions of it that ran
struct RandomRec { demi_random_test_result rec; uint32_t ran; };

// n tests: test i is masks[i * mask_words ..) over the program of trace tr[i], which check_variant accepts.  The tests
// go out in at most two groups, the programs the lane engine takes and the others (so that one HardKill program does
// not send every test to the warp engine), in launches of at most RANDOM_EXECS_PER_LAUNCH executions.
int32_t random_tests_many(demi_handle* h, const ProgramSet& ps, const uint32_t* tr, const uint64_t* masks, size_t n, RandomRec* out) {
  const uint32_t N = (uint32_t)ps.p.n_prefixes, mw = ps.mask_words;
  std::vector<ManyItem> items(n);
  for (size_t i = 0; i < n; i++) items[i] = ManyItem{tr[i], pick_lane_variant(h, ps.prog[tr[i]].info) ? 0u : 1u, masks + i * mw};
  cudaStream_t s = h->stream;
  std::vector<uint32_t> hran;
  std::vector<demi_random_test_result> hrec;
  return launch_many(h, ps, LM_TEST_PARAMS, N, ps.prog.data(), items, mw, RANDOM_EXECS_PER_LAUNCH / N,
                     sizeof(demi_random_test_result) + 4 + 4, [&](ManyLaunch& L) -> int32_t {
    // the caller's bytes: counter | test records | first_hit | executions that ran
    const uint32_t m = L.m;
    unsigned long long* cnt = (unsigned long long*)L.extra;
    demi_random_test_result* odev = (demi_random_test_result*)(L.extra + 16);
    uint32_t* first_hit = (uint32_t*)(odev + m);
    uint32_t* rdev = first_hit + m;
    int32_t rc = h->results_dev.grow(h, std::max<size_t>((size_t)m * N * sizeof(demi_fuzz_result), 32));
    if (rc != DEMI_OK) return rc;
    CUDA_TRY(h, cudaMemsetAsync(first_hit, 0xFF, (size_t)m * 4, s));
    CUDA_TRY(h, cudaMemsetAsync(cnt, 0, sizeof(unsigned long long), s));
    KernelArgs& a = L.plan.args;
    a.results = h->results_dev.get<demi_fuzz_result>();
    a.prog_execs = N;
    a.prog_first_hit = first_hit;
    a.prog_params = L.params;
    if ((rc = launch_plan(h, L.plan, (uint64_t)m * N, s)) != DEMI_OK) return rc;
    random_test_reduce_kernel<true><<<(unsigned)(((uint64_t)m * 32 + 127) / 128), 128, 0, s>>>(a.results, m, N, odev, cnt, rdev);
    CUDA_TRY(h, cudaGetLastError());
    h->perf.kernel_launches++;
    hrec.resize(m); hran.resize(m);
    CUDA_TRY(h, cudaMemcpyAsync(hrec.data(), odev, (size_t)m * sizeof(demi_random_test_result), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(h, cudaMemcpyAsync(hran.data(), rdev, (size_t)m * 4, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(h, cudaStreamSynchronize(s));
    for (uint32_t k = 0; k < m; k++) {
      out[L.item[k]] = RandomRec{hrec[k], hran[k]};
      h->perf.prefixes += hran[k];
    }
    return DEMI_OK;
  });
}

// The call-wide checks of both entry points: what demi_random_test_batch / demi_random_ddmin refuse whatever the program
int32_t check_random_many(demi_handle* h, const char* who, uint32_t n, const demi_ext_event* externals, const uint32_t* ext_offsets,
                          const uint32_t* n_externals, const int64_t* seed_base, const int32_t* max_messages,
                          const uint32_t* looking_for, const demi_fuzz_params* p, uint32_t mask_words) {
  if (!externals || !ext_offsets || !n_externals || !seed_base || !max_messages || !looking_for || !p)
    return fail(h, DEMI_ERR_INVALID, "%s: null argument", who);
  { int32_t mrc = demi_need_model(h); if (mrc != DEMI_OK) return mrc; }
  if (p->n_prefixes == 0 || p->n_prefixes > RANDOM_EXECS_PER_LAUNCH)
    return fail(h, DEMI_ERR_INVALID, "%s: N = n_prefixes must be in 1..%llu", who, (unsigned long long)RANDOM_EXECS_PER_LAUNCH);
  for (uint32_t t = 0; t < n; t++)
    if ((uint64_t)mask_words * 64 < n_externals[t])
      return fail(h, DEMI_ERR_INVALID, "%s: mask_words %u too small for the %u externals of trace %u", who, mask_words, n_externals[t], t);
  return DEMI_OK;
}

typedef ManyRequest<RandomRec> RandomRequest;

// randomDDMin on trace `trace` of a demi_random_ddmin_many call: its batches join the rendezvous
struct ManyRandomDriver : RandomDDMinDriver {
  Rendezvous<RandomRec>* R; uint32_t trace; const ProgramSet* ps;
  int32_t run_tests(const uint64_t* masks, size_t n, demi_random_test_result* res, uint64_t* executed) override {
    const ManyProgram& pg = ps->prog[trace];             // what plan_launch refuses of this trace's launch alone
    int32_t rc = check_variant(ps->h, h, LM_TEST_PARAMS, pg.info, pg.pcap, demi_tosend_cap(pg.info.sends), nullptr);
    if (rc != DEMI_OK) return rc;
    RandomRequest q;
    q.trace = trace; q.masks = masks; q.n = n;
    R->submit(q);
    if (q.rc != DEMI_OK) return q.rc;
    *executed = 0;
    for (size_t k = 0; k < n; k++) { res[k] = q.res[k].rec; *executed += q.res[k].ran; }
    return DEMI_OK;
  }
};

}  // namespace

extern "C" int32_t demi_random_test_batch_many(demi_handle* h, uint32_t n_traces, const demi_ext_event* externals,
                                               const uint32_t* ext_offsets, const uint32_t* n_externals, const int64_t* seed_base,
                                               const int32_t* max_messages, const uint32_t* looking_for,
                                               const uint32_t* trace_of_test, const uint64_t* masks, uint32_t n_tests,
                                               uint32_t mask_words, const demi_fuzz_params* p, demi_random_test_result* out) {
  if (!h) return DEMI_ERR_INVALID;
  static const char* who = "demi_random_test_batch_many";
  int32_t rc = check_random_many(h, who, n_traces, externals, ext_offsets, n_externals, seed_base, max_messages, looking_for, p,
                                 mask_words);
  if (rc != DEMI_OK) return rc;
  if (n_tests && (!trace_of_test || !masks || !out)) return fail(h, DEMI_ERR_INVALID, "%s: null tests or output", who);
  for (uint32_t i = 0; i < n_tests; i++)
    if (trace_of_test[i] >= n_traces) return fail(h, DEMI_ERR_INVALID, "%s: test %u names trace %u of %u", who, i, trace_of_test[i], n_traces);
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  h->perf.kernel_launches = 0; h->perf.prefixes = 0;
  if (!n_tests) return DEMI_OK;
  ProgramSet ps;
  ps.mask_words = mask_words;
  if ((rc = program_set(h, n_traces, externals, ext_offsets, n_externals, seed_base, max_messages, looking_for, p, ps)) != DEMI_OK) return rc;
  // a test fails the call with what its program alone would give
  for (uint32_t i = 0; i < n_tests; i++) {
    const uint32_t t = trace_of_test[i];
    const ManyProgram& pg = ps.prog[t];
    if (ps.pre[t] != DEMI_OK) { h->err = trace_msg(who, t, ps.pre_msg[t]); return ps.pre[t]; }
    if ((rc = check_variant(h, h, LM_TEST_PARAMS, pg.info, pg.pcap, demi_tosend_cap(pg.info.sends), nullptr)) != DEMI_OK) {
      h->err = trace_msg(who, t, h->err);
      return rc;
    }
  }
  std::vector<RandomRec> res(n_tests);
  if ((rc = random_tests_many(h, ps, trace_of_test, masks, n_tests, res.data())) != DEMI_OK) return rc;
  for (uint32_t i = 0; i < n_tests; i++) out[i] = res[i].rec;
  return DEMI_OK;
}

extern "C" int32_t demi_random_ddmin_many(demi_handle* h, uint32_t n_traces, const demi_ext_event* externals,
                                          const uint32_t* ext_offsets, const uint32_t* n_externals, const int64_t* seed_base,
                                          const int32_t* max_messages, const uint32_t* looking_for, const demi_fuzz_params* p,
                                          int32_t check_unmodified, uint64_t* mcs_masks, uint32_t mask_words, uint32_t* iteration_sizes,
                                          uint64_t* iteration_keys, uint32_t cap_iterations, demi_random_ddmin_out* out,
                                          int32_t* status) {
  if (!h) return DEMI_ERR_INVALID;
  static const char* who = "demi_random_ddmin_many";
  if (!n_traces) return DEMI_OK;
  int32_t rc = check_random_many(h, who, n_traces, externals, ext_offsets, n_externals, seed_base, max_messages, looking_for, p,
                                 mask_words);
  if (rc != DEMI_OK) return rc;
  if (!mcs_masks || !out || !status) return fail(h, DEMI_ERR_INVALID, "%s: null output", who);
  const uint32_t n = n_traces;
  uint32_t window;
  if ((rc = many_window(h, n, window)) != DEMI_OK) return rc;
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  memset(out, 0, (size_t)n * sizeof(demi_random_ddmin_out));
  h->perf.kernel_launches = 0; h->perf.prefixes = 0;
  ProgramSet ps;
  ps.mask_words = mask_words;
  if ((rc = program_set(h, n, externals, ext_offsets, n_externals, seed_base, max_messages, looking_for, p, ps)) != DEMI_OK) return rc;
  demi_perf perf{};
  // the union of a round's requests, in request order
  auto serve = [&](std::vector<RandomRequest*>& batch) -> int32_t {
    std::vector<uint32_t> tos;
    std::vector<uint64_t> flat;
    flatten_requests(batch, mask_words, tos, flat);
    std::vector<RandomRec> res(tos.size());
    const int32_t src = random_tests_many(h, ps, tos.data(), flat.data(), tos.size(), res.data());
    perf.kernel_launches += h->perf.kernel_launches; perf.prefixes += h->perf.prefixes;
    h->perf.kernel_launches = 0; h->perf.prefixes = 0;
    if (src != DEMI_OK) return src;
    scatter_results(batch, res);
    return DEMI_OK;
  };
  auto drive = [&](uint32_t t, Rendezvous<RandomRec>& R, demi_handle* eh) -> int32_t {
    if (ps.pre[t] != DEMI_OK) { eh->err = ps.pre_msg[t]; return ps.pre[t]; }
    ManyRandomDriver d;
    d.R = &R; d.trace = t; d.ps = &ps;
    d.h = eh; d.looking_for = looking_for[t]; d.mw = mask_words; d.n_ext = n_externals[t];
    d.ext = externals + ext_offsets[t];
    d.set_width(p->n_prefixes);
    return d.minimize(check_unmodified != 0, mcs_masks + (size_t)t * mask_words,
                      iteration_sizes ? iteration_sizes + (size_t)t * cap_iterations : nullptr,
                      iteration_keys ? iteration_keys + (size_t)t * cap_iterations : nullptr, cap_iterations, out + t);
  };
  rc = run_many<RandomRec>(h, who, n, window, drive, serve, status);
  h->perf.kernel_launches = perf.kernel_launches; h->perf.prefixes = perf.prefixes;
  if (rc != DEMI_OK) return rc;
  for (uint32_t t = 0; t < n; t++)
    if (status[t] != DEMI_OK) { h->err = trace_msg(who, t, h->err); break; }
  return DEMI_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Recording many programs' executions: execution t is the subsequence that mask t keeps of program t, run under its own
// seed, max_messages and looking_for and recorded by the warp engine as demi_fuzz_trace records it.

// Slots per recording launch: record_chunk's, or fewer when DEMI_TEST_FUZZ_MANY_SLOTS is set (tests force several
// launches with it).
static uint32_t fuzz_many_chunk(uint32_t cap_events, uint32_t par_cap) {
  uint32_t c = record_chunk(cap_events, par_cap, 0);
  if (const char* e = getenv("DEMI_TEST_FUZZ_MANY_SLOTS"))
    if (*e) c = std::max(1u, std::min(c, (uint32_t)strtoul(e, nullptr, 10)));
  return c;
}

extern "C" int32_t demi_fuzz_traces_many(demi_handle* h, uint32_t n_traces, const demi_ext_event* externals,
                                         const uint32_t* ext_offsets, const uint32_t* n_externals, const uint64_t* masks,
                                         uint32_t mask_words, const int64_t* seeds, const int32_t* max_messages,
                                         const uint32_t* looking_for, const demi_fuzz_params* p, demi_event* events,
                                         uint32_t cap_events, uint32_t* n_events, uint16_t* dep_parent, uint32_t cap_nodes,
                                         uint32_t* n_nodes, demi_fuzz_result* results, int32_t* status) {
  if (!h) return DEMI_ERR_INVALID;
  static const char* who = "demi_fuzz_traces_many";
  if (!n_traces) return DEMI_OK;
  if (!externals || !ext_offsets || !n_externals || !seeds || !max_messages || !looking_for || !p || !events || !cap_events ||
      !n_events || !status)
    return fail(h, DEMI_ERR_INVALID, "%s: null argument", who);
  if (dep_parent && (!n_nodes || !cap_nodes || cap_nodes > 65536))
    return fail(h, DEMI_ERR_INVALID, "%s: a tree needs n_nodes and cap_nodes in 1..65536", who);
  if (masks)
    for (uint32_t t = 0; t < n_traces; t++)
      if ((uint64_t)mask_words * 64 < n_externals[t])
        return fail(h, DEMI_ERR_INVALID, "%s: mask_words %u too small for the %u externals of trace %u", who, mask_words, n_externals[t], t);
  { int32_t mrc = demi_need_model(h); if (mrc != DEMI_OK) return mrc; }
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  const uint32_t n = n_traces;
  h->perf.kernel_launches = 0; h->perf.prefixes = 0; h->perf.kernel_ms = 0;
  memset(n_events, 0, (size_t)n * sizeof(uint32_t));
  if (n_nodes) memset(n_nodes, 0, (size_t)n * sizeof(uint32_t));
  if (results) memset(results, 0, (size_t)n * sizeof(demi_fuzz_result));
  // demi_set_externals's checks of each program; the programs are uploaded once
  ProgramSet ps;
  int32_t rc = program_set(h, n, externals, ext_offsets, n_externals, seeds, max_messages, looking_for, p, ps);
  if (rc != DEMI_OK) return rc;
  // Then demi_random_test_trace's and plan_launch's of each subsequence.  Every execution runs on the variant its single
  // call picks: the traces are grouped by it, so that a HardKill or SrcDstFIFO program moves no other program.
  uint32_t mw = masks ? mask_words : 1;                // without masks every trace keeps all: one row of ones serves all
  if (!masks) for (uint32_t t = 0; t < n; t++) mw = std::max(mw, (n_externals[t] + 63) / 64);
  const std::vector<uint64_t> ones(mw, ~0ull);
  std::vector<ManyProgram> sub(n);                     // what each trace's mask keeps
  std::vector<ManyItem> items;
  std::vector<std::string> msg(n);
  demi_handle eh;                                      // a trace's refusal
  for (uint32_t t = 0; t < n; t++) {
    status[t] = ps.pre[t];
    if (ps.pre[t] != DEMI_OK) { msg[t] = ps.pre_msg[t]; continue; }
    const demi_ext_event* ev = externals + ext_offsets[t];
    const uint64_t* mk = masks ? masks + (size_t)t * mask_words : ones.data();
    ManyProgram& sp = sub[t];
    for (uint32_t i = 0; i < n_externals[t]; i++)
      if ((mk[i >> 6] >> (i & 63)) & 1ull) {
        sp.len++;
        if (ev[i].kind == DEMI_EXT_SEND) sp.info.sends++;
        if (ev[i].kind == DEMI_EXT_HARD_KILL) sp.info.hard_kill = true;
      }
    if (!sp.len) { status[t] = DEMI_ERR_INVALID; msg[t] = "demi_random_test_trace: the mask keeps no event"; continue; }
    sp.pcap = demi_pending_cap(demi_model_key(h), max_messages[t], sp.info.sends);
    const Variant* v;
    status[t] = check_variant(h, &eh, LM_RECORD_PARAMS, sp.info, sp.pcap, demi_tosend_cap(sp.info.sends), &v);
    if (status[t] != DEMI_OK) { msg[t] = eh.err; continue; }
    items.push_back(ManyItem{t, (uint32_t)(v - variants().data()), mk});
  }
  const uint32_t par_cap = dep_parent ? cap_nodes : 0;
  cudaStream_t s = h->stream;
  DevBuf rbuf;
  std::vector<uint32_t> cnt;
  std::vector<demi_fuzz_result> res;
  std::vector<demi_event> hev;
  std::vector<uint16_t> hpar;
  double ms_all = 0;
  rc = launch_many(h, ps, LM_RECORD_PARAMS, 1, sub.data(), items, mw, fuzz_many_chunk(cap_events, par_cap), 0, [&](ManyLaunch& L) -> int32_t {
    const uint32_t m = L.m;
    Records rec;
    int32_t rc = stage_records(h, &L.plan, m, nullptr, cap_events, par_cap, 0, rbuf, &rec, s);
    if (rc != DEMI_OK) return rc;
    KernelArgs& a = L.plan.args;
    a.sum_steps = nullptr; a.n_violations = nullptr;      // the handle's counters stay as they were
    a.rec_params = L.params;
    CUDA_TRY(h, cudaEventRecord(h->ev0, s));
    if (h->cfg.model == DEMI_MODEL_IR) CUDA_TRY(h, ir_bind(h->ir_dev, s));
    L.plan.v->fn[LM_RECORD_PARAMS]<<<L.plan.grid, WARPS * 32, L.plan.smem, s>>>(a);
    CUDA_TRY(h, cudaGetLastError());
    CUDA_TRY(h, cudaEventRecord(h->ev1, s));
    h->perf.kernel_launches++;
    h->perf.prefixes += m;
    res.resize(m); cnt.resize((size_t)m * 4);
    CUDA_TRY(h, cudaMemcpyAsync(cnt.data(), rec.counts, cnt.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(h, cudaMemcpyAsync(res.data(), rec.results, res.size() * sizeof(demi_fuzz_result), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(h, cudaStreamSynchronize(s));
    float ms = 0.f;
    CUDA_TRY(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
    ms_all += ms;
    // the rows travel as wide as the launch's longest successful recording, then go to their traces' rows
    uint32_t width = 0, pwidth = 0;
    for (uint32_t k = 0; k < m; k++) {
      const uint32_t t = items[L.item[k]].trace;
      n_events[t] = cnt[(size_t)k * 4];
      if (n_nodes) n_nodes[t] = cnt[(size_t)k * 4 + 1];
      if (results) results[t] = res[k];
      if (res[k].status) {
        status[t] = DEMI_ERR_CAPACITY; msg[t] = "demi_fuzz_trace: prefix status " + std::to_string(res[k].status);
      } else {
        width = std::max(width, std::min(cnt[(size_t)k * 4], cap_events));
        pwidth = std::max(pwidth, std::min(cnt[(size_t)k * 4 + 1], par_cap));
      }
    }
    if (width) {
      hev.resize((size_t)m * width);
      CUDA_TRY(h, cudaMemcpy2DAsync(hev.data(), (size_t)width * sizeof(demi_event), rec.events, (size_t)cap_events * sizeof(demi_event),
                                    (size_t)width * sizeof(demi_event), m, cudaMemcpyDeviceToHost, s));
    }
    if (pwidth) {
      hpar.resize((size_t)m * pwidth);
      CUDA_TRY(h, cudaMemcpy2DAsync(hpar.data(), (size_t)pwidth * sizeof(uint16_t), rec.parents, (size_t)par_cap * sizeof(uint16_t),
                                    (size_t)pwidth * sizeof(uint16_t), m, cudaMemcpyDeviceToHost, s));
    }
    if (width || pwidth) CUDA_TRY(h, cudaStreamSynchronize(s));
    for (uint32_t k = 0; k < m; k++) {
      const uint32_t t = items[L.item[k]].trace;
      if (status[t] != DEMI_OK) continue;
      std::copy_n(hev.data() + (size_t)k * width, std::min(n_events[t], cap_events), events + (size_t)t * cap_events);
      if (dep_parent) std::copy_n(hpar.data() + (size_t)k * pwidth, std::min(n_nodes[t], par_cap), dep_parent + (size_t)t * par_cap);
    }
    return DEMI_OK;
  });
  if (rc != DEMI_OK) return rc;
  h->perf.kernel_ms = ms_all;
  // a failing trace has no events and no tree: zeros where they would be
  int64_t bad = -1;
  for (uint32_t t = 0; t < n; t++) {
    if (status[t] == DEMI_OK) continue;
    if (bad < 0) bad = t;
    memset(events + (size_t)t * cap_events, 0, (size_t)cap_events * sizeof(demi_event));
    if (dep_parent) memset(dep_parent + (size_t)t * par_cap, 0, (size_t)par_cap * sizeof(uint16_t));
  }
  if (bad >= 0) h->err = trace_msg(who, (uint32_t)bad, msg[bad]);
  return DEMI_OK;
}

extern "C" int32_t demi_lane_kernel(const demi_handle* h) { return h ? h->lane_kernel : DEMI_ERR_INVALID; }
extern "C" int32_t demi_lane_tree_depth(const demi_handle* h) { return h ? h->lane_tree_depth : DEMI_ERR_INVALID; }
extern "C" int32_t demi_lane_row_bytes(const demi_handle* h) { return h ? h->lane_row_bytes : DEMI_ERR_INVALID; }

extern "C" int32_t demi_stats(const demi_handle* h, demi_perf* out) {
  if (!h || !out) return DEMI_ERR_INVALID;
  *out = h->perf;
  return DEMI_OK;
}
