// capi_replay_many.cu — STSSched replay and DDMin over a set of traces (demi_set_traces): the tests of many traces in
// one K2 launch, and one DDMin per trace, their speculative batches served together.
//
// A minimisation of a small trace asks for tens to a few hundred tests at a time, a small fraction of one wave of the
// replay kernel, and waits for each launch.  Here the drivers of many traces run side by side, each on a host thread
// with a rendezvous (many_rendezvous.hpp): one launch evaluates the union of the requests of every driver in flight.
//
// Internal minimization over a set runs the same way without threads: its driver (intmin_driver.hpp) is not recursive,
// so every trace's driver steps in lock-step rounds of one exact launch and one recording launch.  Wildcard
// minimization (wildcard_driver.hpp) steps the same way, with the WILD kernel for both launches.
#include <functional>
#include "replay_kernel.cuh"
#include "engine.hpp"
#include "ddmin_driver.hpp"
#include "intmin_driver.hpp"
#include "wildcard_driver.hpp"
#include "many_rendezvous.hpp"

using namespace demi;

namespace {

// tests per launch: larger unions are evaluated in several launches
constexpr uint32_t MANY_MAX_TESTS = 1u << 20;
// a recording launch's rows (tests x cap_events events) stay under this many bytes
constexpr uint64_t MANY_MAX_REC_BYTES = 1ull << 30;
// a round of demi_wildcard_minimize_many admits traces while their include masks stay under this many host bytes
// (DEMI_TEST_WC_ROUND_BYTES overrides it, for tests)
constexpr uint64_t WC_MANY_ROUND_BYTES = 256ull << 20;

struct LaunchCounts { uint32_t launches = 0; uint64_t tests = 0, violations = 0, deliveries = 0; double ms = 0; };

// The traces a multi-trace launch reads: the set's, or the working traces of demi_internal_minimize_many
struct Views {
  const std::vector<ReplayTraceView>* host; const ReplayTraceView* dev;
  static Views of(const demi_handle::TraceSet& S) { return Views{&S.view, S.views.get<const ReplayTraceView>()}; }
};
// A recording launch (the REC kernel): each test's EventTrace, at most `cap` events, is handed to take(test, events,
// count, ignored, n_ignored) in input order once the launch is done; a wildcard recording also hands over the trace
// positions of the deliveries the test ignored (none otherwise)
struct Recording {
  uint32_t cap;
  std::function<void(uint32_t, const demi_event*, uint32_t, const uint32_t*, uint32_t)> take;
};
// A wildcard launch (the WILD kernel): the masks are include masks over each trace's deliveries, modes[t] is trace t's
// mode table on the device, and a recording test reports at most ign_cap ignored deliveries
struct Wild { const uint32_t* const* modes; uint32_t ign_cap; };

// One K2 launch over tests [0, n): test i replays mask i (every external when masks is null) on trace trace_of_test[i]
// (validated by the caller), leaving out trace event skips[i] (none when skips is null or it is 0xFFFFFFFF).  Tests
// are grouped by trace into warp tiles, longest trace first; results come back in input order.  With `wild`, mask i is
// test i's include mask (mw words) instead.
int32_t launch_many(demi_handle* h, const Views& V, const uint32_t* trace_of_test, const uint64_t* masks,
                    const uint32_t* skips, uint32_t n, uint32_t mw, const uint32_t* looking_for, uint32_t flags,
                    demi_replay_result* out, LaunchCounts& lc, const Recording* rec, const Wild* wild) {
  const std::vector<ReplayTraceView>& view = *V.host;
  const uint32_t n_traces = (uint32_t)view.size();
  // counting sort of the tests by the rank of their trace (longer traces first, then by index)
  std::vector<uint32_t> count(n_traces + 1, 0);
  for (uint32_t i = 0; i < n; i++) count[trace_of_test[i]]++;
  std::vector<uint32_t> order_t;
  for (uint32_t t = 0; t < n_traces; t++) if (count[t]) order_t.push_back(t);
  std::stable_sort(order_t.begin(), order_t.end(), [&](uint32_t a, uint32_t b) { return view[a].n_events > view[b].n_events; });
  std::vector<uint32_t> first(n_traces, 0);
  std::vector<uint4> tiles;
  ReplayTraceView geometry{};                       // the scratch's: the largest of the launch's traces
  uint32_t pos = 0;
  for (uint32_t t : order_t) {
    first[t] = pos;
    for (uint32_t k = 0; k < count[t]; k += 32) tiles.push_back(make_uint4(t, pos + k, std::min(32u, count[t] - k), looking_for[t]));
    pos += count[t];
    const ReplayTraceView& v = view[t];
    geometry.table_slots = std::max(geometry.table_slots, v.table_slots);
    geometry.tosend_cap = std::max(geometry.tosend_cap, v.tosend_cap);
    geometry.n_uniq_words = std::max(geometry.n_uniq_words, v.n_uniq_words);
    geometry.pending_cap = std::max(geometry.pending_cap, v.pending_cap);
  }
  std::vector<uint32_t> slot(n);                    // test i runs at position slot[i] of the grouped order
  std::vector<uint64_t> grouped(masks ? (size_t)n * mw : 0);
  std::vector<uint32_t> grouped_skips(skips ? n : 0);
  for (uint32_t i = 0; i < n; i++) {
    slot[i] = first[trace_of_test[i]]++;
    if (masks) std::copy(masks + (size_t)i * mw, masks + (size_t)(i + 1) * mw, grouped.begin() + (size_t)slot[i] * mw);
    if (skips) grouped_skips[slot[i]] = skips[i];
  }
  cudaStream_t s = h->stream;
  int32_t rc;
  const size_t mbytes = grouped.size() * sizeof(uint64_t), tbytes = tiles.size() * sizeof(uint4);
  const size_t sbytes = grouped_skips.size() * sizeof(uint32_t);
  const size_t rbytes = (size_t)n * sizeof(demi_replay_result);
  if ((rc = h->rp_masks.grow(h, tbytes + mbytes + sbytes)) != DEMI_OK) return rc;
  if ((rc = h->rp_results.grow(h, rbytes)) != DEMI_OK) return rc;
  char* base = h->rp_masks.get<char>();
  CUDA_TRY(h, cudaMemcpyAsync(base, tiles.data(), tbytes, cudaMemcpyHostToDevice, s));
  if (masks) CUDA_TRY(h, cudaMemcpyAsync(base + tbytes, grouped.data(), mbytes, cudaMemcpyHostToDevice, s));
  if (skips) CUDA_TRY(h, cudaMemcpyAsync(base + tbytes + mbytes, grouped_skips.data(), sbytes, cudaMemcpyHostToDevice, s));
  ReplayArgs a = replay_args(h, geometry, 0, flags);
  a.masks = masks ? (const uint64_t*)(base + tbytes) : nullptr; a.n_masks = n; a.mask_words = mw;
  a.skips = skips ? (const uint32_t*)(base + tbytes + mbytes) : nullptr;
  a.results = h->rp_results.get<demi_replay_result>();
  if (wild) {                                       // every external is replayed; the masks select deliveries
    a.wc_include = a.masks; a.wc_words = mw;
    a.masks = nullptr; a.mask_words = 1;
    std::copy(h->clock_incr, h->clock_incr + 8, a.wc_incr);
  }
  const size_t row_bytes = rec ? (size_t)rec->cap * sizeof(demi_event) : 0;
  const size_t ign_cap = rec && wild ? wild->ign_cap : 0, count_off = n * row_bytes, ign_off = count_off + (size_t)n * sizeof(uint32_t);
  if (rec) {                                        // rows, one count per test; a wildcard's ignored rows and counts
    if ((rc = h->rp_rec.grow(h, ign_off + (size_t)n * (ign_cap + (ign_cap ? 1 : 0)) * sizeof(uint32_t))) != DEMI_OK) return rc;
    a.rec_events = h->rp_rec.get<demi_event>(); a.rec_cap = rec->cap;
    a.rec_count = (uint32_t*)(h->rp_rec.get<char>() + count_off);
    if (ign_cap) {
      a.wc_ignored = (uint32_t*)(h->rp_rec.get<char>() + ign_off); a.wc_ignored_cap = (uint32_t)ign_cap;
      a.wc_ignored_count = a.wc_ignored + (size_t)n * ign_cap;
    }
  }
  const ReplayTiles many{V.dev, (const uint4*)base, (uint32_t)tiles.size(), wild ? wild->modes : nullptr};
  if ((rc = replay_launch(h, a, wild != nullptr, rec != nullptr, &many, true, s)) != DEMI_OK) return rc;
  std::vector<demi_replay_result> res(n);
  std::vector<uint32_t> rec_count(rec ? n : 0), ign_count(ign_cap ? n : 0);
  unsigned long long c[2] = {0, 0};
  CUDA_TRY(h, cudaMemcpyAsync(res.data(), a.results, rbytes, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaMemcpyAsync(c, a.counters, sizeof(c), cudaMemcpyDeviceToHost, s));
  if (rec) CUDA_TRY(h, cudaMemcpyAsync(rec_count.data(), a.rec_count, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  if (ign_cap) CUDA_TRY(h, cudaMemcpyAsync(ign_count.data(), a.wc_ignored_count, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaStreamSynchronize(s));
  float ms = 0;
  CUDA_TRY(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  for (uint32_t i = 0; i < n; i++) out[i] = res[slot[i]];
  if (rec) {
    // the rows as far as the longest recording of the launch reaches, in one strided copy (and so the ignored rows)
    const uint32_t width = std::min(rec->cap, *std::max_element(rec_count.begin(), rec_count.end()));
    std::vector<demi_event> rows((size_t)n * width);
    if (width)
      CUDA_TRY(h, cudaMemcpy2D(rows.data(), width * sizeof(demi_event), a.rec_events, row_bytes, width * sizeof(demi_event), n,
                               cudaMemcpyDeviceToHost));
    const uint32_t iw = ign_cap ? std::min<uint32_t>((uint32_t)ign_cap, *std::max_element(ign_count.begin(), ign_count.end())) : 0;
    std::vector<uint32_t> ign((size_t)n * iw);
    if (iw)
      CUDA_TRY(h, cudaMemcpy2D(ign.data(), iw * sizeof(uint32_t), a.wc_ignored, ign_cap * sizeof(uint32_t), iw * sizeof(uint32_t), n,
                               cudaMemcpyDeviceToHost));
    for (uint32_t i = 0; i < n; i++)
      rec->take(i, rows.data() + (size_t)slot[i] * width, rec_count[slot[i]], ign.data() + (size_t)slot[i] * iw,
                ign_cap ? std::min<uint32_t>(ign_count[slot[i]], iw) : 0);
  }
  lc.launches++; lc.tests += n; lc.ms += ms; lc.violations += c[0]; lc.deliveries += c[1];
  return DEMI_OK;
}

void set_perf(demi_handle* h, const LaunchCounts& lc) {
  h->perf.kernel_launches = lc.launches; h->perf.prefixes = lc.tests; h->perf.kernel_ms = lc.ms;
  h->perf.violations = lc.violations; h->perf.deliveries = lc.deliveries;
}

// n tests in launches of at most MANY_MAX_TESTS (and, recording, of at most MANY_MAX_REC_BYTES of rows)
int32_t replay_many(demi_handle* h, const Views& V, const uint32_t* trace_of_test, const uint64_t* masks,
                    const uint32_t* skips, uint32_t n, uint32_t mw, const uint32_t* looking_for, uint32_t flags,
                    demi_replay_result* out, LaunchCounts& lc, const Recording* rec = nullptr, const Wild* wild = nullptr) {
  uint32_t per_launch = MANY_MAX_TESTS;
  if (rec) {
    const uint64_t row = (uint64_t)rec->cap * sizeof(demi_event) + (wild ? ((uint64_t)wild->ign_cap + 1) * sizeof(uint32_t) : 0);
    per_launch = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(per_launch, MANY_MAX_REC_BYTES / row));
  }
  for (uint32_t off = 0; off < n; off += per_launch) {
    const uint32_t m = std::min(per_launch, n - off);
    Recording part;
    if (rec)
      part = Recording{rec->cap, [&](uint32_t i, const demi_event* ev, uint32_t k, const uint32_t* ign, uint32_t ni) {
                         rec->take(off + i, ev, k, ign, ni);
                       }};
    const int32_t rc = launch_many(h, V, trace_of_test + off, masks ? masks + (size_t)off * mw : nullptr,
                                   skips ? skips + off : nullptr, m, mw, looking_for, flags, out + off, lc, rec ? &part : nullptr,
                                   wild);
    if (rc != DEMI_OK) return rc;
  }
  return DEMI_OK;
}

// ---------------------------------------------------------------------- rounds of DDMin drivers
typedef ManyRequest<demi_replay_result> Request;

// STSSched as DDMin's TestOracle on trace `trace` of the set, as StsDDMinDriver (capi_replay.cu) on the single trace
struct SetDDMinDriver : DDMinDriver {
  Rendezvous<demi_replay_result>* R; uint32_t trace;
  int32_t evaluate(const uint64_t* masks, size_t n, signed char* out) override {
    Request q; q.trace = trace; q.masks = masks; q.n = n;
    R->submit(q);
    return q.rc != DEMI_OK ? q.rc : replay_verdicts(h, q.res.data(), n, out);
  }
};

}  // namespace

extern "C" int32_t demi_set_traces(demi_handle* h, uint32_t n_traces,
                                   const demi_event* events, const uint32_t* event_offsets, const uint32_t* n_events,
                                   const demi_ext_event* externals, const uint32_t* ext_offsets, const uint32_t* n_externals) {
  if (!h) return DEMI_ERR_INVALID;
  if (!n_traces) return fail(h, DEMI_ERR_INVALID, "demi_set_traces: no traces");
  if (!events || !event_offsets || !n_events || !externals || !ext_offsets || !n_externals)
    return fail(h, DEMI_ERR_INVALID, "demi_set_traces: null buffer");
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  { int32_t mrc = demi_need_model(h); if (mrc != DEMI_OK) return mrc; }
  // the new set is built aside and replaces the old one only when every trace passed and every upload succeeded
  std::vector<demi_event> ev_all; std::vector<uint16_t> ord_all, sidx_all; std::vector<demi_ext_event> ext_all;
  std::vector<size_t> ev_off(n_traces), ext_off(n_traces), sidx_off(n_traces);
  std::map<std::pair<uint32_t, uint32_t>, std::pair<size_t, size_t>> ext_seen;   // a program shared by traces is stored once
  demi_handle::TraceSet S;
  S.n = n_traces;
  S.ext.resize(n_traces); S.view.resize(n_traces);
  char who[64];
  TraceTables t;
  for (uint32_t i = 0; i < n_traces; i++) {
    snprintf(who, sizeof(who), "demi_set_traces: trace %u", i);
    const demi_event* ev = events + event_offsets[i];
    const demi_ext_event* ex = externals + ext_offsets[i];
    int32_t rc = check_trace(h, who, ev, n_events[i], ex, n_externals[i]);
    if (rc == DEMI_OK) rc = trace_tables(h, who, ev, n_events[i], ex, n_externals[i], t);
    if (rc != DEMI_OK) return rc;
    ev_off[i] = ev_all.size();
    ev_all.insert(ev_all.end(), ev, ev + n_events[i]);
    ord_all.insert(ord_all.end(), t.ordinal.begin(), t.ordinal.end());
    auto key = std::make_pair(ext_offsets[i], n_externals[i]);
    auto it = ext_seen.find(key);
    if (it == ext_seen.end()) {
      it = ext_seen.emplace(key, std::make_pair(ext_all.size(), sidx_all.size())).first;
      ext_all.insert(ext_all.end(), ex, ex + n_externals[i]);
      sidx_all.insert(sidx_all.end(), t.sidx.begin(), t.sidx.end());
    }
    ext_off[i] = it->second.first; sidx_off[i] = it->second.second;
    S.ext[i].assign(ex, ex + n_externals[i]);
    S.view[i] = trace_view(t, n_events[i], n_externals[i]);
  }
  if (sidx_all.empty()) sidx_all.push_back(0);
  int32_t rc;
  if ((rc = S.events.upload(h, ev_all.data(), ev_all.size() * sizeof(demi_event))) != DEMI_OK) return rc;
  if ((rc = S.ordinal.upload(h, ord_all.data(), ord_all.size() * sizeof(uint16_t))) != DEMI_OK) return rc;
  if ((rc = S.externals.upload(h, ext_all.data(), ext_all.size() * sizeof(demi_ext_event))) != DEMI_OK) return rc;
  if ((rc = S.send_index.upload(h, sidx_all.data(), sidx_all.size() * sizeof(uint16_t))) != DEMI_OK) return rc;
  for (uint32_t i = 0; i < n_traces; i++) {
    ReplayTraceView& v = S.view[i];
    v.events = S.events.get<const uint4>() + ev_off[i]; v.ev_ordinal = S.ordinal.get<const uint16_t>() + ev_off[i];
    v.ext = S.externals.get<const uint4>() + ext_off[i]; v.send_ext_index = S.send_index.get<const uint16_t>() + sidx_off[i];
  }
  if ((rc = S.views.upload(h, S.view.data(), S.view.size() * sizeof(ReplayTraceView))) != DEMI_OK) return rc;
  if ((rc = h->rp_counters.grow(h, 2 * sizeof(unsigned long long))) != DEMI_OK) return rc;
  h->set = std::move(S);
  return DEMI_OK;
}

extern "C" int32_t demi_replay_batch_many(demi_handle* h, const uint32_t* trace_of_test, const uint64_t* masks, uint32_t n_tests,
                                          uint32_t mask_words, const uint32_t* looking_for, uint32_t flags,
                                          demi_replay_result* out) {
  if (!h) return DEMI_ERR_INVALID;
  if (!trace_of_test || !masks || !looking_for || !out) return fail(h, DEMI_ERR_INVALID, "demi_replay_batch_many: null buffer");
  if (!h->set.n) return fail(h, DEMI_ERR_STATE, "demi_set_traces has not been called");
  for (uint32_t i = 0; i < n_tests; i++) {
    const uint32_t t = trace_of_test[i];
    if (t >= h->set.n) return fail(h, DEMI_ERR_INVALID, "demi_replay_batch_many: test %u names trace %u of %u", i, t, h->set.n);
    if ((uint64_t)mask_words * 64 < h->set.ext[t].size())
      return fail(h, DEMI_ERR_INVALID, "mask_words %u too small for the %zu externals of trace %u", mask_words, h->set.ext[t].size(), t);
  }
  if (n_tests == 0) return DEMI_OK;
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  LaunchCounts lc;
  const int32_t rc = replay_many(h, Views::of(h->set), trace_of_test, masks, nullptr, n_tests, mask_words, looking_for, flags, out, lc);
  set_perf(h, lc);
  return rc;
}

extern "C" int32_t demi_ddmin_many(demi_handle* h, const uint32_t* looking_for, uint32_t flags, int32_t check_unmodified,
                                   uint64_t* mcs_masks, uint32_t mask_words, uint32_t* iteration_sizes, uint32_t cap_iterations,
                                   demi_ddmin_out* out, int32_t* status) {
  if (!h) return DEMI_ERR_INVALID;
  if (!looking_for || !mcs_masks || !out || !status) return fail(h, DEMI_ERR_INVALID, "demi_ddmin_many: null buffer");
  const uint32_t n = h->set.n;
  if (!n) return fail(h, DEMI_ERR_STATE, "demi_set_traces has not been called");
  for (uint32_t t = 0; t < n; t++)
    if ((uint64_t)mask_words * 64 < h->set.ext[t].size())
      return fail(h, DEMI_ERR_INVALID, "mask_words %u too small for the %zu externals of trace %u", mask_words, h->set.ext[t].size(), t);
  // drivers in flight: DEMI_DDMIN_MANY_WINDOW (many_window)
  uint32_t window;
  { int32_t wrc = many_window(h, n, window); if (wrc != DEMI_OK) return wrc; }
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  memset(out, 0, (size_t)n * sizeof(demi_ddmin_out));
  auto drive = [&](uint32_t t, Rendezvous<demi_replay_result>& R, demi_handle* eh) -> int32_t {
    SetDDMinDriver d;
    d.R = &R; d.trace = t;
    d.h = eh; d.looking_for = looking_for[t]; d.flags = flags; d.mw = mask_words;
    d.n_ext = (uint32_t)h->set.ext[t].size(); d.ext = h->set.ext[t].data();
    return ddmin_sts(d, check_unmodified, mcs_masks + (size_t)t * mask_words,
                     iteration_sizes ? iteration_sizes + (size_t)t * cap_iterations : nullptr, cap_iterations, out + t);
  };
  LaunchCounts lc;
  auto serve = [&](std::vector<Request*>& batch) -> int32_t {
    std::vector<uint32_t> tr;
    std::vector<uint64_t> flat;
    flatten_requests(batch, mask_words, tr, flat);
    std::vector<demi_replay_result> res(tr.size());
    const int32_t rc = replay_many(h, Views::of(h->set), tr.data(), flat.data(), nullptr, (uint32_t)tr.size(), mask_words, looking_for,
                                   flags, res.data(), lc);
    if (rc != DEMI_OK) return rc;
    scatter_results(batch, res);
    return DEMI_OK;
  };
  const int32_t rc = run_many<demi_replay_result>(h, "demi_ddmin_many", n, window, drive, serve, status);
  set_perf(h, lc);
  return rc;
}

extern "C" int32_t demi_replay_traces_many(demi_handle* h, const uint32_t* trace_of_test, const uint64_t* masks,
                                           const uint32_t* skip_events, uint32_t n_tests, uint32_t mask_words,
                                           const uint32_t* looking_for, uint32_t flags,
                                           demi_event* events, uint32_t cap_events, uint32_t* n_events,
                                           demi_replay_result* results) {
  if (!h) return DEMI_ERR_INVALID;
  if (!trace_of_test || !looking_for || !events || !cap_events || !n_events || !results)
    return fail(h, DEMI_ERR_INVALID, "demi_replay_traces_many: null buffer");
  if (!h->set.n) return fail(h, DEMI_ERR_STATE, "demi_set_traces has not been called");
  for (uint32_t i = 0; i < n_tests; i++) {
    const uint32_t t = trace_of_test[i];
    if (t >= h->set.n) return fail(h, DEMI_ERR_INVALID, "demi_replay_traces_many: test %u names trace %u of %u", i, t, h->set.n);
    if (masks && (uint64_t)mask_words * 64 < h->set.ext[t].size())
      return fail(h, DEMI_ERR_INVALID, "mask_words %u too small for the %zu externals of trace %u", mask_words, h->set.ext[t].size(), t);
  }
  if (n_tests == 0) return DEMI_OK;
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  LaunchCounts lc;
  const Recording rec{cap_events, [&](uint32_t i, const demi_event* ev, uint32_t k, const uint32_t*, uint32_t) {
    n_events[i] = k;
    std::copy(ev, ev + k, events + (size_t)i * cap_events);
  }};
  const int32_t rc = replay_many(h, Views::of(h->set), trace_of_test, masks, skip_events, n_tests, mask_words, looking_for,
                                 flags, results, lc, &rec);
  set_perf(h, lc);
  return rc;
}

extern "C" int32_t demi_internal_minimize_many(demi_handle* h, const uint32_t* looking_for, uint32_t flags,
                                               demi_event* out_traces, uint32_t cap_events,
                                               uint32_t* internal_sizes, uint32_t cap_sizes,
                                               demi_intmin_out* out, int32_t* status) {
  if (!h) return DEMI_ERR_INVALID;
  if (!looking_for || !out_traces || !cap_events || !out || !status)
    return fail(h, DEMI_ERR_INVALID, "demi_internal_minimize_many: null buffer");
  const demi_handle::TraceSet& S = h->set;
  const uint32_t n = S.n;
  if (!n) return fail(h, DEMI_ERR_STATE, "demi_set_traces has not been called");
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  const bool use_fifo = (flags & DEMI_IM_SRC_DST_FIFO) != 0;
  flags &= ~DEMI_IM_SRC_DST_FIFO;
  // the set's traces, read back once; the set itself is left as it is
  std::vector<demi_event> all(S.events.bytes() / sizeof(demi_event));
  if (!all.empty()) CUDA_TRY(h, cudaMemcpy(all.data(), S.events.get(), all.size() * sizeof(demi_event), cudaMemcpyDeviceToHost));
  std::vector<demi::IntMinDriver> d(n);
  for (uint32_t t = 0; t < n; t++) {
    const demi_event* ev = all.data() + (S.view[t].events - S.events.get<const uint4>());
    d[t].init(ev, S.view[t].n_events, demi_ext_type_mask(h), use_fifo, out + t);
    status[t] = DEMI_OK;
  }
  // The working traces: a view table of their own.  A trace that advances gets its recorded trace and ordinals in the
  // round's upload; its externals and their Send index stay the set's.
  std::vector<ReplayTraceView> work = S.view;
  DevBuf work_dev;
  std::vector<DevBuf> rounds;                        // every round's new traces (a view may point into any of them)
  std::vector<std::string> msg(n);
  std::vector<uint8_t> live(n, 1);
  auto fail_trace = [&](uint32_t t, int32_t code, const std::string& m) { status[t] = code; msg[t] = m; live[t] = 0; };
  LaunchCounts lc;
  int32_t rc;
  for (;;) {
    // 1. every unfinished driver's candidates
    std::vector<uint32_t> tr, skip, first(n, 0);
    for (uint32_t t = 0; t < n; t++) {
      if (!live[t]) continue;
      const std::vector<uint32_t>& cand = d[t].candidates();
      if (cand.empty()) { live[t] = 0; continue; }
      first[t] = (uint32_t)tr.size();
      tr.insert(tr.end(), cand.size(), t);
      skip.insert(skip.end(), cand.begin(), cand.end());
    }
    if (tr.empty()) break;
    // 2. their union in one exact launch; 3. each driver commits
    std::vector<demi_replay_result> res(tr.size());
    const Views V{&work, work_dev.bytes() ? work_dev.get<const ReplayTraceView>() : S.views.get<const ReplayTraceView>()};
    if ((rc = replay_many(h, V, tr.data(), nullptr, skip.data(), (uint32_t)tr.size(), 1, looking_for, flags, res.data(), lc)) != DEMI_OK)
      break;
    std::vector<uint32_t> rec_tr, rec_skip;
    for (uint32_t t = 0; t < n; t++) {
      if (!live[t]) continue;
      uint32_t s = 0;
      const demi::IntMinDriver::Step step = d[t].commit(res.data() + first[t], &s);
      if (step == demi::IntMinDriver::FAILED) fail_trace(t, d[t].error, d[t].msg);
      else if (step == demi::IntMinDriver::DONE) live[t] = 0;
      else { rec_tr.push_back(t); rec_skip.push_back(s); }
    }
    if (rec_tr.empty()) continue;
    // 4. every success re-run in one recording launch; the recorded trace advances its driver
    std::vector<demi_replay_result> rres(rec_tr.size());
    std::vector<uint32_t> advanced;
    const Recording rec{cap_events, [&](uint32_t i, const demi_event* ev, uint32_t k, const uint32_t*, uint32_t) {
      const uint32_t t = rec_tr[i];
      if (rres[i].status == DEMI_PS_EVENT_OVF)
        return fail_trace(t, DEMI_ERR_CAPACITY, "demi_internal_minimize_many: trace " + std::to_string(t) +
                                                " needs a recording longer than cap_events " + std::to_string(cap_events));
      if (!d[t].advance(rres[i], ev, k)) return fail_trace(t, d[t].error, d[t].msg);
      advanced.push_back(t);
    }};
    if ((rc = replay_many(h, V, rec_tr.data(), nullptr, rec_skip.data(), (uint32_t)rec_tr.size(), 1, looking_for, flags,
                          rres.data(), lc, &rec)) != DEMI_OK)
      break;
    // 5. the advanced traces' side tables on the host, their records in one upload, the view table in another
    std::vector<demi_event> ev_all; std::vector<uint16_t> ord_all;
    std::vector<size_t> off;
    TraceTables tt;
    char who[80];
    for (uint32_t t : advanced) {
      const std::vector<demi_event>& cur = d[t].cur;
      snprintf(who, sizeof(who), "demi_internal_minimize_many: trace %u", t);
      if ((rc = trace_tables(h, who, cur.data(), (uint32_t)cur.size(), S.ext[t].data(), (uint32_t)S.ext[t].size(), tt)) != DEMI_OK) {
        fail_trace(t, rc, h->err);
        off.push_back(SIZE_MAX);
        continue;
      }
      off.push_back(ev_all.size());
      ev_all.insert(ev_all.end(), cur.begin(), cur.end());
      ord_all.insert(ord_all.end(), tt.ordinal.begin(), tt.ordinal.end());
      const ReplayTraceView v = trace_view(tt, (uint32_t)cur.size(), (uint32_t)S.ext[t].size());
      ReplayTraceView& w = work[t];
      w.n_events = v.n_events; w.n_uniq_words = v.n_uniq_words;
      w.pending_cap = v.pending_cap; w.tosend_cap = v.tosend_cap; w.table_slots = v.table_slots;
    }
    rc = DEMI_OK;
    if (ev_all.empty()) continue;
    const size_t ev_bytes = ev_all.size() * sizeof(demi_event);
    rounds.emplace_back();
    DevBuf& b = rounds.back();
    if ((rc = b.grow(h, ev_bytes + ord_all.size() * sizeof(uint16_t))) != DEMI_OK) break;
    CUDA_TRY(h, cudaMemcpyAsync(b.get(), ev_all.data(), ev_bytes, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(b.get<char>() + ev_bytes, ord_all.data(), ord_all.size() * sizeof(uint16_t),
                                cudaMemcpyHostToDevice, h->stream));
    for (size_t k = 0; k < advanced.size(); k++) {
      if (off[k] == SIZE_MAX) continue;
      ReplayTraceView& w = work[advanced[k]];
      w.events = b.get<const uint4>() + off[k];
      w.ev_ordinal = (const uint16_t*)(b.get<char>() + ev_bytes) + off[k];
    }
    if ((rc = work_dev.grow(h, work.size() * sizeof(ReplayTraceView))) != DEMI_OK) break;
    CUDA_TRY(h, cudaMemcpyAsync(work_dev.get(), work.data(), work.size() * sizeof(ReplayTraceView), cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));    // the host vectors go out of scope
  }
  set_perf(h, lc);
  if (rc != DEMI_OK) return rc;
  for (uint32_t t = 0; t < n; t++)
    if (status[t] == DEMI_OK)
      d[t].finish(out_traces + (size_t)t * cap_events, cap_events, internal_sizes ? internal_sizes + (size_t)t * cap_sizes : nullptr,
                  cap_sizes);
  for (uint32_t t = 0; t < n; t++)
    if (status[t] != DEMI_OK) { h->err = msg[t]; break; }
  return DEMI_OK;
}

// ---------------------------------------------------------------------- wildcard tests over the set
namespace {

// The wildcard form of the set's traces, built once per call: each used trace's mode table (one upload, a device
// pointer per trace), and a view table of the call's own whose pending capacity is the wildcard one with the list's
// room equal to it, as wc_launch (capi_wildcard.cu) sets them for the single trace.  The set is left as it is.
struct WildSet {
  std::vector<demi_event> all;                       // the set's events, read back once
  std::vector<WcTrace> t;
  std::vector<ReplayTraceView> view;
  DevBuf view_dev, modes_dev;
  uint32_t ign_cap = 1;                              // the most deliveries of a used trace, plus one
  Wild wild() const { return Wild{(const uint32_t* const*)modes_dev.get<char>(), ign_cap}; }
  Views views() const { return Views{&view, view_dev.get<const ReplayTraceView>()}; }
};

// Mode tables of the traces with use[t] set; a trace whose Uniq ids repeat gets bad[t] = 1 and its message (bad may
// be null: then that trace fails the call with DEMI_ERR_INVALID)
int32_t wild_set(demi_handle* h, const char* who, const std::vector<uint8_t>& use, WildSet& W, std::vector<uint8_t>* bad,
                 std::vector<std::string>* msg) {
  const demi_handle::TraceSet& S = h->set;
  const uint32_t n = S.n;
  std::vector<demi_event>& all = W.all;
  all.resize(S.events.bytes() / sizeof(demi_event));
  if (!all.empty()) CUDA_TRY(h, cudaMemcpy(all.data(), S.events.get(), all.size() * sizeof(demi_event), cudaMemcpyDeviceToHost));
  W.t.assign(n, WcTrace());
  W.view = S.view;
  std::vector<uint32_t> modes;
  std::vector<size_t> off(n, SIZE_MAX);
  char name[96];
  for (uint32_t t = 0; t < n; t++) {
    if (!use[t]) continue;
    const demi_event* ev = all.data() + (S.view[t].events - S.events.get<const uint4>());
    std::string m;
    snprintf(name, sizeof(name), "%s: trace %u", who, t);
    if (!W.t[t].build(ev, S.view[t].n_events, demi_ext_type_mask(h), h->clock_incr, name, m)) {
      if (!bad) return fail(h, DEMI_ERR_INVALID, "%s", m.c_str());
      (*bad)[t] = 1; (*msg)[t] = m;
      continue;
    }
    off[t] = modes.size();
    modes.insert(modes.end(), W.t[t].ev.begin(), W.t[t].ev.end());
    ReplayTraceView& v = W.view[t];
    v.pending_cap = demi_wildcard_pending_cap(demi_model_key(h), (uint32_t)W.t[t].pos.size(), v.n_sends);
    v.table_slots = v.pending_cap;                   // list storage (the kernel compacts it in place)
    W.ign_cap = std::max<uint32_t>(W.ign_cap, (uint32_t)W.t[t].pos.size() + 1);
  }
  // the pointer table, then the mode tables
  const size_t ptr_bytes = ((size_t)n * sizeof(uint32_t*) + 15) & ~(size_t)15;
  int32_t rc;
  if ((rc = W.modes_dev.grow(h, ptr_bytes + std::max<size_t>(modes.size(), 1) * sizeof(uint32_t))) != DEMI_OK) return rc;
  const uint32_t* dev_modes = (const uint32_t*)(W.modes_dev.get<char>() + ptr_bytes);
  std::vector<const uint32_t*> ptr(n, nullptr);
  for (uint32_t t = 0; t < n; t++) if (off[t] != SIZE_MAX) ptr[t] = dev_modes + off[t];
  CUDA_TRY(h, cudaMemcpy(W.modes_dev.get(), ptr.data(), n * sizeof(uint32_t*), cudaMemcpyHostToDevice));
  if (!modes.empty()) CUDA_TRY(h, cudaMemcpy((void*)dev_modes, modes.data(), modes.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  return W.view_dev.upload(h, W.view.data(), W.view.size() * sizeof(ReplayTraceView));
}

}  // namespace

extern "C" int32_t demi_wildcard_replay_batch_many(demi_handle* h, const uint32_t* trace_of_test, const uint64_t* include_masks,
                                                   uint32_t n_tests, uint32_t mask_words, const uint32_t* looking_for,
                                                   uint32_t flags, demi_replay_result* out) {
  if (!h) return DEMI_ERR_INVALID;
  static const char* who = "demi_wildcard_replay_batch_many";
  if (!trace_of_test || !include_masks || !looking_for || !out) return fail(h, DEMI_ERR_INVALID, "%s: null buffer", who);
  int32_t rc;
  if ((rc = wc_check_flags(h, who, flags)) != DEMI_OK) return rc;
  if (!h->set.n) return fail(h, DEMI_ERR_STATE, "demi_set_traces has not been called");
  std::vector<uint8_t> use(h->set.n, 0);
  for (uint32_t i = 0; i < n_tests; i++) {
    const uint32_t t = trace_of_test[i];
    if (t >= h->set.n) return fail(h, DEMI_ERR_INVALID, "%s: test %u names trace %u of %u", who, i, t, h->set.n);
    use[t] = 1;
  }
  if (n_tests == 0) return DEMI_OK;
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  WildSet W;
  if ((rc = wild_set(h, who, use, W, nullptr, nullptr)) != DEMI_OK) return rc;
  for (uint32_t t = 0; t < h->set.n; t++)
    if (use[t] && mask_words < W.t[t].words)
      return fail(h, DEMI_ERR_INVALID, "%s: mask_words %u too small for the %zu deliveries of trace %u", who, mask_words,
                  W.t[t].pos.size(), t);
  LaunchCounts lc;
  const Wild wild = W.wild();
  rc = replay_many(h, W.views(), trace_of_test, include_masks, nullptr, n_tests, mask_words, looking_for, flags, out, lc,
                   nullptr, &wild);
  set_perf(h, lc);
  return rc;
}

extern "C" int32_t demi_wildcard_minimize_many(demi_handle* h, const uint32_t* looking_for, uint32_t flags,
                                               demi_event* out_traces, uint32_t cap_events,
                                               uint32_t* internal_sizes, uint32_t cap_sizes,
                                               demi_intmin_out* out, int32_t* status) {
  if (!h) return DEMI_ERR_INVALID;
  static const char* who = "demi_wildcard_minimize_many";
  if (!looking_for || !out_traces || !cap_events || !out || !status) return fail(h, DEMI_ERR_INVALID, "%s: null buffer", who);
  int32_t rc;
  if ((rc = wc_check_flags(h, who, flags)) != DEMI_OK) return rc;
  const demi_handle::TraceSet& S = h->set;
  const uint32_t n = S.n;
  if (!n) return fail(h, DEMI_ERR_STATE, "demi_set_traces has not been called");
  uint64_t budget = WC_MANY_ROUND_BYTES;
  if (const char* b = getenv("DEMI_TEST_WC_ROUND_BYTES")) if (*b) budget = strtoull(b, nullptr, 10);
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  memset(out, 0, (size_t)n * sizeof(demi_intmin_out));
  std::vector<std::string> msg(n);
  std::vector<uint8_t> live(n, 1), bad(n, 0);
  WildSet W;
  if ((rc = wild_set(h, who, live, W, &bad, &msg)) != DEMI_OK) return rc;
  auto fail_trace = [&](uint32_t t, int32_t code, const std::string& m) { status[t] = code; msg[t] = m; live[t] = 0; };
  // each trace of the set is the base trace of its driver, which takes over the deliveries and modes wild_set built
  std::vector<WildcardDriver> d(n);
  auto fail_driver = [&](uint32_t t) { fail_trace(t, d[t].error, trace_msg(who, t, d[t].msg)); };
  for (uint32_t t = 0; t < n; t++) {
    status[t] = DEMI_OK;
    if (bad[t]) { fail_trace(t, DEMI_ERR_INVALID, msg[t]); continue; }
    const demi_event* ev = W.all.data() + (S.view[t].events - S.events.get<const uint4>());
    d[t].init(std::move(W.t[t]), ev, S.view[t].n_events, h->clock_rule, h->clock_incr, out + t);
  }
  const Views V = W.views();
  const Wild wild = W.wild();
  LaunchCounts lc;
  rc = DEMI_OK;
  for (;;) {
    // 1. the candidates of unfinished drivers in index order, while their include masks fit the budget (at least one)
    std::vector<uint32_t> adm;
    size_t n_cand = 0; uint32_t mw = 1;
    for (uint32_t t = 0; t < n; t++) {
      if (!live[t]) continue;
      const size_t k = d[t].candidates().empty() ? 0 : d[t].n_candidates();
      if (!k) { live[t] = 0; continue; }
      const uint32_t w = std::max(mw, d[t].t.words);
      if (!adm.empty() && (n_cand + k) * w * sizeof(uint64_t) > budget) break;
      adm.push_back(t); n_cand += k; mw = w;
    }
    if (adm.empty()) break;
    std::vector<uint32_t> tr, first(n, 0);
    std::vector<uint64_t> masks(n_cand * mw, 0);
    for (uint32_t t : adm) {
      const WildcardDriver& x = d[t];
      const uint32_t w = x.t.words;
      first[t] = (uint32_t)tr.size();
      for (size_t c = 0; c < x.n_candidates(); c++)
        std::copy(x.cand.begin() + c * w, x.cand.begin() + (c + 1) * w, masks.begin() + (tr.size() + c) * mw);
      tr.insert(tr.end(), x.n_candidates(), t);
    }
    // 2. their union in one exact launch; 3. each driver commits
    std::vector<demi_replay_result> res(tr.size());
    if ((rc = replay_many(h, V, tr.data(), masks.data(), nullptr, (uint32_t)tr.size(), mw, looking_for, flags, res.data(), lc,
                          nullptr, &wild)) != DEMI_OK)
      break;
    std::vector<uint32_t> rec_tr;
    std::vector<uint64_t> rec_masks;
    for (uint32_t t : adm) {
      const uint64_t* m = nullptr;
      const WildcardDriver::Step step = d[t].commit(res.data() + first[t], &m);
      if (step == WildcardDriver::FAILED) fail_driver(t);
      else if (step == WildcardDriver::RECORD) {
        rec_tr.push_back(t);
        rec_masks.resize(rec_tr.size() * mw, 0);
        std::copy(m, m + d[t].t.words, rec_masks.end() - mw);
      }
    }
    if (rec_tr.empty()) continue;
    // 4. every success re-run in one recording launch; the recording and its ignored deliveries advance its driver
    std::vector<demi_replay_result> rres(rec_tr.size());
    const Recording rec{cap_events, [&](uint32_t i, const demi_event* ev, uint32_t k, const uint32_t* ign, uint32_t ni) {
      const uint32_t t = rec_tr[i];
      if (rres[i].status == DEMI_PS_EVENT_OVF)
        return fail_trace(t, DEMI_ERR_CAPACITY, std::string(who) + ": trace " + std::to_string(t) +
                                                " needs a recording longer than cap_events " + std::to_string(cap_events));
      if (!d[t].advance(rres[i], ev, k, ign, ni)) fail_driver(t);
    }};
    if ((rc = replay_many(h, V, rec_tr.data(), rec_masks.data(), nullptr, (uint32_t)rec_tr.size(), mw, looking_for, flags,
                          rres.data(), lc, &rec, &wild)) != DEMI_OK)
      break;
  }
  set_perf(h, lc);
  if (rc != DEMI_OK) return rc;
  for (uint32_t t = 0; t < n; t++)
    if (status[t] == DEMI_OK)
      d[t].finish(out_traces + (size_t)t * cap_events, cap_events, internal_sizes ? internal_sizes + (size_t)t * cap_sizes : nullptr,
                  cap_sizes);
  for (uint32_t t = 0; t < n; t++)
    if (status[t] != DEMI_OK) { h->err = msg[t]; break; }
  return DEMI_OK;
}
