// capi_intmin.cu — internal-event minimization: STSSchedMinimizer
// (minification/internal_minimization/ScheduleCheckers.scala:19-107) with the
// LeftToRightOneAtATime (OneAtATimeRemoval.scala:17-137) or SrcDstFIFORemoval (:139-251) removal strategy.
//
// IntMinDriver (intmin_driver.hpp) makes the decisions; here they are served on the handle's single trace: the
// whole remaining candidate list of the current base trace is evaluated in one K2 launch (demi_replay_batch_ex with
// skip_events), the first success is re-run in recording mode (demi_replay_trace), and the recorded trace becomes
// the handle's trace.  Decisions, counters and the final trace are the sequential ones.
#include "engine.hpp"
#include "intmin_driver.hpp"

extern "C" int32_t demi_internal_minimize(demi_handle* h, uint32_t looking_for, uint32_t flags,
                                          demi_event* out_trace, uint32_t cap_events,
                                          uint32_t* internal_sizes, uint32_t cap_sizes, demi_intmin_out* out) {
  if (!h) return DEMI_ERR_INVALID;
  if (!out) return fail(h, DEMI_ERR_INVALID, "demi_internal_minimize: null output");
  if (h->trace_host.empty()) return fail(h, DEMI_ERR_STATE, "demi_set_trace has not been called");
  const bool use_fifo = (flags & DEMI_IM_SRC_DST_FIFO) != 0;
  flags &= ~DEMI_IM_SRC_DST_FIFO;
  const std::vector<demi_ext_event> ext = h->trace_ext_host;
  const uint32_t mw = std::max<uint32_t>(1, ((uint32_t)ext.size() + 63) / 64);
  demi::IntMinDriver d;
  d.init(h->trace_host.data(), (uint32_t)h->trace_host.size(), demi_ext_type_mask(h), use_fifo, out);
  std::vector<demi_event> rec(65536);
  for (;;) {
    const std::vector<uint32_t>& cand = d.candidates();
    if (cand.empty()) break;
    std::vector<demi_replay_result> res(cand.size());
    int32_t rc = demi_replay_batch_ex(h, nullptr, cand.data(), (uint32_t)cand.size(), mw, looking_for, flags, res.data());
    if (rc != DEMI_OK) return rc;
    uint32_t skip = 0;
    const demi::IntMinDriver::Step step = d.commit(res.data(), &skip);
    if (step == demi::IntMinDriver::FAILED) return fail(h, d.error, "%s", d.msg.c_str());
    if (step == demi::IntMinDriver::DONE) break;
    uint32_t n_rec = 0; demi_replay_result r1;
    rc = demi_replay_trace(h, nullptr, mw, skip, looking_for, flags, rec.data(), (uint32_t)rec.size(), &n_rec, &r1);
    if (rc != DEMI_OK) return rc;
    if (!d.advance(r1, rec.data(), n_rec)) return fail(h, d.error, "%s", d.msg.c_str());
    rc = demi_set_trace(h, d.cur.data(), (uint32_t)d.cur.size(), ext.data(), (uint32_t)ext.size());
    if (rc != DEMI_OK) return rc;
  }
  d.finish(out_trace, cap_events, internal_sizes, cap_sizes);
  return DEMI_OK;
}
