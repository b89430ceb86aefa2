// replay_trace.hpp — one trace as K2 (replay_kernel.cuh) reads it, shared by the kernels and the handle that keeps it.
#pragma once
#include <stdint.h>
#include <vector_types.h>

namespace demi {

// The ReplayArgs fields that differ from trace to trace (bind_trace).  The capacities are the trace's own, so that every
// test reports the status it would report with that trace alone.
struct ReplayTraceView {
  const uint4* events; const uint16_t* ev_ordinal; const uint4* ext; const uint16_t* send_ext_index;
  uint32_t n_events, n_ext, n_sends, n_uniq_words;
  uint32_t pending_cap, tosend_cap, table_slots, pad;
};

// Match mode of one delivery of a wildcard test's base trace (ClockClusterizer, wildcard_driver.hpp)
enum : uint32_t { WC_EXACT = 0, WC_CLASS = 1, WC_CLOCK = 2 };

}  // namespace demi
