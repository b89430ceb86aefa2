// fuzz_kernel.cuh — K1: the persistent random-fuzz kernel.  One warp owns one
// schedule prefix (one RandomScheduler execution) at a time and loops over the
// prefix indices assigned to it; a block is WARPS independent warps.
// PROG (campaigns, demi_fuzz_campaign): prefix idx runs program idx of the arena in `args.prog_*`, with that
// program's capacities; the launch's own ext / n_ext / caps are the campaign's largest and size the scratch.
// PROG + TESTS (random-oracle tests, demi_random_test_batch): prefix idx is execution idx % prog_execs of program
// idx / prog_execs (prog_test_bind), skipped above its program's first hit.  A separate instantiation, so that the
// campaign kernels stay as they were.
// PROG + TESTS + PARAMS (demi_random_test_batch_many): the same, with each program's seed base, max_messages and
// looking_for taken from `args.prog_params` (the programs of one launch belong to different traces).
// PROG + RECORD + PARAMS (demi_fuzz_traces_many): work-list slot idx records one execution of program idx under its own
// seed, max_messages and looking_for (`args.rec_params`) and that program's capacities.  The only recording PROG kernel.
#pragma once
#include "machine.cuh"
#include "models/models.cuh"

namespace demi {

template <class MODEL, int PCAP, int TCAP, bool PEND_GLOBAL, bool RECORD, int WARPS, bool PROG = false, bool TESTS = false,
          bool PARAMS = false>
__global__ void __launch_bounds__(WARPS * 32)
fuzz_kernel(const __grid_constant__ KernelArgs args) {
  static_assert(!(PROG && RECORD) || (PARAMS && !TESTS),
                "a campaign execution is recorded through demi_fuzz_trace on its program, or with its own parameters");
  static_assert(PROG || !TESTS, "random-oracle tests bind their programs as campaigns do");
  static_assert(TESTS || !PARAMS || RECORD, "per-program parameters are those of random-oracle tests or recordings");
  using M = Machine<MODEL, PCAP, TCAP, PEND_GLOBAL, RECORD>;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t gw = (uint64_t)blockIdx.x * WARPS + warp;
  const uint64_t total_warps = (uint64_t)gridDim.x * WARPS;

  M m;
  m.sm = reinterpret_cast<typename M::Smem*>(smem_raw + (size_t)warp * sizeof(typename M::Smem));
  KernelArgs la;
  if constexpr (PROG) { la = args; m.A = &la; } else m.A = &args;
  m.lane = lane;
  m.nodes_g = args.node_scratch + gw * args.node_cap;
  m.pend_g = PEND_GLOBAL ? (args.pend_scratch + gw * (uint64_t)PCAP) : nullptr;
  if (PEND_GLOBAL && args.fifo_scratch) {
    uint16_t* f = args.fifo_scratch + gw * (uint64_t)(M::HALF + 3 * FIFO_PAIRS);
    m.f_next = f; m.f_head = f + M::HALF; m.f_tail = m.f_head + FIFO_PAIRS; m.f_pairs = m.f_tail + FIFO_PAIRS;
  } else {
    m.f_next = m.f_head = m.f_tail = m.f_pairs = nullptr;
  }

  const bool by_pos = RECORD && args.pos_list;      // the slots the lane engine's recording launch deferred
  const uint64_t count = by_pos ? (uint64_t)(*args.pos_count) : args.index_list ? (uint64_t)(*args.index_count) : args.n_prefixes;
  unsigned long long my_steps = 0, my_viol = 0;

  for (uint64_t k = gw; k < count; k += total_warps) {
    const uint64_t it = by_pos ? (uint64_t)args.pos_list[k] : k;
    const uint64_t idx = args.index_list ? (uint64_t)args.index_list[it] : it;
    demi_fuzz_result r;
    if (RECORD) m.rec_ev = args.rec_events + it * (uint64_t)args.rec_cap;
    if constexpr (TESTS) {
      uint64_t prog; int64_t seed;
      if (prog_test_bind<PARAMS>(la, args, idx, false, prog, seed)) {
        m.run(seed, r);
        if (lane == 0) prog_note_hit(args, idx, prog, r);
      } else {
        r = demi_fuzz_result{};
        r.status = PS_SKIPPED;
      }
    } else if constexpr (PROG && RECORD) {
      int64_t seed;
      prog_bind(la, args, idx, false, prog_params_bind(la, args.rec_params[idx], 0, seed));
      m.run(seed, r);
    } else {
      if constexpr (PROG) prog_bind(la, args, idx, false);
      m.run(seed_at(args.seed_base, idx), r);
    }
    const bool retry = args.ovf_list && (r.status == DEMI_PS_PENDING_OVF || r.status == DEMI_PS_NODE_OVF);
    if (retry) {
      if (lane == 0) { uint32_t pos = atomicAdd(args.ovf_count, 1u); args.ovf_list[pos] = (uint32_t)idx; }
    } else {
      if (lane == 0) {
        // recording launches number their outputs by work-list position, batches by prefix index
        uint4* dst = reinterpret_cast<uint4*>(args.results + (RECORD ? it : idx));
        dst[0] = make_uint4(r.violation, r.steps, (uint32_t)r.state_hash, (uint32_t)(r.state_hash >> 32));
        dst[1] = make_uint4((uint32_t)r.trace_hash, (uint32_t)(r.trace_hash >> 32),
                            (uint32_t)r.n_nodes | ((uint32_t)r.n_events << 16),
                            (uint32_t)r.max_pending | ((uint32_t)r.status << 16));
      }
      my_steps += r.steps;
      my_viol += r.violation ? 1u : 0u;
    }
    if (RECORD) {
      // single-prefix launch: export counts and the DepTracker tree (DepTracker.scala:111-116)
      __syncwarp();
      if (lane == 0) {
        uint32_t* c = args.rec_counts + it * 4;
        c[0] = m.n_events; c[1] = m.n_nodes; c[3] = r.violation;
        // ViolationFingerprint.affectedNodes of the violation the execution stopped on
        c[2] = (r.status == 0 && r.violation) ? MODEL::affected(m.sm->states, args.model_flags, r.violation) : 0u;
      }
      if (args.rec_parent)
        for (uint32_t i = lane; i < m.n_nodes && i < args.rec_parent_cap; i += 32)
          args.rec_parent[it * (uint64_t)args.rec_parent_cap + i] = (uint16_t)__ldcg(&m.nodes_g[i]).w;
    }
  }
  if (lane == 0 && args.sum_steps && (my_steps | my_viol)) {
    atomicAdd(args.sum_steps, my_steps);
    atomicAdd(args.n_violations, my_viol);
  }
}

}  // namespace demi
