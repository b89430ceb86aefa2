// actor_step.cuh — the Instrumenter rules of the executors that replay one delivery per thread: K2 (ReplayMachine,
// replay_kernel.cuh), K3 (DporMachine, dpor_kernel.cuh) and K3F (FrExec, frontier_kernel.cuh).
//
// A delivery re-arms a repeating timer, then runs receive() and applies its operations in program order (`!`,
// scheduleOnce and cancel() act synchronously inside receive() in the reference).  Timers are slots in two bitmasks:
// `registry`, the repeating timers, and `cancelled`, the timers whose next produced message is dropped.  A compiled
// model numbers its finite timer universe itself (MODEL::timer_slot); a model that declares DYNAMIC_TIMERS can arm any
// (dst, type, p0, p1), and its slots are indices into a per-execution table of keys (TimerTable below).
//
// The functions here take the machine m, which supplies:
//   Model, BLOCK                         the model and the block size (m's shared-memory stride);
//   smw, A->model_flags, actor(a), status;
//   registry, cancelled                  of type TimerTable<Model>::mask_t;
//   TimerTable<Model>                    as a base, timer_reset() at the start of an execution;
//   UNSUPPORTED, QUEUE_OVF               its status codes for a timer without a slot and for a full queue;
//   event_produced(src, dst, type, p0, p1)   a produced message into its pending structure, after timer_dropped;
//   enqueue_timer(slot)                  what firing a timer means;
//   cancel_pending(self, slot, type, p0, p1) removes a cancelled timer's pending copy.
#pragma once
#include <type_traits>
#include "lane_kernel.cuh"

namespace demi {

// May receive()'s operations be applied as they are issued (no staged outbox)?  Yes unless the model says otherwise
// (`static constexpr bool REPLAY_DIRECT = false`): a built-in model's receive() never exceeds its outbox, so nothing
// observable depends on staging; a loaded IR program can overflow it, and the queue-overflow status is observable.
template <class M, class = void>
struct model_replay_direct { static constexpr bool value = true; };
template <class M>
struct model_replay_direct<M, std::void_t<decltype(M::REPLAY_DIRECT)>> { static constexpr bool value = M::REPLAY_DIRECT; };

// Does the model arm timers with keys that have no compile-time numbering (`static constexpr bool DYNAMIC_TIMERS = true`)?
template <class M, class = void>
struct model_dynamic_timers { static constexpr bool value = false; };
template <class M>
struct model_dynamic_timers<M, std::void_t<decltype(M::DYNAMIC_TIMERS)>> { static constexpr bool value = M::DYNAMIC_TIMERS; };

// The timer slots of one execution: a base of the machine.  Compiled model: nothing to keep (an empty base), 32-bit
// masks over MODEL::timer_slot.
template <class MODEL, bool DYNAMIC = model_dynamic_timers<MODEL>::value>
struct TimerTable {
  using mask_t = uint32_t;
};
// DYNAMIC_TIMERS: a key's index in the table is its slot.  A slot is live while it is in the machine's registry or
// cancelled mask or in `held`; any other slot is free and is reused, so a slot number means nothing outside the
// execution and must never reach a result, a hash, a recorded event or an ordering.  `held` are the slots a machine
// has queued for its next flush (K2's messagesToSend; K3 and K3F send a fired timer at once and hold none):
// timer_queued() adds one, timer_flushed() drops them all when the queue has been emptied.  A copy that cancel() takes
// out of the queue stays held until that flush, which costs nothing but the slot.
// Bound: registry and cancelled hold at most DEMI_TIMERSET_CAP (16) slots each, and between two flushes lies one
// delivery, which queues at most one re-arm and DEMI_IR_OUTBOX (16) scheduled timers: 16 + 16 + 17 = 49 live slots at
// most, so a table of 64 never fills and the capacity that ends an execution is always one of the reference's.
template <class MODEL>
struct TimerTable<MODEL, true> {
  using mask_t = uint64_t;
  static constexpr int SLOTS = 64;
  static_assert(2 * DEMI_TIMERSET_CAP + MODEL::REPLAY_OUTBOX + 1 <= SLOTS, "the table must not be the binding limit");
  uint32_t key_hdr[SLOTS], key_p0[SLOTS], key_p1[SLOTS];                              // hdr = dst | type << 8
  mask_t held;
  // the slot among `among` that holds the key, or -1 (live keys are distinct, so the search order is immaterial)
  __device__ __forceinline__ int slot_find(mask_t among, uint32_t h, uint32_t q0, uint32_t q1) const {
    for (; among; among &= among - 1) {
      const int s = __ffsll((long long)among) - 1;
      if (key_hdr[s] == h && key_p0[s] == q0 && key_p1[s] == q1) return s;
    }
    return -1;
  }
  __device__ __forceinline__ int slot_intern(mask_t live, uint32_t h, uint32_t q0, uint32_t q1) {
    int s = slot_find(live, h, q0, q1);
    if (s >= 0 || !~live) return s;
    s = __ffsll((long long)~live) - 1;
    key_hdr[s] = h; key_p0[s] = q0; key_p1[s] = q1;
    return s;
  }
};

template <class M> using timer_mask_t = typename TimerTable<typename M::Model>::mask_t;
__device__ __forceinline__ int timer_popc(uint32_t x) { return __popc(x); }
__device__ __forceinline__ int timer_popc(uint64_t x) { return __popcll(x); }

template <class M>
__device__ __forceinline__ void timer_reset(M& m) {
  if constexpr (model_dynamic_timers<typename M::Model>::value) m.held = 0;
}
template <class M>
__device__ __forceinline__ void timer_queued(M& m, uint32_t slot) {
  if constexpr (model_dynamic_timers<typename M::Model>::value) m.held |= timer_mask_t<M>(1) << slot;
}
template <class M>
__device__ __forceinline__ void timer_flushed(M& m) {
  if constexpr (model_dynamic_timers<typename M::Model>::value) m.held = 0;
}
// The slot of a timer key in a dynamic table.  CANCELLED: the caller goes on to test the cancelled mask, else the
// registry, and that mask is all there is to search.  (The rules below choose between these and MODEL::timer_slot with
// a constant conditional, not inside a wrapper: a wrapper around timer_slot changes the code ptxas makes for the
// compiled models.)
template <bool CANCELLED, class M>
__device__ __forceinline__ int timer_table_find(M& m, uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) {
  if constexpr (model_dynamic_timers<typename M::Model>::value)
    return m.slot_find(CANCELLED ? m.cancelled : m.registry, dst | (type << 8), p0, p1);
  else return -1;
}
// ... of a key that is about to be armed or cancelled: it is given a slot if it has none
template <class M>
__device__ __forceinline__ int timer_table_intern(M& m, uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) {
  if constexpr (model_dynamic_timers<typename M::Model>::value)
    return m.slot_intern(m.registry | m.cancelled | m.held, dst | (type << 8), p0, p1);
  else return -1;
}
// The message a slot's timer fires
template <class M>
__device__ __forceinline__ void timer_msg(M& m, uint32_t slot, uint32_t& dst, uint32_t& type, uint32_t& p0, uint32_t& p1) {
  if constexpr (model_dynamic_timers<typename M::Model>::value) {
    dst = m.key_hdr[slot] & 0xFFu; type = m.key_hdr[slot] >> 8; p0 = m.key_p0[slot]; p1 = m.key_p1[slot];
  } else M::Model::slot_msg(slot, dst, type, p0, p1);
}

template <class M>
__device__ __forceinline__ void actor_init(M& m) {
  using MODEL = typename M::Model;
  for (uint32_t i = 0; i < MODEL::N_ACTORS * MODEL::STATE_WORDS; i++) m.smw[i * M::BLOCK] = MODEL::init_word(i, m.A->model_flags);
}

// The cancelled-timer drop of Instrumenter.aroundDispatch (Instrumenter.scala:1090-1096): true = dropped
template <class M>
__device__ __forceinline__ bool timer_dropped(M& m, uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) {
  const int slot = model_dynamic_timers<typename M::Model>::value ? timer_table_find<true>(m, dst, type, p0, p1) : M::Model::timer_slot(dst, type, p0, p1);
  if (m.cancelled && slot >= 0 && ((m.cancelled >> slot) & 1u)) { m.cancelled &= ~(timer_mask_t<M>(1) << slot); return true; }
  return false;
}

// scheduler.scheduleOnce / schedule (Instrumenter.scala:1126-1190)
template <class M>
__device__ __forceinline__ void timer_schedule(M& m, uint32_t kind, uint32_t self, uint32_t type, uint32_t p0, uint32_t p1) {
  if (m.status) return;
  const int slot = model_dynamic_timers<typename M::Model>::value ? timer_table_intern(m, self, type, p0, p1) : M::Model::timer_slot(self, type, p0, p1);
  if (slot < 0) { m.status = M::UNSUPPORTED; return; }
  if ((m.registry >> slot) & 1u) return;                                // "Non-unique timer"
  if (kind == OP_SCHED_REPEAT) {
    if (timer_popc(m.registry) >= DEMI_TIMERSET_CAP) { m.status = M::QUEUE_OVF; return; }
    m.registry |= timer_mask_t<M>(1) << slot;
  }
  m.enqueue_timer((uint32_t)slot);
}

// Cancellable.cancel: notify_timer_cancel (STSScheduler.scala:846-868, DPORwHeuristics.scala:961-985)
template <class M>
__device__ __forceinline__ void timer_cancel(M& m, uint32_t self, uint32_t type, uint32_t p0, uint32_t p1) {
  if (m.status) return;
  const int slot = model_dynamic_timers<typename M::Model>::value ? timer_table_intern(m, self, type, p0, p1) : M::Model::timer_slot(self, type, p0, p1);
  if (slot < 0) { m.status = M::UNSUPPORTED; return; }
  const timer_mask_t<M> bit = timer_mask_t<M>(1) << slot;
  if (!(m.cancelled & bit) && timer_popc(m.cancelled) >= DEMI_TIMERSET_CAP) { m.status = M::QUEUE_OVF; return; }
  m.cancelled |= bit;
  m.registry &= ~bit;
  m.cancel_pending(self, (uint32_t)slot, type, p0, p1);
}

// receive()'s view when its operations are applied as they are issued: no staging in shared memory
template <class M>
struct DirectOutbox {
  M* m; uint32_t self;
  __device__ __forceinline__ bool reserve(uint32_t) { return true; }     // each send checks its own capacities
  __device__ __forceinline__ void send(uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) { m->event_produced(self, dst, type, p0, p1); }
  __device__ __forceinline__ void schedule_once(uint32_t type, uint32_t p0, uint32_t p1) { timer_schedule(*m, OP_SCHED_ONCE, self, type, p0, p1); }
  __device__ __forceinline__ void schedule_repeating(uint32_t type, uint32_t p0, uint32_t p1) { timer_schedule(*m, OP_SCHED_REPEAT, self, type, p0, p1); }
  __device__ __forceinline__ void cancel_timer(uint32_t type, uint32_t p0, uint32_t p1) { timer_cancel(*m, self, type, p0, p1); }
};

// Instrumenter.dispatch_new_message begins by re-arming a repeating timer (Instrumenter.scala:1008-1016) ...
template <class M>
__device__ __forceinline__ void timer_rearm(M& m, uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) {
  const int slot = model_dynamic_timers<typename M::Model>::value ? timer_table_find<false>(m, dst, type, p0, p1) : M::Model::timer_slot(dst, type, p0, p1);
  if (slot >= 0 && ((m.registry >> slot) & 1u)) m.enqueue_timer((uint32_t)slot);
}

// ... then runs receive() and applies its operations in program order.  DIRECT: through DirectOutbox; otherwise
// through a LaneOutbox staged in the REPLAY_OUTBOX * 3 shared-memory words that follow the actor states; when it
// overflows, the status is QUEUE_OVF and none of the operations are applied.
template <bool DIRECT, class M>
__device__ __forceinline__ void actor_receive(M& m, uint32_t src, uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) {
  using MODEL = typename M::Model;
  constexpr int BD = M::BLOCK;
  if constexpr (DIRECT) {
    DirectOutbox<M> direct{&m, dst};
    MODEL::receive(direct, dst, m.actor(dst), src, type, p0, p1, m.A->model_flags);
  } else {
    LaneOutbox<MODEL::REPLAY_OUTBOX> ob;
    ob.base = m.smw + MODEL::N_ACTORS * MODEL::STATE_WORDS * BD; ob.bd = BD; ob.n = 0; ob.self = dst; ob.overflow = false;
    MODEL::receive(ob, dst, m.actor(dst), src, type, p0, p1, m.A->model_flags);
    if (ob.overflow) { m.status = M::QUEUE_OVF; return; }
    for (uint32_t i = 0; i < ob.n && !m.status; i++) {
      const uint32_t w0 = ob.base[(i * 3) * BD], q0 = ob.base[(i * 3 + 1) * BD], q1 = ob.base[(i * 3 + 2) * BD];
      const uint32_t kind = w0 & 0xFF, odst = (w0 >> 8) & 0xFF, otype = (w0 >> 16) & 0xFF;
      if (kind == OP_SEND) m.event_produced(dst, odst, otype, q0, q1);
      else if (kind == OP_CANCEL) timer_cancel(m, odst, otype, q0, q1);
      else timer_schedule(m, kind, odst, otype, q0, q1);
    }
  }
}

}  // namespace demi
