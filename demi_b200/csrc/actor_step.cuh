// actor_step.cuh — the Instrumenter rules of the executors that replay one delivery per thread: K2 (ReplayMachine,
// replay_kernel.cuh), K3 (DporMachine, dpor_kernel.cuh) and K3F (FrExec, frontier_kernel.cuh).
//
// A delivery re-arms a repeating timer, then runs receive() and applies its operations in program order (`!`,
// scheduleOnce and cancel() act synchronously inside receive() in the reference).  Timers are slots of the model's
// timer universe (MODEL::timer_slot) in two bitmasks: `registry`, the repeating timers, and `cancelled`, the timers
// whose next produced message is dropped.
//
// The functions here take the machine m, which supplies:
//   Model, BLOCK                         the model and the block size (m's shared-memory stride);
//   smw, A->model_flags, actor(a), registry, cancelled, status;
//   UNSUPPORTED, QUEUE_OVF               its status codes for a timer outside the slot universe and for a full queue;
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

template <class M>
__device__ __forceinline__ void actor_init(M& m) {
  using MODEL = typename M::Model;
  for (uint32_t i = 0; i < MODEL::N_ACTORS * MODEL::STATE_WORDS; i++) m.smw[i * M::BLOCK] = MODEL::init_word(i, m.A->model_flags);
}

// The cancelled-timer drop of Instrumenter.aroundDispatch (Instrumenter.scala:1090-1096): true = dropped
template <class M>
__device__ __forceinline__ bool timer_dropped(M& m, uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) {
  const int slot = M::Model::timer_slot(dst, type, p0, p1);
  if (m.cancelled && slot >= 0 && ((m.cancelled >> slot) & 1u)) { m.cancelled &= ~(1u << slot); return true; }
  return false;
}

// scheduler.scheduleOnce / schedule (Instrumenter.scala:1126-1190)
template <class M>
__device__ __forceinline__ void timer_schedule(M& m, uint32_t kind, uint32_t self, uint32_t type, uint32_t p0, uint32_t p1) {
  if (m.status) return;
  const int slot = M::Model::timer_slot(self, type, p0, p1);
  if (slot < 0) { m.status = M::UNSUPPORTED; return; }
  if ((m.registry >> slot) & 1u) return;                                // "Non-unique timer"
  if (kind == OP_SCHED_REPEAT) {
    if (__popc(m.registry) >= DEMI_TIMERSET_CAP) { m.status = M::QUEUE_OVF; return; }
    m.registry |= 1u << slot;
  }
  m.enqueue_timer((uint32_t)slot);
}

// Cancellable.cancel: notify_timer_cancel (STSScheduler.scala:846-868, DPORwHeuristics.scala:961-985)
template <class M>
__device__ __forceinline__ void timer_cancel(M& m, uint32_t self, uint32_t type, uint32_t p0, uint32_t p1) {
  if (m.status) return;
  const int slot = M::Model::timer_slot(self, type, p0, p1);
  if (slot < 0) { m.status = M::UNSUPPORTED; return; }
  const uint32_t bit = 1u << slot;
  if (!(m.cancelled & bit) && __popc(m.cancelled) >= DEMI_TIMERSET_CAP) { m.status = M::QUEUE_OVF; return; }
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
  const int slot = M::Model::timer_slot(dst, type, p0, p1);
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
