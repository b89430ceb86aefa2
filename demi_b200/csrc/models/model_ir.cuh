// model_ir.cuh — the device interpreter of the model IR (include/demi_model_ir.h): a model the host loaded with
// demi_load_model runs through the same engine interfaces as the compiled models of models.cuh.  receive() and the
// invariant are register programs in global memory (read-only, L1/L2 resident: a few hundred words); every loaded
// model has the state geometry 16 actors x 8 words.  A SEND to an index that is not one of the loaded model's actors is
// dropped here, before any engine sees it; more than DEMI_IR_OUTBOX operations in one receive() set the outbox's
// overflow flag, which every engine reports as its queue-overflow status.  Timers are available through the outbox like in any model.  A
// loaded program can arm any (type, p0, p1), so the model has no compile-time timer numbering: DYNAMIC_TIMERS makes
// replay (K2), DPOR batches and IncrementalDDMin (K3) and frontier DPOR (K3F) intern the keys per execution
// (TimerTable, actor_step.cuh); timer_slot stays −1 for the lane fuzz engine, which hands a loaded model that arms
// timers to the general warp engine.
#pragma once
#include "../machine.cuh"
#include "../../../include/demi_model_ir.h"

namespace demi {

typedef demi_ir_device IrDevice;
// one copy per translation unit; bound by ir_bind() before a launch of that unit's kernels
static __device__ IrDevice g_ir;
// bind the handle's loaded model to this translation unit's kernels (stream-ordered)
static inline cudaError_t ir_bind(const demi_ir_device& d, cudaStream_t s) {
  return cudaMemcpyToSymbolAsync(g_ir, &d, sizeof(d), 0, cudaMemcpyHostToDevice, s);
}

struct IrModel {
  static constexpr int N_ACTORS = DEMI_IR_ACTORS;
  static constexpr int STATE_WORDS = DEMI_IR_STATE_WORDS;
  static constexpr int ID = DEMI_MODEL_IR;
  static constexpr int LANE_OUTBOX = DEMI_IR_OUTBOX;
  static constexpr int REPLAY_OUTBOX = DEMI_IR_OUTBOX;
  static constexpr bool REPLAY_DIRECT = false;    // a loaded program can overflow the outbox: DEMI_PS_QUEUE_OVF is observable
  static constexpr bool DYNAMIC_TIMERS = true;    // a loaded program arms any (type, p0, p1): replay and DPOR intern the keys

  __device__ static __forceinline__ uint32_t init_word(uint32_t i, uint32_t) {
    const uint32_t a = i / STATE_WORDS, w = i % STATE_WORDS;
    return (a < g_ir.n_actors && w < g_ir.state_words) ? __ldg(g_ir.init + a * g_ir.state_words + w) : 0u;
  }

  // OWN(i) -> reference to own state word i; ALL(a, i) -> value of actor a's word i;
  // EMIT(op, dst, type, p0, p1) -> false stops the program (operation limit exceeded)
  template <class OWN, class ALL, class EMIT>
  __device__ static uint32_t run(const uint32_t* code, uint32_t len, uint32_t* r, bool own, bool all, OWN&& own_w, ALL&& all_w,
                                 EMIT&& emit, uint32_t* affected) {
    uint32_t pc = 0;
#pragma unroll 1
    for (uint32_t steps = 0; steps < DEMI_IR_MAX_STEPS && pc < len; steps++) {
      const uint32_t ins = __ldg(code + pc++);
      const uint32_t op = ins & 0xFF, a = (ins >> 8) & 15, b = (ins >> 16) & 15, c = (ins >> 24) & 15;
      uint32_t imm = 0;
      if (op == DEMI_IR_LDI || (op >= DEMI_IR_JMP && op <= DEMI_IR_JGE)) { if (pc >= len) return 0; imm = __ldg(code + pc++); }
      switch (op) {
        case DEMI_IR_HALT: return 0;
        case DEMI_IR_LDI: r[a] = imm; break;
        case DEMI_IR_MOV: r[a] = r[b]; break;
        case DEMI_IR_ADD: r[a] = r[b] + r[c]; break;
        case DEMI_IR_SUB: r[a] = r[b] - r[c]; break;
        case DEMI_IR_MUL: r[a] = r[b] * r[c]; break;
        case DEMI_IR_AND: r[a] = r[b] & r[c]; break;
        case DEMI_IR_OR:  r[a] = r[b] | r[c]; break;
        case DEMI_IR_XOR: r[a] = r[b] ^ r[c]; break;
        case DEMI_IR_SHL: r[a] = r[b] << (r[c] & 31); break;
        case DEMI_IR_SHR: r[a] = r[b] >> (r[c] & 31); break;
        case DEMI_IR_MOD: r[a] = r[c] ? r[b] % r[c] : 0u; break;
        case DEMI_IR_LDW: r[a] = (own && r[b] < (uint32_t)STATE_WORDS) ? own_w(r[b]) : 0u; break;
        case DEMI_IR_STW: if (own && r[a] < (uint32_t)STATE_WORDS) own_w(r[a]) = r[b]; break;
        case DEMI_IR_LDA: r[a] = (all && r[b] < (uint32_t)N_ACTORS && r[c] < (uint32_t)STATE_WORDS) ? all_w(r[b], r[c]) : 0u; break;
        case DEMI_IR_JMP: pc = imm; break;
        case DEMI_IR_JEQ: if (r[a] == r[b]) pc = imm; break;
        case DEMI_IR_JNE: if (r[a] != r[b]) pc = imm; break;
        case DEMI_IR_JLT: if (r[a] < r[b]) pc = imm; break;
        case DEMI_IR_JGE: if (r[a] >= r[b]) pc = imm; break;
        case DEMI_IR_SEND: if (!emit(0u, r[a] & 0xFFu, r[b] & 0xFFu, r[c], r[(c + 1) & 15])) return 0; break;
        case DEMI_IR_SCHED_ONCE: if (!emit(1u, 0u, r[a] & 0xFFu, r[b], r[c])) return 0; break;
        case DEMI_IR_SCHED_REPEAT: if (!emit(2u, 0u, r[a] & 0xFFu, r[b], r[c])) return 0; break;
        case DEMI_IR_CANCEL: if (!emit(3u, 0u, r[a] & 0xFFu, r[b], r[c])) return 0; break;
        case DEMI_IR_RET: if (affected) *affected = r[(a + 1) & 15]; return r[a];
        default: return 0;
      }
    }
    return 0;
  }

  template <class S, class O>
  __device__ static void receive(O& out, uint32_t self, S st, uint32_t src, uint32_t type, uint32_t p0, uint32_t p1, uint32_t flags) {
    uint32_t r[16];
#pragma unroll
    for (int i = 0; i < 16; i++) r[i] = 0;
    r[0] = self; r[1] = src; r[2] = type; r[3] = p0; r[4] = p1; r[5] = flags;
    uint32_t n_ops = 0;
    run(g_ir.recv, g_ir.recv_len, r, true, false,
        [&](uint32_t i) -> uint32_t& { return st.w(i); }, [](uint32_t, uint32_t) { return 0u; },
        [&](uint32_t op, uint32_t dst, uint32_t ty, uint32_t q0, uint32_t q1) -> bool {
          if (op == 0 && dst >= g_ir.n_actors) return true;                  // no such actor: dropped
          if (++n_ops > (uint32_t)DEMI_IR_OUTBOX) { out.overflow = true; return false; }
          if (op == 0) out.send(dst, ty, q0, q1);
          else if (op == 1) out.schedule_once(ty, q0, q1);
          else if (op == 2) out.schedule_repeating(ty, q0, q1);
          else out.cancel_timer(ty, q0, q1);
          return true;
        }, nullptr);
  }
  template <class ALL>
  __device__ static uint32_t run_invariant(ALL&& all_w, uint32_t flags, uint32_t* affected) {
    uint32_t r[16];
#pragma unroll
    for (int i = 0; i < 16; i++) r[i] = 0;
    r[5] = flags;
    uint32_t* scratch = r;                 // never dereferenced: an invariant program has no own state (own = false)
    return run(g_ir.inv, g_ir.inv_len, r, false, true, [scratch](uint32_t) -> uint32_t& { return scratch[0]; }, all_w,
               [](uint32_t, uint32_t, uint32_t, uint32_t, uint32_t) { return true; }, affected);
  }
  template <class A>
  __device__ static uint32_t invariant(A all, uint32_t flags) {
    return run_invariant([&](uint32_t a, uint32_t i) { return all.actor(a).w(i); }, flags, nullptr);
  }
  __device__ static uint32_t invariant_lane(const uint32_t* states, uint32_t flags, uint32_t lane) {
    if (lane != 0) return 0;
    return run_invariant([&](uint32_t a, uint32_t i) { return states[a * STATE_WORDS + i]; }, flags, nullptr);
  }
  __device__ static uint32_t affected(const uint32_t* states, uint32_t flags, uint32_t code) {
    uint32_t aff = 0;
    const uint32_t got = run_invariant([&](uint32_t a, uint32_t i) { return states[a * STATE_WORDS + i]; }, flags, &aff);
    return got == code ? aff : 0u;
  }
  __device__ static __forceinline__ int timer_slot(uint32_t, uint32_t, uint32_t, uint32_t) { return -1; }
  __device__ static __forceinline__ void slot_msg(uint32_t, uint32_t& dst, uint32_t& type, uint32_t& p0, uint32_t& p1) { dst = type = p0 = p1 = 0; }
};

}  // namespace demi
