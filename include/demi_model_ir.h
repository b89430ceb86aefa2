/*
 * demi_model_ir.h — the data-only actor model a host hands to demi_load_model (SURVEY.md §7 build-order 1, §8b).
 *
 * In the reference the transition function is the application's own receive() (Instrumenter.scala:913-1017,
 * WeaveActor.aj:90-108) and the invariant a JVM closure (TestOracle.scala:27).  A host that wants the engine to
 * explore ITS application describes it as data: a register program for receive(), one for the invariant, the
 * initial actor states, the external-message filter (EventTypes.setExternalMessageFilter, ExternalEvents.scala:160-166)
 * and the actor-name table that maps the reference's actor names to the indices the C ABI uses (blockedActors,
 * demi_ext_event.a, demi_event.src/dst).  The engine interprets the programs on the device; the built-in models
 * (DEMI_MODEL_PINGPONG3 ...) remain as compiled fast paths of the same interface.
 *
 * Blob = little-endian u32 words:
 *   [0] magic 'DMIR'  [1] version  [2] n_actors (<= 16)  [3] state_words (<= 8)  [4] n_types
 *   [5] recv_len  [6] inv_len  [7] external_type_mask  [8] max sends of one receive() (<= 16)  [9] names_bytes
 *   [10..15] reserved
 *   recv program (recv_len words), invariant program (inv_len words), initial state (n_actors * state_words words),
 *   names: n_actors + n_types NUL-terminated strings (actor names, then message-type names), padded to 4 bytes.
 * Every loaded model has the same state geometry on the device — 16 actors x 8 words, unused words zero — so one
 * kernel instantiation serves them all.
 *
 * Instruction = op | a << 8 | b << 16 | c << 24 over registers r0..r15 (u32); LDI and the jumps take the next word.
 *   receive():  r0 = self, r1 = sender (0xFF = deadLetters/timer), r2 = type, r3 = p0, r4 = p1, r5 = model_flags
 *   invariant:  r5 = model_flags; DEMI_IR_RET a returns the violation code r[a] and the affected-actor mask r[a+1]
 * A program that runs more than DEMI_IR_MAX_STEPS instructions halts (receive: state as left; invariant: code 0).
 *
 * Rules every engine and the oracle apply identically:
 *  - Non-existent receiver: a SEND whose destination (r[a] & 0xFF) is not below n_actors — including 0xFF, the
 *    "sender" of an external message or a timer — is dropped where it is issued, as the reference drops a message to a
 *    receiver that does not exist (Instrumenter.scala:397-401).  It gets no Uniq, no MsgSend record, no DepTracker node
 *    and does not count against the operation limit.
 *  - Operation limit: one receive() may issue at most DEMI_IR_OUTBOX SEND / SCHED_ONCE / SCHED_REPEAT / CANCEL
 *    operations that reach the scheduler.  One more ends the execution with the queue-overflow status of the engine
 *    that runs it (DEMI_PS_QUEUE_OVF for fuzzing and replay, DEMI_DS_QUEUE_OVF for DPOR); none of that receive()'s
 *    operations is applied.  Header word 8 is only the capacity hint the pending-set size is derived from.
 *  - Timers: SCHED_ONCE / SCHED_REPEAT / CANCEL name a timer by (type, p0, p1) of the actor that issues them; any
 *    values may be used.  Fuzzing, replay, the minimizers and frontier DPOR all run them.  Per execution at most
 *    DEMI_TIMERSET_CAP (16) repeating timers can be registered at a time and at most 16 cancelled timers can be waiting
 *    for their message to be dropped; one more ends the execution with the queue-overflow status, as for the compiled
 *    models.  Scheduling a repeating timer that is already registered does nothing.
 *  - External types: the external-message filter is a 32-bit mask; type t is external iff t < 32 and bit t of the mask
 *    is set (demi_type_is_external, demi_limits.h).  Types 32..255 are always internal.
 */
#ifndef DEMI_MODEL_IR_H
#define DEMI_MODEL_IR_H
#include <stdint.h>

#define DEMI_MODEL_IR 100            /* demi_config.model of a handle that takes demi_load_model */
#define DEMI_IR_MAGIC 0x52494D44u    /* 'DMIR' */
#define DEMI_IR_VERSION 1u
#define DEMI_IR_ACTORS 16
#define DEMI_IR_STATE_WORDS 8
#define DEMI_IR_OUTBOX 16
#define DEMI_IR_HEADER_WORDS 16
#define DEMI_IR_MAX_CODE 4096
#define DEMI_IR_MAX_STEPS 4096

enum {
  DEMI_IR_HALT = 0,
  DEMI_IR_LDI = 1,      /* r[a] = imm                                  */
  DEMI_IR_MOV = 2,      /* r[a] = r[b]                                 */
  DEMI_IR_ADD = 3, DEMI_IR_SUB = 4, DEMI_IR_MUL = 5, DEMI_IR_AND = 6, DEMI_IR_OR = 7, DEMI_IR_XOR = 8,
  DEMI_IR_SHL = 9, DEMI_IR_SHR = 10, DEMI_IR_MOD = 11,                  /* r[a] = r[b] op r[c]; shifts use c & 31; x mod 0 = 0 */
  DEMI_IR_LDW = 12,     /* r[a] = own state word r[b] (0 outside the state)          */
  DEMI_IR_STW = 13,     /* own state word r[a] = r[b]                                */
  DEMI_IR_LDA = 14,     /* r[a] = state word r[c] of actor r[b] (invariant programs) */
  DEMI_IR_JMP = 15,     /* pc = imm                                                  */
  DEMI_IR_JEQ = 16, DEMI_IR_JNE = 17, DEMI_IR_JLT = 18, DEMI_IR_JGE = 19,   /* if (r[a] ? r[b]) pc = imm   (unsigned) */
  DEMI_IR_SEND = 20,    /* `r[a] ! (type r[b], p0 r[c], p1 r[c+1])`                  */
  DEMI_IR_SCHED_ONCE = 21, DEMI_IR_SCHED_REPEAT = 22, DEMI_IR_CANCEL = 23,  /* timer (type r[a], p0 r[b], p1 r[c]) to self */
  DEMI_IR_RET = 24      /* invariant: return r[a] (code), r[a+1] (affected actors)   */
};


/* engine-internal: where a loaded model lives on the device */
typedef struct demi_ir_device {
  const uint32_t* recv; const uint32_t* inv; const uint32_t* init;
  uint32_t recv_len, inv_len, n_actors, state_words;
} demi_ir_device;

#endif
