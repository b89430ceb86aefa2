/*
 * demi_limits.h — capacity rules and hash constants that are part of the
 * engine's observable behaviour (a prefix that overflows a structure reports
 * DEMI_PS_*_OVF instead of a result), so the CUDA engine and the CPU oracle
 * must apply the same numbers.  Interface constants only; no algorithm here.
 */
#ifndef DEMI_LIMITS_H
#define DEMI_LIMITS_H

#include <stdint.h>

/* messagesToSend / timersToResend / justScheduledTimers / timer registry /
 * timersCancelledThisStep capacities (entries). */
#define DEMI_TIMERSET_CAP 16

/* Shared by host and device code (the campaign kernels apply the capacity rules per program). */
#if defined(__CUDACC__)
#define DEMI_HD __host__ __device__ __forceinline__
#else
#define DEMI_HD static inline
#endif

/* Pending-set capacity class for a (model, max_messages) pair: smallest power
 * of two >= the model's worst-case bound, clamped to [64, 8192]. */
DEMI_HD uint32_t demi_pow2_at_least(uint32_t x, uint32_t lo, uint32_t hi) {
  uint32_t c = lo;
  while (c < x && c < hi) c <<= 1;
  return c;
}

/* Worst-case pending bound per model (see DESIGN.md §3 for the derivations):
 *  pingpong3: every external Send may be pending at once  -> n_ext_sends + 8
 *  raft5:     10 timers + net +4 per delivery              -> 16 + 4*(max_messages+1)
 *  bcast32:   net +30 per delivery                         -> 8 + 31*(max_messages+1) */
/* model IR (demi_model_ir.h): the bound comes from the blob's "max sends of one receive()", model = 100 + 256 * fanout */
DEMI_HD uint32_t demi_pending_bound(int model, int32_t max_messages, uint32_t n_ext_sends) {
  uint32_t d = (max_messages < 0) ? 0u : (uint32_t)max_messages;
  if (d > 100000u) d = 100000u;
  if ((model & 0xFF) == 100) return n_ext_sends + 8u + (uint32_t)(model >> 8) * (d + 1u);
  switch (model) {
    case 1: return n_ext_sends + 8u;
    case 2: return n_ext_sends + 16u + 4u * (d + 1u);
    case 3: return n_ext_sends + 8u + 31u * (d + 1u);
    default: return 64u;
  }
}
DEMI_HD uint32_t demi_pending_cap(int model, int32_t max_messages, uint32_t n_ext_sends) {
  return demi_pow2_at_least(demi_pending_bound(model, max_messages, n_ext_sends), 64u, 8192u);
}
/* messagesToSend capacity: externals of one segment + timers. */
DEMI_HD uint32_t demi_tosend_cap(uint32_t n_ext_sends) {
  return demi_pow2_at_least(n_ext_sends + DEMI_TIMERSET_CAP, 32u, 1024u);
}
/* DepTracker node capacity: one node per enabled message + root. u16 ids. */
DEMI_HD uint32_t demi_node_cap(uint32_t pending_cap) {
  uint32_t c = 2u * pending_cap + 64u;
  return c > 65535u ? 65535u : c;
}

/* STSSched replay: at most every recorded send can be pending at once. */
static inline uint32_t demi_replay_pending_cap(uint32_t n_send_events) {
  return demi_pow2_at_least(n_send_events + 8u, 64u, 8192u);
}
/* EventTypes.externalMessageFilter by message type, per built-in model
 * (pingpong3: PING; raft5: BOOT, CLIENT_CMD; bcast32: INJECT). */
static inline uint32_t demi_external_type_mask(int model) {      /* model IR: taken from the blob instead */
  switch (model) { case 1: return 1u << 1; case 2: return (1u << 1) | (1u << 2); case 3: return 1u << 2; default: return 0; }
}

/* ---- hashes ---------------------------------------------------------------
 * Order-sensitive and cheap on a GPU: a 64-bit SUM of per-item terms; each
 * term hashes the item's words together with its sequence number. */

/* EventTypes.isExternal by message type: the filter is a 32-bit mask, so a type >= 32 (possible in a loaded model)
 * is never external; it must not alias onto bit (type & 31). */
DEMI_HD uint32_t demi_type_is_external(uint32_t mask, uint32_t type) {
  return type < 32u && ((mask >> type) & 1u);
}

DEMI_HD uint32_t demi_fmix32(uint32_t h) {
  h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
  return h;
}
/* Multilinear hash of six 32-bit words into 64 bits: six 32x32->64 multiply-adds
 * (IMAD.WIDE on the GPU) and one 64-bit finaliser.  The two halves are exposed:
 * demi_hash6_lin is linear in each word mod 2^64, so a caller that hashes a run of
 * items whose words differ by known amounts may advance the linear part by
 * DEMI_HASH6_K* times the differences and apply demi_hash6_fin per item. */
#define DEMI_HASH6_KA 0x9E3779B1u
#define DEMI_HASH6_KB 0x85EBCA77u
#define DEMI_HASH6_KC 0xC2B2AE3Du
#define DEMI_HASH6_KD 0x27D4EB2Fu
#define DEMI_HASH6_KE 0x165667B1u
#define DEMI_HASH6_KF 0xD3A2646Du
DEMI_HD uint64_t demi_hash6_lin(uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t e, uint32_t f) {
  return (uint64_t)a * DEMI_HASH6_KA + (uint64_t)b * DEMI_HASH6_KB + (uint64_t)c * DEMI_HASH6_KC +
         (uint64_t)d * DEMI_HASH6_KD + (uint64_t)e * DEMI_HASH6_KE + (uint64_t)f * DEMI_HASH6_KF +
         0x6A09E667BB67AE85ull;
}
DEMI_HD uint64_t demi_hash6_fin(uint64_t acc) {
  acc ^= acc >> 32;
  acc *= 0x9E3779B97F4A7C15ull;
  acc ^= acc >> 29;
  return acc;
}
DEMI_HD uint64_t demi_hash6(uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t e, uint32_t f) {
  return demi_hash6_fin(demi_hash6_lin(a, b, c, d, e, f));
}
/* One EventTrace element: words as laid out in demi_event (w0 = kind | src<<8 |
 * dst<<16 | type<<24, w3 = uniq | node<<16), seq = position in the trace,
 * parent = DepTracker parent of `node` for sends (else 0). */
DEMI_HD uint64_t demi_event_term(uint32_t w0, uint32_t p0, uint32_t p1, uint32_t w3,
                                 uint32_t seq, uint32_t parent) {
  return demi_hash6(w0, p0, p1, w3, seq, parent);
}
/* One 32-bit word of actor state at word index i. */
DEMI_HD uint64_t demi_state_term(uint32_t word, uint32_t i) {
  return demi_hash6(word, i, 0x5D, 0, 0, 0);
}

/* One pending message (sender, receiver, type | payload); summed, so order-free. */
DEMI_HD uint64_t demi_pending_term(uint32_t hdr_noflags, uint32_t p0, uint32_t p1) {
  return demi_hash6(hdr_noflags, p0, p1, 0x50454E44u, 0, 0);
}

/* ---- frontier DPOR (demi_dpor_frontier): content-addressed dependency-graph ids, explored-pair keys and the
 * queue order of a backtrack point are part of the observable behaviour, so engine and oracle share them. */
#define DEMI_FR_ROOT_ID 0x9E3779B97F4A7C15ull
/* id of the message (snd, rcv, fingerprint) created while `parent` is being delivered: the child-reuse rule of
 * DPORwHeuristics.getMessage (:773-801) as a hash.  hdr = src | dst << 8 | type << 16. */
DEMI_HD uint64_t demi_fr_child_id(uint64_t parent, uint32_t hdr, uint32_t p0, uint32_t p1) {
  return demi_hash6((uint32_t)parent, (uint32_t)(parent >> 32), hdr, p0, p1, 0x46524944u);
}
/* ordered pair (first, second) of node ids -> explored-set key (0 is the empty slot) */
DEMI_HD uint64_t demi_fr_pair_key(uint64_t first, uint64_t second) {
  uint64_t k = demi_hash6((uint32_t)first, (uint32_t)(first >> 32), (uint32_t)second, (uint32_t)(second >> 32), 0x50414952u, 0);
  return k ? k : 1ull;
}
/* queue order: ascending `ord` = deeper branch first, then trace slot, later position, earlier position */
#define DEMI_FR_MAX_POS 4095u
DEMI_HD uint64_t demi_fr_ord(uint32_t branch, uint32_t slot, uint32_t li, uint32_t ei) {
  return ((uint64_t)(DEMI_FR_MAX_POS - branch) << 52) | ((uint64_t)slot << 24) | ((uint64_t)li << 12) | (uint64_t)ei;
}
DEMI_HD uint32_t demi_fr_ord_branch(uint64_t o) { return DEMI_FR_MAX_POS - (uint32_t)(o >> 52); }
DEMI_HD uint32_t demi_fr_ord_slot(uint64_t o) { return (uint32_t)(o >> 24) & 0x0FFFFFFFu; }
DEMI_HD uint32_t demi_fr_ord_later(uint64_t o) { return (uint32_t)(o >> 12) & 0xFFFu; }
DEMI_HD uint32_t demi_fr_ord_earlier(uint64_t o) { return (uint32_t)o & 0xFFFu; }
DEMI_HD uint64_t demi_fr_explored_slot(uint64_t key, uint64_t slots) {
  return ((key * 0x9E3779B97F4A7C15ull) >> 20) & (slots - 1);
}
/* executor capacities per interleaving: messages created (pool entries never outlive the execution) */
static inline uint32_t demi_fr_pool_entries(int model, int32_t max_messages, uint32_t n_ext_sends) {
  uint32_t d = (uint32_t)max_messages + 1u;
  if ((model & 0xFF) == 100) return n_ext_sends + 8u + ((uint32_t)(model >> 8) + 1u) * d;     /* loaded model: fan-out in the key */
  switch (model) {
    case 1: return n_ext_sends + 2u * d + 8u;
    case 2: return n_ext_sends + 16u + 7u * d;     /* <= 6 outbox ops + one re-arm per delivery */
    case 3: return n_ext_sends + 8u + 32u * d;
    default: return 64u;
  }
}

/* ---- wildcard replay (demi_wildcard_replay_*): a wildcard delivery may deliver another message than the trace
 * did, so the base trace's own sends no longer bound the pending set.  Bound: what an execution of at most
 * n_deliveries deliveries can create (the executor rule above), clamped like the other pending capacities.  A test
 * whose pending set would exceed it reports DEMI_PS_PENDING_OVF, in the engine and in the oracle alike. */
static inline uint32_t demi_wildcard_pending_cap(int model, uint32_t n_deliveries, uint32_t n_ext_sends) {
  return demi_pow2_at_least(demi_fr_pool_entries(model, (int32_t)n_deliveries, n_ext_sends), 64u, 8192u);
}

#endif /* DEMI_LIMITS_H */
