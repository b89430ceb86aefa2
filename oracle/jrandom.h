/*
 * ORACLE — test infrastructure only.  Never linked into the product path.
 *
 * java.util.Random restated from the Java SE specification (the JDK is a
 * third-party dependency of the reference and is not under /root/reference).
 * Reference call sites: RandomizedHashSet seeds `new Random(seed)` at
 * src/main/scala/verification/schedulers/Util.scala:115 and draws with
 * `rand.nextInt(arr.length)` at Util.scala:172 and :181.
 */
#ifndef ORACLE_JRANDOM_H
#define ORACLE_JRANDOM_H
#include <stdint.h>

typedef struct { uint64_t s; } jrandom;

/* Redraws of nextInt(bound)'s rejection loop since the last oracle_jrandom_reset_rejections(), over every generator
 * and thread of the library (fuzz.c).  Tests read it to show that a crafted seed took the loop.  It is counted on the
 * loop's body only, which runs about once in 10^9 draws at this project's bounds. */
extern uint64_t oracle_jr_rejections;

/* The seed of execution `off` of a batch at `base`.  Java's long addition wraps, and only the low 48 bits reach the
 * generator, so the sum is taken in uint64_t: int64_t addition would be undefined past INT64_MAX. */
static inline int64_t jr_seed_at(int64_t base, uint64_t off) { return (int64_t)((uint64_t)base + off); }

#define JR_MULT 0x5DEECE66DULL
#define JR_ADD  0xBULL
#define JR_MASK ((1ULL << 48) - 1)

static inline void jr_seed(jrandom* r, int64_t seed) {
  r->s = ((uint64_t)seed ^ JR_MULT) & JR_MASK;
}
/* protected int next(int bits) */
static inline int32_t jr_next(jrandom* r, int bits) {
  r->s = (r->s * JR_MULT + JR_ADD) & JR_MASK;
  return (int32_t)(int64_t)(r->s >> (48 - bits));
}
static inline int32_t jr_next_int(jrandom* r) { return jr_next(r, 32); }
/* public int nextInt(int bound), bound > 0 */
static inline int32_t jr_next_int_bound(jrandom* r, int32_t bound) {
  int32_t v = jr_next(r, 31);
  int32_t m = bound - 1;
  if ((bound & m) == 0) {
    return (int32_t)(((int64_t)bound * (int64_t)v) >> 31);
  }
  int32_t u = v;
  /* (u - (v = u % bound) + m) overflows to negative => reject */
  while ((int32_t)((uint32_t)u - (uint32_t)(v = u % bound) + (uint32_t)m) < 0) {
    __atomic_fetch_add(&oracle_jr_rejections, 1, __ATOMIC_RELAXED);
    u = jr_next(r, 31);
  }
  return v;
}
#endif
