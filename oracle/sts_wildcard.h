/* ORACLE — test infrastructure only (see machine.h header). */
#ifndef ORACLE_STS_WILDCARD_H
#define ORACLE_STS_WILDCARD_H
#include "sts.h"

/* STSScheduler.test of ClockClusterizer's trace (sts_wildcard.c): `include` has one bit per MsgEvent of the trace,
 * `incr` is the 256-bit causesClockIncrement type set. */
void oracle_sts_replay_wild(const demi_config* cfg, const demi_replay_input* in, const uint64_t* include,
                            const uint32_t* incr, uint32_t looking_for, uint32_t flags, demi_replay_result* out,
                            demi_event* rec, uint32_t cap_rec, uint32_t* n_rec,
                            uint32_t* ignored, uint32_t cap_ignored, uint32_t* n_ignored);
#endif
