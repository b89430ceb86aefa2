"""Loaded models (include/demi_model_ir.h) that arm timers, on the CPU: the C oracle against the Python restatement
(tests/micro_oracle.py) on a hand-written timeout-driven leader election and on the timer-set capacity edges, for
STSSched replay (with and without filterKnownAbsents, under ignoreTimers), internal minimization and DPORSearch.
The models and programs here are also what tests/test_ir_timers_gpu.py runs on the engine."""
import numpy as np

import demi_b200 as D
from demi_b200 import model_ir, _native as N
import ir_gen
import micro_oracle as M
from test_micro_oracle import flat, name_idx, to_prog, unflat
from test_model_ir_random import sts_case

PS_QUEUE_OVF, DS_QUEUE_OVF = 2, 2
EV7 = ("kind", "src", "dst", "type", "p0", "p1", "uniq")

# ---------------------------------------------------------------- a timeout-driven leader election
KICK, ELECT, REQ, VOTE, HB, TICK = 1, 2, 3, 4, 5, 6
ELECTION_BUG = 1            # model_flags bit 0: a vote is granted whatever was voted before, so two leaders can share a term
TWO_LEADERS = 9


def election_blob():
    """3 actors, words: term, role (0 follower, 1 candidate, 2 leader), votes, term voted in, heartbeats seen.
    Kick (external) arms the repeating election timer.  ElectionTimeout: a non-leader starts a candidacy for term + 1.
    RequestVote(t) / Vote(t): one vote per term unless ELECTION_BUG; two votes make a leader, who arms the once-timer
    HeartbeatTick(term).  HeartbeatTick: the leader sends Heartbeat(term) and re-arms the tick.  Heartbeat(t >= term):
    step down, cancel the election timer (its pending copy goes) and arm it again."""
    send_others = lambda: [("ADD", "r14", "r0", "r7"), ("MOD", "r14", "r14", "r15"), ("SEND", "r14", "r11", "r12"),
                           ("ADD", "r14", "r0", "r8"), ("MOD", "r14", "r14", "r15"), ("SEND", "r14", "r11", "r12")]
    recv = [("LDI", "r6", 0), ("LDI", "r7", 1), ("LDI", "r8", 2), ("LDI", "r15", 3),
            ("LDW", "r9", "r6"), ("LDW", "r10", "r7")]                                   # r9 = term, r10 = role
    for t, lab in ((KICK, "kick"), (ELECT, "elect"), (REQ, "req"), (VOTE, "vote"), (TICK, "tick"), (HB, "hb")):
        recv += [("LDI", "r11", t), ("JEQ", "r2", "r11", lab)]
    recv += [("HALT",),
             ("label", "kick"), ("LDI", "r11", ELECT), ("SCHED_REPEAT", "r11", "r6", "r6"), ("HALT",),
             ("label", "elect"), ("JEQ", "r10", "r8", "done"),
             ("ADD", "r9", "r9", "r7"), ("STW", "r6", "r9"), ("STW", "r7", "r7"), ("STW", "r8", "r7"), ("STW", "r15", "r9"),
             ("LDI", "r11", REQ), ("MOV", "r12", "r9"), ("LDI", "r13", 0)] + send_others() + [("HALT",),
             ("label", "req"), ("JGE", "r9", "r3", "req_known"),
             ("MOV", "r9", "r3"), ("STW", "r6", "r9"), ("STW", "r7", "r6"),
             ("label", "req_known"), ("JLT", "r3", "r9", "done"),
             ("LDW", "r11", "r15"), ("AND", "r12", "r5", "r7"), ("JNE", "r12", "r6", "grant"), ("JGE", "r11", "r3", "done"),
             ("label", "grant"), ("STW", "r15", "r3"),
             ("LDI", "r11", VOTE), ("MOV", "r12", "r3"), ("LDI", "r13", 0), ("SEND", "r1", "r11", "r12"), ("HALT",),
             ("label", "vote"), ("JNE", "r10", "r7", "done"), ("JNE", "r3", "r9", "done"),
             ("LDW", "r11", "r8"), ("ADD", "r11", "r11", "r7"), ("STW", "r8", "r11"), ("JLT", "r11", "r8", "done"),
             ("STW", "r7", "r8"), ("LDI", "r11", TICK), ("SCHED_ONCE", "r11", "r9", "r6"), ("HALT",),
             ("label", "tick"), ("JNE", "r10", "r8", "done"),
             ("LDI", "r11", HB), ("MOV", "r12", "r9"), ("LDI", "r13", 0)] + send_others() + [
             ("LDI", "r11", TICK), ("SCHED_ONCE", "r11", "r9", "r6"), ("HALT",),
             ("label", "hb"), ("JLT", "r3", "r9", "done"),
             ("MOV", "r9", "r3"), ("STW", "r6", "r9"), ("STW", "r7", "r6"),
             ("LDI", "r11", 4), ("LDW", "r12", "r11"), ("ADD", "r12", "r12", "r7"), ("STW", "r11", "r12"),
             ("LDI", "r11", ELECT), ("CANCEL", "r11", "r6", "r6"), ("SCHED_REPEAT", "r11", "r6", "r6"), ("HALT",),
             ("label", "done"), ("HALT",)]
    inv = [("LDI", "r6", 0), ("LDI", "r7", 1), ("LDI", "r8", 2)]
    for k, (a, b) in enumerate(((0, 1), (0, 2), (1, 2))):
        nxt = "next%d" % k
        inv += [("LDI", "r9", a), ("LDI", "r10", b),
                ("LDA", "r11", "r9", "r7"), ("JNE", "r11", "r8", nxt), ("LDA", "r11", "r10", "r7"), ("JNE", "r11", "r8", nxt),
                ("LDA", "r11", "r9", "r6"), ("LDA", "r12", "r10", "r6"), ("JNE", "r11", "r12", nxt),
                ("LDI", "r0", TWO_LEADERS), ("LDI", "r1", (1 << a) | (1 << b)), ("RET", "r0"), ("label", nxt)]
    inv += [("LDI", "r0", 0), ("LDI", "r1", 0), ("RET", "r0")]
    return model_ir.build_blob(["n0", "n1", "n2"], ["-", "Kick", "ElectionTimeout", "RequestVote", "Vote", "Heartbeat", "HeartbeatTick"],
                               5, recv, inv, external_types=(KICK,), fanout=4)


def election_model():
    return ir_gen.Model(0, election_blob(), 3, 5, 7, [KICK], 4, True, ELECTION_BUG)


def election_program(wait=True):
    prog = [D.Start(a) for a in range(3)] + [D.Send(a, KICK, 0) for a in range(3)]
    return prog + [D.WaitQuiescence()] if wait else prog


ELECTION_MAXM, ELECTION_INTERVAL = 40, 1


def election_violation(oracle, n=400):
    """(ext, seed, events) of the first execution of the buggy election that ends with two leaders in one term."""
    oracle.load_model(election_blob())
    ext = D.pack_externals(election_program())
    res = oracle.fuzz_batch(N.MODEL_IR, ext, 1, n, ELECTION_MAXM, ELECTION_INTERVAL, model_flags=ELECTION_BUG)
    hits = np.nonzero((res["violation"] == TWO_LEADERS) & (res["status"] == 0))[0]
    assert len(hits) > 0
    seed = 1 + int(hits[0])
    ev, par, r = oracle.fuzz_trace(N.MODEL_IR, ext, seed, ELECTION_MAXM, ELECTION_INTERVAL, model_flags=ELECTION_BUG)
    assert int(r["violation"]) == TWO_LEADERS
    return ext, seed, ev


# ---------------------------------------------------------------- the timer-set capacity edges
ARM, TIMER, DISARM, GHOST, ONCE, FIRED = 1, 2, 4, 3, 5, 6
DISTINCT = 1                # model_flags bit 0: the key is p0 itself; without it p0 & 7, so at most 8 keys exist


def edges_blob():
    """1 actor.  Arm(k): SCHED_REPEAT Timer(k').  Disarm(k): CANCEL Ghost(k'), a timer that is never armed, so the key
    stays in the cancelled set.  Once(k): SCHED_ONCE Fired(k), cancelled beforehand when k is odd (its message is then
    dropped when it is produced).  k' = k with DISTINCT, else k & 7.  Every delivery counts in word 0."""
    recv = [("LDI", "r6", 0), ("LDI", "r7", 1), ("LDW", "r8", "r6"), ("ADD", "r8", "r8", "r7"), ("STW", "r6", "r8"),
            ("MOV", "r9", "r3"), ("AND", "r10", "r5", "r7"), ("JNE", "r10", "r6", "keyed"),
            ("LDI", "r10", 7), ("AND", "r9", "r9", "r10"),
            ("label", "keyed"),
            ("LDI", "r11", ARM), ("JEQ", "r2", "r11", "arm"), ("LDI", "r11", DISARM), ("JEQ", "r2", "r11", "disarm"),
            ("LDI", "r11", ONCE), ("JEQ", "r2", "r11", "once"), ("HALT",),
            ("label", "arm"), ("LDI", "r11", TIMER), ("SCHED_REPEAT", "r11", "r9", "r6"), ("HALT",),
            ("label", "disarm"), ("LDI", "r11", GHOST), ("CANCEL", "r11", "r9", "r6"), ("HALT",),
            ("label", "once"), ("LDI", "r11", FIRED), ("AND", "r10", "r3", "r7"), ("JEQ", "r10", "r6", "fire"),
            ("CANCEL", "r11", "r3", "r6"),
            ("label", "fire"), ("SCHED_ONCE", "r11", "r3", "r6"), ("HALT",)]
    inv = [("LDI", "r0", 0), ("RET", "r0")]
    return model_ir.build_blob(["a"], ["-", "Arm", "Timer", "Ghost", "Disarm", "Once", "Fired"], 1, recv, inv,
                               external_types=(ARM, DISARM, ONCE), fanout=4)


def edges_model(flags):
    return ir_gen.Model(0, edges_blob(), 1, 1, 7, [ARM, DISARM, ONCE], 4, True, flags)


def edges_program(kind, ks, wait=True):
    prog = [D.Start(0)] + [D.Send(0, kind, int(k)) for k in ks]
    return prog + [D.WaitQuiescence()] if wait else prog


def edges_recorded(oracle, kind, ks, maxm=60):
    """A trace of the program recorded without DISTINCT (8 keys at most, so no capacity is near): replayed with
    DISTINCT, the same externals register one key each."""
    oracle.load_model(edges_blob())
    ext = D.pack_externals(edges_program(kind, ks))
    ev, par, r = oracle.fuzz_trace(N.MODEL_IR, ext, 1, maxm, 0, model_flags=0)
    assert int(r["status"]) == 0
    return ext, ev


def prefix_masks(oracle, ext, counts):
    """One mask per count c: the Start and the first c Sends."""
    full = np.asarray(oracle.full_mask(ext), dtype=np.uint64).reshape(-1)
    masks = np.zeros((len(counts), len(full)), dtype=np.uint64)
    for j, c in enumerate(counts):
        for i in range(1 + c):
            masks[j, i >> 6] |= np.uint64(1) << np.uint64(i & 63)
    return masks & full[None, :]


# ---------------------------------------------------------------- oracle == restatement
def python_replay(m, ev, ext, mask, fka=False, ignore_timers=False, looking_for=None):
    irm = M.IRModel(m.blob)
    subseq = [i for i in range(len(ext)) if (int(mask[i >> 6]) >> (i & 63)) & 1]
    sts = M.STSReplay(irm.make_actors(m.flags), unflat(ev), to_prog(D.unpack_externals(ext)), irm.invariant(m.flags),
                      irm.is_external, filter_known_absents=fka, looking_for=looking_for, ignore_timers=ignore_timers)
    return sts, (sts.test(subseq) or 0), irm


def test_election_replays_match_the_restatement(oracle):
    """Random external subsequences of violating executions, with and without filterKnownAbsents: verdict, counts and
    the recorded trace; then the same replays under ignoreTimers, where no ElectionTimeout is ever sent."""
    m = election_model()
    ext, seed, ev = election_violation(oracle)
    rng = np.random.default_rng(5)
    checked = sum(sts_case(oracle, m, election_program(), s, ELECTION_MAXM, ELECTION_INTERVAL, rng, 6) for s in (seed, seed + 1, seed + 2))
    assert checked >= 20
    full = np.asarray(oracle.full_mask(ext), dtype=np.uint64).reshape(-1)
    for fka in (0, 1):
        sts, got, irm = python_replay(m, ev, ext, full, bool(fka), ignore_timers=True, looking_for=TWO_LEADERS)
        res, rec = oracle.replay_trace(N.MODEL_IR, ev, ext, full, looking_for=TWO_LEADERS, flags=fka, model_flags=m.flags,
                                       ignore_timers=1)
        assert (got, sts.delivered, sts.ignored) == (int(res["violation"]), int(res["delivered"]), int(res["ignored"]))
        assert [row[:7] for row in flat(sts.events)] == [tuple(int(e[f]) for f in EV7) for e in rec]
        assert int(res["delivered"]) == 3 and int(res["ignored"]) > 0 and irm.stats.get("SCHED_REPEAT", 0) == 3
        on, _ = oracle.replay_trace(N.MODEL_IR, ev, ext, full, looking_for=TWO_LEADERS, flags=fka, model_flags=m.flags)
        assert int(on["violation"]) == TWO_LEADERS and int(on["ignored"]) == 0


def test_election_internal_minimization_matches_the_restatement(oracle):
    m = election_model()
    ext, seed, ev = election_violation(oracle)
    prog = election_program()
    full = np.asarray(oracle.full_mask(ext), dtype=np.uint64).reshape(-1)
    rr, vtrace = oracle.replay_trace(N.MODEL_IR, ev, ext, full, looking_for=TWO_LEADERS, model_flags=m.flags)
    assert int(rr["violation"]) == TWO_LEADERS
    mcs_prog = [prog[k] for k in range(len(ext)) if (int(full[k >> 6]) >> (k & 63)) & 1]
    mcs_ext, mcs_events = D.pack_externals(mcs_prog), to_prog(mcs_prog)
    irm = M.IRModel(m.blob)

    def test(candidate):
        sts = M.STSReplay(irm.make_actors(m.flags), candidate, mcs_events, irm.invariant(m.flags), irm.is_external,
                          looking_for=TWO_LEADERS)
        return sts.events if sts.test(list(range(len(mcs_events)))) == TWO_LEADERS else None
    verified = unflat(vtrace)
    for flags, strategy in ((0, M.LeftToRightOneAtATime), (N.IM_SRC_DST_FIFO, M.SrcDstFIFORemoval)):
        rc, ctrace, total, sizes, unig = oracle.internal_minimize(N.MODEL_IR, vtrace, mcs_ext, TWO_LEADERS, flags=flags,
                                                                  model_flags=m.flags)
        assert rc == 0
        sm = M.STSSchedMinimizer(mcs_events, verified, TWO_LEADERS, strategy(verified, irm.is_external), test)
        final = sm.minimize()
        assert (sm.total_replays, sm.internal_sizes, sm.strategy.unignorable) == (total, [int(x) for x in sizes], unig)
        assert [row[:7] for row in flat(final)] == [tuple(int(e[f]) for f in EV7) for e in ctrace]
        assert len(ctrace) < len(vtrace)


def test_election_dpor_matches_the_restatement(oracle):
    """DPORSearch over the election: the same schedules in the same order, timers and cancels included."""
    m = election_model()
    oracle.load_model(m.blob)
    prog = election_program(wait=False)
    irm = M.IRModel(m.blob)
    for maxm, budget in ((10, 300), (16, 200)):
        rc, r, viol, hashes = oracle.dpor_search(N.MODEL_IR, D.pack_externals(prog), maxm, budget, model_flags=m.flags)
        assert rc == 0 and int(r["status"]) == 0
        s = M.DPORSearch(lambda: irm.make_actors(m.flags), to_prog(prog), irm.invariant(m.flags), maxm, stop_if_found=False)
        s.search(budget)

        def sched_hash(trace):
            h = 0
            for i, u in enumerate(trace):
                if i:
                    snd, rcv, (t, p0, p1) = s.event[u]
                    h = (h + M.hash6(name_idx(snd) | (int(rcv) << 8) | (t << 16), p0, p1, i, 0, 0)) & ((1 << 64) - 1)
            return h
        assert [sched_hash(t) for t in s.traces] == [int(h) for h in hashes]
        assert s.races == int(r["races"]) and len(s.traces) == int(r["interleavings"]) >= 10
    assert irm.stats.get("SCHED_REPEAT", 0) > 0 and irm.stats.get("CANCEL", 0) > 0 and irm.stats.get("SCHED_ONCE", 0) > 0


def test_timer_set_edges_on_the_oracle(oracle):
    """16 registered repeating timers and 16 cancelled keys fit; the 17th ends the replay with DEMI_PS_QUEUE_OVF, and the
    restatement, which has no such limit, agrees on every replay below it.  Registering a key again at a full registry
    is no overflow.  80 distinct once-timers, every second one cancelled first, run through."""
    counts = [0, 1, 8, 15, 16, 17, 20]
    for kind in (ARM, DISARM):
        ext, ev = edges_recorded(oracle, kind, range(20))
        masks = prefix_masks(oracle, ext, counts)
        res = oracle.replay_batch(N.MODEL_IR, ev, ext, masks, model_flags=DISTINCT)
        assert [int(x) for x in res["status"]] == [0, 0, 0, 0, 0, PS_QUEUE_OVF, PS_QUEUE_OVF], kind
        for j, c in enumerate(counts[:5]):
            sts, got, _ = python_replay(edges_model(DISTINCT), ev, ext, masks[j])
            assert (sts.delivered, sts.ignored) == (int(res[j]["delivered"]), int(res[j]["ignored"])) and sts.delivered >= c
    ext, ev = edges_recorded(oracle, ARM, list(range(16)) + [3, 15, 0])
    full = np.asarray(oracle.full_mask(ext), dtype=np.uint64).reshape(-1)
    res, _ = oracle.replay_trace(N.MODEL_IR, ev, ext, full, model_flags=DISTINCT)
    assert int(res["status"]) == 0 and int(res["delivered"]) >= 19
    ext, ev = edges_recorded(oracle, ONCE, range(80), maxm=400)
    full = np.asarray(oracle.full_mask(ext), dtype=np.uint64).reshape(-1)
    res, rec = oracle.replay_trace(N.MODEL_IR, ev, ext, full, model_flags=DISTINCT)
    sts, got, irm = python_replay(edges_model(DISTINCT), ev, ext, full)
    assert int(res["status"]) == 0 and int(res["delivered"]) == sts.delivered == 120       # 80 Once + the 40 even timers
    assert [row[:7] for row in flat(sts.events)] == [tuple(int(e[f]) for f in EV7) for e in rec]
    assert irm.stats["SCHED_ONCE"] == 80 and irm.stats["CANCEL"] == 40
    # K3F's side of the registry and cancelled edges
    for kind in (ARM, DISARM):
        for k, want in ((16, 0), (17, DS_QUEUE_OVF)):
            F = oracle.frontier_params(40, 20, 1)
            rc, fres, _, _ = oracle.dpor_frontier(N.MODEL_IR, D.pack_externals(edges_program(kind, range(k), wait=False)), F, 1,
                                                  model_flags=DISTINCT)
            assert int(fres[0]["status"]) == want, (kind, k)
