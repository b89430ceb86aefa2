"""Fungible clocks, known answers derived by hand from the Scala (wildcard_minimization/ClockClusterizer.scala,
AmbiguityResolutionStrategies.scala, schedulers/STSScheduler.scala): the include sets ClockClusterizer issues for a
fixed success pattern, and single wildcard replays, checked on the C oracle and on the Python restatement."""
import numpy as np

import demi_b200 as D
from demi_b200 import _native as N
from oracle import wildcard_binding as W
import micro_oracle as M
import micro_oracle_wildcard as MW
from test_micro_oracle import flat, to_prog

EV_DTYPE = N.EVENT_DTYPE

# ---- ClockClusterizer on a synthetic trace: eight deliveries d0..d7 (raft5's rules: the term is p0 & 0xFF of types
# 4, 5, 7, 8; type 3 increments the clock; type 6 has no clock)
#        d0    d1    d2    d3    d4    d5    d6    d7
IDS = [10, 5, 7, 12, 3, 8, 20, 15]
TYPES = [3, 4, 3, 5, 7, 6, 3, 8]
CLOCKS = [0, 1, 0, 1, 2, 0, 0, 3]
# timers (type 3): ids 10, 7, 20 -> tried in Uniq order 7, 10, 20 (toRemove = all.toSeq.sorted, :249), i.e. d2, d0, d6
# clocked ids: 5, 12 (clock 1), 3 (clock 2), 15 (clock 3); clocks = [1, 2, 3]
ALL_FAIL = [0xFF, 0xFB, 0xFE, 0xBF,      # first cluster: everything, then without timer 7 (d2), 10 (d0), 20 (d6)
            0xF5, 0xF1, 0xF4, 0xB5,      # clock 1 removed (d1, d3), then the same three timers
            0xEF, 0xEB, 0xEE, 0xAF,      # clock 2 (d4)
            0x7F, 0x7B, 0x7E, 0x3F]      # clock 3 (d7); then None


def synthetic_c():
    ev = np.zeros(len(IDS), dtype=EV_DTYPE)
    for j, (u, t, c) in enumerate(zip(IDS, TYPES, CLOCKS)):
        ev[j] = (N.EV_MSG_EVENT, 0, 1, t, c, 0, u, 0)
    return ev


def synthetic_py():
    return [("MsgEvent", "0", "1", (t, c, 0), u, 0) for u, t, c in zip(IDS, TYPES, CLOCKS)]


def py_sequence(outcomes, ignored=()):
    """Drive the Python ClockClusterizer: test k reports outcomes[k] (ignoredAbsentIds ignored[k]); later tests fail."""
    fp = MW.FingerprintFactory(getLogicalClock=lambda m: (m[1] & 0xFF) if m[0] in (4, 5, 7, 8) else None,
                              causesClockIncrement=lambda m: m[0] == 3)
    cz = MW.ClockClusterizer(synthetic_py(), fp, MW.BackTrackStrategy(), lambda m: False)
    masks, k, v, ign = [], 0, False, set()
    while True:
        nxt = cz.getNextTrace(v, ign)
        if nxt is None:
            return masks
        kept = set(e[4] for e in nxt if e[0] == "MsgEvent")
        masks.append(sum(1 << j for j, u in enumerate(IDS) if u in kept))
        v = bool(outcomes[k]) if k < len(outcomes) else False
        ign = set(ignored[k]) if k < len(ignored) else set()
        k += 1


def both(oracle, outcomes, ignored=()):
    py = py_sequence(outcomes, ignored)
    c = [int(m[0]) for m in W.wildcard_cluster_sequence(synthetic_c(), *D.raft5_clock_rules(), outcomes, ignored)]
    assert py == c
    return py


def test_every_test_fails(oracle):
    """The first cluster includes everything; timers are removed one at a time in Uniq order; then each clock."""
    assert both(oracle, []) == ALL_FAIL


def test_success_in_the_first_cluster_blacklists_the_timer(oracle):
    """Removing timer 7 (d2) works: it stays removed while the remaining timers are tried (:279-282)."""
    got = both(oracle, [0, 1])
    assert got[:5] == [0xFF, 0xFB, 0xFA, 0xBB, 0xF1]
    # the next clusters only try the timers that are left: 10 and 20
    assert got[5:8] == [0xF0, 0xB1, 0xEB]


def test_success_outside_the_first_cluster_moves_to_the_next_clock(oracle):
    """ALL_TIMERS_FIRST_ITR: a success in a later cluster skips that cluster's remaining timers (:80-94), and the
    clock-1 ids that were left out stay out."""
    got = both(oracle, [0, 0, 0, 0, 1])
    assert got[:7] == [0xFF, 0xFB, 0xFE, 0xBF, 0xF5, 0xE5, 0xE1]


def test_ignored_absents_are_blacklisted(oracle):
    """A success whose replay ignored timer 20 blacklists it with the timer whose removal succeeded (:279-282)."""
    got = both(oracle, [0, 1], [[], [20]])
    assert got[:4] == [0xFF, 0xFB, 0xBA, 0xBB]


def test_empty_clock_list_restarts_from_the_lowest_clock(oracle):
    """computeRemainingClocks after the last clock was taken: clocks.headOption.getOrElse(0) is 0, so every clock
    that is not blacklisted comes back, the already-tried ones included (:162-173).  Here the clock-3 cluster
    succeeds ignoring id 5: the blacklist is {15, 5} and the clusters restart at clock 1."""
    outcomes = [0] * 12 + [1]
    ignored = [[]] * 12 + [[5]]
    got = both(oracle, outcomes, ignored)
    assert got[:12] == ALL_FAIL[:12] and got[12] == 0x7F
    assert got[13:17] == [0x75, 0x71, 0x74, 0x35]      # clock 1 again, without 5, 12 and 15
    assert got[17] == 0x6D                              # then clock 2 (id 3): 12 is back in
    assert len(got) == 21


# ---- single wildcard replays on pingpong3: three PINGs to actor 0 (payloads 5, 6, 5) make it send PONG(5), PONG(6),
# PONG(5) to actor 1 (Uniq 4, 5, 6); the trace's last delivery is the first PONG, d3.
def pingpong_case():
    prog = [D.Start(0), D.Start(1), D.Start(2), D.Send(0, 1, 5, 0), D.Send(0, 1, 6, 0), D.Send(0, 1, 5, 0)]
    ext = D.pack_externals(prog)
    rows = [(3, 0xFF, 0, 0, 0, 0, 0), (3, 0xFF, 1, 0, 0, 0, 0), (3, 0xFF, 2, 0, 0, 0, 0),
            (1, 0xFF, 0, 1, 5, 0, 1), (1, 0xFF, 0, 1, 6, 0, 2), (1, 0xFF, 0, 1, 5, 0, 3),
            (2, 0xFF, 0, 1, 5, 0, 1), (1, 0, 1, 2, 5, 0, 4),
            (2, 0xFF, 0, 1, 6, 0, 2), (1, 0, 1, 2, 6, 0, 5),
            (2, 0xFF, 0, 1, 5, 0, 3), (1, 0, 1, 2, 5, 0, 6),
            (2, 0, 1, 2, 5, 0, 4)]
    ev = np.array([r + (0,) for r in rows], dtype=EV_DTYPE)
    return prog, ext, ev


def delivered_last(rec):
    d = [e for e in rec if int(e["kind"]) == N.EV_MSG_EVENT]
    return (int(d[-1]["type"]), int(d[-1]["p0"]), int(d[-1]["uniq"]))


def test_the_trace_is_an_exact_replay(oracle):
    prog, ext, ev = pingpong_case()
    res, rec = oracle.replay_trace(N.MODEL_PINGPONG3, ev, ext, oracle.full_mask(ext))
    assert int(res["ignored"]) == 0 and int(res["delivered"]) == 4
    assert [tuple(int(e[f]) for f in ("kind", "src", "dst", "type", "p0", "p1", "uniq")) for e in rec] == \
        [tuple(int(e[f]) for f in ("kind", "src", "dst", "type", "p0", "p1", "uniq")) for e in ev]


def _python(prog, ev, strategy, incr=()):
    fp = MW.FingerprintFactory(causesClockIncrement=lambda m: m[0] in incr)
    base = [("MsgEvent" if int(e["kind"]) == 2 else "MsgSend" if int(e["kind"]) == 1 else "Spawn",) +
            ((M.DEADLETTERS if int(e["src"]) == 0xFF else str(int(e["src"])), str(int(e["dst"])),
              (int(e["type"]), int(e["p0"]), int(e["p1"])), int(e["uniq"]), 0) if int(e["kind"]) in (1, 2)
             else (str(int(e["dst"])),)) for e in ev]
    cz = MW.ClockClusterizer(base, fp, strategy, lambda m: m[0] == 1)
    ids = set(int(e["uniq"]) for e in ev if int(e["kind"]) == 2)
    timers = set(e[4] for e in base if e[0] == "MsgEvent" and fp.causesClockIncrement(e[3]))
    nxt = cz.wildcarded(timers, ids - timers)
    sts = MW.WildcardSTSReplay({str(i): M.PingPongActor(i) for i in range(3)}, nxt, to_prog(prog), M.pingpong_invariant(0),
                              lambda m: m[0] == 1)
    sts.test(list(range(len(prog))))
    return [r for r in flat(sts.events) if r[0] == 2][-1][3:7:1]


def test_first_and_last_resolution_choose_different_messages(oracle):
    """Queues of (0, 1) by head Uniq: PONG(5) [4, 6], PONG(6) [5].  BackTrackStrategy delivers the first matching head,
    Uniq 4; LastOnlyStrategy the last matching head, Uniq 5 — not the newest matching message, Uniq 6."""
    prog, ext, ev = pingpong_case()
    full = np.array([0xF], dtype=np.uint64)
    r0, rec0, ign0 = W.wildcard_replay(N.MODEL_PINGPONG3, ev, ext, full, ())
    r1, rec1, ign1 = W.wildcard_replay(N.MODEL_PINGPONG3, ev, ext, full, (), flags=N.WC_LAST_ONLY)
    assert delivered_last(rec0) == (2, 5, 4)
    assert delivered_last(rec1) == (2, 6, 5)
    assert int(r0["ignored"]) == int(r1["ignored"]) == 0 and len(ign0) == len(ign1) == 0
    assert int(r0["state_hash"]) != int(r1["state_hash"])
    assert _python(prog, ev, MW.BackTrackStrategy()) == (2, 5, 0, 4)
    assert _python(prog, ev, MW.LastOnlyStrategy()) == (2, 6, 0, 5)


def test_the_clock_increment_selector_wins_over_the_resolution(oracle):
    """With PONG marked clock-incrementing, d3 is the CausesClockIncrement wildcard: the first incrementing head, Uniq 4,
    whatever the resolution strategy (ClockClusterizer.scala:107-112)."""
    prog, ext, ev = pingpong_case()
    full = np.array([0xF], dtype=np.uint64)
    _, rec, _ = W.wildcard_replay(N.MODEL_PINGPONG3, ev, ext, full, (2,), flags=N.WC_LAST_ONLY)
    assert delivered_last(rec) == (2, 5, 4)
    assert _python(prog, ev, MW.LastOnlyStrategy(), incr=(2,)) == (2, 5, 0, 4)


def test_a_blocked_receiver_makes_the_wildcard_absent(oracle):
    """messagePending is false while the receiver is blocked: the delivery is ignored and reported at its trace
    position (the ignoreAbsentCallback of STSScheduler.scala:529)."""
    prog, ext, ev = pingpong_case()
    full = np.array([0xF], dtype=np.uint64)
    r, rec, ign = W.wildcard_replay(N.MODEL_PINGPONG3, ev, ext, full, (), blocked_mask=1 << 1)
    assert int(r["ignored"]) == 1 and int(r["delivered"]) == 3 and list(ign) == [12]


def test_a_cleared_bit_leaves_the_delivery_out_and_external_ones_stay_exact(oracle):
    prog, ext, ev = pingpong_case()
    r, rec, ign = W.wildcard_replay(N.MODEL_PINGPONG3, ev, ext, np.array([0], dtype=np.uint64), ())
    assert int(r["delivered"]) == 3 and int(r["ignored"]) == 0 and len(ign) == 0
    assert [int(e["type"]) for e in rec if int(e["kind"]) == N.EV_MSG_EVENT] == [1, 1, 1]
