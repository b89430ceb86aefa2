"""SchedulerConfig's two execution switches, blockedActors (a static mask, DESIGN.md §8) and ignoreTimers, checked on the
C oracle's DPOR and STSSched paths against the independent Python restatement (tests/micro_oracle.py).

The reference reads ignoreTimers in one place, ExternalEventInjector.handle_timer (ExternalEventInjector.scala:283-285).
RandomScheduler and STSScheduler route their timers through it; DPORwHeuristics does not: its enqueue_timer is
Scheduler's default enqueue_message (Scheduler.scala:73), an immediate `!` (DPORwHeuristics.scala:946-955) that
Instrumenter.handleTick (Instrumenter.scala:1185-1196) sends whatever the flag says.  So a DPOR search with ignoreTimers
set must equal the same search without it."""
import numpy as np

import demi_b200 as D
from demi_b200 import _native as N
import micro_oracle as M
from test_dpor_gpu import raft_programs
from test_micro_oracle import flat, name_idx, to_prog

PP_FLAGS = 1 | (2 << 8)          # PingPong3: violation 7 once actor 0 has received 2 pongs
RAFT_TIMER_TYPES = (M.ELECTION_TICK, M.HEARTBEAT_TICK)
EV_FIELDS = ("kind", "src", "dst", "type", "p0", "p1", "uniq")


def model_parts(model, flags):
    if model == N.MODEL_RAFT5:
        return (lambda: {str(i): M.RaftActor(i, flags) for i in range(5)}), M.raft_invariant, (lambda m: m[0] in (1, 2))
    return (lambda: {str(i): M.PingPongActor(i) for i in range(3)}), M.pingpong_invariant(flags), (lambda m: m[0] == 1)


def bits_of(actors):
    return sum(1 << a for a in actors)


# ------------------------------------------------------------------------------------------------------------ DPOR
class _TimersDropped(M.DPORSearch):
    """What a DPOR that obeyed ignoreTimers would do: a scheduled timer is registered but never sent."""

    def handleTick(self, rcv, msg):
        if not self.timerToCancellable[(rcv, msg)]:
            del self.timerToCancellable[(rcv, msg)]


def python_dpor(model, prog, flags, maxm, budget, blocked=(), stop=False, cls=M.DPORSearch):
    make, inv, _ = model_parts(model, flags)
    s = cls(make, to_prog(prog), inv, maxm, stop_if_found=stop, blocked=[str(b) for b in blocked])
    exhausted = s.search(budget)

    def sched_hash(trace):
        h = 0
        for i, u in enumerate(trace):
            if i == 0:
                continue
            snd, rcv, (t, p0, p1) = s.event[u]
            h = (h + M.hash6(name_idx(snd) | (int(rcv) << 8) | (t << 16), p0, p1, i, 0, 0)) & ((1 << 64) - 1)
        return h
    return s, exhausted, [sched_hash(t) for t in s.traces]


def dpor_case(oracle, model, prog, flags, maxm, budget, blocked=(), ignore_timers=0, stop=False):
    """The C oracle's search under (blocked, ignore_timers) against the restatement under `blocked`: the same schedules
    in the same order, counters and violations.  Returns the C oracle's (result, schedule hashes)."""
    rc, r, viol, hashes = oracle.dpor_search(model, D.pack_externals(prog), maxm, budget, stop_if_found=1 if stop else 0,
                                             model_flags=flags, blocked_mask=bits_of(blocked), ignore_timers=ignore_timers)
    assert rc == 0 and int(r["status"]) == 0
    s, exhausted, py_hashes = python_dpor(model, prog, flags, maxm, budget, blocked, stop)
    assert len(s.traces) == int(r["interleavings"]), (blocked, ignore_timers, len(s.traces), int(r["interleavings"]))
    assert py_hashes == [int(h) for h in hashes], (blocked, ignore_timers)
    assert sum(len(t) - 1 for t in s.traces) == int(r["deliveries"])
    assert s.races == int(r["races"]) and s.next_id == int(r["n_nodes"]) and len(s.explored) == int(r["n_explored"])
    assert [(k, v) for k, v in s.violations] == [(int(x["interleaving"]), int(x["code"])) for x in viol]
    assert bool(exhausted) == bool(r["exhausted"])
    return r, [int(h) for h in hashes]


def differs(a, b):
    (ra, ha), (rb, hb) = a, b
    return ha != hb or any(int(ra[f]) != int(rb[f]) for f in ("interleavings", "violations", "deliveries", "races"))


def test_dpor_with_blocked_actors_matches_the_restatement(oracle):
    """getMatchingMessage consumes a nextTrace entry whose receiver is blocked and returns None (:478, :518);
    getPendingEvent skips queues whose receiver is blocked (:455)."""
    pprog = [D.Start(0), D.Start(1), D.Start(2), D.Send(2, 1, 0), D.Send(2, 1, 1), D.Send(0, 1, 2)]
    base = dpor_case(oracle, N.MODEL_PINGPONG3, pprog, PP_FLAGS, 40, 500)
    for b in range(3):
        assert differs(dpor_case(oracle, N.MODEL_PINGPONG3, pprog, PP_FLAGS, 40, 500, blocked=(b,)), base), b
    r, hashes = dpor_case(oracle, N.MODEL_PINGPONG3, pprog, PP_FLAGS, 40, 500, blocked=(0, 1, 2))
    assert int(r["deliveries"]) == 0 and int(r["interleavings"]) == 1
    rng = np.random.default_rng(21)
    for i, prog in enumerate(raft_programs(5, rng)):
        base = dpor_case(oracle, N.MODEL_RAFT5, prog, 1, 24, 400)
        for blocked in ((i % 5,), (i % 5, (i + 2) % 5)):
            assert differs(dpor_case(oracle, N.MODEL_RAFT5, prog, 1, 24, 400, blocked=blocked), base), (i, blocked)


def test_dpor_delivers_timers_under_ignore_timers(oracle):
    """DPORwHeuristics never reads ignoreTimers: the flag leaves every search as it is, while a search that dropped the
    timers would be a different one."""
    rng = np.random.default_rng(22)
    for i, prog in enumerate(raft_programs(4, rng)):
        blocked = () if i % 2 == 0 else ((i + 1) % 5,)
        on = dpor_case(oracle, N.MODEL_RAFT5, prog, 1, 24, 400, blocked=blocked, ignore_timers=1)
        off = dpor_case(oracle, N.MODEL_RAFT5, prog, 1, 24, 400, blocked=blocked)
        assert not differs(on, off)
        dropped, _, dropped_hashes = python_dpor(N.MODEL_RAFT5, prog, 1, 24, 400, blocked, cls=_TimersDropped)
        assert dropped_hashes != on[1] and len(dropped.traces) < int(on[0]["interleavings"])


# ---------------------------------------------------------------------------------------------- RandomScheduler
class _StaticBlocked(M.Execution):
    """blockedActors as the engine offers it (DESIGN.md §8): a static set; a Start does not unblock the actor."""

    def inject_until_quiescence(self):
        M.Execution.inject_until_quiescence(self)
        self.blockedActors |= self.static_blocked


def record(oracle, model, prog, seed, maxm, interval, flags, blocked=(), ignore_timers=0):
    """One RandomScheduler execution under the switches, on both sides: (C events, restatement events, verdict)."""
    make, inv, is_ext = model_parts(model, flags)
    ex = _StaticBlocked(make(), to_prog(prog), seed, maxm, interval, inv, is_ext, blocked=[str(b) for b in blocked],
                        ignore_timers=bool(ignore_timers))
    ex.static_blocked = set(str(b) for b in blocked)
    v = ex.run() or 0
    ev, par, r = oracle.fuzz_trace(model, D.pack_externals(prog), seed, maxm, interval, model_flags=flags,
                                   blocked_mask=bits_of(blocked), ignore_timers=ignore_timers)
    assert [tuple(int(e[f]) for f in EV_FIELDS) for e in ev] == [row[:7] for row in flat(ex.events)], seed
    assert int(r["violation"]) == v
    return ev, ex.events, v


def test_fuzz_with_ignore_timers_matches_the_restatement(oracle):
    """RandomScheduler under ignoreTimers on raft5: no timer is ever sent, so no election starts."""
    prog = D.raft5_program(client_cmds=3)
    ext = D.pack_externals(prog)
    make, inv, is_ext = model_parts(N.MODEL_RAFT5, 1)
    seeds = list(range(1, 301))
    for it in (1, 0):
        res = oracle.fuzz_batch(N.MODEL_RAFT5, ext, seeds[0], len(seeds), 60, 5, model_flags=1, ignore_timers=it)
        for k, seed in enumerate(seeds):
            ex = M.Execution(make(), to_prog(prog), seed, 60, 5, inv, is_ext, ignore_timers=bool(it))
            v = ex.run() or 0
            r = res[k]
            assert (int(r["violation"]), int(r["steps"]), int(r["n_nodes"]), int(r["n_events"]), int(r["max_pending"]),
                    int(r["status"])) == (v, ex.messagesScheduledSoFar, ex.depTracker.next_id, len(ex.events),
                                          ex.max_pending, 0), (it, seed)
            if k % 10 == 0:
                record(oracle, N.MODEL_RAFT5, prog, seed, 60, 5, 1, ignore_timers=it)
        if it:
            timer_sends = [e for e in ex.events if e[0] == "MsgSend" and e[1] == "Timer"]
            assert not timer_sends and (res["steps"] == 8).all()          # 5 boots and 3 client commands, nothing else
        else:
            assert (res["steps"] > 8).all() and res["violation"].any()


# ------------------------------------------------------------------------------------------------ STSScheduler
class _StaticBlockedReplay(M.STSReplay):
    """STSReplay with the static mask: trigger_start's unblocking (the Spawn in advance_replay) does not hold."""

    def message_pending(self, snd, rcv, msg):
        self.blockedActors |= self.static_blocked
        return M.STSReplay.message_pending(self, snd, rcv, msg)


def replay_case(oracle, model, prog, flags, ev, py_events, code, n_masks, rng, blocked=(), ignore_timers=0):
    """STSScheduler.test of random external subsequences of one recorded trace under the switches, restatement against
    oracle_replay_trace (verdict, delivered, ignored, whole recorded EventTrace) and oracle_replay_batch.  Returns the
    (violation, delivered, ignored) of every replay, in (mask, filter) order."""
    make, inv, is_ext = model_parts(model, flags)
    ext = D.pack_externals(prog)
    events = to_prog(prog)
    n_ext, mw = len(ext), oracle.mask_words(len(ext))
    full = np.asarray(oracle.full_mask(ext), dtype=np.uint64).reshape(-1)
    masks = np.zeros((n_masks, mw), dtype=np.uint64)
    for t in range(n_masks):
        keep = rng.random(n_ext) < rng.choice([0.95, 0.8, 0.5]) if t else np.ones(n_ext, dtype=bool)
        for i in np.nonzero(keep)[0]:
            masks[t, i >> 6] |= np.uint64(1) << np.uint64(i & 63)
        masks[t] &= full
    sw = dict(blocked_mask=bits_of(blocked), ignore_timers=ignore_timers)
    out = []
    for fka in (0, 1):
        batch = oracle.replay_batch(model, ev, ext, masks, looking_for=code, flags=fka, model_flags=flags, **sw)
        for t in range(n_masks):
            subseq = [i for i in range(n_ext) if (int(masks[t, i >> 6]) >> (i & 63)) & 1]
            sts = _StaticBlockedReplay(make(), py_events, events, inv, is_ext, filter_known_absents=bool(fka),
                                       looking_for=code or None, blocked=[str(b) for b in blocked],
                                       ignore_timers=bool(ignore_timers))
            sts.static_blocked = set(str(b) for b in blocked)
            got = (sts.test(subseq) or 0, sts.delivered, sts.ignored)
            res, rec = oracle.replay_trace(model, ev, ext, masks[t], looking_for=code, flags=fka, model_flags=flags, **sw)
            assert int(res["status"]) == 0
            assert got == (int(res["violation"]), int(res["delivered"]), int(res["ignored"])), (t, fka, blocked, ignore_timers)
            assert [row[:7] for row in flat(sts.events)] == [tuple(int(e[f]) for f in EV_FIELDS) for e in rec], (t, fka)
            assert tuple(int(batch[t][f]) for f in ("violation", "delivered", "ignored")) == got, (t, fka)
            out.append(got)
    return out


def violating_seed(oracle, model, prog, maxm, interval, flags, n=400, **sw):
    res = oracle.fuzz_batch(model, D.pack_externals(prog), 1, n, maxm, interval, model_flags=flags, **sw)
    hits = np.nonzero(res["violation"])[0]
    assert len(hits)
    return 1 + int(hits[0])


def test_sts_replay_with_blocked_actors_matches_the_restatement(oracle):
    """A blocked receiver's delivery is never enabled (STSScheduler.messagePending, :381-403): it is ignored."""
    rng = np.random.default_rng(23)
    cases = [(N.MODEL_RAFT5, D.raft5_program(client_cmds=3), 60, 5, 1, (2,)),
             (N.MODEL_RAFT5, D.raft5_program(client_cmds=3), 60, 5, 1, (0, 3)),
             (N.MODEL_PINGPONG3, D.pingpong3_program(20), -1, 3, 1 | (4 << 8), (1,))]
    for model, prog, maxm, interval, flags, blocked in cases:
        # a trace recorded under the mask, replayed under it
        seed = violating_seed(oracle, model, prog, maxm, interval, flags, blocked_mask=bits_of(blocked))
        ev, py_events, code = record(oracle, model, prog, seed, maxm, interval, flags, blocked=blocked)
        replay_case(oracle, model, prog, flags, ev, py_events, code, 12, rng, blocked=blocked)
        # a trace recorded without it: the mask decides what the replay delivers
        seed = violating_seed(oracle, model, prog, maxm, interval, flags)
        ev, py_events, code = record(oracle, model, prog, seed, maxm, interval, flags)
        on = replay_case(oracle, model, prog, flags, ev, py_events, code, 12, rng, blocked=blocked)
        off = replay_case(oracle, model, prog, flags, ev, py_events, code, 4, rng)
        assert on[0][2] > 0 and off[0] == (code, off[0][1], 0)           # full subsequence: ignored only under the mask


def test_sts_replay_with_ignore_timers_matches_the_restatement(oracle):
    """STSScheduler's timers go through handle_timer, so under ignoreTimers none is sent.  A raft5 trace recorded with
    timers and replayed under the flag: every recorded timer delivery is ignored, and so is whatever it caused."""
    rng = np.random.default_rng(24)
    prog = D.raft5_program(client_cmds=3)
    seed = violating_seed(oracle, N.MODEL_RAFT5, prog, 60, 5, 1)
    ev, py_events, code = record(oracle, N.MODEL_RAFT5, prog, seed, 60, 5, 1)
    on = replay_case(oracle, N.MODEL_RAFT5, prog, 1, ev, py_events, code, 16, rng, ignore_timers=1)
    timer_deliveries = sum(1 for e in ev if int(e["kind"]) == N.EV_MSG_EVENT and int(e["type"]) in RAFT_TIMER_TYPES)
    external_deliveries = sum(1 for e in ev if int(e["kind"]) == N.EV_MSG_EVENT and int(e["type"]) in (M.BOOT, M.CLIENT_CMD))
    assert timer_deliveries > 0
    # only the boots and client commands are delivered; every timer delivery is ignored
    assert on[0][0] == 0 and on[0][1] == external_deliveries and on[0][2] >= timer_deliveries
    off = replay_case(oracle, N.MODEL_RAFT5, prog, 1, ev, py_events, code, 4, rng)
    assert off[0] == (code, off[0][1], 0)
    # a trace recorded under the flag replays under it in full, with the blocked-actor mask on top
    ev, py_events, code = record(oracle, N.MODEL_RAFT5, prog, 3, 60, 5, 1, ignore_timers=1)
    out = replay_case(oracle, N.MODEL_RAFT5, prog, 1, ev, py_events, code, 8, rng, ignore_timers=1)
    assert out[0] == (0, 8, 0)
    replay_case(oracle, N.MODEL_RAFT5, prog, 1, ev, py_events, code, 8, rng, blocked=(1,), ignore_timers=1)
