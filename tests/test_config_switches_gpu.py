"""GPU parity of SchedulerConfig's two execution switches, blockedActors (a static mask, DESIGN.md §8) and ignoreTimers,
on the replay (K2), DPOR (K3, K3F), provenance and wildcard paths: each engine against the CPU oracle under the same
configuration, bit-exact on every result field, schedule-hash sequence and recorded event.

No case is vacuous: each switched case also runs with the switch off and the two must differ, except ignoreTimers on
DPOR, which DPORwHeuristics never reads (DESIGN.md §6): there the two must be equal.  A trace recorded under a switch
carries its effect already (no delivery to a blocked actor, no timer), so its replay cannot tell the switch from its
absence; the on/off comparison of the replay paths is made on a trace recorded without the switch."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
import micro_oracle as M
from oracle import binding as O
from oracle import wildcard_binding as W

pytestmark = pytest.mark.gpu

RAFT, PP, BC = N.MODEL_RAFT5, N.MODEL_PINGPONG3, N.MODEL_BCAST32
DPOR_FIELDS = ["interleavings", "violations", "deliveries", "races", "n_nodes", "n_explored", "heap_left", "exhausted",
               "budget_exhausted", "status"]
FR_FIELDS = ["interleavings", "violations", "deliveries", "races", "keys_enqueued", "keys_dropped", "explored_pairs",
             "pool_left", "rounds", "exhausted", "budget_exhausted", "status", "trace_slots"]
EV_FIELDS = ["kind", "src", "dst", "type", "p0", "p1", "uniq", "node"]
PP_FLAGS = 1 | (2 << 8)


def engine(model, flags, blocked=0, it=False):
    return D.Engine(D.SchedulerConfig(model, model_flags=flags, blocked_mask=blocked, ignoreTimers=it))


def sw(blocked=0, it=False):
    return dict(blocked_mask=blocked, ignore_timers=1 if it else 0)


def rows(a):
    return [tuple(int(e[f]) for f in EV_FIELDS) for e in a]


def raft_programs(n, rng):
    progs = []
    for _ in range(n):
        order = rng.permutation(5)
        ev = [D.Start(int(a)) for a in order]
        k = int(rng.integers(3, 6))
        ev += [D.Send(int(a), 1, 0x1F) for a in rng.permutation(5)[:k]]
        ev += [D.Send(int(rng.integers(0, 5)), 2, int(rng.integers(1, 50))) for _ in range(int(rng.integers(0, 3)))]
        progs.append(ev)
    return progs


def random_masks(ext, n, seed):
    rng = np.random.default_rng(seed)
    mw = O.mask_words(len(ext))
    full = O.full_mask(ext)
    m = np.zeros((n, mw), dtype=np.uint64)
    for t in range(n):
        keep = rng.random(len(ext)) < rng.choice([0.95, 0.8, 0.5])
        for i in np.nonzero(keep)[0]:
            m[t, i >> 6] |= np.uint64(1) << np.uint64(i & 63)
    m &= full[None, :]
    m[0] = full
    return m


def recorded(model, prog, flags, maxm, interval, n=2000, **rec_sw):
    """The first violating execution under the recording switches (or seed 1 when none violates): (ext, events, code)."""
    ext = D.pack_externals(prog)
    res = O.fuzz_batch(model, ext, 1, n, maxm, interval, model_flags=flags, **rec_sw)
    hits = np.nonzero(res["violation"])[0]
    seed = 1 + int(hits[0]) if len(hits) else 1
    ev, par, r = O.fuzz_trace(model, ext, seed, maxm, interval, model_flags=flags, **rec_sw)
    return ext, ev, int(r["violation"])


# ------------------------------------------------------------------------------------------------------------- K2
K2_CASES = [
    ("raft5_blocked_one", RAFT, D.raft5_program(client_cmds=4), 1, 50, 5, 1 << 2, False),
    ("raft5_blocked_two", RAFT, D.raft5_program(client_cmds=4), 1, 50, 5, (1 << 0) | (1 << 3), False),
    ("raft5_ignore_timers", RAFT, D.raft5_program(client_cmds=4), 1, 50, 5, 0, True),
    ("raft5_both", RAFT, D.raft5_program(client_cmds=4), 1, 50, 5, 1 << 1, True),
    ("pingpong3_blocked", PP, D.pingpong3_program(20), 1 | (4 << 8), -1, 3, 1 << 1, False),
    ("bcast32_blocked", BC, D.bcast32_program(2), 3, 120, 10, (1 << 5) | (1 << 17), False),
]


def k2_check(model, flags, ext, ev, code, blocked, it, n_masks=400, seed=0):
    """replay_batch (plain, filterKnownAbsents, strict), replay_batch_ex with skip_events and replay_trace under the
    switches against the oracle.  Returns the plain replay_batch results."""
    eng = engine(model, flags, blocked, it)
    eng.set_trace(ev, ext)
    masks = random_masks(ext, n_masks, seed)
    out = None
    for fl in (0, N.RF_FILTER_KNOWN_ABSENTS, N.RF_STRICT):
        gpu = eng.replay_batch(masks, code, fl)
        cpu = O.replay_batch(model, ev, ext, masks, looking_for=code, flags=fl, model_flags=flags, **sw(blocked, it))
        bad = np.nonzero(gpu != cpu)[0]
        assert len(bad) == 0, (fl, bad[:5], gpu[bad[:3]], cpu[bad[:3]])
        out = gpu if out is None else out
    deliveries = np.nonzero(ev["kind"] == N.EV_MSG_EVENT)[0].astype(np.uint32)
    skips = deliveries[np.linspace(0, len(deliveries) - 1, min(16, len(deliveries))).astype(int)]
    gpu = eng.replay_batch_ex(None, skips, code)
    all_ext = O.full_mask(ext, False)
    for j, idx in enumerate(skips):
        rc, _ = O.replay_trace(model, ev, ext, all_ext, looking_for=code, model_flags=flags, skip_event=int(idx),
                               **sw(blocked, it))
        assert gpu[j] == rc, j
    for t in range(3):
        for fl in (0, N.RF_FILTER_KNOWN_ABSENTS):
            r, rec = eng.replay_trace(masks[t], looking_for=code, flags=fl)
            rc, crec = O.replay_trace(model, ev, ext, masks[t], looking_for=code, flags=fl, model_flags=flags,
                                      **sw(blocked, it))
            assert r == rc and rows(rec) == rows(crec), (t, fl)
    return out


@pytest.mark.parametrize("case", K2_CASES, ids=[c[0] for c in K2_CASES])
def test_replay_under_switches(oracle, case):
    _, model, prog, flags, maxm, interval, blocked, it = case
    # a trace recorded under the same switches
    ext, ev, code = recorded(model, prog, flags, maxm, interval, **sw(blocked, it))
    k2_check(model, flags, ext, ev, code, blocked, it, seed=1)
    # a trace recorded without them: the switch decides what the replay delivers
    ext, ev, code = recorded(model, prog, flags, maxm, interval)
    on = k2_check(model, flags, ext, ev, code, blocked, it, seed=2)
    off = k2_check(model, flags, ext, ev, code, 0, False, n_masks=400, seed=2)
    assert on[0]["ignored"] > 0 and off[0]["ignored"] == 0
    assert (on != off).sum() > len(on) // 4


def blocked_candidates(model, prog, flags, maxm, interval, actors, n=4000, limit=12):
    """(ext, events, code, blocked) of violating traces recorded without a mask whose full replay under `blocked` still
    shows the violation while ignoring deliveries: the traces the minimizers can run on with and without the mask."""
    ext = D.pack_externals(prog)
    res = O.fuzz_batch(model, ext, 1, n, maxm, interval, model_flags=flags)
    full = O.full_mask(ext)
    for i in np.nonzero(res["violation"])[0][:limit]:
        ev, par, r = O.fuzz_trace(model, ext, 1 + int(i), maxm, interval, model_flags=flags)
        code = int(r["violation"])
        for a in actors:
            rr = O.replay_batch(model, ev, ext, [full], looking_for=code, model_flags=flags, blocked_mask=1 << a)
            if int(rr[0]["violation"]) == code and int(rr[0]["ignored"]) > 0:
                yield ext, ev, code, 1 << a


@pytest.mark.parametrize("model,prog,flags,maxm,interval,actors,ddmin_changes", [
    (RAFT, D.raft5_program(client_cmds=8), 1, 50, 5, range(5), True),
    (PP, D.pingpong3_program(24), 1 | (5 << 8), -1, 3, (1, 2), False),
], ids=["raft5", "pingpong3"])
def test_ddmin_and_internal_minimization_under_a_mask(oracle, model, prog, flags, maxm, interval, actors, ddmin_changes):
    """DDMin (MCS, total replays, iteration sizes) and STSSchedMinimizer (minimized trace, replays, sizes) under a
    blocked-actor mask against the oracle, on a trace where the mask changes the outcome of both on raft5.  On
    pingpong3 the pongs a blocked actor misses never decide actor 0's violation, so there the mask changes the
    internal minimization only; DDMin is still compared under it."""
    found = 0
    for ext, ev, code, blocked in blocked_candidates(model, prog, flags, maxm, interval, actors):
        rc, cmcs, total, iters, verified = O.ddmin_sts(model, ev, ext, code, model_flags=flags, blocked_mask=blocked)
        rc0, cmcs0, total0, iters0, _ = O.ddmin_sts(model, ev, ext, code, model_flags=flags)
        full = O.full_mask(ext)
        _, vtrace = O.replay_trace(model, ev, ext, full, looking_for=code, model_flags=flags)
        irc, ctrace, itotal, sizes, unig = O.internal_minimize(model, vtrace, ext[ext["kind"] != N.EXT_WAIT_QUIESCENCE], code,
                                                               model_flags=flags, blocked_mask=blocked)
        irc0, ctrace0, itotal0, sizes0, _ = O.internal_minimize(model, vtrace, ext[ext["kind"] != N.EXT_WAIT_QUIESCENCE],
                                                                code, model_flags=flags)
        assert rc == rc0 == irc == irc0 == 0
        dd_differs = not np.array_equal(cmcs, cmcs0) or total != total0 or not np.array_equal(iters, iters0)
        im_differs = rows(ctrace) != rows(ctrace0) or itotal != itotal0 or not np.array_equal(sizes, sizes0)
        if not (im_differs and (dd_differs or not ddmin_changes)):
            continue
        eng = engine(model, flags, blocked)
        eng.set_trace(ev, ext)
        mcs, giters, out = eng.ddmin(code)
        assert np.array_equal(mcs, cmcs) and out.total_replays == total and list(giters) == [int(x) for x in iters]
        assert out.verified == verified
        eng.set_trace(vtrace, ext[ext["kind"] != N.EXT_WAIT_QUIESCENCE])
        mtrace, msizes, mout = eng.internal_minimize(code)
        assert rows(mtrace) == rows(ctrace) and mout.total_replays == itotal
        assert [int(x) for x in msizes] == [int(x) for x in sizes] and mout.unignorable == unig
        found += 1
        if found == 2:
            break
    assert found >= 1


# ------------------------------------------------------------------------------------------------------------- K3
def dpor_check(model, progs, flags, maxm, maxi, blocked=0, it=False, looking_for=0, stop=False, node_cap=4096,
               explored_slots=1 << 16, heap_cap=1 << 15):
    eng = engine(model, flags, blocked, it)
    res, viol, hashes = eng.dpor_batch(progs, maxm, maxi, looking_for, stop, -1, node_cap=node_cap,
                                       explored_slots=explored_slots, heap_cap=heap_cap, cap_viol=32, want_hashes=True)
    out = []
    for s, prog in enumerate(progs):
        rc, r, cviol, chashes = O.dpor_search(model, D.pack_externals(prog), maxm, maxi, looking_for, 1 if stop else 0, -1,
                                              model_flags=flags, node_cap=node_cap, explored_slots=explored_slots,
                                              heap_cap=heap_cap, cap_viol=32, **sw(blocked, it))
        for f in DPOR_FIELDS:
            assert res[s][f] == r[f], (s, f, res[s], r)
        n = int(r["interleavings"])
        assert (hashes[s][:n] == chashes).all(), s
        nv = min(int(r["violations"]), 32)
        assert (viol[s][:nv] == cviol[:nv]).all(), s
        out.append((tuple(int(res[s][f]) for f in DPOR_FIELDS), tuple(int(h) for h in hashes[s][:n])))
    return out


def test_dpor_batch_under_blocked_masks(oracle):
    rng = np.random.default_rng(31)
    progs = raft_programs(12, rng)
    off = dpor_check(RAFT, progs, 1, 24, 400)
    for blocked in (1 << 0, 1 << 3, (1 << 1) | (1 << 4), (1 << 2) | (1 << 0)):
        on = dpor_check(RAFT, progs, 1, 24, 400, blocked)
        assert all(a != b for a, b in zip(on, off)), blocked
    on = dpor_check(RAFT, progs, 1, 24, 400, 0x1F)
    assert all(r[0][2] == 0 and r[0][0] == 1 for r in on)           # every receiver blocked: nothing is delivered
    pprogs = [[D.Start(a) for a in range(3)] + [D.Send(int(a), 1, k) for k, a in enumerate(rng.integers(0, 3, size=5))]
              for _ in range(8)]
    off = dpor_check(PP, pprogs, PP_FLAGS, 40, 500, looking_for=7)
    for blocked in (1 << 0, 1 << 1, 1 << 2, (1 << 0) | (1 << 2)):
        on = dpor_check(PP, pprogs, PP_FLAGS, 40, 500, blocked, looking_for=7)
        assert all(a != b for a, b in zip(on, off)), blocked
    on = dpor_check(PP, pprogs, PP_FLAGS, 40, 500, 0x7, looking_for=7)
    assert all(r[0][2] == 0 and r[0][0] == 1 for r in on)


@pytest.mark.parametrize("maxm", [40, 100])
def test_dpor_batch_bcast32(oracle, maxm):
    """bcast32's instantiation of K3, no switch."""
    progs = [D.bcast32_program(ttl)[:-1] for ttl in (1, 2, 3)]
    progs += [[D.Start(a) for a in range(32)] + [D.Send(a, 2, 2) for a in (0, 9, 31)]]
    out = dpor_check(BC, progs, 3, maxm, 200, node_cap=1 << 14, explored_slots=1 << 18, heap_cap=1 << 17)
    assert all(r[0][9] == 0 for r in out) and any(r[0][0] > 1 for r in out)


class _TimersDropped(M.DPORSearch):
    """What a DPOR that obeyed ignoreTimers would do: a scheduled timer is registered but never sent."""

    def handleTick(self, rcv, msg):
        if not self.timerToCancellable[(rcv, msg)]:
            del self.timerToCancellable[(rcv, msg)]


def test_dpor_ignores_ignore_timers(oracle):
    """DPORwHeuristics sends timers whatever ignoreTimers says: K3 and K3F with the flag equal the oracle's and their
    own results without it, on raft5, whose searches dropping the timers would change."""
    rng = np.random.default_rng(32)
    progs = raft_programs(8, rng)
    for blocked in (0, 1 << 2):
        on = dpor_check(RAFT, progs, 1, 24, 400, blocked, it=True)
        off = dpor_check(RAFT, progs, 1, 24, 400, blocked)
        assert on == off
    for prog, r in zip(progs[:3], on):
        s = _TimersDropped(lambda: {str(i): M.RaftActor(i, 1) for i in range(5)}, _micro_prog(prog), M.raft_invariant, 24,
                           stop_if_found=False, blocked=["2"])
        s.search(400)
        assert len(s.traces) < r[0][0]
    for width in (1, 64):
        for prog in progs[:3]:
            a = frontier_check(RAFT, prog, 3, 40, 300, width, it=True)
            b = frontier_check(RAFT, prog, 3, 40, 300, width)
            assert a == b


def _micro_prog(prog):
    out = []
    for e in prog:
        if type(e).__name__ == "Start":
            out.append(("Start", str(e.a)))
        else:
            out.append(("Send", str(e.a), (e.type, e.p0, e.p1)))
    return out


def seeded_world():
    eng = engine(RAFT, 1)
    prog = D.raft5_program()
    eng.set_externals(prog)
    ext_all = D.pack_externals(prog)
    dext = ext_all[(ext_all["kind"] == N.EXT_START) | (ext_all["kind"] == N.EXT_SEND)]
    res = eng.fuzz_batch(1, 3000, 40, 5)
    i = int(np.nonzero(res["violation"] == 1)[0][0])
    ev, par, r = eng.fuzz_trace(1 + i, 40, 5)
    return dext, ev, par, int(r["steps"])


def test_dpor_batch_ex_and_incremental_ddmin_under_a_mask(oracle):
    """RunnerUtils.editDistanceDporDDMin's configuration (seeded graph, ArvindDistanceOrdering, prioritized pending)
    under a mask: the recorded trace's deliveries to the blocked actor are consumed without a match."""
    dext, ev, par, steps = seeded_world()
    rng = np.random.default_rng(33)
    programs = [dext]
    for _ in range(11):
        keep = np.ones(len(dext), dtype=bool)
        keep[rng.integers(5, len(dext), size=int(rng.integers(1, 3)))] = False
        programs.append(dext[keep])
    flags = N.DF_ARVIND_ORDERING | N.DF_PRIORITIZE_PENDING
    results = {}
    for blocked in (0, 1 << 3):
        eng = engine(RAFT, 1, blocked)
        res, hashes = eng.dpor_batch_ex(programs, steps, 60, seed=(ev, par), flags=flags, looking_for=1, want_hashes=True)
        got = []
        for t, p in enumerate(programs):
            inst = O.DporInstance(RAFT, p, steps, 60, seed=O.dpor_seed(ev, par), arvind=1, prioritize_pending=1,
                                  model_flags=1, looking_for=1, blocked_mask=blocked)
            r, h = inst.test(-1)
            inst.close()
            for f in ("interleavings", "violations", "deliveries", "races", "n_nodes", "n_explored", "heap_left", "status"):
                assert int(res[t][f]) == int(r[f]), (blocked, t, f)
            assert hashes[t][:len(h)].tolist() == h.tolist(), (blocked, t)
            got.append((int(r["interleavings"]), int(r["violations"]), h.tolist()))
        results[blocked] = got
    assert all(a != b for a, b in zip(results[0], results[1 << 3]))
    stats = {}
    for blocked in (0, 1 << 3):
        rc, mcs_o, st = O.incremental_ddmin(RAFT, dext, steps, 2000, O.dpor_seed(ev, par), model_flags=1, looking_for=1,
                                            stop_at_size=1, max_max_distance=64, blocked_mask=blocked)
        assert rc == 0
        mcs, out = engine(RAFT, 1, blocked).incremental_ddmin(dext, steps, 2000, (ev, par), looking_for=1, stop_at_size=1,
                                                              max_max_distance=64, heap_cap=1 << 16)
        assert np.array_equal(mcs, mcs_o)
        assert (out.total_replays, out.rounds, out.instances) == (st["total_replays"], st["rounds"], st["instances"])
        stats[blocked] = (mcs_o.tolist(), st["total_replays"], st["rounds"], st["interleavings"])
    assert stats[0] != stats[1 << 3]


# ------------------------------------------------------------------------------------------------------------ K3F
def frontier_check(model, prog, flags, maxm, maxi, width, blocked=0, it=False, **kw):
    eng = engine(model, flags, blocked, it)
    F = eng.frontier_params(maxm, maxi, width, explored_slots=1 << 20, pool_cap=1 << 21, **kw)
    r, viol, hashes = eng.dpor_frontier(prog, F)
    OF = O.frontier_params(maxm, maxi, width, explored_slots=1 << 20, pool_cap=1 << 21, **kw)
    rc, ores, oviol, ohashes = O.dpor_frontier(model, D.pack_externals(prog), OF, 1, model_flags=flags, **sw(blocked, it))
    assert rc == 0
    for f in FR_FIELDS:
        assert r[f] == ores[0][f], (f, r, ores[0])
    assert (hashes == ohashes[0]).all()
    assert (viol == oviol[0]).all()
    return tuple(int(r[f]) for f in FR_FIELDS), tuple(int(h) for h in hashes)


@pytest.mark.parametrize("width", [1, 64, 1024])
def test_frontier_under_a_mask(oracle, width):
    rng = np.random.default_rng(34)
    for k, prog in enumerate(raft_programs(3, rng)):
        blocked = 1 << (k + 1)
        on = frontier_check(RAFT, prog, 3, 60, 150, width, blocked)
        off = frontier_check(RAFT, prog, 3, 60, 150, width)
        assert on != off and on[0][11] == 0
        on = frontier_check(RAFT, prog, 3, 100, 5000, width, blocked | (1 << 4))
        assert on[0][11] == 0


def test_frontier_exhaustive_set_parity_under_a_mask(oracle):
    """A bounded-exhaustive wide search under a mask visits the same set of schedules as the sequential one."""
    rng = np.random.default_rng(35)
    cases = [(RAFT, prog, 3, 40, 1 << 2) for prog in raft_programs(2, rng)]
    cases.append((PP, [D.Start(a) for a in range(3)] + [D.Send(k % 3, 1, k) for k in range(8)], PP_FLAGS, 18, 1 << 1))
    for model, prog, flags, maxm, blocked in cases:
        sets = {}
        for b in (blocked, 0):
            rc, sr, sviol, shashes = O.dpor_search(model, D.pack_externals(prog), maxm, 100000, 0, 0, -1, model_flags=flags,
                                                   node_cap=1 << 16, explored_slots=1 << 22, heap_cap=1 << 22,
                                                   cap_viol=100000, blocked_mask=b)
            assert rc == 0 and sr["exhausted"] == 1
            sets[b] = (set(int(x) for x in shashes), set(int(x) for x in sviol["schedule_hash"]))
        assert sets[blocked][0] != sets[0][0]
        eng = engine(model, flags, blocked)
        F = eng.frontier_params(maxm, 100000, 256, explored_slots=1 << 22, pool_cap=1 << 22)
        r, viol, hashes = eng.dpor_frontier(prog, F, cap_viol=100000)
        assert r["exhausted"] == 1 and r["status"] == 0
        assert (set(int(x) for x in hashes), set(int(x) for x in viol["schedule_hash"])) == sets[blocked]


# ----------------------------------------------------------------------------------------- provenance, wildcard
@pytest.mark.parametrize("blocked,it", [(1 << 2, False), (0, True)], ids=["blocked_warp", "ignore_timers_lane"])
def test_fuzz_provenance_under_switches(oracle, blocked, it):
    ext = D.pack_externals(D.raft5_program())
    n = 6000
    recs = {}
    for b, i in ((blocked, it), (0, False)):
        eng = engine(RAFT, 1, b, i)
        eng.set_externals(ext)
        res = eng.fuzz_batch(1, n, 50, 5)
        assert (res == O.fuzz_batch(RAFT, ext, 1, n, 50, 5, model_flags=1, **sw(b, i))).all()
        viol = np.nonzero(res["violation"])[0].astype(np.uint32)
        idx = np.concatenate([viol[:120], np.nonzero(res["violation"] == 0)[0][:8].astype(np.uint32)])
        keep, out, rec = eng.fuzz_provenance(1, idx, 50, 5)
        assert np.array_equal(rec["trace_hash"], res["trace_hash"][idx])
        for j, k in enumerate(idx):
            kk, o = O.fuzz_provenance(RAFT, ext, 1 + int(k), 50, 5, keep.shape[1], model_flags=1, **sw(b, i))
            assert o["status"] == out[j]["status"] == 0
            assert np.array_equal(kk, keep[j]), int(k)
            for f in ("violation", "affected_mask", "n_trace", "n_kept"):
                assert o[f] == out[j][f], (f, int(k))
        recs[(b, i)] = (res, idx, keep, out)
    on, off = recs[(blocked, it)], recs[(0, False)]
    assert not np.array_equal(on[0]["trace_hash"], off[0]["trace_hash"])
    if blocked:
        assert len(on[1]) > 8 and not np.array_equal(on[2], off[2][:len(on[2])])


def test_wildcard_minimize_under_a_mask(oracle):
    rules, incr = D.raft5_clock_rules()
    rules, incr = list(rules), list(incr)
    prog = D.raft5_program(client_cmds=2)
    done = 0
    for ext, ev, code, blocked in blocked_candidates(RAFT, prog, 1, 40, 5, range(5)):
        mcs_ext = ext[ext["kind"] != N.EXT_WAIT_QUIESCENCE]
        _, vtrace = O.replay_trace(RAFT, ev, ext, O.full_mask(ext), looking_for=code, model_flags=1)
        outs = {}
        for b in (blocked, 0):
            rc, ctrace, total, csizes = W.wildcard_minimize(RAFT, vtrace, mcs_ext, rules, incr, code, model_flags=1,
                                                            blocked_mask=b)
            assert rc == 0
            outs[b] = (rows(ctrace), total, [int(x) for x in csizes])
        if outs[blocked] == outs[0]:
            continue
        eng = engine(RAFT, 1, blocked)
        eng.set_trace(vtrace, mcs_ext)
        eng.set_clock_rules(rules, incr)
        trace, sizes, out = eng.wildcard_minimize(code)
        assert (rows(trace), out.total_replays, [int(x) for x in sizes]) == outs[blocked]
        done += 1
        if done == 2:
            break
    assert done >= 1
