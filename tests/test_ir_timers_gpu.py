"""Loaded models that arm timers on the device: replay (K2), DDMin, internal and wildcard minimization and frontier
DPOR (K3F) against the C oracle, every field bit-exact — on the hand-written leader election of
tests/test_ir_timers_oracle.py, on the generated models of tests/ir_gen.py that use timers, and at the timer-set
capacity edges.  No answer may be DEMI_RS_UNSUPPORTED or DEMI_DS_UNSUPPORTED."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
from oracle import wildcard_binding as W
import ir_gen
import micro_oracle as M
from test_config_switches_gpu import FR_FIELDS, random_masks, rows
from test_dpor_frontier_multi_gpu import FIELDS as MULTI_FIELDS
from test_ir_timers_oracle import (ARM, DISARM, DISTINCT, DS_QUEUE_OVF, ELECT, ELECTION_BUG, ELECTION_INTERVAL, ELECTION_MAXM,
                                   ONCE, PS_QUEUE_OVF, TWO_LEADERS, edges_blob, edges_program, edges_recorded,
                                   election_blob, election_model, election_program, election_violation, prefix_masks,
                                   python_replay)
from test_wildcard_gpu import compare_minimize, compare_replays

pytestmark = pytest.mark.gpu
DS_UNSUPPORTED = 6


def ir_engine(blob, flags, ignore_timers=False):
    eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, model_flags=flags, ignoreTimers=ignore_timers))
    eng.load_model(blob)
    return eng


def frontier_case(oracle, eng, prog, model_flags, maxm, budget, width, ignore_timers=0, **kw):
    F = eng.frontier_params(maxm, budget, width, explored_slots=1 << 18, pool_cap=1 << 20, **kw)
    OF = oracle.frontier_params(maxm, budget, width, explored_slots=1 << 18, pool_cap=1 << 20, **kw)
    rc, ores, oviol, ohashes = oracle.dpor_frontier(N.MODEL_IR, D.pack_externals(prog), OF, 1, model_flags=model_flags,
                                                    ignore_timers=ignore_timers)
    try:
        r, viol, hashes = eng.dpor_frontier(prog, F)
    except D.DemiError:
        r = eng.last_frontier
        assert int(r["status"]) == int(ores[0]["status"]) != 0 and int(r["status"]) != DS_UNSUPPORTED
        return int(r["status"]), None
    for f in FR_FIELDS:
        assert r[f] == ores[0][f], (f, r, ores[0])
    assert (hashes == ohashes[0]).all() and (viol == oviol[0]).all()
    return tuple(int(r[f]) for f in FR_FIELDS), tuple(int(h) for h in hashes)


def replays_equal(oracle, eng, ev, ext, masks, code, flags, ignore_timers=0):
    out = {}
    for fl in (0, N.RF_FILTER_KNOWN_ABSENTS, N.RF_STRICT):
        gpu = eng.replay_batch(masks, code, fl)
        cpu = oracle.replay_batch(N.MODEL_IR, ev, ext, masks, looking_for=code, flags=fl, model_flags=flags,
                                  ignore_timers=ignore_timers)
        bad = np.nonzero(gpu != cpu)[0]
        assert len(bad) == 0, (fl, bad[:5], gpu[bad[:3]], cpu[bad[:3]])
        assert not (gpu["status"] == N.RS_UNSUPPORTED).any()
        out[fl] = gpu
    for t in range(3):
        for fl in (0, N.RF_FILTER_KNOWN_ABSENTS):
            r, rec = eng.replay_trace(masks[t], looking_for=code, flags=fl)
            rc, crec = oracle.replay_trace(N.MODEL_IR, ev, ext, masks[t], looking_for=code, flags=fl, model_flags=flags,
                                           ignore_timers=ignore_timers)
            assert r == rc and rows(rec) == rows(crec), (t, fl)
    return out[0]


def test_election_pipeline(oracle):
    """fuzz -> replay -> DDMin -> internal minimization -> wildcards -> frontier DPOR on the buggy election."""
    m = election_model()
    blob, flags = m.blob, m.flags
    ext, seed, ev = election_violation(oracle)
    W.load_model(blob)
    eng = ir_engine(blob, flags)
    eng.set_externals(ext)
    gpu = eng.fuzz_batch(1, 400, ELECTION_MAXM, ELECTION_INTERVAL)
    assert (gpu == oracle.fuzz_batch(N.MODEL_IR, ext, 1, 400, ELECTION_MAXM, ELECTION_INTERVAL, model_flags=flags)).all()
    assert seed == 1 + int(np.nonzero((gpu["violation"] == TWO_LEADERS) & (gpu["status"] == 0))[0][0])
    gev, gpar, _ = eng.fuzz_trace(seed, ELECTION_MAXM, ELECTION_INTERVAL)
    assert (gev == ev).all()
    # replay
    eng.set_trace(ev, ext)
    masks = random_masks(ext, 65, 7)
    on = replays_equal(oracle, eng, ev, ext, masks, TWO_LEADERS, flags)
    assert int(on[0]["violation"]) == TWO_LEADERS and int(on[0]["ignored"]) == 0
    # DDMin
    rc, cmcs, total, citers, ver = oracle.ddmin_sts(N.MODEL_IR, ev, ext, TWO_LEADERS, model_flags=flags)
    mcs, iters, dd = eng.ddmin(TWO_LEADERS)
    assert rc == 0 and (mcs == cmcs).all() and dd.total_replays == total and list(iters) == list(citers) and dd.verified == ver
    r = eng.replay_batch(mcs.reshape(1, -1), TWO_LEADERS)                   # verify_mcs: the MCS still shows the violation
    assert int(r[0]["violation"]) == TWO_LEADERS
    # internal minimization, both removal strategies
    full = np.asarray(oracle.full_mask(ext), dtype=np.uint64).reshape(-1)
    _, vtrace = oracle.replay_trace(N.MODEL_IR, ev, ext, full, looking_for=TWO_LEADERS, model_flags=flags)
    prog = election_program()
    mcs_prog = [prog[k] for k in range(len(ext)) if (int(full[k >> 6]) >> (k & 63)) & 1]
    mcs_ext = D.pack_externals(mcs_prog)
    for imflags in (0, N.IM_SRC_DST_FIFO):
        eng.set_trace(vtrace, mcs_ext)                                      # a minimization leaves its result in the handle
        rc, ctrace, ctotal, csizes, cunig = oracle.internal_minimize(N.MODEL_IR, vtrace, mcs_ext, TWO_LEADERS, flags=imflags,
                                                                     model_flags=flags)
        gtrace, gsizes, gout = eng.internal_minimize(TWO_LEADERS, flags=imflags)
        assert rc == 0 and rows(gtrace) == rows(ctrace) and gout.total_replays == ctotal
        assert list(gsizes) == list(csizes) and gout.unignorable == cunig and len(gtrace) < len(vtrace)
    # wildcards: the term is the logical clock of RequestVote, Vote and Heartbeat; the election timer increments it
    rules = [N.clock_rule(t, 0, 0, 32) for t in (3, 4, 5)]
    case = (vtrace, mcs_prog, mcs_ext, TWO_LEADERS)
    seen = compare_replays(oracle, eng, N.MODEL_IR, case, rules, (ELECT,), flags, np.random.default_rng(2), n_masks=16, n_rec=3)
    assert seen > 0
    for wflags in (0, N.WC_LAST_ONLY):
        compare_minimize(oracle, eng, N.MODEL_IR, case, rules, (ELECT,), flags, wflags)
    # ignoreTimers: no ElectionTimeout is ever sent, so nothing past the three Kicks is delivered
    ieng = ir_engine(blob, flags, ignore_timers=True)
    ieng.set_trace(ev, ext)
    off = replays_equal(oracle, ieng, ev, ext, masks, TWO_LEADERS, flags, ignore_timers=1)
    assert int(off[0]["violation"]) == 0 and int(off[0]["ignored"]) > 0 and (on != off).sum() > len(on) // 2
    rc, cmcs, total, citers, ver = oracle.ddmin_sts(N.MODEL_IR, ev, ext, TWO_LEADERS, model_flags=flags, ignore_timers=1)
    try:
        imcs, iiters, idd = ieng.ddmin(TWO_LEADERS)
        assert rc == 0 and (imcs == cmcs).all() and idd.total_replays == total and list(iiters) == list(citers)
        assert idd.verified == ver and (idd.verified != dd.verified or idd.total_replays != dd.total_replays)
    except D.DemiError:
        assert rc != 0


@pytest.mark.parametrize("width", [1, 64, 1024])
def test_election_frontier(oracle, width):
    m = election_model()
    oracle.load_model(m.blob)
    prog = election_program(wait=False)
    eng = ir_engine(m.blob, m.flags)
    a = frontier_case(oracle, eng, prog, m.flags, 20, 3000, width)
    assert a[0][11] == 0 and a[0][0] > 20
    b = frontier_case(oracle, ir_engine(m.blob, m.flags, ignore_timers=True), prog, m.flags, 20, 3000, width, ignore_timers=1)
    assert a == b                                                     # DPORwHeuristics never reads ignoreTimers
    found = frontier_case(oracle, eng, prog, m.flags, 24, 4000, width, looking_for=TWO_LEADERS)
    assert found[0][11] == 0


def test_election_frontier_exhaustive_set_parity(oracle):
    """trackHistory off, bounded-exhaustive: the wide search visits the set of schedules of the sequential one."""
    m = election_model()
    oracle.load_model(m.blob)
    prog = election_program(wait=False)
    rc, sr, sviol, shashes = oracle.dpor_search(N.MODEL_IR, D.pack_externals(prog), 9, 200000, 0, 0, -1, model_flags=m.flags,
                                                node_cap=1 << 16, explored_slots=1 << 22, heap_cap=1 << 22, cap_viol=100000)
    assert rc == 0 and sr["exhausted"] == 1
    eng = ir_engine(m.blob, m.flags)
    F = eng.frontier_params(9, 200000, 256, explored_slots=1 << 22, pool_cap=1 << 22)
    r, viol, hashes = eng.dpor_frontier(prog, F, cap_viol=100000)
    assert r["exhausted"] == 1 and r["status"] == 0
    assert set(int(x) for x in hashes) == set(int(x) for x in shashes)
    assert set(int(x) for x in viol["schedule_hash"]) == set(int(x) for x in sviol["schedule_hash"])
    frontier_case(oracle, eng, prog, m.flags, 12, 2000, 64, flags=N.FR_NO_HISTORY)


def test_generated_models_with_timers(oracle):
    """Every generated model of seeds 1..200 whose receive() has timer operations: nothing is declined, everything
    equals the oracle, and the replays really ran SCHED_ONCE, SCHED_REPEAT and CANCEL."""
    stats = {}
    counts = {"models": 0, "replay": 0, "ddmin": 0, "intmin": 0, "frontier": 0}
    for s in range(1, 201):
        m = ir_gen.generate(s)
        if not m.uses_timers:
            continue
        counts["models"] += 1
        oracle.load_model(m.blob)
        fprog = ir_gen.program(m, s, kills=False)
        fext = D.pack_externals(fprog)
        eng = ir_engine(m.blob, m.flags)
        res = oracle.fuzz_batch(N.MODEL_IR, fext, 1, 64, 40, 3, model_flags=m.flags)
        good = np.nonzero(res["status"] == 0)[0]
        if len(good):
            vi = np.nonzero((res["violation"] != 0) & (res["status"] == 0))[0]
            seed = 1 + int(vi[0] if len(vi) else good[0])
            ev, par, r = oracle.fuzz_trace(N.MODEL_IR, fext, seed, 40, 3, model_flags=m.flags)
            code = int(r["violation"])
            eng.set_trace(ev, fext)
            rng = np.random.default_rng(s)
            full = np.asarray(oracle.full_mask(fext), dtype=np.uint64).reshape(-1)
            masks = np.stack([full] + [full & rng.integers(0, 1 << 63, size=eng.mask_words(), dtype=np.uint64) for _ in range(15)])
            for fka in (0, 1):
                g = eng.replay_batch(masks, looking_for=code, flags=fka)
                c = oracle.replay_batch(N.MODEL_IR, ev, fext, masks, looking_for=code, flags=fka, model_flags=m.flags)
                assert not (g["status"] == N.RS_UNSUPPORTED).any(), (m, fka)
                assert (g == c).all(), (m, fka, np.nonzero(g != c)[0][:4])
                counts["replay"] += len(masks)
            try:
                _, _, irm = python_replay(m, ev, fext, full)
            except M.OperationLimit:
                irm = None
            for k in ("SCHED_ONCE", "SCHED_REPEAT", "CANCEL"):
                stats[k] = stats.get(k, 0) + (irm.stats.get(k, 0) if irm else 0)
            if code:
                rc, cmcs, total, citers, ver = oracle.ddmin_sts(N.MODEL_IR, ev, fext, code, model_flags=m.flags)
                try:
                    mcs, iters, dd = eng.ddmin(code)
                except D.DemiError as e:
                    assert rc != 0, (m, e.code)
                else:
                    assert rc == 0 and (mcs == cmcs).all() and dd.total_replays == total and list(iters) == list(citers), m
                    counts["ddmin"] += 1
                full_ev, _ = oracle.replay_trace(N.MODEL_IR, ev, fext, full, looking_for=code, model_flags=m.flags)
                if int(full_ev["violation"]) == code:
                    rc, cev2, ctotal, csizes, cunig = oracle.internal_minimize(N.MODEL_IR, ev, fext, code, model_flags=m.flags)
                    try:
                        gev, gsizes, gout = eng.internal_minimize(code)
                    except D.DemiError as e:
                        assert rc != 0, (m, e.code)
                    else:
                        assert rc == 0 and (gev == cev2).all() and list(gsizes) == list(csizes), m
                        counts["intmin"] += 1
        dprog = [e for e in fprog if type(e).__name__ in ("Start", "Send")][:m.n_actors + 4]
        for width in (1, 64):
            frontier_case(oracle, eng, dprog, m.flags, 12, 2000, width)
            counts["frontier"] += 1
        eng.close()
    assert counts["models"] >= 60 and counts["replay"] > 1000 and counts["frontier"] >= 120, counts
    assert counts["ddmin"] + counts["intmin"] > 0, counts
    assert all(stats.get(k, 0) > 0 for k in ("SCHED_ONCE", "SCHED_REPEAT", "CANCEL")), stats


def test_timer_set_capacity_edges(oracle):
    """16 registered repeating timers / 16 cancelled keys fit and the 17th is the queue-overflow status, at the same
    replay as on the oracle, in K2 and K3F; a registered key armed again at a full registry is no overflow; 80 distinct
    once-timers run through a table of 64 slots."""
    blob = edges_blob()
    eng = ir_engine(blob, DISTINCT)
    counts = [0, 1, 8, 15, 16, 17, 20]
    for kind in (ARM, DISARM):
        ext, ev = edges_recorded(oracle, kind, range(20))
        eng.set_trace(ev, ext)
        masks = prefix_masks(oracle, ext, counts)
        for fl in (0, N.RF_FILTER_KNOWN_ABSENTS):
            g = eng.replay_batch(masks, flags=fl)
            c = oracle.replay_batch(N.MODEL_IR, ev, ext, masks, flags=fl, model_flags=DISTINCT)
            assert (g == c).all(), (kind, fl, g, c)
            assert [int(x) for x in g["status"]] == [0, 0, 0, 0, 0, PS_QUEUE_OVF, PS_QUEUE_OVF]
        for k, want in ((16, 0), (17, DS_QUEUE_OVF)):
            got = frontier_case(oracle, eng, edges_program(kind, range(k), wait=False), DISTINCT, 40, 20, 1)
            assert (got[0] if want else got[0][11]) == want, (kind, k)
    for ks, maxm in ((list(range(16)) + [3, 15, 0], 60), (list(range(80)), 400)):
        kind = ARM if maxm == 60 else ONCE
        ext, ev = edges_recorded(oracle, kind, ks, maxm=maxm)
        eng.set_trace(ev, ext)
        full = np.asarray(oracle.full_mask(ext), dtype=np.uint64).reshape(-1)
        r, rec = eng.replay_trace(full)
        rc, crec = oracle.replay_trace(N.MODEL_IR, ev, ext, full, model_flags=DISTINCT)
        assert r == rc and rows(rec) == rows(crec) and int(r["status"]) == 0
        g = eng.replay_batch(random_masks(ext, 32, 3))
        assert (g == oracle.replay_batch(N.MODEL_IR, ev, ext, random_masks(ext, 32, 3), model_flags=DISTINCT)).all()
    assert int(r["delivered"]) == 120
    got = frontier_case(oracle, eng, edges_program(ONCE, range(80), wait=False), DISTINCT, 200, 6, 1)
    assert got[0][11] == 0


def test_election_frontier_on_two_ranks(oracle):
    """demi_dpor_frontier_multi on a loaded model with timers: every rank equals the simulated protocol's."""
    import ctypes as C
    L = N.lib()
    n = 2
    if L.demi_device_count() < n:
        pytest.skip("needs %d GPUs" % n)
    m = election_model()
    oracle.load_model(m.blob)
    cfg = N.Config(0, N.MODEL_IR, m.flags, 0, 0, 0)
    devs = (C.c_int32 * n)(*range(n))
    hs = (C.c_void_p * n)()
    assert L.demi_create_multi(C.byref(cfg), devs, n, hs) == 0, L.demi_last_error(None)
    for i in range(n):
        assert L.demi_load_model(hs[i], bytes(m.blob), len(m.blob)) == 0, L.demi_last_error(hs[i])
    kw = dict(explored_slots=1 << 18, pool_cap=1 << 20, rounds_per_exchange=2, steal_max=128)
    F = D.Engine.frontier_params(14, 3000, 32, **kw)
    ext = D.pack_externals(election_program(wait=False))
    cap_viol, cap_h = 4096, int(F.max_interleavings) + int(F.width) + 1
    res = np.zeros(n, dtype=N.FRONTIER_RESULT_DTYPE)
    viol = np.zeros((n, cap_viol), dtype=N.DPOR_VIOL_DTYPE)
    hashes = np.zeros((n, cap_h), dtype=np.uint64)
    rc = L.demi_dpor_frontier_multi(hs, n, ext.ctypes.data, len(ext), C.byref(F), res.ctypes.data, viol.ctypes.data, cap_viol,
                                    hashes.ctypes.data, cap_h)
    err = [L.demi_last_error(hs[i]) for i in range(n)]
    for i in range(n):
        L.demi_destroy(hs[i])
    assert rc == 0, err
    OF = oracle.frontier_params(14, 3000, 32, **kw)
    orc, ores, oviol, ohashes = oracle.dpor_frontier(N.MODEL_IR, ext, OF, n, model_flags=m.flags)
    assert orc == 0
    for r in range(n):
        for f in MULTI_FIELDS:
            assert res[r][f] == ores[r][f], (r, f, res[r], ores[r])
        assert (hashes[r, :int(res[r]["interleavings"])] == ohashes[r]).all()
        assert (viol[r, :int(res[r]["violations"])] == oviol[r]).all()
    assert (res["interleavings"] > 0).all()
