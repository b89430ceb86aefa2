"""demi_incremental_ddmin_many (IncrementalDDMin over ResumableDPOR for many violating executions, their DPOR tests in
shared K3 launches) and demi_fuzz_traces_tree (the batched recording that returns each execution's DepTracker tree):
every trace equals demi_incremental_ddmin on that trace alone in every field, and oracle_incremental_ddmin in MCS,
replays, rounds and instances; results do not depend on the set, its order, the window or how a round is split into
launches; a trace that fails does so alone."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import model_ir, _native as N
from test_ir_dpor_oracle import ELECTION_SEEDS, PP_CODE, PP_FLAGS, election_recorded, pingpong_program
from test_ir_timers_oracle import TWO_LEADERS, election_model, election_program

pytestmark = pytest.mark.gpu

FIELDS = ("mcs_size", "total_replays", "rounds", "instances", "tests_executed", "batches", "interleavings_executed")
ALL_FLAGS = N.DF_ARVIND_ORDERING | N.DF_PRIORITIZE_PENDING
BUDGET = 300


def dpor_ext(prog):
    ext = D.pack_externals(prog)
    return ext[(ext["kind"] == N.EXT_START) | (ext["kind"] == N.EXT_SEND)]


@pytest.fixture(scope="module")
def raft():
    """Violating raft5 executions recorded by demi_fuzz_traces_tree, each row and tree checked against demi_fuzz_trace."""
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    eng.set_externals(D.raft5_program())
    res = eng.fuzz_batch(1, 4000, 40, 5)
    viol = np.nonzero((res["violation"] == 1) & (res["status"] == 0))[0][:10]
    assert len(viol) == 10
    ev, ne, par, nn, rr = eng.fuzz_traces_tree(1, viol, 40, 5, cap_events=1024, cap_nodes=1024)
    recs = []
    for i, k in enumerate(viol):
        sev, spar, sr = eng.fuzz_trace(1 + int(k), 40, 5, cap_events=1024, cap_nodes=1024)
        assert ne[i] == len(sev) and np.array_equal(ev[i, :ne[i]], sev), i
        assert nn[i] == len(spar) and np.array_equal(par[i, :nn[i]], spar), i
        assert rr[i] == sr
        recs.append((ev[i, :ne[i]].copy(), par[i, :nn[i]].copy(), int(rr[i]["steps"])))
    return eng, dpor_ext(D.raft5_program()), recs


def solo(eng, prog, maxm, seed, looking_for, flags, **kw):
    mcs, out = eng.incremental_ddmin(prog, maxm, kw.pop("budget", BUDGET), seed, looking_for=looking_for, flags=flags, **kw)
    return mcs, out


def assert_same(mcs_m, out_m, mcs_s, out_s, what):
    n = len(mcs_s)
    assert np.array_equal(mcs_m[:n], mcs_s) and not mcs_m[n:].any(), what
    for f in FIELDS:
        assert int(out_m[f]) == int(getattr(out_s, f)), (what, f)


def run_set(eng, progs, maxms, seeds, looking_for, flags, **kw):
    kw.setdefault("heap_cap", 1 << 16)
    return eng.incremental_ddmin_many(progs, maxms, kw.pop("budget", BUDGET), seeds, looking_for=looking_for, flags=flags,
                                      max_max_distance=64, stop_at_size=1, **kw)


@pytest.mark.parametrize("flags", [ALL_FLAGS, N.DF_PRIORITIZE_PENDING, 0])
def test_mixed_set_equals_single_calls(raft, flags):
    """Per-trace programs and max_messages: every trace equals its single call in every field."""
    eng, dext, recs = raft
    rng = np.random.default_rng(flags)
    progs, maxms, seeds = [], [], []
    for t, (ev, par, steps) in enumerate(recs):
        keep = np.ones(len(dext), dtype=bool)
        if t % 3 == 1:
            keep[rng.integers(0, len(dext), size=2)] = False
        progs.append(dext[keep])
        maxms.append(steps + (t % 4))
        seeds.append((ev, par))
    mcs, out, status = run_set(eng, progs, maxms, seeds, 1, flags)
    assert (status == 0).all()
    for t in range(len(recs)):
        ms, os_ = solo(eng, progs[t], maxms[t], seeds[t], 1, flags, max_max_distance=64, stop_at_size=1, heap_cap=1 << 16)
        assert_same(mcs[t], out[t], ms, os_, t)


def test_raft5_set_matches_the_oracle(raft, oracle):
    eng, dext, recs = raft
    mcs, out, status = run_set(eng, dext, [r[2] for r in recs], [(r[0], r[1]) for r in recs], 1, ALL_FLAGS)
    assert (status == 0).all()
    for t, (ev, par, steps) in enumerate(recs):
        rc, mcs_o, st = oracle.incremental_ddmin(N.MODEL_RAFT5, dext, steps, BUDGET, oracle.dpor_seed(ev, par), model_flags=1,
                                                 looking_for=1, stop_at_size=1, max_max_distance=64)
        assert rc == 0
        assert np.array_equal(mcs[t, :len(mcs_o)], mcs_o), t
        assert (int(out[t]["total_replays"]), int(out[t]["rounds"]), int(out[t]["instances"])) == \
            (st["total_replays"], st["rounds"], st["instances"]), t


def test_subsets_permutations_window_and_split(raft, monkeypatch):
    """The same traces in a subset, in another order, with one driver in flight, and with a footprint that forces more
    than one launch per round: every trace's outputs are unchanged."""
    eng, dext, recs = raft
    maxms, seeds = [r[2] for r in recs], [(r[0], r[1]) for r in recs]
    mcs, out, status = run_set(eng, dext, maxms, seeds, 1, ALL_FLAGS)
    assert (status == 0).all()
    base_launches = eng.stats().kernel_launches
    perm = np.random.default_rng(3).permutation(len(recs))
    for idx in (perm, perm[:4], np.array([7, 2])):
        m2, o2, s2 = run_set(eng, dext, [maxms[i] for i in idx], [seeds[i] for i in idx], 1, ALL_FLAGS)
        assert (s2 == 0).all()
        for j, i in enumerate(idx):
            assert np.array_equal(m2[j], mcs[i]) and o2[j] == out[i], (idx, i)
    monkeypatch.setenv("DEMI_DDMIN_MANY_WINDOW", "1")
    m2, o2, s2 = run_set(eng, dext, maxms, seeds, 1, ALL_FLAGS)
    assert (s2 == 0).all() and np.array_equal(m2, mcs) and (o2 == out).all()
    monkeypatch.delenv("DEMI_DDMIN_MANY_WINDOW")
    # 2^26 explored slots: 512 MiB per search, so a launch holds at most a few dozen searches
    m3, o3, s3 = run_set(eng, dext, maxms, seeds, 1, ALL_FLAGS, explored_slots=1 << 26)
    assert (s3 == 0).all()
    split_launches = eng.stats().kernel_launches
    ms, os_ = solo(eng, dext, maxms[0], seeds[0], 1, ALL_FLAGS, max_max_distance=64, stop_at_size=1, heap_cap=1 << 16,
                   explored_slots=1 << 26)
    assert_same(m3[0], o3[0], ms, os_, "split")
    assert np.array_equal(m3, mcs) and (o3 == out).all()
    assert split_launches > base_launches, (split_launches, base_launches)


def solo_or_code(eng, prog, maxm, seed, **kw):
    try:
        return 0, solo(eng, prog, maxm, seed, 1, ALL_FLAGS, max_max_distance=64, stop_at_size=1, **kw)
    except D.DemiError as e:
        return e.code, None


def check_against_solo(eng, progs, maxms, seeds, **kw):
    kw.setdefault("heap_cap", 1 << 16)
    mcs, out, status = run_set(eng, progs, maxms, seeds, 1, ALL_FLAGS, **dict(kw))
    for t in range(len(progs)):
        code, got = solo_or_code(eng, progs[t], maxms[t], seeds[t], **kw)
        assert int(status[t]) == code, (t, int(status[t]), code)
        if code == 0:
            assert_same(mcs[t], out[t], got[0], got[1], t)
    return status


def test_failures_stay_with_their_trace(raft):
    """A Kill external (DEMI_ERR_INVALID), a seed over node_cap and a heap too small for a search (DEMI_ERR_CAPACITY)
    fail their own trace; the others equal their single calls and the call returns OK."""
    eng, dext, recs = raft
    maxms = [r[2] for r in recs[:4]]
    seeds = [(r[0], r[1]) for r in recs[:4]]
    kill = np.concatenate([dext, D.pack_externals([D.Kill(0)])])
    status = check_against_solo(eng, [dext, kill, dext, dext], maxms, seeds)
    assert list(status) == [0, N.ERR_INVALID, 0, 0]
    sizes = sorted(len(s[1]) for s in seeds)
    status = check_against_solo(eng, [dext] * 4, maxms, seeds, node_cap=sizes[-1] - 1)
    assert N.ERR_CAPACITY in list(status)
    # a 24-entry heap: the full program's search overflows it, a three-external one with few messages does not
    status = check_against_solo(eng, [dext, dext[:3], dext], [maxms[0], 3, maxms[2]], seeds[:3], heap_cap=24)
    assert N.ERR_CAPACITY in list(status)


def test_election_with_timers(oracle):
    m = election_model()
    eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, model_flags=m.flags))
    eng.load_model(m.blob)
    dext = D.pack_externals(election_program(wait=False))
    recs = [election_recorded(oracle, s) for s in ELECTION_SEEDS]
    mcs, out, status = eng.incremental_ddmin_many(dext, [r[2] for r in recs], 60, [(r[0], r[1]) for r in recs],
                                                  looking_for=TWO_LEADERS, max_max_distance=64, stop_at_size=1,
                                                  heap_cap=1 << 16)
    assert (status == 0).all()
    for t, (ev, par, steps, _) in enumerate(recs):
        ms, os_ = eng.incremental_ddmin(dext, steps, 60, (ev, par), looking_for=TWO_LEADERS, max_max_distance=64,
                                        stop_at_size=1, heap_cap=1 << 16)
        assert_same(mcs[t], out[t], ms, os_, t)
        rc, mcs_o, st = oracle.incremental_ddmin(N.MODEL_IR, dext, steps, 60, oracle.dpor_seed(ev, par), max_max_distance=64,
                                                 stop_at_size=1, looking_for=TWO_LEADERS, model_flags=m.flags)
        assert rc == 0 and np.array_equal(mcs[t], mcs_o)
        assert (int(out[t]["total_replays"]), int(out[t]["rounds"]), int(out[t]["instances"])) == \
            (st["total_replays"], st["rounds"], st["instances"])
    eng.close()


def test_loaded_pingpong3(oracle):
    blob = model_ir.pingpong3_blob()
    eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, model_flags=PP_FLAGS))
    eng.load_model(blob)
    pext = D.pack_externals(pingpong_program())
    fext = D.pack_externals(pingpong_program(wait=True))
    oracle.load_model(blob)
    recs = []
    for seed in (1, 2, 4):
        ev, par, r = oracle.fuzz_trace(N.MODEL_IR, fext, seed, 30, 1, model_flags=PP_FLAGS)
        recs.append((ev, par, int(r["steps"])))
    mcs, out, status = eng.incremental_ddmin_many(pext, [r[2] for r in recs], 200, [(r[0], r[1]) for r in recs],
                                                  looking_for=PP_CODE, max_max_distance=16, stop_at_size=1, heap_cap=1 << 16)
    assert (status == 0).all()
    for t, (ev, par, steps) in enumerate(recs):
        ms, os_ = eng.incremental_ddmin(pext, steps, 200, (ev, par), looking_for=PP_CODE, max_max_distance=16, stop_at_size=1,
                                        heap_cap=1 << 16)
        assert_same(mcs[t], out[t], ms, os_, t)
        rc, mcs_o, st = oracle.incremental_ddmin(N.MODEL_IR, pext, steps, 200, oracle.dpor_seed(ev, par), max_max_distance=16,
                                                 stop_at_size=1, looking_for=PP_CODE, model_flags=PP_FLAGS)
        assert rc == 0 and np.array_equal(mcs[t], mcs_o)
        assert int(out[t]["total_replays"]) == st["total_replays"] and int(out[t]["instances"]) == st["instances"]
    eng.close()


def test_minimize_many_host_class(raft):
    """IncrementalDDMin.minimize_many: one MCS per execution, each what minimize() returns for it."""
    eng, dext, recs = raft
    prog = [e for e in D.raft5_program() if e.kind in (N.EXT_START, N.EXT_SEND)]
    cfg = D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1)
    ev, par, steps = recs[0]
    oracle = D.ResumableDPOR(cfg, ev, par, max_messages=steps, max_interleavings=BUDGET, engine=eng)
    ddmin = D.IncrementalDDMin(oracle, maxMaxDistance=64, stopAtSize=1)
    got = ddmin.minimize_many([(prog, r[0], r[1], r[2]) for r in recs[:3]], 1)
    for t, (ev, par, steps) in enumerate(recs[:3]):
        o = D.ResumableDPOR(cfg, ev, par, max_messages=steps, max_interleavings=BUDGET, engine=eng)
        want = D.IncrementalDDMin(o, maxMaxDistance=64, stopAtSize=1).minimize(prog, 1)
        assert [e._id for e in got[t]] == [e._id for e in want], t
