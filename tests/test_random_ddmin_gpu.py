"""DDMin with RandomScheduler as the TestOracle on the device (demi_random_test_batch / demi_random_ddmin), bit for bit
against the C oracle (oracle/random_ddmin.c)."""
import ctypes as C
import os

import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
from test_random_ddmin_oracle import CASES, PP_FLAGS, RAFT_FLAGS, atoms_cover, bits, _oracle_cfg

pytestmark = pytest.mark.gpu
FIELDS = ("first_hit", "executions_run", "violation", "status")


@pytest.fixture(scope="module")
def rd():
    from demi_b200 import build
    build.build_oracle()
    from oracle import random_ddmin_binding
    random_ddmin_binding.lib()
    return random_ddmin_binding


def engine(model, flags, c, lane_cap=None):
    if lane_cap is not None:
        os.environ["DEMI_LANE_PENDING_CAP"] = str(lane_cap)
    try:
        eng = D.Engine(D.SchedulerConfig(model, flags, blocked_mask=_oracle_cfg(c)["blocked_mask"],
                                         strategy=c.get("strategy", 0)))
    finally:
        os.environ.pop("DEMI_LANE_PENDING_CAP", None)
    if c.get("rules"):
        eng.set_user_filter(c["rules"])
    return eng


def rows(recs):
    return [tuple(int(r[f]) for f in FIELDS) for r in recs]


def random_masks(n_ext, n, rng):
    ms = [sorted(int(i) for i in np.nonzero(rng.random(n_ext) < p)[0]) for p in rng.uniform(0.3, 0.95, n)]
    ms += [[i for i in range(n_ext) if i != k] for k in range(n_ext)] + [list(range(n_ext)), []]
    return np.stack([bits(m, n_ext) for m in ms])


def batch_case(rd, model, flags, prog, maxm, interval, n, seed, c, looking=0, lane_cap=None, eng=None):
    eng = eng or engine(model, flags, c, lane_cap)
    eng.set_externals(prog)
    masks = random_masks(len(prog), 60, np.random.default_rng(seed))
    got = eng.random_test_batch(masks, n, seed, maxm, interval, looking)
    rd.set_user_filter(c.get("rules", []))
    try:
        want = rd.random_test_batch(model, D.pack_externals(prog), masks, n, seed, maxm, interval, looking_for=looking,
                                    model_flags=flags, **_oracle_cfg(c))
    finally:
        rd.set_user_filter([])
    assert rows(got) == rows(want)
    return got, eng


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_batch_matches_the_oracle(rd, case):
    name, model, flags, prog, maxm, interval, n, seed, c = case
    got, eng = batch_case(rd, model, flags, prog, maxm, interval, n, seed, c)
    assert (got["first_hit"] > 0).any() or model == N.MODEL_PINGPONG3
    batch_case(rd, model, flags, prog, maxm, interval, 64, seed + 1, c, eng=eng)
    # executions deferred from the lane engine to the warp engine (a tiny lane pending cap) give the same records
    if not c and not any(isinstance(e, D.HardKill) for e in prog):      # HardKill programs run on the warp engine alone
        eng2 = engine(model, flags, c, lane_cap=6)
        batch_case(rd, model, flags, prog, maxm, interval, 64, seed + 1, c, eng=eng2)
        assert eng2.stats().deferred > 0


def test_bcast32_batch(rd):
    prog = D.bcast32_program(ttl=3)[:-1] + [D.WaitQuiescence(), D.Send(5, 2, 2), D.WaitQuiescence()]
    batch_case(rd, N.MODEL_BCAST32, 0, prog, 200, 0, 16, 3, {})


def test_generated_models_with_capacity_statuses(rd):
    """Loaded models: the records equal the oracle's, statuses included."""
    import ir_gen
    from oracle import random_ddmin_binding
    statuses = 0
    for s in range(1, 13):
        m = ir_gen.generate(s)
        random_ddmin_binding.load_model(m.blob)
        eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, m.flags))
        eng.load_model(m.blob)
        got, _ = batch_case(rd, N.MODEL_IR, m.flags, ir_gen.program(m, s, hard_kill=(s % 3 == 1)), 40, 2, 16, s, {}, eng=eng)
        statuses += int((got["status"] != 0).sum())
    assert statuses > 0


def test_seeds_j_and_j_plus_1_differ(rd):
    """Execution j runs FullyRandom(seed + j): shifting the seed base by one changes some records, and both agree."""
    name, model, flags, prog, maxm, interval, n, seed, c = CASES[0]
    a, eng = batch_case(rd, model, flags, prog, maxm, interval, 4, seed, c)
    b, _ = batch_case(rd, model, flags, prog, maxm, interval, 4, seed + 1, c, eng=eng)
    assert rows(a) != rows(b)


def test_all_ones_first_hit_is_explores_first_violation():
    name, model, flags, prog, maxm, interval, n, seed, c = CASES[0]
    sched = D.RandomScheduler(D.SchedulerConfig(model, flags), max_executions=64, invariant_check_interval=interval, seed=seed)
    sched.setMaxMessages(maxm)
    assert sched.explore(prog) is not None
    first = int(np.nonzero(sched.last_results["violation"])[0][0])
    sched.engine.set_externals(prog)
    r = sched.engine.random_test_batch(bits(range(len(prog)), len(prog)), 64, seed, maxm, interval)[0]
    assert int(r["first_hit"]) == first and int(r["executions_run"]) == first + 1


def ddmin_case(rd, model, flags, prog, maxm, interval, n, seed, c, eng=None):
    eng = eng or engine(model, flags, c)
    rd.set_user_filter(c.get("rules", []))
    try:
        ext = D.pack_externals(prog)
        full = rd.random_test_batch(model, ext, bits(range(len(prog)), len(prog)), 64, seed, maxm, interval, model_flags=flags,
                                    **_oracle_cfg(c))[0]
        looking = int(full["violation"])
        want = rd.random_ddmin(model, ext, n, seed, maxm, looking, interval, model_flags=flags, **_oracle_cfg(c))
    finally:
        rd.set_user_filter([])
    eng.set_externals(prog)
    if want["rc"] == -4:
        with pytest.raises(D.DemiError) as ei:
            eng.random_ddmin(n, seed, maxm, looking, interval)
        assert ei.value.code == N.ERR_CAPACITY
        return None
    assert want["rc"] == 0
    mcs, sizes, keys, out = eng.random_ddmin(n, seed, maxm, looking, interval)
    assert list(mcs) == list(want["mcs"])
    assert out.tests == len(want["tests"]) and out.total_replays == want["total_replays"]
    assert list(sizes) == list(want["sizes"]) and list(keys) == list(want["keys"])
    assert out.verified == want["verified"] and out.mcs_size == sum(bin(int(w)).count("1") for w in mcs)
    assert out.tests_evaluated >= out.tests and out.executions_executed >= 1
    return out


@pytest.mark.parametrize("n", [1, 64])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_whole_minimization_matches_the_oracle(rd, case, n):
    name, model, flags, prog, maxm, interval, _, seed, c = case
    ddmin_case(rd, model, flags, prog, maxm, interval, n, seed, c)


def test_generated_models_whole_minimization(rd):
    import ir_gen
    from oracle import random_ddmin_binding
    done = 0
    for s in range(1, 30):
        m = ir_gen.generate(s)
        prog = ir_gen.program(m, s)
        if not atoms_cover(prog):
            continue
        random_ddmin_binding.load_model(m.blob)
        eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, m.flags))
        eng.load_model(m.blob)
        full = rd.random_test_batch(N.MODEL_IR, D.pack_externals(prog), bits(range(len(prog)), len(prog)), 64, s, 40, 2,
                                    model_flags=m.flags)[0]
        if not full["violation"]:
            continue
        ddmin_case(rd, N.MODEL_IR, m.flags, prog, 40, 2, 16, s, {}, eng=eng)
        done += 1
    assert done >= 3


def test_rejected_inputs():
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, RAFT_FLAGS))
    L = N.lib()
    p = N.FuzzParams(0, 8, 50, 5, 0, 0)
    masks = np.zeros(4, dtype=np.uint64)
    out = np.zeros(4, dtype=N.RANDOM_TEST_DTYPE)
    rout = N.RandomDDMinOut()
    mcs = np.zeros(4, dtype=np.uint64)
    assert L.demi_random_test_batch(eng._h, masks.ctypes.data, 1, 1, C.byref(p), out.ctypes.data) == N.ERR_STATE
    assert L.demi_random_ddmin(eng._h, C.byref(p), 0, mcs.ctypes.data, 1, None, None, 0, C.byref(rout)) == N.ERR_STATE
    eng.set_externals(D.raft5_program(client_cmds=60))                   # 71 events: 2 mask words
    assert L.demi_random_test_batch(eng._h, masks.ctypes.data, 1, 1, C.byref(p), out.ctypes.data) == N.ERR_INVALID
    assert L.demi_random_ddmin(eng._h, C.byref(p), 0, mcs.ctypes.data, 1, None, None, 0, C.byref(rout)) == N.ERR_INVALID
    p0 = N.FuzzParams(0, 0, 50, 5, 0, 0)
    assert L.demi_random_test_batch(eng._h, masks.ctypes.data, 1, 2, C.byref(p0), out.ctypes.data) == N.ERR_INVALID
    assert L.demi_random_ddmin(eng._h, C.byref(p0), 0, mcs.ctypes.data, 2, None, None, 0, C.byref(rout)) == N.ERR_INVALID
    assert L.demi_random_test_batch(eng._h, masks.ctypes.data, 1, 2, None, out.ctypes.data) == N.ERR_INVALID
    assert L.demi_random_test_batch(eng._h, masks.ctypes.data, 1, 2, C.byref(p), None) == N.ERR_INVALID
    assert L.demi_random_ddmin(eng._h, C.byref(p), 0, None, 2, None, None, 0, C.byref(rout)) == N.ERR_INVALID
    assert L.demi_random_ddmin(eng._h, C.byref(p), 0, mcs.ctypes.data, 2, None, None, 0, None) == N.ERR_INVALID


PP_HK = D.pingpong3_program(n_sends=6)[:-1] + [D.WaitQuiescence(), D.HardKill(1), D.Send(0, 1, 50), D.Send(2, 1, 51),
                                               D.WaitQuiescence()]


def test_hard_kill_violation_minimizes_end_to_end(rd):
    """A violation RandomScheduler.explore finds on a program with HardKill (which STSSched replay and DPOR reject)
    minimizes through randomDDMin, and the result equals the oracle's.  (pingpong3 quiesces, so the invariant is checked
    at the end of each execution under randomDDMin's interval 0.)"""
    assert atoms_cover(PP_HK)
    cfg = D.SchedulerConfig(N.MODEL_PINGPONG3, PP_FLAGS)
    sched = D.RandomScheduler(cfg, max_executions=64, invariant_check_interval=0, seed=7)
    found = sched.explore(PP_HK)
    assert found is not None
    trace, violation = found
    mcs, stats, verified, v = D.randomDDMin(cfg, trace, PP_HK, violation, stats=D.MinimizationStats(), max_executions=16, seed=7)
    assert v == violation and 0 < len(mcs) < len(PP_HK)
    want = rd.random_ddmin(N.MODEL_PINGPONG3, D.pack_externals(PP_HK), 16, 7, len(trace), violation, 0, model_flags=PP_FLAGS)
    assert want["rc"] == 0
    assert (verified is not None) == bool(want["verified"])           # verify_mcs: None when the MCS does not reproduce
    assert [PP_HK.index(e) for e in mcs] == [i for i in range(len(PP_HK)) if (int(want["mcs"][0]) >> i) & 1]
    assert stats.total_replays == want["total_replays"]
    assert stats.inner().iterationSize == {int(k): int(v) for k, v in zip(want["keys"], want["sizes"])}   # keyed by executions
    # the DDMin front end over a RandomScheduler oracle gives the same MCS
    sched2 = D.RandomScheduler(cfg, max_executions=16, seed=7)
    sched2.setMaxMessages(len(trace))
    assert D.DDMin(sched2).minimize(violation, PP_HK) == mcs


def _closure(prog):
    """Every test DDMin's decision tree over `prog` can ask for (both halves of every frame, with every remainder the
    recursion and the interference step give): what the first speculative batch holds when it fits."""
    import micro_oracle as M
    from test_micro_oracle import to_prog
    mp = list(enumerate(to_prog(prog)))
    seen, tests, stack = set(), set(), [(tuple(range(len(prog))), ())]
    while stack:
        dag, rem = stack.pop()
        if (dag, rem) in seen:
            continue
        seen.add((dag, rem))
        atoms = M.atomic_events([mp[i] for i in dag])
        if len(atoms) <= 1:
            continue
        h = [tuple(sorted(x[0] for a in chunk for x in a)) for chunk in M.split_list(atoms, 2)]
        for k in (0, 1):
            tests.add(tuple(sorted(set(h[k]) | set(rem))))
        stack += [(h[0], rem), (h[1], rem), (h[0], tuple(sorted(set(h[1]) | set(rem)))),
                  (h[1], tuple(sorted(set(h[0]) | set(rem))))]
    return sorted(tests)


def test_speculative_only_status_does_not_fail_the_call(rd):
    """A loaded model whose DDMin tree holds tests with capacity statuses that the sequential walk never consumes: the
    oracle's walk succeeds, the engine evaluates those tests speculatively (its one batch is the whole tree) and still
    returns the oracle's minimization."""
    import ir_gen
    from oracle import random_ddmin_binding
    s, maxm, n = 210, 40, 16
    m = ir_gen.generate(s)
    prog = ir_gen.program(m, s)
    assert atoms_cover(prog)
    random_ddmin_binding.load_model(m.blob)
    ext = D.pack_externals(prog)
    looking = int(rd.random_test_batch(N.MODEL_IR, ext, bits(range(len(prog)), len(prog)), n, s, maxm, 2,
                                       model_flags=m.flags)[0]["violation"])
    assert looking
    want = rd.random_ddmin(N.MODEL_IR, ext, n, s, maxm, looking, 2, model_flags=m.flags)
    assert want["rc"] == 0 and all(int(r["status"]) == 0 for r in want["records"])
    tree = _closure(prog)
    masks = np.stack([bits(t, len(prog)) for t in tree])
    eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, m.flags))
    eng.load_model(m.blob)
    eng.set_externals(prog)
    recs = eng.random_test_batch(masks, n, s, maxm, 2, looking)
    assert (recs["status"] != 0).sum() > 0                        # tests with a status are in the tree ...
    mcs, sizes, keys, out = eng.random_ddmin(n, s, maxm, looking, 2)
    assert out.batches == 1 and out.tests_evaluated == len(tree)  # ... and were evaluated speculatively
    assert list(mcs) == list(want["mcs"]) and out.total_replays == want["total_replays"]
    assert list(sizes) == list(want["sizes"]) and list(keys) == list(want["keys"])


def test_subsequence_trace_accepts_adjacent_wait_quiescence(rd, oracle):
    """demi_random_test_trace records a subsequence that demi_set_externals would reject (adjacent, leading and
    trailing WaitQuiescence), event for event as the oracle records it; the handle's program is unchanged."""
    name, model, flags, prog, maxm, interval, n, seed, c = CASES[0]
    eng = engine(model, flags, c)
    eng.set_externals(prog)
    wq = [i for i, e in enumerate(prog) if isinstance(e, D.WaitQuiescence)]
    keeps = [[i for i in range(len(prog)) if not wq[1] < i < wq[2]],                     # adjacent
             [i for i in range(len(prog)) if not (wq[2] < i < wq[3] or wq[1] < i < wq[2])],
             [0] + list(range(1, 6)) + wq[1:]]                                          # leading, adjacent, trailing
    for keep in keeps:
        kinds = [type(prog[i]).__name__ for i in keep]
        assert any(a == b == "WaitQuiescence" for a, b in zip(kinds, kinds[1:]))
        sub = [prog[i] for i in keep]
        for s in (seed, seed + 3):
            r, ev = eng.random_test_trace(bits(keep, len(prog)), s, maxm, interval)
            want_ev, _, want_r = oracle.fuzz_trace(model, D.pack_externals(sub), s, maxm, interval, model_flags=flags)
            assert [tuple(e) for e in ev] == [tuple(e) for e in want_ev]
            assert (int(r["violation"]), int(r["steps"]), int(r["status"])) == \
                   (int(want_r["violation"]), int(want_r["steps"]), int(want_r["status"]))
    with pytest.raises(D.DemiError):
        eng.set_externals([prog[i] for i in keeps[0]])          # the rule of demi_set_externals is unchanged
    assert len(eng.random_test_batch(bits(range(len(prog)), len(prog)), 2, seed, maxm, interval)) == 1


def test_many_launches_per_call(rd):
    """N = 2^21: two tests per launch, so the call runs its masks in several launches (mask and record offsets, the
    first_hit words reset per launch).  Each record equals the one the mask gives alone, and the oracle's where the
    first hit is below 64."""
    name, model, flags, prog, maxm, interval, n, seed, c = CASES[0]
    eng = engine(model, flags, c)
    eng.set_externals(prog)
    keeps = [list(range(len(prog)))] + [[i for i in range(len(prog)) if i != k] for k in range(0, len(prog), 2)] + [[]]
    masks = np.stack([bits(k, len(prog)) for k in keeps])
    big = 1 << 21
    got = eng.random_test_batch(masks, big, seed, maxm, interval)
    assert eng.stats().kernel_launches > 4
    for k in range(len(masks)):
        assert rows(got[k:k + 1]) == rows(eng.random_test_batch(masks[k:k + 1], big, seed, maxm, interval))
    small = rd.random_test_batch(model, D.pack_externals(prog), masks, 64, seed, maxm, interval, model_flags=flags)
    for g, w in zip(got, small):
        if 0 <= int(w["first_hit"]):
            assert (int(g["first_hit"]), int(g["violation"])) == (int(w["first_hit"]), int(w["violation"]))
    assert (got["first_hit"] < 0).any() and (got["first_hit"] >= 0).any()
