"""K3 on loaded models: DPOR batches (demi_dpor_batch / demi_dpor_batch_ex) and IncrementalDDMin
(demi_incremental_ddmin) of a model loaded with demi_load_model, against the C oracle, every field bit-exact — on the
loaded pingpong3 (also against compiled K3 pingpong3), on the leader election of tests/test_ir_timers_oracle.py, whose
timers are armed, fired and cancelled inside the searches, on the generated models of tests/ir_gen.py that use
timers, and at the timer-set and operation-limit capacity edges.  No answer may be DEMI_DS_UNSUPPORTED."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import model_ir, _native as N
import ir_gen
from test_dpor_gpu import FIELDS
from test_ir_dpor_oracle import ELECTION_SEEDS, PP_CODE, PP_FLAGS, SHRINKING_SEED, election_recorded, pingpong_program
from test_ir_timers_oracle import (ARM, DISARM, DISTINCT, DS_QUEUE_OVF, KICK, ONCE, TWO_LEADERS, edges_blob, edges_program,
                                   election_model, election_program)
from test_model_ir_random import _fanout_model

pytestmark = pytest.mark.gpu
DS_UNSUPPORTED = 6
CAPS = [0, 2, 4, 8, 16, -1]


def ir_engine(blob, flags):
    eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, model_flags=flags))
    eng.load_model(blob)
    return eng


def check(oracle, eng, model, progs, maxm, maxi, flags, looking_for=0, stop=False, depth_bound=-1, blob=None, cap_viol=32,
          node_cap=4096, explored_slots=1 << 16, heap_cap=1 << 15):
    """One K3 launch of every program against oracle_dpor_search per program: results, schedule hashes, violations."""
    res, viol, hashes = eng.dpor_batch(progs, maxm, maxi, looking_for, stop, depth_bound, node_cap=node_cap,
                                       explored_slots=explored_slots, heap_cap=heap_cap, cap_viol=cap_viol, want_hashes=True)
    if blob is not None:
        oracle.load_model(blob)
    for s, prog in enumerate(progs):
        rc, r, cviol, chashes = oracle.dpor_search(model, D.pack_externals(prog), maxm, maxi, looking_for, 1 if stop else 0,
                                                    depth_bound, model_flags=flags, node_cap=node_cap,
                                                    explored_slots=explored_slots, heap_cap=heap_cap, cap_viol=cap_viol)
        for f in FIELDS:
            assert res[s][f] == r[f], (s, f, res[s], r)
        assert (hashes[s][:int(r["interleavings"])] == chashes).all(), s
        nv = min(int(r["violations"]), cap_viol)
        assert (viol[s][:nv] == cviol[:nv]).all(), s
    assert not (res["status"] == DS_UNSUPPORTED).any()
    return res, viol, hashes


def test_pingpong3_blob_equals_oracle_and_compiled_k3(oracle):
    """The loaded pingpong3 through K3: every result field, schedule hash and violation record equals the oracle's on
    the loaded model and compiled K3 pingpong3's, with and without looking_for / stopIfViolationFound / a depth
    bound, and at a depth whose scan table no longer fits in shared memory (max_messages 40)."""
    blob = model_ir.pingpong3_blob()
    rng = np.random.default_rng(11)
    progs = [pingpong_program()] + [pingpong_program(tuple(int(x) for x in rng.integers(0, 3, size=int(rng.integers(2, 7)))))
                                    for _ in range(39)]
    ir = ir_engine(blob, PP_FLAGS)
    compiled = D.Engine(D.SchedulerConfig(N.MODEL_PINGPONG3, model_flags=PP_FLAGS))
    found = 0
    for maxm, looking_for, stop, depth in ((14, 0, False, -1), (20, PP_CODE, True, -1), (20, PP_CODE, False, -1),
                                           (20, 0, False, 5), (40, PP_CODE, False, -1)):
        a = check(oracle, ir, N.MODEL_IR, progs, maxm, 400, PP_FLAGS, looking_for, stop, depth, blob=blob)
        b = compiled.dpor_batch(progs, maxm, 400, looking_for, stop, depth, cap_viol=32, want_hashes=True)
        for x, y in zip(a, b):
            assert (x == y).all(), (maxm, looking_for, stop, depth)
        assert (a[0]["status"] == 0).sum() > len(progs) // 2
        found += int(a[0]["violations"].sum())
    assert found > 0


def election_programs(n, rng):
    """The election's six Start / Kick externals and random subsequences of them, some with an extra Kick (a repeating
    timer armed again is not registered twice): searches of mixed length."""
    base = election_program(wait=False)
    progs = [base]
    while len(progs) < n:
        sub = [e for e in base if rng.random() < 0.75]
        if rng.random() < 0.3:
            sub.append(D.Send(int(rng.integers(0, 3)), KICK, int(rng.integers(0, 4))))
        if sub:
            progs.append(sub)
    return progs


def test_election_many_searches_in_one_launch(oracle):
    m = election_model()
    progs = election_programs(72, np.random.default_rng(3))
    eng = ir_engine(m.blob, m.flags)
    res, _, _ = check(oracle, eng, N.MODEL_IR, progs, 16, 300, m.flags, blob=m.blob)
    assert (res["status"] == 0).all() and len(set(int(x) for x in res["interleavings"])) > 3
    assert res["exhausted"].sum() > 0 and res["races"].sum() > 0
    check(oracle, eng, N.MODEL_IR, progs, 24, 200, m.flags, looking_for=TWO_LEADERS, stop=True, blob=m.blob)


def oracle_history(oracle, m, dext, seed, steps, caps, arvind, prio, budget):
    inst = oracle.DporInstance(N.MODEL_IR, dext, steps, budget, seed=seed, arvind=arvind, prioritize_pending=prio,
                               model_flags=m.flags, looking_for=TWO_LEADERS)
    tot = {"interleavings": 0, "deliveries": 0, "races": 0}
    hashes, last = [], None
    for c in caps:
        r, h = inst.test(c)
        for k in tot:
            tot[k] += int(r[k])
        hashes += h.tolist()
        last = r
    inst.close()
    return tot, hashes, last


@pytest.mark.parametrize("arvind,prio,seeded", [(1, 1, True), (0, 1, True), (0, 0, True), (1, 0, True), (0, 0, False),
                                                (0, 1, False)])
def test_election_instances_match_oracle(oracle, arvind, prio, seeded):
    """demi_dpor_batch_ex on the election against oracle DporInstances put through the same setMaxDistance history."""
    m = election_model()
    rng = np.random.default_rng(5 + arvind + 2 * prio)
    dprog = election_program(wait=False)
    budget = 60
    eng = ir_engine(m.blob, m.flags)
    found = 0
    for rec_seed in (SHRINKING_SEED, ELECTION_SEEDS[0]):
        ev, par, steps, _ = election_recorded(oracle, rec_seed)
        seed = oracle.dpor_seed(ev, par) if seeded else None
        programs, caps = [], []
        for t in range(24):
            keep = np.ones(len(dprog), dtype=bool)
            if t:
                keep[rng.integers(0, len(dprog), size=int(rng.integers(0, 3)))] = False
            hist = CAPS[:int(rng.integers(1, len(CAPS) + 1))]
            if not arvind:
                hist = [c if c < 0 else 0 for c in hist]       # without the distance ordering every key has distance 0
            programs.append(D.pack_externals([e for e, k in zip(dprog, keep) if k])); caps.append(hist)
        flags = (N.DF_ARVIND_ORDERING if arvind else 0) | (N.DF_PRIORITIZE_PENDING if prio else 0)
        res, hashes = eng.dpor_batch_ex(programs, steps, budget, seed=(ev, par) if seeded else None, flags=flags, caps=caps,
                                        looking_for=TWO_LEADERS, want_hashes=True, heap_cap=1 << 16)
        oracle.load_model(m.blob)
        for t in range(len(programs)):
            tot, oh, last = oracle_history(oracle, m, programs[t], seed, steps, caps[t], arvind, prio, budget)
            r = res[t]
            assert r["status"] == 0 == last["status"]
            for k in tot:
                assert int(r[k]) == tot[k], (rec_seed, t, k)
            for k in ("n_nodes", "n_explored", "heap_left"):
                assert int(r[k]) == int(last[k]), (rec_seed, t, k)
            assert hashes[t][:len(oh)].tolist() == oh, (rec_seed, t)
            found += int(r["violations"] > 0)
    if seeded:
        assert found > 0          # the seeded instance of the whole program replays the recorded violation


def test_incremental_ddmin_matches_oracle(oracle):
    """demi_incremental_ddmin against oracle_incremental_ddmin on the election recordings and on violating executions
    of the loaded pingpong3: MCS, total replays, rounds and instances."""
    m = election_model()
    eng = ir_engine(m.blob, m.flags)
    dext = D.pack_externals(election_program(wait=False))
    shrunk = 0
    for rec_seed in ELECTION_SEEDS:
        ev, par, steps, _ = election_recorded(oracle, rec_seed)
        for mmd in (8, 64):
            rc, cmcs, st = oracle.incremental_ddmin(N.MODEL_IR, dext, steps, 60, oracle.dpor_seed(ev, par), max_max_distance=mmd,
                                                    stop_at_size=1, looking_for=TWO_LEADERS, model_flags=m.flags)
            assert rc == 0
            mcs, out = eng.incremental_ddmin(dext, steps, 60, (ev, par), looking_for=TWO_LEADERS, stop_at_size=1,
                                             max_max_distance=mmd, heap_cap=1 << 16)
            assert np.array_equal(mcs, cmcs), (rec_seed, mmd)
            assert (out.total_replays, out.rounds, out.instances) == (st["total_replays"], st["rounds"], st["instances"])
            assert out.mcs_size == bin(int(cmcs[0])).count("1") and out.tests_executed >= out.total_replays
            shrunk += int(out.mcs_size < len(dext))
    assert shrunk >= 2
    blob = model_ir.pingpong3_blob()
    peng = ir_engine(blob, PP_FLAGS)
    pext = D.pack_externals(pingpong_program())
    fext = D.pack_externals(pingpong_program(wait=True))
    for seed in (1, 2, 4):
        oracle.load_model(blob)
        ev, par, r = oracle.fuzz_trace(N.MODEL_IR, fext, seed, 30, 1, model_flags=PP_FLAGS)
        assert int(r["violation"]) == PP_CODE
        rc, cmcs, st = oracle.incremental_ddmin(N.MODEL_IR, pext, int(r["steps"]), 200, oracle.dpor_seed(ev, par),
                                                max_max_distance=16, stop_at_size=1, looking_for=PP_CODE, model_flags=PP_FLAGS)
        assert rc == 0
        mcs, out = peng.incremental_ddmin(pext, int(r["steps"]), 200, (ev, par), looking_for=PP_CODE, stop_at_size=1,
                                          max_max_distance=16, heap_cap=1 << 16)
        assert np.array_equal(mcs, cmcs) and out.mcs_size < len(pext), seed
        assert (out.total_replays, out.rounds, out.instances) == (st["total_replays"], st["rounds"], st["instances"])


def test_host_mirror_classes_on_a_loaded_model(oracle):
    """ResumableDPOR / IncrementalDDMin / DPORwHeuristics given an engine that carries a loaded model."""
    m = election_model()
    eng = ir_engine(m.blob, m.flags)
    cfg = D.SchedulerConfig(N.MODEL_IR, model_flags=m.flags)
    ev, par, steps, _ = election_recorded(oracle, SHRINKING_SEED)
    prog = election_program(wait=False)
    heuristic = D.ArvindDistanceOrdering()
    heuristic.init(ev, par)
    ro = D.ResumableDPOR(cfg, ev, par, max_messages=steps, max_interleavings=60, engine=eng, backtrackHeuristic=heuristic)
    dd = D.IncrementalDDMin(ro, maxMaxDistance=8, stopAtSize=1)
    mcs = dd.minimize(prog, TWO_LEADERS)
    rc, cmcs, st = oracle.incremental_ddmin(N.MODEL_IR, D.pack_externals(prog), steps, 60, oracle.dpor_seed(ev, par),
                                            max_max_distance=8, stop_at_size=1, looking_for=TWO_LEADERS, model_flags=m.flags)
    assert rc == 0 and len(mcs) < len(prog)
    assert [e._id for e in mcs] == [e._id for k, e in enumerate(prog) if (int(cmcs[0]) >> k) & 1]
    assert dd._stats.total_replays == st["total_replays"]
    ro.setMaxDistance(0)
    assert ro.test(prog, TWO_LEADERS) and ro.test(prog, TWO_LEADERS)
    # DPORwHeuristics: the unseeded election search runs out of backtrack points without two leaders; pingpong3 finds 7
    for blob, flags, p, code, maxm in ((m.blob, m.flags, election_program(), TWO_LEADERS, 24),
                                       (model_ir.pingpong3_blob(), PP_FLAGS, pingpong_program(wait=True), PP_CODE, 20)):
        dpor = D.DPORwHeuristics(D.SchedulerConfig(N.MODEL_IR, model_flags=flags), stopIfViolationFound=True,
                                 max_interleavings=300, engine=ir_engine(blob, flags))
        dpor.setMaxMessagesToSchedule(maxm)
        hit = dpor.test(p, code)
        oracle.load_model(blob)
        rc, r, cviol, _ = oracle.dpor_search(N.MODEL_IR, D.pack_externals(dpor_prog(p)), maxm, 300, code, 1, -1,
                                             model_flags=flags, node_cap=4096, explored_slots=1 << 16, heap_cap=1 << 15)
        for f in FIELDS:
            assert dpor.last[f] == r[f], (f, dpor.last, r)
        assert (hit is None) == (code == TWO_LEADERS) and (hit is None or hit == cviol[0])


def dpor_prog(prog):
    """convertToDPORTrace: the Starts and Sends of a program."""
    return [e for e in prog if e.kind in (N.EXT_START, N.EXT_SEND)]


def test_generated_models_with_timers(oracle):
    """Every generated model of seeds 1..200 whose receive() has timer operations: one K3 launch of a few programs
    per model, every search equal to the oracle's, nothing declined."""
    counts = {"models": 0, "searches": 0, "statuses": {}}
    for s in range(1, 201):
        m = ir_gen.generate(s)
        if not m.uses_timers:
            continue
        counts["models"] += 1
        fprog = ir_gen.program(m, s, kills=False)
        dprog = dpor_prog(fprog)[:m.n_actors + 4]
        rng = np.random.default_rng(s)
        progs = [dprog] + [[e for e in dprog if rng.random() < 0.8] for _ in range(3)]
        progs = [p for p in progs if p]
        eng = ir_engine(m.blob, m.flags)
        res, _, _ = check(oracle, eng, N.MODEL_IR, progs, 12, 200, m.flags, blob=m.blob)
        eng.close()
        counts["searches"] += len(progs)
        for st in res["status"]:
            counts["statuses"][int(st)] = counts["statuses"].get(int(st), 0) + 1
    assert counts["models"] >= 60 and counts["searches"] >= 200, counts
    assert counts["statuses"].get(0, 0) > counts["searches"] // 2, counts


def test_capacity_edges(oracle):
    """16 registered repeating timers / 16 cancelled keys fit and the 17th is DEMI_DS_QUEUE_OVF, at the same
    interleaving as the oracle; 80 distinct once-timers run through the 64-slot table; a receive() with 17 operations
    is DEMI_DS_QUEUE_OVF and one with 16 is not."""
    blob = edges_blob()
    eng = ir_engine(blob, DISTINCT)
    for kind in (ARM, DISARM):
        progs = [edges_program(kind, range(k), wait=False) for k in (15, 16, 17, 20)]
        res, _, _ = check(oracle, eng, N.MODEL_IR, progs, 40, 20, DISTINCT, blob=blob)
        assert [int(x) for x in res["status"]] == [0, 0, DS_QUEUE_OVF, DS_QUEUE_OVF], kind
    res, _, _ = check(oracle, eng, N.MODEL_IR, [edges_program(ONCE, range(80), wait=False)], 200, 6, DISTINCT, blob=blob,
                      explored_slots=1 << 18, heap_cap=1 << 17)
    assert int(res[0]["status"]) == 0 and int(res[0]["interleavings"]) == 6
    prog = [D.Start(0), D.Send(0, 1, 0)]
    for k, want in ((16, 0), (17, DS_QUEUE_OVF)):
        fb = _fanout_model(k)
        res, _, _ = check(oracle, ir_engine(fb, 0), N.MODEL_IR, [prog], 10, 100, 0, blob=fb)
        assert int(res[0]["status"]) == want, k


def test_errors(oracle):
    """No model loaded: DEMI_ERR_STATE from every K3 and K3F entry point; an external naming an actor at or above the
    loaded count, or of a kind other than Start and Send: DEMI_ERR_INVALID."""
    m = election_model()
    prog = election_program(wait=False)
    ev, par, steps, _ = election_recorded(oracle, SHRINKING_SEED)
    calls = (lambda e, p: e.dpor_batch([p], 10, 10),
             lambda e, p: e.dpor_batch_ex([p], 10, 10, seed=(ev, par), flags=N.DF_ARVIND_ORDERING),
             lambda e, p: e.incremental_ddmin(p, steps, 10, (ev, par), looking_for=TWO_LEADERS),
             lambda e, p: e.dpor_frontier(p, e.frontier_params(10, 10, 16)))
    bare = D.Engine(D.SchedulerConfig(N.MODEL_IR, model_flags=m.flags))
    for call in calls:
        with pytest.raises(D.DemiError) as e:
            call(bare, prog)
        assert e.value.code == N.ERR_STATE
    eng = ir_engine(m.blob, m.flags)
    for bad in (prog + [D.Start(3)], prog + [D.Send(3, KICK, 0)], [D.Start(15)], prog + [D.WaitQuiescence()]):
        for call in calls:
            with pytest.raises(D.DemiError) as e:
                call(eng, bad)
            assert e.value.code == N.ERR_INVALID
    for call in calls:
        call(eng, prog)
