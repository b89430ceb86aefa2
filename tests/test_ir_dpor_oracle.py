"""Resumable, edit-distance bounded DPOR and IncrementalDDMin on loaded models, on the CPU: the C oracle against the
Python restatement (tests/micro_oracle.py) on the leader election of tests/test_ir_timers_oracle.py, whose timers are
armed, fired and cancelled inside the searches, and the loaded pingpong3 (model_ir.pingpong3_blob) against the
compiled one.  The recordings and programs here are also what tests/test_ir_dpor_gpu.py runs on the engine."""
import demi_b200 as D
from demi_b200 import model_ir, _native as N
import micro_oracle as M
from test_micro_oracle import name_idx, to_prog
from test_ir_timers_oracle import ELECTION_INTERVAL, ELECTION_MAXM, TWO_LEADERS, election_blob, election_model, election_program

PP_FLAGS = 1 | (4 << 8)          # pingpong3: violation 7 once actor 0 has received 4 pongs
PP_CODE = 7


def election_recorded(oracle, seed):
    """(events, dep_parent, steps, violation) of fuzz execution `seed` of the election: a recording IncrementalDDMin
    and the seeded DPOR instances start from."""
    oracle.load_model(election_blob())
    ext = D.pack_externals(election_program())
    ev, par, r = oracle.fuzz_trace(N.MODEL_IR, ext, seed, ELECTION_MAXM, ELECTION_INTERVAL, model_flags=election_model().flags)
    return ev, par, int(r["steps"]), int(r["violation"])


# violating seeds of the election: on 10 and 29 IncrementalDDMin drops two of the six externals, on the others it
# keeps all six
ELECTION_SEEDS = (8, 10, 14, 18, 29)
SHRINKING_SEED = 10


def pingpong_program(dests=(2, 0, 2, 1, 2, 2), wait=False):
    """Start x3, then Ping(k) to dests[k]: four of them to actor 2, whose Pongs go to actor 0."""
    prog = [D.Start(a) for a in range(3)] + [D.Send(a, 1, k) for k, a in enumerate(dests)]
    return prog + [D.WaitQuiescence()] if wait else prog


def py_init_nodes(nodes):
    nm = lambda x: M.DEADLETTERS if x == 0xFF else str(x)
    return [(nm(int(w[0]) & 0xFF), str((int(w[0]) >> 8) & 0xFF), ((int(w[0]) >> 16) & 0xFF, int(w[1]), int(w[2])), int(w[3]))
            for w in nodes]


def sched_hash(py, trace):
    h = 0
    for i, u in enumerate(trace):
        if i:
            snd, rcv, (t, p0, p1) = py.event[u]
            h = (h + M.hash6(name_idx(snd) | (int(rcv) << 8) | (t << 16), p0, p1, i, 0, 0)) & ((1 << 64) - 1)
    return h


def test_election_instances_match_the_restatement(oracle):
    """Seeded DporInstances of the election, ArvindDistanceOrdering on and off, prioritizePendingUponDivergence on and
    off, several setMaxDistance histories and external subsequences: per test() call the same schedules in the same
    order, the same verdict, races, graph size and explored-pair count."""
    m = election_model()
    irm = M.IRModel(m.blob)
    dprog = election_program(wait=False)
    checked = found = 0
    cases = ((10, [0, 2, 4, 8, -1], 1, 1, ()), (8, [0, 2, -1], 1, 1, ()), (18, [0, 0, 2, 4, 16], 1, 0, (4,)),
             (10, [-1], 0, 1, ()), (29, [0, 0, -1, -1], 0, 0, (3,)), (14, [0, 4, -1], 1, 1, (5,)))
    for seed, caps, arv, prio, drop in cases:
        ev, par, steps, _ = election_recorded(oracle, seed)
        sub = [e for k, e in enumerate(dprog) if k not in drop]
        nodes, trace = oracle.dpor_seed(ev, par)
        inst = oracle.DporInstance(N.MODEL_IR, D.pack_externals(sub), steps, 300, seed=(nodes, trace), arvind=arv,
                                   prioritize_pending=prio, model_flags=m.flags, looking_for=TWO_LEADERS)
        py = M.ResumableDPORInstance(lambda: irm.make_actors(m.flags), to_prog(sub), irm.invariant(m.flags), steps,
                                     init_nodes=py_init_nodes(nodes), init_trace=[int(x) for x in trace], arvind=bool(arv),
                                     prioritize_pending=bool(prio), stop_if_found=True, looking_for=TWO_LEADERS)
        for cap in caps:
            races_before = py.races
            rc, hashes = inst.test(cap)
            ran, hit = py.test(cap, 300)
            assert int(rc["status"]) == 0
            assert (len(ran), bool(hit)) == (int(rc["interleavings"]), int(rc["violations"]) > 0), (seed, cap)
            assert [sched_hash(py, t) for t in ran] == [int(h) for h in hashes], (seed, cap)
            assert (py.races - races_before, py.next_id, len(py.explored)) == \
                (int(rc["races"]), int(rc["n_nodes"]), int(rc["n_explored"])), (seed, cap)
            checked += 1
            found += int(hit)
        inst.close()
    assert checked >= 20 and found > 0
    assert irm.stats.get("SCHED_REPEAT", 0) > 0 and irm.stats.get("CANCEL", 0) > 0 and irm.stats.get("SCHED_ONCE", 0) > 0


def python_incremental_ddmin(m, irm, devents, nodes, trace, steps, code, max_max_distance, budget):
    """IncrementalDDMin over ResumableDPOR, restated: (mask, total replays, rounds, instances, MCS sizes)."""
    init_nodes = py_init_nodes(nodes)
    instances = {}
    state = {"dist": 0}

    def test(sub):
        key = tuple(id(e) for e in sub)
        if key not in instances:
            instances[key] = M.ResumableDPORInstance(lambda: irm.make_actors(m.flags), list(sub), irm.invariant(m.flags), steps,
                                                     init_nodes=init_nodes, init_trace=[int(x) for x in trace], arvind=True,
                                                     prioritize_pending=True, stop_if_found=True, looking_for=code)
        return instances[key].test(state["dist"], budget)[1]
    current = list(enumerate(devents))
    total = rounds = 0
    sizes = []
    while state["dist"] < max_max_distance and len(current) > 1:
        dd = M.DDMin(test)
        current = dd.ddmin2(current, [])
        total += dd.total_replays
        rounds += 1
        sizes.append(len(current))
        state["dist"] = 2 if state["dist"] == 0 else state["dist"] << 1
    return sum(1 << i for i, _ in current), total, rounds, len(instances), sizes


def test_election_incremental_ddmin_matches_the_restatement(oracle):
    """IncrementalDDMin on violating election recordings: MCS, total replays, rounds, instances and the MCS size of
    every round equal oracle_incremental_ddmin's; on one recording the MCS is smaller than the program."""
    m = election_model()
    irm = M.IRModel(m.blob)
    dprog = election_program(wait=False)
    dext = D.pack_externals(dprog)
    shrunk = 0
    for seed in ELECTION_SEEDS:
        ev, par, steps, v = election_recorded(oracle, seed)
        assert v == TWO_LEADERS
        nodes, trace = oracle.dpor_seed(ev, par)
        for mmd in (8, 64):
            rc, cmcs, info = oracle.incremental_ddmin(N.MODEL_IR, dext, steps, 60, (nodes, trace), max_max_distance=mmd,
                                                      stop_at_size=1, looking_for=TWO_LEADERS, model_flags=m.flags)
            assert rc == 0
            got = python_incremental_ddmin(m, irm, to_prog(dprog), nodes, trace, steps, TWO_LEADERS, mmd, 60)
            assert got[:4] == (int(cmcs[0]), info["total_replays"], info["rounds"], info["instances"]), (seed, mmd)
            assert got[4] == [int(x) for x in info["mcs_sizes"]], (seed, mmd)
            shrunk += int(bin(int(cmcs[0])).count("1") < len(dprog))
    assert shrunk >= 2
    ev, par, steps, _ = election_recorded(oracle, SHRINKING_SEED)
    rc, cmcs, info = oracle.incremental_ddmin(N.MODEL_IR, dext, steps, 60, oracle.dpor_seed(ev, par), max_max_distance=8,
                                              stop_at_size=1, looking_for=TWO_LEADERS, model_flags=m.flags)
    assert int(cmcs[0]) == 0b11011


def test_loaded_pingpong3_equals_compiled_in_dpor(oracle):
    """model_ir.pingpong3_blob() under DEMI_MODEL_IR and DEMI_MODEL_PINGPONG3 give the same DPOR searches (every
    counter, every schedule hash, every violation record) and the same IncrementalDDMin."""
    blob = model_ir.pingpong3_blob()
    prog = pingpong_program()
    ext = D.pack_externals(prog)
    for maxm in (14, 20):
        for looking_for, stop, depth in ((0, 0, -1), (PP_CODE, 1, -1), (PP_CODE, 0, -1), (0, 0, 5)):
            oracle.load_model(blob)
            a = oracle.dpor_search(N.MODEL_IR, ext, maxm, 400, looking_for, stop, depth, model_flags=PP_FLAGS)
            b = oracle.dpor_search(N.MODEL_PINGPONG3, ext, maxm, 400, looking_for, stop, depth, model_flags=PP_FLAGS)
            assert a[0] == b[0] == 0 and a[1] == b[1], (maxm, looking_for, stop, depth)
            assert (a[2] == b[2]).all() and (a[3] == b[3]).all()
            assert int(a[1]["interleavings"]) > (0 if stop else 10) and int(a[1]["violations"]) > 0
    fext = D.pack_externals(pingpong_program(wait=True))
    done = 0
    for seed in range(1, 60):
        oracle.load_model(blob)
        ev, par, r = oracle.fuzz_trace(N.MODEL_IR, fext, seed, 30, 1, model_flags=PP_FLAGS)
        cev, cpar, cr = oracle.fuzz_trace(N.MODEL_PINGPONG3, fext, seed, 30, 1, model_flags=PP_FLAGS)
        assert (ev == cev).all() and (par == cpar).all()
        assert (int(r["violation"]), int(r["steps"])) == (int(cr["violation"]), int(cr["steps"]))
        if int(r["violation"]) != PP_CODE:
            continue
        seed_rec = oracle.dpor_seed(ev, par)
        oracle.load_model(blob)
        a = oracle.incremental_ddmin(N.MODEL_IR, ext, int(r["steps"]), 200, seed_rec, max_max_distance=16, stop_at_size=1,
                                     looking_for=PP_CODE, model_flags=PP_FLAGS)
        b = oracle.incremental_ddmin(N.MODEL_PINGPONG3, ext, int(r["steps"]), 200, seed_rec, max_max_distance=16,
                                     stop_at_size=1, looking_for=PP_CODE, model_flags=PP_FLAGS)
        assert a[0] == b[0] == 0 and (a[1] == b[1]).all()
        assert {k: v for k, v in a[2].items() if k != "mcs_sizes"} == {k: v for k, v in b[2].items() if k != "mcs_sizes"}
        assert (a[2]["mcs_sizes"] == b[2]["mcs_sizes"]).all()
        done += 1
        if done == 3:
            break
    assert done == 3
