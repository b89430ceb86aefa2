"""The lane fuzz kernel's steady instantiation against the CPU oracle, on both sides of every edge of its eligibility.

A batch over the handle's program starts every execution from the program's pre-delivery snapshot (taken once, by
demi_set_externals) and runs an instantiation without code for externals, partitions, isolated actors, ignoreTimers, a
violation filter or the node capacity, when lane_steady_eligible (demi_b200/csrc/lane_steady.hpp) allows it; every
other launch runs the generic instantiation.  Each case here names the instantiation it must run (demi_lane_kernel
reports it, so a silent fall-back to the generic one fails) and compares every result field per seed."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N

pytestmark = pytest.mark.gpu

FIELDS = ["violation", "steps", "state_hash", "trace_hash", "n_nodes", "n_events", "max_pending", "status"]
R, P, B = N.MODEL_RAFT5, N.MODEL_PINGPONG3, N.MODEL_BCAST32
BOOT, CLIENT_CMD = 1, 2
STEADY, GENERIC = N.LANE_STEADY, N.LANE_GENERIC
SOME, ALL, ANY = "some", "all", "any"           # what the lane engine defers to the warp engine


def starts(n=5):
    return [D.Start(a) for a in range(n)]


def boots():
    return [D.Send(a, BOOT, 0x1F) for a in range(5)]


def case(model, prog, kernel, flags=1, maxm=50, interval=5, n=4000, ignore=0, looking_for=0, lane_cap=None, deferred=ANY):
    return dict(model=model, prog=prog, kernel=kernel, flags=flags, maxm=maxm, interval=interval, n=n, ignore=ignore,
                looking_for=looking_for, lane_cap=lane_cap, deferred=deferred)


W = D.WaitQuiescence
CASES = {
    # the benchmark's workload
    "bench-d50": case(R, D.raft5_program(), STEADY, n=100_003),
    # one segment only: an external after the first quiescence wait keeps the generic kernel
    "second-segment": case(R, D.raft5_program() + [D.Send(0, CLIENT_CMD, 9), W()], GENERIC),
    # an actor killed before the wait stays isolated; killed and started again, nobody is
    "kill-before-wait": case(R, starts() + boots() + [D.Kill(3), W()], GENERIC),
    "kill-and-restart-before-wait": case(R, starts() + boots() + [D.Kill(3), D.Start(3), W()], STEADY),
    # any Partition / UnPartition, even one undone before the wait
    "partition": case(R, starts() + [D.Partition(0, 1)] + boots() + [W()], GENERIC),
    "partition-undone": case(R, starts() + [D.Partition(0, 1), D.UnPartition(0, 1)] + boots() + [W()], GENERIC),
    # a violation filter, and ignoreTimers
    "looking-for-1": case(R, D.raft5_program(), GENERIC, looking_for=1),
    "looking-for-2": case(R, D.raft5_program(), GENERIC, looking_for=2),
    "ignore-timers": case(R, D.raft5_program(), GENERIC, maxm=-1, interval=0, ignore=1),
    # more than the five BOOTs in the snapshot: 11 entries, then 16, which fill its rows and messagesToSend exactly
    "clients-6": case(R, D.raft5_program(client_cmds=6), STEADY, n=20000),
    "clients-11": case(R, D.raft5_program(client_cmds=11), STEADY, n=20000),
    # a 17th Send fits neither: the first segment defers, there is no snapshot, and every execution goes to the warp engine
    "clients-12": case(R, D.raft5_program(client_cmds=12), GENERIC, n=2000, deferred=ALL),
    # no invariant checks, and another model_flags (the snapshot holds no actor state)
    "no-invariant-flags0": case(R, D.raft5_program(client_cmds=3), STEADY, flags=0, interval=0, n=20000),
    # the node capacity: 6 nodes in the snapshot and at most 7 per delivery against demi_node_cap = 16448 at the
    # largest pending capacity.  6 + 2348 * 7 = 16442 fits, 6 + 2349 * 7 = 16449 does not.
    "node-proof-holds": case(R, D.raft5_program(), STEADY, maxm=2347, n=300),
    "node-proof-fails": case(R, D.raft5_program(), GENERIC, maxm=2348, n=300),
    "unbounded-depth": case(P, D.pingpong3_program(12), GENERIC, flags=0, maxm=-1, interval=0),
    # a lowered lane pending capacity: steady executions defer at it; below the snapshot's size there is nothing to start from
    "lane-cap-24": case(R, D.raft5_program(), STEADY, n=20000, lane_cap=24, deferred=SOME),
    "lane-cap-5": case(R, D.raft5_program(), STEADY, lane_cap=5),
    "lane-cap-4": case(R, D.raft5_program(), GENERIC, n=2000, lane_cap=4, deferred=ALL),
    # the other models' single-segment programs
    "pingpong3": case(P, D.pingpong3_program(12), STEADY, flags=0, maxm=40, interval=0),
    "pingpong3-17-sends": case(P, D.pingpong3_program(17), GENERIC, flags=0, maxm=40, interval=0, n=1000, deferred=ALL),
    "bcast32-ttl2": case(B, D.bcast32_program(2), STEADY, flags=0, maxm=200, interval=0, n=500),
}


def assert_same(a, b, what):
    for f in FIELDS:
        bad = np.nonzero(a[f] != b[f])[0]
        assert len(bad) == 0, "%s: field %s differs at %d prefixes, first idx %d: %s vs %s" % (
            what, f, len(bad), bad[0], a[bad[0]], b[bad[0]])


def engine(c):
    eng = D.Engine(D.SchedulerConfig(c["model"], model_flags=c["flags"], ignoreTimers=bool(c["ignore"])))
    eng.set_externals(D.pack_externals(c["prog"]))
    return eng


@pytest.mark.parametrize("name", sorted(CASES))
def test_instantiation_and_results(oracle, monkeypatch, name):
    c = CASES[name]
    monkeypatch.delenv("DEMI_DISABLE_LANE_ENGINE", raising=False)
    monkeypatch.delenv("DEMI_LANE_PENDING_CAP", raising=False)
    if c["lane_cap"] is not None:
        monkeypatch.setenv("DEMI_LANE_PENDING_CAP", str(c["lane_cap"]))
    eng = engine(c)
    got = eng.fuzz_batch(1, c["n"], c["maxm"], c["interval"], looking_for=c["looking_for"])
    assert eng.lane_kernel() == c["kernel"]
    deferred = eng.stats().deferred
    eng.close()
    cpu = oracle.fuzz_batch(c["model"], D.pack_externals(c["prog"]), 1, c["n"], c["maxm"], c["interval"],
                            model_flags=c["flags"], ignore_timers=c["ignore"], looking_for=c["looking_for"])
    assert_same(got, cpu, name)
    if c["deferred"] == ALL:
        assert deferred == c["n"]
    elif c["deferred"] == SOME:
        assert 0 < deferred < c["n"]


def test_snapshot_follows_the_program(oracle, monkeypatch):
    """One handle, program after program: each batch starts from the snapshot of the program it runs, and a handle
    goes back and forth between the two instantiations."""
    monkeypatch.delenv("DEMI_DISABLE_LANE_ENGINE", raising=False)
    monkeypatch.delenv("DEMI_LANE_PENDING_CAP", raising=False)
    eng = D.Engine(D.SchedulerConfig(R, model_flags=1))
    for name in ["clients-6", "second-segment", "bench-d50", "partition", "clients-11", "bench-d50"]:
        c = CASES[name]
        ext = D.pack_externals(c["prog"])
        eng.set_externals(ext)
        for looking_for, kernel in ((0, c["kernel"]), (1, GENERIC)):
            got = eng.fuzz_batch(7, 3000, 50, 5, looking_for=looking_for)
            assert eng.lane_kernel() == kernel, name
            assert_same(got, oracle.fuzz_batch(R, ext, 7, 3000, 50, 5, model_flags=1, looking_for=looking_for), name)
    eng.close()


def test_other_launches_report_their_engine(monkeypatch):
    """Recording launches run the generic instantiation; with the lane engine disabled there is none."""
    monkeypatch.delenv("DEMI_DISABLE_LANE_ENGINE", raising=False)
    c = CASES["bench-d50"]
    eng = engine(c)
    res = eng.fuzz_batch(1, 3000, 50, 5)
    assert eng.lane_kernel() == STEADY
    idx = np.nonzero(res["violation"] != 0)[0][:8].astype(np.uint32)
    _, _, rec = eng.fuzz_provenance(1, idx, 50, 5)
    assert eng.lane_kernel() == GENERIC
    assert np.array_equal(rec["trace_hash"], res["trace_hash"][idx])
    eng.close()
    monkeypatch.setenv("DEMI_DISABLE_LANE_ENGINE", "1")
    eng = engine(c)
    warp = eng.fuzz_batch(1, 3000, 50, 5)
    assert eng.lane_kernel() == N.LANE_NONE
    assert_same(warp, res, "warp engine alone vs steady")
    eng.close()
