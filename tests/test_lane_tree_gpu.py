"""The steady lane kernel's tree of first deliveries against the CPU oracle.

A steady batch starts each execution at the node of the program's tree (demi_b200/csrc/lane_steady.hpp) that its
first pick indices lead to, so every input of those deliveries is part of the tree's key: the program, model_flags,
the invariant interval, maxMessages and the lane pending capacity.  Each case compares every result field per seed,
and names the depth it must have walked where that is known (demi_lane_tree_depth), so that a silent fall-back to
the bare snapshot fails."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N

pytestmark = pytest.mark.gpu

FIELDS = ["violation", "steps", "state_hash", "trace_hash", "n_nodes", "n_events", "max_pending", "status"]
R, P, B = N.MODEL_RAFT5, N.MODEL_PINGPONG3, N.MODEL_BCAST32


@pytest.fixture(autouse=True)
def lane_engine(monkeypatch):
    monkeypatch.delenv("DEMI_DISABLE_LANE_ENGINE", raising=False)
    monkeypatch.delenv("DEMI_LANE_PENDING_CAP", raising=False)
    return monkeypatch


def assert_same(a, b, what):
    for f in FIELDS:
        bad = np.nonzero(a[f] != b[f])[0]
        assert len(bad) == 0, "%s: field %s differs at %d prefixes, first idx %d: %s vs %s" % (
            what, f, len(bad), bad[0], a[bad[0]], b[bad[0]])


def run(oracle, model, prog, n, maxm, interval, flags=1, seed=1, min_depth=0, eng=None):
    own = eng is None
    if own:
        eng = D.Engine(D.SchedulerConfig(model, model_flags=flags))
    ext = D.pack_externals(prog)
    eng.set_externals(ext)
    got = eng.fuzz_batch(seed, n, maxm, interval)
    assert eng.lane_kernel() == N.LANE_STEADY
    depth = eng.lane_tree_depth()
    assert depth >= min_depth
    deferred = eng.stats().deferred
    if own:
        eng.close()
    cpu = oracle.fuzz_batch(model, ext, seed, n, maxm, interval, model_flags=flags)
    assert_same(got, cpu, "model %d maxm %d interval %d flags %d" % (model, maxm, interval, flags))
    return depth, deferred


def test_bench_workload(oracle):
    """The benchmark's batch walks at least four levels."""
    depth, _ = run(oracle, R, D.raft5_program(), 100_003, 50, 5, seed=10_000_001, min_depth=4)
    assert depth <= 8


@pytest.mark.parametrize("interval", [1, 2, 3, 4, 5, 6])
def test_interval_and_max_messages(oracle, interval):
    """maxMessages 0..6 stop executions at or inside the tree; 50 runs through it."""
    for maxm in list(range(7)) + [50]:
        run(oracle, R, D.raft5_program(), 3000, maxm, interval, seed=77 + maxm)


@pytest.mark.parametrize("flags", [0, 1, 2, 3])
def test_model_flags(oracle, flags):
    run(oracle, R, D.raft5_program(), 20000, 50, 5, flags=flags, min_depth=1)


@pytest.mark.parametrize("clients", [3, 6, 11])
def test_client_commands(oracle, clients):
    """More rows per node: some nodes exceed the record's rows and the tree stops at their parents."""
    run(oracle, R, D.raft5_program(client_cmds=clients), 20000, 50, 5)


@pytest.mark.parametrize("cap", [6, 8, 12])
def test_low_lane_pending_cap(oracle, lane_engine, cap):
    """A lane pending capacity just above the snapshot's five rows: executions inside the tree defer."""
    lane_engine.setenv("DEMI_LANE_PENDING_CAP", str(cap))
    _, deferred = run(oracle, R, D.raft5_program(), 20000, 50, 5)
    assert deferred > 0


@pytest.mark.parametrize("model,prog,maxm", [(B, D.bcast32_program(2), 200), (B, D.bcast32_program(3), 200),
                                             (P, D.pingpong3_program(12), 40)],
                         ids=["bcast32-ttl2", "bcast32-ttl3", "pingpong3"])
def test_other_models(oracle, model, prog, maxm):
    run(oracle, model, prog, 2000, maxm, 0, flags=0)


def test_key_changes_on_one_handle(oracle):
    """One handle: the tree follows interval, maxMessages and the program, and comes back to earlier keys."""
    eng = D.Engine(D.SchedulerConfig(R, model_flags=1))
    bench, clients = D.raft5_program(), D.raft5_program(client_cmds=3)
    for prog, maxm, interval in [(bench, 50, 5), (bench, 50, 1), (bench, 50, 5), (bench, 3, 5), (bench, 50, 5),
                                 (clients, 50, 5), (bench, 50, 5), (bench, 50, 5)]:
        run(oracle, R, prog, 5000, maxm, interval, seed=3 + maxm + interval, eng=eng)
    eng.close()


def test_handles_with_different_model_flags(oracle):
    engs = [D.Engine(D.SchedulerConfig(R, model_flags=f)) for f in (0, 1, 3)]
    for rnd in range(2):
        for f, eng in zip((0, 1, 3), engs):
            run(oracle, R, D.raft5_program(), 5000, 50, 5, flags=f, seed=11 + rnd, eng=eng)
    for eng in engs:
        eng.close()
