"""The raft5 lane fuzz kernel on programs other than the bench's: partitions and kills make sends and timers cross
partitions (a node and a sequence number, no pending entry), restarts and client commands vary the first flush, and a
low lane pending capacity makes the lane engine defer mid-execution, so that lane-engine and warp-engine prefixes
alternate in one batch.  Every result field is compared per seed with the oracle, and the recorded traces of violating
executions (the lane engine's recording instantiation) event by event through their provenance masks."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N

pytestmark = pytest.mark.gpu

FIELDS = ["violation", "steps", "state_hash", "trace_hash", "n_nodes", "n_events", "max_pending", "status"]
BOOT, CLIENT_CMD = 1, 2


def boots(actors):
    return [D.Send(a, BOOT, 0x1F) for a in actors]


PROGRAMS = {
    # isolated pairs and a dead actor for the whole execution: sends and timers that cross them
    "partition-kill": lambda: ([D.Start(a) for a in range(5)] + [D.Partition(0, 1), D.Partition(3, 2), D.Kill(4)]
                               + boots(range(5)) + [D.Send(1, CLIENT_CMD, 7)] + [D.WaitQuiescence()]),
    # a restart and a healed partition before the bootstraps, client commands in the first flush
    "restart-clients": lambda: ([D.Start(a) for a in range(5)] + [D.Kill(2), D.Partition(1, 0), D.Start(2),
                                                                  D.UnPartition(1, 0)]
                                + boots(range(5)) + [D.Send(i % 5, CLIENT_CMD, 1 + i) for i in range(4)]
                                + [D.WaitQuiescence()]),
    # one actor never booted: its timers never start, messages to it stay pending
    "partial-boot": lambda: [D.Start(a) for a in range(5)] + boots([0, 1, 2, 4]) + [D.WaitQuiescence()],
}


def assert_same(gpu, cpu):
    for f in FIELDS:
        bad = np.nonzero(gpu[f] != cpu[f])[0]
        assert len(bad) == 0, "field %s differs at %d prefixes, first idx %d: gpu=%s cpu=%s" % (
            f, len(bad), bad[0], gpu[bad[0]], cpu[bad[0]])


@pytest.mark.parametrize("lane_cap", [None, 24])
@pytest.mark.parametrize("name", sorted(PROGRAMS))
def test_programs_match_oracle(oracle, monkeypatch, name, lane_cap):
    if lane_cap is not None:
        monkeypatch.setenv("DEMI_LANE_PENDING_CAP", str(lane_cap))
    ext = D.pack_externals(PROGRAMS[name]())
    n, maxm, interval = 20000, 50, 5
    for flags in (1, 0):
        eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=flags))
        eng.set_externals(ext)
        gpu = eng.fuzz_batch(1, n, maxm, interval)
        deferred = eng.stats().deferred
        eng.close()
        cpu = oracle.fuzz_batch(N.MODEL_RAFT5, ext, 1, n, maxm, interval, model_flags=flags)
        assert_same(gpu, cpu)
        assert (gpu["status"] == 0).all()
        if lane_cap is not None:
            assert 0 < deferred < n          # both engines ran
            assert (gpu["max_pending"] > lane_cap).any()


@pytest.mark.parametrize("name", sorted(PROGRAMS))
def test_recorded_traces_match_oracle(oracle, monkeypatch, name):
    """Violating executions recorded by the lane engine (and, past a lowered pending capacity, by the warp engine):
    trace hash, verdict, and the provenance masks, which follow every event's position and DepTracker parent."""
    monkeypatch.setenv("DEMI_LANE_PENDING_CAP", "24")
    ext = D.pack_externals(PROGRAMS[name]())
    n, maxm, interval = 20000, 50, 5
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    eng.set_externals(ext)
    res = eng.fuzz_batch(1, n, maxm, interval)
    viol = np.nonzero(res["violation"] != 0)[0]
    small = viol[res["max_pending"][viol] <= 24][:40]
    big = viol[res["max_pending"][viol] > 24][:20]
    assert len(small) >= 10
    idx = np.concatenate([small, big]).astype(np.uint32)
    keep, out, rec = eng.fuzz_provenance(1, idx, maxm, interval)
    assert np.array_equal(rec["trace_hash"], res["trace_hash"][idx])
    assert np.array_equal(rec["violation"], res["violation"][idx])
    for j, i in enumerate(idx):
        k, o = oracle.fuzz_provenance(N.MODEL_RAFT5, ext, 1 + int(i), maxm, interval, keep.shape[1], model_flags=1)
        assert o["status"] == out[j]["status"] == 0
        assert np.array_equal(k, keep[j]), int(i)
        for f in ("violation", "affected_mask", "n_trace", "n_kept"):
            assert o[f] == out[j][f], (f, int(i))
    eng.close()
