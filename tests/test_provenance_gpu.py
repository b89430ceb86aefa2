"""GPU parity for provenance pruning (ProvenanceTracker, schedulers/Util.scala:267-376): the mask-propagation
kernel against the oracle's literal pair-set closure, through the C ABI."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
from oracle import binding as O
from test_provenance_kat import PARENT, TRACE, deliveries

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    e.set_externals(D.raft5_program())
    return e


def same(a, b):
    ka, oa = a
    kb, ob = b
    assert oa["status"] == ob["status"]
    assert np.array_equal(ka, kb)
    for f in ("affected_mask", "n_trace", "n_kept"):
        assert oa[f] == ob[f], f


def test_hand_derived_cases(eng):
    for aff in (0b01, 0b10, 0b11, 0, 0b100):
        same(eng.provenance(TRACE, PARENT, aff, 1), O.provenance(TRACE, PARENT, aff, 1))
    keep, out = eng.provenance(TRACE, PARENT, 0b10, 1)
    assert int(keep[0]) == 0b000111
    for seq in ([(1, 0)], [(1, 0), (1, 0), (2, 0)], [(1, 0), (2, 0), (1, 0)]):
        par = [0] * (1 + max(n for n, _ in seq))
        same(eng.provenance(deliveries(seq), par, 1, 1), O.provenance(deliveries(seq), par, 1, 1))
    assert eng.provenance(deliveries([(1, 0), (2, 0), (1, 0)]), [0, 0, 0], 1, 1)[1]["status"] == N.PV_CYCLE
    assert eng.provenance(deliveries([(1, 0)] * 70), [0, 0], 1, 1)[1]["status"] == N.PV_OVERFLOW


def random_execution(rng, n_actors, steps, dup_rate):
    """A random DepTracker tree + delivery order: every delivery creates 0-3 messages whose parent it is."""
    parent, rcv_of = [0], [255]
    pending, seq = [], []
    for _ in range(int(rng.integers(1, 4))):                 # externals hang off the root
        parent.append(0); rcv_of.append(int(rng.integers(0, n_actors))); pending.append(len(parent) - 1)
    for _ in range(steps):
        if not pending:
            break
        if seq and rng.random() < dup_rate:
            node = seq[int(rng.integers(0, len(seq)))][0]    # a Unique delivered again (repeating timer)
        else:
            node = pending.pop(int(rng.integers(0, len(pending))))
        seq.append((node, rcv_of[node]))
        for _ in range(int(rng.integers(0, 4))):
            parent.append(node); rcv_of.append(int(rng.integers(0, n_actors))); pending.append(len(parent) - 1)
    return deliveries(seq), parent


@pytest.mark.parametrize("n_actors,dup_rate", [(2, 0.0), (5, 0.0), (5, 0.08), (32, 0.0), (32, 0.03)])
def test_random_executions_match_literal_closure(eng, n_actors, dup_rate):
    rng = np.random.default_rng(1000 + n_actors)
    cycles = kept = 0
    for _ in range(60):
        ev, par = random_execution(rng, n_actors, int(rng.integers(1, 120)), dup_rate)
        aff = int(rng.integers(0, 1 << min(n_actors, 31)))
        got, ref = eng.provenance(ev, par, aff, 2), O.provenance(ev, par, aff, 2)
        same(got, ref)
        cycles += int(ref[1]["status"] == 1)
        kept += int(ref[1]["n_kept"])
    assert kept > 0
    if dup_rate:
        assert cycles > 0


def test_fuzz_provenance_batch_matches_oracle(eng):
    ext = D.pack_externals(D.raft5_program())
    n = 20000
    res = eng.fuzz_batch(1, n, 50, 5)
    viol = np.nonzero(res["violation"])[0].astype(np.uint32)
    assert len(viol) > 50
    idx = np.concatenate([viol[:300], np.nonzero(res["violation"] == 0)[0][:5].astype(np.uint32)])   # + clean ones: nothing affected
    keep, out, rec = eng.fuzz_provenance(1, idx, 50, 5)
    assert np.array_equal(rec["trace_hash"], res["trace_hash"][idx])
    assert np.array_equal(rec["violation"], res["violation"][idx])
    for j, i in enumerate(idx):
        k, o = O.fuzz_provenance(N.MODEL_RAFT5, ext, 1 + int(i), 50, 5, keep.shape[1], model_flags=1)
        assert o["status"] == out[j]["status"] == 0
        assert np.array_equal(k, keep[j]), int(i)
        for f in ("violation", "affected_mask", "n_trace", "n_kept"):
            assert o[f] == out[j][f], (f, int(i))
    assert (out["n_kept"][:len(viol[:300])] > 0).all() and (out["n_kept"][-5:] == 0).all()
    # pruning helps: it removes a real share of the deliveries
    assert out["n_kept"][:300].sum() < 0.9 * out["n_trace"][:300].sum()


def test_fuzz_provenance_reports_its_own_launches_and_prefixes(eng):
    """demi_perf after fuzz_provenance describes that call alone: the same call gives the same launch count, and
    `prefixes` counts its executions, not those of the batch before it."""
    res = eng.fuzz_batch(1, 20000, 50, 5)
    idx = np.nonzero(res["violation"])[0][:100].astype(np.uint32)
    assert 0 < len(idx) < 20000
    seen = []
    for _ in range(2):
        eng.fuzz_provenance(1, idx, 50, 5)
        seen.append((eng.stats().kernel_launches, eng.stats().prefixes))
    assert seen[0] == seen[1] and seen[0][1] == len(idx) and seen[0][0] >= 2


def test_fuzz_provenance_slots_deferred_by_the_lane_engine(monkeypatch):
    """The lane engine records what it can prove exact; slots it defers (here: more than 24 pending messages, a bound
    lowered for the test) are recorded by the general engine, addressed by work-list position.  Both kinds in one
    batch, against the oracle."""
    monkeypatch.setenv("DEMI_LANE_PENDING_CAP", "24")
    ext = D.pack_externals(D.raft5_program())
    eng2 = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    eng2.set_externals(ext)
    n, maxm, interval = 20000, 50, 5
    res = eng2.fuzz_batch(1, n, maxm, interval)
    assert 0 < eng2.stats().deferred < n
    cpu = O.fuzz_batch(N.MODEL_RAFT5, ext, 1, n, maxm, interval, model_flags=1)
    assert (res == cpu).all()
    big = np.nonzero((res["violation"] != 0) & (res["max_pending"] > 24))[0].astype(np.uint32)      # deferred
    small = np.nonzero((res["violation"] != 0) & (res["max_pending"] <= 24))[0].astype(np.uint32)   # recorded by the lane engine
    assert len(big) > 20 and len(small) > 20
    idx = np.empty(0, dtype=np.uint32)
    for a, b in zip(big[:60], small[:60]):          # interleaved, so positions and prefix indexes differ
        idx = np.append(idx, [b, a]).astype(np.uint32)
    keep, out, rec = eng2.fuzz_provenance(1, idx, maxm, interval)
    assert np.array_equal(rec["trace_hash"], res["trace_hash"][idx])
    assert np.array_equal(rec["violation"], res["violation"][idx])
    for j, i in enumerate(idx):
        k, o = O.fuzz_provenance(N.MODEL_RAFT5, ext, 1 + int(i), maxm, interval, keep.shape[1], model_flags=1)
        assert o["status"] == out[j]["status"] == 0
        assert np.array_equal(k, keep[j]), int(i)
        for f in ("violation", "affected_mask", "n_trace", "n_kept"):
            assert o[f] == out[j][f], (f, int(i))
    eng2.close()
