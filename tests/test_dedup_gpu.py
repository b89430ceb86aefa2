"""GPU checks for K5 (state-hash dedup) / K4 (stable compaction) and the bcast32 configuration."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N

pytestmark = pytest.mark.gpu
FF_HASH_PENDING = 1


def expected_unique(res):
    """numpy restatement: per distinct state_hash keep the record with the smallest index, in index order."""
    _, first = np.unique(res["state_hash"], return_index=True)
    idx = np.sort(first)
    return res[idx], idx.astype(np.uint32)


def test_dedup_keeps_first_occurrence_in_index_order(oracle):
    ext = D.pack_externals(D.raft5_program())
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    eng.set_externals(ext)
    n = 300_000
    res = eng.fuzz_batch(1, n, 6, 5, flags=FF_HASH_PENDING)           # short prefixes: many coinciding states
    cpu = oracle.fuzz_batch(N.MODEL_RAFT5, ext, 1, 20000, 6, 5, model_flags=1, flags=FF_HASH_PENDING)
    assert (res[:20000] == cpu).all()                                  # the pending-multiset term is in parity too
    nohash = eng.fuzz_batch(1, 1000, 6, 5)
    assert (nohash["state_hash"] != res["state_hash"][:1000]).any()
    uniq, idx = eng.dedup_compact(res, 0)
    eu, ei = expected_unique(res)
    assert len(uniq) == len(eu) and len(uniq) < n
    assert (idx == ei).all() and (uniq == eu).all()
    # idempotent
    u2, i2 = eng.dedup_compact(uniq, 0)
    assert (u2 == uniq).all() and (i2 == np.arange(len(uniq))).all()
    # violating-prefix compaction is stable too
    full = eng.fuzz_batch(1, n, 50, 5)
    viol, vidx = eng.dedup_compact(full, 1)
    evidx = np.nonzero(full["violation"])[0]
    assert (vidx == evidx).all() and (viol == full[evidx]).all()


def test_dedup_edge_cases():
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5))
    empty = np.zeros(0, dtype=N.RESULT_DTYPE)
    u, i = eng.dedup_compact(empty, 0)
    assert len(u) == 0
    one = np.zeros(1, dtype=N.RESULT_DTYPE); one["state_hash"] = 0xFFFFFFFFFFFFFFFF   # the table's sentinel value
    u, i = eng.dedup_compact(np.repeat(one, 777), 0)
    assert len(u) == 1 and i[0] == 0
    # ~0 marks an empty slot; it must stay distinct from every real key, whichever of the two comes first
    ones, other = 0xFFFFFFFFFFFFFFFF, 0x5D5D5D5D5D5D5D5D
    for a, b in ((ones, other), (other, ones)):
        alias = np.zeros(5, dtype=N.RESULT_DTYPE); alias["state_hash"] = [a, b, a, b, 0]
        alias["steps"] = np.arange(5)
        u, i = eng.dedup_compact(alias, 0)
        assert i.tolist() == [0, 1, 4] and u.tobytes() == alias[[0, 1, 4]].tobytes()
    ragged = np.zeros(1025, dtype=N.RESULT_DTYPE); ragged["state_hash"] = np.arange(1025) % 7
    u, i = eng.dedup_compact(ragged, 0)
    assert (i == np.arange(7)).all()


def test_bcast32_config5_fuzz_with_dedup(oracle):
    """BASELINE configs[4]: 32-actor broadcast storm, depth-200 fuzz, state-hash dedup on."""
    prog = D.bcast32_program(3)
    ext = D.pack_externals(prog)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_BCAST32))
    eng.set_externals(ext)
    n = 3000
    res = eng.fuzz_batch(1, n, 200, 0, flags=FF_HASH_PENDING)
    cpu = oracle.fuzz_batch(N.MODEL_BCAST32, ext, 1, n, 200, 0, flags=FF_HASH_PENDING)
    assert (res == cpu).all() and (res["status"] == 0).all()
    assert (res["steps"] == 201).all() and res["max_pending"].max() > 2000
    uniq, idx = eng.dedup_compact(res, 0)
    eu, ei = expected_unique(res)
    assert (idx == ei).all() and (uniq == eu).all()
