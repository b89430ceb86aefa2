"""K3F at the widths the benchmark runs, compared with oracle/dpor_frontier.c in slot order: every result field and
every schedule hash.  Each no-history case first shows, from the oracle, that the code path it is there for ran:
without history a round executes min(W, pool_left, budget left) points (more than FR_TILE = 1024 of them use several
enqueue tiles) and its selection window holds min(pool_left, win_cap) entries, win_cap = min(max(4W, 4096), 2^22)
(more than 1024 blocks of 256 need a second pass of fr_sel_blockscan_kernel)."""
import ctypes as C

import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N

pytestmark = pytest.mark.gpu

FIELDS = ["interleavings", "violations", "deliveries", "races", "keys_enqueued", "keys_dropped", "explored_pairs",
          "pool_left", "records_sent", "records_received", "bytes_sent", "rounds", "exchanges", "exhausted",
          "budget_exhausted", "status", "trace_slots"]
PROG = D.raft5_program(client_cmds=2)[:-1]


def rounds(oracle, prog, mf, maxm, budget, width, **kw):
    """(points executed, window entries) of every round after the root, from the oracle run with the budget cut at
    the previous round"""
    win_cap = min(max(4 * width, 4096), 1 << 22)
    out, done = [], 1
    while done < budget:
        F = oracle.frontier_params(maxm, done, width, flags=N.FR_NO_HISTORY, **kw)
        rc, res, _, _ = oracle.dpor_frontier(N.MODEL_RAFT5, D.pack_externals(prog), F, 1, model_flags=mf)
        assert rc == 0 and res[0]["interleavings"] == done
        pool = int(res[0]["pool_left"])
        n = min(width, pool, budget - done)
        out.append((n, min(pool, win_cap)))
        done += n
    return out


def compare(oracle, eng, prog, mf, F, OF, ranks=1):
    r, viol, hashes = eng.dpor_frontier(prog, F)
    rc, ores, oviol, ohashes = oracle.dpor_frontier(N.MODEL_RAFT5, D.pack_externals(prog), OF, ranks, model_flags=mf)
    assert rc == 0
    for f in FIELDS:
        assert r[f] == ores[0][f], (f, r, ores[0])
    assert len(hashes) == len(ohashes[0]) and (hashes == ohashes[0]).all()
    assert (viol == oviol[0]).all()
    return r, hashes


def nh_case(oracle, maxm, budget, width, pool_cap=1 << 22):
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=3))
    F = eng.frontier_params(maxm, budget, width, explored_slots=1 << 10, pool_cap=pool_cap, flags=N.FR_NO_HISTORY)
    OF = oracle.frontier_params(maxm, budget, width, explored_slots=1 << 10, pool_cap=pool_cap, flags=N.FR_NO_HISTORY)
    r, hashes = compare(oracle, eng, PROG, 3, F, OF)
    assert r["budget_exhausted"] == 1 and r["status"] == 0
    return eng, F, OF, r, hashes


@pytest.mark.parametrize("width", [1024, 1025])
def test_enqueue_tiles(oracle, width):
    budget = 1 + 3 * width
    rs = rounds(oracle, PROG, 3, 30, budget, width)
    assert max(n for n, _ in rs) == width                     # a round of 1024 points is one tile, of 1025 two
    nh_case(oracle, 30, budget, width)


@pytest.mark.parametrize("width, blocks", [(65536, 1024), (65537, 1025)])
def test_selection_scan_passes(oracle, width, blocks):
    rs = rounds(oracle, PROG, 3, 24, 131072, width)
    assert max((w + 255) // 256 for _, w in rs) == blocks     # a window of 262 144 entries, then of 262 148
    assert max(n for n, _ in rs) > 1024
    nh_case(oracle, 24, 131072, width)


def test_bench_geometry_and_its_call_pair(oracle):
    """The benchmark's no-history search (model_flags 3, depth 100, width 131 072) through root, round 2 and one full
    round, called twice on one handle as the benchmark does (warm-up, then the timed call on the cached tables)."""
    W, budget = 131072, 131816
    rs = rounds(oracle, PROG, 3, 100, budget, W, pool_cap=1 << 26)
    assert rs[-1][0] == W and len(rs) == 2
    eng, F, OF, r, hashes = nh_case(oracle, 100, budget, W, pool_cap=1 << 26)
    r2, viol2, hashes2 = eng.dpor_frontier(PROG, F)
    for f in FIELDS:
        assert r2[f] == r[f], f
    assert (hashes2 == hashes).all()


def test_bench_history_search(oracle):
    """The benchmark's history-on search at its parameters: equal to the frontier oracle, and its schedule set equal
    to the sequential search's."""
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=3))
    kw = dict(explored_slots=1 << 16, pool_cap=1 << 18, trace_cap=1 << 16)
    F = eng.frontier_params(100, 1 << 16, 16384, **kw)
    OF = oracle.frontier_params(100, 1 << 16, 16384, **kw)
    r, hashes = compare(oracle, eng, PROG, 3, F, OF)
    assert r["exhausted"] == 1 and r["status"] == 0
    rc, sr, sviol, shashes = oracle.dpor_search(N.MODEL_RAFT5, D.pack_externals(PROG), 100, 1 << 16, 0, 0, -1, model_flags=3,
                                                node_cap=1 << 14, explored_slots=1 << 18, heap_cap=1 << 20)
    assert rc == 0 and sr["exhausted"] == 1
    assert set(int(x) for x in hashes) == set(int(x) for x in shashes)


def test_reused_handle_equals_a_fresh_one(oracle):
    """One handle: the same search twice, another program with the same Send count (the cached tables are reused),
    then history switched on and off.  Every result equals a fresh handle's."""
    other = [D.Start(a) for a in (4, 2, 0, 1, 3)] + [D.Send(a, 1, 0x1F) for a in (3, 1, 4, 0, 2)] + [D.Send(2, 2, 7), D.Send(0, 2, 9)]
    W = 512
    calls = [(PROG, N.FR_NO_HISTORY), (PROG, N.FR_NO_HISTORY), (other, N.FR_NO_HISTORY), (other, 0), (PROG, 0),
             (PROG, N.FR_NO_HISTORY)]
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=3))
    for prog, flags in calls:
        F = eng.frontier_params(40, 3000, W, explored_slots=1 << 20, pool_cap=1 << 22, flags=flags)
        assert (1 << 20) >= 2 * (W * 42 * 41 // 2 + W)
        r, viol, hashes = eng.dpor_frontier(prog, F)
        fresh = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=3))
        r0, viol0, hashes0 = fresh.dpor_frontier(prog, F)
        for f in FIELDS:
            assert r[f] == r0[f], (f, flags)
        assert (hashes == hashes0).all() and (viol == viol0).all()
        OF = oracle.frontier_params(40, 3000, W, explored_slots=1 << 20, pool_cap=1 << 22, flags=flags)
        rc, ores, _, ohashes = oracle.dpor_frontier(N.MODEL_RAFT5, D.pack_externals(prog), OF, 1, model_flags=3)
        assert rc == 0 and (hashes == ohashes[0]).all() and r["interleavings"] == ores[0]["interleavings"]


def test_two_ranks_reuse_their_handles(oracle):
    """Two ranks, a no-history search and then a history search on the same handles: the history search must share
    explored pairs between the ranks exactly as the simulated protocol does."""
    L = N.lib()
    if L.demi_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cfg = N.Config(0, N.MODEL_RAFT5, 3, 0, 0, 0)
    devs = (C.c_int32 * 2)(0, 1)
    hs = (C.c_void_p * 2)()
    assert L.demi_create_multi(C.byref(cfg), devs, 2, hs) == 0, L.demi_last_error(None)
    ext = D.pack_externals(PROG)
    try:
        for flags in (N.FR_NO_HISTORY, 0, N.FR_NO_HISTORY):
            kw = dict(explored_slots=1 << 20, pool_cap=1 << 22, rounds_per_exchange=2, steal_max=64, flags=flags)
            F = D.Engine.frontier_params(40, 3000, 64, **kw)
            res = np.zeros(2, dtype=N.FRONTIER_RESULT_DTYPE)
            viol = np.zeros((2, 4096), dtype=N.DPOR_VIOL_DTYPE)
            cap_h = 3000 + 64 + 1
            hashes = np.zeros((2, cap_h), dtype=np.uint64)
            rc = L.demi_dpor_frontier_multi(hs, 2, ext.ctypes.data, len(ext), C.byref(F), res.ctypes.data, viol.ctypes.data,
                                            4096, hashes.ctypes.data, cap_h)
            assert rc == 0, [L.demi_last_error(hs[i]) for i in range(2)]
            OF = oracle.frontier_params(40, 3000, 64, **kw)
            orc, ores, _, ohashes = oracle.dpor_frontier(N.MODEL_RAFT5, ext, OF, 2, model_flags=3)
            assert orc == 0
            for q in range(2):
                for f in FIELDS:
                    assert res[q][f] == ores[q][f], (flags, q, f)
                assert (hashes[q, :int(res[q]["interleavings"])] == ohashes[q]).all()
    finally:
        for i in range(2):
            L.demi_destroy(hs[i])
