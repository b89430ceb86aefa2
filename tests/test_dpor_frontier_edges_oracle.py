"""What a frontier DPOR search (oracle/dpor_frontier.c) reports when it meets a capacity.

pool_cap bounds the arena (every backtrack point enqueued or received over the search), not the live queue.  A round
that ends in a capacity status adds nothing to the executed work: its counters, hashes and violations are those of the
same search with the budget cut at the interleavings it reports."""
import pytest

import demi_b200 as D
from demi_b200 import _native as N

FIELDS = ["interleavings", "violations", "deliveries", "races", "keys_enqueued", "keys_dropped", "explored_pairs",
          "pool_left", "records_sent", "records_received", "bytes_sent", "rounds", "exchanges", "exhausted",
          "budget_exhausted", "status", "trace_slots"]
EXECUTED = ["interleavings", "violations", "deliveries", "races", "keys_enqueued", "rounds", "trace_slots"]
HEAP_OVF, EXPLORED_OVF, TRACE_OVF = 4, 3, 5

NO_HISTORY = (N.MODEL_RAFT5, D.raft5_program(client_cmds=2)[:-1], 3, 30, 2000, 64, N.FR_NO_HISTORY)
HISTORY = (N.MODEL_RAFT5, D.raft5_program()[:-1], 3, 100, 100000, 64, 0)
PINGPONG = (N.MODEL_PINGPONG3, [D.Start(a) for a in range(3)] + [D.Send(k % 3, 1, k) for k in range(8)], 1 | (2 << 8), 18,
            100000, 4, 0)


def search(oracle, case, ranks=1, **kw):
    model, prog, mf, maxm, budget, width, flags = case
    kw = dict(dict(explored_slots=1 << 22, pool_cap=1 << 22, flags=flags), **kw)
    budget = kw.pop("budget", budget)
    F = oracle.frontier_params(maxm, budget, width, **kw)
    return oracle.dpor_frontier(model, D.pack_externals(prog), F, ranks, model_flags=mf, cap_viol=100000)


def same(a, b, fields):
    for f in fields:
        assert a[f] == b[f], (f, a, b)


def check_failed_round(oracle, case, failed, **kw):
    """the failed search's executed work = the same search with the budget cut where it stopped"""
    rc, res, vs, hs = failed
    n = int(res[0]["interleavings"])
    assert n > 1                                               # it failed after some rounds, not at the root
    rc2, res2, vs2, hs2 = search(oracle, case, budget=n, **kw)
    assert rc2 == 0 and res2[0]["budget_exhausted"] == 1
    same(res[0], res2[0], EXECUTED)
    assert (hs[0] == hs2[0]).all()
    assert (vs[0] == vs2[0]).all()


@pytest.mark.parametrize("case", [NO_HISTORY, HISTORY, PINGPONG], ids=["no_history", "history", "pingpong"])
def test_pool_cap_bounds_the_arena(oracle, case):
    rc, res, vs, hs = search(oracle, case)
    assert rc == 0 and res[0]["status"] == 0
    need = int(res[0]["keys_enqueued"])
    assert need > res[0]["pool_left"]                          # the arena is larger than the live queue ...
    if case is HISTORY:
        assert res[0]["exhausted"] == 1 and res[0]["interleavings"] == 742 and need == 179005   # ... far larger here
    rc1, res1, vs1, hs1 = search(oracle, case, pool_cap=need)
    assert rc1 == 0
    same(res[0], res1[0], FIELDS)
    assert (hs[0] == hs1[0]).all() and (vs[0] == vs1[0]).all()
    failed = search(oracle, case, pool_cap=need - 1)
    assert failed[0] != 0 and failed[1][0]["status"] == HEAP_OVF
    assert failed[1][0]["keys_enqueued"] < need
    check_failed_round(oracle, case, failed)


def test_pool_cap_on_two_ranks_counts_received_points(oracle):
    """with steals a rank's arena holds what it enqueued and what it received"""
    kw = dict(rounds_per_exchange=2, steal_max=64)
    for case in [NO_HISTORY, (N.MODEL_RAFT5, D.raft5_program()[:-1], 3, 40, 100000, 16, 0)]:
        rc, res, vs, hs = search(oracle, case, ranks=2, **kw)
        assert rc == 0 and res["records_received"].sum() > 0
        arena = res["keys_enqueued"] + res["records_received"]
        need = int(arena.max())
        rc1, res1, vs1, hs1 = search(oracle, case, ranks=2, pool_cap=need, **kw)
        assert rc1 == 0
        for q in range(2):
            same(res[q], res1[q], FIELDS)
            assert (hs[q] == hs1[q]).all()
        rc2, res2, _, _ = search(oracle, case, ranks=2, pool_cap=need - 1, **kw)
        assert rc2 != 0 and HEAP_OVF in set(int(s) for s in res2["status"])
        assert (res2["keys_enqueued"] + res2["records_received"] <= need - 1).all()


@pytest.mark.parametrize("case", [NO_HISTORY, HISTORY, PINGPONG], ids=["no_history", "history", "pingpong"])
def test_trace_cap_is_decided_for_the_whole_round(oracle, case):
    rc, res, vs, hs = search(oracle, case)
    need = int(res[0]["trace_slots"])
    rc1, res1, _, hs1 = search(oracle, case, trace_cap=need)
    assert rc1 == 0
    same(res[0], res1[0], FIELDS)
    failed = search(oracle, case, trace_cap=need - 1)
    assert failed[0] != 0 and failed[1][0]["status"] == TRACE_OVF
    check_failed_round(oracle, case, failed)


@pytest.mark.parametrize("case", [HISTORY, PINGPONG], ids=["history", "pingpong"])
def test_explored_slots_are_decided_after_the_round(oracle, case):
    """EXPLORED_OVF when a round leaves explored_pairs · 2 >= explored_slots: the power of two above twice the final
    count passes, the one below fails"""
    rc, res, vs, hs = search(oracle, case)
    final = int(res[0]["explored_pairs"])
    ok = 1
    while ok <= 2 * final:
        ok *= 2
    rc1, res1, _, hs1 = search(oracle, case, explored_slots=ok)
    assert rc1 == 0
    same(res[0], res1[0], FIELDS)
    failed = search(oracle, case, explored_slots=ok // 2)
    assert failed[0] != 0 and failed[1][0]["status"] == EXPLORED_OVF
    # explored_pairs is the failed round's getNext: the round's own scan is not counted
    assert failed[1][0]["explored_pairs"] < ok // 4 + case[5]
    check_failed_round(oracle, case, failed)


def test_a_failed_root_round_reports_nothing_executed(oracle):
    rc, res, vs, hs = search(oracle, HISTORY, pool_cap=1)
    r = res[0]
    assert rc != 0 and r["status"] == HEAP_OVF
    for f in EXECUTED:
        assert r[f] == 0, f
    assert r["pool_left"] == 0 and r["explored_pairs"] == 0 and len(hs[0]) == 0
