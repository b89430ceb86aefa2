"""K3F (demi_dpor_frontier) at its capacity edges, against oracle/dpor_frontier.c: pool_cap (the arena of every point
enqueued or received), trace_cap and explored_slots at the exact need and one below it.  A search that stops on a
capacity must report what the oracle reports in every field, hash and violation record, not only the status.

No case may use an explored table that one round could fill (a full table is only handled by the bounded probe in
fr_e_has and the check after the round): `safe()` asserts explored_slots >= 2 * (W * rcap + W) before each launch."""
import pytest

import demi_b200 as D
from demi_b200 import _native as N

pytestmark = pytest.mark.gpu

FIELDS = ["interleavings", "violations", "deliveries", "races", "keys_enqueued", "keys_dropped", "explored_pairs",
          "pool_left", "records_sent", "records_received", "bytes_sent", "rounds", "exchanges", "exhausted",
          "budget_exhausted", "status", "trace_slots"]
HEAP_OVF, EXPLORED_OVF, TRACE_OVF = 4, 3, 5

NO_HISTORY = (N.MODEL_RAFT5, D.raft5_program(client_cmds=2)[:-1], 3, 30, 2000, 64, N.FR_NO_HISTORY)
HISTORY = (N.MODEL_RAFT5, D.raft5_program()[:-1], 3, 100, 100000, 64, 0)   # arena 179 005 points, live queue far smaller
# one point per round at depth 43: W * (rcap + 1) = 947 new pairs at most per round, within half of 2048 slots
PINGPONG = (N.MODEL_PINGPONG3, [D.Start(a) for a in range(3)] + [D.Send(0, 1, k) for k in range(30)], 0, 43, 100000, 1, 0)
PINGPONG30 = (N.MODEL_PINGPONG3, [D.Start(a) for a in range(3)] + [D.Send(k % 3, 1, k) for k in range(60)], 1, 30, 100000, 1, 0)


def safe(case, explored_slots):
    _, _, _, maxm, _, width, flags = case
    T1 = maxm + 2
    rcap = T1 * (T1 - 1) // 2
    assert explored_slots >= 2 * (width * rcap + width), (explored_slots, width, rcap)


def both(oracle, case, **kw):
    model, prog, mf, maxm, budget, width, flags = case
    kw = dict(dict(explored_slots=1 << 20, pool_cap=1 << 22, flags=flags), **kw)
    safe(case, kw["explored_slots"])
    eng = D.Engine(D.SchedulerConfig(model, model_flags=mf))
    F = eng.frontier_params(maxm, budget, width, **kw)
    try:
        r, viol, hashes = eng.dpor_frontier(prog, F, cap_viol=100000)
    except D.DemiError:
        r = eng.last_frontier
        viol = hashes = None
    OF = oracle.frontier_params(maxm, budget, width, **kw)
    rc, ores, oviol, ohashes = oracle.dpor_frontier(model, D.pack_externals(prog), OF, 1, model_flags=mf, cap_viol=100000)
    for f in FIELDS:
        assert r[f] == ores[0][f], (f, r, ores[0])
    if hashes is None:                                      # a failed call: read what the handle kept of the search
        assert rc != 0 and r["status"] != 0
        eng2 = D.Engine(D.SchedulerConfig(model, model_flags=mf))
        F2 = eng2.frontier_params(maxm, int(r["interleavings"]), width, **kw)
        r2, viol, hashes = eng2.dpor_frontier(prog, F2, cap_viol=100000)
        for f in ("interleavings", "violations", "deliveries", "races", "keys_enqueued", "rounds", "trace_slots"):
            assert r2[f] == r[f], (f, r2, r)
    else:
        assert rc == 0 and r["status"] == 0
    assert len(hashes) == len(ohashes[0]) and (hashes == ohashes[0]).all()
    assert (viol == oviol[0]).all()
    return r


@pytest.mark.parametrize("case", [NO_HISTORY, HISTORY], ids=["no_history", "history"])
def test_pool_cap_at_the_arena_edge(oracle, case):
    r = both(oracle, case)
    need = int(r["keys_enqueued"])
    assert need > r["pool_left"]
    if case is HISTORY:
        assert need == 179005 and r["interleavings"] == 742 and r["exhausted"] == 1
    else:
        assert need == 55424 and r["pool_left"] == 53425
    assert both(oracle, case, pool_cap=need)["status"] == 0
    r = both(oracle, case, pool_cap=need - 1)
    assert r["status"] == HEAP_OVF and r["interleavings"] > 1


@pytest.mark.parametrize("case", [NO_HISTORY, HISTORY], ids=["no_history", "history"])
def test_trace_cap_edge(oracle, case):
    need = int(both(oracle, case)["trace_slots"])
    assert both(oracle, case, trace_cap=need)["status"] == 0
    r = both(oracle, case, trace_cap=need - 1)
    assert r["status"] == TRACE_OVF and r["interleavings"] > 1


@pytest.mark.parametrize("case", [PINGPONG, PINGPONG30], ids=["pingpong43", "pingpong30"])
def test_explored_slots_edge(oracle, case):
    """The power of two above twice the final count passes with every field equal.  The one below would fail, but
    no model here reaches it with a table that one round cannot fill; that side is checked against the oracle
    alone (test_dpor_frontier_edges_oracle.py)."""
    final = int(both(oracle, case)["explored_pairs"])
    ok = 1024
    while ok <= 2 * final:
        ok *= 2
    r = both(oracle, case, explored_slots=ok)
    assert r["status"] == 0 and r["explored_pairs"] == final


def test_a_failed_round_keeps_the_last_completed_round(oracle):
    """HEAP_OVF from a history search: the engine drops the failed round as the oracle does, and the handle's next
    search with room is unaffected"""
    model, prog, mf, maxm, budget, width, flags = HISTORY
    eng = D.Engine(D.SchedulerConfig(model, model_flags=mf))
    F = eng.frontier_params(maxm, budget, width, explored_slots=1 << 20, pool_cap=100000)
    with pytest.raises(D.DemiError):
        eng.dpor_frontier(prog, F)
    failed = eng.last_frontier
    assert failed["status"] == HEAP_OVF
    F = eng.frontier_params(maxm, budget, width, explored_slots=1 << 20, pool_cap=1 << 22)
    r, _, _ = eng.dpor_frontier(prog, F)
    assert r["status"] == 0 and r["interleavings"] == 742
