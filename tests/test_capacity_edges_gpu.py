"""The engine at its capacity edges (DESIGN.md §4), against the C oracle record by record: the last state that fits
(status 0 with the counter equal to its cap) and one step past it (the named DEMI_PS_* status, and an otherwise
all-zero record).  The programs are pinned on the oracle in tests/test_capacity_edges_oracle.py.  Every case runs
on the lane engine with the warp engine behind it, and on the warp engine alone."""
import ctypes as C

import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N, model_ir
from test_capacity_edges_oracle import (DPOR_BASE, DPOR_BUCKET_EDGES, DPOR_HEAP_BUDGET, DPOR_HEAP_EDGES, DS_QUEUE_OVF,
                                        HARD_KILL_K, PS_EVENT_OVF, PS_NODE_OVF, PS_PENDING_OVF, SMALL_CAPS,
                                        bcast32_node_edge, bcast32_small_cap, dpor_bucket_program, dpor_heap_instance,
                                        dpor_queue_program, hard_kill_program, long_seed_search, raft5_seed_world,
                                        uniq_wrap_program)
from test_dpor_gpu import FIELDS as DPOR_FIELDS, check as dpor_check
from test_fuzz_parity_gpu import assert_same, engine_mode  # noqa: F401  (the fixture)
from test_random_ddmin_oracle import bits

pytestmark = pytest.mark.gpu


def overflowed_records_are_zero(r):
    bad = r[r["status"] != 0]
    for f in ("violation", "steps", "state_hash", "trace_hash", "n_nodes", "n_events", "max_pending"):
        assert (bad[f] == 0).all(), f


def fuzz_case(oracle, model, prog, n, maxm, interval=0, model_flags=0, blocked_mask=0, lane_eligible=False,
              engine_mode="warp-only"):
    ext = D.pack_externals(prog)
    eng = D.Engine(D.SchedulerConfig(model, model_flags=model_flags, blocked_mask=blocked_mask))
    eng.set_externals(ext)
    gpu = eng.fuzz_batch(1, n, maxm, interval)
    cpu = oracle.fuzz_batch(model, ext, 1, n, maxm, interval, model_flags=model_flags, blocked_mask=blocked_mask)
    assert_same(gpu, cpu)
    overflowed_records_are_zero(gpu)
    if lane_eligible and engine_mode == "lane+warp":
        assert eng.stats().deferred > 0
    return eng, gpu


def raw_trace(eng, seed, maxm, interval, cap_events, cap_nodes=65536):
    """demi_fuzz_trace without the wrapper's raise, so that an overflowed record can be read."""
    p = N.FuzzParams(seed, 1, maxm, interval, 0, 0)
    ev = np.zeros(max(cap_events, 1), dtype=N.EVENT_DTYPE)
    par = np.zeros(max(cap_nodes, 1), dtype=np.uint16)
    ne, nn = C.c_uint32(), C.c_uint32()
    res = np.zeros(1, dtype=N.RESULT_DTYPE)
    rc = N.lib().demi_fuzz_trace(eng._h, C.byref(p), seed, ev.ctypes.data, cap_events, C.byref(ne), par.ctypes.data,
                                 cap_nodes, C.byref(nn), res.ctypes.data)
    return rc, ev[:ne.value], par[:min(nn.value, cap_nodes)], res[0], nn.value


def test_pending_cap_edges_on_bcast32(oracle, engine_mode):
    for n_flood, n_quiet, cap, counts, at_cap in SMALL_CAPS:
        _, r = fuzz_case(oracle, N.MODEL_BCAST32, bcast32_small_cap(n_flood, n_quiet), 400, -1, lane_eligible=True,
                         engine_mode=engine_mode)
        ok = r["status"] == 0
        assert (r["status"][~ok] == PS_PENDING_OVF).all() and int(ok.sum()) == counts[0]
        assert int((r["max_pending"][ok] == cap).sum()) == at_cap


def test_pending_cap_clamp_on_bcast32(oracle, engine_mode):
    _, r = fuzz_case(oracle, N.MODEL_BCAST32, D.bcast32_program(4), 500, 900, lane_eligible=True, engine_mode=engine_mode)
    assert int((r["status"] == PS_PENDING_OVF).sum()) == 190
    assert int(r["max_pending"][r["status"] == 0].max()) == 8190


def test_node_cap_edge_on_bcast32(oracle, engine_mode):
    _, r = fuzz_case(oracle, N.MODEL_BCAST32, bcast32_node_edge(0), 300, -1, lane_eligible=True, engine_mode=engine_mode)
    assert (r["status"] == 0).all() and (r["n_nodes"] == 320).all()
    _, r = fuzz_case(oracle, N.MODEL_BCAST32, bcast32_node_edge(1), 300, -1, lane_eligible=True, engine_mode=engine_mode)
    assert (r["status"] == PS_NODE_OVF).all()


@pytest.mark.parametrize("k", HARD_KILL_K)
def test_hard_kill_of_many_pending_messages(oracle, engine_mode, k):
    """k Pings pending for the blocked actor 1, then HardKill(1): status 0 for every k, on fuzz_batch, fuzz_trace and
    random_test_batch.  With k <= 111 the program fits the PingPong3 128 tier (pending and send queue); listing the
    k matches needs room for 2k entries, which only the HBM tiers have."""
    prog = hard_kill_program(k)
    eng, r = fuzz_case(oracle, N.MODEL_PINGPONG3, prog, 64, -1, blocked_mask=0b010, engine_mode=engine_mode)
    assert (r["status"] == 0).all() and (r["max_pending"] == k).all() and (r["steps"] == 1).all()
    ext = D.pack_externals(prog)
    for seed in (1, 2):
        rc, ev, par, res, _ = raw_trace(eng, seed, -1, 0, 1024)
        cev, cpar, cres = oracle.fuzz_trace(N.MODEL_PINGPONG3, ext, seed, -1, 0, blocked_mask=0b010)
        assert rc == 0 and res == cres and np.array_equal(ev, cev) and np.array_equal(par, cpar)
    from oracle import random_ddmin_binding as rd
    rd.lib()
    n_ext = len(prog)
    masks = np.stack([bits(range(n_ext), n_ext), bits([i for i in range(n_ext) if i != 3], n_ext),
                      bits([i for i in range(n_ext) if i != n_ext - 2], n_ext)])
    got = eng.random_test_batch(masks, 8, 1, -1)
    want = rd.random_test_batch(N.MODEL_PINGPONG3, ext, masks, 8, 1, -1, blocked_mask=0b010)
    for f in ("first_hit", "executions_run", "violation", "status"):
        assert np.array_equal(got[f], want[f]), f
    assert (got["status"] == 0).all()


@pytest.mark.parametrize("k", (65, 111))
def test_hard_kill_on_a_loaded_model(oracle, engine_mode, k):
    """The same family on pingpong3 loaded as IR; k <= 111 fits the IrModel 128 tier."""
    blob = model_ir.pingpong3_blob()
    oracle.load_model(blob)
    prog = hard_kill_program(k)
    ext = D.pack_externals(prog)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, blocked_mask=0b010))
    eng.load_model(blob)
    eng.set_externals(ext)
    gpu = eng.fuzz_batch(1, 64, -1, 0)
    cpu = oracle.fuzz_batch(N.MODEL_IR, ext, 1, 64, -1, 0, blocked_mask=0b010)
    assert_same(gpu, cpu)
    assert (gpu["status"] == 0).all() and (gpu["max_pending"] == k).all()


def test_uniq_ids_past_65535(oracle, engine_mode):
    """68 000 Uniq ids on 3 DepTracker nodes: the ids wrap at 2^16 and never reach the node field."""
    prog = uniq_wrap_program()
    eng, r = fuzz_case(oracle, N.MODEL_PINGPONG3, prog, 4, -1, engine_mode=engine_mode)
    assert (r["status"] == 0).all() and (r["n_nodes"] == 3).all() and (r["steps"] == 68000).all()
    ext = D.pack_externals(prog)
    rc, ev, par, res, _ = raw_trace(eng, 1, -1, 0, 1 << 18)
    cev, cpar, cres = oracle.fuzz_trace(N.MODEL_PINGPONG3, ext, 1, -1, 0, cap_events=1 << 18)
    assert rc == 0 and res == cres and len(ev) == len(cev) > 0xFFFF
    assert np.array_equal(ev, cev) and np.array_equal(par, cpar)
    assert int(ev["node"].max()) == 2


@pytest.mark.parametrize("model,prog,maxm,interval,flags", [
    (N.MODEL_RAFT5, D.raft5_program(), 50, 5, 1),                  # Raft5 256, recording, shared memory
    (N.MODEL_PINGPONG3, D.pingpong3_program(40), -1, 0, 0),        # HBM recording tier
    (N.MODEL_BCAST32, D.bcast32_program(2), 200, 0, 0),            # HBM recording tier
])
def test_event_cap_edge(oracle, model, prog, maxm, interval, flags):
    """fuzz_trace with cap_events equal to the trace length fits; one less ends with EVENT_OVF and an all-zero
    record.  A dep_parent buffer shorter than the tree receives its first cap_nodes parents, n_nodes the full count.
    (fuzz_trace always runs on the warp engine, so this test does not take the engine_mode fixture.)"""
    ext = D.pack_externals(prog)
    eng = D.Engine(D.SchedulerConfig(model, model_flags=flags))
    eng.set_externals(ext)
    for seed in (1, 7):
        cev, cpar, cres = oracle.fuzz_trace(model, ext, seed, maxm, interval, model_flags=flags)
        n = len(cev)
        rc, ev, par, res, _ = raw_trace(eng, seed, maxm, interval, n)
        assert rc == 0 and res == cres and np.array_equal(ev, cev) and np.array_equal(par, cpar)
        rc, _, _, res, _ = raw_trace(eng, seed, maxm, interval, n - 1)
        _, _, ores = oracle.fuzz_trace(model, ext, seed, maxm, interval, model_flags=flags, cap_events=n - 1)
        assert rc == N.ERR_CAPACITY and res == ores and int(res["status"]) == PS_EVENT_OVF
        overflowed_records_are_zero(np.array([res]))
        half = max(1, len(cpar) // 2)
        rc, ev, par, res, nn = raw_trace(eng, seed, maxm, interval, n, cap_nodes=half)
        cev2, cpar2, cres2 = oracle.fuzz_trace(model, ext, seed, maxm, interval, model_flags=flags, cap_nodes=half)
        assert rc == 0 and res == cres2 == cres and np.array_equal(ev, cev) and np.array_equal(ev, cev2)
        assert np.array_equal(par, cpar[:half]) and np.array_equal(cpar2, par)
        assert half < len(cpar) and nn == len(cpar) == int(cres["n_nodes"])


@pytest.mark.parametrize("ttl,flags,maxm,interval,n", [
    (4, 40, 900, 10, 200),       # PENDING_OVF at the 8192 clamp, mixed with violation 3 (40 floods received)
    (3, 0, 20000, 0, 64),        # past the clamp, node_cap 16 448 < the nodes of 20 000 deliveries: NODE_OVF too
])
def test_provenance_of_overflowed_prefixes(oracle, engine_mode, ttl, flags, maxm, interval, n):
    """fuzz_provenance over prefixes that end in PENDING_OVF or NODE_OVF, mixed with each other or with violating ones:
    the overflowed ones report DEMI_PV_PREFIX_FAILED, the others match the oracle's pruning."""
    ext = D.pack_externals(D.bcast32_program(ttl))
    eng = D.Engine(D.SchedulerConfig(N.MODEL_BCAST32, model_flags=flags))
    eng.set_externals(ext)
    res = eng.fuzz_batch(1, n, maxm, interval)
    assert_same(res, oracle.fuzz_batch(N.MODEL_BCAST32, ext, 1, n, maxm, interval, model_flags=flags))
    failed = np.nonzero(res["status"] != 0)[0]
    rest = np.nonzero(res["status"] == 0)[0]
    assert len(failed) > 10
    if ttl == 3:                 # every prefix overflows here, one way or the other
        assert (res["status"] == PS_NODE_OVF).sum() > 5 and (res["status"] == PS_PENDING_OVF).sum() > 5
    else:
        assert (res["violation"][rest] != 0).sum() > 20
    idx = np.concatenate([failed[:20], rest[:20]]).astype(np.uint32)
    idx = idx[np.random.default_rng(0).permutation(len(idx))]
    keep, out, rec = eng.fuzz_provenance(1, idx, maxm, interval)
    for j, i in enumerate(idx):
        k, o = oracle.fuzz_provenance(N.MODEL_BCAST32, ext, 1 + int(i), maxm, interval, keep.shape[1], model_flags=flags)
        assert int(out[j]["status"]) == int(o["status"]), int(i)
        if res["status"][i] != 0:
            assert int(out[j]["status"]) == N.PV_PREFIX_FAILED
        else:
            assert int(out[j]["status"]) == 0 and np.array_equal(k, keep[j]), int(i)
            for f in ("violation", "affected_mask", "n_trace", "n_kept"):
                assert o[f] == out[j][f], (f, int(i))


def dpor_caps(key, value):
    return dict(DPOR_BASE, **{key: value})


@pytest.mark.parametrize("key,edge,below,status", DPOR_BUCKET_EDGES, ids=[e[0] for e in DPOR_BUCKET_EDGES])
def test_dpor_cap_edges_bucket_queue(oracle, key, edge, below, status):
    """demi_dpor_batch (default ordering: the bucket queue) at each cap's smallest passing value and one below:
    counters, schedule hashes and violations equal the oracle's, and the status is 0 and then the cap's."""
    prog = [dpor_bucket_program()]
    res, _, _ = dpor_check(N.MODEL_RAFT5, prog, 1, 24, 400, oracle, **dpor_caps(key, edge))
    assert int(res[0]["status"]) == 0
    res, _, _ = dpor_check(N.MODEL_RAFT5, prog, 1, 24, 400, oracle, **dpor_caps(key, below))
    assert int(res[0]["status"]) == status


@pytest.mark.parametrize("key,edge,below,status", DPOR_HEAP_EDGES, ids=[e[0] for e in DPOR_HEAP_EDGES])
def test_dpor_cap_edges_arvind_heap(oracle, key, edge, below, status):
    """demi_dpor_batch_ex with ArvindDistanceOrdering (the binary heap), seeded, at the same two points."""
    dext, ev, par, steps = raft5_seed_world(oracle)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    prog = dext[np.arange(len(dext)) != 7]
    for value, want in ((edge, 0), (below, status)):
        caps = dict(DPOR_BASE, heap_cap=1 << 16); caps[key] = value
        res, hashes = eng.dpor_batch_ex([prog], steps, DPOR_HEAP_BUDGET, seed=(ev, par),
                                        flags=N.DF_ARVIND_ORDERING | N.DF_PRIORITIZE_PENDING, stop_if_found=False,
                                        want_hashes=True, **caps)
        r, h = dpor_heap_instance(oracle, dext, ev, par, steps, **{key: value})
        for f in DPOR_FIELDS:
            assert res[0][f] == r[f], (key, value, f)
        assert hashes[0][:int(r["interleavings"])].tolist() == h.tolist()
        assert int(r["status"]) == want


def test_dpor_queue_edge(oracle):
    """256 messages on one (snd, rcv) FIFO fit DPOR_QCAP; 257 end the search with QUEUE_OVF, on both sides."""
    res, _, _ = dpor_check(N.MODEL_PINGPONG3, [dpor_queue_program(256), dpor_queue_program(257)], 0, 4, 8, oracle)
    assert [int(x) for x in res["status"]] == [0, DS_QUEUE_OVF]


def test_dpor_follows_the_whole_initial_trace(oracle):
    """A seeded search whose initial trace is longer than max_messages + 2 follows all of it, as the oracle does."""
    ext_all = D.pack_externals(D.raft5_program())
    dext = ext_all[(ext_all["kind"] == N.EXT_SEND) | (ext_all["kind"] == N.EXT_START)]
    ev, par, _ = oracle.fuzz_trace(N.MODEL_RAFT5, ext_all, 1, 40, 5, model_flags=1)
    r, h = long_seed_search(oracle, dext, ev, par)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    res, hashes = eng.dpor_batch_ex([dext[np.arange(len(dext)) != 5]], 8, 30, seed=(ev, par),
                                    flags=N.DF_PRIORITIZE_PENDING, looking_for=1, stop_if_found=True, heap_cap=1 << 17,
                                    want_hashes=True)
    for f in DPOR_FIELDS:
        assert res[0][f] == r[f], f
    assert hashes[0][:int(r["interleavings"])].tolist() == h.tolist()
