"""Recording many programs' executions in one call (demi_fuzz_traces_many): per trace, the status, EventTrace, count and
record of demi_set_externals + demi_random_test_trace on a handle of its own (demi_fuzz_trace for a full program), the
DepTracker tree of demi_fuzz_trace or of the C oracle's oracle_fuzz_trace over the kept subsequence, whichever traces
share the launches; and the pipelines it feeds, against the per-trace loop."""
import ctypes as C

import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
from demi_b200.fuzzer import ClientCommandGenerator, Fuzzer, FuzzerWeights, fuzzer_config
from oracle import binding as O
import ir_gen
from test_random_ddmin_gpu import PP_HK, engine, random_masks
from test_random_ddmin_oracle import PP_FLAGS, RAFT_FLAGS, RAFT_HK, RAFT_PART, RAFT_WQ, bits
from test_capacity_edges_oracle import PS_EVENT_OVF, PS_PENDING_OVF, SMALL_CAPS, bcast32_small_cap

pytestmark = pytest.mark.gpu
CAP_EV, CAP_NODES = 1024, 1024


def raft5_campaign(n, num_events=(6, 10, 14)):
    """Fuzzer programs of a raft5 campaign of mixed lengths (the Fuzzer draws Kill and Partition events)"""
    return [Fuzzer(num_events[s % len(num_events)], FuzzerWeights(), ClientCommandGenerator(2), D.raft5_program()[:-1],
                   seed=7000 + s).generateFuzzTest() for s in range(n)]


def single(eng, prog, mask, seed, maxm, looking, interval, cap_events=CAP_EV):
    """demi_set_externals + demi_random_test_trace: (rc, events, n_events, result)"""
    ext = D.pack_externals(prog)
    L = N.lib()
    rc = L.demi_set_externals(eng._h, ext.ctypes.data if len(ext) else None, len(ext))
    ev = np.zeros(cap_events, dtype=N.EVENT_DTYPE)
    n = C.c_uint32()
    res = np.zeros(1, dtype=N.RESULT_DTYPE)
    if rc == 0:
        m = np.ascontiguousarray(mask if mask is not None else bits(range(len(prog)), len(prog)), dtype=np.uint64)
        p = N.FuzzParams(seed, 1, maxm, interval, looking, 0)
        rc = L.demi_random_test_trace(eng._h, m.ctypes.data, len(m), C.byref(p), seed, ev.ctypes.data, cap_events,
                                      C.byref(n), res.ctypes.data)
    return rc, ev, n.value, res[0]


def full_tree(eng, prog, seed, maxm, looking, interval, cap_events=CAP_EV, cap_nodes=CAP_NODES):
    """demi_set_externals + demi_fuzz_trace's tree: (events, dep_parent)"""
    eng.set_externals(prog)
    ev, par, _ = eng.fuzz_trace(seed, maxm, interval, looking, cap_events=cap_events, cap_nodes=cap_nodes)
    return ev, par


def kept(prog, mask):
    return [e for i, e in enumerate(prog) if mask is None or (int(mask[i >> 6]) >> (i & 63)) & 1]


def check(eng, ref, progs, seeds, maxms, lookings, interval, masks=None, cap_events=CAP_EV, cap_nodes=None, want=None,
          oracle=None, mask_words=None):
    """demi_fuzz_traces_many over progs equals the single sequence on `ref` per trace; the trees equal demi_fuzz_trace's
    (full programs) and, on every `oracle`-th trace, the C oracle's over the subsequence.  Returns the call's outputs."""
    out = eng.fuzz_traces_many(progs, seeds, maxms, lookings, interval, masks=masks, cap_events=cap_events,
                               cap_nodes=cap_nodes, mask_words=mask_words)
    ev, ne, par, nn, res, status = out
    for t, prog in enumerate(progs):
        mask = None if masks is None else masks[t]
        rc, ev1, n1, r1 = single(ref, prog, mask, seeds[t], maxms[t], lookings[t], interval, cap_events)
        assert int(status[t]) == rc, (t, int(status[t]), rc, eng.last_error())
        if want is not None:
            assert rc == want[t], (t, rc)
        if rc:
            assert not ev[t].view(np.uint8).any(), t                       # zeros where the events would be
            if cap_nodes:
                assert not par[t].any(), t
            if rc == N.ERR_CAPACITY and n1:                                 # a prefix status: its count and result
                assert int(ne[t]) == n1 and res[t].tobytes() == r1.tobytes(), t
            continue
        assert int(ne[t]) == n1 and res[t].tobytes() == r1.tobytes(), t
        assert ev[t, :n1].tobytes() == ev1[:n1].tobytes(), t
        if cap_nodes and mask is None:
            fe, fp = full_tree(ref, prog, seeds[t], maxms[t], lookings[t], interval, cap_events, cap_nodes)
            assert fe.tobytes() == ev1[:n1].tobytes()
            assert int(nn[t]) == len(fp) and par[t, :len(fp)].tobytes() == fp.tobytes(), t
        if oracle is not None and t % oracle[0] == 0:
            model, flags, cfg = oracle[1], oracle[2], oracle[3] if len(oracle) > 3 else {}
            cev, cpar, cres = O.fuzz_trace(model, D.pack_externals(kept(prog, mask)), seeds[t], maxms[t], interval,
                                           model_flags=flags, looking_for=lookings[t], cap_events=cap_events,
                                           cap_nodes=cap_nodes or CAP_NODES, **cfg)
            assert cev.tobytes() == ev[t, :n1].tobytes(), t
            if cap_nodes:
                assert par[t, :int(nn[t])].tobytes() == cpar.tobytes(), t
    return out


def mixed_masks(progs, rng, mw):
    """per trace: all ones, a random subsequence, or one that drops an event between two WaitQuiescence"""
    out = np.zeros((len(progs), mw), dtype=np.uint64)
    for t, prog in enumerate(progs):
        n = len(prog)
        if t % 3 == 0:
            m = bits(range(n), n)
        elif t % 3 == 1:
            m = random_masks(n, 1, rng)[0]
        else:
            wq = [i for i, e in enumerate(prog) if isinstance(e, D.WaitQuiescence)]
            drop = {i + 1 for i in wq[:-1] if i + 1 < n and (i + 2 < n and isinstance(prog[i + 2], D.WaitQuiescence))}
            m = bits([i for i in range(n) if i not in drop], n)
        out[t, :len(m)] = m
    return out


@pytest.fixture(scope="module")
def raft():
    return engine(N.MODEL_RAFT5, RAFT_FLAGS, {}), engine(N.MODEL_RAFT5, RAFT_FLAGS, {})


def test_raft5_mixed_programs_full_and_masked(raft):
    """Campaign programs of mixed lengths with Kill / Partition, a HardKill program (the HBM variant) and one with
    leading and repeated WaitQuiescence; full programs with trees, then masks (adjacent and leading WaitQuiescence)."""
    eng, ref = raft
    progs = raft5_campaign(12) + [RAFT_HK, RAFT_WQ, RAFT_PART]
    n = len(progs)
    seeds = [100 + 13 * t for t in range(n)]
    maxms = [40 + 5 * (t % 4) for t in range(n)]
    lookings = [0 if t % 2 else 1 for t in range(n)]
    check(eng, ref, progs, seeds, maxms, lookings, 5, cap_nodes=CAP_NODES, oracle=(3, N.MODEL_RAFT5, RAFT_FLAGS))
    mw = max(1, (max(len(p) for p in progs) + 63) // 64)
    masks = mixed_masks(progs, np.random.default_rng(4), mw)
    # RAFT_WQ keeps its leading WaitQuiescence and loses its last Send: two adjacent ones
    wq = len(progs) - 2
    masks[wq, :] = 0
    masks[wq, :1] = bits([i for i in range(len(RAFT_WQ)) if i not in (len(RAFT_WQ) - 2,)], len(RAFT_WQ))
    check(eng, ref, progs, seeds, maxms, lookings, 5, masks=masks, cap_nodes=CAP_NODES,
          oracle=(2, N.MODEL_RAFT5, RAFT_FLAGS), mask_words=mw)


def test_pingpong3_and_bcast32():
    pp = [PP_HK, D.pingpong3_program(n_sends=6), PP_HK[:-3] + [D.WaitQuiescence(), D.WaitQuiescence()],
          D.pingpong3_program(n_sends=40)]
    eng, ref = D.Engine(D.SchedulerConfig(N.MODEL_PINGPONG3, PP_FLAGS)), D.Engine(D.SchedulerConfig(N.MODEL_PINGPONG3, PP_FLAGS))
    # the third program has adjacent WaitQuiescence, which demi_set_externals refuses: it fails alone
    check(eng, ref, pp, [7, 8, 9, 10], [40, 30, 40, 200], [0, 0, 0, 0], 0, cap_nodes=CAP_NODES, want=[0, 0, N.ERR_INVALID, 0],
          oracle=(1, N.MODEL_PINGPONG3, PP_FLAGS))
    # PP_HK without its HardKill and the two Sends after it: a subsequence with adjacent WaitQuiescence, accepted
    pp[2] = PP_HK
    hk = [i for i, e in enumerate(PP_HK) if isinstance(e, D.HardKill)][0]
    masks = np.vstack([bits(range(len(p)), len(p))[:1] for p in pp]).astype(np.uint64)
    masks[2] = bits([i for i in range(len(PP_HK)) if i not in (hk, hk + 1, hk + 2)], len(PP_HK))[:1]
    check(eng, ref, pp, [7, 8, 9, 10], [40, 30, 40, 200], [0, 0, 0, 0], 0, masks=masks, cap_nodes=CAP_NODES,
          want=[0, 0, 0, 0], oracle=(1, N.MODEL_PINGPONG3, PP_FLAGS), mask_words=1)
    bc = [D.bcast32_program(ttl=2), D.bcast32_program(ttl=3)]
    eng, ref = D.Engine(D.SchedulerConfig(N.MODEL_BCAST32, 0)), D.Engine(D.SchedulerConfig(N.MODEL_BCAST32, 0))
    check(eng, ref, bc, [3, 4], [30, 60], [0, 0], 0, cap_events=8192, cap_nodes=4096, oracle=(1, N.MODEL_BCAST32, 0))


@pytest.mark.parametrize("timers", [False, True])
def test_loaded_models(timers):
    done = 0
    for s in range(1, 200):
        m = ir_gen.generate(s)
        if m.uses_timers != timers:
            continue
        progs = [ir_gen.program(m, s), ir_gen.program(m, s + 1000, hard_kill=True), ir_gen.program(m, s + 2000)]
        O.load_model(m.blob)
        eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, m.flags))
        eng.load_model(m.blob)
        ref = D.Engine(D.SchedulerConfig(N.MODEL_IR, m.flags))
        ref.load_model(m.blob)
        seeds = [s + k for k in range(len(progs))]
        check(eng, ref, progs, seeds, [40, 30, 50], [0, 0, 0], 2, cap_nodes=CAP_NODES, oracle=(1, N.MODEL_IR, m.flags))
        mw = max(1, (max(len(p) for p in progs) + 63) // 64)
        check(eng, ref, progs, seeds, [40, 30, 50], [0, 0, 0], 2, masks=mixed_masks(progs, np.random.default_rng(s), mw),
              cap_nodes=CAP_NODES, oracle=(1, N.MODEL_IR, m.flags), mask_words=mw)
        done += 1
        if done == 3:
            return
    raise AssertionError("not enough generated models")


@pytest.mark.parametrize("c", [dict(strategy=1), dict(rules=[(0b00110, 0b11111, 1 << 5, 0)]), dict(blocked=(4,)),
                               dict(ignore_timers=True)], ids=["fifo", "filter", "blocked", "ignore_timers"])
def test_switches(c):
    """One handle per configuration: SrcDstFIFO (the HBM variant for every program), a user filter, a blocked actor and
    ignoreTimers, each against the single calls under the same configuration and the oracle."""
    def mk():
        if c.get("ignore_timers"):
            return D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=RAFT_FLAGS, ignoreTimers=True))
        return engine(N.MODEL_RAFT5, RAFT_FLAGS, c)
    eng, ref = mk(), mk()
    progs = raft5_campaign(6) + [RAFT_WQ]
    if not c.get("strategy"):
        progs.append(RAFT_HK)
    n = len(progs)
    seeds, maxms, lookings = [30 + t for t in range(n)], [60] * n, [0] * n
    cfg = dict(strategy=c.get("strategy", 0), blocked_mask=sum(1 << b for b in c.get("blocked", ())),
               ignore_timers=1 if c.get("ignore_timers") else 0)
    O.set_user_filter(c.get("rules", []))
    try:
        check(eng, ref, progs, seeds, maxms, lookings, 5, cap_nodes=CAP_NODES, oracle=(2, N.MODEL_RAFT5, RAFT_FLAGS, cfg))
    finally:
        O.set_user_filter([])
    if c.get("strategy"):
        # SrcDstFIFO offers no HardKill: that trace fails alone, as plan_launch refuses it
        st = eng.fuzz_traces_many(progs + [RAFT_HK], seeds + [1], maxms + [60], lookings + [0], 5)[5]
        assert list(st) == [0] * n + [N.ERR_INVALID]


def test_per_trace_failures(raft):
    eng, ref = raft
    progs = raft5_campaign(4)
    seeds, maxms = [11, 12, 13, 14], [50] * 4
    base = eng.fuzz_traces_many(progs, seeds, maxms, 0, 5)
    lens = [int(x) for x in base[1]]
    bad = [D.Start(0), D.WaitQuiescence(), D.WaitQuiescence()]          # demi_set_externals rejects it
    big = [D.Start(a) for a in range(5)] + [D.Send(0, 2, k) for k in range(1100)]     # tosend_cap 2048: no variant
    ps = [progs[0], bad, progs[1], [], progs[2], big, progs[3]]
    sd, mm, lf = [11, 1, 12, 1, 13, 1, 14], [50] * 7, [0] * 7
    out = check(eng, ref, ps, sd, mm, lf, 5, cap_nodes=CAP_NODES,
                want=[0, N.ERR_INVALID, 0, N.ERR_STATE, 0, N.ERR_CAPACITY, 0])
    assert "trace 1" in eng.last_error()
    for k, t in enumerate([0, 2, 4, 6]):
        assert out[0][t].tobytes() == base[0][k].tobytes()
    # a mask that keeps no event
    mw = max(1, (max(len(p) for p in progs) + 63) // 64)
    masks = np.vstack([np.pad(bits(range(len(p)), len(p)), (0, mw - max(1, (len(p) + 63) // 64))) for p in progs])
    masks[1] = 0
    check(eng, ref, progs, seeds, maxms, [0] * 4, 5, masks=masks, mask_words=mw, want=[0, N.ERR_INVALID, 0, 0])
    # DEMI_PS_EVENT_OVF at the exact edge: cap_events = the longest recording passes, one less fails that trace alone
    top = int(np.argmax(lens))
    check(eng, ref, progs, seeds, maxms, [0] * 4, 5, cap_events=lens[top], cap_nodes=CAP_NODES, want=[0] * 4)
    want = [N.ERR_CAPACITY if lens[t] > lens[top] - 1 else 0 for t in range(4)]
    out = check(eng, ref, progs, seeds, maxms, [0] * 4, 5, cap_events=lens[top] - 1, cap_nodes=CAP_NODES, want=want)
    assert int(out[4][top]["status"]) == PS_EVENT_OVF


def test_pending_capacity_edge():
    """A pending-set status at its exact edge (test_capacity_edges_oracle's small-capacity bcast32 program): executions
    that end with exactly `cap` pending messages record, the ones one past it fail alone with DEMI_PS_PENDING_OVF; one
    program shared by every trace through ext_offsets 0."""
    n_flood, n_quiet, cap, _, _ = SMALL_CAPS[0]
    prog = bcast32_small_cap(n_flood, n_quiet)
    eng, ref = D.Engine(D.SchedulerConfig(N.MODEL_BCAST32, 0)), D.Engine(D.SchedulerConfig(N.MODEL_BCAST32, 0))
    seeds = list(range(1, 65))
    out = check(eng, ref, [prog] * len(seeds), seeds, [-1] * len(seeds), [0] * len(seeds), 0, cap_events=8192)
    shared = eng.fuzz_traces_many(prog, seeds, -1, 0, 0, cap_events=8192)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(out, shared) if a is not None)
    st = out[4]["status"]
    assert (st == PS_PENDING_OVF).any() and (out[5] == N.ERR_CAPACITY).sum() == (st != 0).sum()
    assert (out[4]["max_pending"][st == 0] == cap).any()


def test_grouping_permutation_split_and_shared_program(raft, monkeypatch):
    eng, ref = raft
    progs = raft5_campaign(9) + [RAFT_HK]
    n = len(progs)
    seeds, maxms, lookings = [200 + t for t in range(n)], [45] * n, [0] * n
    full = eng.fuzz_traces_many(progs, seeds, maxms, lookings, 5, cap_nodes=CAP_NODES)

    def same(sel, got):
        for k, t in enumerate(sel):
            assert got[5][k] == full[5][t] and got[1][k] == full[1][t] and got[4][k].tobytes() == full[4][t].tobytes()
            assert got[0][k].tobytes() == full[0][t].tobytes() or got[0][k, :got[1][k]].tobytes() == full[0][t, :full[1][t]].tobytes()
            assert got[2][k, :got[3][k]].tobytes() == full[2][t, :full[3][t]].tobytes()
    order = list(np.random.default_rng(1).permutation(n))
    same(order, eng.fuzz_traces_many([progs[t] for t in order], [seeds[t] for t in order], maxms, lookings, 5,
                                     cap_nodes=CAP_NODES))
    same(range(0, 4), eng.fuzz_traces_many(progs[:4], seeds[:4], 45, 0, 5, cap_nodes=CAP_NODES))
    same(range(4, n), eng.fuzz_traces_many(progs[4:], seeds[4:], 45, 0, 5, cap_nodes=CAP_NODES))
    # forced launch splits: three slots per launch
    monkeypatch.setenv("DEMI_TEST_FUZZ_MANY_SLOTS", "3")
    same(range(n), eng.fuzz_traces_many(progs, seeds, maxms, lookings, 5, cap_nodes=CAP_NODES))
    assert eng.stats().kernel_launches >= 2 * 4
    monkeypatch.delenv("DEMI_TEST_FUZZ_MANY_SLOTS")
    # one program through ext_offsets 0 equals demi_fuzz_traces(_tree) for the same seeds
    prog = D.raft5_program(client_cmds=2)
    idx = [3, 17, 40, 41, 99, 250]
    got = eng.fuzz_traces_many(prog, [1000 + i for i in idx], 50, 0, 5, cap_nodes=CAP_NODES)
    assert not got[5].any()
    eng.set_externals(prog)
    ev, ne, par, nn, res = eng.fuzz_traces_tree(1000, idx, 50, 5, cap_events=CAP_EV, cap_nodes=CAP_NODES)
    ev2, ne2, res2 = eng.fuzz_traces(1000, idx, 50, 5, cap_events=CAP_EV)
    for k in range(len(idx)):
        assert got[1][k] == ne[k] == ne2[k] and got[4][k].tobytes() == res[k].tobytes() == res2[k].tobytes()
        assert got[0][k, :ne[k]].tobytes() == ev[k, :ne[k]].tobytes() == ev2[k, :ne[k]].tobytes()
        assert got[3][k] == nn[k] and got[2][k, :nn[k]].tobytes() == par[k, :nn[k]].tobytes()


def test_handle_untouched_and_rejected_arguments(raft):
    eng, _ = raft
    prog = D.raft5_program(client_cmds=1)
    eng.set_externals(prog)
    before = eng.fuzz_trace(5, 50, 5)
    eng.fuzz_traces_many(raft5_campaign(3), [1, 2, 3], 50, 0, 5)
    after = eng.fuzz_trace(5, 50, 5)
    assert before[0].tobytes() == after[0].tobytes() and before[1].tobytes() == after[1].tobytes()
    L = N.lib()
    ext = D.pack_externals(prog)
    z, n_ext = np.zeros(1, dtype=np.uint32), np.array([len(ext)], dtype=np.uint32)
    sd, mm, lf = np.zeros(1, dtype=np.int64), np.array([50], dtype=np.int32), np.zeros(1, dtype=np.uint32)
    p = N.FuzzParams(0, 0, -1, 5, 0, 0)
    ev = np.zeros(64, dtype=N.EVENT_DTYPE)
    ne, nn, st = np.zeros(1, dtype=np.uint32), np.zeros(1, dtype=np.uint32), np.zeros(1, dtype=np.int32)
    par = np.zeros(70000, dtype=np.uint16)
    mask = np.zeros(1, dtype=np.uint64)

    def call(masks=None, mw=0, events=ev.ctypes.data, parent=None, cap_nodes=0, nodes=None, n_externals=n_ext):
        return L.demi_fuzz_traces_many(eng._h, 1, ext.ctypes.data, z.ctypes.data, n_externals.ctypes.data, masks, mw,
                                       sd.ctypes.data, mm.ctypes.data, lf.ctypes.data, C.byref(p), events, 64,
                                       ne.ctypes.data, parent, cap_nodes, nodes, None, st.ctypes.data)
    assert call(events=None) == N.ERR_INVALID
    assert call(masks=mask.ctypes.data, mw=0) == N.ERR_INVALID                       # mask_words * 64 < n_externals
    assert call(parent=par.ctypes.data, cap_nodes=0, nodes=nn.ctypes.data) == N.ERR_INVALID
    assert call(parent=par.ctypes.data, cap_nodes=65537, nodes=nn.ctypes.data) == N.ERR_INVALID
    assert call(parent=par.ctypes.data, cap_nodes=64, nodes=None) == N.ERR_INVALID
    assert call() == N.OK


def campaign_violations(eng, want, seed_base=1, pseed=500_000):
    fz = Fuzzer(20, FuzzerWeights(), ClientCommandGenerator(2), D.raft5_program()[:-1])
    eng.set_fuzzer(fuzzer_config(fz), D.raft5_program()[:-1])
    res = eng.fuzz_campaign(seed_base, 1 << 14, 50, 5, pseed)
    out = []
    for i in np.nonzero((res["violation"] != 0) & (res["status"] == 0))[0][:want]:
        out.append((D.unpack_externals(eng.fuzzer_program(pseed + int(i))), seed_base + int(i), int(res["violation"][i])))
    assert len(out) == want
    return out


def test_pipelines_equal_the_per_violation_loop(raft):
    """campaign violations -> demi_fuzz_traces_many -> demi_set_traces -> demi_ddmin_many (and, with trees,
    demi_incremental_ddmin_many) equal the same pipelines fed by demi_set_externals + demi_fuzz_trace per violation."""
    eng, ref = raft
    vs = campaign_violations(eng, 12)
    progs, seeds, codes = [v[0] for v in vs], [v[1] for v in vs], [v[2] for v in vs]
    ev, ne, par, nn, res, st = eng.fuzz_traces_many(progs, seeds, 50, 0, 5, cap_nodes=CAP_NODES)
    assert not st.any()
    loop = [full_tree(ref, p, s, 50, 0, 5) for p, s in zip(progs, seeds)]
    for t in range(len(vs)):
        assert ev[t, :ne[t]].tobytes() == loop[t][0].tobytes() and par[t, :nn[t]].tobytes() == loop[t][1].tobytes()
    lf = np.array(codes, dtype=np.uint32)

    def same(a, b):                                  # every output, the records' reserved words aside
        assert len(a) == len(b)
        for u, v in zip(a, b):
            u, v = np.asarray(u), np.asarray(v)
            if u.dtype.names:
                assert all(np.array_equal(u[f], v[f]) for f in u.dtype.names if f != "reserved")
            else:
                assert u.tobytes() == v.tobytes()
    packed = [D.pack_externals(p) for p in progs]
    eng.set_traces((ev, ne), packed)
    ref.set_traces([x[0] for x in loop], packed)
    a, b = eng.ddmin_many(lf), ref.ddmin_many(lf)
    same(a, b)
    a = eng.incremental_ddmin_many(progs, 50, 200, [(ev[t, :ne[t]], par[t, :nn[t]]) for t in range(len(vs))], codes)
    b = ref.incremental_ddmin_many(progs, 50, 200, loop, codes)
    same(a, b)


def test_random_ddmin_verified_traces():
    """demi_random_ddmin_many, then the MCS traces recorded in one call with seeds seed + mcs_first_hit: randomDDMin_many's
    verified traces (pingpong3, whose violation shows under randomDDMin's invariant interval 0, HardKill included)."""
    cfg = D.SchedulerConfig(N.MODEL_PINGPONG3, PP_FLAGS)
    eng, ref = D.Engine(cfg), D.Engine(cfg)
    execs, seeds = [], []
    for k, prog in enumerate([PP_HK, D.pingpong3_program(n_sends=6), D.pingpong3_program(n_sends=4),
                              D.pingpong3_program(n_sends=8)] * 3):
        seed = 7 + 11 * k
        ref.set_externals(prog)
        tr, _, r = ref.fuzz_trace(seed, 40, 0)
        if int(r["status"]) == 0 and int(r["violation"]):
            execs.append((tr, prog, int(r["violation"])))
            seeds.append(seed)
    assert len(execs) >= 3
    results, status = D.randomDDMin_many(cfg, execs, 16, seeds, engine=ref)
    progs = [list(x[1]) for x in execs]
    mw = max(1, (max(len(p) for p in progs) + 63) // 64)
    mcs, _, _, out, st2 = eng.random_ddmin_many(progs, 16, seeds, [len(x[0]) for x in execs], [x[2] for x in execs],
                                                mask_words=mw)
    assert list(st2) == list(status)
    sel = [t for t in range(len(execs)) if not status[t] and results[t][2] is not None and len(results[t][0]) < len(progs[t])]
    assert sel
    got = eng.fuzz_traces_many([progs[t] for t in sel], [seeds[t] + int(out[t]["mcs_first_hit"]) for t in sel],
                               [len(execs[t][0]) for t in sel], [execs[t][2] for t in sel], 0, masks=mcs[sel],
                               cap_events=65536, mask_words=mw)
    assert not got[5].any()
    for k, t in enumerate(sel):
        verified = results[t][2]
        assert got[0][k, :got[1][k]].tobytes() == np.asarray(verified, dtype=N.EVENT_DTYPE).tobytes(), t
