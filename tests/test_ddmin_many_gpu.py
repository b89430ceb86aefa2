"""Many traces at once: demi_fuzz_traces, demi_set_traces, demi_replay_batch_many and demi_ddmin_many against the
single-trace entry points and the CPU oracle, record by record."""
import ctypes as C

import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N

pytestmark = pytest.mark.gpu

MAXM, INTERVAL, RAFT_FLAGS = 50, 5, 1          # the headline workload (bench.py)
PS_EVENT_OVF = 4                               # DEMI_PS_EVENT_OVF


def raft_engine(prog):
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=RAFT_FLAGS))
    eng.set_externals(prog)
    return eng


def raft_hits(eng, n_seeds, want):
    res = eng.fuzz_batch(1, n_seeds, MAXM, INTERVAL)
    hits = np.nonzero((res["violation"] != 0) & (res["status"] == 0))[0]
    assert len(hits) >= want
    return hits[:want].astype(np.uint32), res


def fuzz_traces_raw(eng, seed_base, idx, maxm, interval, cap):
    """demi_fuzz_traces with its return code: the records are filled whether or not some execution fails."""
    p = N.FuzzParams(seed_base, len(idx), maxm, interval, 0, 0)
    ev = np.zeros((len(idx), cap), dtype=N.EVENT_DTYPE)
    ne = np.zeros(len(idx), dtype=np.uint32)
    res = np.zeros(len(idx), dtype=N.RESULT_DTYPE)
    i32 = np.ascontiguousarray(idx, dtype=np.uint32)
    rc = N.lib().demi_fuzz_traces(eng._h, C.byref(p), i32.ctypes.data, len(idx), ev.ctypes.data, cap, ne.ctypes.data,
                                  res.ctypes.data)
    return rc, ev, ne, res


def fuzz_trace_raw(eng, seed, maxm, interval, cap):
    """demi_fuzz_trace with its return code, count and result, which it reports also when it fails."""
    p = N.FuzzParams(seed, 1, maxm, interval, 0, 0)
    ev = np.zeros(cap, dtype=N.EVENT_DTYPE)
    n = C.c_uint32()
    res = np.zeros(1, dtype=N.RESULT_DTYPE)
    rc = N.lib().demi_fuzz_trace(eng._h, C.byref(p), seed, ev.ctypes.data, cap, C.byref(n), None, 0, None, res.ctypes.data)
    return rc, ev[:n.value].copy() if rc == N.OK else None, n.value, res[0]


def compare_fuzz_traces(eng, oracle, model, ext, seed_base, idx, maxm, interval, cap, flags):
    """Record by record: demi_fuzz_traces == demi_fuzz_trace (events, count, result, failure) == the oracle's fuzz_trace."""
    rc, ev, ne, res = fuzz_traces_raw(eng, seed_base, idx, maxm, interval, cap)
    failing = res["status"] != 0
    assert rc == (N.ERR_CAPACITY if failing.any() else N.OK)
    if failing.any():
        assert "demi_fuzz_traces: execution %d " % int(np.argmax(failing)) in eng.last_error()
    for i, k in enumerate(idx):
        seed = seed_base + int(k)
        src, sev, sn, sr = fuzz_trace_raw(eng, seed, maxm, interval, cap)
        assert ne[i] == sn and res[i] == sr, (i, seed)
        if src != N.OK:
            assert src == N.ERR_CAPACITY and failing[i], (i, seed)
            if not failing.all():
                assert (ev[i].view(np.uint8)[:16] == 0).all()           # no events of a failing execution
            continue
        assert not failing[i] and (ev[i, :ne[i]] == sev).all(), (i, seed)
        if oracle is not None:
            cev, _, cr = oracle.fuzz_trace(model, ext, seed, maxm, interval, model_flags=flags, cap_events=cap)
            assert (cev == sev).all() and cr == sr, (i, seed)
    return ev, ne, res


def test_fuzz_traces_raft5_headline(oracle):
    prog = D.raft5_program()
    ext = D.pack_externals(prog)
    eng = raft_engine(prog)
    hits, res = raft_hits(eng, 20000, 256)
    quiet = np.nonzero(res["violation"] == 0)[0][:64].astype(np.uint32)
    idx = np.concatenate([hits, quiet])
    ev, ne, r = compare_fuzz_traces(eng, oracle, N.MODEL_RAFT5, ext, 1, idx, MAXM, INTERVAL, 4096, RAFT_FLAGS)
    assert (r["violation"][:256] != 0).all() and (r["violation"][256:] == 0).all() and (r["status"] == 0).all()
    # a cap_events too small for some executions: those fail as demi_fuzz_trace does, the others are recorded
    small = int(np.median(ne[:64]))
    _, _, r = compare_fuzz_traces(eng, oracle, N.MODEL_RAFT5, ext, 1, idx[:64], MAXM, INTERVAL, small, RAFT_FLAGS)
    assert (r["status"] == PS_EVENT_OVF).any() and (r["status"] == 0).any()


def test_fuzz_traces_pingpong_bcast(oracle):
    prog = [D.Start(a) for a in range(3)] + [D.Send(k % 3, 1, k) for k in range(10)]
    prog += [D.WaitQuiescence(), D.Partition(0, 1), D.Kill(2)] + [D.Send(k % 3, 1, 100 + k) for k in range(10)]
    prog += [D.WaitQuiescence(), D.UnPartition(0, 1), D.Start(2)] + [D.Send(k % 3, 1, 200 + k) for k in range(9)]
    for model, flags, p, maxm, interval in ((N.MODEL_PINGPONG3, 1 | (6 << 8), prog, -1, 0),
                                            (N.MODEL_BCAST32, 3, D.bcast32_program(2), 120, 10)):
        eng = D.Engine(D.SchedulerConfig(model, model_flags=flags))
        eng.set_externals(p)
        idx = np.arange(0, 96, 3, dtype=np.uint32)
        compare_fuzz_traces(eng, oracle, model, D.pack_externals(p), 5, idx, maxm, interval, 65536, flags)


def test_fuzz_traces_loaded_model_with_timers(oracle):
    from test_ir_timers_oracle import ELECTION_INTERVAL, ELECTION_MAXM, election_model, election_program
    m = election_model()
    eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, model_flags=m.flags))
    eng.load_model(m.blob)
    eng.set_externals(election_program())
    oracle.load_model(m.blob)
    compare_fuzz_traces(eng, oracle, N.MODEL_IR, D.pack_externals(election_program()), 1, np.arange(40, dtype=np.uint32),
                        ELECTION_MAXM, ELECTION_INTERVAL, 65536, m.flags)


def raft_set(n, client_cmds=0, seeds=40000):
    prog = D.raft5_program(client_cmds=client_cmds)
    ext = D.pack_externals(prog)
    eng = raft_engine(prog)
    hits, res = raft_hits(eng, seeds, n)
    ev, ne, r = eng.fuzz_traces(1, hits, MAXM, INTERVAL, cap_events=1024)
    return eng, ext, ev, ne, r["violation"].astype(np.uint32)


def long_raft_trace(oracle):
    """One ~2 000-event raft5 trace (max_messages 1000)."""
    prog = D.raft5_program(client_cmds=6)
    ext = D.pack_externals(prog)
    res = oracle.fuzz_batch(N.MODEL_RAFT5, ext, 1, 400, 1000, 0, model_flags=RAFT_FLAGS)
    k = int(np.argmax(res["n_events"]))
    ev, _, r = oracle.fuzz_trace(N.MODEL_RAFT5, ext, 1 + k, 1000, 0, model_flags=RAFT_FLAGS)
    assert len(ev) > 1000
    return ev, ext, int(r["violation"])


def random_masks(n_ext, n, rng):
    mw = max(1, (n_ext + 63) // 64)
    bits = rng.integers(0, 2, size=(n, n_ext)).astype(np.uint64)
    m = np.zeros((n, mw), dtype=np.uint64)
    for j in range(n_ext):
        m[:, j >> 6] |= bits[:, j] << np.uint64(j & 63)
    m[0] = 0
    for j in range(n_ext):
        m[0, j >> 6] |= np.uint64(1) << np.uint64(j & 63)
    return m


def test_replay_batch_many_matches_single_and_oracle(oracle):
    eng, ext, ev, ne, viol = raft_set(12, client_cmds=6)
    lev, lext, lcode = long_raft_trace(oracle)
    traces = [ev[i, :ne[i]].copy() for i in range(len(ne))] + [lev]
    exts = [ext] * len(ne) + [lext]
    codes = list(viol) + [lcode]
    eng.set_traces(traces, exts)
    rng = np.random.default_rng(3)
    per = 70
    tr = np.repeat(np.arange(len(traces), dtype=np.uint32), per)
    masks = np.concatenate([random_masks(len(exts[t]), per, rng) for t in range(len(traces))])
    perm = rng.permutation(len(tr))
    tr, masks = tr[perm], masks[perm]
    for flags in (0, N.RF_FILTER_KNOWN_ABSENTS, N.RF_STRICT):
        many = eng.replay_batch_many(tr, masks, codes, flags)
        assert eng.stats().kernel_launches == 1 and eng.stats().prefixes == len(tr)
        for t in range(len(traces)):
            sel = np.nonzero(tr == t)[0]
            eng.set_trace(traces[t], exts[t])
            solo = eng.replay_batch(masks[sel, :eng.mask_words()], codes[t], flags)
            assert (many[sel].view(np.uint8) == solo.view(np.uint8)).all(), (t, flags)
            if t % 4 == 0 or t == len(traces) - 1:
                cpu = oracle.replay_batch(N.MODEL_RAFT5, traces[t], exts[t], masks[sel, :eng.mask_words()], looking_for=codes[t],
                                          flags=flags, model_flags=RAFT_FLAGS)
                assert (many[sel] == cpu).all(), (t, flags)


def test_replay_batch_many_capacity_status_is_per_trace(oracle):
    """A bcast32 trace without its internal MsgSends sizes its pending set for its few external Sends, so its replays
    overflow it; the full trace replayed in the same launch does not."""
    prog = D.bcast32_program(2)
    ext = D.pack_externals(prog)
    ev, _, r = oracle.fuzz_trace(N.MODEL_BCAST32, ext, 3, 120, 10, model_flags=3)
    keep = (ev["kind"] != N.EV_MSG_SEND) | (ev["type"] == 2)          # 2: bcast32's external INJECT
    short = ev[keep].copy()
    eng = D.Engine(D.SchedulerConfig(N.MODEL_BCAST32, model_flags=3))
    eng.set_traces([ev, short], [ext, ext])
    masks = random_masks(len(ext), 40, np.random.default_rng(4))
    tr = np.array([0, 1] * 40, dtype=np.uint32)
    m2 = np.repeat(masks, 2, axis=0)
    many = eng.replay_batch_many(tr, m2, [3, 3])
    assert (many["status"][tr == 0] == 0).all()
    assert (many["status"][tr == 1] != 0).any()
    assert many["status"][1] == 1                           # DEMI_PS_PENDING_OVF on the full subsequence
    for t, trace in enumerate((ev, short)):
        eng.set_trace(trace, ext)
        solo = eng.replay_batch(masks, 3)
        assert (many[tr == t].view(np.uint8) == solo.view(np.uint8)).all()
        cpu = oracle.replay_batch(N.MODEL_BCAST32, trace, ext, masks, looking_for=3, model_flags=3)
        assert (many[tr == t] == cpu).all()


def solo_ddmin(eng, trace, ext, code, mw, check=True):
    eng.set_trace(trace, ext)
    mcs = np.zeros(mw, dtype=np.uint64)
    iters = np.zeros(256, dtype=np.uint32)
    out = N.DDMinOut()
    rc = N.lib().demi_ddmin(eng._h, int(code), 0, 1 if check else 0, mcs.ctypes.data, mw, iters.ctypes.data, 256, C.byref(out))
    return rc, mcs, iters, out


def assert_same_as_solo(eng, traces, ext, codes, res, check=True, oracle=None):
    mcs, iters, out, status = res
    mw = mcs.shape[1]
    for t in range(len(traces)):
        rc, smcs, siters, sout = solo_ddmin(eng, traces[t], ext, codes[t], mw, check)
        assert status[t] == rc, t
        if rc != N.OK:
            continue
        assert (mcs[t] == smcs).all() and (iters[t] == siters).all(), t
        for f in ("mcs_size", "total_replays", "n_iterations", "replays_executed", "batches", "verified"):
            assert out[t][f] == getattr(sout, f), (t, f)
        if oracle is not None and t % 16 == 0:
            crc, cmcs, total, citers, ver = oracle.ddmin_sts(N.MODEL_RAFT5, traces[t], ext, int(codes[t]), model_flags=RAFT_FLAGS)
            assert crc == 0 and (cmcs == mcs[t]).all() and total == out[t]["total_replays"] and ver == out[t]["verified"]
            assert list(citers) == list(iters[t, :out[t]["n_iterations"]])


@pytest.mark.parametrize("wide", [None, "64"])
def test_ddmin_many_equals_solo_and_oracle(oracle, monkeypatch, wide):
    if wide:
        monkeypatch.setenv("DEMI_DDMIN_WIDE", wide)
    eng, ext, ev, ne, viol = raft_set(96, client_cmds=6)
    traces = [ev[i, :ne[i]].copy() for i in range(len(ne))]
    eng.set_traces((ev, ne), ext)
    res = eng.ddmin_many(viol)
    assert (res[3] == N.OK).all()
    launches = eng.stats().kernel_launches
    assert 0 < launches < sum(int(b) for b in res[2]["batches"])       # drivers shared launches
    assert_same_as_solo(eng, traces, ext, viol, res, oracle=oracle)
    # grouping independence: reversed order, two calls, a window of 7
    eng.set_traces(traces[::-1], ext)
    r2 = eng.ddmin_many(viol[::-1])
    fields = ["mcs_size", "total_replays", "n_iterations", "replays_executed", "batches", "verified"]
    assert (r2[0][::-1] == res[0]).all() and (r2[1][::-1] == res[1]).all() and (r2[3][::-1] == res[3]).all()
    assert (r2[2][::-1][fields] == res[2][fields]).all()
    half = len(traces) // 2
    for lo, hi in ((0, half), (half, len(traces))):
        eng.set_traces(traces[lo:hi], ext)
        r3 = eng.ddmin_many(viol[lo:hi])
        assert (r3[0] == res[0][lo:hi]).all() and (r3[1] == res[1][lo:hi]).all()
    monkeypatch.setenv("DEMI_DDMIN_MANY_WINDOW", "7")
    eng.set_traces((ev, ne), ext)
    r4 = eng.ddmin_many(viol)
    assert (r4[0] == res[0]).all() and (r4[1] == res[1]).all() and (r4[2][fields] == res[2][fields]).all()


def test_ddmin_many_single_and_4096_traces():
    eng, ext, ev, ne, viol = raft_set(4096, seeds=200000)
    eng.set_traces((ev[:1], ne[:1]), ext)
    r1 = eng.ddmin_many(viol[:1])
    assert r1[3][0] == N.OK
    assert_same_as_solo(eng, [ev[0, :ne[0]]], ext, viol[:1], r1)
    eng.set_traces((ev, ne), ext)
    r = eng.ddmin_many(viol)
    assert (r[3] == N.OK).all()
    sample = list(range(0, 4096, 97))
    assert_same_as_solo(eng, [ev[i, :ne[i]] for i in sample], ext, viol[sample], tuple(x[sample] for x in r))


def test_ddmin_many_failure_isolation():
    eng, ext, ev, ne, viol = raft_set(8)
    res = eng.fuzz_batch(1, 2000, MAXM, INTERVAL)
    quiet = np.nonzero(res["violation"] == 0)[0][:1].astype(np.uint32)
    qev, qne, _ = eng.fuzz_traces(1, quiet, MAXM, INTERVAL, cap_events=1024)
    traces = [ev[i, :ne[i]].copy() for i in range(3)] + [qev[0, :qne[0]].copy()] + [ev[i, :ne[i]].copy() for i in range(3, 8)]
    codes = np.concatenate([viol[:3], [viol[0]], viol[3:]]).astype(np.uint32)
    eng.set_traces(traces, ext)
    r = eng.ddmin_many(codes)
    assert r[3][3] == N.ERR_INVALID and (np.delete(r[3], 3) == N.OK).all()
    assert "Unmodified trace does not trigger violation" in eng.last_error()
    assert_same_as_solo(eng, traces, ext, codes, r)


def test_handle_state_and_arguments(monkeypatch):
    eng, ext, ev, ne, viol = raft_set(4)
    L = N.lib()
    with pytest.raises(D.DemiError) as ei:                   # the Python binding reports the library's state error
        eng.ddmin_many([])
    assert ei.value.code == N.ERR_STATE
    # no set yet
    lf = np.zeros(1, dtype=np.uint32)
    out = np.zeros(1, dtype=N.DDMIN_OUT_DTYPE)
    st = np.zeros(1, dtype=np.int32)
    mcs = np.zeros(1, dtype=np.uint64)
    assert L.demi_ddmin_many(eng._h, lf.ctypes.data, 0, 1, mcs.ctypes.data, 1, None, 0, out.ctypes.data, st.ctypes.data) == N.ERR_STATE
    rr = np.zeros(1, dtype=N.REPLAY_DTYPE)
    t0 = np.zeros(1, dtype=np.uint32)
    assert L.demi_replay_batch_many(eng._h, t0.ctypes.data, mcs.ctypes.data, 1, 1, lf.ctypes.data, 0, rr.ctypes.data) == N.ERR_STATE
    # the single trace, its conjoined atoms and its replays
    eng.set_trace(ev[0, :ne[0]], ext)
    eng.conjoin_atoms(0, 1)
    masks = random_masks(len(ext), 64, np.random.default_rng(5))
    before = eng.replay_batch(masks, int(viol[0]))
    eng.set_traces((ev, ne), ext)
    eng.ddmin_many(viol)
    assert (eng.replay_batch(masks, int(viol[0])).view(np.uint8) == before.view(np.uint8)).all()
    with pytest.raises(D.DemiError) as ei:
        eng.conjoin_atoms(1, 2)                              # still conjoined: the single trace's dag is untouched
    assert ei.value.code == N.ERR_STATE
    # a rejected set names the bad trace and keeps the previous one
    bad = [ev[i, :ne[i]].copy() for i in range(4)]
    bad[2][0]["dst"] = 40
    with pytest.raises(D.DemiError) as ei:
        eng.set_traces(bad, ext)
    assert ei.value.code == N.ERR_INVALID and "trace 2" in str(ei.value)
    r = eng.ddmin_many(viol)
    assert (r[3] == N.OK).all()
    # arguments
    m4 = np.tile(masks[:1], (4, 1))
    t4 = np.arange(4, dtype=np.uint32)
    r4 = np.zeros(4, dtype=N.REPLAY_DTYPE)
    assert L.demi_replay_batch_many(eng._h, None, m4.ctypes.data, 4, 1, viol.ctypes.data, 0, r4.ctypes.data) == N.ERR_INVALID
    t4[3] = 4
    assert L.demi_replay_batch_many(eng._h, t4.ctypes.data, m4.ctypes.data, 4, 1, viol.ctypes.data, 0, r4.ctypes.data) == N.ERR_INVALID
    assert "names trace 4" in eng.last_error()
    out4 = np.zeros(4, dtype=N.DDMIN_OUT_DTYPE)
    st4 = np.zeros(4, dtype=np.int32)
    mc4 = np.zeros(4, dtype=np.uint64)
    assert L.demi_ddmin_many(eng._h, viol.ctypes.data, 0, 1, mc4.ctypes.data, 1, None, 0, None, st4.ctypes.data) == N.ERR_INVALID
    assert L.demi_ddmin_many(eng._h, viol.ctypes.data, 0, 1, mc4.ctypes.data, 0, None, 0, out4.ctypes.data, st4.ctypes.data) == N.ERR_INVALID
    assert "too small" in eng.last_error()
    # the window of drivers in flight is validated
    mc4 = np.zeros((4, 1), dtype=np.uint64)
    for bad in ("0", "-1", "4097", "x"):
        monkeypatch.setenv("DEMI_DDMIN_MANY_WINDOW", bad)
        assert L.demi_ddmin_many(eng._h, viol.ctypes.data, 0, 1, mc4.ctypes.data, 1, None, 0, out4.ctypes.data,
                                 st4.ctypes.data) == N.ERR_INVALID
        assert "DEMI_DDMIN_MANY_WINDOW" in eng.last_error()
    monkeypatch.setenv("DEMI_DDMIN_MANY_WINDOW", "1")
    assert L.demi_ddmin_many(eng._h, viol.ctypes.data, 0, 1, mc4.ctypes.data, 1, None, 0, out4.ctypes.data,
                             st4.ctypes.data) == N.OK and (st4 == N.OK).all()
