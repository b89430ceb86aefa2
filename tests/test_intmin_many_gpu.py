"""Internal minimization of many traces at once: demi_replay_traces_many and demi_internal_minimize_many against the
single-trace entry points (demi_set_trace + demi_replay_trace / demi_internal_minimize) and the CPU oracle."""

import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
from test_ddmin_many_gpu import INTERVAL, MAXM, RAFT_FLAGS, long_raft_trace, raft_engine, raft_hits, random_masks

pytestmark = pytest.mark.gpu

NONE = 0xFFFFFFFF
PS_EVENT_OVF = 4                               # DEMI_PS_EVENT_OVF
FLAG_SETS = [0, N.IM_SRC_DST_FIFO, N.RF_FILTER_KNOWN_ABSENTS, N.IM_SRC_DST_FIFO | N.RF_FILTER_KNOWN_ABSENTS]


def as_bytes(a):
    return np.ascontiguousarray(a).view(np.uint8)


def solo_record(eng, trace, ext, mask, skip, code, flags, cap):
    eng.set_trace(trace, ext)
    return eng.replay_trace(mask, skip, code, flags, cap)


def solo_intmin(eng, trace, ext, code, flags, cap=4096):
    """(status, message, trace, sizes, out) of demi_set_trace + demi_internal_minimize."""
    eng.set_trace(trace, ext)
    try:
        t, s, o = eng.internal_minimize(code, flags, cap_events=cap)
    except D.DemiError as e:
        return e.code, eng.last_error(), None, None, None
    out = np.zeros(1, dtype=N.INTMIN_OUT_DTYPE)
    out.view(np.uint8)[:] = np.frombuffer(bytes(o), dtype=np.uint8)
    return N.OK, "", t, s, out[0]


def check_against_solo(eng, traces, exts, codes, flags, many, cap=4096, solo_cap=None):
    ev, sizes, out, status = many
    for t in range(len(traces)):
        st, msg, strace, ssizes, sout = solo_intmin(eng, traces[t], exts[t], codes[t], flags, solo_cap or cap)
        assert status[t] == st, (t, flags, status[t], st, msg)
        if st != N.OK:
            continue
        assert as_bytes(out[t]).tobytes() == as_bytes(sout).tobytes(), (t, flags)
        n = min(int(out[t]["n_events"]), cap)
        assert (ev[t, :n] == strace[:n]).all(), (t, flags)
        assert (sizes[t, :out[t]["n_internal_sizes"]] == ssizes).all(), (t, flags)


# ---------------------------------------------------------------- inputs: verified MCS traces
_CACHE = {}


def mcs_set(client_cmds, n):
    """n violating executions of the headline workload (with client_cmds) after DDMin and the recorded verify_mcs:
    (engine, program, MCS traces, MCS externals, codes).  Executions whose MCS does not reproduce are left out."""
    key = (client_cmds, n)
    if key in _CACHE:
        return _CACHE[key]
    prog = D.raft5_program(client_cmds=client_cmds)
    ext = D.pack_externals(prog)
    eng = raft_engine(prog)
    hits, _ = raft_hits(eng, 40000, n + n // 2)
    ev, ne, r = eng.fuzz_traces(1, hits, MAXM, INTERVAL, cap_events=1024)
    codes = r["violation"].astype(np.uint32)
    eng.set_traces((ev, ne), ext)
    mw = eng.set_mask_words()
    mcs, _, dd, status = eng.ddmin_many(codes)
    assert (status == N.OK).all()
    rev, rne, rres = eng.replay_traces_many(np.arange(len(ne), dtype=np.uint32), mcs, None, codes, cap_events=1024)
    ok = np.nonzero((rres["status"] == 0) & (rres["violation"] == codes))[0][:n]
    assert len(ok) == n
    traces = [rev[i, :rne[i]].copy() for i in ok]
    exts = [D.pack_externals(D.events_of(prog, mcs[i, :mw])) for i in ok]
    _CACHE[key] = (eng, prog, traces, exts, codes[ok].copy(), (ev, ne, mcs, codes))
    return _CACHE[key]


# ---------------------------------------------------------------- 1. recording
def test_replay_traces_many_matches_single_and_oracle(oracle):
    prog = D.raft5_program(client_cmds=6)
    ext = D.pack_externals(prog)
    eng = raft_engine(prog)
    hits, _ = raft_hits(eng, 40000, 12)
    ev, ne, r = eng.fuzz_traces(1, hits, MAXM, INTERVAL, cap_events=1024)
    lev, lext, lcode = long_raft_trace(oracle)
    traces = [ev[i, :ne[i]].copy() for i in range(len(ne))] + [lev]
    exts = [ext] * len(ne) + [lext]
    codes = list(r["violation"].astype(np.uint32)) + [lcode]
    eng.set_traces(traces, exts)
    rng = np.random.default_rng(5)
    per = 6
    tr = np.repeat(np.arange(len(traces), dtype=np.uint32), per)
    masks = np.concatenate([random_masks(len(exts[t]), per, rng) for t in range(len(traces))])
    skips = np.array([NONE if k % 3 == 0 else int(rng.choice(np.nonzero(traces[t]["kind"] == N.EV_MSG_EVENT)[0]))
                      for k, t in enumerate(tr)], dtype=np.uint32)
    perm = rng.permutation(len(tr))
    tr, masks, skips = tr[perm], masks[perm], skips[perm]
    for flags in (0, N.RF_FILTER_KNOWN_ABSENTS, N.RF_STRICT):
        for m, sk in ((masks, skips), (None, skips), (masks, None)):
            rev, rne, rres = eng.replay_traces_many(tr, m, sk, codes, flags, cap_events=4096)
            assert eng.stats().kernel_launches == 1 and eng.stats().prefixes == len(tr)
            for i, t in enumerate(tr):
                mask = None if m is None else m[i, :max(1, (len(exts[t]) + 63) // 64)]
                skip = NONE if sk is None else int(sk[i])
                sres, sev = solo_record(eng, traces[t], exts[t], mask, skip, codes[t], flags, 4096)
                assert as_bytes(rres[i:i + 1]).tobytes() == as_bytes(np.array([sres])).tobytes(), (i, t, flags)
                assert rne[i] == len(sev) and (rev[i, :rne[i]] == sev).all(), (i, t, flags)
                if i % 9 == 0:
                    om = oracle.full_mask(exts[t], False) if m is None else mask
                    cres, cev = oracle.replay_trace(N.MODEL_RAFT5, traces[t], exts[t], om, looking_for=int(codes[t]),
                                                    flags=flags, model_flags=RAFT_FLAGS, skip_event=skip)
                    assert cres == sres and len(cev) == len(sev) and (cev == sev).all(), (i, t, flags)


def test_replay_traces_many_event_overflow_matches_single():
    eng, prog, traces, exts, codes, _ = mcs_set(0, 64)
    eng.set_traces(traces, exts)
    tr = np.arange(len(traces), dtype=np.uint32)
    cap = int(np.median([len(t) for t in traces]))
    rev, rne, rres = eng.replay_traces_many(tr, None, None, codes, 0, cap_events=cap)
    assert (rres["status"] == PS_EVENT_OVF).any() and (rres["status"] == 0).any()
    for t in range(len(traces)):
        sres, sev = solo_record(eng, traces[t], exts[t], None, NONE, codes[t], 0, cap)
        assert as_bytes(rres[t:t + 1]).tobytes() == as_bytes(np.array([sres])).tobytes(), t
        assert rne[t] == len(sev) and (rev[t, :rne[t]] == sev).all(), t


# ---------------------------------------------------------------- 2. the pipeline, 3. grouping
@pytest.mark.parametrize("client_cmds", [0, 6])
def test_pipeline_matches_single_path_and_oracle(oracle, client_cmds):
    eng, prog, traces, exts, codes, _ = mcs_set(client_cmds, 64)
    eng.set_traces(traces, exts)
    for flags in FLAG_SETS:
        many = eng.internal_minimize_many(codes, flags)
        assert (many[3] == N.OK).all(), eng.last_error()
        assert eng.stats().kernel_launches <= 2 * int(many[2]["batches"].max())
        check_against_solo(eng, traces, exts, codes, flags, many)
        ev, sizes, out, _ = many
        for t in range(0, len(traces), 4):
            rc, ctrace, total, csizes, unig = oracle.internal_minimize(N.MODEL_RAFT5, traces[t], exts[t], int(codes[t]),
                                                                       flags=flags, model_flags=RAFT_FLAGS)
            assert rc == 0
            n = int(out[t]["n_events"])
            assert n == len(ctrace) and (ev[t, :n] == ctrace).all(), (t, flags)
            assert out[t]["total_replays"] == total and out[t]["unignorable"] == unig, (t, flags)
            assert (sizes[t, :out[t]["n_internal_sizes"]] == csizes).all(), (t, flags)


def test_results_do_not_depend_on_grouping():
    eng, prog, traces, exts, codes, _ = mcs_set(0, 64)
    eng.set_traces(traces, exts)
    flags = N.IM_SRC_DST_FIFO
    ev, sizes, out, status = eng.internal_minimize_many(codes, flags)
    sub = np.random.default_rng(9).permutation(len(traces))[:23]
    eng.set_traces([traces[i] for i in sub], [exts[i] for i in sub])
    ev2, sizes2, out2, status2 = eng.internal_minimize_many(codes[sub], flags)
    assert (status2 == status[sub]).all()
    assert as_bytes(out2).tobytes() == as_bytes(out[sub]).tobytes()
    for k, t in enumerate(sub):
        n = int(out[t]["n_events"])
        assert (ev2[k, :n] == ev[t, :n]).all() and (sizes2[k] == sizes[t]).all()


# ---------------------------------------------------------------- 4. other models
def verified_full(eng, model, ext, evs, codes):
    """Traces recorded by replaying each execution's full externals (a verified trace whose MCS is everything)."""
    eng.set_traces(evs, [ext] * len(evs))
    rev, rne, rres = eng.replay_traces_many(np.arange(len(evs), dtype=np.uint32), None, None, codes, 0, cap_events=65536)
    assert (rres["status"] == 0).all()
    return [rev[i, :rne[i]].copy() for i in range(len(evs))]


def other_model_case(oracle, model, flags, prog, maxm, interval, n, blob=None, seeds=4000):
    ext = D.pack_externals(prog)
    if blob is not None:
        oracle.load_model(blob)
    res = oracle.fuzz_batch(model, ext, 1, seeds, maxm, interval, model_flags=flags)
    hits = np.nonzero((res["violation"] != 0) & (res["status"] == 0))[0][:n]
    assert len(hits) > 0
    evs, codes = [], []
    for k in hits:
        ev, _, r = oracle.fuzz_trace(model, ext, 1 + int(k), maxm, interval, model_flags=flags)
        evs.append(ev)
        codes.append(int(r["violation"]))
    eng = D.Engine(D.SchedulerConfig(model, model_flags=flags))
    if blob is not None:
        eng.load_model(blob)
    codes = np.array(codes, dtype=np.uint32)
    traces = verified_full(eng, model, ext, evs, codes)
    eng.set_traces(traces, [ext] * len(traces))
    for im in (0, N.IM_SRC_DST_FIFO):
        many = eng.internal_minimize_many(codes, im, cap_events=65536)
        check_against_solo(eng, traces, [ext] * len(traces), codes, im, many, cap=65536)
        ev, sizes, out, status = many
        for t in range(0, len(traces), 3):
            rc, ctrace, total, csizes, unig = oracle.internal_minimize(model, traces[t], ext, int(codes[t]), flags=im,
                                                                       model_flags=flags)
            assert rc == 0 and status[t] == N.OK
            n = int(out[t]["n_events"])
            assert n == len(ctrace) and (ev[t, :n] == ctrace).all() and out[t]["total_replays"] == total, (model, t, im)
            assert (sizes[t, :out[t]["n_internal_sizes"]] == csizes).all()


def test_other_models(oracle):
    prog = [D.Start(a) for a in range(3)] + [D.Send(k % 3, 1, k) for k in range(10)] + [D.WaitQuiescence()]
    other_model_case(oracle, N.MODEL_PINGPONG3, 1, prog, -1, 0, 8)
    other_model_case(oracle, N.MODEL_BCAST32, 3, D.bcast32_program(2), 120, 10, 6)
    from test_ir_timers_oracle import ELECTION_INTERVAL, ELECTION_MAXM, election_model, election_program
    m = election_model()
    other_model_case(oracle, N.MODEL_IR, m.flags, election_program(), ELECTION_MAXM, ELECTION_INTERVAL, 8, blob=m.blob,
                     seeds=400)


# ---------------------------------------------------------------- 5. failures, 6. state and arguments
def test_a_failing_trace_fails_alone(oracle):
    prog = D.bcast32_program(2)
    ext = D.pack_externals(prog)
    ev, _, r = oracle.fuzz_trace(N.MODEL_BCAST32, ext, 3, 120, 10, model_flags=3)
    keep = (ev["kind"] != N.EV_MSG_SEND) | (ev["type"] == 2)
    short = ev[keep].copy()
    eng = D.Engine(D.SchedulerConfig(N.MODEL_BCAST32, model_flags=3))
    traces = [ev, short, ev]
    eng.set_traces(traces, [ext] * 3)
    many = eng.internal_minimize_many([3, 3, 3], 0, cap_events=65536)
    status = many[3]
    assert status[0] == N.OK and status[2] == N.OK and status[1] != N.OK
    msg = eng.last_error()
    st, smsg, _, _, _ = solo_intmin(eng, short, ext, 3, 0, 65536)
    assert st == status[1] and smsg == msg
    check_against_solo(eng, traces, [ext] * 3, [3, 3, 3], 0, many, cap=65536)


def test_too_small_cap_fails_only_the_traces_that_need_more():
    eng, prog, traces, exts, codes, _ = mcs_set(0, 64)
    eng.set_traces(traces, exts)
    lens = np.array([len(t) for t in traces])
    cap = int(np.percentile(lens, 60))
    ev, sizes, out, status = eng.internal_minimize_many(codes, 0, cap_events=cap)
    failing = np.nonzero(status != N.OK)[0]
    assert len(failing) > 0 and (status[failing] == N.ERR_CAPACITY).all()
    assert (lens[failing] > cap).all()
    assert "trace %d " % failing[0] in eng.last_error()
    for t in np.nonzero(status == N.OK)[0]:
        st, _, strace, ssizes, sout = solo_intmin(eng, traces[t], exts[t], codes[t], 0, 65536)
        assert st == N.OK and as_bytes(out[t]).tobytes() == as_bytes(sout).tobytes()
        n = min(int(out[t]["n_events"]), cap)
        assert (ev[t, :n] == strace[:n]).all()


def test_state_and_arguments():
    eng, prog, traces, exts, codes, _ = mcs_set(0, 64)
    fresh = raft_engine(prog)
    with pytest.raises(D.DemiError) as ei:
        fresh.internal_minimize_many(codes[:1])
    assert ei.value.code == N.ERR_STATE
    with pytest.raises(D.DemiError) as ei:
        fresh.replay_traces_many([0], None, None, codes[:1])
    assert ei.value.code == N.ERR_STATE
    eng.set_traces(traces, exts)
    L = N.lib()
    ev = np.zeros((len(traces), 64), dtype=N.EVENT_DTYPE)
    out = np.zeros(len(traces), dtype=N.INTMIN_OUT_DTYPE)
    st = np.zeros(len(traces), dtype=np.int32)
    lf = np.ascontiguousarray(codes, dtype=np.uint32)
    assert L.demi_internal_minimize_many(eng._h, None, 0, ev.ctypes.data, 64, None, 0, out.ctypes.data, st.ctypes.data) == N.ERR_INVALID
    assert L.demi_internal_minimize_many(eng._h, lf.ctypes.data, 0, None, 64, None, 0, out.ctypes.data, st.ctypes.data) == N.ERR_INVALID
    assert L.demi_internal_minimize_many(eng._h, lf.ctypes.data, 0, ev.ctypes.data, 64, None, 0, None, st.ctypes.data) == N.ERR_INVALID
    tr = np.zeros(1, dtype=np.uint32)
    ne = np.zeros(1, dtype=np.uint32)
    res = np.zeros(1, dtype=N.REPLAY_DTYPE)
    assert L.demi_replay_traces_many(eng._h, tr.ctypes.data, None, None, 1, 1, lf.ctypes.data, 0, None, 64, ne.ctypes.data,
                                     res.ctypes.data) == N.ERR_INVALID
    bad = np.array([len(traces)], dtype=np.uint32)
    assert L.demi_replay_traces_many(eng._h, bad.ctypes.data, None, None, 1, 1, lf.ctypes.data, 0, ev.ctypes.data, 64,
                                     ne.ctypes.data, res.ctypes.data) == N.ERR_INVALID
    # the set is left as it was
    rng = np.random.default_rng(2)
    trs = np.repeat(np.arange(len(traces), dtype=np.uint32), 3)
    masks = np.concatenate([random_masks(len(exts[t]), 3, rng) for t in range(len(traces))])
    before = eng.replay_batch_many(trs, masks, codes)
    eng.internal_minimize_many(codes, N.IM_SRC_DST_FIFO)
    after = eng.replay_batch_many(trs, masks, codes)
    assert as_bytes(before).tobytes() == as_bytes(after).tobytes()


# ---------------------------------------------------------------- 7. scale
def test_four_thousand_traces_in_one_call():
    prog = D.raft5_program()
    ext = D.pack_externals(prog)
    eng = raft_engine(prog)
    hits, _ = raft_hits(eng, 200000, 4096)
    ev, ne, r = eng.fuzz_traces(1, hits, MAXM, INTERVAL, cap_events=1024)
    codes = r["violation"].astype(np.uint32)
    eng.set_traces((ev, ne), ext)
    rev, rne, rres = eng.replay_traces_many(np.arange(len(ne), dtype=np.uint32), None, None, codes, 0, cap_events=1024)
    assert (rres["status"] == 0).all()
    traces = [rev[i, :rne[i]].copy() for i in range(len(rne))]
    eng.set_traces(traces, ext)
    many = eng.internal_minimize_many(codes, 0, cap_events=1024)
    assert (many[3] == N.OK).all()
    assert eng.stats().kernel_launches <= 2 * int(many[2]["batches"].max())
    check_against_solo(eng, traces, [ext] * len(traces), codes, 0, many, cap=1024)
