"""Wildcard minimization of many traces at once: demi_wildcard_replay_batch_many and demi_wildcard_minimize_many against
the single-trace entry points (demi_set_trace + demi_wildcard_replay_batch / demi_wildcard_minimize) and the CPU
oracle."""

import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
from oracle import wildcard_binding as W
import many_sets as S
from test_ddmin_many_gpu import INTERVAL, MAXM, RAFT_FLAGS, raft_engine, raft_hits
from test_intmin_many_gpu import mcs_set

pytestmark = pytest.mark.gpu

FLAG_SETS = [0, N.WC_LAST_ONLY, N.RF_FILTER_KNOWN_ABSENTS, N.WC_LAST_ONLY | N.RF_FILTER_KNOWN_ABSENTS]
RULES, INCR = D.raft5_clock_rules()


def as_bytes(a):
    return np.ascontiguousarray(a).view(np.uint8)


def n_deliv(trace):
    return int((trace["kind"] == N.EV_MSG_EVENT).sum())


def words(trace):
    return max(1, (n_deliv(trace) + 63) // 64)


def engine(model, flags, rules, incr, blob=None, **kw):
    eng = D.Engine(D.SchedulerConfig(model, model_flags=flags, **kw))
    if blob is not None:
        eng.load_model(blob)
    eng.set_clock_rules(rules, incr)
    return eng


def recorded(eng, traces, exts, codes, cap=65536):
    """Each trace replayed once over its externals: the recordings (distinct Uniq ids) that reproduce their code."""
    eng.set_traces(traces, exts)
    rev, rne, rres = eng.replay_traces_many(np.arange(len(traces), dtype=np.uint32), None, None, codes, 0, cap_events=cap)
    ok = [i for i in range(len(traces)) if rres[i]["status"] == 0 and rres[i]["violation"] == codes[i]]
    return [rev[i, :rne[i]].copy() for i in ok], [exts[i] for i in ok], np.asarray(codes)[ok].astype(np.uint32)


def include_masks(trace, n, mw, rng):
    """n include masks over trace's deliveries (mask 0 includes all), mw words, random bits past the deliveries."""
    d = n_deliv(trace)
    m = rng.integers(0, 1 << 64, size=(n, mw), dtype=np.uint64, endpoint=False)
    m[0, :] = ~np.uint64(0)
    keep = rng.random((n, d)) < rng.choice([0.97, 0.85, 0.5], size=n)[:, None]
    for j in range(d):
        bit = np.uint64(1) << np.uint64(j & 63)
        m[:, j >> 6] = np.where(keep[:, j] | (np.arange(n) == 0), m[:, j >> 6] | bit, m[:, j >> 6] & ~bit)
    return m


def solo_wc(eng, trace, ext, code, flags, cap=4096):
    """(status, message, trace, sizes, out) of demi_set_trace + demi_wildcard_minimize on `eng`, an engine or a function
    that makes a fresh one."""
    if not isinstance(eng, D.Engine):
        eng = eng()
    eng.set_trace(trace, ext)
    try:
        t, s, o = eng.wildcard_minimize(code, flags, cap_events=cap)
    except D.DemiError as e:
        return e.code, eng.last_error(), None, None, None
    out = np.zeros(1, dtype=N.INTMIN_OUT_DTYPE)
    out.view(np.uint8)[:] = np.frombuffer(bytes(o), dtype=np.uint8)
    return N.OK, "", t, s, out[0]


def check_against_solo(solo, traces, exts, codes, flags, many, cap=4096):
    """Each trace of `many` against the single call on a fresh handle from solo()."""
    ev, sizes, out, status = many
    for t in range(len(traces)):
        st, msg, strace, ssizes, sout = solo_wc(solo, traces[t], exts[t], codes[t], flags, cap)
        assert status[t] == st, (t, flags, status[t], st, msg)
        if st != N.OK:
            continue
        assert as_bytes(out[t]).tobytes() == as_bytes(sout).tobytes(), (t, flags)
        n = min(int(out[t]["n_events"]), cap)
        assert (ev[t, :n] == strace[:n]).all(), (t, flags)
        assert (sizes[t, :out[t]["n_internal_sizes"]] == ssizes).all(), (t, flags)


def check_oracle(model, model_flags, traces, exts, codes, rules, incr, flags, many, step, **cfg):
    ev, sizes, out, status = many
    for t in range(0, len(traces), step):
        rc, ctrace, total, csizes = W.wildcard_minimize(model, traces[t], exts[t], rules, incr, int(codes[t]), flags=flags,
                                                        model_flags=model_flags, **cfg)
        assert rc == 0 and status[t] == N.OK
        n = int(out[t]["n_events"])
        assert n == len(ctrace) and (ev[t, :n] == ctrace).all(), (t, flags)
        assert out[t]["total_replays"] == total and (sizes[t, :out[t]["n_internal_sizes"]] == csizes).all(), (t, flags)


# ---------------------------------------------------------------- inputs
_CACHE = {}


def intmin_set(client_cmds, n):
    """n headline violations after ddmin_many, the recorded verify_mcs and internal_minimize_many: what the wildcard
    stage starts from.  (engine, traces, MCS externals, codes)."""
    key = (client_cmds, n)
    if key not in _CACHE:
        eng, prog, traces, exts, codes, _ = mcs_set(client_cmds, n)
        eng.set_clock_rules(RULES, INCR)
        eng.set_traces(traces, exts)
        ev, _, out, status = eng.internal_minimize_many(codes, N.IM_SRC_DST_FIFO)
        assert (status == N.OK).all()
        _CACHE[key] = (eng, [ev[t, :out[t]["n_events"]].copy() for t in range(n)], exts, codes)
    return _CACHE[key]


def raft_mixed_recorded():
    if "mixed" not in _CACHE:
        traces, exts, codes = S.raft5_mixed()
        eng = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR)
        _CACHE["mixed"] = (eng,) + recorded(eng, traces, exts, codes)
    return _CACHE["mixed"]


# ---------------------------------------------------------------- 1. replays
def test_wildcard_replay_batch_many_matches_single():
    eng, traces, exts, codes = raft_mixed_recorded()
    solo = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR)
    eng.set_traces(traces, exts)
    rng = np.random.default_rng(3)
    mw = max(words(t) for t in traces) + 1
    per = 12
    tr = np.repeat(np.arange(len(traces), dtype=np.uint32), per)
    masks = np.concatenate([include_masks(t, per, mw, rng) for t in traces])
    perm = rng.permutation(len(tr))
    tr, masks = tr[perm], masks[perm]
    for flags in FLAG_SETS:
        got = eng.wildcard_replay_batch_many(tr, masks, codes, flags)
        assert eng.stats().kernel_launches == 1 and eng.stats().prefixes == len(tr)
        for t in range(len(traces)):
            sel = np.nonzero(tr == t)[0]
            solo.set_trace(traces[t], exts[t])
            want = solo.wildcard_replay_batch(masks[sel, :words(traces[t])], codes[t], flags)
            assert as_bytes(got[sel]).tobytes() == as_bytes(want).tobytes(), (t, flags)
        assert (got["violation"] != 0).any() and (got["violation"] == 0).any()


def test_wildcard_replay_batch_many_split_and_many_tiles_per_warp():
    """2^20 + 37 tests: two launches, each warp running several tiles."""
    eng, traces, exts, codes = raft_mixed_recorded()
    solo = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR)
    eng.set_traces(traces, exts)
    rng = np.random.default_rng(4)
    n = (1 << 20) + 37
    mw = max(words(t) for t in traces)
    tr = (np.arange(n) % len(traces)).astype(np.uint32)
    masks = np.zeros((n, mw), dtype=np.uint64)
    base = [include_masks(t, 64, mw, rng) for t in traces]
    pick = rng.integers(0, 64, size=n)
    for t in range(len(traces)):
        sel = tr == t
        masks[sel] = base[t][pick[sel]]
    got = eng.wildcard_replay_batch_many(tr, masks, codes, N.WC_LAST_ONLY)
    assert eng.stats().kernel_launches == 2 and eng.stats().prefixes == n
    for t in range(len(traces)):
        solo.set_trace(traces[t], exts[t])
        want = solo.wildcard_replay_batch(base[t][:, :words(traces[t])], codes[t], N.WC_LAST_ONLY)
        sel = np.nonzero(tr == t)[0]
        assert as_bytes(got[sel]).tobytes() == as_bytes(want[pick[sel]]).tobytes(), t


# ---------------------------------------------------------------- 2. minimization
@pytest.mark.parametrize("client_cmds", [0, 6])
def test_minimize_many_matches_single_and_oracle(client_cmds):
    eng, traces, exts, codes = intmin_set(client_cmds, 64)
    solo = lambda: engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR)
    eng.set_traces(traces, exts)
    for flags in FLAG_SETS:
        many = eng.wildcard_minimize_many(codes, flags)
        assert (many[3] == N.OK).all(), eng.last_error()
        assert eng.stats().kernel_launches <= 2 * int(many[2]["batches"].max())
        check_against_solo(solo, traces, exts, codes, flags, many)
        check_oracle(N.MODEL_RAFT5, RAFT_FLAGS, traces, exts, codes, RULES, INCR, flags, many, 8)
    assert (many[2]["deliveries_after"] < many[2]["deliveries_before"]).any()


def test_minimize_many_under_blocked_actors_and_ignore_timers():
    _, traces, exts, codes = intmin_set(0, 64)
    for kw in (dict(blocked_mask=1 << 4), dict(ignoreTimers=True)):
        eng = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR, **kw)
        solo = lambda: engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR, **kw)
        eng.set_traces(traces[:24], exts[:24])
        for flags in (0, N.WC_LAST_ONLY | N.RF_FILTER_KNOWN_ABSENTS):
            many = eng.wildcard_minimize_many(codes[:24], flags)
            check_against_solo(solo, traces[:24], exts[:24], codes[:24], flags, many)


def test_other_models(oracle):
    # pingpong3: a clock in p0's low bits, no incrementing type
    traces, exts, codes = S.pingpong3_set()
    eng = engine(N.MODEL_PINGPONG3, S.PP_FLAGS, [N.clock_rule(1, 0, 0, 2)], ())
    traces, exts, codes = recorded(eng, traces, exts, codes)
    assert len(traces) >= 6
    solo = lambda: engine(N.MODEL_PINGPONG3, S.PP_FLAGS, [N.clock_rule(1, 0, 0, 2)], ())
    eng.set_traces(traces, exts)
    for flags in (0, N.WC_LAST_ONLY):
        many = eng.wildcard_minimize_many(codes, flags, cap_events=65536)
        check_against_solo(solo, traces, exts, codes, flags, many, cap=65536)
        check_oracle(N.MODEL_PINGPONG3, S.PP_FLAGS, traces, exts, codes, [N.clock_rule(1, 0, 0, 2)], [], flags, many, 3)
    # the timer-driven election: its timer is the incrementing type, the terms are clocks
    from test_ir_timers_oracle import ELECT, HB, REQ, VOTE
    m, traces, exts, codes = S.election_set()
    W.load_model(m.blob)
    rules = [N.clock_rule(t, 0, 0, 8) for t in (REQ, VOTE, HB)]
    eng = engine(N.MODEL_IR, m.flags, rules, [ELECT], blob=m.blob)
    traces, exts, codes = recorded(eng, traces, exts, codes)
    assert len(traces) >= 4
    solo = lambda: engine(N.MODEL_IR, m.flags, rules, [ELECT], blob=m.blob)
    eng.set_traces(traces, exts)
    for flags in FLAG_SETS:
        many = eng.wildcard_minimize_many(codes, flags, cap_events=65536)
        assert (many[3] == N.OK).all(), eng.last_error()
        check_against_solo(solo, traces, exts, codes, flags, many, cap=65536)
        check_oracle(N.MODEL_IR, m.flags, traces, exts, codes, rules, [ELECT], flags, many, 2)
    # generated models that arm timers, with their first timer-armed type incrementing
    for gm, gtr, gext, gcodes in S.generated_timer_sets(seeds=range(1, 25), per=3)[:3]:
        rules = [N.clock_rule(t, 0, 0, 8) for t in range(1, min(gm.n_types, 4))]
        eng = engine(N.MODEL_IR, gm.flags, rules, [1], blob=gm.blob)
        gtr, gext, gcodes = recorded(eng, gtr, gext, gcodes)
        if not gtr:
            continue
        solo = lambda gm=gm, rules=rules: engine(N.MODEL_IR, gm.flags, rules, [1], blob=gm.blob)
        eng.set_traces(gtr, gext)
        many = eng.wildcard_minimize_many(gcodes, N.WC_LAST_ONLY, cap_events=65536)
        check_against_solo(solo, gtr, gext, gcodes, N.WC_LAST_ONLY, many, cap=65536)


# ---------------------------------------------------------------- 3. grouping, 4. the round budget
def test_results_do_not_depend_on_grouping():
    eng, traces, exts, codes = intmin_set(0, 64)
    eng.set_traces(traces, exts)
    flags = N.WC_LAST_ONLY
    ev, sizes, out, status = eng.wildcard_minimize_many(codes, flags)
    sub = np.random.default_rng(9).permutation(len(traces))[:23]
    eng.set_traces([traces[i] for i in sub], [exts[i] for i in sub])
    ev2, sizes2, out2, status2 = eng.wildcard_minimize_many(codes[sub], flags)
    assert (status2 == status[sub]).all()
    assert as_bytes(out2).tobytes() == as_bytes(out[sub]).tobytes()
    for k, t in enumerate(sub):
        n = int(out[t]["n_events"])
        assert (ev2[k, :n] == ev[t, :n]).all() and (sizes2[k] == sizes[t]).all()


def test_round_budget_changes_no_result(monkeypatch):
    eng, traces, exts, codes = intmin_set(6, 64)
    eng.set_traces(traces, exts)
    want = eng.wildcard_minimize_many(codes, 0)
    rounds = eng.stats().kernel_launches
    monkeypatch.setenv("DEMI_TEST_WC_ROUND_BYTES", "2048")           # a few traces per round, one when they are large
    got = eng.wildcard_minimize_many(codes, 0)
    assert eng.stats().kernel_launches > rounds
    for a, b in zip(want, got):
        assert as_bytes(a).tobytes() == as_bytes(b).tobytes()


# ---------------------------------------------------------------- 5. failures, 6. state and arguments
def test_a_failing_trace_fails_alone():
    """Repeated Uniq ids (DEMI_ERR_INVALID) and a recording longer than cap_events (DEMI_ERR_CAPACITY), each alongside
    traces that succeed."""
    eng, traces, exts, codes = intmin_set(0, 64)
    solo = lambda: engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR)
    eng.set_traces(traces, exts)
    _, _, full, _ = eng.wildcard_minimize_many(codes, 0, cap_events=4096)
    # a trace whose minTrace was replaced by a recording: that recording is n_events long
    rec = [t for t in range(len(traces)) if full[t]["deliveries_after"] < full[t]["deliveries_before"]]
    assert rec
    long_t = max(rec, key=lambda t: int(full[t]["n_events"]))
    cap = int(full[long_t]["n_events"]) - 1
    dup = traces[5].copy()
    d = np.nonzero(dup["kind"] == N.EV_MSG_EVENT)[0]
    dup["uniq"][d[-1]] = dup["uniq"][d[0]]                             # a Uniq id names two deliveries
    pick = [0, 1, 5, long_t] + [t for t in range(2, len(traces)) if t not in (5, long_t)][:8]
    tr = [traces[t] for t in pick]
    tr[2] = dup
    ex, cd = [exts[t] for t in pick], np.array([codes[t] for t in pick], dtype=np.uint32)
    eng.set_traces(tr, ex)
    many = eng.wildcard_minimize_many(cd, 0, cap_events=cap)
    status = many[3]
    assert status[2] == N.ERR_INVALID and status[3] == N.ERR_CAPACITY
    long_ = [t for t in range(len(tr)) if t != 2 and status[t] != N.OK]
    assert long_ and all(status[t] == N.ERR_CAPACITY for t in long_)
    assert (status == N.OK).any()
    low = int(np.nonzero(status != N.OK)[0][0])
    msg = eng.last_error()
    assert ("trace %d:" % low) in msg or ("trace %d " % low) in msg, msg
    st, _, _, _, _ = solo_wc(solo, dup, ex[2], cd[2], 0)
    assert st == N.ERR_INVALID
    for t in np.nonzero(status == N.OK)[0]:
        st, _, strace, ssizes, sout = solo_wc(solo, tr[t], ex[t], cd[t], 0, 65536)
        assert st == N.OK and as_bytes(many[2][t]).tobytes() == as_bytes(sout).tobytes()
        n = min(int(many[2][t]["n_events"]), cap)
        assert (many[0][t, :n] == strace[:n]).all()


# bcast32 floods with the invariant checked once, at max_messages deliveries: at 700 deliveries the wildcard pending
# capacity is clamped at 8192 entries, and a wildcard replay that delivers other floods than the trace did can need more
BC_RULES = [N.clock_rule(1, 0, 0, 8)]                                   # FLOOD(ttl): the ttl as its clock


def bcast_set():
    """(traces, externals, codes): bcast32 ttl-3 executions of 700 and of 200 deliveries.  Their Uniq ids are distinct."""
    if "bcast" not in _CACHE:
        ext = D.pack_externals(D.bcast32_program(3))
        traces, codes = [], []
        for maxm, n in ((700, 4), (200, 3)):
            for ev, c in S.violating(S.BC, ext, 1, maxm, maxm, n, 16):
                traces.append(ev)
                codes.append(c)
        _CACHE["bcast"] = (traces, [ext] * len(traces), np.array(codes, dtype=np.uint32))
    return _CACHE["bcast"]


def test_bcast32_replays_and_a_pending_overflow_that_fails_alone():
    traces, exts, codes = bcast_set()
    eng = engine(N.MODEL_BCAST32, 1, BC_RULES, ())
    eng.set_traces(traces, exts)
    # the replays: the set's wildcard pending capacity is each trace's own, overflows included
    rng = np.random.default_rng(8)
    mw = max(words(t) for t in traces)
    per = 10
    tr = np.repeat(np.arange(len(traces), dtype=np.uint32), per)
    masks = np.concatenate([include_masks(t, per, mw, rng) for t in traces])
    solo = engine(N.MODEL_BCAST32, 1, BC_RULES, ())
    for flags in (0, N.WC_LAST_ONLY):
        got = eng.wildcard_replay_batch_many(tr, masks, codes, flags)
        for t in range(len(traces)):
            sel = np.nonzero(tr == t)[0]
            solo.set_trace(traces[t], exts[t])
            want = solo.wildcard_replay_batch(masks[sel, :words(traces[t])], codes[t], flags)
            assert as_bytes(got[sel]).tobytes() == as_bytes(want).tobytes(), (t, flags)
        if flags == 0:                              # BackTrack: every delivery of the first trace overflows (mask 0)
            assert got["status"][0] == S.PS_PENDING_OVF and (got["status"] == 0).any()
    # the minimization: a trace whose first test overflows fails alone, as the single call fails
    for flags in (0, N.WC_LAST_ONLY):
        many = eng.wildcard_minimize_many(codes, flags, cap_events=65536)
        status = many[3]
        assert (status == N.OK).any() and ((status == N.OK) | (status == N.ERR_CAPACITY)).all(), status
        if flags == 0:
            assert status[0] == N.ERR_CAPACITY
            msg = eng.last_error()
            assert "trace 0:" in msg and "status %d" % S.PS_PENDING_OVF in msg, msg
        check_against_solo(lambda: engine(N.MODEL_BCAST32, 1, BC_RULES, ()), traces, exts, codes, flags, many, cap=65536)


def test_state_and_arguments():
    eng, traces, exts, codes = intmin_set(0, 64)
    fresh = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR)
    with pytest.raises(D.DemiError) as ei:
        fresh.wildcard_minimize_many(codes[:1])
    assert ei.value.code == N.ERR_STATE
    with pytest.raises(D.DemiError) as ei:
        fresh.wildcard_replay_batch_many([0], np.zeros((1, 1), np.uint64), codes[:1])
    assert ei.value.code == N.ERR_STATE
    eng.set_traces(traces, exts)
    eng.set_trace(traces[7], exts[7])
    L = N.lib()
    n = len(traces)
    # what the set and the handle's trace replay to: unchanged after every call below
    rng = np.random.default_rng(2)
    mw = max(words(t) for t in traces)
    trs = np.repeat(np.arange(n, dtype=np.uint32), 3)
    masks = np.concatenate([include_masks(t, 3, mw, rng) for t in traces])
    own = masks[trs == 7][:, :words(traces[7])]
    before = as_bytes(eng.wildcard_replay_batch_many(trs, masks, codes)).tobytes()
    single = as_bytes(eng.wildcard_replay_batch(own, codes[7])).tobytes()

    def unchanged():
        assert as_bytes(eng.wildcard_replay_batch_many(trs, masks, codes)).tobytes() == before
        assert as_bytes(eng.wildcard_replay_batch(own, codes[7])).tobytes() == single

    ev = np.zeros((n, 64), dtype=N.EVENT_DTYPE)
    out = np.zeros(n, dtype=N.INTMIN_OUT_DTYPE)
    st = np.zeros(n, dtype=np.int32)
    lf = np.ascontiguousarray(codes, dtype=np.uint32)
    args = [lf.ctypes.data, 0, ev.ctypes.data, 64, None, 0, out.ctypes.data, st.ctypes.data]
    for k in (0, 2, 6, 7):
        bad = list(args)
        bad[k] = None
        assert L.demi_wildcard_minimize_many(eng._h, *bad) == N.ERR_INVALID
        unchanged()
    for flags in (N.RF_STRICT, 0x40000, N.IM_SRC_DST_FIFO):
        bad = list(args)
        bad[1] = flags
        assert L.demi_wildcard_minimize_many(eng._h, *bad) == N.ERR_INVALID
        unchanged()
    tr = np.zeros(1, dtype=np.uint32)
    m = np.zeros(1, dtype=np.uint64)
    res = np.zeros(1, dtype=N.REPLAY_DTYPE)
    assert L.demi_wildcard_replay_batch_many(eng._h, tr.ctypes.data, None, 1, 1, lf.ctypes.data, 0, res.ctypes.data) == N.ERR_INVALID
    unchanged()
    assert L.demi_wildcard_replay_batch_many(eng._h, tr.ctypes.data, m.ctypes.data, 1, 1, lf.ctypes.data, N.RF_STRICT,
                                             res.ctypes.data) == N.ERR_INVALID
    unchanged()
    far = np.array([n], dtype=np.uint32)
    assert L.demi_wildcard_replay_batch_many(eng._h, far.ctypes.data, m.ctypes.data, 1, 1, lf.ctypes.data, 0,
                                             res.ctypes.data) == N.ERR_INVALID
    big = int(np.argmax([n_deliv(t) for t in traces]))
    if words(traces[big]) > 1:
        one = np.array([big], dtype=np.uint32)
        assert L.demi_wildcard_replay_batch_many(eng._h, one.ctypes.data, m.ctypes.data, 1, 1, lf.ctypes.data, 0,
                                                 res.ctypes.data) == N.ERR_INVALID
    unchanged()
    # the successful calls leave them too
    for flags in (0, N.WC_LAST_ONLY):
        eng.wildcard_minimize_many(codes, flags)
        unchanged()


# ---------------------------------------------------------------- 7. one handle, every kind of launch
def test_one_handle_runs_every_kind_of_launch_in_turn():
    eng, traces, exts, codes = intmin_set(0, 64)
    tr8, ex8, cd8 = traces[:8], exts[:8], codes[:8]
    rng = np.random.default_rng(6)
    mw = max(words(t) for t in tr8)
    trs = np.repeat(np.arange(8, dtype=np.uint32), 4)
    inc = np.concatenate([include_masks(t, 4, mw, rng) for t in tr8])
    emw = max(1, (max(len(e) for e in ex8) + 63) // 64)
    ext_masks = np.full((len(trs), emw), ~np.uint64(0), dtype=np.uint64)

    def steps(h, fresh):
        got = []
        if fresh: h = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR)
        h.set_trace(tr8[2], ex8[2])
        got.append(h.wildcard_replay_batch(inc[trs == 2][:, :words(tr8[2])], cd8[2], N.WC_LAST_ONLY))
        if fresh: h = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR)
        h.set_traces(tr8, ex8)
        got.append(h.wildcard_replay_batch_many(trs, inc, cd8))
        if fresh: h = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR); h.set_traces(tr8, ex8)
        got.append(h.replay_batch_many(trs, ext_masks, cd8, mask_words=emw))
        if fresh: h = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR); h.set_traces(tr8, ex8)
        got += list(h.wildcard_minimize_many(cd8, 0))
        if fresh: h = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR); h.set_traces(tr8, ex8)
        got += list(h.internal_minimize_many(cd8, 0))
        if fresh: h = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR); h.set_traces(tr8, ex8)
        got.append(h.replay_batch_many(trs, ext_masks, cd8, mask_words=emw))
        if fresh: h = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR)
        h.set_trace(tr8[3], ex8[3])
        got.append(h.wildcard_minimize(cd8[3], 0)[0])
        return got

    shared = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR)
    for a, b in zip(steps(shared, False), steps(None, True)):
        assert as_bytes(a).tobytes() == as_bytes(b).tobytes()


# ---------------------------------------------------------------- 8. the chain at scale
def test_full_chain_on_1024_violations_equals_the_per_trace_chain():
    prog = D.raft5_program()
    ext = D.pack_externals(prog)
    eng = raft_engine(prog)
    eng.set_clock_rules(RULES, INCR)
    hits, _ = raft_hits(eng, 200000, 1200)
    ev, ne, r = eng.fuzz_traces(1, hits, MAXM, INTERVAL, cap_events=1024)
    codes = r["violation"].astype(np.uint32)
    eng.set_traces((ev, ne), ext)
    mw = eng.set_mask_words()
    mcs, _, _, status = eng.ddmin_many(codes)
    assert (status == N.OK).all()
    rev, rne, rres = eng.replay_traces_many(np.arange(len(ne), dtype=np.uint32), mcs, None, codes, cap_events=1024)
    ok = np.nonzero((rres["status"] == 0) & (rres["violation"] == codes))[0]
    traces = [rev[i, :rne[i]].copy() for i in ok]
    exts = [D.pack_externals(D.events_of(prog, mcs[i, :mw])) for i in ok]
    cd = codes[ok]
    eng.set_traces(traces, exts)
    iev, _, iout, ist = eng.internal_minimize_many(cd, N.IM_SRC_DST_FIFO, cap_events=1024)
    keep = np.nonzero(ist == N.OK)[0]
    itr = [iev[t, :iout[t]["n_events"]].copy() for t in keep]
    iex, icd = [exts[t] for t in keep], cd[keep]
    assert len(itr) >= 1024
    eng.set_traces(itr, iex)
    w1 = eng.wildcard_minimize_many(icd, 0, cap_events=1024)
    ok1 = np.nonzero(w1[3] == N.OK)[0]
    eng.set_traces([w1[0][t, :w1[2][t]["n_events"]].copy() for t in ok1], [iex[t] for t in ok1])
    w2 = eng.wildcard_minimize_many(icd[ok1], N.WC_LAST_ONLY, cap_events=1024)
    k = 0
    for t in range(len(itr)):
        solo = engine(N.MODEL_RAFT5, RAFT_FLAGS, RULES, INCR)             # a fresh handle per trace, for both stages
        st, _, t1, _, o1 = solo_wc(solo, itr[t], iex[t], icd[t], 0, 1024)
        assert st == w1[3][t], t
        if st != N.OK:
            continue
        assert as_bytes(w1[2][t]).tobytes() == as_bytes(o1).tobytes(), t
        st2, _, t2, s2, o2 = solo_wc(solo, t1, iex[t], icd[t], N.WC_LAST_ONLY, 1024)
        assert st2 == w2[3][k], t
        if st2 == N.OK:
            assert as_bytes(w2[2][k]).tobytes() == as_bytes(o2).tobytes(), t
            n = int(o2["n_events"])
            assert (w2[0][k, :n] == t2[:n]).all(), t
        k += 1
