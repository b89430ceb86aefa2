"""The calls over a set of traces (demi_set_traces, demi_replay_batch_many, demi_ddmin_many, demi_replay_traces_many,
demi_internal_minimize_many) where a kernel or host path that mixed up two traces would go wrong: warps that run tiles
of several traces, sets of mixed lengths, capacities, programs and mask widths, every model, both execution switches,
mask bits past a trace's externals, launches split by size, and one handle running every kind of launch in turn.

Every record is compared bit for bit with the single-trace entry points on a fresh handle, and a sample of traces
(at least one in 20, all of its tests) with the CPU oracle.  tests/test_many_traces_edges_oracle.py checks on the
oracle that these inputs show what they are here to show: per-trace capacity statuses, several codes, a code that
is not met, switches that change the records, traces of 1, 2 and 3 mask words."""
import ctypes as C

import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
import many_sets as S
from oracle import binding as O
from test_config_switches_gpu import K2_CASES, blocked_candidates

pytestmark = pytest.mark.gpu

NONE = 0xFFFFFFFF
FLAGS = (0, N.RF_FILTER_KNOWN_ABSENTS, N.RF_STRICT)
DD_FIELDS = ["mcs_size", "total_replays", "n_iterations", "replays_executed", "batches", "verified"]


def as_bytes(a):
    return np.ascontiguousarray(a).view(np.uint8)


def engine(model, flags, blob=None, blocked=0, it=False):
    eng = D.Engine(D.SchedulerConfig(model, model_flags=flags, blocked_mask=blocked, ignoreTimers=it))
    if blob is not None:
        eng.load_model(blob)
    return eng


def own_mw(ext):
    return O.mask_words(len(ext))


def resident_warps():
    import torch
    return 64 * torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------------- the sets
def model_sets():
    """(name, model, model_flags, blob, traces, externals, codes) of every model."""
    out = [("raft5", S.RAFT, S.RAFT_FLAGS, None) + S.raft5_mixed(),
           ("pingpong3", S.PP, S.PP_FLAGS, None) + S.pingpong3_set(),
           ("bcast32", S.BC, S.BC_FLAGS, None) + S.bcast32_set()]
    m, tr, ex, co = S.election_set()
    out.append(("election", S.IR, m.flags, m.blob, tr, ex, co))
    return out


_SETS = {}


def sets():
    if not _SETS:
        for s in model_sets():
            _SETS[s[0]] = s
    return _SETS


def load(model_blob):
    if model_blob is not None:
        O.load_model(model_blob)


def shuffled_tests(exts, counts, rng, pool=64):
    """Tests of trace t: counts[t] rows drawn from a pool of S.masks; in shuffled order.  -> (trace_of_test, masks at
    the set's width, pool index of each test, pools)."""
    pools = [S.masks(e, pool, rng) for e in exts]
    mw = max(own_mw(e) for e in exts)
    tr = np.repeat(np.arange(len(exts), dtype=np.uint32), counts)
    pick = np.concatenate([rng.integers(0, pool, size=c) for c in counts])
    pick[np.concatenate([[0], np.cumsum(counts)[:-1]])] = 0                  # every trace replays its full program once
    m = np.zeros((len(tr), mw), dtype=np.uint64)
    for t in range(len(exts)):
        sel = tr == t
        m[sel, :pools[t].shape[1]] = pools[t][pick[sel]]
    perm = rng.permutation(len(tr))
    return tr[perm], m[perm], pick[perm], pools


# --------------------------------------------------------------------------------- 1. warps that switch traces
@pytest.mark.parametrize("name", ["raft5", "bcast32", "pingpong3", "election"])
def test_warps_switch_traces(name):
    """replay_batch_many with at least three tiles on every resident warp of the GPU: each warp binds several traces
    in turn, longest first, so a field kept from the previous tile (events, externals, capacities, looking_for) changes
    the records.  Peak memory: ~2.5 M tests, ~60 MB host, ~90 MB device."""
    _, model, flags, blob, traces, exts, codes = sets()[name]
    load(blob)
    rng = np.random.default_rng(11)
    need = 3 * resident_warps()
    per = -(-need * 21 // 20 // len(traces))                                  # tiles per trace, 5 % to spare
    counts = np.array([32 * (per - 1) + int(rng.integers(1, 33)) for _ in traces])
    tiles = int(sum(-(-c // 32) for c in counts))
    assert tiles >= need
    tr, masks, pick, pools = shuffled_tests(exts, counts, rng)
    eng = engine(model, flags, blob)
    eng.set_traces(traces, exts)
    solo = engine(model, flags, blob)
    overflowed = set()
    for fl in FLAGS:
        many = eng.replay_batch_many(tr, masks, codes, fl)
        assert eng.stats().kernel_launches == 1 and eng.stats().prefixes == len(tr)
        for t in range(len(traces)):
            sel = np.nonzero(tr == t)[0]
            solo.set_trace(traces[t], exts[t])
            one = solo.replay_batch(masks[sel, :own_mw(exts[t])], int(codes[t]), fl)
            assert (as_bytes(many[sel]) == as_bytes(one)).all(), (name, t, fl)
            if (many["status"][sel] == S.PS_PENDING_OVF).any():
                overflowed.add(t)
            if t % 7 == 0 or t == len(traces) - 1:
                cpu = O.replay_batch(model, traces[t], exts[t], pools[t], looking_for=int(codes[t]), flags=fl,
                                     model_flags=flags)
                assert (many[sel] == cpu[pick[sel]]).all(), (name, t, fl)
    if name in ("raft5", "bcast32"):
        # the short copies overflow their own pending set in this regime; the traces they were made from do not
        n_ev = np.array([len(t) for t in traces])
        assert overflowed and all(n_ev[t] < max(n_ev) for t in overflowed)
        assert any((traces[t]["kind"] == N.EV_MSG_SEND).sum() < (traces[t]["kind"] == N.EV_MSG_EVENT).sum()
                   for t in overflowed)


# ------------------------------------------------------------------------------------- 2. ddmin_many, every model
def solo_ddmin(eng, trace, ext, code, flags):
    eng.set_trace(trace, ext)
    mw = own_mw(ext)
    mcs = np.zeros(mw, dtype=np.uint64)
    iters = np.zeros(256, dtype=np.uint32)
    out = N.DDMinOut()
    rc = N.lib().demi_ddmin(eng._h, int(code), flags, 1, mcs.ctypes.data, mw, iters.ctypes.data, 256, C.byref(out))
    return rc, mcs, iters, out


def check_ddmin_many(model, flags, blob, traces, exts, codes, fl, mw=None, oracle_every=8):
    eng = engine(model, flags, blob)
    eng.set_traces(traces, exts)
    mcs, iters, out, status = eng.ddmin_many(codes, fl, mask_words=mw)
    solo = engine(model, flags, blob)
    for t in range(len(traces)):
        rc, smcs, siters, sout = solo_ddmin(solo, traces[t], exts[t], codes[t], fl)
        assert status[t] == rc, (t, fl, status[t], rc)
        if rc != N.OK:
            continue
        w = own_mw(exts[t])
        assert (mcs[t, :w] == smcs).all() and (mcs[t, w:] == 0).all(), (t, fl)
        assert (iters[t] == siters).all(), (t, fl)
        for f in DD_FIELDS:
            assert out[t][f] == getattr(sout, f), (t, fl, f)
        if t % oracle_every == 0:
            crc, cmcs, total, citers, ver = O.ddmin_sts(model, traces[t], exts[t], int(codes[t]), flags=fl, model_flags=flags)
            assert crc == 0 and (cmcs == smcs).all() and total == sout.total_replays and ver == sout.verified, (t, fl)
            assert list(citers) == list(siters[:sout.n_iterations]), (t, fl)
    return mcs, status


@pytest.mark.parametrize("wide", [None, "64"])
@pytest.mark.parametrize("name", ["raft5", "bcast32", "pingpong3", "election"])
def test_ddmin_many_every_model(monkeypatch, name, wide):
    """Every trace against a solo demi_ddmin at its own mask width, for flags 0, filterKnownAbsents and strict."""
    if wide:
        monkeypatch.setenv("DEMI_DDMIN_WIDE", wide)
    _, model, flags, blob, traces, exts, codes = sets()[name]
    load(blob)
    ok = 0
    for fl in FLAGS:
        _, status = check_ddmin_many(model, flags, blob, traces, exts, codes, fl)
        ok += int((status == N.OK).sum())
    assert ok > 0
    if name == "raft5":
        # the traces of 1 and 2 mask words, at their set's width (2) and at 3
        sub = [t for t in range(len(traces)) if own_mw(exts[t]) <= 2]
        args = ([traces[t] for t in sub], [exts[t] for t in sub], codes[sub])
        assert {own_mw(e) for e in args[1]} == {1, 2}
        a = check_ddmin_many(model, flags, blob, *args, 0)
        b = check_ddmin_many(model, flags, blob, *args, 0, mw=3)
        assert (a[1] == b[1]).all() and (b[0][:, :2] == a[0]).all() and (b[0][:, 2] == 0).all()


def test_ddmin_many_generated_timer_models():
    """Generated loaded models that arm timers (tests/ir_gen.py), a set of 4 violating executions each."""
    got = S.generated_timer_sets(range(1, 121))
    assert len(got) >= 3
    for m, traces, exts, codes in got:
        O.load_model(m.blob)
        for fl in FLAGS:
            check_ddmin_many(S.IR, m.flags, m.blob, traces, exts, codes, fl, oracle_every=2)


# --------------------------------------------------------------- 3. recording and internal minimization on mixed sets
def check_replay_traces(eng, solo, model, flags, traces, exts, codes, tr, masks, skips, fl, cap, oracle_every=9):
    rev, rne, rres = eng.replay_traces_many(tr, masks, skips, codes, fl, cap_events=cap)
    for i, t in enumerate(tr):
        w = own_mw(exts[t])
        mask = None if masks is None else masks[i, :w]
        skip = NONE if skips is None else int(skips[i])
        solo.set_trace(traces[t], exts[t])
        sres, sev = solo.replay_trace(mask, skip, int(codes[t]), fl, cap)
        assert as_bytes(rres[i:i + 1]).tobytes() == as_bytes(np.array([sres])).tobytes(), (i, t, fl)
        assert rne[i] == len(sev) and (rev[i, :rne[i]] == sev).all(), (i, t, fl)
        if oracle_every and i % oracle_every == 0:
            om = O.full_mask(exts[t], False) if mask is None else mask
            cres, cev = O.replay_trace(model, traces[t], exts[t], om, looking_for=int(codes[t]), flags=fl, model_flags=flags,
                                       skip_event=skip)
            assert cres == sres and len(cev) == len(sev) and (cev == sev).all(), (i, t, fl)
    return rev, rne, rres


def intmin_solo(eng, trace, ext, code, fl, cap):
    eng.set_trace(trace, ext)
    try:
        t, s, o = eng.internal_minimize(int(code), fl, cap_events=cap)
    except D.DemiError as e:
        return e.code, None, None, None
    out = np.zeros(1, dtype=N.INTMIN_OUT_DTYPE)
    out.view(np.uint8)[:] = np.frombuffer(bytes(o), dtype=np.uint8)
    return N.OK, t, s, out[0]


def check_intmin_many(model, flags, blob, traces, exts, codes, fl, cap=4096, oracle_every=4, switches=None):
    sw = switches or {}
    eng = engine(model, flags, blob, sw.get("blocked_mask", 0), bool(sw.get("ignore_timers", 0)))
    eng.set_traces(traces, exts)
    ev, sizes, out, status = eng.internal_minimize_many(codes, fl, cap_events=cap)
    solo = engine(model, flags, blob, sw.get("blocked_mask", 0), bool(sw.get("ignore_timers", 0)))
    for t in range(len(traces)):
        st, strace, ssizes, sout = intmin_solo(solo, traces[t], exts[t], codes[t], fl, cap)
        assert status[t] == st, (t, fl)
        if st != N.OK:
            continue
        assert as_bytes(out[t]).tobytes() == as_bytes(sout).tobytes(), (t, fl)
        n = int(out[t]["n_events"])
        assert (ev[t, :n] == strace).all() and (sizes[t, :out[t]["n_internal_sizes"]] == ssizes).all(), (t, fl)
        if t % oracle_every == 0:
            rc, ctrace, total, csizes, unig = O.internal_minimize(model, traces[t], exts[t], int(codes[t]), flags=fl,
                                                                  model_flags=flags, **sw)
            assert rc == 0 and n == len(ctrace) and (ev[t, :n] == ctrace).all(), (t, fl)
            assert out[t]["total_replays"] == total and out[t]["unignorable"] == unig, (t, fl)
            assert (sizes[t, :out[t]["n_internal_sizes"]] == csizes).all(), (t, fl)
    return ev, out, status


def verified(eng, traces, exts, codes, cap=4096):
    """Each trace's recorded replay of its full program: a verified trace whose MCS is every external."""
    eng.set_traces(traces, exts)
    rev, rne, rres = eng.replay_traces_many(np.arange(len(traces), dtype=np.uint32), None, None, codes, 0, cap_events=cap)
    keep = np.nonzero((rres["status"] == 0) & (rres["violation"] == codes) & (codes != 0))[0]
    return [rev[i, :rne[i]].copy() for i in keep], [exts[i] for i in keep], codes[keep]


@pytest.mark.parametrize("name", ["raft5", "bcast32", "election"])
def test_replay_traces_and_internal_minimize_many_mixed(name):
    _, model, flags, blob, traces, exts, codes = sets()[name]
    load(blob)
    rng = np.random.default_rng(12)
    eng = engine(model, flags, blob)
    eng.set_traces(traces, exts)
    solo = engine(model, flags, blob)
    counts = rng.integers(3, 9, size=len(traces))
    tr, masks, _, _ = shuffled_tests(exts, counts, rng)
    skips = np.array([NONE if k % 3 == 0 else int(rng.choice(np.nonzero(traces[t]["kind"] == N.EV_MSG_EVENT)[0]))
                      for k, t in enumerate(tr)], dtype=np.uint32)
    for fl in FLAGS:
        for m, sk in ((masks, skips), (None, skips), (masks, None)):
            check_replay_traces(eng, solo, model, flags, traces, exts, codes, tr, m, sk, fl, 4096)
            assert eng.stats().kernel_launches == 1
    vt, vx, vc = verified(eng, traces, exts, codes)
    assert len(vt) >= 4 and len({len(t) for t in vt}) > 1
    for fl in (0, N.IM_SRC_DST_FIFO, N.RF_FILTER_KNOWN_ABSENTS):
        check_intmin_many(model, flags, blob, vt, vx, vc, fl)


def test_recordings_of_many_traces_per_warp():
    """demi_replay_traces_many with one test on each of more than 3 x 64 x SMs raft5 traces: every warp records tiles
    of several traces.  Peak memory: ~0.9 GB host (the rows), ~1 GB device."""
    prog = D.raft5_program()
    ext = D.pack_externals(prog)
    eng = engine(S.RAFT, S.RAFT_FLAGS)
    eng.set_externals(prog)
    n = 3 * resident_warps() * 21 // 20
    ev, ne, r = eng.fuzz_traces(1, np.arange(n, dtype=np.uint32), 50, 5, cap_events=1024)
    assert (r["status"] == 0).all()
    codes = r["violation"].astype(np.uint32)
    eng.set_traces((ev, ne), ext)
    rng = np.random.default_rng(13)
    masks = S.masks(ext, n, rng)
    tr = rng.permutation(n).astype(np.uint32)
    cap = 1024
    rev, rne, rres = eng.replay_traces_many(tr, masks[tr], None, codes, 0, cap_events=cap)
    assert eng.stats().kernel_launches == 1
    solo = engine(S.RAFT, S.RAFT_FLAGS)
    for i, t in enumerate(tr):
        solo.set_trace(ev[t, :ne[t]], ext)
        sres, sev = solo.replay_trace(masks[t], NONE, int(codes[t]), 0, cap)
        assert as_bytes(rres[i:i + 1]).tobytes() == as_bytes(np.array([sres])).tobytes(), (i, t)
        assert rne[i] == len(sev) and (rev[i, :rne[i]] == sev).all(), (i, t)
        if i % 997 == 0:
            cres, cev = O.replay_trace(S.RAFT, ev[t, :ne[t]], ext, masks[t], looking_for=int(codes[t]), model_flags=S.RAFT_FLAGS)
            assert cres == sres and (cev == sev).all(), (i, t)


# ---------------------------------------------------------------------------------------------------- 4. switches
def switch_set(model, prog, flags, maxm, interval, n=4):
    ext = D.pack_externals(prog)
    got = S.violating(model, ext, flags, maxm, interval, n, 4000)
    return [g[0] for g in got], [ext] * n, np.array([g[1] for g in got], dtype=np.uint32)


@pytest.mark.parametrize("case", K2_CASES, ids=[c[0] for c in K2_CASES])
def test_set_replays_under_switches(case):
    """replay_batch_many, replay_traces_many and ddmin_many under blockedActors / ignoreTimers against the oracle under
    the same switches, on traces recorded without them; the records differ from the unswitched ones."""
    _, model, prog, flags, maxm, interval, blocked, it = case
    sw = dict(blocked_mask=blocked, ignore_timers=1 if it else 0)
    traces, exts, codes = switch_set(model, prog, flags, maxm, interval)
    rng = np.random.default_rng(14)
    tr, masks, pick, pools = shuffled_tests(exts, [40] * len(traces), rng)
    on, off = engine(model, flags, blocked=blocked, it=it), engine(model, flags)
    on.set_traces(traces, exts)
    off.set_traces(traces, exts)
    for fl in FLAGS:
        a = on.replay_batch_many(tr, masks, codes, fl)
        b = off.replay_batch_many(tr, masks, codes, fl)
        assert (a != b).sum() > len(a) // 4
        if fl != N.RF_STRICT:                          # strict replays diverge where the others ignore a delivery
            assert a["ignored"].sum() > b["ignored"].sum()
        for t in range(len(traces)):
            sel = tr == t
            cpu = O.replay_batch(model, traces[t], exts[t], pools[t], looking_for=int(codes[t]), flags=fl, model_flags=flags, **sw)
            assert (a[sel] == cpu[pick[sel]]).all(), (t, fl)
    rev, rne, rres = on.replay_traces_many(tr[:24], masks[:24], None, codes, 0, cap_events=4096)
    for i, t in enumerate(tr[:24]):
        cres, cev = O.replay_trace(model, traces[t], exts[t], masks[i, :own_mw(exts[t])], looking_for=int(codes[t]),
                                   model_flags=flags, **sw)
        assert cres == rres[i] and rne[i] == len(cev) and (rev[i, :rne[i]] == cev).all(), i
    mcs, _, out, status = on.ddmin_many(codes)
    for t in range(len(traces)):
        crc, cmcs, total, citers, ver = O.ddmin_sts(model, traces[t], exts[t], int(codes[t]), model_flags=flags, **sw)
        assert (status[t] == N.OK) == (crc == 0), t
        if crc == 0:
            assert (mcs[t] == cmcs).all() and out[t]["total_replays"] == total and out[t]["verified"] == ver, t


@pytest.mark.parametrize("name,model,prog,flags,maxm,interval,actors", [
    ("raft5", S.RAFT, D.raft5_program(client_cmds=8), 1, 50, 5, range(5)),
    ("pingpong3", S.PP, D.pingpong3_program(24), 1 | (5 << 8), -1, 3, (1, 2)),
])
def test_set_minimizers_under_a_mask(name, model, prog, flags, maxm, interval, actors):
    """ddmin_many and internal_minimize_many under a blocked-actor mask against the oracle, on the traces of
    test_config_switches_gpu's blocked_candidates (the mask changes their minimization), grouped by mask."""
    by_mask = {}
    for ext, ev, code, blocked in blocked_candidates(model, prog, flags, maxm, interval, actors, limit=8):
        by_mask.setdefault(blocked, []).append((ext, ev, code))
    assert by_mask
    for blocked, cases in by_mask.items():
        sw = dict(blocked_mask=blocked)
        exts = [c[0] for c in cases]
        traces = [c[1] for c in cases]
        codes = np.array([c[2] for c in cases], dtype=np.uint32)
        eng = engine(model, flags, blocked=blocked)
        eng.set_traces(traces, exts)
        mcs, _, out, status = eng.ddmin_many(codes)
        for t in range(len(cases)):
            crc, cmcs, total, citers, ver = O.ddmin_sts(model, traces[t], exts[t], int(codes[t]), model_flags=flags, **sw)
            assert crc == 0 and status[t] == N.OK and (mcs[t] == cmcs).all() and out[t]["total_replays"] == total, t
        vt, vx = [], []
        for ext, ev, code in cases:
            _, v = O.replay_trace(model, ev, ext, O.full_mask(ext), looking_for=code, model_flags=flags)
            vt.append(v)
            vx.append(ext[ext["kind"] != N.EXT_WAIT_QUIESCENCE])
        check_intmin_many(model, flags, None, vt, vx, codes, 0, oracle_every=1, switches=sw)


@pytest.mark.parametrize("model,prog,flags,maxm,interval", [
    (S.RAFT, D.raft5_program(client_cmds=4), 1, 50, 5),
])
def test_ddmin_many_under_ignore_timers(model, prog, flags, maxm, interval):
    """ddmin_many under ignoreTimers against the oracle under the same switch.  (raft5 elects through its timers, so
    its violating traces stop violating without them: there is no verified trace to minimize internally.)"""
    traces, exts, codes = switch_set(model, prog, flags, maxm, interval, n=6)
    sw = dict(ignore_timers=1)
    eng = engine(model, flags, it=True)
    eng.set_traces(traces, exts)
    mcs, _, out, status = eng.ddmin_many(codes)
    for t in range(len(traces)):
        crc, cmcs, total, citers, ver = O.ddmin_sts(model, traces[t], exts[t], int(codes[t]), model_flags=flags, **sw)
        assert (status[t] == N.OK) == (crc == 0), t
        if crc == 0:
            assert (mcs[t] == cmcs).all() and out[t]["total_replays"] == total, t


# ---------------------------------------------------------------------------------------------- 5. mask padding
def test_mask_bits_past_the_externals_are_ignored():
    """Random bits at and past each trace's n_externals, within the call's mask_words, give the clean masks' records:
    replay_batch_many, replay_traces_many and demi_replay_batch."""
    _, model, flags, blob, traces, exts, codes = sets()["raft5"]
    rng = np.random.default_rng(15)
    tr, masks, _, _ = shuffled_tests(exts, [24] * len(traces), rng)
    dirty = np.concatenate([S.pad(masks[i:i + 1, :own_mw(exts[t])], exts[t], 3, rng) for i, t in enumerate(tr)])
    assert (dirty != masks).any(axis=1).all()
    eng = engine(model, flags)
    eng.set_traces(traces, exts)
    for fl in FLAGS:
        assert (as_bytes(eng.replay_batch_many(tr, dirty, codes, fl)) == as_bytes(eng.replay_batch_many(tr, masks, codes, fl))).all()
    a = eng.replay_traces_many(tr, dirty, None, codes, 0, cap_events=4096)
    b = eng.replay_traces_many(tr, masks, None, codes, 0, cap_events=4096)
    assert (a[1] == b[1]).all() and (as_bytes(a[2]) == as_bytes(b[2])).all()
    for i in range(len(tr)):
        assert (a[0][i, :a[1][i]] == b[0][i, :b[1][i]]).all()
    L = N.lib()
    for t in range(len(traces)):
        sel = np.nonzero(tr == t)[0]
        eng.set_trace(traces[t], exts[t])
        for m in (dirty, masks):
            out = np.zeros(len(sel), dtype=N.REPLAY_DTYPE)
            mm = np.ascontiguousarray(m[sel])
            assert L.demi_replay_batch(eng._h, mm.ctypes.data, len(sel), 3, int(codes[t]), 0, out.ctypes.data) == N.OK
            if m is dirty:
                first = out
        assert (as_bytes(first) == as_bytes(out)).all(), t


# ---------------------------------------------------------------------------------------------- 6. launch splits
def small_pingpong():
    traces, exts, codes = S.pingpong3_set()
    keep = [t for t in range(len(traces)) if len(exts[t]) <= 24]
    return [traces[t] for t in keep], [exts[t] for t in keep], codes[keep]


def test_exact_launch_splits_above_a_million_tests():
    """2^20 + 33 tests in shuffled order run as two launches; every record equals solo.  Peak memory: ~120 MB host,
    ~40 MB device."""
    traces, exts, codes = small_pingpong()
    rng = np.random.default_rng(16)
    n = (1 << 20) + 33
    counts = np.full(len(traces), n // len(traces))
    counts[: n - counts.sum()] += 1
    tr, masks, _, _ = shuffled_tests(exts, counts, rng, pool=256)
    eng = engine(S.PP, S.PP_FLAGS)
    eng.set_traces(traces, exts)
    many = eng.replay_batch_many(tr, masks, codes)
    assert eng.stats().kernel_launches == 2 and eng.stats().prefixes == n
    solo = engine(S.PP, S.PP_FLAGS)
    for t in range(len(traces)):
        sel = np.nonzero(tr == t)[0]
        solo.set_trace(traces[t], exts[t])
        assert (as_bytes(many[sel]) == as_bytes(solo.replay_batch(masks[sel, :own_mw(exts[t])], int(codes[t])))).all(), t


@pytest.mark.parametrize("n,launches", [(1025, 2), (2049, 3)])
def test_recording_launch_splits_at_a_gibibyte_of_rows(n, launches):
    """At cap_events = 65 536 a launch records at most 1 024 tests (1 GiB of rows).  Every row and count equals solo,
    those of the tests right after each split included.  Peak memory: the output is n x 1 MiB of np.zeros, of which only
    the recorded events are touched (~10 MB host); ~1 GiB device."""
    traces, exts, codes = small_pingpong()
    rng = np.random.default_rng(17)
    cap = 65536
    counts = np.full(len(traces), n // len(traces))
    counts[: n - counts.sum()] += 1
    tr, masks, pick, pools = shuffled_tests(exts, counts, rng, pool=8)
    eng = engine(S.PP, S.PP_FLAGS)
    eng.set_traces(traces, exts)
    rev, rne, rres = eng.replay_traces_many(tr, masks, None, codes, 0, cap_events=cap)
    assert eng.stats().kernel_launches == launches
    solo = engine(S.PP, S.PP_FLAGS)
    want = {}
    for t in range(len(traces)):
        solo.set_trace(traces[t], exts[t])
        for p in range(len(pools[t])):
            want[(t, p)] = solo.replay_trace(pools[t][p], NONE, int(codes[t]), 0, cap)
    for i, t in enumerate(tr):
        sres, sev = want[(int(t), int(pick[i]))]
        assert as_bytes(rres[i:i + 1]).tobytes() == as_bytes(np.array([sres])).tobytes(), i
        assert rne[i] == len(sev) > 0 and (rev[i, :rne[i]] == sev).all(), i


# -------------------------------------------------------------------------------- 7. one handle, many kinds of launch
def test_one_handle_many_kinds_of_launch():
    """On one raft5 handle: replay_batch, replay_batch_many, replay_traces_many, replay_batch, wildcard_replay_batch,
    internal_minimize_many, replay_batch_many; each equals the same call on a fresh handle."""
    _, model, flags, _, traces, exts, codes = sets()["raft5"]
    rng = np.random.default_rng(18)
    tr, masks, _, _ = shuffled_tests(exts, [20] * len(traces), rng)
    single, sext, scode = traces[4], exts[4], int(codes[4])
    smasks = S.masks(sext, 200, rng)
    eng = engine(model, flags)
    vt, vx, vc = verified(engine(model, flags), traces, exts, codes)
    n_del = int((single["kind"] == N.EV_MSG_EVENT).sum())
    wmasks = rng.integers(0, 1 << 64, size=(64, max(1, (n_del + 63) // 64)), dtype=np.uint64, endpoint=False)

    def fresh():
        return engine(model, flags)

    def batch(e):
        e.set_trace(single, sext)
        return as_bytes(e.replay_batch(smasks, scode)).tobytes()

    def batch_many(e):
        e.set_traces(traces, exts)
        return as_bytes(e.replay_batch_many(tr, masks, codes, N.RF_FILTER_KNOWN_ABSENTS)).tobytes()

    def traces_many(e):
        e.set_traces(traces, exts)
        ev, ne, res = e.replay_traces_many(tr, masks, None, codes, 0, cap_events=4096)
        return as_bytes(res).tobytes(), ne.tobytes(), b"".join(as_bytes(ev[i, :ne[i]]).tobytes() for i in range(len(ne)))

    def wildcard(e):
        e.set_trace(single, sext)
        return as_bytes(e.wildcard_replay_batch(wmasks, scode)).tobytes()

    def intmin_many(e):
        e.set_traces(vt, vx)
        ev, sizes, out, status = e.internal_minimize_many(vc, N.IM_SRC_DST_FIFO)
        return ev.tobytes(), sizes.tobytes(), as_bytes(out).tobytes(), status.tobytes()

    for step in (batch, batch_many, traces_many, batch, wildcard, intmin_many, batch_many):
        assert step(eng) == step(fresh()), step.__name__
