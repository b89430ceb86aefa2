"""randomDDMin over many programs in one call (demi_random_test_batch_many / demi_random_ddmin_many): per trace, the
records of demi_random_test_batch on that program alone and the C oracle's, and the outputs of demi_set_externals +
demi_random_ddmin on that program, whichever traces share the launches."""
import ctypes as C

import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
from demi_b200.fuzzer import ClientCommandGenerator, Fuzzer, FuzzerWeights
import ir_gen
from test_random_ddmin_gpu import PP_HK, engine, random_masks, rows
from test_random_ddmin_oracle import PP_FLAGS, RAFT_FLAGS, RAFT_WQ, atoms_cover, bits, _oracle_cfg

pytestmark = pytest.mark.gpu
OUT_FIELDS = ("mcs_size", "tests", "n_iterations", "verified", "total_replays", "tests_evaluated", "batches",
              "mcs_first_hit")


@pytest.fixture(scope="module")
def rd():
    from demi_b200 import build
    build.build_oracle()
    from oracle import random_ddmin_binding
    random_ddmin_binding.lib()
    return random_ddmin_binding


def raft5_programs(n, num_events=(6, 10, 14)):
    """Fuzzer programs of a raft5 campaign (bench_random_ddmin.py's Fuzzer) of mixed lengths"""
    out = []
    for s in range(n):
        ne = num_events[s % len(num_events)]
        out.append(Fuzzer(ne, FuzzerWeights(), ClientCommandGenerator(2), D.raft5_program()[:-1], seed=5000 + s).generateFuzzTest())
    return out


def oracle_violation(rd, model, flags, prog, n, seed, maxm, interval, c=None):
    full = rd.random_test_batch(model, D.pack_externals(prog), bits(range(len(prog)), len(prog)), n, seed, maxm, interval,
                                model_flags=flags, **_oracle_cfg(c or {}))[0]
    return int(full["violation"]) if int(full["status"]) == 0 else 0


def single(eng, prog, n, seed, maxm, looking, interval, check, mw, cap=1024):
    """demi_set_externals + demi_random_ddmin: (status, mcs, sizes, keys, out)"""
    eng.set_externals(prog)
    p = N.FuzzParams(seed, n, maxm, interval, looking, 0)
    mcs = np.zeros(mw, dtype=np.uint64)
    sizes = np.zeros(cap, dtype=np.uint32)
    keys = np.zeros(cap, dtype=np.uint64)
    out = N.RandomDDMinOut()
    rc = N.lib().demi_random_ddmin(eng._h, C.byref(p), 1 if check else 0, mcs.ctypes.data, mw, sizes.ctypes.data,
                                   keys.ctypes.data, cap, C.byref(out))
    k = min(out.n_iterations, cap)
    return rc, mcs, sizes[:k], keys[:k], out


def check_many(eng, progs, n, seeds, maxms, lookings, interval, check, single_eng=None, want_status=None):
    """demi_random_ddmin_many over progs equals the single sequence per trace; returns the many call's outputs"""
    mw = max(1, (max(len(p) for p in progs) + 63) // 64)
    mcs, sizes, keys, out, status = eng.random_ddmin_many(progs, n, seeds, maxms, lookings, interval, check, mask_words=mw)
    se = single_eng or eng
    for t, prog in enumerate(progs):
        rc, m1, s1, k1, o1 = single(se, prog, n, seeds[t], maxms[t], lookings[t], interval, check, mw)
        assert int(status[t]) == rc, (t, int(status[t]), rc, eng.last_error())
        if want_status is not None:
            assert rc == want_status[t]
        if rc:
            continue
        assert list(mcs[t]) == list(m1)
        ni = int(out[t]["n_iterations"])
        assert list(sizes[t, :ni]) == list(s1) and list(keys[t, :ni]) == list(k1)
        for f in OUT_FIELDS:
            assert int(out[t][f]) == int(getattr(o1, f)), (t, f)
        # executions_executed: this trace's own count, between what its tests needed and tests_evaluated x N
        assert int(out[t]["executions_executed"]) <= int(out[t]["tests_evaluated"]) * n
        assert int(out[t]["executions_executed"]) >= 1
    return mcs, sizes, keys, out, status


def oracle_check(rd, model, flags, progs, n, seeds, maxms, lookings, interval, check, mcs, out, status, c=None):
    for t, prog in enumerate(progs):
        if status[t]:
            continue
        want = rd.random_ddmin(model, D.pack_externals(prog), n, seeds[t], maxms[t], lookings[t], interval,
                               check_unmodified=check, model_flags=flags, **_oracle_cfg(c or {}))
        assert want["rc"] == 0
        assert list(mcs[t][:len(want["mcs"])]) == list(want["mcs"])
        assert int(out[t]["total_replays"]) == want["total_replays"] and int(out[t]["tests"]) == len(want["tests"])
        assert int(out[t]["verified"]) == want["verified"]


def raft5_set(rd, count, n, interval=5):
    progs, seeds, maxms, lookings = [], [], [], []
    for k, prog in enumerate(raft5_programs(4 * count)):
        if not atoms_cover(prog):
            continue
        seed, maxm = 100 + k, 40 + 5 * (k % 3)
        v = oracle_violation(rd, N.MODEL_RAFT5, RAFT_FLAGS, prog, 16, seed, maxm, interval)
        if not v:
            continue
        progs.append(prog); seeds.append(seed); maxms.append(maxm); lookings.append(v)
        if len(progs) == count:
            break
    assert len(progs) == count
    return progs, seeds, maxms, lookings


def test_batch_many_matches_the_oracle_per_trace(rd):
    """Mixed sets: raft5 campaign programs (lane engine) and pingpong3 with and without HardKill (the two groups)."""
    for model, flags, progs in ((N.MODEL_RAFT5, RAFT_FLAGS, raft5_programs(5) + [RAFT_WQ]),
                                (N.MODEL_PINGPONG3, PP_FLAGS, [PP_HK, D.pingpong3_program(n_sends=6), PP_HK[:-3] + [D.WaitQuiescence()]])):
        eng = D.Engine(D.SchedulerConfig(model, flags))
        rng = np.random.default_rng(3)
        seeds = [11 + 7 * t for t in range(len(progs))]
        maxms = [40 + 10 * (t % 3) for t in range(len(progs))]
        lookings = [0 if t % 2 else 1 for t in range(len(progs))]
        mw = max(1, (max(len(p) for p in progs) + 63) // 64)
        tr, masks = [], []
        for t, prog in enumerate(progs):
            m = random_masks(len(prog), 20, rng)
            m = np.hstack([m, np.zeros((len(m), mw - m.shape[1]), dtype=np.uint64)])
            tr += [t] * len(m)
            masks.append(m)
        order = rng.permutation(len(tr))                      # traces interleaved in the request
        tr, masks = np.array(tr, dtype=np.uint32)[order], np.vstack(masks)[order]
        for n, interval in ((64, 5), (1, 0)):
            got = eng.random_test_batch_many(progs, tr, masks, n, seeds, maxms, interval, lookings, mask_words=mw)
            for t, prog in enumerate(progs):
                sel = np.nonzero(tr == t)[0]
                pm = masks[sel][:, :max(1, (len(prog) + 63) // 64)]
                want = rd.random_test_batch(model, D.pack_externals(prog), pm, n, seeds[t], maxms[t], interval,
                                            looking_for=lookings[t], model_flags=flags)
                assert rows(got[sel]) == rows(want), (model, t)


@pytest.mark.parametrize("n,interval,check", [(1, 5, False), (64, 5, True), (64, 5, False), (1024, 5, True)])
def test_raft5_campaign_programs(rd, n, interval, check):
    progs, seeds, maxms, lookings = raft5_set(rd, 6 if n < 1024 else 3, n, interval)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, RAFT_FLAGS))
    mcs, _, _, out, status = check_many(eng, progs, n, seeds, maxms, lookings, interval, check)
    assert not status.any()
    if n <= 64:
        oracle_check(rd, N.MODEL_RAFT5, RAFT_FLAGS, progs, n, seeds, maxms, lookings, interval, check, mcs, out, status)


def test_pingpong3_hard_kill_and_lane_programs(rd):
    progs = [PP_HK, D.pingpong3_program(n_sends=6), PP_HK[:-3] + [D.WaitQuiescence()], D.pingpong3_program(n_sends=4)]
    seeds, maxms = [7, 8, 9, 10], [40, 40, 30, 40]
    lookings = [oracle_violation(rd, N.MODEL_PINGPONG3, PP_FLAGS, p, 16, s, m, 0) for p, s, m in zip(progs, seeds, maxms)]
    eng = D.Engine(D.SchedulerConfig(N.MODEL_PINGPONG3, PP_FLAGS))
    for check in (False, True):
        want = [0 if (lk or not check) else N.ERR_INVALID for lk in lookings]
        mcs, _, _, out, status = check_many(eng, progs, 16, seeds, maxms, lookings, 0, check, want_status=want)
        oracle_check(rd, N.MODEL_PINGPONG3, PP_FLAGS, progs, 16, seeds, maxms, lookings, 0, check, mcs, out, status)


@pytest.mark.parametrize("c", [dict(strategy=1), dict(rules=[(0b00110, 0b11111, 1 << 5, 0)]), dict(blocked=(4,))],
                         ids=["fifo", "filter", "blocked"])
def test_switches(rd, c):
    progs, seeds, maxms, lookings = [], [], [], []
    for k, prog in enumerate([RAFT_WQ] + raft5_programs(12)):
        if not atoms_cover(prog):
            continue
        rd.set_user_filter(c.get("rules", []))
        try:
            v = oracle_violation(rd, N.MODEL_RAFT5, RAFT_FLAGS, prog, 16, 30 + k, 60, 5, c)
        finally:
            rd.set_user_filter([])
        if v:
            progs.append(prog); seeds.append(30 + k); maxms.append(60); lookings.append(v)
        if len(progs) == 3:
            break
    assert len(progs) >= 2
    eng = engine(N.MODEL_RAFT5, RAFT_FLAGS, c)
    mcs, _, _, out, status = check_many(eng, progs, 16, seeds, maxms, lookings, 5, False)
    rd.set_user_filter(c.get("rules", []))
    try:
        oracle_check(rd, N.MODEL_RAFT5, RAFT_FLAGS, progs, 16, seeds, maxms, lookings, 5, False, mcs, out, status, c)
    finally:
        rd.set_user_filter([])


@pytest.mark.parametrize("timers", [False, True])
def test_loaded_models(rd, timers):
    from oracle import random_ddmin_binding
    done = 0
    for s in range(1, 200):
        m = ir_gen.generate(s)
        if m.uses_timers != timers:
            continue
        progs = [ir_gen.program(m, s), ir_gen.program(m, s + 1000, hard_kill=True)]
        progs = [p for p in progs if atoms_cover(p)]
        random_ddmin_binding.load_model(m.blob)
        seeds = [s + k for k in range(len(progs))]
        lookings = [oracle_violation(rd, N.MODEL_IR, m.flags, p, 16, sd, 40, 2) for p, sd in zip(progs, seeds)]
        if not any(lookings):
            continue
        eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, m.flags))
        eng.load_model(m.blob)
        mcs, _, _, out, status = check_many(eng, progs, 16, seeds, [40] * len(progs), lookings, 2, False)
        oracle_check(rd, N.MODEL_IR, m.flags, progs, 16, seeds, [40] * len(progs), lookings, 2, False, mcs, out, status)
        done += 1
        if done == 3:
            return
    raise AssertionError("not enough generated models")


def test_subsets_permutations_window_and_splits(rd, monkeypatch):
    progs, seeds, maxms, lookings = raft5_set(rd, 6, 64)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, RAFT_FLAGS))
    mw = max(1, (max(len(p) for p in progs) + 63) // 64)
    full = eng.random_ddmin_many(progs, 64, seeds, maxms, lookings, 5, mask_words=mw)

    def same(sel, got):
        for k, t in enumerate(sel):
            ni = int(full[3][t]["n_iterations"])
            assert list(got[0][k]) == list(full[0][t]) and list(got[1][k, :ni]) == list(full[1][t, :ni])
            assert list(got[2][k, :ni]) == list(full[2][t, :ni])
            for f in OUT_FIELDS:
                assert int(got[3][k][f]) == int(full[3][t][f])
    for sel in ([4, 1], [5, 3, 0, 2, 4, 1]):
        same(sel, eng.random_ddmin_many([progs[t] for t in sel], 64, [seeds[t] for t in sel], [maxms[t] for t in sel],
                                        [lookings[t] for t in sel], 5, mask_words=mw))
    monkeypatch.setenv("DEMI_DDMIN_MANY_WINDOW", "1")
    same(range(6), eng.random_ddmin_many(progs, 64, seeds, maxms, lookings, 5, mask_words=mw))
    monkeypatch.delenv("DEMI_DDMIN_MANY_WINDOW")
    # N = 2^15: 128 tests per launch and 32 per trace and batch, so the first round of six traces takes two launches
    big = 1 << 15
    got = eng.random_ddmin_many(progs, big, seeds, maxms, lookings, 5, mask_words=mw)
    assert eng.stats().kernel_launches > 4 * (int(got[3]["batches"].max()) + 1)     # four kernels per launch
    check_many(eng, progs, big, seeds, maxms, lookings, 5, False)


def capacity_failure(rd):
    """A loaded model whose randomDDMin consumes a test with a capacity status (the oracle's -4)"""
    from oracle import random_ddmin_binding
    for s in range(1, 80):
        m = ir_gen.generate(s)
        prog = ir_gen.program(m, s)
        if not atoms_cover(prog):
            continue
        random_ddmin_binding.load_model(m.blob)
        v = oracle_violation(rd, N.MODEL_IR, m.flags, prog, 16, s, 40, 2)
        want = rd.random_ddmin(N.MODEL_IR, D.pack_externals(prog), 16, s, 40, v, 2, model_flags=m.flags)
        if want["rc"] == -4:
            ok = [(p, s + 1000 + k) for k, p in enumerate([ir_gen.program(m, s + 500 + j) for j in range(20)])
                  if atoms_cover(p)]
            for p, sd in ok:
                v2 = oracle_violation(rd, N.MODEL_IR, m.flags, p, 16, sd, 40, 2)
                if v2 and rd.random_ddmin(N.MODEL_IR, D.pack_externals(p), 16, sd, 40, v2, 2, model_flags=m.flags)["rc"] == 0:
                    return m, (prog, s, v), (p, sd, v2)
    raise AssertionError("no loaded model with a consumed capacity status")


def test_failures_stay_with_their_trace(rd):
    progs, seeds, maxms, lookings = raft5_set(rd, 3, 16)
    bad = [D.Start(0), D.WaitQuiescence(), D.WaitQuiescence()]              # demi_set_externals rejects it
    quiet = D.raft5_program(client_cmds=1)[:3]                              # no violation: fails under check_unmodified
    ps = [progs[0], bad, progs[1], quiet, progs[2], []]
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, RAFT_FLAGS))
    mw = max(1, (max(len(p) for p in ps) + 63) // 64)
    mcs, sizes, keys, out, status = eng.random_ddmin_many(ps, 16, seeds[:1] + [1] + seeds[1:2] + [1] + seeds[2:] + [1],
                                                          maxms[:1] + [40] + maxms[1:2] + [40] + maxms[2:] + [40],
                                                          lookings[:1] + [1] + lookings[1:2] + [1] + lookings[2:] + [1], 5,
                                                          True, mask_words=mw)
    assert [int(x) for x in status] == [0, N.ERR_INVALID, 0, N.ERR_INVALID, 0, N.ERR_STATE]
    assert "trace 1" in eng.last_error()
    for k, t in enumerate([0, 2, 4]):
        rc, m1, s1, k1, o1 = single(eng, progs[k], 16, seeds[k], maxms[k], lookings[k], 5, True, mw)
        assert rc == 0 and list(mcs[t]) == list(m1) and int(out[t]["total_replays"]) == o1.total_replays
    # a consumed test's capacity status fails its trace alone, with the single call's code
    m, (p_bad, s_bad, v_bad), (p_ok, s_ok, v_ok) = capacity_failure(rd)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, m.flags))
    eng.load_model(m.blob)
    check_many(eng, [p_ok, p_bad, p_ok], 16, [s_ok, s_bad, s_ok], [40] * 3, [v_ok, v_bad, v_ok], 2, False,
               want_status=[0, N.ERR_CAPACITY, 0])


def test_handle_program_untouched_and_alloc_failure(rd, monkeypatch):
    progs, seeds, maxms, lookings = raft5_set(rd, 3, 16)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, RAFT_FLAGS))
    eng.set_externals(progs[0])
    before = eng.random_ddmin(16, seeds[0], maxms[0], lookings[0], 5)
    eng.random_ddmin_many(progs[1:], 16, seeds[1:], maxms[1:], lookings[1:], 5)
    after = eng.random_ddmin(16, seeds[0], maxms[0], lookings[0], 5)
    assert list(before[0]) == list(after[0]) and list(before[2]) == list(after[2])
    assert before[3].total_replays == after[3].total_replays
    monkeypatch.setenv("DEMI_TEST_ALLOC_LIMIT", "4096")
    with pytest.raises(D.DemiError) as ei:
        eng.random_ddmin_many(progs, 16, seeds, maxms, lookings, 5)
    assert ei.value.code == N.ERR_CUDA
    monkeypatch.delenv("DEMI_TEST_ALLOC_LIMIT")
    mcs, _, _, out, status = eng.random_ddmin_many(progs, 16, seeds, maxms, lookings, 5)
    assert not status.any() and list(mcs[0][:len(before[0])]) == list(before[0])


def test_rejected_arguments():
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, RAFT_FLAGS))
    prog = D.pack_externals(RAFT_WQ)
    z = np.zeros(1, dtype=np.uint32)
    n_ext = np.array([len(prog)], dtype=np.uint32)
    sb, mm, lf = np.zeros(1, dtype=np.int64), np.array([40], dtype=np.int32), np.zeros(1, dtype=np.uint32)
    out = np.zeros(1, dtype=N.RANDOM_DDMIN_OUT_DTYPE)
    st = np.zeros(1, dtype=np.int32)
    mcs = np.zeros(4, dtype=np.uint64)
    L = N.lib()
    p = N.FuzzParams(0, 0, 40, 5, 0, 0)
    assert L.demi_random_ddmin_many(eng._h, 1, prog.ctypes.data, z.ctypes.data, n_ext.ctypes.data, sb.ctypes.data,
                                    mm.ctypes.data, lf.ctypes.data, C.byref(p), 0, mcs.ctypes.data, 1, None, None, 0,
                                    out.ctypes.data, st.ctypes.data) == N.ERR_INVALID            # N = 0
    p = N.FuzzParams(0, 8, 40, 5, 0, 0)
    big = np.array([200], dtype=np.uint32)
    assert L.demi_random_ddmin_many(eng._h, 1, prog.ctypes.data, z.ctypes.data, big.ctypes.data, sb.ctypes.data,
                                    mm.ctypes.data, lf.ctypes.data, C.byref(p), 0, mcs.ctypes.data, 1, None, None, 0,
                                    out.ctypes.data, st.ctypes.data) == N.ERR_INVALID            # mask_words too small
    tr = np.array([1], dtype=np.uint32)
    rec = np.zeros(1, dtype=N.RANDOM_TEST_DTYPE)
    assert L.demi_random_test_batch_many(eng._h, 1, prog.ctypes.data, z.ctypes.data, n_ext.ctypes.data, sb.ctypes.data,
                                         mm.ctypes.data, lf.ctypes.data, tr.ctypes.data, mcs.ctypes.data, 1, 1, C.byref(p),
                                         rec.ctypes.data) == N.ERR_INVALID              # trace_of_test out of range
