"""Fuzzing campaigns on the device (demi_fuzz_campaign): record i equals demi_set_externals(program i) followed by
demi_fuzz_batch(seed_base + i, n = 1), and oracle_fuzz_campaign; the RunnerUtils.fuzz driver; demi_set_fuzzer's
rejections."""
import ctypes as C

import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
from demi_b200 import fuzzer as F
from oracle import campaign_binding as CB
import ir_gen

pytestmark = pytest.mark.gpu


def cfgs(num_events, send_type, kill=0.01, send=0.3, wait_quiescence=0.1, partition=0.1, unpartition=0.1):
    w = (kill, send, wait_quiescence, partition, unpartition, num_events, send_type)
    return N.FuzzerConfig(*w), CB.FuzzerConfig(*w)


def engine(model, model_flags=0, blocked_mask=0, strategy=0, blob=None):
    eng = D.Engine(D.SchedulerConfig(model, model_flags=model_flags, blocked_mask=blocked_mask, strategy=strategy))
    if blob is not None:
        eng.load_model(blob)
    return eng


def check_campaign(model, prefix, postfix, cfg_pair, n, max_messages, interval, model_flags=0, blocked_mask=0, strategy=0,
                   blob=None, rules=None, n_fixed=24, seed_base=1000, program_seed_base=55):
    """The campaign against oracle_fuzz_campaign on all n records and the fixed-program path on a sample."""
    cfg, ocfg = cfg_pair
    pre, post = D.pack_externals(prefix), D.pack_externals(postfix)
    eng = engine(model, model_flags, blocked_mask, strategy, blob)
    if rules:
        eng.set_user_filter(rules)
    eng.set_fuzzer(cfg, pre, post)
    got = eng.fuzz_campaign(seed_base, n, max_messages, interval, program_seed_base)
    if blob is not None:
        CB.load_model(blob)
    if rules:
        CB.set_user_filter(rules)
    try:
        want = CB.fuzz_campaign(model, ocfg, pre, post, seed_base, n, max_messages, interval, program_seed_base,
                                model_flags=model_flags, blocked_mask=blocked_mask, strategy=strategy)
    finally:
        if rules:
            CB.set_user_filter([])
    assert got.tobytes() == want.tobytes(), np.nonzero(got != want)[0][:5]
    fixed = engine(model, model_flags, blocked_mask, strategy, blob)
    if rules:
        fixed.set_user_filter(rules)
    for i in np.linspace(0, n - 1, n_fixed).astype(int):
        fixed.set_externals(eng.fuzzer_program(program_seed_base + int(i)))
        one = fixed.fuzz_batch(seed_base + int(i), 1, max_messages, interval)
        assert one.tobytes() == got[i:i + 1].tobytes(), int(i)
    return eng, got


@pytest.mark.parametrize("flags", [0, 1, 2])
def test_raft5(flags):
    _, got = check_campaign(N.MODEL_RAFT5, D.raft5_program(), [], cfgs(40, 2), 6000, 50, 5, model_flags=flags)
    assert (got["status"] == 0).all()
    if flags == 1:                                                   # the double-vote bug shows up within 6000 executions
        assert (got["violation"] != 0).any()


def test_raft5_chunks_and_halves():
    """n not a multiple of the chunk size; two half campaigns equal one whole one."""
    cfg, _ = cfgs(10, 2)
    eng = engine(N.MODEL_RAFT5, 1)
    eng.set_fuzzer(cfg, D.pack_externals(D.raft5_program()))
    n = (2 << 20) + 12345
    whole = eng.fuzz_campaign(7, n, 50, 5, 9)
    a = eng.fuzz_campaign(7, n // 2, 50, 5, 9)
    b = eng.fuzz_campaign(7 + n // 2, n - n // 2, 50, 5, 9 + n // 2)
    assert np.concatenate([a, b]).tobytes() == whole.tobytes()
    fixed = engine(N.MODEL_RAFT5, 1)
    for i in (0, n // 2 - 1, n // 2, (2 << 20) - 1, 2 << 20, n - 1):
        fixed.set_externals(eng.fuzzer_program(9 + i))
        assert fixed.fuzz_batch(7 + i, 1, 50, 5).tobytes() == whole[i:i + 1].tobytes(), i


def test_dev_path_and_summary():
    import torch
    cfg, _ = cfgs(40, 2)
    eng = engine(N.MODEL_RAFT5, 1)
    eng.set_fuzzer(cfg, D.pack_externals(D.raft5_program()))
    n = 20000
    host = eng.fuzz_campaign(3, n, 50, 5, 4)
    buf = torch.empty(n * 32, dtype=torch.uint8, device="cuda")
    eng.fuzz_campaign_dev(3, n, 50, 5, 4, buf.data_ptr())
    nv, steps = eng.fuzz_summary_dev()
    dev = buf.cpu().numpy().view(N.RESULT_DTYPE)
    assert dev.tobytes() == host.tobytes()
    assert nv == int((host["violation"] != 0).sum()) and steps == int(host["steps"].sum())
    assert eng.stats().prefixes == n and eng.stats().kernel_launches >= 2


def test_pingpong3_and_bcast32():
    check_campaign(N.MODEL_PINGPONG3, D.pingpong3_program(20), [D.Send(1, 1, 500)], cfgs(40, 1, partition=0.3), 4000, 60, 3)
    check_campaign(N.MODEL_BCAST32, D.bcast32_program(2), [], cfgs(30, 2, send=0.2, partition=0.3), 2000, 200, 0)


@pytest.mark.parametrize("model,prefix,send_type", [
    (N.MODEL_PINGPONG3, D.pingpong3_program(20), 1),       # fixed Sends p0 = 0..19, generated p0 = 1..40: made distinct below
    (N.MODEL_BCAST32, D.bcast32_program(2), 2),
])
def test_lane_prog_kernels_pingpong3_bcast32(monkeypatch, model, prefix, send_type):
    """Fixed Sends that no generated (send_type, 1..num_events, 0) Send can equal: the campaign runs on the lane engine."""
    prefix = [D.Send(e.a, e.type, 1000 + e.p0) if isinstance(e, D.Send) else e for e in prefix]
    monkeypatch.setenv("DEMI_LANE_PENDING_CAP", "8")                  # the lane engine ran iff it deferred something
    eng, _ = check_campaign(model, prefix, [], cfgs(30, send_type, partition=0.2), 2000, 60, 3)
    assert eng.stats().deferred > 0
    monkeypatch.delenv("DEMI_LANE_PENDING_CAP")
    monkeypatch.setenv("DEMI_DISABLE_LANE_ENGINE", "1")
    eng, _ = check_campaign(model, prefix, [], cfgs(30, send_type, partition=0.2), 2000, 60, 3)
    assert eng.stats().deferred == 0


def test_per_program_caps_mix_overflow():
    """bcast32 unbounded: programs with 88-89 Sends get pending_cap 128, with 90-91 Sends 256; some records overflow."""
    prefix = [D.Start(a) for a in range(32)] + [D.Send(a % 32, 1, 0) for a in range(88)] + [D.WaitQuiescence()]
    _, got = check_campaign(N.MODEL_BCAST32, prefix, [], cfgs(2, 2, kill=0.0, send=0.6, wait_quiescence=0.4, partition=0.0,
                                                                  unpartition=0.0), 600, -1, 0)
    assert (got["status"] == 0).any() and (got["status"] == 1).any()          # DEMI_PS_PENDING_OVF


def test_src_dst_fifo_blocked_filter_hard_kill():
    check_campaign(N.MODEL_RAFT5, D.raft5_program(), [], cfgs(30, 2), 3000, 50, 5, model_flags=1, strategy=1)
    check_campaign(N.MODEL_RAFT5, D.raft5_program(), [], cfgs(30, 2), 3000, 50, 5, model_flags=1, blocked_mask=0b100)
    check_campaign(N.MODEL_RAFT5, D.raft5_program(), [], cfgs(30, 2), 3000, 50, 5, model_flags=1, rules=[(0b1, 0b10, 0xFFFFFFFF, 0)])
    hk = D.raft5_program()[:-1] + [D.WaitQuiescence(), D.HardKill(2), D.Start(2), D.Send(2, 1, 0x1F)]
    check_campaign(N.MODEL_RAFT5, hk, [], cfgs(30, 2), 3000, 50, 5, model_flags=1)


def test_lane_engine_disabled_and_deferring(monkeypatch):
    monkeypatch.setenv("DEMI_DISABLE_LANE_ENGINE", "1")
    check_campaign(N.MODEL_RAFT5, D.raft5_program(), [], cfgs(40, 2), 3000, 50, 5, model_flags=1)
    monkeypatch.delenv("DEMI_DISABLE_LANE_ENGINE")
    monkeypatch.setenv("DEMI_LANE_PENDING_CAP", "12")
    eng, _ = check_campaign(N.MODEL_RAFT5, D.raft5_program(), [], cfgs(40, 2), 3000, 50, 5, model_flags=1)
    assert eng.stats().deferred > 0


@pytest.mark.parametrize("timers", [False, True])
def test_generated_loaded_models(timers):
    done = 0
    for s in range(400):
        m = ir_gen.generate(s)
        if m.uses_timers != timers:
            continue
        prefix = [e for e in ir_gen.program(m, s, kills=False)]
        cfg = cfgs(20, m.ext_types[0], partition=0.2)
        check_campaign(N.MODEL_IR, prefix, [], cfg, 300, 40, 3, model_flags=m.flags, blob=m.blob, n_fixed=6)
        done += 1
        if done == 6:
            break
    assert done == 6


def test_set_fuzzer_rejections():
    eng = engine(N.MODEL_RAFT5)
    ok = D.pack_externals(D.raft5_program())
    cfg, _ = cfgs(10, 2)
    L = N.lib()

    def rc(c, pre, post=None):
        pre = D.pack_externals(pre) if isinstance(pre, list) else pre
        post = D.pack_externals(post or [])
        return L.demi_set_fuzzer(eng._h, C.byref(c), pre.ctypes.data if len(pre) else None, len(pre),
                                 post.ctypes.data if len(post) else None, len(post))

    p = N.FuzzParams(0, 4, 50, 5, 0, 0)
    out = np.zeros(4, dtype=N.RESULT_DTYPE)
    assert L.demi_fuzz_campaign(eng._h, C.byref(p), 0, out.ctypes.data) == N.ERR_STATE          # no Fuzzer yet
    assert rc(cfg, ok) == N.OK
    bad_kind = ok.copy(); bad_kind[3]["kind"] = 9
    assert rc(cfg, bad_kind) == N.ERR_INVALID
    assert rc(cfg, [D.Start(0), D.Send(7, 2, 1)]) == N.ERR_INVALID                                # unknown actor
    assert rc(cfg, [D.Start(0)], [D.Partition(0, 9)]) == N.ERR_INVALID
    assert rc(cfg, [D.Send(0, 1, 1), D.WaitQuiescence()]) == N.ERR_INVALID                        # no Start
    assert rc(cfg, [D.Start(0), D.WaitQuiescence(), D.WaitQuiescence()]) == N.ERR_INVALID
    assert rc(cfg, [D.Start(0)], [D.Send(0, 2, 1), D.WaitQuiescence(), D.WaitQuiescence()]) == N.ERR_INVALID
    assert rc(cfg, [D.Start(0)], [D.WaitQuiescence(), D.Send(0, 2, 1)]) == N.ERR_INVALID        # postfix begins with WQ
    assert rc(cfgs(10, 9)[0], ok) == N.ERR_INVALID                                                 # raft5 types are 1..8
    for w in (dict(kill=-0.1), dict(send=float("inf")), dict(partition=float("nan")),
              dict(kill=0.0, send=0.0, wait_quiescence=0.0, partition=0.0, unpartition=0.0)):
        assert rc(cfgs(10, 2, **w)[0], ok) == N.ERR_INVALID, w
    assert rc(cfgs(N.FUZZER_MAX_EVENTS + 1, 2)[0], ok) == N.ERR_INVALID
    assert rc(cfgs(N.FUZZER_MAX_EVENTS, 2)[0], ok) == N.OK
    b = engine(N.MODEL_BCAST32)
    c33 = D.pack_externals([D.Start(a % 32) for a in range(33)])
    assert L.demi_set_fuzzer(b._h, C.byref(cfg), c33.ctypes.data, 33, None, 0) == N.ERR_INVALID     # > 32 Starts
    # demi_set_fuzzer leaves the handle's externals alone
    eng.set_externals(D.raft5_program())
    before = eng.fuzz_batch(5, 100, 50, 5)
    assert rc(cfg, ok) == N.OK
    assert eng.fuzz_batch(5, 100, 50, 5).tobytes() == before.tobytes()


# ---- the driver (RunnerUtils.fuzz)
def raft_fuzzer(num_events=40):
    return F.Fuzzer(num_events, F.FuzzerWeights(), F.ClientCommandGenerator(2), D.raft5_program())


def host_loop(fz, flags, budget, accept, mm=50, interval=5, pbase=D.PROGRAM_SEED_OFFSET):
    """The same search from existing calls: demi_fuzzer_generate, demi_set_externals, demi_fuzz_batch one at a time."""
    eng = engine(N.MODEL_RAFT5, flags)
    cfg = F.fuzzer_config(fz)
    pre = D.pack_externals(fz.prefix)
    for k in range(budget):
        eng.set_externals(N.fuzzer_generate(cfg, pbase + k, pre))
        r = eng.fuzz_batch(k, 1, mm, interval)[0]
        if r["status"] == 0 and r["violation"] and accept(int(r["violation"])):
            return k, int(r["violation"])
    return None


def test_driver_matches_host_loop_and_oracle_trace(oracle):
    sc = D.SchedulerConfig(N.MODEL_RAFT5, model_flags=3)
    for budget in (5, 40, 300):
        want = host_loop(raft_fuzzer(), 3, budget, lambda v: True, pbase=0)
        got = D.fuzz(raft_fuzzer(), sc, maxMessages=50, invariant_check_interval=5, max_executions=budget, chunk=17,
                 program_seed_base=0)
        if want is None:
            assert got is None
            continue
        assert (got.execution, got.violation) == want
        ev, par, r = oracle.fuzz_trace(N.MODEL_RAFT5, got.externals, got.execution, 50, 5, model_flags=3)
        assert np.array_equal(ev, got.trace) and np.array_equal(par, got.dep_graph) and int(r["violation"]) == got.violation


def test_driver_predicate_budget_provenance_and_replay():
    sc = D.SchedulerConfig(N.MODEL_RAFT5, model_flags=3)
    first = D.fuzz(raft_fuzzer(), sc, maxMessages=50, invariant_check_interval=5, max_executions=2000)
    assert first is not None
    assert (first.execution, first.violation) == host_loop(raft_fuzzer(), 3, 2000, lambda v: True)   # default program seeds
    other = D.fuzz(raft_fuzzer(), sc, maxMessages=50, invariant_check_interval=5, max_executions=5000,
                   violationWereLookingFor=lambda v: v != first.violation)
    want = host_loop(raft_fuzzer(), 3, 5000, lambda v: v != first.violation)
    if want is None:
        assert other is None
    else:
        assert (other.execution, other.violation) == want and other.violation != first.violation
    assert D.fuzz(raft_fuzzer(), sc, maxMessages=50, invariant_check_interval=5, max_executions=first.execution) is None
    prov = D.fuzz(raft_fuzzer(), sc, maxMessages=50, invariant_check_interval=5, max_executions=2000, computeProvenance=True,
                  validate_replay=True)
    assert prov.execution == first.execution
    eng = engine(N.MODEL_RAFT5, 3)
    eng.set_externals(prov.externals)
    _, out, _ = eng.fuzz_provenance(prov.execution, [0], 50, 5)
    keep, o = eng.provenance(prov.trace, prov.dep_graph, int(out[0]["affected_mask"]))
    idx = np.nonzero(prov.trace["kind"] == N.EV_MSG_EVENT)[0]
    bits = np.unpackbits(keep.view(np.uint8), bitorder="little")[1:len(idx) + 1].astype(bool)
    assert np.array_equal(prov.filtered, prov.trace[idx[bits]])
    assert prov.initialTrace[0] == 0 and len(prov.initialTrace) == len(idx) + 1
