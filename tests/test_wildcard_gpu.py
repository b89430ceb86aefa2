"""Fungible clocks on the device: the WILD instantiation of the K2 replay kernel and demi_wildcard_minimize, bit-exact
against the sequential C oracle (oracle/sts_wildcard.c, oracle/wildcard.c) — per-test results, recorded traces
and ignored positions, and the whole minimizer — on raft5 (several seeds and the configs[3] trace), pingpong3 (no
clocks: only the first cluster) and timer-free loaded models; plus the inputs that are rejected before any launch."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
from oracle import wildcard_binding as W
import ir_gen
from test_wildcard_kat import pingpong_case
from test_wildcard_oracle import raft_cases, raft_rules, recorded

pytestmark = pytest.mark.gpu
FIELDS = ("kind", "src", "dst", "type", "p0", "p1", "uniq", "node")
RFIELDS = ("violation", "status", "delivered", "ignored", "state_hash")


def rows(a):
    return [tuple(int(e[f]) for f in FIELDS) for e in a]


def rres(r):
    return tuple(int(r[f]) for f in RFIELDS)


def deliveries(a):
    return int((a["kind"] == N.EV_MSG_EVENT).sum())


def random_masks(rng, n_deliv, n):
    mw = max(1, (n_deliv + 63) // 64)
    masks = np.zeros((n, mw), dtype=np.uint64)
    for k in range(n):
        keep = rng.random(n_deliv) < (1.0 if k == 0 else rng.choice([0.95, 0.8, 0.5]))
        for j in np.nonzero(keep)[0]:
            masks[k, j >> 6] |= np.uint64(1) << np.uint64(j & 63)
    return masks


def compare_replays(oracle, eng, model, case, rules, incr, model_flags, rng, n_masks=24, n_rec=3):
    vtrace, _, mcs_ext, code = case
    eng.set_trace(vtrace, mcs_ext)
    eng.set_clock_rules(rules, incr)
    masks = random_masks(rng, deliveries(vtrace), n_masks)
    seen = 0
    for flags in (0, N.WC_LAST_ONLY, N.RF_FILTER_KNOWN_ABSENTS, N.WC_LAST_ONLY | N.RF_FILTER_KNOWN_ABSENTS):
        got = eng.wildcard_replay_batch(masks, looking_for=code, flags=flags)
        for k in range(n_masks):
            r, rec, ign = W.wildcard_replay(model, vtrace, mcs_ext, masks[k], incr, looking_for=code, flags=flags,
                                                model_flags=model_flags)
            assert rres(got[k]) == rres(r), (k, flags)
            if k < n_rec:
                g, grec, gign = eng.wildcard_replay_trace(masks[k], looking_for=code, flags=flags)
                assert rres(g) == rres(r) and rows(grec) == rows(rec) and list(gign) == list(ign), (k, flags)
            seen += int(r["violation"]) != 0
    return seen


def compare_minimize(oracle, eng, model, case, rules, incr, model_flags, flags):
    vtrace, _, mcs_ext, code = case
    eng.set_trace(vtrace, mcs_ext)
    eng.set_clock_rules(rules, incr)
    trace, sizes, out = eng.wildcard_minimize(code, flags=flags)
    rc, ctrace, total, csizes = W.wildcard_minimize(model, vtrace, mcs_ext, rules, incr, code, flags=flags,
                                                         model_flags=model_flags)
    assert rc == 0
    assert rows(trace) == rows(ctrace)
    assert out.total_replays == total and [int(x) for x in sizes] == [int(x) for x in csizes]
    assert out.deliveries_before == deliveries(vtrace) and out.deliveries_after == deliveries(ctrace)
    assert out.n_events == len(ctrace) and out.unignorable == 0 and out.replays_executed >= total
    # the handle now holds minTrace; replayed in full it still shows the violation
    r, _ = eng.replay_trace(None, looking_for=code, flags=flags & N.RF_FILTER_KNOWN_ABSENTS)
    assert int(r["violation"]) == code
    return out


def test_rejected_before_any_launch():
    eng = D.Engine(D.SchedulerConfig(N.MODEL_PINGPONG3))
    prog, ext, ev = pingpong_case()
    eng.set_trace(ev, ext)
    for bad in ([N.clock_rule(4, 0, 0, 8), N.clock_rule(4, 1, 0, 8)],      # two rules for one type
                [N.clock_rule(4, 0, 0, 0)], [N.clock_rule(4, 0, 0, 33)],    # bits outside 1..32
                [N.clock_rule(4, 2, 0, 8)], [N.clock_rule(4, 0, 32, 8)]):   # word 2, shift 32
        with pytest.raises(D.DemiError) as e:
            eng.set_clock_rules(bad, ())
        assert e.value.code == N.ERR_INVALID
    eng.set_clock_rules([N.clock_rule(2, 0, 0, 32)], (3,))                  # accepted
    full = np.array([0xF], dtype=np.uint64)
    for flags in (N.RF_STRICT, N.RF_STRICT | N.WC_LAST_ONLY, N.IM_SRC_DST_FIFO):
        with pytest.raises(D.DemiError) as e:
            eng.wildcard_replay_batch(full, flags=flags)
        assert e.value.code == N.ERR_INVALID
        with pytest.raises(D.DemiError) as e:
            eng.wildcard_minimize(0, flags=flags)
        assert e.value.code == N.ERR_INVALID
    dup = ev.copy()
    dup[12]["uniq"] = 1                                                    # two deliveries with Uniq id 1
    eng.set_trace(dup, ext)
    for call in (lambda: eng.wildcard_replay_batch(full), lambda: eng.wildcard_replay_trace(full),
                 lambda: eng.wildcard_minimize(0)):
        with pytest.raises(D.DemiError) as e:
            call()
        assert e.value.code == N.ERR_INVALID


def test_pingpong_known_answers_on_the_device(oracle):
    """The hand-derived cases of test_wildcard_kat.py, on the engine: First, Last, the clock selector, a blocked
    receiver, a cleared bit."""
    prog, ext, ev = pingpong_case()
    full = np.array([0xF], dtype=np.uint64)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_PINGPONG3))
    eng.set_trace(ev, ext)
    last = lambda rec: [(int(e["type"]), int(e["p0"]), int(e["uniq"])) for e in rec if int(e["kind"]) == 2][-1]
    assert last(eng.wildcard_replay_trace(full)[1]) == (2, 5, 4)
    assert last(eng.wildcard_replay_trace(full, flags=N.WC_LAST_ONLY)[1]) == (2, 6, 5)
    eng.set_clock_rules([], (2,))
    assert last(eng.wildcard_replay_trace(full, flags=N.WC_LAST_ONLY)[1]) == (2, 5, 4)
    r, _, ign = eng.wildcard_replay_trace(np.array([0], dtype=np.uint64))
    assert int(r["delivered"]) == 3 and len(ign) == 0
    blk = D.Engine(D.SchedulerConfig(N.MODEL_PINGPONG3, blocked_mask=1 << 1))
    blk.set_trace(ev, ext)
    r, _, ign = blk.wildcard_replay_trace(full)
    assert int(r["ignored"]) == 1 and list(ign) == [12]
    ro, _, oign = W.wildcard_replay(N.MODEL_PINGPONG3, ev, ext, full, (), blocked_mask=1 << 1)
    assert rres(r) == rres(ro) and list(oign) == [12]


def test_raft5_replays_and_minimizer_match_the_oracle(oracle):
    cases = raft_cases(oracle, 8)
    rules, incr = raft_rules()
    rng = np.random.default_rng(3)
    engines = {f: D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=f)) for f in (1, 3)}
    viol = removed = multi_batch = 0
    for k, (flags, *case) in enumerate(cases):
        eng = engines[flags]
        viol += compare_replays(oracle, eng, N.MODEL_RAFT5, case, rules, incr, flags, rng)
        for wflags in (0, N.WC_LAST_ONLY, N.RF_FILTER_KNOWN_ABSENTS if k % 2 else N.WC_LAST_ONLY | N.RF_FILTER_KNOWN_ABSENTS):
            out = compare_minimize(oracle, eng, N.MODEL_RAFT5, case, rules, incr, flags, wflags)
            removed += out.deliveries_after < out.deliveries_before
            multi_batch += out.batches > 1
    assert viol > 50 and removed > 2 and multi_batch > 0


def test_the_wildcard_minimizer_class(oracle):
    """WildcardMinimizer with the reference's stats calls: one strategy record, the size series of the engine."""
    flags, vtrace, mcs_prog, mcs_ext, code = raft_cases(oracle, 2)[0]
    cfg = D.SchedulerConfig(N.MODEL_RAFT5, model_flags=flags)
    wm = D.WildcardMinimizer(cfg, mcs_prog, vtrace, code, resolutionStrategy=D.LastOnlyStrategy(),
                             clock_rules=D.raft5_clock_rules())
    stats, trace = wm.minimize()
    rules, incr = raft_rules()
    rc, ctrace, total, csizes = W.wildcard_minimize(N.MODEL_RAFT5, vtrace, mcs_ext, rules, incr, code,
                                                         flags=N.WC_LAST_ONLY, model_flags=flags)
    assert rows(trace) == rows(ctrace) and stats.total_replays == total and stats.internal_sizes == [int(x) for x in csizes]
    assert stats.stats[-1].name == "(FungibleClockMinimizer,STSSched)"
    for bad in (dict(testScheduler=D.TestScheduler.DPORwHeuristics), dict(skipClockClusters=True),
                dict(clusteringStrategy=D.ClusteringStrategy.SingletonClusterizer)):
        with pytest.raises(NotImplementedError):
            D.WildcardMinimizer(cfg, mcs_prog, vtrace, code, engine=wm.engine, **bad)


def _c3_case(oracle):
    from tools import secondary as S
    prog = D.raft5_program(client_cmds=S.C3_PROGRAM_CMDS)
    return prog, recorded(oracle, N.MODEL_RAFT5, prog, S.C3_SEED_DEFAULT, S.C3_MAX_MESSAGES, S.C3_INTERVAL, 1)


def test_configs3_trace(oracle):
    """The 2039-event configs[3] trace: per-test results on random masks, the full minimizer, and the chain
    DDMin -> internal minimization (SrcDstFIFO) -> wildcard minimization, which is runTheGamut's order."""
    prog, case = _c3_case(oracle)
    assert case is not None and len(case[0]) >= 2000
    rules, incr = raft_rules()
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    compare_replays(oracle, eng, N.MODEL_RAFT5, case, rules, incr, 1, np.random.default_rng(7), n_masks=64, n_rec=2)
    compare_minimize(oracle, eng, N.MODEL_RAFT5, case, rules, incr, 1, 0)
    # the chain
    vtrace, mcs_prog, mcs_ext, code = case
    eng.set_trace(vtrace, mcs_ext)
    mcs, _, _ = eng.ddmin(code)
    keep = [k for k in range(len(mcs_prog)) if (int(mcs[k >> 6]) >> (k & 63)) & 1]
    mext = D.pack_externals([mcs_prog[k] for k in keep])
    r, mtrace = eng.replay_trace(mcs, looking_for=code)
    assert int(r["violation"]) == code
    eng.set_trace(mtrace, mext)
    itrace, _, _ = eng.internal_minimize(code, flags=N.IM_SRC_DST_FIFO)
    out = compare_minimize(oracle, eng, N.MODEL_RAFT5, (itrace, None, mext, code), rules, incr, 1, 0)
    assert out.deliveries_after <= out.deliveries_before


def test_pingpong3_has_only_the_first_cluster(oracle):
    flags = 1 | (3 << 8)
    prog = [D.Start(a) for a in range(3)] + [D.Send(k % 3, 1, k) for k in range(18)] + [D.WaitQuiescence()]
    ext = D.pack_externals(prog)
    res = oracle.fuzz_batch(N.MODEL_PINGPONG3, ext, 1, 40, -1, 0, model_flags=flags)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_PINGPONG3, model_flags=flags))
    done = 0
    for i in np.nonzero(res["violation"])[0][:3]:
        case = recorded(oracle, N.MODEL_PINGPONG3, prog, 1 + int(i), -1, 0, flags)
        if case is None:
            continue
        compare_replays(oracle, eng, N.MODEL_PINGPONG3, case, [], (), flags, np.random.default_rng(1), n_masks=8)
        out = compare_minimize(oracle, eng, N.MODEL_PINGPONG3, case, [], (), flags, 0)
        assert out.total_replays == 1 and out.batches == 1      # no clocks, no timers: the first cluster only
        done += 1
    assert done >= 1


def test_timer_free_loaded_models(oracle):
    rng = np.random.default_rng(9)
    n_models = n_cases = 0
    seed = 0
    while n_models < 40 and seed < 2000:
        seed += 1
        m = ir_gen.generate(seed)
        if m.uses_timers:
            continue
        n_models += 1
        oracle.load_model(m.blob)
        W.load_model(m.blob)                                         # the wildcard oracle is a library of its own
        prog = ir_gen.program(m, seed)
        ext = D.pack_externals(prog)
        maxm = [40, 60][seed % 2]
        res = oracle.fuzz_batch(N.MODEL_IR, ext, 1, 60, maxm, seed % 4, model_flags=m.flags)
        eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, model_flags=m.flags))
        eng.load_model(m.blob)
        types = list(range(min(m.n_types, 256)))
        rules = [N.clock_rule(int(t), int(rng.integers(0, 2)), int(rng.integers(0, 8)), int(rng.choice([1, 2, 8, 32])))
                 for t in rng.choice(types, size=min(len(types), 3), replace=False)]
        incr = [int(t) for t in rng.choice(types, size=min(len(types), 1), replace=False)]
        for i in np.nonzero(res["violation"] * (res["status"] == 0))[0][:2]:
            case = recorded(oracle, N.MODEL_IR, prog, 1 + int(i), maxm, seed % 4, m.flags)
            if case is None:
                continue
            compare_replays(oracle, eng, N.MODEL_IR, case, rules, incr, m.flags, rng, n_masks=8, n_rec=2)
            compare_minimize(oracle, eng, N.MODEL_IR, case, rules, incr, m.flags, seed % 2 and N.WC_LAST_ONLY)
            n_cases += 1
    assert n_cases >= 15
