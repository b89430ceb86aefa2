"""Fungible clocks on the CPU: the C oracle (oracle/sts_wildcard.c, oracle/wildcard.c) against the Python
restatement of WildcardMinimizer / ClockClusterizer / WildCardMatch (tests/micro_oracle_wildcard.py), which works on message
objects through real closures, as the Scala does, and never sees the packed clock rules or the per-delivery mode table.
Per-test results, recorded traces and ignored positions on random include masks; the whole minimizer; the chain
DDMin -> internal minimization -> wildcard minimization."""
import numpy as np

import demi_b200 as D
from demi_b200 import _native as N
from oracle import wildcard_binding as W
import ir_gen
import micro_oracle as M
import micro_oracle_wildcard as MW
from test_micro_oracle import flat, to_prog, unflat

FIELDS7 = ("kind", "src", "dst", "type", "p0", "p1", "uniq")
RAFT_TERM_TYPES, RAFT_TICK = (4, 5, 7, 8), 3


def raft_fingerprinter():
    """raft5's FingerprintFactory written as closures over a message (type, p0, p1)."""
    return MW.FingerprintFactory(getLogicalClock=lambda m: (m[1] & 0xFF) if m[0] in RAFT_TERM_TYPES else None,
                                causesClockIncrement=lambda m: m[0] == RAFT_TICK)


def raft_rules():
    rules, incr = D.raft5_clock_rules()
    return list(rules), list(incr)


def closures_of(rule_spec, incr_types):
    """Random rules as (type -> (word, shift, bits)) turned into closures, independently of the packing."""
    def clock(m):
        if m[0] not in rule_spec:
            return None
        word, shift, bits = rule_spec[m[0]]
        return (m[1 + word] >> shift) & ((1 << bits) - 1)
    inc = set(incr_types)
    return MW.FingerprintFactory(getLogicalClock=clock, causesClockIncrement=lambda m: m[0] in inc)


def recorded(oracle, model, prog, seed, maxm, interval, model_flags):
    """A violating execution replayed once by STSSched over its own externals (minus WaitQuiescence): the verified
    trace the minimizers start from, and the MCS it replays."""
    ext = D.pack_externals(prog)
    ev, _, r = oracle.fuzz_trace(model, ext, seed, maxm, interval, model_flags=model_flags)
    code = int(r["violation"])
    if not code or int(r["status"]):
        return None
    full = np.asarray(oracle.full_mask(ext), dtype=np.uint64).reshape(-1)
    rr, vtrace = oracle.replay_trace(model, ev, ext, full, looking_for=code, model_flags=model_flags)
    if int(rr["status"]) or int(rr["violation"]) != code:
        return None
    mcs_prog = [prog[k] for k in range(len(ext)) if (int(full[k >> 6]) >> (k & 63)) & 1]
    return vtrace, mcs_prog, D.pack_externals(mcs_prog), code


def raft_cases(oracle, n):
    """n violating raft5 traces: half with the double-vote bug alone (model_flags 1), half with both bugs (3)."""
    prog = D.raft5_program(client_cmds=2)
    ext = D.pack_externals(prog)
    per_flag = {}
    for flags in (1, 3):
        res = oracle.fuzz_batch(N.MODEL_RAFT5, ext, 1, 4000, 40, 5, model_flags=flags)
        per_flag[flags] = []
        for i in np.nonzero(res["violation"])[0]:
            c = recorded(oracle, N.MODEL_RAFT5, prog, 1 + int(i), 40, 5, flags)
            if c is not None:
                per_flag[flags].append((flags,) + c)
            if len(per_flag[flags]) >= n:
                break
    take3 = min(len(per_flag[3]), n // 2)
    return per_flag[3][:take3] + per_flag[1][:n - take3]


def include_ids(vtrace, mask):
    ids, j = set(), 0
    for e in vtrace:
        if int(e["kind"]) == N.EV_MSG_EVENT:
            if (int(mask[j >> 6]) >> (j & 63)) & 1:
                ids.add(int(e["uniq"]))
            j += 1
    return ids


def python_replay(actors, invariant, is_ext, fp, strategy, vtrace, mcs_events, mask, fka, code):
    """ClockClusterizer's trace for the included ids, replayed by the Python STSScheduler."""
    base = unflat(vtrace)
    inc = include_ids(vtrace, mask)
    timers = set(e[4] for e in base if e[0] == "MsgEvent" and fp.causesClockIncrement(e[3])) & inc
    cz = MW.ClockClusterizer(base, fp, strategy, is_ext)
    nxt = cz.wildcarded(timers, inc - timers)
    sts = MW.WildcardSTSReplay(actors, nxt, mcs_events, invariant, is_ext, filter_known_absents=bool(fka), looking_for=code)
    sts.violation = sts.test(list(range(len(mcs_events))))
    return sts


def check_replays(oracle, model, make_actors, invariant, is_ext, fp, incr, case, rng, n_masks, model_flags, stats):
    vtrace, mcs_prog, mcs_ext, code = case
    mcs_events = to_prog(mcs_prog)
    n_deliv = int((vtrace["kind"] == N.EV_MSG_EVENT).sum())
    mw = max(1, (n_deliv + 63) // 64)
    for t in range(n_masks):
        keep = rng.random(n_deliv) < (1.0 if t == 0 else rng.choice([0.9, 0.7, 0.4]))
        mask = np.zeros(mw, dtype=np.uint64)
        for j in np.nonzero(keep)[0]:
            mask[j >> 6] |= np.uint64(1) << np.uint64(j & 63)
        picks = {}
        for last in (0, 1):
            for fka in (0, 1):
                flags = (N.WC_LAST_ONLY if last else 0) | fka
                res, rec, ign = W.wildcard_replay(model, vtrace, mcs_ext, mask, incr, looking_for=code, flags=flags,
                                                      model_flags=model_flags)
                strategy = MW.LastOnlyStrategy() if last else MW.BackTrackStrategy()
                try:
                    sts = python_replay(make_actors(), invariant, is_ext, fp, strategy, vtrace, mcs_events, mask, fka, code)
                except M.OperationLimit:
                    assert int(res["status"]) != 0
                    continue
                if int(res["status"]):
                    stats["status"] += 1
                    continue
                got = (sts.violation or 0, sts.delivered, sts.ignored)
                assert got == (int(res["violation"]), int(res["delivered"]), int(res["ignored"])), (t, last, fka)
                rows = [row[:7] for row in flat(sts.events)]
                assert rows == [tuple(int(e[f]) for f in FIELDS7) for e in rec], (t, last, fka)
                assert [sts.trace[i][4] for i in sts.ignoredAbsentIndices] == [int(vtrace[p]["uniq"]) for p in ign]
                stats["checked"] += 1
                stats["violations"] += int(res["violation"]) != 0
                picks[(last, fka)] = rows
        if (0, 0) in picks and (1, 0) in picks and picks[(0, 0)] != picks[(1, 0)]:
            stats["first_last_differ"] += 1


def python_minimize(make_actors, invariant, is_ext, fp, strategy, vtrace, mcs_events, fka, code):
    def test(nxt):
        sts = MW.WildcardSTSReplay(make_actors(), nxt, mcs_events, invariant, is_ext, filter_known_absents=bool(fka),
                                  looking_for=code)
        sts.violation = sts.test(list(range(len(mcs_events))))
        return sts

    def project(nxt):
        return M.subsequence_intersection(nxt, mcs_events, list(range(len(mcs_events))), is_ext, bool(fka))
    wm = MW.WildcardMinimizer(unflat(vtrace), fp, strategy, is_ext, test, project)
    return wm, wm.minimize()


def check_minimize(oracle, model, make_actors, invariant, is_ext, fp, rules, incr, case, model_flags, last, fka):
    vtrace, mcs_prog, mcs_ext, code = case
    flags = (N.WC_LAST_ONLY if last else 0) | fka
    rc, ctrace, total, sizes = W.wildcard_minimize(model, vtrace, mcs_ext, rules, incr, code, flags=flags,
                                                        model_flags=model_flags)
    assert rc == 0
    strategy = MW.LastOnlyStrategy() if last else MW.BackTrackStrategy()
    wm, final = python_minimize(make_actors, invariant, is_ext, fp, strategy, vtrace, to_prog(mcs_prog), fka, code)
    assert (wm.total_replays, wm.internal_sizes) == (total, [int(x) for x in sizes])
    assert [row[:7] for row in flat(final)] == [tuple(int(e[f]) for f in FIELDS7) for e in ctrace]
    return int((vtrace["kind"] == N.EV_MSG_EVENT).sum()), int((ctrace["kind"] == N.EV_MSG_EVENT).sum()), total


def _raft_actors(flags):
    return lambda: {str(k): M.RaftActor(k, flags) for k in range(5)}


def test_wildcard_replays_match_on_raft5(oracle):
    """>= 20 violating raft5 traces, both bug flags: random include masks, First and Last resolution,
    filterKnownAbsents on and off — verdict, counts, recorded trace and ignored positions."""
    cases = raft_cases(oracle, 20)
    assert len(cases) >= 20 and {c[0] for c in cases} == {1, 3}
    rng = np.random.default_rng(11)
    rules, incr = raft_rules()
    stats = dict(checked=0, violations=0, first_last_differ=0, status=0)
    for flags, *case in cases:
        check_replays(oracle, N.MODEL_RAFT5, _raft_actors(flags), M.raft_invariant, lambda m: m[0] in (1, 2),
                      raft_fingerprinter(), incr, case, rng, 6, flags, stats)
    assert stats["checked"] > 400 and stats["violations"] > 20
    assert stats["first_last_differ"] > 0, stats                     # the two resolutions are told apart


def test_wildcard_minimizer_matches_on_raft5(oracle):
    """The whole WildcardMinimizer on the same traces: minTrace, total_replays and the internal-size series."""
    cases = raft_cases(oracle, 20)
    rules, incr = raft_rules()
    removed = 0
    outcomes = {}
    for k, (flags, *case) in enumerate(cases):
        for last in (0, 1):
            fka = k % 2
            before, after, total = check_minimize(oracle, N.MODEL_RAFT5, _raft_actors(flags), M.raft_invariant,
                                                  lambda m: m[0] in (1, 2), raft_fingerprinter(), rules, incr, case, flags,
                                                  last, fka)
            removed += after < before
            outcomes.setdefault(k, []).append((after, total))
    assert removed > 5                                               # non-vacuity: deliveries do get removed
    assert any(v[0] != v[1] for v in outcomes.values())              # First and Last differ on at least one trace


def test_wildcard_on_generated_timer_free_models(oracle):
    """>= 50 timer-free generated models with random clock rules: replays and the whole minimizer."""
    rng = np.random.default_rng(5)
    n_models = n_cases = removed = replays = 0
    stats = dict(checked=0, violations=0, first_last_differ=0, status=0)
    seed = 0
    while n_models < 50 and seed < 2000:
        seed += 1
        m = ir_gen.generate(seed)
        if m.uses_timers:
            continue
        n_models += 1
        oracle.load_model(m.blob)
        W.load_model(m.blob)                                         # the wildcard oracle is a library of its own
        irm = M.IRModel(m.blob)
        prog = ir_gen.program(m, seed)
        ext = D.pack_externals(prog)
        maxm = [40, 60][seed % 2]
        res = oracle.fuzz_batch(N.MODEL_IR, ext, 1, 60, maxm, seed % 4, model_flags=m.flags)
        viol = [1 + int(i) for i in np.nonzero(res["violation"] * (res["status"] == 0))[0][:3]]
        types = list(range(min(m.n_types, 256)))
        spec = {}
        for t in rng.choice(types, size=min(len(types), int(rng.integers(1, 5))), replace=False):
            spec[int(t)] = (int(rng.integers(0, 2)), int(rng.integers(0, 8)), int(rng.choice([1, 2, 3, 8, 32])))
        incr = [int(t) for t in rng.choice(types, size=min(len(types), int(rng.integers(0, 3))), replace=False)]
        rules = [N.clock_rule(t, w, s, b) for t, (w, s, b) in spec.items()]
        fp = closures_of(spec, incr)
        for s in viol:
            case = recorded(oracle, N.MODEL_IR, prog, s, maxm, seed % 4, m.flags)
            if case is None:
                continue
            n_cases += 1
            make = lambda: irm.make_actors(m.flags)
            check_replays(oracle, N.MODEL_IR, make, irm.invariant(m.flags), irm.is_external, fp, incr, case, rng, 3, m.flags, stats)
            try:
                before, after, total = check_minimize(oracle, N.MODEL_IR, make, irm.invariant(m.flags), irm.is_external,
                                                      fp, rules, incr, case, m.flags, seed % 2, 0)
                removed += after < before
                replays += total
            except M.OperationLimit:
                pass
    assert n_models >= 50 and n_cases >= 20 and stats["checked"] > 100, (n_models, n_cases, stats)
    assert removed > 0 and replays > n_cases, (removed, replays)


def test_chain_ddmin_intmin_wildcard(oracle):
    """runTheGamut's order: DDMin over the externals, internal minimization (SrcDstFIFO), then the wildcard stage."""
    prog = D.raft5_program(client_cmds=2)
    ext = D.pack_externals(prog)
    res = oracle.fuzz_batch(N.MODEL_RAFT5, ext, 1, 400, 40, 5, model_flags=1)
    rules, incr = raft_rules()
    done = 0
    for i in np.nonzero(res["violation"])[0][:3]:
        ev, _, r = oracle.fuzz_trace(N.MODEL_RAFT5, ext, 1 + int(i), 40, 5, model_flags=1)
        code = int(r["violation"])
        _, mcs_mask, _, _, _ = oracle.ddmin_sts(N.MODEL_RAFT5, ev, ext, code, model_flags=1)
        mcs_mask = np.asarray(mcs_mask, dtype=np.uint64).reshape(-1)
        rr, vtrace = oracle.replay_trace(N.MODEL_RAFT5, ev, ext, mcs_mask, looking_for=code, model_flags=1)
        if int(rr["violation"]) != code:
            continue
        mcs_prog = [prog[k] for k in range(len(ext)) if (int(mcs_mask[k >> 6]) >> (k & 63)) & 1]
        mcs_ext = D.pack_externals(mcs_prog)
        rc, itrace, _, _, _ = oracle.internal_minimize(N.MODEL_RAFT5, vtrace, mcs_ext, code, model_flags=1,
                                                      flags=N.IM_SRC_DST_FIFO)
        assert rc == 0
        case = (itrace, mcs_prog, mcs_ext, code)
        check_minimize(oracle, N.MODEL_RAFT5, _raft_actors(1), M.raft_invariant, lambda m: m[0] in (1, 2),
                       raft_fingerprinter(), rules, incr, case, 1, 0, 0)
        done += 1
    assert done >= 2
