"""java.util.Random's nextInt(bound) rejection loop, forced on crafted seeds (tests/jrandom_seeds.py), on the CPU side.

The loop runs about once in 10^9 draws at this project's bounds, so ordinary seed ranges never reach it.  Each crafted
seed forces one draw of its execution to a raw value that the bound at that draw rejects, unless the bound there is a
power of two or the execution ended earlier.  A case keeps a seed only if the oracle's rejection counter shows that the
loop ran, and asserts a minimum number of kept seeds per position, so that it cannot pass without reaching the loop.
The kept seeds are then compared between the C oracle and the independent Python restatement (tests/micro_oracle.py):
verdict, counters and the whole EventTrace and DepTracker tree."""
import ctypes as C

import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N, fuzzer as F
import ir_gen
import jrandom_seeds as J
import micro_oracle as M
from test_micro_oracle import flat, run_micro
from test_model_ir_random import run_python

R, P = N.MODEL_RAFT5, N.MODEL_PINGPONG3
FIELDS = ("kind", "src", "dst", "type", "p0", "p1", "uniq", "node")


def test_seed_for_places_the_raw_value_at_its_position(oracle):
    for k in (1, 2, 3, 17, 50, 200):
        for raw in (J.ALWAYS, J.TOP - 3, 0, 12345):
            for low in (0, 1, 0x1FFFF):
                s = J.seed_for(k, raw, low)
                got = oracle.kat_jrandom(s, 0, k)                     # nextInt() = next(32); next(31) is its top 31 bits
                assert (got[k - 1] & 0xFFFFFFFF) >> 1 == raw
                assert J.raw_draws(s, k)[k - 1] == raw
    assert F.JavaRandom(J.seed_for(1, J.ALWAYS)).nextDouble() == ((1 << 26) - 1) * 2.0 ** -26 + \
        (J.raw_draws(J.seed_for(1, J.ALWAYS), 2)[1] >> 4) * 2.0 ** -53
    assert F.JavaRandom(J.seed_for(1, 0)).nextDouble() < 2.0 ** -26


@pytest.mark.parametrize("bound", [3, 5, 6, 7, 10, 11, 13, 100, 1000, 65537])
def test_a_rejected_draw_consumes_exactly_one_more(oracle, bound):
    """nextInt(bound) on the oracle at a forced position: every later value comes one raw draw later."""
    assert J.rejects(J.ALWAYS, bound)
    for k in (1, 2, 9, 40):
        s = J.seed_for(k, J.ALWAYS, 0x2A)
        raws = J.raw_draws(s, 80)
        assert not any(J.rejects(u, bound) for i, u in enumerate(raws) if i != k - 1)
        want = [u % bound for i, u in enumerate(raws) if i != k - 1][:60]
        oracle.reset_jrandom_rejections()
        assert oracle.kat_jrandom(s, bound, 60) == want
        assert oracle.jrandom_rejections() == 1
        r = F.JavaRandom(s)
        assert [r.nextInt(bound) for _ in range(60)] == want
        r = M.JavaRandom(s)
        assert [r.nextInt(bound) for _ in range(60)] == want


def test_rejects_matches_the_oracle_for_raw_values_below_the_top(oracle):
    """Raw value 2^31 - r is rejected exactly by the bounds with 2^31 mod n >= r."""
    seen = set()
    for n in list(range(3, 200)) + [1000, 4099, 65537, (1 << 30) + 1, (1 << 31) - 1]:
        for r in (1, 2, 5, 64, 1000, 100000):
            s = J.seed_for(1, J.TOP - r, 3)
            oracle.reset_jrandom_rejections()
            oracle.kat_jrandom(s, n, 1)
            got = oracle.jrandom_rejections() > 0
            assert got == J.rejects(J.TOP - r, n) == (n & (n - 1) != 0 and J.TOP % n >= r), (n, r)
            seen.add(got)
    assert seen == {True, False}


def kept(lib, run, seeds_by_pos, min_per_position):
    """The seeds whose oracle run (`run(seed)`) counted at least one rejection, per position."""
    out = {}
    for k, seeds in seeds_by_pos.items():
        keep = []
        for s in seeds:
            lib.reset_jrandom_rejections()
            run(s)
            if lib.jrandom_rejections():
                keep.append(s)
        out[k] = keep
    counts = {k: len(v) for k, v in out.items()}
    print("kept seeds per position:", counts)
    assert min(counts.values()) >= min_per_position, counts
    return out


def compare_with_restatement(oracle, model, prog, seed, maxm, interval, flags, py, strategy=0, blocked_mask=0):
    ext = D.pack_externals(prog)
    r = oracle.fuzz_batch(model, ext, seed, 1, maxm, interval, model_flags=flags, strategy=strategy,
                          blocked_mask=blocked_mask, threads=1)[0]
    ex, v = py(seed)
    assert int(r["status"]) == 0, seed
    assert (int(r["violation"]), int(r["steps"]), int(r["n_nodes"]), int(r["n_events"]), int(r["max_pending"])) == \
           (v, ex.messagesScheduledSoFar, ex.depTracker.next_id, len(ex.events), ex.max_pending), seed
    ev, par, _ = oracle.fuzz_trace(model, ext, seed, maxm, interval, model_flags=flags, strategy=strategy,
                                   blocked_mask=blocked_mask)
    assert [tuple(int(e[f]) for f in FIELDS) for e in ev] == flat(ex.events), seed
    assert [int(x) for x in par] == [ex.depTracker.parent_of[i] for i in range(ex.depTracker.next_id)], seed
    return v


def crafted_case(oracle, model, prog, positions, maxm, interval, flags, per_position, min_per_position, raw=J.ALWAYS,
                 strategy=0, blocked=()):
    ext = D.pack_externals(prog)
    bmask = sum(1 << b for b in blocked)
    if blocked:
        def py(seed):
            ex = StaticBlocked(*micro_args(model, prog, seed, maxm, interval, flags), blocked=[str(b) for b in blocked])
            ex.static_blocked = set(str(b) for b in blocked)
            return ex, (ex.run() or 0)
    else:
        def py(seed):
            return run_micro(model, prog, seed, maxm, interval, flags, strategy=strategy)
    seeds = kept(oracle, lambda s: oracle.fuzz_batch(model, ext, s, 1, maxm, interval, model_flags=flags, strategy=strategy,
                                                     blocked_mask=bmask, threads=1),
                 J.crafted(positions, raw, per_position), min_per_position)
    n_viol = 0
    for k, ss in seeds.items():
        for s in ss:
            n_viol += bool(compare_with_restatement(oracle, model, prog, s, maxm, interval, flags, py, strategy, bmask))
    return n_viol


class StaticBlocked(M.Execution):
    """blockedActors as the engine offers it (DESIGN.md §8): a static set; a Start does not unblock the actor."""

    def inject_until_quiescence(self):
        M.Execution.inject_until_quiescence(self)
        self.blockedActors |= self.static_blocked


def micro_args(model, prog, seed, maxm, interval, flags):
    from test_micro_oracle import to_prog
    assert model == R
    actors = {str(i): M.RaftActor(i, flags) for i in range(5)}
    return (actors, to_prog(prog), seed, maxm, interval, M.raft_invariant, lambda m: m[0] in (1, 2))


def test_raft5_bench_program_positions_1_to_51(oracle):
    """The benchmark's workload (maxMessages 50, invariant every 5): a rejected draw at every position of the tree walk
    and of the delivery loop."""
    n_viol = crafted_case(oracle, R, D.raft5_program(), range(1, 52), 50, 5, 1, per_position=6, min_per_position=3)
    assert n_viol > 0


def test_pingpong3(oracle):
    crafted_case(oracle, P, D.pingpong3_program(20), range(1, 35), 40, 3, 0, per_position=4, min_per_position=1)


def test_blocked_actor_redraw(oracle):
    """A blocked receiver makes find_non_blocked_message draw again: the forced draw lands in that loop too.  The first
    draw is over 8 pending messages, a power of two."""
    crafted_case(oracle, R, D.raft5_program(client_cmds=3), range(2, 41), 50, 5, 1, per_position=4, min_per_position=2,
                 blocked=(1,))


def test_src_dst_fifo(oracle):
    """SrcDstFIFO's two generators take the same seed: position k forces whichever draws k-th."""
    crafted_case(oracle, R, D.raft5_program(client_cmds=3), range(1, 41), 50, 5, 1, per_position=4, min_per_position=2,
                 strategy=1)


def test_loaded_ir_model(oracle):
    total = 0
    for s in (5, 12, 40):
        m = ir_gen.generate(s)
        oracle.load_model(m.blob)
        irm = M.IRModel(m.blob)
        prog = ir_gen.program(m, s)
        ext = D.pack_externals(prog)
        seeds = kept(oracle, lambda sd: oracle.fuzz_batch(N.MODEL_IR, ext, sd, 1, 30, 3, model_flags=m.flags, threads=1),
                     J.crafted(range(1, 21), J.ALWAYS, 3), 0)
        for k, ss in seeds.items():
            for sd in ss:
                ex, v, raised = run_python(m, irm, prog, sd, 30, 3)
                r = oracle.fuzz_batch(N.MODEL_IR, ext, sd, 1, 30, 3, model_flags=m.flags, threads=1)[0]
                if raised or int(r["status"]):
                    assert raised == bool(int(r["status"])) or int(r["status"]), (s, sd)
                    continue
                assert (int(r["violation"]), int(r["steps"]), int(r["n_nodes"]), int(r["n_events"])) == \
                       (v, ex.messagesScheduledSoFar, ex.depTracker.next_id, len(ex.events)), (s, sd)
                ev, par, _ = oracle.fuzz_trace(N.MODEL_IR, ext, sd, 30, 3, model_flags=m.flags)
                assert [tuple(int(e[f]) for f in FIELDS) for e in ev] == flat(ex.events), (s, sd)
                total += 1
    print("IR executions with a rejection compared:", total)
    assert total >= 20


# ---------------------------------------------------------------- the Fuzzer
PREFIX = [D.Start(a) for a in range(5)] + [D.Send(a, 1, 0x1F) for a in range(5)]
WEIGHTS = dict(kill=0.01, send=0.4, wait_quiescence=0.1, partition=0.25, unpartition=0.25)
# kills stay rare: once everybody is killed, fuzzer.py raises where the C restatements draw nextInt(0)


def fuzzer_programs(native, campaign, seed, num_events=60):
    """The same program three ways: the campaign oracle's C restatement, demi_b200/fuzzer.py and the C ABI's
    demi_fuzzer_generate (the host build of the device generator)."""
    cfg = campaign.FuzzerConfig(WEIGHTS["kill"], WEIGHTS["send"], WEIGHTS["wait_quiescence"], WEIGHTS["partition"],
                                WEIGHTS["unpartition"], num_events, 2)
    pext = D.pack_externals(PREFIX)
    c = campaign.fuzzer_generate(cfg, seed, pext)
    w = F.FuzzerWeights(WEIGHTS["kill"], WEIGHTS["send"], WEIGHTS["wait_quiescence"], WEIGHTS["partition"],
                        WEIGHTS["unpartition"])
    py = D.pack_externals(F.Fuzzer(num_events, w, F.ClientCommandGenerator(2), PREFIX, seed=seed).generateFuzzTest())
    ncfg = native.FuzzerConfig(*[WEIGHTS[k] for k in ("kill", "send", "wait_quiescence", "partition", "unpartition")],
                               num_events, 2)
    out = np.zeros(len(pext) + num_events + 2, dtype=native.EXT_DTYPE)
    n = C.c_uint32()
    rc = native.lib().demi_fuzzer_generate(C.byref(ncfg), seed, pext.ctypes.data, len(pext), None, 0, out.ctypes.data,
                                           len(out), C.byref(n))
    assert rc == 0
    return c, py, out[:n.value]


def assert_same_programs(c, py, host, seed):
    assert len(c) == len(py) == len(host), seed
    for f in ("kind", "a", "b", "type", "p0", "p1", "id"):
        assert (c[f] == host[f]).all(), (seed, f)
    for f in ("kind", "a", "b", "type", "p0", "p1"):
        assert (c[f] == py[f]).all(), (seed, f)


@pytest.fixture(scope="module")
def campaign():
    from oracle import campaign_binding
    campaign_binding.lib()
    return campaign_binding


def test_fuzzer_rejections_in_the_set_draws(native, campaign):
    """Forced rejections in the draws of `alive` (5 actors, nextInt(5..1)) and of the two pair sets (10 pairs)."""
    seeds = kept(campaign, lambda s: fuzzer_programs(native, campaign, s), J.crafted(range(1, 25), J.ALWAYS, 4), 1)
    n = 0
    for k, ss in seeds.items():
        for s in ss:
            assert_same_programs(*fuzzer_programs(native, campaign, s), s)
            n += 1
    assert n >= 60


@pytest.mark.parametrize("top,cls", [(J.ALWAYS, None), (0, "Kill")], ids=["top-wait-quiescence", "zero-kill"])
def test_fuzzer_next_double_at_both_extremes(native, campaign, monkeypatch, top, cls):
    """A nextDouble whose first half is all ones is at least 1 - 2^-26, the last weight class (WaitQuiescence); all
    zeros is below 2^-26, the Kill class.  Forced at the j-th nextDouble of the program generator."""
    drawn, base = [], F.JavaRandom

    class Logged(base):
        def nextDouble(self):
            drawn.append(base.nextDouble(self))
            return drawn[-1]
    for j in range(1, 30):
        for low in (0x11, 0x777, 0x1F00F):
            s = J.seed_for(2 * j - 1, top, low)
            del drawn[:]
            with monkeypatch.context() as mp:
                mp.setattr(F, "JavaRandom", Logged)
                F.Fuzzer(60, F.FuzzerWeights(**WEIGHTS), F.ClientCommandGenerator(2), PREFIX, seed=s).generateFuzzTest()
            x = drawn[j - 1]
            assert (x >= 1 - 2.0 ** -26 if top else x < 2.0 ** -26), (j, x)
            assert F.FuzzerWeights(**WEIGHTS).getNextEventType(x) == cls
            assert_same_programs(*fuzzer_programs(native, campaign, s), s)
