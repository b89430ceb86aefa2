"""java.util.Random's nextInt(bound) rejection loop on the device, forced on crafted seeds (tests/jrandom_seeds.py).

Every randomized path picks with nextInt(n), and when n is not a power of two Java rejects a raw value in the top
2^31 mod n values and draws again, so every later pick of the execution moves by one draw.  That happens about once in
10^9 draws at this project's bounds.  Each case here first keeps the crafted seeds for which the CPU oracle counts a
rejection, then runs each kept seed s in a window (seed_base = s - 17, 64 executions), so that the rejecting execution
shares its warp with executions that do not loop, and compares every result field of all 64 records with the oracle.
Where the instantiation is known it is asserted, so that a silent fall-back fails."""
import numpy as np
import pytest
import torch

import demi_b200 as D
from demi_b200 import _native as N
from oracle import campaign_binding as CB
from oracle import random_ddmin_binding as RD
import jrandom_seeds as J

pytestmark = pytest.mark.gpu

FIELDS = ["violation", "steps", "state_hash", "trace_hash", "n_nodes", "n_events", "max_pending", "status"]
R, P, B = N.MODEL_RAFT5, N.MODEL_PINGPONG3, N.MODEL_BCAST32
BACK, WINDOW = 17, 64
INT64_MAX, INT64_MIN = (1 << 63) - 1, -(1 << 63)
USER_RULES = [(0b00110, 0b11111, 1 << 5, 0), (0, 0b00001, 1 << 3, 1)]


def wrap64(x):
    return (x + (1 << 63)) % (1 << 64) - (1 << 63)


@pytest.fixture(autouse=True)
def env(monkeypatch):
    monkeypatch.delenv("DEMI_DISABLE_LANE_ENGINE", raising=False)
    monkeypatch.delenv("DEMI_LANE_PENDING_CAP", raising=False)
    return monkeypatch


def assert_same(a, b, what):
    for f in FIELDS:
        bad = np.nonzero(a[f] != b[f])[0]
        assert len(bad) == 0, "%s: field %s differs at %d records, first %d: %s vs %s" % (
            what, f, len(bad), bad[0], a[bad[0]], b[bad[0]])


def kept(lib, run, seeds_by_pos, min_total, min_per_position=0):
    """The crafted seeds whose oracle run counted a rejection, flattened; the counts per position are printed."""
    out, counts = [], {}
    for k, seeds in seeds_by_pos.items():
        c = 0
        for s in seeds:
            lib.reset_jrandom_rejections()
            run(s)
            if lib.jrandom_rejections():
                out.append(s)
                c += 1
        counts[k] = c
    print("kept seeds per position:", counts)
    assert len(out) >= min_total and min(counts.values()) >= min_per_position, counts
    return out


class Case(object):
    """One workload: an engine with its program set, and the oracle's view of it."""

    def __init__(self, oracle, model, prog, maxm, interval, flags=0, blocked_mask=0, strategy=0, looking_for=0,
                 rules=None):
        self.oracle, self.model, self.maxm, self.interval, self.flags = oracle, model, maxm, interval, flags
        self.kw = dict(model_flags=flags, blocked_mask=blocked_mask, strategy=strategy, looking_for=looking_for)
        self.looking_for, self.rules = looking_for, rules
        self.ext = D.pack_externals(prog)
        self.eng = D.Engine(D.SchedulerConfig(model, model_flags=flags, blocked_mask=blocked_mask, strategy=strategy))
        if rules:
            self.eng.set_user_filter(rules)
        self.eng.set_externals(self.ext)
        self.deferred = 0

    def cpu(self, seed_base, n, threads=None):
        self.oracle.set_user_filter(self.rules or [])
        try:
            return self.oracle.fuzz_batch(self.model, self.ext, seed_base, n, self.maxm, self.interval, threads=threads,
                                          **self.kw)
        finally:
            self.oracle.set_user_filter([])

    def seeds(self, positions, per_position, min_total, raw=J.ALWAYS, min_per_position=0):
        return kept(self.oracle, lambda s: self.cpu(s, 1, threads=1), J.crafted(positions, raw, per_position), min_total,
                    min_per_position)

    def window(self, s, kernel=None):
        base = wrap64(s - BACK)
        got = self.eng.fuzz_batch(base, WINDOW, self.maxm, self.interval, looking_for=self.looking_for)
        if kernel is not None:
            assert self.eng.lane_kernel() == kernel
        self.deferred += self.eng.stats().deferred
        assert_same(got, self.cpu(base, WINDOW), "seed %d" % s)
        return got

    def close(self):
        self.eng.close()


# ---------------------------------------------------------------- the steady kernel and its tree
def bench(oracle, **kw):
    return Case(oracle, R, D.raft5_program(), kw.pop("maxm", 50), kw.pop("interval", 5), flags=1, **kw)


def tree_depth(c):
    c.window(1000, kernel=N.LANE_STEADY)
    return c.eng.lane_tree_depth()


def test_steady_tree_walk(oracle):
    """Forced positions 1..depth: the rejection lands in the walk's own draws."""
    c = bench(oracle)
    depth = tree_depth(c)
    assert depth >= 4
    for s in c.seeds(range(1, depth + 1), 8, 5 * depth, min_per_position=2):
        c.window(s, kernel=N.LANE_STEADY)
    c.close()


def test_steady_delivery_loop(oracle):
    """Forced positions depth+1..51: past the tree, in the delivery loop."""
    c = bench(oracle)
    depth = tree_depth(c)
    for s in c.seeds(range(depth + 1, 52), 3, 2 * (51 - depth)):
        c.window(s, kernel=N.LANE_STEADY)
    c.close()


@pytest.mark.parametrize("maxm,interval", [(m, 5) for m in range(9)] + [(50, 1)])
def test_steady_ends_inside_the_tree(oracle, maxm, interval):
    """maxMessages 0..8 and interval 1: executions end, or find a violation, at a node of the tree."""
    c = bench(oracle, maxm=maxm, interval=interval)
    for s in c.seeds(range(1, min(maxm, 9) + 2), 3, 2 if maxm else 1):
        c.window(s, kernel=N.LANE_STEADY)
    c.close()


@pytest.mark.parametrize("variant", ["cap6", "cap8", "clients6", "clients11"])
def test_steady_rollback_at_an_absent_child(oracle, env, variant):
    """Children that defer (a low lane pending cap) or exceed the record's 32 rows (client commands) are not stored:
    the walk stops before them and must leave the generator as it was before that draw, rejected values included."""
    prog = D.raft5_program()
    if variant.startswith("cap"):
        env.setenv("DEMI_LANE_PENDING_CAP", variant[3:])
    else:
        prog = D.raft5_program(client_cmds=int(variant[7:]))
    c = Case(oracle, R, prog, 50, 5, flags=1)
    depth = tree_depth(c)
    for s in c.seeds(range(1, depth + 3), 6, 3 * depth):
        c.window(s, kernel=N.LANE_STEADY)
    if variant.startswith("cap"):
        assert c.deferred > 0
    c.close()


@pytest.mark.parametrize("model,ttl_or_n,maxm,raw", [(B, 2, 200, J.TOP - 4), (B, 3, 200, J.TOP - 16),
                                                     (P, 12, 40, J.TOP - 2)],
                         ids=["bcast32-ttl2", "bcast32-ttl3", "pingpong3"])
def test_steady_other_models(oracle, model, ttl_or_n, maxm, raw):
    """Raw values 2^31 - r with r below 2^31 mod n for most of the model's pending counts."""
    prog = D.bcast32_program(ttl_or_n) if model == B else D.pingpong3_program(ttl_or_n)
    c = Case(oracle, model, prog, maxm, 0)
    positions = list(range(1, 25)) + list(range(30, maxm, 15))
    for s in c.seeds(positions, 3, 20, raw=raw):
        c.window(s, kernel=N.LANE_STEADY)
    c.close()


# ---------------------------------------------------------------- the generic lane kernel and its REC instantiation
def test_generic_lane_kernel_second_segment(oracle):
    prog = D.raft5_program(client_cmds=2)[:-1] + [D.WaitQuiescence(), D.Send(3, 2, 9), D.Send(1, 2, 10), D.WaitQuiescence()]
    c = Case(oracle, R, prog, 60, 5, flags=1)
    for s in c.seeds(range(1, 61, 2), 3, 40):
        c.window(s, kernel=N.LANE_GENERIC)
    c.close()


def test_generic_lane_kernel_looking_for(oracle):
    c = bench(oracle, looking_for=1)
    for s in c.seeds(range(1, 52, 2), 3, 40):
        c.window(s, kernel=N.LANE_GENERIC)
    c.close()


def violating_seeds(oracle, c, count):
    out = []
    for s in c.seeds(range(1, 52), 16, 200):
        if c.cpu(s, 1)[0]["violation"]:
            out.append(s)
    assert len(out) >= count, len(out)
    return out[:count]


def test_lane_rec_provenance_and_trace(oracle):
    """fuzz_provenance records violating executions on the lane REC instantiation; fuzz_trace gives the whole trace."""
    c = bench(oracle)
    for s in violating_seeds(oracle, c, 12):
        base = s - BACK
        res = c.cpu(base, WINDOW)
        idx = np.nonzero(res["violation"])[0]
        assert BACK in idx
        keep, out, rec = c.eng.fuzz_provenance(base, idx, 50, 5)
        assert np.array_equal(rec["trace_hash"], res["trace_hash"][idx]) and np.array_equal(rec["steps"], res["steps"][idx])
        for j, i in enumerate(idx):
            k, o = oracle.fuzz_provenance(R, c.ext, base + int(i), 50, 5, keep.shape[1], model_flags=1)
            assert o["status"] == out[j]["status"] == 0 and np.array_equal(k, keep[j]), (s, int(i))
        ev, par, r = c.eng.fuzz_trace(s, 50, 5)
        cev, cpar, cr = oracle.fuzz_trace(R, c.ext, s, 50, 5, model_flags=1)
        assert ev.tobytes() == cev.tobytes() and par.tobytes() == cpar.tobytes() and r.tobytes() == cr.tobytes(), s
    c.close()


# ---------------------------------------------------------------- the warp engine
@pytest.mark.parametrize("variant", ["fully-random", "blocked", "user-filter", "hard-kill"])
def test_warp_engine(oracle, env, variant):
    env.setenv("DEMI_DISABLE_LANE_ENGINE", "1")
    if variant == "fully-random":
        c = bench(oracle)
    elif variant == "blocked":
        c = Case(oracle, R, D.raft5_program(client_cmds=3), 50, 5, flags=1, blocked_mask=1 << 1)
    elif variant == "user-filter":
        c = bench(oracle, rules=USER_RULES)
    else:
        prog = D.raft5_program(client_cmds=3)[:-1] + [D.WaitQuiescence(), D.HardKill(1), D.Send(1, 2, 40), D.WaitQuiescence(),
                                                      D.Start(1), D.Send(1, 1, 0x1F), D.WaitQuiescence()]
        c = Case(oracle, R, prog, 90, 7, flags=1)
    for s in c.seeds(range(2, 52), 3, 60):
        c.window(s, kernel=N.LANE_NONE)
    c.close()


def test_src_dst_fifo(oracle):
    """SrcDstFIFO's two generators share the seed: position k forces whichever draws k-th."""
    c = Case(oracle, R, D.raft5_program(client_cmds=3), 50, 5, flags=1, strategy=1)
    for s in c.seeds(range(1, 61), 3, 80):
        c.window(s)
    c.close()


# ---------------------------------------------------------------- regression seeds found by counting rejections
@pytest.mark.parametrize("model,prog,maxm,interval,flags,seed",
                         [(R, "bench", 50, 5, 1, 36_096_526), (R, "bench", 50, 5, 1, 21_237), (B, "ttl3", 200, 0, 0, 13_889)],
                         ids=["raft5-36096526", "raft5-21237", "bcast32-ttl3-13889"])
def test_regression_seeds(oracle, model, prog, maxm, interval, flags, seed):
    c = Case(oracle, model, D.raft5_program() if prog == "bench" else D.bcast32_program(3), maxm, interval, flags=flags)
    oracle.reset_jrandom_rejections()
    c.cpu(seed, 1, threads=1)
    assert oracle.jrandom_rejections() == 1
    c.window(seed, kernel=N.LANE_STEADY)
    c.close()


# ---------------------------------------------------------------- campaigns (the Fuzzer on the device)
# The bench program without its WaitQuiescence: the generated client commands, kills and partitions join the first
# segment, so the executions of different programs differ within maxMessages.
CAMPAIGN_PREFIX = D.pack_externals(D.raft5_program()[:-1])


def campaign_setup():
    w = (0.01, 0.4, 0.1, 0.25, 0.25, 40, 2)
    eng = D.Engine(D.SchedulerConfig(R, model_flags=1))
    eng.set_fuzzer(N.FuzzerConfig(*w), CAMPAIGN_PREFIX, D.pack_externals([]))
    return eng, CB.FuzzerConfig(*w)


def campaign_records(eng, seed_base, program_seed_base, dev):
    if not dev:
        return eng.fuzz_campaign(seed_base, WINDOW, 50, 5, program_seed_base)
    buf = torch.empty(WINDOW * N.RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    eng.fuzz_campaign_dev(seed_base, WINDOW, 50, 5, program_seed_base, buf.data_ptr())
    torch.cuda.synchronize()
    return buf.cpu().numpy().view(N.RESULT_DTYPE)


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_campaign_crafted_program_seeds(dev):
    """program_seed_base + i crafted: the generator kernel's set draws reject."""
    eng, ocfg = campaign_setup()
    pre = CAMPAIGN_PREFIX
    ps = kept(CB, lambda s: CB.fuzzer_generate(ocfg, s, pre), J.crafted(range(1, 25), J.ALWAYS, 3), 30)
    for s in ps[::2]:
        got = campaign_records(eng, 1000, s - BACK, dev)
        want = CB.fuzz_campaign(R, ocfg, pre, None, 1000, WINDOW, 50, 5, s - BACK, model_flags=1)
        assert_same(got, want, "program seed %d" % s)
    eng.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_campaign_crafted_execution_seeds(dev):
    """seed_base + i crafted: the executions of generated programs reject."""
    eng, ocfg = campaign_setup()
    pre = CAMPAIGN_PREFIX
    CB.reset_jrandom_rejections()
    CB.fuzzer_generate(ocfg, 55 + BACK, pre)
    assert CB.jrandom_rejections() == 0
    ss = kept(CB, lambda s: CB.fuzz_campaign(R, ocfg, pre, None, s, 1, 50, 5, 55 + BACK, model_flags=1, threads=1),
              J.crafted(range(1, 40), J.ALWAYS, 2), 30)
    for s in ss[::2]:
        got = campaign_records(eng, s - BACK, 55, dev)
        want = CB.fuzz_campaign(R, ocfg, pre, None, s - BACK, WINDOW, 50, 5, 55, model_flags=1)
        assert_same(got, want, "seed %d" % s)
    eng.close()


# ---------------------------------------------------------------- random-oracle tests
def full_and_sub_masks(n_ext, rng):
    masks = [list(range(n_ext))] + [sorted(int(i) for i in np.nonzero(rng.random(n_ext) < 0.8)[0]) for _ in range(7)]
    mw = RD.mask_words(n_ext)
    out = np.zeros((len(masks), mw), dtype=np.uint64)
    for r, m in enumerate(masks):
        for i in m:
            out[r, i // 64] |= np.uint64(1) << np.uint64(i % 64)
    return out


def test_random_test_batch_and_ddmin(oracle):
    prog = D.raft5_program(client_cmds=3)
    c = Case(oracle, R, prog, 50, 5, flags=1)
    masks = full_and_sub_masks(len(c.ext), np.random.default_rng(7))
    viol = violating_seeds(oracle, c, 6)
    for s in viol:
        for base, n in ((s - BACK, WINDOW), (s, 8)):
            got = c.eng.random_test_batch(masks, n, base, 50, 5)
            want = RD.random_test_batch(R, c.ext, masks, n, base, 50, 5, model_flags=1)
            assert got.tobytes() == want.tobytes(), (s, base)
        assert got[0]["first_hit"] == 0
    for s in viol[:3]:
        code = int(c.cpu(s, 1)[0]["violation"])
        want = RD.random_ddmin(R, c.ext, 4, s, 50, code, 5, model_flags=1)
        assert want["rc"] == 0
        mcs, sizes, keys, out = c.eng.random_ddmin(4, s, 50, code, 5)
        assert list(mcs) == list(want["mcs"]) and list(sizes) == list(want["sizes"]) and list(keys) == list(want["keys"])
        assert out.total_replays == want["total_replays"] and out.verified == want["verified"]
    c.close()


# ---------------------------------------------------------------- seed arithmetic: Java's long addition wraps
def test_seeds_equal_modulo_2_to_48_and_negative_bases(oracle):
    c = bench(oracle)
    s = 12_345
    ref = c.eng.fuzz_batch(s, WINDOW, 50, 5)
    assert_same(ref, c.cpu(s, WINDOW), "base")
    for j in (1, -1, 5, -7, 1 << 14):
        b = wrap64(s + j * (1 << 48))
        assert_same(c.eng.fuzz_batch(b, WINDOW, 50, 5), ref, "engine at %d" % b)
        assert_same(c.cpu(b, WINDOW), ref, "oracle at %d" % b)
    neg = c.eng.fuzz_batch(-40, WINDOW, 50, 5)
    assert_same(neg, c.cpu(-40, WINDOW), "negative base")
    c.close()


def test_batch_across_int64_max(oracle):
    """Seeds past INT64_MAX are the seeds written after the wrap, from INT64_MIN."""
    c = bench(oracle)
    base = INT64_MAX - 20
    got = c.eng.fuzz_batch(base, WINDOW, 50, 5)
    after = c.eng.fuzz_batch(INT64_MIN, WINDOW - 21, 50, 5)
    assert_same(got[21:], after, "engine after the wrap")
    want = c.cpu(base, WINDOW)
    assert_same(got, want, "oracle across the wrap")
    assert_same(c.cpu(INT64_MIN, WINDOW - 21), after, "oracle after the wrap")
    c.close()


def test_chunked_batch_whose_later_chunk_starts_past_the_wrap(oracle):
    """More than 2 * 2^21 prefixes run in three chunks; the third chunk's own base lies past INT64_MAX, and the second
    chunk crosses it."""
    chunk = 2 << 20
    n = 2 * chunk + 1
    per = -(-n // 3)
    base = INT64_MAX - per - per // 2
    c = bench(oracle)
    host = c.eng.fuzz_batch(base, n, 50, 5)
    assert wrap64(base + 2 * per) < 0 < wrap64(base + per)
    for a, b in [(0, 256), (per - 256, per + 256), (per + per // 2 - 256, per + per // 2 + 256),
                 (2 * per - 256, 2 * per + 256), (n - 256, n)]:
        assert_same(host[a:b], c.cpu(wrap64(base + a), b - a), "records %d..%d" % (a, b))
    c.close()
