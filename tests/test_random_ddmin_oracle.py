"""DDMin with RandomScheduler as the TestOracle (RunnerUtils.randomDDMin): the C oracle (oracle/random_ddmin.c) against
the Python restatement (tests/micro_oracle_random.py over micro_oracle.Execution) — per-test records, and whole
minimizations: the test order, the MCS, total_replays, the keyed iteration-size series and verify_mcs."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
import micro_oracle as M
import micro_oracle_random as MR
from test_micro_oracle import to_prog

RAFT_FLAGS, PP_FLAGS = 1, 1 | (2 << 8)          # raft5's double-vote bug; pingpong3: actor 0 has seen 2 pongs


@pytest.fixture(scope="module")
def rd():
    from demi_b200 import build
    build.build_oracle()
    from oracle import random_ddmin_binding
    random_ddmin_binding.lib()
    return random_ddmin_binding


class _StaticBlocked(M.Execution):
    """blockedActors as the engine offers it (DESIGN.md §8): a static set."""

    def inject_until_quiescence(self):
        M.Execution.inject_until_quiescence(self)
        self.blockedActors |= self.static_blocked


def micro_runner(model, flags, maxm, interval, looking_for, rules=(), strategy=0, blocked=(), irm=None):
    """run_one(subsequence in micro_oracle's form, seed) -> violation code or 0, on the restatement."""
    if model == N.MODEL_RAFT5:
        fresh, n, inv, ext = (lambda a: M.RaftActor(int(a), flags)), 5, M.raft_invariant, (lambda m: m[0] in (1, 2))
    elif model == N.MODEL_PINGPONG3:
        fresh, n, inv, ext = (lambda a: M.PingPongActor(int(a))), 3, M.pingpong_invariant(flags), (lambda m: m[0] == 1)
    else:
        fresh, inv, ext = irm.fresh(flags), irm.invariant(flags), irm.is_external

    def user_filter(snd, rcv, msg):
        for src_mask, dst_mask, type_mask, fl in rules:
            src_ok = ((src_mask >> int(snd)) & 1) if snd.isdigit() else (fl & 1)
            if src_ok and (dst_mask >> int(rcv)) & 1 and (type_mask >> msg[0]) & 1:
                return False
        return True

    def run_one(sub, seed):
        actors = irm.make_actors(flags) if irm else {str(i): fresh(str(i)) for i in range(n)}
        cls = M.SrcDstFifoExecution if strategy == 1 else _StaticBlocked if blocked else M.Execution
        ex = cls(actors, list(sub), seed, maxm, interval, inv, ext, blocked=[str(b) for b in blocked],
                 looking_for=looking_for or None, user_filter=user_filter if rules else None, fresh_actor=fresh)
        ex.static_blocked = set(str(b) for b in blocked)
        return ex.run() or 0
    return run_one


def bits(idx, n):
    m = np.zeros(max(1, (n + 63) // 64), dtype=np.uint64)
    for i in idx:
        m[i // 64] |= np.uint64(1) << np.uint64(i % 64)
    return m


def wq_shapes(prog, idx_sets):
    """Which WaitQuiescence shapes the subsequences have: adjacent, leading, trailing."""
    out = set()
    for s in idx_sets:
        kinds = [type(prog[i]).__name__ for i in s]
        if kinds and kinds[0] == "WaitQuiescence":
            out.add("leading")
        if kinds and kinds[-1] == "WaitQuiescence":
            out.add("trailing")
        if any(a == b == "WaitQuiescence" for a, b in zip(kinds, kinds[1:])):
            out.add("adjacent")
    return out


RAFT_WQ = [D.WaitQuiescence()] + D.raft5_program(client_cmds=2)[:-1] + [D.WaitQuiescence(), D.Send(1, 2, 40), D.WaitQuiescence(),
                                                                        D.Send(2, 2, 41), D.WaitQuiescence()]
# (no Start after the HardKill: get_atomic_events keeps one Start per actor and asserts that every event is in an atom)
RAFT_HK = D.raft5_program(client_cmds=2)[:-1] + [D.WaitQuiescence(), D.HardKill(1), D.Send(2, 2, 40), D.WaitQuiescence(),
                                                D.Kill(3), D.Send(0, 2, 9), D.WaitQuiescence()]
RAFT_PART = D.raft5_program(client_cmds=1)[:-1] + [D.Partition(0, 1), D.WaitQuiescence(), D.UnPartition(0, 1), D.Send(3, 2, 7),
                                                  D.WaitQuiescence()]
PP = D.pingpong3_program(n_sends=6)[:-1] + [D.WaitQuiescence(), D.Send(0, 1, 50), D.WaitQuiescence()]
# (name, model, flags, program, max_messages, interval, N, seed, config)
CASES = [
    ("raft5_wq", N.MODEL_RAFT5, RAFT_FLAGS, RAFT_WQ, 60, 5, 8, 11, {}),
    ("raft5_hardkill", N.MODEL_RAFT5, RAFT_FLAGS, RAFT_HK, 60, 5, 6, 3, {}),
    ("raft5_partition_fifo", N.MODEL_RAFT5, RAFT_FLAGS, RAFT_PART, 60, 5, 6, 21, dict(strategy=1)),
    ("raft5_filter", N.MODEL_RAFT5, RAFT_FLAGS, D.raft5_program(client_cmds=1), 60, 5, 8, 5,
     dict(rules=[(0b00110, 0b11111, 1 << 5, 0)])),
    ("raft5_blocked", N.MODEL_RAFT5, RAFT_FLAGS, RAFT_WQ, 60, 5, 8, 40, dict(blocked=(4,))),
    ("pingpong3", N.MODEL_PINGPONG3, PP_FLAGS, PP, 40, 0, 4, 1, {}),
]


def atoms_cover(prog):
    """UnmodifiedEventDag.get_atomic_events's `assume`: every event of the program is in an atom (and no Kill lacks
    its Start)."""
    try:
        return sum(len(a) for a in M.atomic_events(list(enumerate(to_prog(prog))))) == len(prog)
    except KeyError:
        return False


def _oracle_cfg(c):
    return dict(strategy=c.get("strategy", 0), blocked_mask=sum(1 << b for b in c.get("blocked", ())))


def _violation(rd, model, flags, prog, maxm, interval, n, seed, c):
    """The code the whole program's first hit shows (the violation randomDDMin minimizes for)."""
    ext = D.pack_externals(prog)
    r = rd.random_test_batch(model, ext, bits(range(len(prog)), len(prog)), 64, seed, maxm, interval, model_flags=flags,
                             **_oracle_cfg(c))[0]
    return int(r["violation"])


def _run_case(rd, name, model, flags, prog, maxm, interval, n, seed, c, irm=None, skip_status=False):
    rd.set_user_filter(c.get("rules", []))
    try:
        looking = _violation(rd, model, flags, prog, maxm, interval, n, seed, c)
        assert looking, name
        ext = D.pack_externals(prog)
        got = rd.random_ddmin(model, ext, n, seed, maxm, looking, interval, model_flags=flags, **_oracle_cfg(c))
        if skip_status and got["rc"] == -4:
            return None                                  # a capacity status, which the restatement does not model
        assert got["rc"] == 0, (name, got["rc"])
        run_one = micro_runner(model, flags, maxm, interval, looking, c.get("rules", ()), c.get("strategy", 0),
                               c.get("blocked", ()), irm)
        mprog = to_prog(prog)
        d, mcs, verified = MR.random_ddmin(run_one, mprog, n, seed)
        tests = [tuple(int(i) for i in range(len(prog)) if (int(t[i // 64]) >> (i % 64)) & 1) for t in got["tests"]]
        assert tests == d.tests, name
        assert [tuple(int(r[f]) for f in ("first_hit", "executions_run", "violation")) for r in got["records"]] == d.records, name
        assert all(int(r["status"]) == 0 for r in got["records"])
        assert [i for i in range(len(prog)) if (int(got["mcs"][i // 64]) >> (i % 64)) & 1] == mcs, name
        assert got["total_replays"] == d.total_replays and list(got["sizes"]) == d.sizes and list(got["keys"]) == d.keys, name
        assert bool(got["verified"]) == verified, name
        # the per-test records of arbitrary masks, batched and threaded
        rng = np.random.default_rng(seed)
        masks = [sorted(int(i) for i in np.nonzero(rng.random(len(prog)) < 0.7)[0]) for _ in range(12)]
        masks += [[i for i in range(len(prog)) if i != k] for k in range(len(prog))]      # leave one out
        recs = rd.random_test_batch(model, ext, np.stack([bits(m, len(prog)) for m in masks]), n, seed, maxm, interval,
                                    looking_for=looking, model_flags=flags, **_oracle_cfg(c))
        for m, r in zip(masks, recs):
            want = MR.random_test(lambda s: run_one([mprog[i] for i in m], s), n, seed)
            assert (int(r["first_hit"]), int(r["executions_run"]), int(r["violation"]), int(r["status"])) == want + (0,), (name, m)
        return d, got, recs, masks
    finally:
        rd.set_user_filter([])


def test_stats_keying_counts_executions():
    """Hand-checked: tests are keyed by the running sum of executions.  Program a b c d (single atoms); a test violates
    iff it keeps c, with its first hit at j = 3 (4 executions); a miss runs all N = 5."""
    prog = [("Send", "0", (1, k, 0)) for k in range(4)]
    d = MR.RandomDDMin(lambda sub: (3, 4, 7) if prog[2] in sub else (-1, 5, 0))
    assert d.minimize(prog) == [2]
    assert d.tests == [(0, 1), (2, 3), (2,)]
    assert d.records == [(-1, 5, 0), (3, 4, 7), (3, 4, 7)]
    assert d.sizes == [4, 4, 2, 1]                   # original - pruned when each test is recorded, then the fencepost
    assert d.keys == [5, 9, 13, 13]                  # a miss adds N = 5, a hit at j = 3 adds 4
    assert d.total_replays == 13


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_equals_the_restatement(rd, case):
    _run_case(rd, *case)


def test_the_cases_are_not_vacuous(rd):
    """Across the cases: hits at j > 0, misses, and subsequences with adjacent, leading and trailing WaitQuiescence."""
    later_hits, misses, shapes = 0, 0, set()
    for case in CASES:
        d, got, recs, masks = _run_case(rd, *case)
        later_hits += sum(1 for r in d.records if r[0] > 0) + int((recs["first_hit"] > 0).sum())
        misses += sum(1 for r in d.records if r[0] < 0) + int((recs["first_hit"] < 0).sum())
        shapes |= wq_shapes(case[3], d.tests + [tuple(m) for m in masks])
    assert later_hits and misses
    assert shapes == {"adjacent", "leading", "trailing"}


def test_generated_models(rd):
    """tests/ir_gen.py models: the oracle equals the restatement on every one whose program shows a violation."""
    import ir_gen
    from oracle import random_ddmin_binding
    done = 0
    for s in range(1, 40):
        m = ir_gen.generate(s)
        irm = M.IRModel(m.blob)
        prog = ir_gen.program(m, s, hard_kill=(s % 3 == 1))
        random_ddmin_binding.load_model(m.blob)
        if not atoms_cover(prog) or not _violation(rd, N.MODEL_IR, m.flags, prog, 40, 2, 8, s, {}):
            continue
        try:
            if _run_case(rd, "ir%d" % s, N.MODEL_IR, m.flags, prog, 40, 2, 8, s, {}, irm=irm, skip_status=True) is None:
                continue
        except M.OperationLimit:
            continue
        done += 1
        if done >= 6:
            break
    assert done >= 3


def test_record_layouts_match_the_header(tmp_path):
    """sizeof() and field offsets of demi_random_test_result / demi_random_ddmin_out equal the ctypes / numpy mirror."""
    import ctypes as C
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "sizes.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "demi_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu\\n", sizeof(demi_random_test_result), offsetof(demi_random_test_result, status),'
                   ' sizeof(demi_random_ddmin_out));\n'
                   '  printf("%zu %zu\\n", offsetof(demi_random_ddmin_out, executions_executed), offsetof(demi_random_ddmin_out, verified));\n'
                   '  return 0;\n}\n')
    exe = tmp_path / "sizes"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [N.RANDOM_TEST_DTYPE.itemsize, N.RANDOM_TEST_DTYPE.fields["status"][1], C.sizeof(N.RandomDDMinOut),
                   N.RandomDDMinOut.executions_executed.offset, N.RandomDDMinOut.verified.offset]
