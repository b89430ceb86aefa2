"""raft5 on external messages of every type (DESIGN.md §3, raft5 rules R1-R3), on the CPU.

The generated programs of raft5_gen.py drive the handlers with payloads no correct peer sends and with deadLetters as the
sender.  Here: the Python restatement (micro_oracle.py) against the C oracle on the whole corpus; the C oracle built with
AddressSanitizer and UndefinedBehaviorSanitizer on the same corpus and on raft5 campaigns of each protocol send type; and
known answers for the three rules on hand-written programs."""
import os
import shutil
import subprocess
import sys
import tempfile

import pytest

import demi_b200 as D
from demi_b200 import _native as N
import micro_oracle as M
import raft5_gen as G
from test_micro_oracle import flat, run_micro

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
ORACLE = os.path.join(ROOT, "oracle")
R = N.MODEL_RAFT5

CORPUS = ([G.generate(s, "forged") for s in range(80)] + [G.generate(s, "timer") for s in range(48)]
          + [G.generate(s, "clean") for s in range(16)] + [G.generate(s, "hardkill") for s in range(16)])


def _depth(p):
    return (50, 100)[p.seed % 2], (0, 5, 30)[p.seed % 3], p.seed % 4


def test_micro_oracle_matches_the_c_oracle_on_generated_programs(oracle):
    """Verdict, steps, node and event counts and max pending on every seed; the whole EventTrace and the DepTracker tree
    on every 10th, with FullyRandom and SrcDstFIFO (HardKill runs on FullyRandom only) and model flags 0-3."""
    k = 0
    n_viol = n_progs = 0
    for p in CORPUS:
        maxm, interval, flags = _depth(p)
        ext = D.pack_externals(p.events)
        for strategy in ((0,) if p.family == "hardkill" else (0, 1)):
            seeds = [1 + 7 * p.seed + j for j in range(6)]
            res = oracle.fuzz_batch(R, ext, seeds[0], len(seeds), maxm, interval, model_flags=flags, strategy=strategy)
            for j, seed in enumerate(seeds):
                ex, v = run_micro(R, p.events, seed, maxm, interval, flags, strategy=strategy)
                r = res[j]
                assert (int(r["violation"]), int(r["steps"]), int(r["n_nodes"]), int(r["n_events"]), int(r["max_pending"]),
                        int(r["status"])) == (v, ex.messagesScheduledSoFar, ex.depTracker.next_id, len(ex.events),
                                              ex.max_pending, 0), (p, strategy, seed)
                n_viol += bool(v)
                if k % 10 == 0:
                    ev, par, _ = oracle.fuzz_trace(R, ext, seed, maxm, interval, model_flags=flags, strategy=strategy)
                    got = [(int(e["kind"]), int(e["src"]), int(e["dst"]), int(e["type"]), int(e["p0"]), int(e["p1"]),
                            int(e["uniq"]), int(e["node"])) for e in ev]
                    rows = flat(ex.events)
                    assert got == rows, (p, strategy, seed, next((i for i in range(min(len(got), len(rows))) if got[i] != rows[i]), -1))
                    assert [int(x) for x in par] == [ex.depTracker.parent_of[i] for i in range(ex.depTracker.next_id)], (p, seed)
                k += 1
            n_progs += 1
    assert n_progs >= 150 and n_viol > 0


def test_corpus_reaches_the_handlers(oracle):
    """The corpus is not vacuous: deliveries from deadLetters of every type 3-8 reach booted actors, forged
    AppendEntries break state-machine safety without a seeded bug (code 2 at model flag 0), and some actor reaches term
    255.  Election safety (code 1) needs the double-vote bug: under R2 a VOTE_REPLY from deadLetters counts for nothing
    and under R3 a vote granted to deadLetters is not a vote, so no forged message gives one voter two votes in a term."""
    delivered_types, codes, top_term = set(), {0: set(), 1: set()}, 0
    for p in CORPUS:
        if p.family == "hardkill":
            continue
        ext = D.pack_externals(p.events)
        for flags in (0, 1):
            res = oracle.fuzz_batch(R, ext, 1, 1000, 100, 5, model_flags=flags)
            codes[flags] |= set(int(c) for c in res["violation"])
        ev, _, _ = oracle.fuzz_trace(R, ext, 1, 100, 5)
        booted, external = set(), set()
        for e in ev:
            if int(e["kind"]) == N.EV_MSG_SEND and int(e["src"]) == 0xFF:   # timers are recorded from "Timer" (0xFE)
                external.add(int(e["uniq"]))
            if int(e["kind"]) == N.EV_MSG_EVENT and int(e["uniq"]) in external:
                if int(e["type"]) == G.BOOT:
                    booted.add(int(e["dst"]))
                elif int(e["dst"]) in booted:
                    delivered_types.add(int(e["type"]))
        ex, _ = run_micro(R, p.events, 1, 100, 5, 0)
        top_term = max([top_term] + [a.term for a in ex.actors.values()])
    assert set(range(3, 9)) <= delivered_types, delivered_types
    assert 2 in codes[0] and 1 not in codes[0] and 1 in codes[1], codes
    assert top_term == 255


def test_timer_family_flushes_timer_keyed_externals(oracle):
    """The timer family's timer-keyed Sends are flushed in some programs (the lane engine hands those executions over)
    and not in others (the segment holding them is never reached), so a batch over the family runs on both engines."""
    flushed = []
    for p in CORPUS:
        if p.family != "timer":
            continue
        keys = set((e.a, e.type) for e in p.timer_keyed)
        ev, _, _ = oracle.fuzz_trace(R, D.pack_externals(p.events), 1, 50, 5)
        flushed.append(any(int(e["kind"]) == N.EV_MSG_SEND and int(e["src"]) == 0xFF and int(e["p0"]) == 0 and
                           int(e["p1"]) == 0 and (int(e["dst"]), int(e["type"])) in keys for e in ev))
    assert any(flushed) and not all(flushed)


# ------------------------------------------------------------------------------------------- the rules, known answers
def _boot_all(actors):
    return [D.Start(a) for a in range(5)] + [D.Send(a, G.BOOT, 0x1F) for a in actors]


def test_r1_no_reply_to_dead_letters(oracle):
    """An external REQUEST_VOTE (granted or not) and external APPEND_ENTRIES (accepted, rejected, stale) are handled
    but answered with nothing: no MsgSend to 255, and the node count of a program whose forged message is replaced by
    one that sends nothing (a CLIENT_CMD to a follower)."""
    forged = [(G.REQUEST_VOTE, 3 | (9 << 8) | (255 << 16)), (G.REQUEST_VOTE, 0), (G.APPEND_ENTRIES, 3),
              (G.APPEND_ENTRIES, 3 | (5 << 8)), (G.APPEND_ENTRIES, 0)]
    for ty, p0 in forged:
        for ignore in (1, 0):
            prog = _boot_all([0]) + [D.Send(0, ty, p0, 1), D.WaitQuiescence()]
            quiet = _boot_all([0]) + [D.Send(0, G.CLIENT_CMD, 5), D.WaitQuiescence()]
            for seed in range(1, 40):
                ev, _, r = oracle.fuzz_trace(R, D.pack_externals(prog), seed, 30, 0, ignore_timers=ignore)
                assert not any(int(e["dst"]) == 0xFF for e in ev if int(e["kind"]) in (N.EV_MSG_SEND, N.EV_MSG_EVENT))
                _, _, q = oracle.fuzz_trace(R, D.pack_externals(quiet), seed, 30, 0, ignore_timers=ignore)
                if ignore:
                    assert int(r["n_nodes"]) == int(q["n_nodes"]) == 3, (ty, seed)
                assert int(r["status"]) == 0


def _elected_leader():
    """Actor 0 elected by 1 and 2 in term 1 (no timers: an ELECTION_TICK with a payload starts the election), 3 and 4
    never booted.  With timers ignored the execution quiesces in the same final state under every schedule."""
    return [D.Start(a) for a in range(5)] + [D.Send(a, G.BOOT, 0x1F) for a in (0, 1, 2)] + \
           [D.WaitQuiescence(), D.Send(0, G.ELECTION_TICK, 7), D.WaitQuiescence()]


class _Ctx(object):
    """What a RaftActor may do inside receive(), recorded."""

    def __init__(self):
        self.ops = []

    def send(self, dst, msg):
        self.ops.append(("send", dst, msg))

    def schedule_repeating(self, msg):
        self.ops.append(("schedule", msg))

    def cancel(self, msg):
        self.ops.append(("cancel", msg))


def _final(oracle, prog, seeds=range(1, 30), flags=0):
    ext = D.pack_externals(prog)
    res = oracle.fuzz_batch(R, ext, seeds[0], len(seeds), -1, 0, model_flags=flags, ignore_timers=1)
    assert (res["status"] == 0).all()
    return res


def test_r2_vote_reply_from_dead_letters_never_elects(oracle):
    """A candidate that receives granted VOTE_REPLYs of its term from deadLetters stays a candidate: its final state
    equals the run without them; a VOTE_REPLY of a higher term applies the term rule only."""
    cand = [D.Start(a) for a in range(5)] + [D.Send(0, G.BOOT, 0x1F), D.WaitQuiescence(), D.Send(0, G.ELECTION_TICK, 7),
                                             D.WaitQuiescence()]
    votes = cand + [D.Send(0, G.VOTE_REPLY, 1 | (1 << 8) | (k << 12)) for k in range(4)] + [D.WaitQuiescence()]
    for flags in range(4):
        base = _final(oracle, cand, flags=flags)
        assert len(set(base["state_hash"].tolist())) == 1
        got = _final(oracle, votes, flags=flags)
        assert (got["state_hash"] == base["state_hash"][0]).all() and (got["violation"] == 0).all()
    a, ctx = M.RaftActor(0, 0), _Ctx()
    a.receive(ctx, M.DEADLETTERS, (G.BOOT, 0x1F, 0))
    a.receive(ctx, M.DEADLETTERS, (G.ELECTION_TICK, 7, 0))
    for k in range(4):
        a.receive(ctx, M.DEADLETTERS, (G.VOTE_REPLY, 1 | (1 << 8) | (k << 12), 0))
    assert (a.role, a.term, a.votes) == (M.CANDIDATE, 1, {0})
    a.receive(ctx, M.DEADLETTERS, (G.VOTE_REPLY, 9, 0))               # a higher term: the term rule still applies
    assert (a.role, a.term, a.voted, a.votes) == (M.FOLLOWER, 9, None, set())


def test_r2_append_reply_from_dead_letters_applies_the_term_rule_only(oracle):
    """An APPEND_REPLY from deadLetters to a leader changes nothing of its term or below (ok or not, any match index),
    and at a higher term does exactly what a VOTE_REPLY of that term does: step down."""
    lead = _elected_leader()
    base = _final(oracle, lead)
    assert len(set(base["state_hash"].tolist())) == 1
    ev, _, _ = oracle.fuzz_trace(R, D.pack_externals(lead), 1, -1, 0, ignore_timers=1)
    assert sum(int(e["kind"]) == N.EV_MSG_SEND and int(e["type"]) == G.APPEND_ENTRIES for e in ev) == 4   # it leads
    a, ctx = M.RaftActor(0, 0), _Ctx()
    a.role, a.term, a.log, a.next, a.match = M.LEADER, 1, [(1, 0x80)], [0] * 5, [0, 1, 0, 0, 0]
    for p0 in (1 | (1 << 8) | (5 << 16), 1 | (1 << 8) | (255 << 16), 1):
        a.receive(ctx, M.DEADLETTERS, (G.APPEND_REPLY, p0, 0))
    assert (a.role, a.commit, a.next, a.match, ctx.ops) == (M.LEADER, 0, [0] * 5, [0, 1, 0, 0, 0], [])
    a.receive(ctx, M.DEADLETTERS, (G.APPEND_REPLY, 2 | (1 << 8), 0))
    assert (a.role, a.term, ctx.ops) == (M.FOLLOWER, 2, [("cancel", (G.HEARTBEAT_TICK, 0, 0))])
    for p0 in (1 | (1 << 8) | (5 << 16), 1 | (1 << 8) | (255 << 16), 1, 0 | (1 << 8) | (8 << 16)):
        got = _final(oracle, lead + [D.Send(0, G.APPEND_REPLY, p0), D.WaitQuiescence()])
        assert (got["state_hash"] == base["state_hash"][0]).all(), hex(p0)
    for t in (2, 255):
        up = _final(oracle, lead + [D.Send(0, G.APPEND_REPLY, t | (1 << 8) | (3 << 16)), D.WaitQuiescence()])
        vr = _final(oracle, lead + [D.Send(0, G.VOTE_REPLY, t | (1 << 8)), D.WaitQuiescence()])
        assert (up["state_hash"] != base["state_hash"][0]).all() and (up["state_hash"] == vr["state_hash"]).all()


def test_r3_granted_vote_to_dead_letters(oracle):
    """A REQUEST_VOTE from deadLetters may be granted: VOTED holds 0xFF (none), so the actor can vote again in that term,
    and HEARD is set."""
    prog = [D.Start(a) for a in range(5)] + [D.Send(0, G.BOOT, 0x1F), D.Send(1, G.BOOT, 0x1F), D.WaitQuiescence(),
                                             D.Send(0, G.REQUEST_VOTE, 1), D.WaitQuiescence(),
                                             D.Send(1, G.ELECTION_TICK, 7), D.WaitQuiescence()]
    for seed in range(1, 20):                                   # the later candidate 1 still gets actor 0's vote in term 1
        ev, _, _ = oracle.fuzz_trace(R, D.pack_externals(prog), seed, -1, 0, ignore_timers=1)
        vr = [e for e in ev if int(e["kind"]) == N.EV_MSG_SEND and int(e["type"]) == G.VOTE_REPLY]
        assert [(int(e["src"]), int(e["dst"]), int(e["p0"])) for e in vr] == [(0, 1, 1 | (1 << 8))]
    a, ctx = M.RaftActor(0, 0), _Ctx()
    a.receive(ctx, M.DEADLETTERS, (G.BOOT, 0x1F, 0))
    a.receive(ctx, M.DEADLETTERS, (G.REQUEST_VOTE, 1, 0))
    assert (a.term, a.voted, a.heard) == (1, None, True) and ctx.ops == [("schedule", (G.ELECTION_TICK, 0, 0))]
    a.receive(ctx, "1", (G.REQUEST_VOTE, 1, 0))
    assert a.voted == 1 and ctx.ops[-1] == ("send", "1", (G.VOTE_REPLY, 1 | (1 << 8), 0))


# ----------------------------------------------------------------------------------------------------- sanitizers
SAN_FLAGS = ["-O1", "-g", "-fno-omit-frame-pointer", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
             "-fPIC", "-shared", "-std=gnu11", "-pthread"]
ORACLE_SRCS = ["machine.c", "models.c", "model_ir.c", "fuzz.c", "ddmin.c", "sts.c", "dpor.c", "dpor_frontier.c",
               "intmin.c", "provenance.c", "campaign.c"]

SAN_DRIVER = r"""
import ctypes as C, sys
sys.path[:0] = [%(root)r, %(tests)r]
from oracle import binding as O, campaign_binding as CB
lib = C.CDLL(%(so)r)
lib.oracle_fuzzer_generate.restype = C.c_uint32
lib.oracle_set_user_filter.restype = None
O._lib = CB._lib = lib
import demi_b200 as D
import raft5_gen as G
R = 2
for fam, n in (("forged", 40), ("timer", 24), ("clean", 8), ("hardkill", 8)):
    for p in G.corpus(n, fam):
        ext = D.pack_externals(p.events)
        for strategy in ((0,) if fam == "hardkill" else (0, 1)):
            for flags in range(4):
                O.fuzz_batch(R, ext, 1, 24, 60, 5, model_flags=flags, strategy=strategy, threads=2)
            O.fuzz_trace(R, ext, 3, 60, 5, model_flags=p.seed %% 4, strategy=strategy)
pre = D.pack_externals(D.raft5_program()[:-1])
for send_type in (4, 5, 7, 8):
    cfg = CB.FuzzerConfig(0.02, 0.6, 0.05, 0.05, 0.05, 30, send_type)
    CB.fuzz_campaign(R, cfg, pre, None, 1, 200, 60, 5, 9, model_flags=send_type %% 4, threads=2)
print("clean")
"""


def _sanitizer_runtimes():
    cc = shutil.which("gcc")
    if not cc:
        return None
    libs = []
    for name in ("libasan.so", "libubsan.so"):
        path = subprocess.run([cc, "-print-file-name=" + name], capture_output=True, text=True).stdout.strip()
        if not os.path.isabs(path) or not os.path.exists(path):
            return None
        libs.append(path)
    return cc, libs


def build_sanitized_oracle(src_dir, out_dir):
    """The oracle (with the campaign loop) compiled with ASan + UBSan into out_dir; None if the compiler cannot."""
    found = _sanitizer_runtimes()
    if not found:
        return None
    cc, _ = found
    so = os.path.join(out_dir, "liboracle_san.so")
    r = subprocess.run([cc] + SAN_FLAGS + ["-o", so] + [os.path.join(src_dir, s) for s in ORACLE_SRCS],
                       capture_output=True, text=True)
    return so if r.returncode == 0 else None


def run_sanitized(so, root=ROOT):
    _, libs = _sanitizer_runtimes()
    env = dict(os.environ, LD_PRELOAD=":".join(libs), ASAN_OPTIONS="detect_leaks=0:halt_on_error=1:abort_on_error=0",
               UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    script = SAN_DRIVER % {"root": root, "tests": os.path.join(root, "tests"), "so": so}
    return subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, env=env, timeout=1800)


def test_oracle_under_sanitizers_on_generated_programs():
    """The generated corpus through oracle_fuzz_batch and oracle_fuzz_trace (both strategies, flags 0-3) and raft5
    campaigns whose generated Sends are REQUEST_VOTE, VOTE_REPLY, APPEND_ENTRIES and APPEND_REPLY, with every
    AddressSanitizer or UndefinedBehaviorSanitizer report fatal."""
    if _sanitizer_runtimes() is None:
        pytest.skip("the C compiler has no AddressSanitizer / UndefinedBehaviorSanitizer runtimes")
    with tempfile.TemporaryDirectory() as tmp:
        so = build_sanitized_oracle(ORACLE, tmp)
        if so is None:
            pytest.skip("the C compiler cannot build with -fsanitize=address,undefined")
        r = run_sanitized(so)
    report = r.stderr[-4000:]
    assert "runtime error" not in r.stderr and "AddressSanitizer" not in r.stderr, report
    assert r.returncode == 0 and r.stdout.strip().endswith("clean"), report
