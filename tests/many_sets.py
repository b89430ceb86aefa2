"""Deterministic sets of violating traces for the set entry points (demi_set_traces and the calls over a set), built on
the CPU oracle alone so that tests without a GPU can check what the GPU tests will run.

Each builder returns (traces, externals, codes): EVENT_DTYPE arrays, one EXT_DTYPE program per trace, and the code
each trace looks for.  `masks` draws the tests the two test files share."""
import numpy as np

import demi_b200 as D
from demi_b200 import _native as N
from oracle import binding as O

RAFT, PP, BC, IR = N.MODEL_RAFT5, N.MODEL_PINGPONG3, N.MODEL_BCAST32, N.MODEL_IR
RAFT_FLAGS, BC_FLAGS = 1, 3
PS_PENDING_OVF = 1                              # DEMI_PS_PENDING_OVF


def violating(model, ext, flags, maxm, interval, n, seeds, code=None, skip=0):
    """The first n violating executions (of `code` when given) among seeds 1..seeds: [(events, code)]."""
    res = O.fuzz_batch(model, ext, 1, seeds, maxm, interval, model_flags=flags)
    hit = (res["violation"] != 0) & (res["status"] == 0)
    if code is not None:
        hit &= res["violation"] == code
    out = []
    for k in np.nonzero(hit)[0][skip:skip + n]:
        ev, _, r = O.fuzz_trace(model, ext, 1 + int(k), maxm, interval, model_flags=flags)
        out.append((ev, int(r["violation"])))
    assert len(out) == n, (model, len(ext), n, len(out))
    return out


def strip_internal_sends(ev, external_types):
    """The trace without its internal MsgSends.  The replay sizes its pending set by the trace's MsgSends, so a short
    copy of a trace with many messages in flight overflows it where the full trace does not."""
    keep = (ev["kind"] != N.EV_MSG_SEND) | np.isin(ev["type"], list(external_types))
    return ev[keep].copy()


def masks(ext, n, rng):
    """n test masks over ext, each external kept with probability 0.95, 0.8 or 0.5; mask 0 keeps every external.  No
    bit is set at or past len(ext)."""
    mw = O.mask_words(len(ext))
    m = np.zeros((n, mw), dtype=np.uint64)
    p = rng.choice([0.95, 0.8, 0.5], size=n)
    keep = rng.random((n, len(ext))) < p[:, None]
    keep[0] = True
    for i in range(len(ext)):
        m[:, i >> 6] |= keep[:, i].astype(np.uint64) << np.uint64(i & 63)
    return m


def pad(m, ext, mw, rng):
    """m (rows of O.mask_words(len(ext)) words) widened to mw words, with random bits at and past len(ext)."""
    out = np.zeros((len(m), mw), dtype=np.uint64)
    out[:, :m.shape[1]] = m
    garbage = rng.integers(0, 1 << 64, size=out.shape, dtype=np.uint64, endpoint=False)
    n = len(ext)
    for w in range(mw):
        lo = w * 64
        if lo + 64 <= n:
            continue
        keep_low = np.uint64((1 << max(0, n - lo)) - 1)
        out[:, w] = (out[:, w] & keep_low) | (garbage[:, w] & ~keep_low)
    return out


# ---------------------------------------------------------------------------------------------------------- raft5
def raft5_variant(client_cmds):
    """A program as long as raft5_program(client_cmds) that starts the actors in the other order and sends other
    commands.  The replay reads Starts from the program and Sends from the trace, so a trace replayed against the
    other program of its length gives other records."""
    ev = [D.Start(a) for a in range(4, -1, -1)] + [D.Send(a, 1, 0x1F) for a in range(5)]
    ev += [D.Send((i + 2) % 5, 2, 50 + 3 * i) for i in range(client_cmds)]
    return ev + [D.WaitQuiescence()]


def raft5_mixed():
    """Violating raft5 executions of raft5_program(c) for c in 0, 6, 60, 120 (11, 17, 71 and 131 externals: 1, 1, 2
    and 3 mask words), of a variant program as long as c = 6's, a ~2 000-event execution (max_messages 1000) and short
    copies without internal MsgSends of four of them.  Codes 1 and 2 both occur, and trace 1 looks for 2, which its
    full replay does not show.  Longest first is not the input order."""
    traces, exts, codes = [], [], []

    def add(prog, maxm, n, code=None, skip=0):
        ext = D.pack_externals(prog)
        for ev, c in violating(RAFT, ext, RAFT_FLAGS, maxm, 5, n, 4000, code, skip):
            traces.append(ev)
            exts.append(ext)
            codes.append(c)

    add(D.raft5_program(0), 50, 3, code=1)
    add(D.raft5_program(0), 50, 1, code=2)
    add(D.raft5_program(6), 50, 3, code=1)
    add(raft5_variant(6), 50, 3)
    add(D.raft5_program(60), 200, 3)
    add(D.raft5_program(120), 200, 3)
    ext6 = D.pack_externals(D.raft5_program(6))
    res = O.fuzz_batch(RAFT, ext6, 1, 400, 1000, 5, model_flags=RAFT_FLAGS)
    ok = np.nonzero((res["violation"] != 0) & (res["status"] == 0))[0]
    k = int(ok[np.argmax(res["n_events"][ok])])
    ev, _, r = O.fuzz_trace(RAFT, ext6, 1 + k, 1000, 5, model_flags=RAFT_FLAGS)
    assert len(ev) > 1000
    traces.append(ev)
    exts.append(ext6)
    codes.append(int(r["violation"]))
    for t in (len(traces) - 1, 0, 12, 15):                       # the long one, c = 0, c = 60, c = 120
        traces.append(strip_internal_sends(traces[t], (1, 2)))
        exts.append(exts[t])
        codes.append(codes[t])
    codes[1] = 2
    return traces, exts, np.array(codes, dtype=np.uint32)


# --------------------------------------------------------------------------------------------- the other models
PP_FLAGS = 1 | (2 << 8)


def pingpong3_set():
    """Violations of pingpong3_program(n) (actor 0 has 2 pongs) for n in 8, 20, 64, 90: 12 to 94 externals."""
    traces, exts, codes = [], [], []
    for n in (8, 20, 64, 90):
        ext = D.pack_externals(D.pingpong3_program(n))
        for ev, c in violating(PP, ext, PP_FLAGS, -1, 3, 3, 200):
            traces.append(ev)
            exts.append(ext)
            codes.append(c)
    return traces, exts, np.array(codes, dtype=np.uint32)


def bcast32_set():
    """bcast32 executions of ttl 2 and 3 and their short copies without internal MsgSends, which overflow their
    pending set."""
    traces, exts, codes = [], [], []
    for ttl in (2, 3):
        ext = D.pack_externals(D.bcast32_program(ttl))
        full = violating(BC, ext, BC_FLAGS, 120, 10, 3, 200)
        for ev, c in full:
            traces += [ev, strip_internal_sends(ev, (2,))]
            exts += [ext, ext]
            codes += [c, c]
    return traces, exts, np.array(codes, dtype=np.uint32)


def election_set(n=8):
    """Violating executions (two leaders in one term) of the timer-driven election of test_ir_timers_oracle."""
    from test_ir_timers_oracle import ELECTION_INTERVAL, ELECTION_MAXM, election_model, election_program
    m = election_model()
    O.load_model(m.blob)
    ext = D.pack_externals(election_program())
    got = violating(IR, ext, m.flags, ELECTION_MAXM, ELECTION_INTERVAL, n, 400)
    return m, [g[0] for g in got], [ext] * n, np.array([g[1] for g in got], dtype=np.uint32)


def generated_timer_sets(seeds=range(1, 41), per=4, maxm=40, interval=3):
    """For each generated model of `seeds` that arms timers and has `per` violating executions of its program among
    64 seeds: (model, traces, externals, codes)."""
    import ir_gen
    out = []
    for s in seeds:
        m = ir_gen.generate(s)
        if not m.uses_timers:
            continue
        O.load_model(m.blob)
        ext = D.pack_externals(ir_gen.program(m, s, kills=False))
        res = O.fuzz_batch(IR, ext, 1, 64, maxm, interval, model_flags=m.flags)
        hits = np.nonzero((res["violation"] != 0) & (res["status"] == 0))[0][:per]
        if len(hits) < per:
            continue
        tr = [O.fuzz_trace(IR, ext, 1 + int(k), maxm, interval, model_flags=m.flags)[0] for k in hits]
        out.append((m, tr, [ext] * per, res["violation"][hits].astype(np.uint32)))
    return out
