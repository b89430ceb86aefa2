"""The inputs of tests/test_many_traces_edges_gpu.py on the CPU oracle: they show what the GPU tests rely on to fail
when a set call mixes up two traces.  Per-trace capacity statuses in short and full traces, violations of more than
one code, a code a trace looks for and does not show, switches that change the records, traces of 1, 2 and 3 mask
words, and the mask contract: bits at and past a trace's externals are ignored."""
import numpy as np

import demi_b200 as D
from demi_b200 import _native as N
import many_sets as S
from oracle import binding as O
from test_config_switches_gpu import K2_CASES          # the switch cases tests/test_many_traces_edges_gpu.py runs

def records(model, flags, traces, exts, codes, n=64, seed=0, **sw):
    rng = np.random.default_rng(seed)
    out = []
    for t in range(len(traces)):
        m = S.masks(exts[t], n, rng)
        out.append((m, O.replay_batch(model, traces[t], exts[t], m, looking_for=int(codes[t]), model_flags=flags, **sw)))
    return out


def test_raft5_mixed_set():
    traces, exts, codes = S.raft5_mixed()
    n_ev = np.array([len(t) for t in traces])
    assert {O.mask_words(len(e)) for e in exts} == {1, 2, 3}
    assert n_ev.max() > 1000 and np.argmax(n_ev) != 0                     # longest first is not the input order
    # two programs of one length that differ: a set must not share their externals
    lens = {}
    for e in exts:
        lens.setdefault(len(e), set()).add(e.tobytes())
    assert any(len(v) > 1 for v in lens.values())
    rec = records(S.RAFT, S.RAFT_FLAGS, traces, exts, codes)
    other = [t for t in range(len(traces)) if len(exts[t]) == len(exts[7]) and exts[t].tobytes() != exts[7].tobytes()]
    swapped = O.replay_batch(S.RAFT, traces[7], exts[other[0]], rec[7][0], looking_for=int(codes[7]), model_flags=S.RAFT_FLAGS)
    assert (swapped != rec[7][1]).sum() > len(swapped) // 4                # and that would show in the records
    st = [r["status"] for _, r in rec]
    short = [t for t in range(len(traces)) if (st[t] == S.PS_PENDING_OVF).any()]
    assert short and all((st[t] == 0).all() for t in range(len(traces)) if t not in short)
    long_t = int(np.argmax(n_ev))
    assert (st[long_t] == 0).all() and any(len(traces[t]) < len(traces[long_t]) for t in short)
    # codes 1 and 2 are both met; trace 1 looks for 2 and meets nothing, though it violates 1
    seen = set(int(v) for _, r in rec for v in r["violation"] if v)
    assert seen == {1, 2}
    assert codes[1] == 2 and (rec[1][1]["violation"] == 0).all()
    any_code = O.replay_batch(S.RAFT, traces[1], exts[1], rec[1][0], looking_for=0, model_flags=S.RAFT_FLAGS)
    assert (any_code["violation"] == 1).any()


def test_other_model_sets():
    traces, exts, codes = S.pingpong3_set()
    assert {O.mask_words(len(e)) for e in exts} == {1, 2} and max(len(e) for e in exts) > 64
    rec = records(S.PP, S.PP_FLAGS, traces, exts, codes)
    assert all((r["violation"] == 7).any() and (r["violation"] == 0).any() for _, r in rec)
    traces, exts, codes = S.bcast32_set()
    rec = records(S.BC, S.BC_FLAGS, traces, exts, codes)
    for t in range(0, len(traces), 2):                                     # full trace, then its short copy
        assert (rec[t][1]["status"] == 0).all() and (rec[t + 1][1]["status"] == S.PS_PENDING_OVF).any()
    m, traces, exts, codes = S.election_set()
    rec = records(S.IR, m.flags, traces, exts, codes)
    assert all((r["violation"] == 9).any() for _, r in rec)
    got = S.generated_timer_sets(range(1, 121))
    assert len(got) >= 3 and all(len(tr) == 4 for _, tr, _, _ in got)


def test_switches_change_the_records():
    for _, model, prog, flags, maxm, interval, blocked, it in K2_CASES:
        ext = D.pack_externals(prog)
        got = S.violating(model, ext, flags, maxm, interval, 4, 4000)
        traces, exts, codes = [g[0] for g in got], [ext] * 4, [g[1] for g in got]
        on = records(model, flags, traces, exts, codes, n=40, blocked_mask=blocked, ignore_timers=1 if it else 0)
        off = records(model, flags, traces, exts, codes, n=40)
        a = np.concatenate([r for _, r in on])
        b = np.concatenate([r for _, r in off])
        assert (a != b).sum() > len(a) // 4 and a["ignored"].sum() > b["ignored"].sum(), (model, blocked, it)


def test_garbage_mask_bits_are_ignored():
    """A mask with random bits at and past n_externals gives the clean mask's record, for every flag."""
    traces, exts, codes = S.raft5_mixed()
    rng = np.random.default_rng(5)
    for t in range(len(traces)):
        m = S.masks(exts[t], 32, rng)
        dirty = S.pad(m, exts[t], m.shape[1], rng)
        assert (dirty != m).any(axis=1).all()
        for fl in (0, N.RF_FILTER_KNOWN_ABSENTS, N.RF_STRICT):
            a = O.replay_batch(S.RAFT, traces[t], exts[t], m, looking_for=int(codes[t]), flags=fl, model_flags=S.RAFT_FLAGS)
            b = O.replay_batch(S.RAFT, traces[t], exts[t], dirty, looking_for=int(codes[t]), flags=fl, model_flags=S.RAFT_FLAGS)
            assert (a == b).all(), (t, fl)
        for i in range(0, 32, 8):
            ra, ea = O.replay_trace(S.RAFT, traces[t], exts[t], m[i], looking_for=int(codes[t]), model_flags=S.RAFT_FLAGS)
            rb, eb = O.replay_trace(S.RAFT, traces[t], exts[t], dirty[i], looking_for=int(codes[t]), model_flags=S.RAFT_FLAGS)
            assert ra == rb and len(ea) == len(eb) and (ea == eb).all(), (t, i)
