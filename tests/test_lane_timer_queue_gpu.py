"""messagesToSend in the lane fuzz kernel at its edges, against the warp engine alone and the CPU oracle.

The lane engine keeps messagesToSend as a 16-entry byte queue in registers: external Sends (0x80 | k) pushed at the
start of a segment, the re-send list and scheduled timers pushed around a delivery, Cancellable.cancel looking a slot
up in it, and the flush taking entries from the front.  The programs here fill the queue to exactly 16 entries and one
past it (the lane engine defers), put a flush item that defers in the middle of the queue (an external equal to a
timer key, a lowered lane pending capacity), ignore timers, and run raft5 leaders into forged higher-term messages so
that they step down and cancel their heartbeat while a re-send list or a fresh schedule is queued.  Every result field
is compared per seed, and the recorded traces of violating executions through their provenance masks."""
import random

import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
import raft5_gen as G

pytestmark = pytest.mark.gpu

FIELDS = ["violation", "steps", "state_hash", "trace_hash", "n_nodes", "n_events", "max_pending", "status"]
R, P, B = N.MODEL_RAFT5, N.MODEL_PINGPONG3, N.MODEL_BCAST32


def boots():
    return [D.Send(a, G.BOOT, 0x1F) for a in range(5)]


def clients(k, base=1):
    return [D.Send(i % 5, G.CLIENT_CMD, base + i) for i in range(k)]


def starts(n=5):
    return [D.Start(a) for a in range(n)]


def forged(seed, k):
    """k distinct protocol messages, half of them at the top terms 254 / 255, so that a leader steps down."""
    rng = random.Random(seed)
    out, seen = [], set()
    while len(out) < k:
        ty = rng.choice([G.REQUEST_VOTE, G.VOTE_REPLY, G.APPEND_ENTRIES, G.APPEND_REPLY])
        p0, p1 = G.payload(rng, ty)
        if rng.random() < 0.5:
            p0 = (p0 & ~0xFF) | rng.choice([254, 255])
        a = rng.randrange(5)
        if (a, ty, p0, p1) not in seen:
            seen.add((a, ty, p0, p1))
            out.append(D.Send(a, ty, p0, p1))
    return out


def interleave(xs, ys):
    out = []
    for i in range(max(len(xs), len(ys))):
        out += xs[i:i + 1] + ys[i:i + 1]
    return out


# name: (model, program, model_flags, max_messages, interval, n, ignore_timers, lane pending cap, every lane prefix defers)
CASES = {
    # 16 Sends in one segment: the queue is full at the first flush, and the lane engine keeps the execution
    "raft5-16-sends": (R, starts() + boots() + clients(11) + [D.WaitQuiescence()], 1, 50, 5, 10000, 0, None, False),
    # one more: the 17th push defers
    "raft5-17-sends": (R, starts() + boots() + clients(12) + [D.WaitQuiescence()], 1, 50, 5, 2000, 0, None, True),
    # an external equal to ELECTION_TICK(2)'s key as the 9th of 16 flush items: the flush defers there
    "raft5-timer-key-mid-flush": (R, starts() + boots() + clients(3) + [D.Send(2, G.ELECTION_TICK, 0, 0)]
                                  + clients(7, 10) + [D.WaitQuiescence()], 1, 50, 5, 2000, 0, None, True),
    # a lane pending capacity of 12: the 13th of 16 flush items defers
    "raft5-pending-cap-mid-flush": (R, starts() + boots() + clients(11) + [D.WaitQuiescence()],
                                    1, 50, 5, 2000, 0, 12, True),
    # timers ignored: no re-send list or scheduled timer ever enters the queue
    "raft5-16-sends-ignore-timers": (R, starts() + boots() + clients(11) + [D.WaitQuiescence()],
                                     1, -1, 0, 2000, 1, None, False),
    # forged higher-term messages among the BOOTs: leaders step down and cancel their heartbeat; long executions
    # without invariant checks let re-send lists grow
    "raft5-forged-stepdown-d100": (R, starts() + interleave(boots(), forged(1, 11)) + [D.WaitQuiescence()],
                                   0, 100, 0, 10000, 0, None, False),
    "raft5-forged-stepdown-bug-d100": (R, starts() + interleave(boots(), forged(2, 11)) + [D.WaitQuiescence()],
                                       1, 100, 5, 10000, 0, None, False),
    # a partition and a kill in a first segment of 16 Sends before the booting one
    "raft5-two-segments": (R, starts() + forged(3, 16) + [D.WaitQuiescence(), D.Partition(0, 1), D.Kill(3),
                                                           D.Start(3)] + boots() + clients(4) + [D.WaitQuiescence()],
                           1, 60, 5, 10000, 0, None, False),
    # pingpong3: 16 and 17 PINGs per segment
    "pingpong3-16-sends": (P, starts(3) + [D.Send(k % 3, 1, k) for k in range(16)] + [D.WaitQuiescence()]
                           + [D.Send(k % 3, 1, 100 + k) for k in range(16)] + [D.WaitQuiescence()],
                           0, -1, 0, 3000, 0, None, False),
    "pingpong3-17-sends": (P, starts(3) + [D.Send(k % 3, 1, k) for k in range(17)] + [D.WaitQuiescence()],
                           0, -1, 0, 1000, 0, None, True),
    "bcast32-ttl2": (B, D.bcast32_program(2), 0, 200, 0, 300, 0, None, False),
}


def assert_same(a, b, what):
    for f in FIELDS:
        bad = np.nonzero(a[f] != b[f])[0]
        assert len(bad) == 0, "%s: field %s differs at %d prefixes, first idx %d: %s vs %s" % (
            what, f, len(bad), bad[0], a[bad[0]], b[bad[0]])


def run(case, monkeypatch, warp_only):
    model, prog, flags, maxm, interval, n, ignore, lane_cap, _ = case
    monkeypatch.delenv("DEMI_DISABLE_LANE_ENGINE", raising=False)
    monkeypatch.delenv("DEMI_LANE_PENDING_CAP", raising=False)
    if warp_only:
        monkeypatch.setenv("DEMI_DISABLE_LANE_ENGINE", "1")
    elif lane_cap is not None:
        monkeypatch.setenv("DEMI_LANE_PENDING_CAP", str(lane_cap))
    eng = D.Engine(D.SchedulerConfig(model, model_flags=flags, ignoreTimers=bool(ignore)))
    eng.set_externals(D.pack_externals(prog))
    res = eng.fuzz_batch(1, n, maxm, interval)
    deferred = eng.stats().deferred
    eng.close()
    return res, deferred


@pytest.mark.parametrize("name", sorted(CASES))
def test_lane_and_warp_match_oracle(oracle, monkeypatch, name):
    case = CASES[name]
    model, prog, flags, maxm, interval, n, ignore, _, all_defer = case
    lane, deferred = run(case, monkeypatch, False)
    warp, _ = run(case, monkeypatch, True)
    cpu = oracle.fuzz_batch(model, D.pack_externals(prog), 1, n, maxm, interval, model_flags=flags,
                            ignore_timers=ignore)
    assert_same(lane, cpu, "lane+warp vs oracle")
    assert_same(warp, cpu, "warp alone vs oracle")
    assert (lane["status"] == 0).all()
    if all_defer:
        assert deferred == n                 # every execution handed over at the same queue edge
    else:
        assert deferred < n                  # the lane engine finished executions through the full queue


@pytest.mark.parametrize("name", ["raft5-16-sends", "raft5-forged-stepdown-bug-d100", "raft5-two-segments"])
def test_recorded_traces_match_oracle(oracle, monkeypatch, name):
    """The lane engine's recording instantiation on violating executions: trace hash, verdict and provenance masks."""
    model, prog, flags, maxm, interval, n, _, _, _ = CASES[name]
    monkeypatch.delenv("DEMI_DISABLE_LANE_ENGINE", raising=False)
    monkeypatch.delenv("DEMI_LANE_PENDING_CAP", raising=False)
    ext = D.pack_externals(prog)
    eng = D.Engine(D.SchedulerConfig(model, model_flags=flags))
    eng.set_externals(ext)
    res = eng.fuzz_batch(1, n, maxm, interval)
    idx = np.nonzero(res["violation"] != 0)[0][:24].astype(np.uint32)
    assert len(idx) >= 4
    keep, out, rec = eng.fuzz_provenance(1, idx, maxm, interval)
    assert np.array_equal(rec["trace_hash"], res["trace_hash"][idx])
    assert np.array_equal(rec["violation"], res["violation"][idx])
    for j, i in enumerate(idx):
        k, o = oracle.fuzz_provenance(model, ext, 1 + int(i), maxm, interval, keep.shape[1], model_flags=flags)
        assert o["status"] == out[j]["status"] == 0
        assert np.array_equal(k, keep[j]), int(i)
        for f in ("violation", "affected_mask", "n_trace", "n_kept"):
            assert o[f] == out[j][f], (f, int(i))
    eng.close()
