"""The steady raft5 lane kernel with 8-byte pending rows (the ROW8 flavour, demi_b200/csrc/lane_steady.hpp) against
the CPU oracle.

A steady raft5 batch runs ROW8 when the host can prove that every row it creates fits the 8-byte layout: every row of
the program's snapshot (its external Sends) fits, and no DepTracker node reaches 2^12.  Otherwise it runs the 16-byte
steady kernel.  demi_lane_row_bytes says which ran, so that a silent fall-back to either fails here.  Every result field
is compared per seed with the oracle."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
import raft5_gen as G

pytestmark = pytest.mark.gpu

FIELDS = ["violation", "steps", "state_hash", "trace_hash", "n_nodes", "n_events", "max_pending", "status"]
R = N.MODEL_RAFT5
BOOT, CLIENT_CMD, REQUEST_VOTE, VOTE_REPLY, APPEND_ENTRIES, APPEND_REPLY = 1, 2, 4, 5, 7, 8
EDGE = 583           # the largest maxMessages whose nodes fit 12 bits on raft5_program(): 6 + 584 * 7 <= 4096


@pytest.fixture(autouse=True)
def lane_engine(monkeypatch):
    monkeypatch.delenv("DEMI_DISABLE_LANE_ENGINE", raising=False)
    monkeypatch.delenv("DEMI_LANE_PENDING_CAP", raising=False)


def assert_same(a, b, what):
    for f in FIELDS:
        bad = np.nonzero(a[f] != b[f])[0]
        assert len(bad) == 0, "%s: field %s differs at %d prefixes, first idx %d: %s vs %s" % (
            what, f, len(bad), bad[0], a[bad[0]], b[bad[0]])


def run(oracle, events, n, maxm, interval, flags=1, seed=1):
    """The batch on the device and on the oracle; returns the device's records, the lane kernel and its row bytes."""
    ext = D.pack_externals(events)
    eng = D.Engine(D.SchedulerConfig(R, model_flags=flags))
    eng.set_externals(ext)
    got = eng.fuzz_batch(seed, n, maxm, interval)
    kernel, row = eng.lane_kernel(), eng.lane_row_bytes()
    eng.close()
    cpu = oracle.fuzz_batch(R, ext, seed, n, maxm, interval, model_flags=flags)
    assert_same(got, cpu, "maxm %d interval %d flags %d" % (maxm, interval, flags))
    return got, kernel, row


def boots():
    return [D.Start(a) for a in range(5)] + [D.Send(a, BOOT, 0x1F) for a in range(5)]


PROGRAMS = {
    "bench": lambda: D.raft5_program(),
    "clients-3": lambda: D.raft5_program(client_cmds=3),
    "clients-11": lambda: D.raft5_program(client_cmds=11),
    "partial-boot": lambda: [D.Start(a) for a in range(5)] + [D.Send(a, BOOT, 0x1F) for a in (0, 1, 2, 4)] +
                            [D.WaitQuiescence()],
}


@pytest.mark.parametrize("interval", [0, 1, 5])
@pytest.mark.parametrize("name", sorted(PROGRAMS))
def test_programs_run_row8(oracle, name, interval):
    for flags in (1, 0):
        _, kernel, row = run(oracle, PROGRAMS[name](), 20000, 50, interval, flags=flags, seed=3 + interval)
        assert (kernel, row) == (N.LANE_STEADY, 8)


def test_bench_workload(oracle):
    got, kernel, row = run(oracle, D.raft5_program(), 100_003, 50, 5, seed=10_000_001)
    assert (kernel, row) == (N.LANE_STEADY, 8)
    assert (got["status"] == 0).all()


def test_node_bound_edge(oracle):
    """maxMessages EDGE packs and EDGE + 1 does not: the 16-byte kernel runs it, with the same records wherever no
    execution reaches EDGE deliveries."""
    for flags, interval in ((1, 5), (3, 1)):
        a, ka, ra = run(oracle, D.raft5_program(), 4000, EDGE, interval, flags=flags, seed=21)
        b, kb, rb = run(oracle, D.raft5_program(), 4000, EDGE + 1, interval, flags=flags, seed=21)
        assert (ka, ra) == (N.LANE_STEADY, 8) and (kb, rb) == (N.LANE_STEADY, 16)
        short = a["steps"] < EDGE
        assert short.any()
        for f in FIELDS:
            assert np.array_equal(a[f][short], b[f][short]), f


# external protocol messages after the bootstraps: (type, p0, p1), and whether the layout holds them
EXTERNALS = [
    ((APPEND_ENTRIES, 3 | 8 << 8 | 2 << 16 | 8 << 24, 1 | 2 << 8 | 0x80 << 16), 8),
    ((APPEND_ENTRIES, 1 | 15 << 8 | 255 << 16 | 15 << 24, 1 | 255 << 8 | 255 << 16), 8),
    ((APPEND_ENTRIES, 3 | 16 << 8, 0), 16),                  # prev in 4 bits
    ((APPEND_ENTRIES, 3 | 2 << 8, 2), 16),                   # p1 byte 0 in 1 bit
    ((APPEND_REPLY, 2 | 1 << 8 | 200 << 16, 0), 8),          # a deadLetters matchIndex is only a byte: NEXT never takes it
    ((REQUEST_VOTE, 255 | 9 << 8 | 255 << 16, 0), 8),
    ((REQUEST_VOTE, 2 | 1 << 8 | 1 << 16 | 1 << 28, 0), 16),  # junk in p0 byte 3
    ((VOTE_REPLY, 2 | 1 << 8, 1 << 24), 16),                 # junk in p1 byte 3
    ((CLIENT_CMD, 0x7F, 0), 8),
    ((CLIENT_CMD, 0xFFFFFFFF, 0), 16),
]


@pytest.mark.parametrize("i", range(len(EXTERNALS)))
def test_external_protocol_messages(oracle, i):
    (ty, p0, p1), want = EXTERNALS[i]
    events = boots() + [D.Send(i % 5, ty, p0, p1), D.WaitQuiescence()]
    for flags, interval in ((1, 5), (0, 0), (3, 1)):
        _, kernel, row = run(oracle, events, 20000, 50, interval, flags=flags, seed=7 + i)
        assert (kernel, row) == (N.LANE_STEADY, want)


def test_generated_programs(oracle):
    """raft5_gen's one-segment programs: forged payloads at the handlers' edges, with junk in the bits they ignore.
    A steady launch runs ROW8 exactly when every Send's payload leaves the layout's header and node bits clear."""
    steady = 0
    for family in ("clean", "forged", "timer"):
        for p in G.corpus(40, family, base=500):
            if sum(isinstance(e, D.WaitQuiescence) for e in p.events) != 1 or \
                    any(isinstance(e, (D.Kill, D.Partition, D.UnPartition, D.HardKill)) for e in p.events):
                continue
            _, kernel, row = run(oracle, p.events, 3000, 50, 5, flags=p.seed % 4, seed=p.seed)
            if kernel == N.LANE_STEADY:
                steady += 1
                fits = all((e.p0 & ~0x0FFF0FFF) == 0 and (e.p1 & ~0x00FFFF01) == 0
                           for e in p.events if isinstance(e, D.Send))
                assert row == (8 if fits else 16), p
    assert steady > 0
