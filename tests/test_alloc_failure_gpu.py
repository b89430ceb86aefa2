"""Device allocations that fail, made to fail on the host side with DEMI_TEST_ALLOC_LIMIT (an allocation of more than
the limit fails as it would on a full device).  A setter that fails leaves the handle as it was: its next calls give
the records they gave before.  A call that cannot allocate its cached or per-call buffers returns DEMI_ERR_CUDA, and
the same call repeated on that handle gives what it gives on a fresh handle."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
from demi_b200 import model_ir
import ir_gen

pytestmark = pytest.mark.gpu

MAXM, INTERVAL = 50, 5                 # raft5 with model_flags = 1, as the benchmark runs it
LIMIT = "DEMI_TEST_ALLOC_LIMIT"


def under_limit(monkeypatch, limit, call):
    """call() with every device allocation above `limit` bytes failing: its result, or the DemiError it raised."""
    monkeypatch.setenv(LIMIT, str(limit))
    try:
        return call()
    except D.DemiError as e:
        return e
    finally:
        monkeypatch.delenv(LIMIT)


def fails(monkeypatch, limit, call):
    e = under_limit(monkeypatch, limit, call)
    assert isinstance(e, D.DemiError) and e.code == N.ERR_CUDA, e


def raft_engine(program=None):
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    eng.set_externals(D.raft5_program(client_cmds=6) if program is None else program)
    return eng


def full_mask(n):
    m = np.zeros((n + 63) // 64, dtype=np.uint64)
    for i in range(n):
        m[i >> 6] |= np.uint64(1) << np.uint64(i & 63)
    return m


def random_masks(n_bits, n, seed):
    rng = np.random.default_rng(seed)
    m = np.zeros((n, (n_bits + 63) // 64), dtype=np.uint64)
    for i in range(n_bits):
        m[:, i >> 6] |= rng.integers(0, 2, size=n, dtype=np.uint64) << np.uint64(i & 63)
    m[0] = full_mask(n_bits)
    return m


@pytest.fixture(scope="module")
def recorded():
    """Two executions of raft5_program(6) that violate the invariant: [(events, dep_parent, record)]."""
    eng = raft_engine()
    hits = np.nonzero(eng.fuzz_batch(1, 20000, MAXM, INTERVAL)["violation"])[0]
    assert len(hits) >= 2
    return [eng.fuzz_trace(1 + int(s), MAXM, INTERVAL) for s in hits[:2]]


# ---------------------------------------------------------------- setters
def test_set_externals_that_fails_keeps_the_program(monkeypatch):
    eng = raft_engine()
    want = eng.fuzz_batch(7, 4096, MAXM, INTERVAL)
    other = D.raft5_program(client_cmds=2)
    assert raft_engine(other).fuzz_batch(7, 4096, MAXM, INTERVAL).tobytes() != want.tobytes()
    fails(monkeypatch, 0, lambda: eng.set_externals(other))
    assert eng.fuzz_batch(7, 4096, MAXM, INTERVAL).tobytes() == want.tobytes()


def test_set_trace_that_fails_keeps_the_trace(monkeypatch, recorded):
    (ev, _, r), (ev2, _, _) = recorded
    ext = D.pack_externals(D.raft5_program(client_cmds=6))
    eng = raft_engine()
    eng.set_trace(ev, ext)
    masks = random_masks(len(ext), 512, 1)
    want = eng.replay_batch(masks, int(r["violation"]))
    trace_bytes = len(ev2) * N.EVENT_DTYPE.itemsize
    assert ev2.tobytes() != ev.tobytes() and len(ext) * N.EXT_DTYPE.itemsize < trace_bytes
    fails(monkeypatch, 0, lambda: eng.set_trace(ev2, ext))
    fails(monkeypatch, trace_bytes - 1, lambda: eng.set_trace(ev2, ext))      # the smaller buffers fit, the trace does not
    assert eng.replay_batch(masks, int(r["violation"])).tobytes() == want.tobytes()
    res, trace = eng.replay_trace(full_mask(len(ext)), looking_for=int(r["violation"]))
    assert res["violation"] == r["violation"] and len(trace) > 0


def test_set_fuzzer_that_fails_keeps_the_fuzzer(monkeypatch):
    eng = raft_engine()
    eng.set_fuzzer(N.FuzzerConfig(0.01, 0.3, 0.1, 0.1, 0.1, 40, 2), D.pack_externals(D.raft5_program()))
    want = eng.fuzz_campaign(1000, 2048, MAXM, INTERVAL, 55)
    other = N.FuzzerConfig(0.0, 0.5, 0.1, 0.0, 0.0, 10, 2)
    fails(monkeypatch, 0, lambda: eng.set_fuzzer(other, D.pack_externals(D.raft5_program(client_cmds=3))))
    assert eng.fuzz_campaign(1000, 2048, MAXM, INTERVAL, 55).tobytes() == want.tobytes()


def test_load_model_that_fails_keeps_the_model(monkeypatch):
    eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, model_flags=1 | (4 << 8)))
    eng.load_model(model_ir.pingpong3_blob())
    eng.set_externals(D.pingpong3_program(20))
    want = eng.fuzz_batch(1, 4096, -1, 3)
    fails(monkeypatch, 0, lambda: eng.load_model(ir_gen.generate(1).blob))
    assert eng.actor_name(0) == "A" and eng.actor_index("C") == 2
    assert eng.fuzz_batch(1, 4096, -1, 3).tobytes() == want.tobytes()


# ---------------------------------------------------------------- cached and per-call buffers
def traced_engine(recorded):
    ev, _, _ = recorded[0]
    eng = raft_engine()
    eng.set_trace(ev, D.pack_externals(D.raft5_program(client_cmds=6)))
    return eng


def dpor_programs():
    return [[D.Start(a) for a in order] + [D.Send(a, 1, 0x1F) for a in order[:3]] for order in ([0, 1, 2, 3, 4], [4, 2, 0, 3, 1])]


def frontier(e):
    F = e.frontier_params(30, 300, 16, explored_slots=1 << 16, pool_cap=1 << 16)
    r, viol, hashes = e.dpor_frontier(dpor_programs()[0], F)
    return r["interleavings"], r["violations"], r["deliveries"], r["status"], viol, hashes


def cases(recorded):
    """name -> (a handle ready for the call, the call)"""
    ev, par, r = recorded[0]
    code = int(r["violation"])
    n_ext = len(D.raft5_program(client_cmds=6))
    n_deliveries = int((ev["kind"] == N.EV_MSG_EVENT).sum())
    records = raft_engine().fuzz_batch(1, 5000, MAXM, INTERVAL)
    return {
        "fuzz_batch": (raft_engine, lambda e: e.fuzz_batch(3, 4096, MAXM, INTERVAL)),
        "fuzz_trace": (raft_engine, lambda e: e.fuzz_trace(5, MAXM, INTERVAL)),
        "replay_trace": (lambda: traced_engine(recorded), lambda e: e.replay_trace(full_mask(n_ext), looking_for=code)),
        "wildcard_replay_trace": (lambda: traced_engine(recorded),
                                  lambda e: e.wildcard_replay_trace(full_mask(n_deliveries), looking_for=code)),
        "provenance": (raft_engine, lambda e: e.provenance(ev, par, 1)),
        "fuzz_provenance": (raft_engine, lambda e: e.fuzz_provenance(1, np.arange(64), MAXM, INTERVAL)),
        "fuzz_traces": (raft_engine, lambda e: e.fuzz_traces(1, np.arange(64), MAXM, INTERVAL)),
        "random_test_trace": (raft_engine, lambda e: e.random_test_trace(full_mask(n_ext), 5, MAXM, INTERVAL)),
        "dedup_compact": (raft_engine, lambda e: e.dedup_compact(records, 0)),
        "dpor_batch": (raft_engine, lambda e: e.dpor_batch(dpor_programs(), 30, 200, cap_viol=8, want_hashes=True)),
        "dpor_frontier": (raft_engine, frontier),
    }


CASES = ["fuzz_batch", "fuzz_trace", "replay_trace", "wildcard_replay_trace", "provenance", "fuzz_provenance",
         "fuzz_traces", "random_test_trace", "dedup_compact", "dpor_batch", "dpor_frontier"]


def as_bytes(x):
    return b"|".join(as_bytes(y) for y in x) if isinstance(x, tuple) else np.asarray(x).tobytes()


@pytest.mark.parametrize("case", CASES)
def test_a_call_that_fails_to_allocate_leaves_a_working_handle(monkeypatch, recorded, case):
    make, call = cases(recorded)[case]
    want = as_bytes(call(make()))
    eng = make()
    fails(monkeypatch, 0, lambda: call(eng))
    for limit in (1 << 12, 1 << 20):        # some buffers fit, as a call that runs out of memory midway leaves them
        got = under_limit(monkeypatch, limit, lambda: call(eng))
        assert (got.code == N.ERR_CUDA) if isinstance(got, D.DemiError) else as_bytes(got) == want, (limit, got)
    assert as_bytes(call(eng)) == want
