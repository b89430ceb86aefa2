"""The device-resident entry points as the benchmark calls them: many calls on one handle, on a non-default stream,
results left in HBM.  K5/K4 dedup against numpy at probe-chain, grid-stride and scan-pass edges and on reused scratch;
demi_fuzz_batch_dev and demi_fuzz_summary_dev against the host path and the oracle, batch after batch, empty batches
included; demi_fuzz_batch's chunked host path against one device launch; demi_replay_batch_dev across the replay
table's generation reset and across traces of different table geometry."""
import numpy as np
import pytest
import torch

import demi_b200 as D
from demi_b200 import _native as N
from test_dedup_gpu import expected_unique
from test_replay_ddmin_gpu import random_masks

pytestmark = pytest.mark.gpu

UNIQUE, VIOLATING = 0, 1
REC = N.RESULT_DTYPE.itemsize
MAXM, INTERVAL = 50, 5                 # the benchmark's workload: raft5_program(), model_flags = 1
ONES = 0xFFFFFFFFFFFFFFFF              # the dedup table's empty-slot marker


def side_stream():
    """A non-default stream that sees everything queued so far on the current one (buffer fills, copies)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    return s


def to_device(arr):
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).reshape(-1).copy()).cuda()


def records_of(buf, n):
    return buf[:n * REC].cpu().numpy().view(N.RESULT_DTYPE)


def sums(rec):
    """What demi_fuzz_summary_dev reports for these records: (violating records, sum of steps)."""
    return int((rec["violation"] != 0).sum()), int(rec["steps"].sum(dtype=np.uint64))


# ---------------------------------------------------------------- K5 / K4: dedup and compaction
def random_records(rng, hashes, violation=None):
    """Records with every byte random except the given state hashes (and violation column)."""
    r = rng.integers(0, 256, size=(len(hashes), REC), dtype=np.uint8).view(N.RESULT_DTYPE).reshape(-1)
    r["state_hash"] = hashes
    if violation is not None:
        r["violation"] = violation
    return r


def random_keys(rng, n):
    return rng.integers(0, ONES, size=n, dtype=np.uint64)        # never the marker itself


def expected(res, mode):
    if mode == UNIQUE:
        return expected_unique(res)
    idx = np.nonzero(res["violation"])[0].astype(np.uint32)
    return res[idx], idx


def check_dedup(eng, res, mode):
    out, idx = eng.dedup_compact(res, mode)
    want, widx = expected(res, mode)
    assert idx.tobytes() == widx.tobytes(), (len(idx), len(widx))
    assert out.tobytes() == want.tobytes()
    return out, idx


def table_slots(n):
    """demi_dedup_compact_dev's table size: the smallest power of two >= 1024 and >= 2n."""
    slots = 1024
    while slots < 2 * n:
        slots <<= 1
    return slots


def dd_slot(keys, slots):
    """dd_slot (dedup_kernel.cuh): a key's home slot, with uint64 wrap-around."""
    k = np.asarray(keys, dtype=np.uint64)
    return ((k ^ (k >> np.uint64(29))) * np.uint64(0x9E3779B97F4A7C15) >> np.uint64(20)) & np.uint64(slots - 1)


@pytest.mark.parametrize("n", [512, 513])
def test_dedup_probe_chains_and_wraparound(n):
    slots = table_slots(n)
    assert slots == (1024 if n == 512 else 2048)
    rng = np.random.default_rng(n)
    cand = np.unique(random_keys(rng, 1 << 22))
    home = dd_slot(cand, slots)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5))
    # one chain of 300 distinct keys that all start probing at the same slot, each key at scattered indices
    chain = cand[home == slots // 3][:300]
    assert len(chain) == 300
    keys = rng.permutation(np.concatenate([chain, rng.choice(chain, n - len(chain))]))
    check_dedup(eng, random_records(rng, keys), UNIQUE)
    # keys homed at the last slot probe on from slot 0, where the keys homed at 0 and 1 compete with them
    wrap = np.concatenate([cand[home == slots - 1][:150], cand[home == 0][:50], cand[home == 1][:50]])
    assert len(wrap) == 250
    keys = rng.permutation(np.concatenate([wrap, rng.choice(wrap, n - len(wrap) - 2), [ONES, ONES]]))
    check_dedup(eng, random_records(rng, keys), UNIQUE)


def test_dedup_first_occurrence_under_contention():
    """More records than one grid-stride pass of the insert kernel (min(blocks, 8 per SM) blocks of 256): one key at
    every third index, keys drawn from a small pool elsewhere; the kept index is each key's first occurrence."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    n = 1_000_003
    assert n > 2 * sm * 8 * 256
    rng = np.random.default_rng(3)
    pool = random_keys(rng, 4096)
    keys = rng.choice(pool, n)
    hot = np.uint64(0x0123456789ABCDEF)
    keys[1::3] = hot
    res = random_records(rng, keys)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5))
    out, idx = check_dedup(eng, res, UNIQUE)
    assert idx[out["state_hash"] == hot].tolist() == [1]


SCAN_SIZES = sorted({256 * b - d for b in (1, 1023, 1024, 1025, 2048, 2049) for d in (0, 1)} | {1, 31, 32, 33, 255, 257})


@pytest.mark.parametrize("n", SCAN_SIZES)
def test_dedup_scan_passes_and_ragged_tails(n):
    """dedup_scan_kernel carries its sums across passes of 1024 block counts; the last block is partly empty."""
    rng = np.random.default_rng(n)
    res = random_records(rng, rng.choice(random_keys(rng, max(1, n // 2)), n))
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5))
    check_dedup(eng, res, UNIQUE)
    i = np.arange(n, dtype=np.uint32)
    for viol in (np.zeros(n, dtype=np.uint32), i % 5 + 1, i % 2):
        res["violation"] = viol
        check_dedup(eng, res, VIOLATING)


def test_dedup_scratch_reuse_on_one_handle():
    """The handle's table, flags and block counts only grow: a call after a larger one sees their stale contents."""
    rng = np.random.default_rng(11)

    def batch(n, distinct, violation=None):
        keys = rng.choice(random_keys(rng, distinct), n)
        keys[rng.choice(n, 3, replace=False)] = ONES
        return random_records(rng, keys, violation)

    calls = [(batch(700_001, 200_000), UNIQUE), (batch(1_000, 300), UNIQUE),
             (batch(50_000, 50_000, rng.integers(0, 3, 50_000)), VIOLATING), (batch(3_001, 1_000), UNIQUE)]
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5))
    for res, mode in calls:
        out, idx = check_dedup(eng, res, mode)
        fresh = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5))
        fo, fi = fresh.dedup_compact(res, mode)
        fresh.close()
        assert out.tobytes() == fo.tobytes() and idx.tobytes() == fi.tobytes()


def test_dedup_compact_dev_on_a_stream():
    rng = np.random.default_rng(5)
    n = 100_003
    keys = rng.choice(random_keys(rng, 30_000), n)
    keys[::997] = ONES
    res = random_records(rng, keys, rng.integers(0, 2, n))
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5))
    inp = to_device(res)
    out = torch.empty(n * REC, dtype=torch.uint8, device="cuda")
    idx = torch.empty(n, dtype=torch.int32, device="cuda")
    cnt = torch.empty(2, dtype=torch.int64, device="cuda")
    side = side_stream()
    for mode in (UNIQUE, VIOLATING):
        want, widx = eng.dedup_compact(res, mode)                    # the host wrapper
        assert widx.tobytes() == expected(res, mode)[1].tobytes()
        for with_index in (False, True):
            with torch.cuda.stream(side):
                cnt.fill_(-1)
                idx.fill_(-1)
                eng.dedup_compact_dev(inp.data_ptr(), n, mode, out.data_ptr(), idx.data_ptr() if with_index else 0,
                                      cnt.data_ptr(), side.cuda_stream)
            side.synchronize()
            c = cnt.cpu().numpy()
            assert c[0] == len(want) and c[1] == -1                   # one uint64 count, nothing written past it
            assert records_of(out, int(c[0])).tobytes() == want.tobytes()
            got_idx = idx.cpu().numpy()
            if with_index:
                assert got_idx[:c[0]].view(np.uint32).tobytes() == widx.tobytes()
            else:
                assert (got_idx == -1).all()                          # a NULL out_index is never written
    # indices are 32-bit: a larger n is refused before any buffer is read (the pointers here are never dereferenced)
    for mode in (UNIQUE, VIOLATING):
        with pytest.raises(D.DemiError) as e:
            eng.dedup_compact_dev(16, 1 << 32, mode, 16, 16, 16, side.cuda_stream)
        assert e.value.code == N.ERR_INVALID
    check_dedup(eng, res, UNIQUE)                                     # and the handle is still usable


# ---------------------------------------------------------------- K1: demi_fuzz_batch_dev and its counters
def raft5_engine():
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    eng.set_externals(D.pack_externals(D.raft5_program()))
    return eng


def run_dev(eng, seed, n, buf, side, maxm=MAXM, interval=INTERVAL):
    """One batch as bench.py runs it, then the summary read on the same stream (which waits for it)."""
    eng.fuzz_batch_dev(seed, n, maxm, interval, buf.data_ptr(), side.cuda_stream)
    summary = eng.fuzz_summary_dev(side.cuda_stream)
    return records_of(buf, n), summary


@pytest.mark.parametrize("lane_cap", [None, 24])
def test_bench_workload_on_a_stream(oracle, monkeypatch, lane_cap):
    """With a lane pending capacity of 24 some prefixes defer to the warp engine: the summary still counts each
    prefix once."""
    if lane_cap is not None:
        monkeypatch.setenv("DEMI_LANE_PENDING_CAP", str(lane_cap))
    n, seed = 100_003, 1
    eng = raft5_engine()
    buf = torch.empty(n * REC, dtype=torch.uint8, device="cuda")
    side = side_stream()
    rec, summary = run_dev(eng, seed, n, buf, side)
    st = eng.stats()
    host_eng = raft5_engine()
    host = host_eng.fuzz_batch(seed, n, MAXM, INTERVAL)
    assert rec.tobytes() == host.tobytes()
    cpu = oracle.fuzz_batch(N.MODEL_RAFT5, D.pack_externals(D.raft5_program()), seed, 20_000, MAXM, INTERVAL, model_flags=1)
    assert rec[:20_000].tobytes() == cpu.tobytes()
    assert summary == sums(rec) and summary[0] > 0
    assert (st.violations, st.deliveries) == summary
    assert st.prefixes == n and st.deferred == host_eng.stats().deferred
    if lane_cap is not None:
        assert 0 < st.deferred < n


def test_back_to_back_batches_report_their_own_counts():
    n1, n2 = 150_001, 30_011
    eng = raft5_engine()
    buf = torch.empty(n1 * REC, dtype=torch.uint8, device="cuda")
    side = side_stream()
    rec1, s1 = run_dev(eng, 1, n1, buf, side)
    assert s1 == sums(rec1) and eng.stats().prefixes == n1
    rec2, s2 = run_dev(eng, 5_000_000, n2, buf, side)
    assert s2 == sums(rec2) and eng.stats().prefixes == n2
    assert rec2.tobytes() == raft5_engine().fuzz_batch(5_000_000, n2, MAXM, INTERVAL).tobytes()
    assert records_of(buf, n1)[n2:].tobytes() == rec1[n2:].tobytes()      # past n2 the buffer is untouched


@pytest.mark.parametrize("entry", ["fuzz_batch_dev", "fuzz_batch", "fuzz_campaign_dev"])
def test_empty_batch_reports_zero_counts(monkeypatch, entry):
    monkeypatch.setenv("DEMI_LANE_PENDING_CAP", "12")                  # the batch before defers some prefixes
    n = 20_000
    eng = raft5_engine()
    if entry == "fuzz_campaign_dev":
        eng.set_fuzzer(N.FuzzerConfig(0.01, 0.3, 0.1, 0.1, 0.1, 40, 2), D.pack_externals(D.raft5_program()))
    buf = torch.empty(n * REC, dtype=torch.uint8, device="cuda")
    side = side_stream()

    def call(m):
        if entry == "fuzz_batch":
            eng.fuzz_batch(1, m, MAXM, INTERVAL, out=np.empty(max(m, 1), dtype=N.RESULT_DTYPE))
        elif entry == "fuzz_batch_dev":
            eng.fuzz_batch_dev(1, m, MAXM, INTERVAL, buf.data_ptr(), side.cuda_stream)
        else:
            eng.fuzz_campaign_dev(1, m, MAXM, INTERVAL, 7, buf.data_ptr(), side.cuda_stream)

    call(n)
    before = eng.fuzz_summary_dev(side.cuda_stream)
    st = eng.stats()
    assert before[0] > 0 and before[1] > 0 and st.prefixes == n and st.deferred > 0
    call(0)
    st = eng.stats()
    assert (st.prefixes, st.deliveries, st.violations, st.deferred) == (0, 0, 0, 0)
    assert eng.fuzz_summary_dev(side.cuda_stream) == (0, 0)
    st = eng.stats()
    assert (st.prefixes, st.deliveries, st.violations, st.deferred) == (0, 0, 0, 0)


@pytest.mark.parametrize("model,prog,maxm,interval,n", [
    (N.MODEL_PINGPONG3, lambda: D.pingpong3_program(12), -1, 0, 20_001),
    (N.MODEL_BCAST32, lambda: D.bcast32_program(2), 200, 0, 5_003),
], ids=["pingpong3", "bcast32"])
def test_other_lane_variants_on_a_stream(oracle, model, prog, maxm, interval, n):
    ext = D.pack_externals(prog())
    eng = D.Engine(D.SchedulerConfig(model))
    eng.set_externals(ext)
    buf = torch.empty(n * REC, dtype=torch.uint8, device="cuda")
    side = side_stream()
    rec, summary = run_dev(eng, 3, n, buf, side, maxm, interval)
    assert eng.stats().kernel_launches == 2               # the lane engine, then the warp engine on what it deferred
    host_eng = D.Engine(D.SchedulerConfig(model))
    host_eng.set_externals(ext)
    assert rec.tobytes() == host_eng.fuzz_batch(3, n, maxm, interval).tobytes()
    assert summary == sums(rec)
    cpu = oracle.fuzz_batch(model, ext, 3, 2000, maxm, interval)
    assert rec[:2000].tobytes() == cpu.tobytes()


# ---------------------------------------------------------------- demi_fuzz_batch's chunks
def test_chunked_host_path_matches_one_launch_and_oracle(oracle):
    """Past 2 * CHUNK prefixes demi_fuzz_batch runs ceil(n / CHUNK) equal chunks (CHUNK = 2^21), each with its own
    seed base, copying one to the host while the next runs."""
    chunk = 2 << 20
    n = 2 * chunk + 1
    per = -(-n // 3)
    assert per == 1_398_102
    seed = 11
    ext = D.pack_externals(D.raft5_program())
    eng = raft5_engine()
    host = eng.fuzz_batch(seed, n, MAXM, INTERVAL)
    st = eng.stats()
    assert st.prefixes == n and (st.violations, st.deliveries) == sums(host)
    buf = torch.empty(n * REC, dtype=torch.uint8, device="cuda")
    side = side_stream()
    eng.fuzz_batch_dev(seed, n, MAXM, INTERVAL, buf.data_ptr(), side.cuda_stream)
    side.synchronize()
    assert records_of(buf, n).tobytes() == host.tobytes()
    del buf
    for a, b in [(0, 1000), (per - 1000, per + 1000), (2 * per - 1000, 2 * per + 1000), (n - 1000, n)]:
        cpu = oracle.fuzz_batch(N.MODEL_RAFT5, ext, seed + a, b - a, MAXM, INTERVAL, model_flags=1)
        assert host[a:b].tobytes() == cpu.tobytes(), (a, b)


# ---------------------------------------------------------------- K2: replay table state across calls
def raft5_traces(oracle, client_cmds, count, maxm=MAXM):
    """The first `count` violating executions of raft5_program(client_cmds) as (externals, trace, violation)."""
    ext = D.pack_externals(D.raft5_program(client_cmds=client_cmds))
    res = oracle.fuzz_batch(N.MODEL_RAFT5, ext, 1, 20000, maxm, INTERVAL, model_flags=1)
    out = []
    for i in np.nonzero(res["violation"])[0][:count]:
        ev, _, r = oracle.fuzz_trace(N.MODEL_RAFT5, ext, 1 + int(i), maxm, INTERVAL, model_flags=1)
        out.append((ext, ev, int(r["violation"])))
    assert len(out) == count
    return out


def pow2_at_least(x, lo, hi):
    c = lo
    while c < x and c < hi:
        c <<= 1
    return c


def replay_table_slots(ev):
    """launch_replay's hash-table slots per test, from the trace's MsgSend count (demi_limits.h)."""
    pending_cap = pow2_at_least(int((ev["kind"] == N.EV_MSG_SEND).sum()) + 8, 64, 8192)
    return pow2_at_least(2 * pending_cap, 256, 1 << 16)


def oracle_replay(oracle, t, masks):
    ext, ev, code = t
    return oracle.replay_batch(N.MODEL_RAFT5, ev, ext, masks, looking_for=code, model_flags=1)


def test_replay_dev_past_the_generation_reset(oracle):
    """64 masks per call give each thread two generation stamps, so the 16-bit range runs out (and the table is
    cleared) about every 32 760 calls; 70 000 calls on one handle cross that point twice."""
    t = raft5_traces(oracle, 6, 1)[0]
    ext, ev, code = t
    masks = random_masks(ext, 64, 5, oracle)
    want = np.frombuffer(oracle_replay(oracle, t, masks).tobytes(), dtype=np.uint8)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    eng.set_trace(ev, ext)
    calls, row = 70_000, 64 * N.REPLAY_DTYPE.itemsize
    masks_dev = to_device(masks)
    out = torch.empty(calls * row, dtype=torch.uint8, device="cuda")
    side = side_stream()
    for k in range(calls):
        eng.replay_batch_dev(masks_dev.data_ptr(), 64, out.data_ptr() + k * row, code, 0, side.cuda_stream)
    side.synchronize()
    got = out.cpu().numpy().reshape(calls, row)
    bad = np.nonzero((got != want[None, :]).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), bad[:5])


@pytest.mark.parametrize("flags", [0, N.RF_FILTER_KNOWN_ABSENTS])
def test_replay_dev_on_a_stream_matches_host(oracle, flags):
    t = raft5_traces(oracle, 6, 1)[0]
    ext, ev, code = t
    masks = random_masks(ext, 3001, 8, oracle)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    eng.set_trace(ev, ext)
    host = eng.replay_batch(masks, code, flags)
    assert host.tobytes() == oracle.replay_batch(N.MODEL_RAFT5, ev, ext, masks, looking_for=code, flags=flags,
                                                 model_flags=1).tobytes()
    masks_dev = to_device(masks)
    out = torch.empty(len(masks) * N.REPLAY_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    side = side_stream()
    eng.replay_batch_dev(masks_dev.data_ptr(), len(masks), out.data_ptr(), code, flags, side.cuda_stream)
    side.synchronize()
    assert out.cpu().numpy().tobytes() == host.tobytes()


def test_replay_alternating_traces(oracle):
    """set_trace back and forth on one handle: between traces whose table geometry differs (the table is cleared on
    each switch) and between traces that share one (the generation stamps carry on over the other trace's entries)."""
    traces = [t for cc, maxm in ((6, 50), (30, 50), (30, 200), (30, 400)) for t in raft5_traces(oracle, cc, 2, maxm)]
    by_slots = {}
    for t in traces:
        by_slots.setdefault(replay_table_slots(t[1]), []).append(t)
    assert len(by_slots) >= 2                           # depth 50 traces use 256 slots, the longer ones 512 or 1024
    different = [by_slots[min(by_slots)][0], by_slots[max(by_slots)][0]]
    same = next(v for v in by_slots.values() if len(v) >= 2)[:2]
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    for pair in (different, same):
        inputs = []
        for k, t in enumerate(pair):
            masks = random_masks(t[0], 500, 20 + k, oracle)
            inputs.append((t, masks, oracle_replay(oracle, t, masks)))
        for rnd in range(3):
            for (ext, ev, code), masks, want in inputs:
                eng.set_trace(ev, ext)
                assert eng.replay_batch(masks, code).tobytes() == want.tobytes(), rnd
