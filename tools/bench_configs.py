"""Secondary workloads of BASELINE.json (configs[2..4]) — one JSON line per config.
Not bench.py; its JSON lines can be kept under profiles/."""
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import demi_b200 as D
from demi_b200 import _native as N
from oracle import binding as O

HBM_PEAK = 6572.2
try:
    HBM_PEAK = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass


def cores():
    n = len(os.sched_getaffinity(0))
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(float(q) / float(p) + 0.5)))
    except Exception:
        pass
    return n


def config4_ddmin():
    """DDMin over a long violating raft5 trace with ~300 externals + a 10^6-mask replay batch."""
    prog = D.raft5_program(client_cmds=290)
    ext = D.pack_externals(prog)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    eng.set_externals(ext)
    # find an execution whose violation shows up late, so the recorded trace is long
    maxm, interval = 700, 100
    res = eng.fuzz_batch(1, 2_000_000, maxm, interval)
    hits = np.nonzero((res["violation"] == 1) & (res["steps"] >= 600))[0]
    seed = 1 + int(hits[0])
    ev, par, r = eng.fuzz_trace(seed, maxm, interval)
    code = int(r["violation"])
    eng.set_trace(ev, ext)
    mw = eng.mask_words()
    rng = np.random.default_rng(0)
    n = 1_000_000
    full = O.full_mask(ext)
    masks = rng.integers(0, 2**63, size=(n, mw), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=(n, mw), dtype=np.uint64)
    masks |= rng.integers(0, 2**63, size=(n, mw), dtype=np.uint64) * np.uint64(2)     # ~75 % dense
    masks &= full[None, :]
    masks[0] = full
    dm = torch.from_numpy(masks.view(np.int64)).cuda()
    dout = torch.empty(n * 16, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream()
    for _ in range(2):
        eng.replay_batch_dev(dm.data_ptr(), n, dout.data_ptr(), code, 0, st.cuda_stream)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(3):
        eng.replay_batch_dev(dm.data_ptr(), n, dout.data_ptr(), code, 0, st.cuda_stream)
    e1.record(st)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 3
    out = dout.cpu().numpy().view(N.REPLAY_DTYPE)
    t0 = time.perf_counter()
    host_out = eng.replay_batch(masks, code)
    e2e = time.perf_counter() - t0
    assert (host_out == out).all() and out[0]["violation"] == code
    nc = 4000 * cores()
    t0 = time.perf_counter()
    cpu = O.replay_batch(N.MODEL_RAFT5, ev, ext, masks[:nc], looking_for=code, model_flags=1, threads=cores())
    cdt = time.perf_counter() - t0
    assert (cpu == out[:nc]).all()
    t0 = time.perf_counter()
    mcs, iters, dd = eng.ddmin(code)
    ddt = time.perf_counter() - t0
    t0 = time.perf_counter()
    rc, cmcs, total, citers, ver = O.ddmin_sts(N.MODEL_RAFT5, ev, ext, code, model_flags=1)
    cddt = time.perf_counter() - t0
    assert (mcs == cmcs).all() and dd.total_replays == total and list(iters) == list(citers)
    alg_bytes = n * (mw * 8 + 16)
    return {"config": "configs[3]: DDMin over a %d-event violating raft5 trace, %d externals; 10^6 STSSched replays batched"
                      % (len(ev), len(ext)),
            "metric": "subsequence replays/s", "value": n / (ms * 1e-3), "e2e_value": n / e2e, "kernel_ms": ms,
            "reproduced": int((out["violation"] != 0).sum()),
            "roofline": {"bound": "hbm", "achieved": alg_bytes / (ms * 1e-3) / 1e9, "peak": HBM_PEAK,
                         "frac": alg_bytes / (ms * 1e-3) / 1e9 / HBM_PEAK, "algorithmic_bytes_per_test": mw * 8 + 16,
                         "note": "replay tests are latency/issue bound: the shared trace is L2-resident"},
            "cpu_baseline": {"value": nc / cdt, "cores": cores(), "kind": "port", "sample": "%d masks" % nc},
            "ddmin": {"externals": int(len(ext)), "mcs_size": int(dd.mcs_size), "sequential_tests": int(dd.total_replays),
                      "tests_executed_on_gpu": int(dd.replays_executed), "batches": int(dd.batches),
                      "verified": int(dd.verified), "gpu_seconds": ddt, "cpu_oracle_seconds": cddt,
                      "mcs_identical_to_sequential_oracle": True}}


def config3_dpor():
    """Independent DPORwHeuristics searches (depth 100), one per external subsequence."""
    rng = np.random.default_rng(7)
    progs = []
    for _ in range(int(os.environ.get("DEMI_C3_SEARCHES", "32768"))):
        ev = [D.Start(int(a)) for a in rng.permutation(5)]
        ev += [D.Send(int(a), 1, 0x1F) for a in rng.permutation(5)[:int(rng.integers(3, 6))]]
        ev += [D.Send(int(rng.integers(0, 5)), 2, int(rng.integers(1, 50))) for _ in range(int(rng.integers(0, 3)))]
        progs.append(ev)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=3))
    maxi = 200
    eng.dpor_batch(progs[:64], 100, 20, heap_cap=1 << 17)
    t0 = time.perf_counter()
    res, viol, _ = eng.dpor_batch(progs, 100, maxi, heap_cap=1 << 17)
    dt = time.perf_counter() - t0
    kms = eng.stats().kernel_ms
    il = int(res["interleavings"].sum())
    nc = 2 * cores()
    t0 = time.perf_counter()
    cil = 0
    for p in progs[:nc]:
        rc, r, _, _ = O.dpor_search(N.MODEL_RAFT5, D.pack_externals(p), 100, maxi, model_flags=3, node_cap=4096,
                                    explored_slots=1 << 16, heap_cap=1 << 17)
        cil += int(r["interleavings"])
    cdt = time.perf_counter() - t0
    return {"config": "configs[2]: raft5 DPORwHeuristics depth-100, %d independent searches x <=%d interleavings" % (len(progs), maxi),
            "metric": "interleavings/s", "value": il / (kms * 1e-3), "e2e_value": il / dt, "kernel_ms": kms,
            "interleavings": il, "deliveries": int(res["deliveries"].sum()), "races_analysed": int(res["races"].sum()),
            "violating_interleavings": int(res["violations"].sum()), "status_ok": bool((res["status"] == 0).all()),
            "cpu_baseline": {"value": cil / cdt, "cores": 1, "kind": "port",
                             "sample": "%d searches sequentially on one core (x%d cores = %.0f/s if perfectly parallel)"
                                       % (nc, cores(), cil / cdt * cores())}}


def provenance():
    """§8(f) rank 4: provenance pruning of every violating prefix a fuzz batch found."""
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    ext = D.pack_externals(D.raft5_program())
    eng.set_externals(ext)
    n = 2_000_000
    res = eng.fuzz_batch(1, n, 50, 5)
    viol = np.nonzero(res["violation"])[0].astype(np.uint32)
    eng.fuzz_provenance(1, viol[:64], 50, 5)
    t0 = time.perf_counter()
    keep, out, _ = eng.fuzz_provenance(1, viol, 50, 5)
    dt = time.perf_counter() - t0
    kms = eng.stats().kernel_ms
    nc = min(len(viol), 2000)
    t0 = time.perf_counter()
    for i in viol[:nc]:
        O.fuzz_provenance(N.MODEL_RAFT5, ext, 1 + int(i), 50, 5, keep.shape[1], model_flags=1)
    cdt = time.perf_counter() - t0
    return {"config": "provenance pruning of the %d violating prefixes among %d raft5 depth-50 prefixes" % (len(viol), n),
            "metric": "executions pruned/s", "value": len(viol) / (kms * 1e-3), "e2e_value": len(viol) / dt, "kernel_ms": kms,
            "status_ok": bool((out["status"] == 0).all()),
            "deliveries": int(out["n_trace"].sum() - len(out)), "deliveries_kept": int(out["n_kept"].sum() - len(out)),
            "cpu_baseline": {"value": nc / cdt, "cores": 1, "kind": "port",
                             "sample": "%d executions, literal pair-set closure, one core" % nc}}


def incddmin():
    """§8(f) rank 2: IncrementalDDMin over ResumableDPOR (RunnerUtils.editDistanceDporDDMin)."""
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1))
    prog = D.raft5_program(client_cmds=6)
    eng.set_externals(prog)
    ext_all = D.pack_externals(prog)
    dext = ext_all[(ext_all["kind"] == 1) | (ext_all["kind"] == 3)]
    res = eng.fuzz_batch(1, 20000, 60, 5)
    viol = np.nonzero(res["violation"] == 1)[0]
    rows = []
    for i in viol[:8]:
        ev, par, r = eng.fuzz_trace(1 + int(i), 60, 5)
        steps = int(r["steps"])
        t0 = time.perf_counter()
        mcs, out = eng.incremental_ddmin(dext, steps, 4000, (ev, par), looking_for=1, stop_at_size=1, max_max_distance=64,
                                         heap_cap=1 << 17)
        gt = time.perf_counter() - t0
        t0 = time.perf_counter()
        rc, mcs_o, st = O.incremental_ddmin(N.MODEL_RAFT5, dext, steps, 4000, O.dpor_seed(ev, par), model_flags=1,
                                            looking_for=1, stop_at_size=1, max_max_distance=64)
        ct = time.perf_counter() - t0
        rows.append({"prefix": int(i), "deliveries": steps, "externals": int(len(dext)), "mcs": int(out.mcs_size),
                     "identical_to_sequential_oracle": bool(rc == 0 and np.array_equal(mcs, mcs_o) and out.total_replays == st["total_replays"]),
                     "sequential_tests": int(out.total_replays), "tests_on_gpu": int(out.tests_executed),
                     "batches": int(out.batches), "interleavings_on_gpu": int(out.interleavings_executed),
                     "oracle_interleavings": int(st["interleavings"]), "gpu_s": gt, "cpu_oracle_s": ct})
    return {"config": "IncrementalDDMin(ResumableDPOR, ArvindDistanceOrdering) on violating raft5 executions, caps 0..32",
            "metric": "minimisations", "rows": rows}


def config5_bcast():
    """bcast32 depth-200 fuzz with state-hash dedup + compaction."""
    eng = D.Engine(D.SchedulerConfig(N.MODEL_BCAST32))
    ext = D.pack_externals(D.bcast32_program(3))
    eng.set_externals(ext)
    n = 200_000
    dres = torch.empty(n * 32, dtype=torch.uint8, device="cuda")
    dout = torch.empty(n * 32, dtype=torch.uint8, device="cuda")
    didx = torch.empty(n, dtype=torch.int32, device="cuda")
    dcnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    eng.fuzz_batch_dev(1, n, 200, 0, dres.data_ptr(), st.cuda_stream, flags=1)
    eng.dedup_compact_dev(dres.data_ptr(), n, 0, dout.data_ptr(), didx.data_ptr(), dcnt.data_ptr(), st.cuda_stream)
    torch.cuda.synchronize()
    ev[0].record(st)
    eng.fuzz_batch_dev(1 + n, n, 200, 0, dres.data_ptr(), st.cuda_stream, flags=1)
    ev[1].record(st)
    eng.dedup_compact_dev(dres.data_ptr(), n, 0, dout.data_ptr(), didx.data_ptr(), dcnt.data_ptr(), st.cuda_stream)
    ev[2].record(st)
    torch.cuda.synchronize()
    fuzz_ms, dd_ms = ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])
    uniq = int(dcnt.item())
    # a dedup-heavy batch for the HBM-bound kernels alone: 2*10^7 records, 10^6 distinct states
    m = 20_000_000
    rec = np.zeros(m, dtype=N.RESULT_DTYPE)
    rec["state_hash"] = np.random.default_rng(1).integers(0, 1_000_000, size=m, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    big = torch.from_numpy(rec.view(np.uint8)).cuda()
    bout = torch.empty_like(big)
    bidx = torch.empty(m, dtype=torch.int32, device="cuda")
    for _ in range(2):
        eng.dedup_compact_dev(big.data_ptr(), m, 0, bout.data_ptr(), bidx.data_ptr(), dcnt.data_ptr(), st.cuda_stream)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(5):
        eng.dedup_compact_dev(big.data_ptr(), m, 0, bout.data_ptr(), bidx.data_ptr(), dcnt.data_ptr(), st.cuda_stream)
    e1.record(st)
    torch.cuda.synchronize()
    k_ms = e0.elapsed_time(e1) / 5
    kept = int(dcnt.item())
    # algorithmic bytes: insert reads 16 B/record + 12 B table probe/update; flag re-reads 16 B + 12 B probe + 1 B flag;
    # compact reads 1 B flag + 32 B + writes 36 B per kept record
    alg = m * (16 + 12 + 16 + 12 + 1 + 1) + kept * (32 + 36)
    return {"config": "configs[4]: bcast32 (32 actors), depth-200 fuzz, state-hash dedup on",
            "metric": "prefixes/s", "value": n / (fuzz_ms * 1e-3), "fuzz_ms": fuzz_ms, "dedup_compact_ms": dd_ms,
            "unique_states": uniq, "unique_states_per_s": uniq / ((fuzz_ms + dd_ms) * 1e-3),
            "dedup_kernels": {"records": m, "distinct": kept, "ms": k_ms, "records_per_s": m / (k_ms * 1e-3),
                              "roofline": {"bound": "hbm", "achieved": alg / (k_ms * 1e-3) / 1e9, "peak": HBM_PEAK,
                                           "frac": alg / (k_ms * 1e-3) / 1e9 / HBM_PEAK,
                                           "algorithmic_bytes": alg}}}


if __name__ == "__main__":
    which = sys.argv[1:] or ["c4", "c3", "c5"]
    for w in which:
        fn = {"c4": config4_ddmin, "c3": config3_dpor, "c5": config5_bcast, "prov": provenance, "incddmin": incddmin}[w]
        print(json.dumps(fn()), flush=True)
