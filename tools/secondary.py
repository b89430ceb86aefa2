"""Secondary workloads of BASELINE.json (configs[2..4]) as legs of bench.py's JSON line.

Each leg runs after, and outside, the headline's timed region, on every rank (legs with an exchange step are
collective), is bounded to a few seconds, and reports its own metric, a `roofline` object for its dominant kernel(s)
and a `cpu_baseline` timed on the host cores (rank 0, N = 1 only — the oracle is test infrastructure, used here as the
reported CPU figure exactly as in the headline)."""
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import demi_b200 as D
from demi_b200 import _native as N

# configs[3]: the violating raft5 execution whose EventTrace has >= 2000 events (found with tools/find_c3_trace.py:
# 290 client commands, maxMessages 1000, invariant every 100 deliveries, seeded double-vote bug)
C3_PROGRAM_CMDS = 290
C3_MAX_MESSAGES = 1000
C3_INTERVAL = 100
C3_SEED = int(os.environ.get("DEMI_C3_SEED", "0")) or None
C3_SEED_DEFAULT = 318        # tools/find_c3_trace.py: 2039 events, 1000 deliveries, violation 1 (two leaders in a term)


def _peak():
    try:
        import json
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]), "measured"
    except Exception:
        return 3350.0, "fallback"                 # H100 SXM data sheet (HBM3)


def _allmax(x, dev, world):
    t = torch.tensor([float(x)], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def _allsum(xs, dev, world):
    t = torch.tensor([float(x) for x in xs], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return [float(v) for v in t.tolist()]


def _barrier(world):
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ configs[2]
def c2_dpor(rank, world, local_rank, cores, with_cpu):
    """akka-raft-like 5 nodes, DPORwHeuristics depth-100 (max_messages = 100), ONE search.
    (a) the search as the reference runs it (trackHistory = true) to exhaustion, on one GPU, next to the sequential CPU
        restatement; (b) the same search with trackHistory = false — every backtrack point is replayed, so the frontier
        is unbounded and only a budget ends it — sharded over all ranks with the in-library NCCL steal round."""
    dev = torch.device("cuda", local_rank)
    prog = D.raft5_program(client_cmds=2)[:-1]
    ext = D.pack_externals(prog)
    out = {"config": "configs[2]: raft5, DPORwHeuristics(max_messages=100, DefaultBacktrackOrdering, stopIfViolationFound=false), "
                     "one search explored as a frontier of backtrack points"}
    # ---- (a) trackHistory = true, to exhaustion
    if rank == 0:
        eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=3, device=local_rank))
        F = eng.frontier_params(100, 1 << 16, 16384, explored_slots=1 << 16, pool_cap=1 << 18, trace_cap=1 << 16)
        eng.dpor_frontier(prog, F)                                   # allocates the tables
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r, viol, hashes = eng.dpor_frontier(prog, F)
        gpu_ms = (time.perf_counter() - t0) * 1e3
        a = {"mode": "trackHistory=true, run until the backtrack set is empty", "interleavings": int(r["interleavings"]),
             "rounds": int(r["rounds"]), "races": int(r["races"]), "explored_pairs": int(r["explored_pairs"]),
             "exhausted": int(r["exhausted"]), "gpu_ms": gpu_ms, "width": 16384,
             "kernel_ms": float(r["exec_ms"] + r["scan_ms"] + r["select_ms"]), "gpu_launches": int(eng.stats().kernel_launches)}
        if with_cpu:
            from oracle import binding as O
            O.dpor_search(N.MODEL_RAFT5, ext, 100, 1 << 16, 0, 0, -1, model_flags=3, node_cap=1 << 14, explored_slots=1 << 18,
                          heap_cap=1 << 20)
            t0 = time.perf_counter()
            rc, sr, sviol, shashes = O.dpor_search(N.MODEL_RAFT5, ext, 100, 1 << 16, 0, 0, -1, model_flags=3, node_cap=1 << 14,
                                                   explored_slots=1 << 18, heap_cap=1 << 20)
            cpu_ms = (time.perf_counter() - t0) * 1e3
            a["cpu_baseline"] = {"value": cpu_ms, "unit": "ms", "cores": 1, "kind": "port",
                                 "sample": "the same search, sequential restatement of DPORwHeuristics (the reference "
                                           "algorithm is sequential: one interleaving per dpor() call)"}
            a["speedup_vs_cpu"] = cpu_ms / gpu_ms
            a["schedule_set_equal_to_sequential"] = bool(set(int(x) for x in hashes) == set(int(x) for x in shashes))
            a["violating_set_equal_to_sequential"] = bool(set(int(x) for x in viol["schedule_hash"]) ==
                                                          set(int(x) for x in sviol["schedule_hash"]))
        out["search"] = a
        eng.close()
    # ---- (b) trackHistory = false, budgeted, all ranks + steal round
    per_gpu = int(os.environ.get("DEMI_C2_BUDGET", str(1 << 22)))
    width = int(os.environ.get("DEMI_C2_WIDTH", "131072"))
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=3, device=local_rank))
    if world > 1:
        uid = torch.zeros(N.COMM_ID_BYTES, dtype=torch.uint8, device=dev)
        if rank == 0:
            uid.copy_(torch.frombuffer(bytearray(D.Engine.comm_unique_id()), dtype=torch.uint8))
        dist.broadcast(uid, 0)
        eng.comm_init(bytes(uid.cpu().numpy().tobytes()), rank, world)
    F = eng.frontier_params(100, per_gpu * world, width, explored_slots=1 << 10, pool_cap=1 << 30,
                            trace_cap=per_gpu + width + 8 * 4096 + 16, rounds_per_exchange=4, steal_max=4096,
                            flags=N.FR_NO_HISTORY)
    eng.dpor_frontier(prog, F, want_hashes=False)                    # warm-up: allocates, first NCCL exchange
    _barrier(world)
    t0 = time.perf_counter()
    r, viol, _ = eng.dpor_frontier(prog, F, want_hashes=False)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    dt = _allmax(dt, dev, world)
    il, dl, races, keys, sent, bsent = _allsum([r["interleavings"], r["deliveries"], r["races"], r["keys_enqueued"],
                                                r["records_sent"], r["bytes_sent"]], dev, world)
    kms = _allmax(float(r["exec_ms"] + r["scan_ms"] + r["select_ms"]), dev, world)
    xms = _allmax(float(r["exchange_ms"]), dev, world)
    alg = dl * 32 + keys * 16 + races * 8
    peak, kind = _peak()
    b = {"mode": "trackHistory=false (DPORwHeuristics.scala:86), budget %d interleavings per GPU, width %d, "
                 "steal every 4 rounds" % (per_gpu, width),
         "metric": "interleavings/s", "value": il / dt, "unit": "interleavings/s", "n_gpus": world, "scaling": "weak",
         "wall_s": dt, "interleavings": il, "deliveries": dl, "races": races, "backtrack_points_enqueued": keys,
         "kernel_ms_max_rank": kms, "exec_ms": float(r["exec_ms"]), "scan_ms": float(r["scan_ms"]),
         "select_ms": float(r["select_ms"]), "rounds_rank0": int(r["rounds"]),
         "steal": {"exchanges": int(r["exchanges"]), "records_sent": sent, "bytes_sent": bsent, "exchange_ms_max_rank": xms,
                   "collective": "ncclAllGather (queue lengths, counts) + grouped ncclSend/ncclRecv of %d-byte records"
                                 % (16 * 104) if world > 1 else None},
         "gpu_launches": int(eng.stats().kernel_launches),
         "roofline": {"bound": "hbm", "achieved": alg * 1.0 / world / (kms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s",
                      "frac": alg * 1.0 / world / (kms * 1e-3) / 1e9 / peak, "peak_kind": kind, "traffic": None,
                      "algorithmic_bytes": "32 B per delivery (16 B trace entry written + 16 B key-trace entry read) + "
                                           "16 B per backtrack point + 8 B per race record",
                      "kernel": "fr_exec_kernel + fr_scan_kernel + fr_count/fr_scatter (per GPU)"}}
    if with_cpu and rank == 0 and world == 1:
        from oracle import binding as O
        OF = O.frontier_params(100, 20000, width, explored_slots=1 << 10, pool_cap=1 << 23, flags=1)
        t0 = time.perf_counter()
        rc, ores, _, _ = O.dpor_frontier(N.MODEL_RAFT5, ext, OF, 1, model_flags=3)
        cdt = time.perf_counter() - t0
        b["cpu_baseline"] = {"value": float(ores[0]["interleavings"]) / cdt, "unit": "interleavings/s", "cores": 1, "kind": "port",
                             "sample": "20000 interleavings of the same search, CPU restatement, one core"}
    out["frontier"] = b
    eng.close()
    return out


# ------------------------------------------------------------------------------------------------ configs[3]
def c3_trace(eng_cfg_device):
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=1, device=eng_cfg_device))
    prog = D.raft5_program(client_cmds=C3_PROGRAM_CMDS)
    ext = D.pack_externals(prog)
    eng.set_externals(ext)
    seed = C3_SEED or C3_SEED_DEFAULT
    ev, par, r = eng.fuzz_trace(seed, C3_MAX_MESSAGES, C3_INTERVAL)
    return eng, ext, ev, par, r, seed


def c3_ddmin(rank, world, local_rank, cores, with_cpu):
    """DDMin over a >= 2000-event violating trace; 10^6 STSSched subsequence replays per GPU in one batch."""
    dev = torch.device("cuda", local_rank)
    eng, ext, ev, par, r, seed = c3_trace(local_rank)
    code = int(r["violation"])
    out = {"config": "configs[3]: DDMin over a %d-event violating raft5 trace (%d externals, seed %d); 10^6 STSSched "
                     "replays per GPU batched" % (len(ev), len(ext), seed)}
    if code == 0 or len(ev) < 2000:
        out["error"] = "the recorded execution has %d events and violation %d" % (len(ev), code)
        return out
    eng.set_trace(ev, ext)
    mw = eng.mask_words()
    rng = np.random.default_rng(rank)
    n = int(os.environ.get("DEMI_C3_MASKS", "1000000"))
    full = np.zeros(mw, dtype=np.uint64)
    for i, e in enumerate(ext):
        if e["kind"] != N.EXT_WAIT_QUIESCENCE:
            full[i // 64] |= np.uint64(1) << np.uint64(i % 64)
    masks = rng.integers(0, 2**63, size=(n, mw), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=(n, mw), dtype=np.uint64)
    masks |= rng.integers(0, 2**63, size=(n, mw), dtype=np.uint64) * np.uint64(2)     # ~75 % dense
    masks &= full[None, :]
    masks[0] = full
    dm = torch.from_numpy(masks.view(np.int64)).to(dev)
    dout = torch.empty(n * 16, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream()
    eng.replay_batch_dev(dm.data_ptr(), n, dout.data_ptr(), code, 0, st.cuda_stream)
    _barrier(world)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    reps = 2
    for _ in range(reps):
        eng.replay_batch_dev(dm.data_ptr(), n, dout.data_ptr(), code, 0, st.cuda_stream)
    e1.record(st)
    torch.cuda.synchronize()
    ms = _allmax(e0.elapsed_time(e1) / reps, dev, world)
    res = dout.cpu().numpy().view(N.REPLAY_DTYPE)
    t0 = time.perf_counter()
    host_out = eng.replay_batch(masks, code)                          # host masks in, host results out
    e2e = _allmax(time.perf_counter() - t0, dev, world)
    ok = bool((host_out == res).all() and res[0]["violation"] == code)
    alg = n * (mw * 8 + 16)
    peak, kind = _peak()
    out.update({"metric": "subsequence replays/s", "value": n * world / (ms * 1e-3), "unit": "replays/s", "n_gpus": world,
                "scaling": "weak", "e2e": {"value": n * world / e2e, "unit": "replays/s", "h2d_bytes_per_step": int(masks.nbytes),
                                            "d2h_bytes_per_step": n * 16},
                "kernel_ms": ms, "reproduced_rank0": int((res["violation"] != 0).sum()), "host_path_identical": ok,
                "gpu_launches": reps,
                "roofline": {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s",
                             "frac": alg / (ms * 1e-3) / 1e9 / peak, "peak_kind": kind, "traffic": None,
                             "algorithmic_bytes_per_test": mw * 8 + 16, "kernel": "replay_lane_kernel<Raft5,256>",
                             "note": "the %d-event trace is shared by the whole batch (L2-resident) and not counted per test" % len(ev)}})
    if rank == 0:
        t0 = time.perf_counter()
        mcs, iters, dd = eng.ddmin(code)
        ddt = time.perf_counter() - t0
        out["ddmin"] = {"externals": int(len(ext)), "mcs_size": int(dd.mcs_size), "sequential_tests": int(dd.total_replays),
                        "tests_executed_on_gpu": int(dd.replays_executed), "batches": int(dd.batches),
                        "verified": int(dd.verified), "gpu_seconds": ddt}
        if with_cpu and world == 1:
            from oracle import binding as O
            nc = 2000 * cores
            t0 = time.perf_counter()
            cpu = O.replay_batch(N.MODEL_RAFT5, ev, ext, masks[:nc], looking_for=code, model_flags=1, threads=cores)
            cdt = time.perf_counter() - t0
            out["cpu_baseline"] = {"value": nc / cdt, "per_core": nc / cdt / cores, "unit": "replays/s", "cores": cores,
                                   "kind": "port", "sample": "%d of the same masks, identical results: %s" % (nc, bool((cpu == res[:nc]).all()))}
            t0 = time.perf_counter()
            rc, cmcs, total, citers, ver = O.ddmin_sts(N.MODEL_RAFT5, ev, ext, code, model_flags=1)
            out["ddmin"]["cpu_oracle_seconds"] = time.perf_counter() - t0
            out["ddmin"]["mcs_identical_to_sequential_oracle"] = bool((mcs == cmcs).all() and dd.total_replays == total and
                                                                      list(iters) == list(citers))
    eng.close()
    return out


# ------------------------------------------------------------------------------------------------ configs[4]
def c4_bcast(eng_headline, rank, world, local_rank, results_dev, n_headline, cores, with_cpu):
    """32-actor broadcast storm, depth-200 fuzz, state-hash dedup on (K5 insert + K4 ordered compaction)."""
    dev = torch.device("cuda", local_rank)
    st = torch.cuda.current_stream()
    peak, kind = _peak()
    out = {"config": "configs[4]: bcast32 (32 actors), depth-200 fuzz, state-hash dedup on"}

    def fuzz_and_dedup(prog, n, flags, label):
        eng = D.Engine(D.SchedulerConfig(N.MODEL_BCAST32, device=local_rank))
        eng.set_externals(D.pack_externals(prog))
        dres = torch.empty(n * 32, dtype=torch.uint8, device=dev)
        dkept = torch.empty(n * 32, dtype=torch.uint8, device=dev)
        didx = torch.empty(n, dtype=torch.int32, device=dev)
        dcnt = torch.zeros(1, dtype=torch.int64, device=dev)
        eng.fuzz_batch_dev(1 + rank * 10 * n, n, 200, 0, dres.data_ptr(), st.cuda_stream, flags=flags)
        eng.dedup_compact_dev(dres.data_ptr(), n, 0, dkept.data_ptr(), didx.data_ptr(), dcnt.data_ptr(), st.cuda_stream)
        _barrier(world)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record(st)
        eng.fuzz_batch_dev(1 + rank * 10 * n + n, n, 200, 0, dres.data_ptr(), st.cuda_stream, flags=flags)
        ev[1].record(st)
        eng.dedup_compact_dev(dres.data_ptr(), n, 0, dkept.data_ptr(), didx.data_ptr(), dcnt.data_ptr(), st.cuda_stream)
        ev[2].record(st)
        torch.cuda.synchronize()
        fms, dms = _allmax(ev[0].elapsed_time(ev[1]), dev, world), _allmax(ev[1].elapsed_time(ev[2]), dev, world)
        uniq = int(dcnt.item())
        steps = float(eng.fuzz_summary_dev(st.cuda_stream)[1])
        u, s = _allsum([uniq, steps], dev, world)
        eng.close()
        return {"program": label, "prefixes_per_gpu": n, "fuzz_ms": fms, "dedup_compact_ms": dms,
                "prefixes_per_s": n * world / ((fms + dms) * 1e-3), "deliveries_per_s": s / (fms * 1e-3),
                "unique_states_sum_over_ranks": u, "unique_fraction": u / (n * world)}

    n = int(os.environ.get("DEMI_C4_PREFIXES", "200000"))
    # (i) the storm itself: one INJECT(ttl=3): 29 823 messages, cut at depth 200 — the reachable states outnumber any
    # sample, so every record is distinct and dedup is a pass-through filter
    out["storm_ttl3"] = fuzz_and_dedup(D.bcast32_program(3), n, 1, "Start x32, INJECT(ttl=3); cut at depth 200, pending multiset hashed")
    # (ii) six small floods that quiesce inside the bound (6 + 6*31 = 192 deliveries): deliveries commute, executions
    # converge to the same final state and dedup collapses the batch
    prog = [D.Start(a) for a in range(32)] + [D.Send(a, 2, 1) for a in range(6)] + [D.WaitQuiescence()]
    out["quiescing_ttl1_x6"] = fuzz_and_dedup(prog, n, 1, "Start x32, INJECT(ttl=1) into actors 0..5; quiesces at 192 deliveries")
    out["metric"] = "prefixes/s (fuzz + dedup)"; out["value"] = out["storm_ttl3"]["prefixes_per_s"]; out["unit"] = "prefixes/s"
    out["n_gpus"] = world; out["scaling"] = "weak"
    # (iii) the HBM-bound kernels on a batch with real duplicates: the headline's last step (10^7 raft5 records per GPU)
    dkept = torch.empty(n_headline * 32, dtype=torch.uint8, device=dev)
    didx = torch.empty(n_headline, dtype=torch.int32, device=dev)
    dcnt = torch.zeros(1, dtype=torch.int64, device=dev)
    eng_headline.dedup_compact_dev(results_dev.data_ptr(), n_headline, 0, dkept.data_ptr(), didx.data_ptr(), dcnt.data_ptr(), st.cuda_stream)
    _barrier(world)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    reps = 3
    for _ in range(reps):
        eng_headline.dedup_compact_dev(results_dev.data_ptr(), n_headline, 0, dkept.data_ptr(), didx.data_ptr(), dcnt.data_ptr(), st.cuda_stream)
    e1.record(st)
    torch.cuda.synchronize()
    kms = _allmax(e0.elapsed_time(e1) / reps, dev, world)
    kept = int(dcnt.item())
    alg = n_headline * (16 + 12 + 16 + 12 + 1 + 1) + kept * (32 + 36)
    out["dedup_kernels"] = {"input": "the %d result records of the headline's last step (raft5 depth-50)" % n_headline,
                            "records_per_gpu": n_headline, "distinct_states_rank0": kept, "ms": kms,
                            "records_per_s": n_headline * world / (kms * 1e-3), "gpu_launches": 4 * reps}
    out["roofline"] = {"bound": "hbm", "achieved": alg / (kms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s",
                       "frac": alg / (kms * 1e-3) / 1e9 / peak, "peak_kind": kind, "traffic": None,
                       "algorithmic_bytes": alg, "kernel": "dedup_insert + dedup_flag + scan + scatter (K5/K4)"}
    if with_cpu and rank == 0 and world == 1:
        sample = results_dev[:2_000_000 * 32].cpu().numpy().view(N.RESULT_DTYPE)
        t0 = time.perf_counter()
        np.unique(sample["state_hash"], return_index=True)
        cdt = time.perf_counter() - t0
        out["cpu_baseline"] = {"value": len(sample) / cdt, "unit": "records/s", "cores": 1, "kind": "port",
                               "sample": "numpy.unique(return_index=True) over %d of the same records" % len(sample)}
    return out


def run_all(eng_headline, rank, world, local_rank, results_dev, n_headline, cores, with_cpu=True):
    out = {}
    for name, fn in (("c2_dpor", lambda: c2_dpor(rank, world, local_rank, cores, with_cpu)),
                     ("c3_ddmin", lambda: c3_ddmin(rank, world, local_rank, cores, with_cpu)),
                     ("c4_bcast_dedup", lambda: c4_bcast(eng_headline, rank, world, local_rank, results_dev, n_headline, cores, with_cpu))):
        t0 = time.perf_counter()
        out[name] = fn()
        out[name]["leg_seconds"] = time.perf_counter() - t0
    return out
