"""IncrementalDDMin over ResumableDPOR (RunnerUtils.editDistanceDporDDMin's minimisation) of many violating executions:
the per-trace loop against the batched path.

  (a) per trace: demi_fuzz_trace (with its DepTracker tree) + demi_incremental_ddmin
  (b) demi_fuzz_traces_tree + demi_incremental_ddmin_many

on the first K violating prefixes of a fuzz batch of raft5 (bench.py's max_messages, interval and model flags), with
the program of 11 externals and the one with six client commands (17).  Each trace's DPOR instances are seeded with its
own recording and setMaxMessagesToSchedule(its recorded deliveries), ArvindDistanceOrdering and
prioritizePendingUponDivergence on.  Reports wall time per trace (recording included), kernel launches, DPOR tests and
whether (a) and (b) agree trace by trace in every output, with the card's name and power limit.  The batched arm alone
runs at the K of --batched-only.

  python tools/bench_incddmin_many.py [--ks 64,1024] [--batched-only 4096] [--out profiles/incddmin_many_h100.txt]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
import demi_b200 as D  # noqa: E402
from demi_b200 import _native as N  # noqa: E402

CAP_EVENTS, CAP_NODES = 1024, 1024
FLAGS = N.DF_ARVIND_ORDERING | N.DF_PRIORITIZE_PENDING
FIELDS = ("mcs_size", "total_replays", "rounds", "instances", "tests_executed", "batches", "interleavings_executed")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def dpor_ext(prog):
    ext = D.pack_externals(prog)
    return np.ascontiguousarray(ext[(ext["kind"] == N.EXT_START) | (ext["kind"] == N.EXT_SEND)])


def params(budget):
    return N.DporParams(0, -1, budget, 1, 1, 4096, 1 << 16, 1 << 16)


def per_trace_loop(eng, hits, dext, budget, mmd, mw):
    """(a): one fuzz_trace and incremental_ddmin per violating prefix."""
    L = N.lib()
    p = N.FuzzParams(1, 1, bench.MAX_MESSAGES, bench.INTERVAL, 0, 0)
    ev = np.zeros(CAP_EVENTS, dtype=N.EVENT_DTYPE)
    par = np.zeros(CAP_NODES, dtype=np.uint16)
    ne, nn = C.c_uint32(), C.c_uint32()
    res = np.zeros(1, dtype=N.RESULT_DTYPE)
    mcs = np.zeros((len(hits), mw), dtype=np.uint64)
    outs = np.zeros(len(hits), dtype=N.INCDDMIN_OUT_DTYPE)
    status = np.zeros(len(hits), dtype=np.int32)
    launches = tests = 0
    t0 = time.perf_counter()
    for i, k in enumerate(hits):
        rc = L.demi_fuzz_trace(eng._h, C.byref(p), 1 + int(k), ev.ctypes.data, CAP_EVENTS, C.byref(ne), par.ctypes.data,
                               CAP_NODES, C.byref(nn), res.ctypes.data)
        assert rc == N.OK, L.demi_last_error(eng._h)
        P = params(budget)
        P.max_messages = int(res[0]["steps"])
        sd = N.DporSeed(ev.ctypes.data, ne.value, par.ctypes.data, nn.value)
        o = N.IncDDMinOut()
        status[i] = L.demi_incremental_ddmin(eng._h, dext.ctypes.data, len(dext), C.byref(P), FLAGS, C.byref(sd), mmd, 1,
                                             mcs[i].ctypes.data, mw, C.byref(o))
        outs[i] = tuple(getattr(o, f) for f in FIELDS)
        launches += 1 + o.batches
        tests += o.tests_executed
    return time.perf_counter() - t0, mcs, outs, status, launches, tests


def batched(eng, hits, dext, budget, mmd, mw):
    """(b): fuzz_traces_tree, incremental_ddmin_many."""
    t0 = time.perf_counter()
    ev, ne, par, nn, res = eng.fuzz_traces_tree(1, hits, bench.MAX_MESSAGES, bench.INTERVAL, cap_events=CAP_EVENTS,
                                                cap_nodes=CAP_NODES)
    fuzz_launches = eng.stats().kernel_launches
    seeds = [(ev[i, :ne[i]], par[i, :nn[i]]) for i in range(len(hits))]
    mcs, outs, status = eng.incremental_ddmin_many(dext, res["steps"].astype(np.int32), budget, seeds, looking_for=1,
                                                   max_max_distance=mmd, stop_at_size=1, flags=FLAGS, heap_cap=1 << 16,
                                                   mask_words=mw)
    dt = time.perf_counter() - t0
    st = eng.stats()
    return dt, mcs, outs, status, fuzz_launches + st.kernel_launches, int(outs["tests_executed"].sum()), st.kernel_ms


def run(name, prog, ks, batched_only, n_fuzz, budget, mmd):
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=bench.MODEL_FLAGS))
    eng.set_externals(prog)
    res = eng.fuzz_batch(1, n_fuzz, bench.MAX_MESSAGES, bench.INTERVAL)
    viol = np.nonzero((res["violation"] == 1) & (res["status"] == 0))[0]
    dext = dpor_ext(prog)
    mw = max(1, (len(dext) + 63) // 64)
    rows = []
    # warm-up: every kernel and buffer the timed runs use
    per_trace_loop(eng, viol[:2].astype(np.uint32), dext, budget, mmd, mw)
    batched(eng, viol[:2].astype(np.uint32), dext, budget, mmd, mw)
    for k in ks + batched_only:
        if k > len(viol):
            rows.append({"program": name, "K": k, "skipped": "only %d violating prefixes in %d" % (len(viol), n_fuzz)})
            continue
        hits = viol[:k].astype(np.uint32)
        row = {"program": name, "K": k, "externals": len(prog), "dpor_externals": len(dext)}
        tb, mb, ob, sb, lb, nb, kms = batched(eng, hits, dext, budget, mmd, mw)
        row.update({"b_ms_per_trace": 1e3 * tb / k, "b_launches": lb, "b_tests": nb, "b_kernel_ms": kms,
                    "ok_traces": int((sb == 0).sum())})
        if k in ks:
            ta, ma, oa, sa, la, na = per_trace_loop(eng, hits, dext, budget, mmd, mw)
            same = (sa == sb) & (ma == mb).all(axis=1) & np.array([oa[f] == ob[f] for f in FIELDS]).all(axis=0)
            row.update({"a_ms_per_trace": 1e3 * ta / k, "speedup": ta / tb, "a_launches": la, "a_tests": na,
                        "identical_traces": int(same.sum())})
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    eng.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="64,1024", help="K at which both arms run")
    ap.add_argument("--batched-only", default="4096", help="K at which only the batched arm runs")
    ap.add_argument("--fuzz", type=int, default=1 << 20, help="prefixes of the fuzz batch the violations come from")
    ap.add_argument("--budget", type=int, default=200, help="max_interleavings of every DPOR instance")
    ap.add_argument("--max-max-distance", type=int, default=16)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ks = [int(x) for x in a.ks.split(",") if x]
    bo = [int(x) for x in a.batched_only.split(",") if x]
    gpu = card()
    rows = run("raft5_program()", D.raft5_program(), ks, bo, a.fuzz, a.budget, a.max_max_distance)
    rows += run("raft5_program(client_cmds=6)", D.raft5_program(client_cmds=6), ks, bo, a.fuzz, a.budget, a.max_max_distance)
    lines = ["# tools/bench_incddmin_many.py: IncrementalDDMin(ResumableDPOR) of K violating raft5 executions",
             "# card (name, power limit, max SM clock): " + gpu,
             "# (a) demi_fuzz_trace + demi_incremental_ddmin per trace; (b) demi_fuzz_traces_tree + "
             "demi_incremental_ddmin_many.  Wall time includes recording.  launches: kernel launches (a counts one "
             "recording launch per trace); tests: DPOR tests evaluated, speculation included.",
             "# fuzz max_messages %d, interval %d, model_flags %d; DPOR: max_messages = each trace's deliveries, "
             "max_interleavings %d, max_max_distance %d, stop_at_size 1, node_cap 4096, explored_slots 2^16, heap_cap 2^16, "
             "ArvindDistanceOrdering + prioritizePendingUponDivergence" % (bench.MAX_MESSAGES, bench.INTERVAL, bench.MODEL_FLAGS,
                                                                           a.budget, a.max_max_distance)]
    lines += [json.dumps(r) for r in rows]
    text = "\n".join(lines) + "\n"
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
