"""STSSched DDMin of many violating executions: the per-trace loop against the batched path.

  (a) per trace: demi_fuzz_trace + demi_set_trace + demi_ddmin
  (b) demi_fuzz_traces + demi_set_traces + demi_ddmin_many

on the first K in {1, 64, 1024, 16384} violating prefixes of a fuzz batch of the headline workload (bench.py's program,
max_messages, interval and model flags), and of the same program with six client commands.  Reports wall time per trace,
kernel launches, tests evaluated and whether (a) and (b) agree trace by trace, with the card's name and power limit.

  python tools/bench_ddmin_many.py [--ks 1,64,1024,16384] [--out profiles/ddmin_many_h100.txt]
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

CAP_EVENTS = 1024
CAP_ITER = 256


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def per_trace_loop(eng, hits, codes, mw):
    """(a): one fuzz_trace, set_trace and ddmin per violating prefix."""
    L = N.lib()
    p = N.FuzzParams(1, 1, bench.MAX_MESSAGES, bench.INTERVAL, 0, 0)
    ev = np.zeros(CAP_EVENTS, dtype=N.EVENT_DTYPE)
    ne = C.c_uint32()
    res = np.zeros(1, dtype=N.RESULT_DTYPE)
    mcs = np.zeros((len(hits), mw), dtype=np.uint64)
    iters = np.zeros((len(hits), CAP_ITER), dtype=np.uint32)
    outs = np.zeros(len(hits), dtype=N.DDMIN_OUT_DTYPE)
    status = np.zeros(len(hits), dtype=np.int32)
    launches, tests = 0, 0
    ext = eng._ext
    t0 = time.perf_counter()
    for i, k in enumerate(hits):
        rc = L.demi_fuzz_trace(eng._h, C.byref(p), 1 + int(k), ev.ctypes.data, CAP_EVENTS, C.byref(ne), None, 0, None,
                               res.ctypes.data)
        assert rc == N.OK, L.demi_last_error(eng._h)
        rc = L.demi_set_trace(eng._h, ev.ctypes.data, ne.value, ext.ctypes.data, len(ext))
        assert rc == N.OK, L.demi_last_error(eng._h)
        o = N.DDMinOut()
        status[i] = L.demi_ddmin(eng._h, int(codes[i]), 0, 1, mcs[i].ctypes.data, mw, iters[i].ctypes.data, CAP_ITER,
                                 C.byref(o))
        outs[i] = tuple(getattr(o, f) for f in ("mcs_size", "total_replays", "n_iterations", "replays_executed",
                                                "batches", "verified")) + (tuple(o.reserved),)
        launches += 1 + o.batches
        tests += o.replays_executed
    return time.perf_counter() - t0, mcs, iters, outs, status, launches, tests


def batched(eng, hits, codes, mw):
    """(b): fuzz_traces, set_traces, ddmin_many."""
    t0 = time.perf_counter()
    ev, ne, res = eng.fuzz_traces(1, hits, bench.MAX_MESSAGES, bench.INTERVAL, cap_events=CAP_EVENTS)
    fuzz_launches = eng.stats().kernel_launches
    eng.set_traces((ev, ne), eng._ext)
    mcs, iters, outs, status = eng.ddmin_many(codes, cap_iterations=CAP_ITER, mask_words=mw)
    dt = time.perf_counter() - t0
    st = eng.stats()
    return dt, mcs, iters, outs, status, fuzz_launches + st.kernel_launches, st.prefixes, st.kernel_ms


def run(name, prog, ks, n_fuzz):
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=bench.MODEL_FLAGS))
    eng.set_externals(prog)
    res = eng.fuzz_batch(1, n_fuzz, bench.MAX_MESSAGES, bench.INTERVAL)
    viol = np.nonzero((res["violation"] != 0) & (res["status"] == 0))[0]
    mw = max(1, (len(prog) + 63) // 64)
    rows = []
    # warm-up: every kernel and buffer the timed runs use
    per_trace_loop(eng, viol[:2].astype(np.uint32), res["violation"][viol[:2]].astype(np.uint32), mw)
    batched(eng, viol[:2].astype(np.uint32), res["violation"][viol[:2]].astype(np.uint32), mw)
    for k in ks:
        if k > len(viol):
            rows.append({"program": name, "K": k, "skipped": "only %d violating prefixes in %d" % (len(viol), n_fuzz)})
            continue
        hits = viol[:k].astype(np.uint32)
        codes = res["violation"][hits].astype(np.uint32)
        ta, ma, ia, oa, sa, la, na = per_trace_loop(eng, hits, codes, mw)
        tb, mb, ib, ob, sb, lb, nb, kms = batched(eng, hits, codes, mw)
        fields = ["mcs_size", "total_replays", "n_iterations", "replays_executed", "batches", "verified"]
        same = (sa == sb) & (ma == mb).all(axis=1) & (ia == ib).all(axis=1) & \
            np.array([oa[f] == ob[f] for f in fields]).all(axis=0)
        rows.append({"program": name, "K": k, "externals": len(prog),
                     "a_ms_per_trace": 1e3 * ta / k, "b_ms_per_trace": 1e3 * tb / k, "speedup": ta / tb,
                     "a_launches": la, "b_launches": lb, "a_tests": na, "b_tests": nb, "b_kernel_ms": kms,
                     "identical_traces": int(same.sum()), "ok_traces": int((sb == 0).sum())})
        print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,64,1024,16384")
    ap.add_argument("--fuzz", type=int, default=1 << 20, help="prefixes of the fuzz batch the violations come from")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ks = [int(x) for x in a.ks.split(",")]
    gpu = card()
    rows = run("raft5_program()", D.raft5_program(), ks, a.fuzz)
    rows += run("raft5_program(client_cmds=6)", D.raft5_program(client_cmds=6), ks, a.fuzz)
    lines = ["# tools/bench_ddmin_many.py: STSSched DDMin of K violating raft5 executions",
             "# card (name, power limit, max SM clock): " + gpu,
             "# (a) demi_fuzz_trace + demi_set_trace + demi_ddmin per trace; (b) demi_fuzz_traces + demi_set_traces + "
             "demi_ddmin_many.  Wall time includes recording.  launches: kernel launches (a counts one recording launch "
             "per trace); tests: replays evaluated.",
             "# max_messages %d, interval %d, model_flags %d, DEMI_DDMIN_WIDE default" % (bench.MAX_MESSAGES, bench.INTERVAL,
                                                                                      bench.MODEL_FLAGS)]
    lines += [json.dumps(r) for r in rows]
    text = "\n".join(lines) + "\n"
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
