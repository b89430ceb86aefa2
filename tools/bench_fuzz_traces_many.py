"""Recording many violating executions of a campaign in one call (demi_fuzz_traces_many) against the per-violation
loop (demi_set_externals + demi_fuzz_trace per execution).

A seeded raft5 campaign with tools/bench_random_ddmin_many.py's Fuzzer settings (MODEL_FLAGS = 1, max_messages 50,
interval 5, raft5_program() prefix, CLIENT_CMD Sends, the reference's default FuzzerWeights, num_events 20) gives its
violating executions in order.  Execution k has its own program (demi_fuzzer_generate with program seed pseed + k) and
its seed seed_base + k.  The first 64, 1 024 and 4 096 of them are recorded, EventTrace and DepTracker tree, both ways,
alternating, `--repeats` times; then the whole pipeline (recording, demi_set_traces, demi_ddmin_many) runs both ways,
alternating.  The campaign is not timed.  Every record, tree and MCS must be identical both ways.

Prints the card's name and power limit first, then one JSON line per size: ms per trace both ways for the recording
alone and for the pipeline, and the launches of the batched call.  Usage: python tools/bench_fuzz_traces_many.py
[--sizes 64,1024,4096] [--repeats R]"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
import demi_b200 as D  # noqa: E402
from demi_b200 import _native as N  # noqa: E402
from demi_b200.fuzzer import ClientCommandGenerator, Fuzzer, FuzzerWeights, fuzzer_config  # noqa: E402

MM, INTERVAL, FLAGS, CLIENT_CMD = 50, 5, 1, 2
CAP_EV, CAP_NODES = 1024, 1024


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def violating_executions(eng, want, seed_base, pseed):
    fz = Fuzzer(20, FuzzerWeights(), ClientCommandGenerator(CLIENT_CMD), D.raft5_program()[:-1])
    eng.set_fuzzer(fuzzer_config(fz), D.raft5_program()[:-1])
    out, off, chunk = [], 0, 1 << 16
    while len(out) < want:
        res = eng.fuzz_campaign(seed_base + off, chunk, MM, INTERVAL, pseed + off)
        for i in np.nonzero((res["violation"] != 0) & (res["status"] == 0))[0]:
            k = off + int(i)
            out.append((np.ascontiguousarray(eng.fuzzer_program(pseed + k), dtype=N.EXT_DTYPE), seed_base + k,
                        int(res["violation"][i])))
        off += chunk
    return out[:want]


def loop(eng, execs):
    """demi_set_externals + demi_fuzz_trace per execution: (events [n, CAP_EV], n_events, dep_parent, n_nodes)"""
    n = len(execs)
    ev = np.zeros((n, CAP_EV), dtype=N.EVENT_DTYPE)
    par = np.zeros((n, CAP_NODES), dtype=np.uint16)
    ne, nn = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint32)
    L = N.lib()
    for t, (prog, seed, _) in enumerate(execs):
        assert L.demi_set_externals(eng._h, prog.ctypes.data, len(prog)) == 0
        p = N.FuzzParams(seed, 1, MM, INTERVAL, 0, 0)
        a, b = C.c_uint32(), C.c_uint32()
        assert L.demi_fuzz_trace(eng._h, C.byref(p), seed, ev[t].ctypes.data, CAP_EV, C.byref(a), par[t].ctypes.data, CAP_NODES,
                                 C.byref(b), None) == 0
        ne[t], nn[t] = a.value, b.value
    return ev, ne, par, nn


def many(eng, execs):
    ev, ne, par, nn, _, status = eng.fuzz_traces_many([e[0] for e in execs], [e[1] for e in execs], MM, 0, INTERVAL,
                                                      cap_events=CAP_EV, cap_nodes=CAP_NODES)
    assert not status.any()
    return ev, ne, par, nn


def pipeline(eng, execs, record):
    ev, ne, _, _ = record(eng, execs)
    eng.set_traces((ev, ne), [e[0] for e in execs])
    mcs, _, out, status = eng.ddmin_many(np.array([e[2] for e in execs], dtype=np.uint32))
    return mcs, out["mcs_size"].copy(), status


def same_records(a, b):
    ev1, ne1, par1, nn1 = a
    ev2, ne2, par2, nn2 = b
    if not (np.array_equal(ne1, ne2) and np.array_equal(nn1, nn2)):
        return False
    return all(ev1[t, :ne1[t]].tobytes() == ev2[t, :ne1[t]].tobytes() and
               par1[t, :nn1[t]].tobytes() == par2[t, :nn1[t]].tobytes() for t in range(len(ne1)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="64,1024,4096")
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps({"card": card()}))
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, FLAGS))
    sizes = [int(x) for x in a.sizes.split(",")]
    seed_base = 1000
    execs_all = violating_executions(eng, max(sizes), seed_base, seed_base + D.PROGRAM_SEED_OFFSET)
    print(json.dumps({"violating_executions": len(execs_all),
                      "program_events": [min(len(e[0]) for e in execs_all), max(len(e[0]) for e in execs_all)]}))
    for size in sizes:
        execs = execs_all[:size]
        many(eng, execs[:8]), loop(eng, execs[:8])                 # warm-up: modules, buffers
        t_many, t_loop, p_many, p_loop = [], [], [], []
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            got = many(eng, execs)
            t_many.append(time.perf_counter() - t0)
            launches = eng.stats().kernel_launches
            t0 = time.perf_counter()
            want = loop(eng, execs)
            t_loop.append(time.perf_counter() - t0)
            assert same_records(got, want), "records differ"
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            got = pipeline(eng, execs, many)
            p_many.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            want = pipeline(eng, execs, loop)
            p_loop.append(time.perf_counter() - t0)
            assert all(np.array_equal(x, y) for x, y in zip(got, want)), "MCSs differ"
        print(json.dumps({"traces": size,
                          "record_many_ms_per_trace": [round(1e3 * t / size, 4) for t in t_many],
                          "record_loop_ms_per_trace": [round(1e3 * t / size, 4) for t in t_loop],
                          "record_speedup_best": round(min(t_loop) / min(t_many), 2), "many_launches": launches,
                          "pipeline_many_ms_per_trace": [round(1e3 * t / size, 3) for t in p_many],
                          "pipeline_loop_ms_per_trace": [round(1e3 * t / size, 3) for t in p_loop],
                          "pipeline_speedup_best": round(min(p_loop) / min(p_many), 2),
                          "failed_ddmin_traces": int((got[2] != 0).sum()), "identical": True}))
        sys.stdout.flush()


if __name__ == "__main__":
    main()
