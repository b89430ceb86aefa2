"""randomDDMin over many violating executions in one call (demi_random_ddmin_many) against the per-trace loop
(demi_set_externals + demi_random_ddmin per execution).

A seeded raft5 campaign with tools/bench_random_ddmin.py's Fuzzer settings (MODEL_FLAGS = 1, max_messages 50, interval
5, raft5_program() prefix, CLIENT_CMD Sends, the reference's default FuzzerWeights, num_events 20) gives its violating
executions in order.  Execution k has its own program (demi_fuzzer_generate with program seed pseed + k), its seed
seed_base + k, max_messages = the length of its recorded EventTrace (randomDDMin's setMaxMessages(trace.size)) and
looking_for = its violation.  The first 64, 1 024 and 4 096 of them are minimized with N = 1 and N = 64 executions per
test, both ways, alternating, `--repeats` times; the setup is not timed.  Every trace's status, MCS, iteration series
and demi_random_ddmin_out fields (executions_executed aside) must be identical both ways.

Prints the card's name and power limit first, then one JSON line per (traces, N): ms per trace both ways, the
launches of the many call and the speculative batches of the loop.  Usage: python tools/bench_random_ddmin_many.py [--sizes 64,1024,4096]
[--ns 1,64] [--repeats R]"""
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
FIELDS = ("mcs_size", "tests", "n_iterations", "verified", "total_replays", "tests_evaluated", "batches", "mcs_first_hit")
CAP = 1024


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
            out.append((eng.fuzzer_program(pseed + k), seed_base + k, int(res["n_events"][i]), int(res["violation"][i])))
        off += chunk
    return out[:want]


def loop(eng, execs, n):
    """the per-trace sequence: (status, mcs, sizes, keys, out) per trace, and the speculative batches (each at least
    four launches: subsequences, lane engine, warp engine, reduction)"""
    res, batches = [], 0
    mw = max(1, (max(len(e[0]) for e in execs) + 63) // 64)
    for prog, seed, maxm, v in execs:
        eng.set_externals(prog)
        p = N.FuzzParams(seed, n, maxm, INTERVAL, v, 0)
        mcs = np.zeros(mw, dtype=np.uint64)
        sizes = np.zeros(CAP, dtype=np.uint32)
        keys = np.zeros(CAP, dtype=np.uint64)
        out = N.RandomDDMinOut()
        rc = N.lib().demi_random_ddmin(eng._h, C.byref(p), 0, mcs.ctypes.data, mw, sizes.ctypes.data, keys.ctypes.data, CAP,
                                       C.byref(out))
        batches += out.batches
        k = min(out.n_iterations, CAP)
        res.append((rc, mcs, sizes[:k], keys[:k], {f: int(getattr(out, f)) for f in FIELDS}))
    return res, batches


def many(eng, execs, n):
    mw = max(1, (max(len(e[0]) for e in execs) + 63) // 64)
    mcs, sizes, keys, out, status = eng.random_ddmin_many([e[0] for e in execs], n, [e[1] for e in execs],
                                                          [e[2] for e in execs], [e[3] for e in execs], INTERVAL,
                                                          cap_iterations=CAP, mask_words=mw)
    res = []
    for t in range(len(execs)):
        k = min(int(out[t]["n_iterations"]), CAP)
        res.append((int(status[t]), mcs[t], sizes[t, :k], keys[t, :k], {f: int(out[t][f]) for f in FIELDS}))
    return res, eng.stats().kernel_launches


def same(a, b):
    return all(x[0] == y[0] and (x[0] != 0 or (list(x[1]) == list(y[1]) and list(x[2]) == list(y[2]) and
                                               list(x[3]) == list(y[3]) and x[4] == y[4])) for x, y in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="64,1024,4096")
    ap.add_argument("--ns", default="1,64")
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    print(json.dumps({"card": card()}))
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, FLAGS))
    sizes = [int(x) for x in a.sizes.split(",")]
    seed_base = 1000
    execs_all = violating_executions(eng, max(sizes), seed_base, seed_base + D.PROGRAM_SEED_OFFSET)
    print(json.dumps({"violating_executions": len(execs_all),
                      "program_events": [min(len(e[0]) for e in execs_all), max(len(e[0]) for e in execs_all)],
                      "max_messages": [min(e[2] for e in execs_all), max(e[2] for e in execs_all)]}))
    for size in sizes:
        execs = execs_all[:size]
        for n in [int(x) for x in a.ns.split(",")]:
            many(eng, execs[:8], n)                                  # warm-up: modules, buffers
            loop(eng, execs[:8], n)
            t_many, t_loop = [], []
            for _ in range(a.repeats):
                t0 = time.perf_counter()
                got, launches_many = many(eng, execs, n)
                t_many.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                want, batches_loop = loop(eng, execs, n)
                t_loop.append(time.perf_counter() - t0)
                assert same(got, want), "outputs differ"
            print(json.dumps({"traces": size, "N": n, "many_ms_per_trace": [round(1e3 * t / size, 3) for t in t_many],
                              "loop_ms_per_trace": [round(1e3 * t / size, 3) for t in t_loop],
                              "speedup_best": round(min(t_loop) / min(t_many), 2), "many_launches": launches_many, "loop_batches": batches_loop,
                              "failed_traces": sum(1 for x in got if x[0]), "identical": True}))
            sys.stdout.flush()


if __name__ == "__main__":
    main()
