"""DDMin with RandomScheduler as the TestOracle (demi_random_ddmin) on a violating raft5 program.

A seeded fuzzing campaign (raft5, MODEL_FLAGS = 1, max_messages 50, interval 5, raft5_program() prefix, CLIENT_CMD Sends,
the reference's default FuzzerWeights, num_events 20) gives the first violating execution k; its program is then
minimized with N = 1, 64 and 1024 executions per test, execution j under FullyRandom(seed_base + k + j), interval 5 and
max_messages = the length of the recorded EventTrace (randomDDMin's setMaxMessages(trace.size)).

Per N: engine wall time, batches, tests, tests_evaluated, total_replays and executions_executed; the C oracle's
minimization on the host (oracle/random_ddmin.c: the sequential walk in one thread, each test's executions in turn);
the threaded C oracle (oracle_random_test_batch on every host core) and the engine on the sequential walk's tests as
one batch; the MCS sizes; and the STSSched demi_ddmin MCS of the same recorded execution.  Prints the card's name and power limit
first.  Usage: python tools/bench_random_ddmin.py [--ns 1,64,1024] [--repeats R]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, ".")
import demi_b200 as D  # noqa: E402
from demi_b200 import _native as N  # noqa: E402
from demi_b200.fuzzer import ClientCommandGenerator, Fuzzer, FuzzerWeights  # noqa: E402
from oracle import random_ddmin_binding as RB  # noqa: E402

MM, INTERVAL, FLAGS, CLIENT_CMD = 50, 5, 1, 2


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ns", default="1,64,1024")
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps({"card": card(), "host_cores": os.cpu_count()}))
    cfg = D.SchedulerConfig(N.MODEL_RAFT5, FLAGS)
    eng = D.Engine(cfg)
    fz = Fuzzer(20, FuzzerWeights(), ClientCommandGenerator(CLIENT_CMD), D.raft5_program()[:-1])
    seed_base, pseed = 1000, 1000 + D.PROGRAM_SEED_OFFSET
    found = D.fuzz(fz, cfg, invariant_check_interval=INTERVAL, maxMessages=MM, max_executions=1 << 16, seed_base=seed_base,
                   program_seed_base=pseed, engine=eng)
    assert found is not None, "no violation in the campaign"
    program, k, trace, violation = found.externals, found.execution, found.trace, found.violation
    prog_events = D.unpack_externals(program)
    print(json.dumps({"execution": k, "program_events": len(program), "trace_events": len(trace), "violation": violation}))
    eng.set_trace(trace, program)
    sts_mcs, _, sts_out = eng.ddmin(violation)
    print(json.dumps({"stssched_ddmin_mcs": int(sts_out.mcs_size), "stssched_total_replays": int(sts_out.total_replays)}))
    for n in [int(x) for x in a.ns.split(",")]:
        times = []
        for _ in range(a.repeats):
            eng.set_externals(prog_events)
            t0 = time.perf_counter()
            mcs, sizes, keys, out = eng.random_ddmin(n, seed_base + k, len(trace), violation, INTERVAL)
            times.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        want = RB.random_ddmin(N.MODEL_RAFT5, program, n, seed_base + k, len(trace), violation, INTERVAL, model_flags=FLAGS)
        t_oracle = time.perf_counter() - t0
        assert want["rc"] == 0 and list(want["mcs"]) == list(mcs) and want["total_replays"] == out.total_replays
        # the tests of the sequential walk as one batch: the threaded oracle on every host core against the engine
        t0 = time.perf_counter()
        RB.random_test_batch(N.MODEL_RAFT5, program, want["tests"], n, seed_base + k, len(trace), INTERVAL, looking_for=violation,
                             model_flags=FLAGS, threads=os.cpu_count())
        t_threaded = time.perf_counter() - t0
        eng.set_externals(prog_events)
        t0 = time.perf_counter()
        eng.random_test_batch(want["tests"], n, seed_base + k, len(trace), INTERVAL, violation)
        t_engine_batch = time.perf_counter() - t0
        print(json.dumps({"N": n, "engine_wall_s": [round(t, 4) for t in times], "batches": out.batches, "tests": out.tests,
                          "tests_evaluated": out.tests_evaluated, "total_replays": out.total_replays,
                          "executions_executed": int(out.executions_executed), "mcs_size": out.mcs_size,
                          "verified": out.verified, "oracle_wall_s": round(t_oracle, 3), "oracle_equal": True,
                          "walk_tests_batch": {"tests": len(want["tests"]), "engine_s": round(t_engine_batch, 4),
                                               "threaded_oracle_s": round(t_threaded, 4), "threads": os.cpu_count()}}))


if __name__ == "__main__":
    main()
