"""Fuzzing-campaign throughput (demi_fuzz_campaign_dev): RunnerUtils.fuzz's loop with a fresh Fuzzer program per
execution, on raft5 with MODEL_FLAGS = 1, max_messages = 50 and interval 5 as in bench.py.  The Fuzzer: prefix
raft5_program(), Sends of CLIENT_CMD, the reference's default FuzzerWeights, num_events 10 and 40.

Per num_events, in one process and alternated step by step:
  campaign : executions/s and deliveries/s of demi_fuzz_campaign_dev (kernel time includes generation)
  fixed    : demi_fuzz_batch_dev on raft5_program() alone (one fixed program, the bench.py headline workload)
then the share of the campaign's kernel time spent in the generator kernel (torch.profiler, a separate pass), and the
CPU oracle's campaign on all host cores.

Prints the card's name and power limit first; every number below was measured on that card in the same run.
Usage: python tools/bench_campaign.py [--n N] [--steps K] [--warmup W]"""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, ".")
import numpy as np  # noqa: E402
import torch  # noqa: E402

import demi_b200 as D  # noqa: E402
from demi_b200 import _native as N  # noqa: E402
from oracle import campaign_binding as CB  # noqa: E402

MM, INTERVAL, FLAGS, CLIENT_CMD = 50, 5, 1, 2
DEFAULT_WEIGHTS = dict(kill=0.01, send=0.3, wait_quiescence=0.1, partition=0.1, unpartition=0.1)   # Fuzzer.scala:24-29


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError) as e:
        return "unknown (%s)" % e


def timed(fn, stream):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(stream)
    fn()
    t1.record(stream)
    t1.synchronize()
    return t0.elapsed_time(t1)


def leg(num_events, n, steps, warmup):
    w = DEFAULT_WEIGHTS
    cfg = N.FuzzerConfig(w["kill"], w["send"], w["wait_quiescence"], w["partition"], w["unpartition"], num_events, CLIENT_CMD)
    prog = D.pack_externals(D.raft5_program())
    camp = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=FLAGS))
    camp.set_fuzzer(cfg, prog)
    fixed = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=FLAGS))
    fixed.set_externals(prog)
    out = torch.empty(n * 32, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream()
    c_ms, f_ms, c_del, f_del = [], [], [], []
    for step in range(warmup + steps):
        base = step * n
        ms = timed(lambda: camp.fuzz_campaign_dev(base, n, MM, INTERVAL, base, out.data_ptr(), s.cuda_stream), s)
        nv, dl = camp.fuzz_summary_dev(s.cuda_stream)
        if step >= warmup:
            c_ms.append(ms); c_del.append(dl)
        ms = timed(lambda: fixed.fuzz_batch_dev(base, n, MM, INTERVAL, out.data_ptr(), s.cuda_stream), s)
        nv, dl = fixed.fuzz_summary_dev(s.cuda_stream)
        if step >= warmup:
            f_ms.append(ms); f_del.append(dl)
    # generation share: kernel times by name, one profiled campaign call
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        camp.fuzz_campaign_dev(0, n, MM, INTERVAL, 0, out.data_ptr(), s.cuda_stream)
        torch.cuda.synchronize()
    gen = tot = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        if "fuzz" in e.key:
            tot += t
            if "fuzzer_gen_kernel" in e.key:
                gen += t
    st = camp.stats()
    print("num_events %2d | n %d x %d steps | campaign %.3e exec/s (%.3e deliveries/s), kernel ms %s, deferred %d | "
          "fixed program %.3e exec/s (%.3e deliveries/s), kernel ms %s | generation %.1f %% of the campaign's kernel time"
          % (num_events, n, steps, n * steps / (sum(c_ms) / 1e3), sum(c_del) / (sum(c_ms) / 1e3),
             ",".join("%.2f" % x for x in c_ms), st.deferred, n * steps / (sum(f_ms) / 1e3), sum(f_del) / (sum(f_ms) / 1e3),
             ",".join("%.2f" % x for x in f_ms), 100.0 * gen / tot if tot else float("nan")))
    # the CPU oracle on all host cores
    ocfg = CB.FuzzerConfig(w["kill"], w["send"], w["wait_quiescence"], w["partition"], w["unpartition"], num_events, CLIENT_CMD)
    on = 200000
    t0 = time.perf_counter()
    res = CB.fuzz_campaign(N.MODEL_RAFT5, ocfg, prog, None, 0, on, MM, INTERVAL, 0, model_flags=FLAGS)
    dt = time.perf_counter() - t0
    host = np.empty(on, dtype=N.RESULT_DTYPE)
    camp.fuzz_campaign(0, on, MM, INTERVAL, 0, out=host)
    print("num_events %2d | cpu oracle campaign on %d threads: %.3e exec/s (%d executions, %.2f s) | gpu records identical: %s"
          % (num_events, os.cpu_count() or 1, on / dt, on, dt, host.tobytes() == res.tobytes()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 23)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    print("card (name, power limit):", card())
    for ne in (10, 40):
        leg(ne, a.n, a.steps, a.warmup)


if __name__ == "__main__":
    main()
