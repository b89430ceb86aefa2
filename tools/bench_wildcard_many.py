"""Wildcard minimization (WildcardMinimizer, STSSched, ClockClusterizer) of many violating executions: the per-trace
loop against the batched path.  Both start from the same internally minimized traces (untimed: demi_ddmin_many, the
recorded MCS replay and demi_internal_minimize_many, LeftToRightOneAtATime), with raft5's clock rules:

  (a) per trace: demi_set_trace + demi_wildcard_minimize (BackTrack), then demi_wildcard_minimize (DEMI_WC_LAST_ONLY)
      on its output, which the first call leaves on the handle
  (b) demi_set_traces + demi_wildcard_minimize_many (BackTrack), demi_set_traces (its outputs) +
      demi_wildcard_minimize_many (DEMI_WC_LAST_ONLY)

on the first K in {1, 64, 1024, 16384} violating prefixes of a fuzz batch of the headline workload (bench.py's program,
max_messages, interval and model flags), and of the same program with six client commands.  Both paths run --repeats
times in turn on the same input; reports the median wall time per trace and its range, kernel launches, tests evaluated,
deliveries before and after, and whether (a) and (b) agree trace by trace in every repeat, with the card's name, power
limit and max SM clock.  (b)'s launches and tests are counted; (a)'s are derived (see run()).

  python tools/bench_wildcard_many.py [--ks 1,64,1024,16384] [--repeats 3] [--out profiles/wildcard_many_h100.txt]
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
CAP_SIZES = 1024
STAGES = (0, N.WC_LAST_ONLY)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def per_trace_loop(eng, traces, exts, codes):
    """(a): per trace, demi_set_trace then demi_wildcard_minimize twice (BackTrack, LastOnly)."""
    L = N.lib()
    k = len(traces)
    out_tr = np.zeros((k, CAP_EVENTS), dtype=N.EVENT_DTYPE)
    sizes = np.zeros((k, CAP_SIZES), dtype=np.uint32)
    outs = np.zeros((len(STAGES), k), dtype=N.INTMIN_OUT_DTYPE)
    status = np.zeros(k, dtype=np.int32)
    t0 = time.perf_counter()
    for i in range(k):
        rc = L.demi_set_trace(eng._h, traces[i].ctypes.data, len(traces[i]), exts[i].ctypes.data, len(exts[i]))
        assert rc == N.OK, L.demi_last_error(eng._h)
        for s, flags in enumerate(STAGES):
            o = N.IntMinOut()
            status[i] = L.demi_wildcard_minimize(eng._h, int(codes[i]), flags, out_tr[i].ctypes.data, CAP_EVENTS,
                                                 sizes[i].ctypes.data, CAP_SIZES, C.byref(o))
            outs[s, i] = tuple(getattr(o, f) for f, _ in N.IntMinOut._fields_)
            if status[i] != N.OK:
                break
    return time.perf_counter() - t0, out_tr, sizes, outs, status


def batched(eng, traces, exts, codes):
    """(b): set_traces + wildcard_minimize_many, twice."""
    k = len(traces)
    launches = tests = 0
    outs = np.zeros((len(STAGES), k), dtype=N.INTMIN_OUT_DTYPE)
    status = np.zeros(k, dtype=np.int32)
    alive = np.arange(k)
    t0 = time.perf_counter()
    cur = traces
    for s, flags in enumerate(STAGES):
        eng.set_traces(cur, [exts[i] for i in alive])
        tr, sizes, out, st = eng.wildcard_minimize_many(codes[alive], flags, cap_events=CAP_EVENTS, cap_sizes=CAP_SIZES)
        launches += eng.stats().kernel_launches
        tests += eng.stats().prefixes
        outs[s, alive] = out
        status[alive] = st
        ok = np.nonzero(st == N.OK)[0]
        cur = [tr[j, :min(out[j]["n_events"], CAP_EVENTS)] for j in ok]
        full_tr, full_sizes = np.zeros((k, CAP_EVENTS), dtype=N.EVENT_DTYPE), np.zeros((k, CAP_SIZES), dtype=np.uint32)
        full_tr[alive], full_sizes[alive] = tr, sizes
        alive = alive[ok]
    return time.perf_counter() - t0, full_tr, full_sizes, outs, status, launches, tests


def prepare(eng, prog, hits, codes, mw):
    """The shared starting point (untimed): the executions recorded, DDMin over each, the MCS recorded, its internal
    events minimized.  (traces, MCS externals, codes) of the executions that come through every stage."""
    ext = D.pack_externals(prog)
    ev, ne, _ = eng.fuzz_traces(1, hits, bench.MAX_MESSAGES, bench.INTERVAL, cap_events=CAP_EVENTS)
    eng.set_traces((ev, ne), ext)
    mcs, _, _, status = eng.ddmin_many(codes, mask_words=mw)
    assert (status == N.OK).all(), eng.last_error()
    mcs_ext = [D.pack_externals(D.events_of(prog, m)) for m in mcs]
    rev, rne, rres = eng.replay_traces_many(np.arange(len(ne), dtype=np.uint32), mcs, None, codes, cap_events=CAP_EVENTS)
    eng.set_traces([rev[i, :rne[i]] for i in range(len(ne))], mcs_ext)
    it, _, io, ist = eng.internal_minimize_many(codes, 0, cap_events=CAP_EVENTS, cap_sizes=CAP_SIZES)
    ok = [i for i in range(len(ne)) if ist[i] == N.OK and rres[i]["violation"] == codes[i]]
    return ([np.ascontiguousarray(it[i, :io[i]["n_events"]]) for i in ok], [mcs_ext[i] for i in ok],
            np.ascontiguousarray(codes[ok], dtype=np.uint32))


def agree(n, a, b):
    """Per trace: the two paths' statuses, records of both stages, final traces and sizes are identical."""
    ta, tra, sa, oa, sta = a
    tb, trb, sb, ob, stb = b[:5]
    last = oa[-1]
    same = (sta == stb) & (oa.view(np.uint32).reshape(len(STAGES), n, -1) ==
                           ob.view(np.uint32).reshape(len(STAGES), n, -1)).all(axis=(0, 2))
    same &= np.array([(tra[i, :min(last[i]["n_events"], CAP_EVENTS)] == trb[i, :min(ob[-1][i]["n_events"], CAP_EVENTS)]).all()
                      and (sa[i, :last[i]["n_internal_sizes"]] == sb[i, :ob[-1][i]["n_internal_sizes"]]).all()
                      for i in range(n)])
    return same


def run(name, prog, ks, n_fuzz, repeats):
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=bench.MODEL_FLAGS))
    eng.set_externals(prog)
    eng.set_clock_rules(*D.raft5_clock_rules())
    res = eng.fuzz_batch(1, n_fuzz, bench.MAX_MESSAGES, bench.INTERVAL)
    viol = np.nonzero((res["violation"] != 0) & (res["status"] == 0))[0]
    mw = max(1, (len(prog) + 63) // 64)
    rows = []
    # warm-up: every kernel and buffer the timed runs use
    hits = viol[:2].astype(np.uint32)
    traces, exts, codes = prepare(eng, prog, hits, res["violation"][hits].astype(np.uint32), mw)
    per_trace_loop(eng, traces, exts, codes)
    batched(eng, traces, exts, codes)
    for k in ks:
        if k > len(viol):
            rows.append({"program": name, "K": k, "skipped": "only %d violating prefixes in %d" % (len(viol), n_fuzz)})
            continue
        hits = viol[:k].astype(np.uint32)
        traces, exts, codes = prepare(eng, prog, hits, res["violation"][hits].astype(np.uint32), mw)
        n = len(traces)
        ta_s, tb_s, same = [], [], np.ones(n, dtype=bool)
        for _ in range(repeats):
            b = batched(eng, traces, exts, codes)
            a = per_trace_loop(eng, traces, exts, codes)
            ta_s.append(a[0])
            tb_s.append(b[0])
            same &= agree(n, a, b)
        oa, stb, lb, nb = a[3], b[4], b[5], b[6]
        # (a)'s launches and tests are not counted but derived: one launch per batch (batches) and one recording per
        # success, whose count is taken from (b) (its recording tests, nb - replays_executed), the same successes when
        # the paths agree, as identical_traces checks
        successes = int(nb - oa["replays_executed"].sum())
        la = int(oa["batches"].sum()) + successes
        na = int(oa["replays_executed"].sum()) + successes
        ta, tb = float(np.median(ta_s)), float(np.median(tb_s))
        rows.append({"program": name, "K": k, "traces": n, "repeats": repeats,
                     "a_ms_per_trace": 1e3 * ta / n, "a_ms_range": [1e3 * min(ta_s) / n, 1e3 * max(ta_s) / n],
                     "b_ms_per_trace": 1e3 * tb / n, "b_ms_range": [1e3 * min(tb_s) / n, 1e3 * max(tb_s) / n],
                     "speedup": ta / tb, "a_launches_derived": la, "b_launches": lb, "a_tests_derived": na, "b_tests": nb,
                     "deliveries_before": float(oa[0]["deliveries_before"].mean()),
                     "deliveries_after": float(oa[-1]["deliveries_after"].mean()),
                     "identical_traces": int(same.sum()), "ok_traces": int((stb == 0).sum())})
        print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,64,1024,16384")
    ap.add_argument("--fuzz", type=int, default=1 << 20, help="prefixes of the fuzz batch the violations come from")
    ap.add_argument("--repeats", type=int, default=3, help="timed runs of each path per K, alternating")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ks = [int(x) for x in a.ks.split(",")]
    gpu = card()
    rows = run("raft5_program()", D.raft5_program(), ks, a.fuzz, a.repeats)
    rows += run("raft5_program(client_cmds=6)", D.raft5_program(client_cmds=6), ks, a.fuzz, a.repeats)
    lines = ["# tools/bench_wildcard_many.py: WildcardMinimizer (STSSched, ClockClusterizer, raft5_clock_rules) of K "
             "violating raft5 executions after DDMin and internal minimization, BackTrack then LastOnly",
             "# card (name, power limit, max SM clock): " + gpu,
             "# (a) demi_set_trace + demi_wildcard_minimize twice per trace; (b) demi_set_traces + "
             "demi_wildcard_minimize_many, twice.  Both start from the same internally minimized traces and run %d times in "
             "turn: ms per trace is the median, ms_range the fastest and slowest run.  launches: kernel launches; tests: "
             "replays evaluated, recordings included.  (b)'s are counted; (a)'s are derived from (a)'s batches and "
             "executed replays plus (b)'s recordings, which are (a)'s too only when the paths agree "
             "(identical_traces).  deliveries: mean before the first stage and after the second." % a.repeats,
             "# max_messages %d, interval %d, model_flags %d" % (bench.MAX_MESSAGES, bench.INTERVAL, bench.MODEL_FLAGS)]
    lines += [json.dumps(r) for r in rows]
    text = "\n".join(lines) + "\n"
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
