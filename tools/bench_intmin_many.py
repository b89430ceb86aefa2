"""Internal-event minimization (STSSchedMinimizer) of many violating executions: the per-trace loop against the batched
path.  Both start from the same demi_ddmin_many output (the MCS of each execution):

  (a) per trace: demi_set_trace (the execution) + demi_replay_trace (MCS, verify_mcs's recording) + demi_set_trace
      (the recorded trace, the MCS) + demi_internal_minimize
  (b) demi_replay_traces_many (every MCS) + demi_set_traces (the recorded traces, their MCS) +
      demi_internal_minimize_many

on the first K in {1, 64, 1024, 16384} violating prefixes of a fuzz batch of the headline workload (bench.py's program,
max_messages, interval and model flags), and of the same program with six client commands, with LeftToRightOneAtATime.
Reports wall time per trace, kernel launches, tests evaluated and whether (a) and (b) agree trace by trace, with the
card's name, power limit and max SM clock.

  python tools/bench_intmin_many.py [--ks 1,64,1024,16384] [--out profiles/intmin_many_h100.txt]
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def per_trace_loop(eng, ev, ne, ext, mcs, mcs_ext, codes, mw):
    """(a): per execution, the recorded MCS replay, then demi_internal_minimize on it."""
    L = N.lib()
    k = len(ne)
    rec = np.zeros(CAP_EVENTS, dtype=N.EVENT_DTYPE)
    nrec = C.c_uint32()
    r1 = np.zeros(1, dtype=N.REPLAY_DTYPE)
    traces = np.zeros((k, CAP_EVENTS), dtype=N.EVENT_DTYPE)
    sizes = np.zeros((k, CAP_SIZES), dtype=np.uint32)
    outs = np.zeros(k, dtype=N.INTMIN_OUT_DTYPE)
    status = np.zeros(k, dtype=np.int32)
    t0 = time.perf_counter()
    for i in range(k):
        rc = L.demi_set_trace(eng._h, ev[i].ctypes.data, int(ne[i]), ext.ctypes.data, len(ext))
        assert rc == N.OK, L.demi_last_error(eng._h)
        rc = L.demi_replay_trace(eng._h, mcs[i].ctypes.data, mw, 0xFFFFFFFF, int(codes[i]), 0, rec.ctypes.data, CAP_EVENTS,
                                 C.byref(nrec), r1.ctypes.data)
        assert rc == N.OK, L.demi_last_error(eng._h)
        rc = L.demi_set_trace(eng._h, rec.ctypes.data, nrec.value, mcs_ext[i].ctypes.data, len(mcs_ext[i]))
        assert rc == N.OK, L.demi_last_error(eng._h)
        o = N.IntMinOut()
        status[i] = L.demi_internal_minimize(eng._h, int(codes[i]), 0, traces[i].ctypes.data, CAP_EVENTS, sizes[i].ctypes.data,
                                             CAP_SIZES, C.byref(o))
        outs[i] = tuple(getattr(o, f) for f, _ in N.IntMinOut._fields_)
    return time.perf_counter() - t0, traces, sizes, outs, status


def batched(eng, ne, mcs, mcs_ext, codes):
    """(b): replay_traces_many, set_traces, internal_minimize_many (the set holds the executions)."""
    k = len(ne)
    t0 = time.perf_counter()
    rev, rne, _ = eng.replay_traces_many(np.arange(k, dtype=np.uint32), mcs, None, codes, cap_events=CAP_EVENTS)
    rec_launches, rec_ms = eng.stats().kernel_launches, eng.stats().kernel_ms
    eng.set_traces([rev[i, :rne[i]] for i in range(k)], mcs_ext)
    traces, sizes, outs, status = eng.internal_minimize_many(codes, 0, cap_events=CAP_EVENTS, cap_sizes=CAP_SIZES)
    dt = time.perf_counter() - t0
    st = eng.stats()
    return dt, traces, sizes, outs, status, rec_launches + st.kernel_launches, k + st.prefixes, rec_ms + st.kernel_ms, st.prefixes


def prepare(eng, prog, hits, codes, mw):
    """The shared starting point: the executions recorded, set, and minimized by demi_ddmin_many (untimed)."""
    ext = D.pack_externals(prog)
    ev, ne, _ = eng.fuzz_traces(1, hits, bench.MAX_MESSAGES, bench.INTERVAL, cap_events=CAP_EVENTS)
    eng.set_traces((ev, ne), ext)
    mcs, _, _, status = eng.ddmin_many(codes, mask_words=mw)
    assert (status == N.OK).all(), eng.last_error()
    mcs_ext = [D.pack_externals(D.events_of(prog, m)) for m in mcs]
    return ext, ev, ne, mcs, mcs_ext


def run(name, prog, ks, n_fuzz):
    eng = D.Engine(D.SchedulerConfig(N.MODEL_RAFT5, model_flags=bench.MODEL_FLAGS))
    eng.set_externals(prog)
    res = eng.fuzz_batch(1, n_fuzz, bench.MAX_MESSAGES, bench.INTERVAL)
    viol = np.nonzero((res["violation"] != 0) & (res["status"] == 0))[0]
    mw = max(1, (len(prog) + 63) // 64)
    rows = []
    # warm-up: every kernel and buffer the timed runs use
    hits = viol[:2].astype(np.uint32)
    codes = res["violation"][hits].astype(np.uint32)
    ext, ev, ne, mcs, mcs_ext = prepare(eng, prog, hits, codes, mw)
    per_trace_loop(eng, ev, ne, ext, mcs, mcs_ext, codes, mw)
    eng.set_traces((ev, ne), ext)
    batched(eng, ne, mcs, mcs_ext, codes)
    for k in ks:
        if k > len(viol):
            rows.append({"program": name, "K": k, "skipped": "only %d violating prefixes in %d" % (len(viol), n_fuzz)})
            continue
        hits = viol[:k].astype(np.uint32)
        codes = res["violation"][hits].astype(np.uint32)
        ext, ev, ne, mcs, mcs_ext = prepare(eng, prog, hits, codes, mw)
        tb, trb, sb, ob, stb, lb, nb, kms, intmin_tests = batched(eng, ne, mcs, mcs_ext, codes)
        ta, tra, sa, oa, sta = per_trace_loop(eng, ev, ne, ext, mcs, mcs_ext, codes, mw)
        same = (sta == stb) & (oa.view(np.uint32).reshape(k, -1) == ob.view(np.uint32).reshape(k, -1)).all(axis=1)
        same &= np.array([(tra[i, :min(oa[i]["n_events"], CAP_EVENTS)] == trb[i, :min(ob[i]["n_events"], CAP_EVENTS)]).all() and
                          (sa[i, :oa[i]["n_internal_sizes"]] == sb[i, :ob[i]["n_internal_sizes"]]).all() for i in range(k)])
        # (a)'s launches: one recording per trace, one exact launch per batch and one recording per successful removal;
        # the recordings of successful removals are (b)'s recording tests, the same removals when the paths agree
        successes = int(intmin_tests - oa["replays_executed"].sum())
        la = k + int(oa["batches"].sum()) + successes
        na = k + int(oa["replays_executed"].sum()) + successes
        rows.append({"program": name, "K": k, "externals": len(prog),
                     "a_ms_per_trace": 1e3 * ta / k, "b_ms_per_trace": 1e3 * tb / k, "speedup": ta / tb,
                     "a_launches": la, "b_launches": lb, "a_tests": na, "b_tests": nb, "b_kernel_ms": kms,
                     "deliveries_before": float(oa["deliveries_before"].mean()),
                     "deliveries_after": float(oa["deliveries_after"].mean()), "max_batches": int(ob["batches"].max()),
                     "identical_traces": int(same.sum()), "ok_traces": int((stb == 0).sum())})
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
    lines = ["# tools/bench_intmin_many.py: STSSchedMinimizer (LeftToRightOneAtATime) of K violating raft5 executions "
             "after DDMin",
             "# card (name, power limit, max SM clock): " + gpu,
             "# (a) demi_set_trace + demi_replay_trace (MCS) + demi_set_trace + demi_internal_minimize per trace; "
             "(b) demi_replay_traces_many + demi_set_traces + demi_internal_minimize_many.  Both start from the same "
             "demi_ddmin_many output; wall time includes the MCS recording.  launches: kernel launches; tests: replays "
             "evaluated, recordings included.",
             "# max_messages %d, interval %d, model_flags %d" % (bench.MAX_MESSAGES, bench.INTERVAL, bench.MODEL_FLAGS)]
    lines += [json.dumps(r) for r in rows]
    text = "\n".join(lines) + "\n"
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
