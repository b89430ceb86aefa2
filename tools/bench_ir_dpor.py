"""K3 on a loaded model: what the IR interpreter costs a DPOR batch, and IncrementalDDMin on the engine against the
sequential CPU oracle.

  batch   : one demi_dpor_batch launch of N pingpong3 searches (random Ping programs, max_messages 20, at most 400
            interleavings each) on the loaded model_ir.pingpong3_blob() and on compiled pingpong3.  The two give the
            same results (checked); the kernel time (CUDA events) of each, min of REPS launches after one untimed.
  incddmin: demi_incremental_ddmin on the leader election of tests/test_ir_timers_oracle.py (recording seed 10) and on
            a violating execution of the loaded pingpong3, against oracle_incremental_ddmin on the host: wall times,
            and whether MCS and counters agree.

Prints the card's name and power limit first; every number below was measured on that card in the same run."""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import demi_b200 as D  # noqa: E402
from demi_b200 import model_ir, _native as N  # noqa: E402
from oracle import binding as O  # noqa: E402
from test_ir_dpor_oracle import PP_CODE, PP_FLAGS, SHRINKING_SEED, election_recorded, pingpong_program  # noqa: E402
from test_ir_timers_oracle import TWO_LEADERS, election_model, election_program  # noqa: E402

REPS = 3


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError) as e:
        return "unknown (%s)" % e


def timed_batch(eng, progs, maxm, budget):
    ms = []
    for rep in range(REPS + 1):                       # the first launch loads the module and sizes the buffers
        res, viol, hashes = eng.dpor_batch(progs, maxm, budget, want_hashes=True)
        if rep:
            ms.append(eng.stats().kernel_ms)
    return res, hashes, min(ms)


def batch(n):
    rng = np.random.default_rng(1)
    progs = [pingpong_program(tuple(int(x) for x in rng.integers(0, 3, size=int(rng.integers(3, 7))))) for _ in range(n)]
    ir = D.Engine(D.SchedulerConfig(N.MODEL_IR, model_flags=PP_FLAGS))
    ir.load_model(model_ir.pingpong3_blob())
    compiled = D.Engine(D.SchedulerConfig(N.MODEL_PINGPONG3, model_flags=PP_FLAGS))
    a, ah, ams = timed_batch(ir, progs, 20, 400)
    b, bh, bms = timed_batch(compiled, progs, 20, 400)
    il = int(a["interleavings"].sum())
    print("batch    %5d searches, %7d interleavings, %8d deliveries | loaded %8.2f ms (%.3g interleavings/s) | "
          "compiled %8.2f ms (%.3g interleavings/s) | loaded / compiled %.2fx | identical %s"
          % (n, il, int(a["deliveries"].sum()), ams, il / ams * 1e3, bms, il / bms * 1e3, ams / bms,
             bool((a == b).all() and (ah == bh).all())))


def incddmin(name, eng, model, dext, steps, budget, rec, code, flags, mmd):
    walls = []
    for rep in range(REPS + 1):
        t0 = time.perf_counter()
        mcs, out = eng.incremental_ddmin(dext, steps, budget, rec, looking_for=code, stop_at_size=1, max_max_distance=mmd,
                                         heap_cap=1 << 16)
        if rep:
            walls.append(time.perf_counter() - t0)
    t0 = time.perf_counter()
    rc, cmcs, st = O.incremental_ddmin(model, dext, steps, budget, O.dpor_seed(*rec), max_max_distance=mmd, stop_at_size=1,
                                       looking_for=code, model_flags=flags)
    cdt = time.perf_counter() - t0
    same = bool(rc == 0 and np.array_equal(mcs, cmcs) and out.total_replays == st["total_replays"]
                and out.rounds == st["rounds"] and out.instances == st["instances"])
    print("incddmin %-9s %d externals -> %d | total_replays %3d, rounds %d, instances %3d, tests executed %4d in %3d "
          "batches | engine wall %8.2f ms (min of %d) | cpu oracle %8.2f ms | identical %s"
          % (name, len(dext), out.mcs_size, out.total_replays, out.rounds, out.instances, out.tests_executed, out.batches,
             min(walls) * 1e3, REPS, cdt * 1e3, same))


def main():
    print("card (name, power limit):", card())
    for n in (1024, 8192):
        batch(n)
    m = election_model()
    ev, par, steps, _ = election_recorded(O, SHRINKING_SEED)
    eng = D.Engine(D.SchedulerConfig(N.MODEL_IR, model_flags=m.flags))
    eng.load_model(m.blob)
    incddmin("election", eng, N.MODEL_IR, D.pack_externals(election_program(wait=False)), steps, 60, (ev, par), TWO_LEADERS,
             m.flags, 64)
    blob = model_ir.pingpong3_blob()
    O.load_model(blob)
    ev, par, r = O.fuzz_trace(N.MODEL_IR, D.pack_externals(pingpong_program(wait=True)), 1, 30, 1, model_flags=PP_FLAGS)
    peng = D.Engine(D.SchedulerConfig(N.MODEL_IR, model_flags=PP_FLAGS))
    peng.load_model(blob)
    incddmin("pingpong3", peng, N.MODEL_IR, D.pack_externals(pingpong_program()), int(r["steps"]), 200, (ev, par), PP_CODE,
             PP_FLAGS, 16)


if __name__ == "__main__":
    main()
