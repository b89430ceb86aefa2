"""Wildcard (fungible-clock) minimization wall-clock on the configs[3] raft5 trace: demi_wildcard_minimize against the
sequential CPU oracle, with BackTrackStrategy (WildcardsNoBackTracks) and LastOnlyStrategy (WildcardsLastOnly).

  chain : DDMin -> internal minimization (SrcDstFIFO) -> wildcard minimization, runTheGamut's order; the wildcard
          step is timed.
  full  : the wildcard minimizer run directly on the whole 2039-event trace.

Prints the card's name and power limit first; every number below was measured on that card in the same run."""
import subprocess
import sys
import time

sys.path.insert(0, ".")
import numpy as np  # noqa: E402

import demi_b200 as D  # noqa: E402
from demi_b200 import _native as N  # noqa: E402
from tools import secondary as S  # noqa: E402
from oracle import binding as O  # noqa: E402
from oracle import wildcard_binding as W  # noqa: E402

REPS = 3


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError) as e:
        return "unknown (%s)" % e


def leg(name, eng, trace, mcs_ext, code, rules, incr, flags):
    eng.set_clock_rules(rules, incr)
    walls = []
    for rep in range(REPS + 1):                     # the first run loads the module and sizes the buffers: not timed
        eng.set_trace(trace, mcs_ext)
        t0 = time.perf_counter()
        out_trace, sizes, out = eng.wildcard_minimize(code, flags=flags)
        dt = time.perf_counter() - t0
        if rep:
            walls.append(dt)
    t0 = time.perf_counter()
    rc, ctrace, total, csizes = W.wildcard_minimize(N.MODEL_RAFT5, trace, mcs_ext, rules, incr, code, flags=flags,
                                                    model_flags=1)
    cdt = time.perf_counter() - t0
    same = bool(rc == 0 and len(out_trace) == len(ctrace) and (out_trace == ctrace).all() and out.total_replays == total
                and list(sizes) == list(csizes))
    print("%-6s %-9s base %4d events / %4d deliveries -> %4d deliveries | gpu wall %8.1f ms (min of %d; runs %s) | "
          "total_replays %5d, replays_executed %5d in %3d batches | cpu oracle %8.1f ms | identical %s"
          % (name, "LastOnly" if flags & N.WC_LAST_ONLY else "BackTrack", len(trace), out.deliveries_before,
             out.deliveries_after, min(walls) * 1e3, REPS, ", ".join("%.1f" % (w * 1e3) for w in walls),
             out.total_replays, out.replays_executed, out.batches, cdt * 1e3, same))


def main():
    print("card (name, power limit):", card())
    eng, ext, ev, par, r, seed = S.c3_trace(0)
    code = int(r["violation"])
    prog = D.raft5_program(client_cmds=S.C3_PROGRAM_CMDS)
    rules, incr = D.raft5_clock_rules()
    full = np.asarray(O.full_mask(ext), dtype=np.uint64).reshape(-1)
    eng.set_trace(ev, ext)
    rr, vtrace = eng.replay_trace(full, looking_for=code)
    full_ext = D.pack_externals([prog[k] for k in range(len(ext)) if (int(full[k >> 6]) >> (k & 63)) & 1])
    # chain: DDMin, then internal minimization, on the engine
    eng.set_trace(ev, ext)
    mcs, _, _ = eng.ddmin(code)
    mext = D.pack_externals([prog[k] for k in range(len(ext)) if (int(mcs[k >> 6]) >> (k & 63)) & 1])
    _, mtrace = eng.replay_trace(mcs, looking_for=code)
    eng.set_trace(mtrace, mext)
    itrace, _, _ = eng.internal_minimize(code, flags=N.IM_SRC_DST_FIFO)
    print("configs[3]: seed %d, %d events, violation %d; DDMin MCS %d externals, internal minimization %d -> %d events"
          % (seed, len(ev), code, len(mext), len(mtrace), len(itrace)))
    for flags in (0, N.WC_LAST_ONLY):
        leg("chain", eng, itrace, mext, code, rules, incr, flags)
    for flags in (0, N.WC_LAST_ONLY):
        leg("full", eng, vtrace, full_ext, code, rules, incr, flags)


if __name__ == "__main__":
    main()
