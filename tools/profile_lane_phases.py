"""Where the raft5 lane fuzz kernel's warp cycles go, phase by phase, on the bench workload.

  python tools/profile_lane_phases.py [--lib PATH] [--prefixes N] [--json OUT]     (on an H100)
  python tools/profile_lane_phases.py --build-only --lib PATH                      (no GPU needed)

The library is built with DEMI_K1_PHASE_CLOCK=1 under its own name (PATH, by default in a temporary directory), so
the clock build never replaces demi_b200/libdemi_b200.so.  In that build lane 0 of each warp of fuzz_lane_kernel adds
up, per phase, the clock64() cycles from the phase's entry to the next phase's entry and the active lanes at the
entry (lane_kernel.cuh, LanePhaseClock).  The workload is bench.py's headline: raft5, depth 50, invariant every 5
deliveries, model_flags=1, one launch of 10^7 prefixes after one warm-up launch.  The clock reads and the lane-0
bookkeeping slow the kernel down, so the shares are of the clock build's cycles, not of the bench build's time.

For each phase it prints the share of warp cycles, the cycles per warp-step (one pick of all 32 lanes), and the
average active lanes at the phase's entry."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ["flush", "pick", "receive", "send", "cancel", "schedule", "invariant", "tail"]   # LanePhase order
MODEL_RAFT5, MAX_MESSAGES, INTERVAL, MODEL_FLAGS = 2, 50, 5, 1


def build_phase_lib(out):
    from demi_b200 import build as b
    srcs = b._sources(b.CSRC, (".cu", ".cuh", ".h", ".hpp"))
    cus = sorted(s for s in srcs if s.endswith(".cu"))
    cmd = (["nvcc"] + b.NVCC_FLAGS + ["-DDEMI_K1_PHASE_CLOCK=1", "-DDEMI_BUILD_ID=\"%s\"" % b.source_id(),
                                       "-DDEMI_K1_ID=\"%s-phase\"" % b.k1_source_id(), "-o", out] + cus)
    subprocess.check_call(cmd, cwd=ROOT, stdout=sys.stderr)
    return out


def profile(lib_path, prefixes):
    from demi_b200 import _native
    _native.LIB_PATH = lib_path                  # must precede the first load of the library
    import demi_b200 as D
    import torch
    L = _native.lib()
    L.demi_k1_phase_read.restype = C.c_int32
    L.demi_k1_phase_read.argtypes = [C.c_void_p, C.c_int32]
    eng = D.Engine(D.SchedulerConfig(MODEL_RAFT5, model_flags=MODEL_FLAGS))
    eng.set_externals(D.pack_externals(D.raft5_program()))
    out = torch.empty(prefixes * 32, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream()
    eng.fuzz_batch_dev(1, prefixes, MAX_MESSAGES, INTERVAL, out.data_ptr(), stream.cuda_stream)    # warm-up
    torch.cuda.synchronize()
    if L.demi_k1_phase_read(None, 1) != len(PHASES):
        raise SystemExit("profile_lane_phases: %s has another phase list" % lib_path)
    seed = 1 + prefixes
    eng.fuzz_batch_dev(seed, prefixes, MAX_MESSAGES, INTERVAL, out.data_ptr(), stream.cuda_stream)
    nv, steps = eng.fuzz_summary_dev(stream.cuda_stream)
    buf = (C.c_ulonglong * (3 * len(PHASES)))()
    if L.demi_k1_phase_read(C.addressof(buf), 1) != len(PHASES):
        raise SystemExit("profile_lane_phases: demi_k1_phase_read failed")
    sums = list(buf)
    total = sum(sums[3 * p] for p in range(len(PHASES)))
    warp_steps = sums[3 * PHASES.index("pick") + 2]
    rows = []
    for p, name in enumerate(PHASES):
        cyc, lanes, n = sums[3 * p:3 * p + 3]
        rows.append({"phase": name, "cycle_share": cyc / total if total else 0.0,
                     "cycles_per_warp_step": cyc / warp_steps if warp_steps else 0.0,
                     "entries_per_warp_step": n / warp_steps if warp_steps else 0.0,
                     "active_lanes": lanes / n if n else 0.0})
    return {"prefixes": prefixes, "seed": seed, "deliveries": int(steps), "violations": int(nv),
            "warp_steps": int(warp_steps), "warp_cycles": int(total), "device": torch.cuda.get_device_name(),
            "k1_id": _native.lib().demi_version().decode().split(" k1 ")[-1], "phases": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="the clock build (built here unless it exists)")
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--prefixes", type=int, default=10_000_000)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    lib = os.path.abspath(a.lib) if a.lib else os.path.join(tempfile.mkdtemp(prefix="demi_phase_"), "libdemi_b200_phase.so")
    if not os.path.exists(lib):
        build_phase_lib(lib)
    if a.build_only:
        print(lib)
        return 0
    r = profile(lib, a.prefixes)
    print("%s  k1 %s  %d prefixes, %d deliveries, %d warp-steps" % (r["device"], r["k1_id"], r["prefixes"],
                                                                     r["deliveries"], r["warp_steps"]))
    print("%-10s %8s %14s %10s %13s" % ("phase", "cycles", "cyc/warp-step", "entries", "active lanes"))
    for row in r["phases"]:
        print("%-10s %7.1f%% %14.0f %10.2f %13.1f" % (row["phase"], 100 * row["cycle_share"], row["cycles_per_warp_step"],
                                                      row["entries_per_warp_step"], row["active_lanes"]))
    if a.json:
        json.dump(r, open(a.json, "w"), indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
