"""Regenerate profiles/k1_profile.json: the profile-derived figures bench.py reports for the headline kernel.

  (on an H100)  python tools/profile_k1.py            # runs ncu on tools/profile_k1.py --workload, parses the capture

One `ncu --set full --clock-control none` capture of fuzz_lane_kernel over PREFIXES prefixes of the bench workload.
The JSON records the hash of the kernel's sources (demi_b200.build.k1_source_id); bench.py refuses figures taken
from other sources.  The ncu report itself (profiles/k1_profile.ncu-rep) is not kept in git."""
import csv
import io
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PREFIXES = 4_000_000
OUT = os.path.join(ROOT, "profiles", "k1_profile.json")
REP = os.path.join(ROOT, "profiles", "k1_profile")


def workload():
    import demi_b200 as D
    import torch
    eng = D.Engine(D.SchedulerConfig(2, model_flags=1))
    eng.set_externals(D.pack_externals(D.raft5_program()))
    out = torch.empty(PREFIXES * 32, dtype=torch.uint8, device="cuda")
    for s in range(3):
        eng.fuzz_batch_dev(1 + s * PREFIXES, PREFIXES, 50, 5, out.data_ptr(), 0)
    torch.cuda.synchronize()


def metric(rows, name):
    for r in rows:
        if r.get("Metric Name") == name:
            return float(r["Metric Value"].replace(",", ""))
    return None


def main():
    if "--workload" in sys.argv:
        return workload()
    if "--parse" in sys.argv:                       # re-read an existing capture (no GPU needed)
        raw = subprocess.run(["ncu", "-i", REP + ".ncu-rep", "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
        prof = parse(raw)
        json.dump(prof, open(OUT, "w"), indent=1)
        print(json.dumps(prof))
        return
    os.makedirs(os.path.dirname(REP), exist_ok=True)
    subprocess.check_call(["ncu", "--set", "full", "--clock-control", "none", "--import-source", "on", "-k", "regex:fuzz_lane_kernel",
                           "-s", "2", "-c", "1", "-f", "-o", REP, sys.executable, os.path.abspath(__file__), "--workload"])
    raw = subprocess.run(["ncu", "-i", REP + ".ncu-rep", "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    prof = parse(raw)
    json.dump(prof, open(OUT, "w"), indent=1)
    print(json.dumps(prof))


SCALE = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12,
         "ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3, "second": 1e3}     # bytes; milliseconds


def parse(raw):
    """`ncu --page raw --csv`: a header row, a units row, then one row per captured launch."""
    rd = list(csv.reader(io.StringIO(raw)))
    hdr, units, vals = rd[0], rd[1], rd[-1]
    m = {h: (u, v) for h, u, v in zip(hdr, units, vals)}

    def g(name):
        u, v = m.get(name, ("", ""))
        try:
            return float(v.replace(",", "")) * SCALE.get(u, 1.0)
        except ValueError:
            return None
    from demi_b200 import build
    k1_id = build.k1_source_id()
    inst = g("smsp__inst_executed.sum")
    dram = (g("dram__bytes_read.sum") or 0) + (g("dram__bytes_write.sum") or 0)
    return {
        "capture": "ncu --set full --clock-control none, fuzz_lane_kernel<Raft5,256,96>, %d prefixes (3rd launch)" % PREFIXES,
        "k1_id": k1_id, "prefixes": PREFIXES,
        "duration_ms": g("gpu__time_duration.sum"),
        "dram_bytes_read": g("dram__bytes_read.sum"), "dram_bytes_write": g("dram__bytes_write.sum"),
        "dram_bytes_per_prefix": dram / PREFIXES,
        "warp_instructions_per_prefix": inst / PREFIXES if inst else None,
        "active_lanes_per_instruction": g("smsp__thread_inst_executed_per_inst_executed.ratio"),
        "issue_slot_utilisation": (g("smsp__issue_active.avg.pct_of_peak_sustained_active") or 0) / 100.0,
        "registers_per_thread": g("launch__registers_per_thread"),
        "achieved_occupancy_pct": g("sm__warps_active.avg.pct_of_peak_sustained_active"),
        "l1_hit_rate_pct": g("l1tex__t_sector_hit_rate.pct"), "l2_hit_rate_pct": g("lts__t_sector_hit_rate.pct"),
    }


if __name__ == "__main__":
    main()
