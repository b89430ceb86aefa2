"""The headline with and without the lane kernel's steady instantiation: this tree against a checkout of its parent
commit, alternated in one session on one GPU.

  git worktree add build/parent HEAD~1          (or any checkout of the commit to compare with)
  python tools/bench_lane_steady.py --parent build/parent [--runs 4] [--out DIR]     (on an H100)
  python tools/bench_lane_steady.py --parent build/parent --build-only               (no GPU needed)

Each tree's libraries are built by its own demi_b200/build.py if they are missing.  The card's name, power limit and
maximum SM clock are printed first (an nvidia-smi query; they are part of every figure below).  Then each tree's
`bench.py --gpus 1 --steps 20 --warmup 5 --dump-outputs DIR` runs `--runs` times, parent and this tree in turn, so
that a drift of the card's clocks falls on both alike.  bench.py times the same seeds in every run, so the dumped
arrays (a seeded sample of the last step's records, and that step's counters) must be identical in all of them: they
are compared array for array.  The verdict line says whether the slowest run of this tree beat the fastest of the
parent."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SECONDARY = ["c2_dpor", "c3_ddmin", "c4_bcast_dedup"]


def secondary_value(j, leg):
    """(value, unit) of a secondary leg of a bench.py line (configs[2]'s figure is its frontier search's), or None."""
    r = j.get("secondary", {}).get(leg, {})
    r = r if "value" in r else r.get("frontier", {})
    return (r["value"], r.get("unit", "")) if "value" in r else None


def build(tree):
    if not os.path.exists(os.path.join(tree, "demi_b200", "libdemi_b200.so")) or \
            not os.path.exists(os.path.join(tree, "oracle", "liboracle.so")):
        subprocess.check_call([sys.executable, os.path.join(tree, "demi_b200", "build.py")], cwd=tree, stdout=sys.stderr)


def bench(tree, out_dir, steps, warmup):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
           "--dump-outputs", out_dir]
    out = subprocess.run(cmd, cwd=tree, capture_output=True, text=True)
    if out.returncode != 0:
        raise SystemExit("bench.py failed in %s:\n%s" % (tree, out.stderr[-4000:]))
    return json.loads(out.stdout.strip().splitlines()[-1])


def same_arrays(a, b):
    """Names of the arrays that differ between two --dump-outputs directories (a missing file differs)."""
    names = sorted(set(os.listdir(a)) | set(os.listdir(b)))
    bad = []
    for n in names:
        pa, pb = os.path.join(a, n), os.path.join(b, n)
        if not (os.path.exists(pa) and os.path.exists(pb)) or not np.array_equal(np.load(pa), np.load(pb)):
            bad.append(n)
    return names, bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True, help="a checkout of the commit to compare with")
    ap.add_argument("--runs", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="where the --dump-outputs directories go (default: a temporary directory)")
    ap.add_argument("--build-only", action="store_true")
    a = ap.parse_args()
    trees = {"parent": os.path.abspath(a.parent), "steady": ROOT}
    for t in trees.values():
        build(t)
    if a.build_only:
        return 0
    out = os.path.abspath(a.out) if a.out else tempfile.mkdtemp(prefix="demi_lane_steady_")
    os.makedirs(out, exist_ok=True)
    print(subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], text=True).strip())
    print("bench.py --gpus 1 --steps %d --warmup %d, %d runs per build, alternated (parent first)" % (a.steps, a.warmup, a.runs))
    runs = {k: [] for k in trees}
    for r in range(a.runs):
        for k, tree in trees.items():
            d = os.path.join(out, "%s_%d" % (k, r))
            j = bench(tree, d, a.steps, a.warmup)
            runs[k].append((j, d))
            sec = {s: secondary_value(j, s) for s in SECONDARY}
            print("%-6s run %d  k1 %s  %.4e prefixes/s  %.3f ms/step  violations_last_step %d  launches %d  e2e %.4e  | %s" % (
                k, r, j["k1_id"], j["value"], j["ms_per_step"], j["violations_last_step"], j["gpu_launches"], j["e2e"]["value"],
                "  ".join("%s %.4e %s" % ((s,) + sec[s]) for s in SECONDARY if sec[s])))
            sys.stdout.flush()
    ref = runs["parent"][0][1]
    names, _ = same_arrays(ref, ref)
    differing = {}
    for k in trees:
        for j, d in runs[k]:
            _, bad = same_arrays(ref, d)
            if bad:
                differing[os.path.basename(d)] = bad
    counters = {os.path.basename(d): np.load(os.path.join(d, "step_counters.npy")).astype(np.uint64).tolist()
                for k in trees for _, d in runs[k]}
    print("dumped arrays (%d: %s): %s" % (len(names), " ".join(n[:-4] for n in names),
                                        "identical in all %d runs" % (2 * a.runs) if not differing else "DIFFER: %r" % differing))
    print("step_counters [violations, deliveries] of the last step: %s" % (
        "%r in every run" % counters["parent_0"] if len({tuple(v) for v in counters.values()}) == 1 else repr(counters)))
    v = {k: [j["value"] for j, _ in runs[k]] for k in trees}
    for k in trees:
        print("%-6s prefixes/s  min %.4e  max %.4e  spread %.2f %%" % (k, min(v[k]), max(v[k]), 100 * (max(v[k]) / min(v[k]) - 1)))
    print("slowest steady run / fastest parent run = %.4f   mean / mean = %.4f" % (
        min(v["steady"]) / max(v["parent"]), np.mean(v["steady"]) / np.mean(v["parent"])))
    for s in SECONDARY:
        sv = {k: [secondary_value(j, s)[0] for j, _ in runs[k] if secondary_value(j, s)] for k in trees}
        if sv["parent"] and sv["steady"]:
            print("%-15s parent %.4e .. %.4e   steady %.4e .. %.4e" % (s, min(sv["parent"]), max(sv["parent"]),
                                                                        min(sv["steady"]), max(sv["steady"])))
    return 1 if differing else 0


if __name__ == "__main__":
    sys.exit(main())
