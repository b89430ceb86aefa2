"""How many loop trips a warp of the raft5 lane fuzz kernel pays per step for a delivery's sends and the next flush,
with two loops (max(sends) + max(flush items)) and with one (max(sends + flush items)), from oracle traces.

  python tools/lane_trip_model.py [--lanes 32] [--rounds 24] [--seed 10000001]          (CPU only)

The workload is bench.py's headline: raft5, depth 50, invariant every 5 deliveries, model_flags=1.  Lane l of the
modelled warp runs the prefixes seed + l + 32 r, r < rounds, one after another; warp-step i is step i of every lane
that still has one.  A lane's step is the actor sends recorded after its delivery k (sender an actor) and the timer
and external sends recorded before delivery k + 1 (sender "Timer" or deadLetters); a prefix's first step is its
initial flush.  Timers dropped as cancelled leave no event and are not counted.  This is a model of lock-step
execution, not a measurement: lanes of a real warp also wait for each other inside the receive() switch, the pick and
the invariant."""
import argparse
import os
import sys


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MAX_MESSAGES, INTERVAL, MODEL_FLAGS = 50, 5, 1


def lane_steps(O, N, ext, seed):
    """[(sends, flush items)] per step of one prefix, from its oracle trace."""
    ev, _, _ = O.fuzz_trace(N.MODEL_RAFT5, ext, seed, MAX_MESSAGES, INTERVAL, model_flags=MODEL_FLAGS)
    steps, sends, flush = [], 0, 0
    for kind, src in zip(ev["kind"].tolist(), ev["src"].tolist()):
        if kind == N.EV_MSG_EVENT:
            steps.append((sends, flush))
            sends, flush = 0, 0
        elif kind == N.EV_MSG_SEND:
            if src in (N.TIMER_SND, N.DEADLETTERS):
                flush += 1
            else:
                sends += 1
    steps.append((sends, flush))
    return steps


def model(lanes, rounds, seed):
    import demi_b200 as D
    from demi_b200 import _native as N
    from demi_b200 import build
    build.build_oracle()
    from oracle import binding as O
    ext = D.pack_externals(D.raft5_program())
    per_lane = []
    for l in range(lanes):
        st = []
        for r in range(rounds):
            st += lane_steps(O, N, ext, seed + l + lanes * r)
        per_lane.append(st)
    n_ws = max(len(s) for s in per_lane)
    sep = one = items = sends_max = flush_max = 0
    lane_sends = lane_flush = lane_steps_n = 0
    hist_s, hist_f = {}, {}
    for i in range(n_ws):
        cur = [s[i] for s in per_lane if i < len(s)]
        ms, mf = max(c[0] for c in cur), max(c[1] for c in cur)
        sends_max += ms; flush_max += mf
        sep += ms + mf
        one += max(c[0] + c[1] for c in cur)
        items += sum(c[0] + c[1] for c in cur)
        for c in cur:
            lane_sends += c[0]; lane_flush += c[1]; lane_steps_n += 1
            hist_s[c[0]] = hist_s.get(c[0], 0) + 1
            hist_f[c[1]] = hist_f.get(c[1], 0) + 1
    return {"warp_steps": n_ws, "separate": sep / n_ws, "separate_sends": sends_max / n_ws,
            "separate_flush": flush_max / n_ws, "one": one / n_ws,
            "util_separate": items / (lanes * sep), "util_one": items / (lanes * one),
            "sends_per_lane_step": lane_sends / lane_steps_n, "flush_per_lane_step": lane_flush / lane_steps_n,
            "sends_hist": {k: v / lane_steps_n for k, v in sorted(hist_s.items())},
            "flush_hist": {k: v / lane_steps_n for k, v in sorted(hist_f.items())}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=24)
    ap.add_argument("--seed", type=int, default=10000001)
    a = ap.parse_args()
    r = model(a.lanes, a.rounds, a.seed)
    print("%d lanes x %d prefixes from seed %d: %d warp-steps" % (a.lanes, a.rounds, a.seed, r["warp_steps"]))
    print("%-38s %24s %10s" % ("per warp-step", "separate loops", "one loop"))
    print("%-38s %7.2f (%.2f send + %.2f flush) %6.2f (%+.0f %%)" % (
        "trips", r["separate"], r["separate_sends"], r["separate_flush"], r["one"],
        100 * (r["one"] / r["separate"] - 1)))
    print("%-38s %24.2f %10.2f" % ("useful lane-items / (lanes x trips)", r["util_separate"], r["util_one"]))
    print("per lane-step: %.2f sends, %.2f flush items" % (r["sends_per_lane_step"], r["flush_per_lane_step"]))
    print("send counts:  " + "  ".join("%d: %.0f %%" % (k, 100 * v) for k, v in r["sends_hist"].items()))
    print("flush counts: " + "  ".join("%d: %.0f %%" % (k, 100 * v) for k, v in r["flush_hist"].items()))
    return 0


if __name__ == "__main__":
    sys.exit(main())
