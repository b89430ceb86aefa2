"""raft5 on external messages of every type (DESIGN.md §3, raft5 rules R1-R3), on the device against the CPU oracle.

The programs of raft5_gen.py reach the handlers with forged payloads and deadLetters as the sender, the lane engine's
defer paths (externals that equal a timer key) and its heartbeat-copy bookkeeping (leaders forced to step down).  Every
result field is compared bit for bit: fuzzing on both K1 engines, the warp engine alone, a low lane pending capacity and
SrcDstFIFO; recorded traces, provenance, raft5 campaigns of each protocol send type, STSSched replay with DDMin, and
frontier DPOR, all of which run the same Raft5::receive."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
import raft5_gen as G
from test_campaign_gpu import cfgs, check_campaign
from test_replay_ddmin_gpu import random_masks

pytestmark = pytest.mark.gpu

R = N.MODEL_RAFT5
FIELDS = ["violation", "steps", "state_hash", "trace_hash", "n_nodes", "n_events", "max_pending", "status"]
COUNTS = {"forged": 24, "timer": 20, "clean": 12, "hardkill": 8}
PROGRAMS = {f: G.corpus(n, f) for f, n in COUNTS.items()}
MODES = ["lane+warp", "warp-only", "lane-cap-24", "src-dst-fifo"]


def assert_same(gpu, cpu, what=""):
    for f in FIELDS:
        bad = np.nonzero(gpu[f] != cpu[f])[0]
        assert len(bad) == 0, "%s: field %s differs at %d prefixes, first idx %d: gpu=%s cpu=%s" % (
            what, f, len(bad), bad[0], gpu[bad[0]], cpu[bad[0]])


def depth(p):
    """Depth 50 / 100, invariant interval 0 / 5 / 30 and model flags 0-3, every combination over 12 seeds."""
    return (50, 100)[p.seed % 2], (0, 5, 30)[p.seed % 3], p.seed % 4


@pytest.fixture(params=MODES)
def mode(request, monkeypatch):
    monkeypatch.delenv("DEMI_DISABLE_LANE_ENGINE", raising=False)
    monkeypatch.delenv("DEMI_LANE_PENDING_CAP", raising=False)
    if request.param == "warp-only":
        monkeypatch.setenv("DEMI_DISABLE_LANE_ENGINE", "1")
    elif request.param == "lane-cap-24":
        monkeypatch.setenv("DEMI_LANE_PENDING_CAP", "24")
    return request.param


@pytest.mark.parametrize("family", sorted(COUNTS))
def test_fuzz_batch_matches_oracle(oracle, mode, family):
    fifo = mode == "src-dst-fifo"
    if fifo and family == "hardkill":
        pytest.skip("HardKill runs under FullyRandom only (actorTerminated -> FullyRandom.removeAll)")
    n, total, deferred = 2000, 0, 0
    for p in PROGRAMS[family]:
        maxm, interval, flags = depth(p)
        ext = D.pack_externals(p.events)
        eng = D.Engine(D.SchedulerConfig(R, model_flags=flags, strategy=1 if fifo else 0))
        eng.set_externals(ext)
        gpu = eng.fuzz_batch(1, n, maxm, interval, flags=1 if fifo else 0)
        deferred += eng.stats().deferred
        eng.close()
        cpu = oracle.fuzz_batch(R, ext, 1, n, maxm, interval, model_flags=flags, strategy=1 if fifo else 0,
                                flags=1 if fifo else 0)
        assert_same(gpu, cpu, repr(p))
        assert (gpu["status"] == 0).all()
        total += n
    if mode == "lane+warp" and family == "timer":
        assert 0 < deferred < total                  # executions that flush a timer-keyed external go to the warp engine
    if mode == "lane+warp" and family == "clean":
        assert deferred == 0                         # no timer keys, no kills: the lane engine keeps every execution


@pytest.mark.parametrize("family", sorted(COUNTS))
def test_event_trace_and_dep_tree_match_oracle(oracle, family):
    """The whole EventTrace and the DepTracker parents of 5 seeds of three programs of each family."""
    for p in PROGRAMS[family][:3]:
        maxm, interval, flags = depth(p)
        ext = D.pack_externals(p.events)
        eng = D.Engine(D.SchedulerConfig(R, model_flags=flags))
        eng.set_externals(ext)
        for seed in (1, 2, 3, 12345, -7):
            gev, gpar, gres = eng.fuzz_trace(seed, maxm, interval)
            cev, cpar, cres = oracle.fuzz_trace(R, ext, seed, maxm, interval, model_flags=flags)
            assert len(gev) == len(cev) and len(gpar) == len(cpar), (p, seed)
            assert (gev == cev).all() and (gpar == cpar).all(), (p, seed)
            for f in FIELDS:
                assert gres[f] == cres[f], (p, seed, f)
            assert eng.fuzz_batch(seed, 1, maxm, interval)[0]["trace_hash"] == gres["trace_hash"]
        eng.close()


@pytest.mark.parametrize("family", ["forged", "timer"])
def test_recorded_traces_match_oracle(oracle, monkeypatch, family):
    """Violating executions re-executed in recording mode (lane and warp engines): trace hash, verdict and the
    provenance masks, which follow every event's position and DepTracker parent."""
    monkeypatch.setenv("DEMI_LANE_PENDING_CAP", "24")
    checked = 0
    for p in PROGRAMS[family]:
        maxm, interval = 50, 5
        ext = D.pack_externals(p.events)
        eng = D.Engine(D.SchedulerConfig(R, model_flags=1))
        eng.set_externals(ext)
        res = eng.fuzz_batch(1, 4000, maxm, interval)
        idx = np.nonzero(res["violation"] != 0)[0][:12].astype(np.uint32)
        if len(idx) == 0:
            eng.close()
            continue
        keep, out, rec = eng.fuzz_provenance(1, idx, maxm, interval)
        assert np.array_equal(rec["trace_hash"], res["trace_hash"][idx])
        assert np.array_equal(rec["violation"], res["violation"][idx])
        for j, i in enumerate(idx):
            k, o = oracle.fuzz_provenance(R, ext, 1 + int(i), maxm, interval, keep.shape[1], model_flags=1)
            assert o["status"] == out[j]["status"] == 0
            assert np.array_equal(k, keep[j]), (p, int(i))
            for f in ("violation", "affected_mask", "n_trace", "n_kept"):
                assert o[f] == out[j][f], (p, f, int(i))
            checked += 1
        eng.close()
    assert checked >= 20


@pytest.mark.parametrize("send_type", [G.REQUEST_VOTE, G.VOTE_REPLY, G.APPEND_ENTRIES, G.APPEND_REPLY])
def test_campaign_of_protocol_sends(send_type):
    """A raft5 campaign whose generated Sends are protocol messages from deadLetters, interleaved with the BOOTs: record i
    equals oracle_fuzz_campaign's and demi_fuzz_batch of program i."""
    prefix = D.raft5_program()[:-1]
    _, got = check_campaign(R, prefix, [], cfgs(30, send_type, kill=0.02, send=0.6, wait_quiescence=0.05),
                            3000, 60, 5, model_flags=send_type % 4)
    assert (got["status"] == 0).all()


def _violating(oracle, programs, flags, maxm, interval, limit):
    for p in programs:
        ext = D.pack_externals(p.events)
        res = oracle.fuzz_batch(R, ext, 1, 3000, maxm, interval, model_flags=flags)
        hits = np.nonzero(res["violation"])[0]
        if len(hits):
            ev, _, r = oracle.fuzz_trace(R, ext, 1 + int(hits[0]), maxm, interval, model_flags=flags)
            yield p, ext, ev, int(r["violation"])
            limit -= 1
            if not limit:
                return


def test_sts_replay_and_ddmin_match_oracle(oracle):
    """STSSched replay of recorded traces of forged programs under random external subsequences, and DDMin over it."""
    done = 0
    for p, ext, ev, code in _violating(oracle, PROGRAMS["forged"], 1, 50, 5, 6):
        cfg = D.SchedulerConfig(R, model_flags=1)
        eng = D.Engine(cfg)
        eng.set_trace(ev, ext)
        masks = random_masks(ext, 800, p.seed, oracle)
        for fl in (0, N.RF_FILTER_KNOWN_ABSENTS):
            gpu = eng.replay_batch(masks, code, fl)
            cpu = oracle.replay_batch(R, ev, ext, masks, looking_for=code, flags=fl, model_flags=1)
            bad = np.nonzero(gpu != cpu)[0]
            assert len(bad) == 0, (p, fl, bad[:5], gpu[bad[:3]], cpu[bad[:3]])
        eng.close()
        rc, cmcs, total_replays, iters, verified = oracle.ddmin_sts(R, ev, ext, code, model_flags=1)
        if rc != 0:                                  # the recorded run does not reproduce under STSSched: nothing to minimize
            continue
        dd = D.DDMin(D.STSScheduler(cfg, ev, p.events), checkUnmodifed=True)
        mcs = dd.minimize(code)
        assert (D.mask_of(p.events, mcs) == cmcs).all(), p
        assert dd._stats.total_replays == total_replays and dd._stats.iteration_size == [int(x) for x in iters]
        assert dd.last.verified == verified
        done += 1
    assert done >= 2


FRONTIER_FIELDS = ["interleavings", "violations", "deliveries", "races", "keys_enqueued", "keys_dropped",
                   "explored_pairs", "pool_left", "rounds", "exhausted", "budget_exhausted", "status", "trace_slots"]


@pytest.mark.parametrize("width", [1, 64])
def test_frontier_dpor_matches_oracle(oracle, width):
    """Frontier DPOR over the Starts and Sends of forged programs (protocol-type externals included), small budget."""
    for p in PROGRAMS["forged"][:4] + PROGRAMS["timer"][:2]:
        prog = [e for e in p.events if isinstance(e, (D.Start, D.Send))]
        flags = p.seed % 4
        eng = D.Engine(D.SchedulerConfig(R, model_flags=flags))
        F = eng.frontier_params(30, 200, width, explored_slots=1 << 18, pool_cap=1 << 20)
        r, viol, hashes = eng.dpor_frontier(prog, F)
        OF = oracle.frontier_params(30, 200, width, explored_slots=1 << 18, pool_cap=1 << 20)
        rc, ores, oviol, ohashes = oracle.dpor_frontier(R, D.pack_externals(prog), OF, 1, model_flags=flags)
        assert rc == 0 and r["status"] == 0
        for f in FRONTIER_FIELDS:
            assert r[f] == ores[0][f], (p, f, r, ores[0])
        assert (hashes == ohashes[0]).all() and (viol == oviol[0]).all(), p
        eng.close()
