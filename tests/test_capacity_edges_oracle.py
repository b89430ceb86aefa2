"""The capacity edges tests/test_capacity_edges_gpu.py runs the engine at, pinned on the C oracle: each program sits
exactly at a limit of DESIGN.md §4 (the last state that fits) or one step past it.  A change to the oracle, the
program generators or the capacity formulas that moves a program off its edge fails here first.  The program that
issues more than 65 535 Uniq ids is also run through the Python restatement (tests/micro_oracle.py), event by
event."""
import collections

import numpy as np

import demi_b200 as D
from demi_b200 import _native as N
import micro_oracle as M
from test_dpor_gpu import raft_programs
from test_micro_oracle import flat, to_prog

INJECT, PING = 2, 1
PS_PENDING_OVF, PS_NODE_OVF, PS_EVENT_OVF = 1, 3, 4                     # DEMI_PS_* (include/demi_b200.h)
DS_NODE_OVF, DS_QUEUE_OVF, DS_EXPLORED_OVF, DS_HEAP_OVF = 1, 2, 3, 4    # DEMI_DS_*
BCAST32_START = [D.Start(a) for a in range(32)]


def bcast32_small_cap(n_flood, n_quiet):
    """bcast32, one segment: n_flood distinct ttl-1 injects (31 floods each) and n_quiet distinct ttl-0 injects."""
    return BCAST32_START + [D.Send(1 + j, INJECT, 1) for j in range(n_flood)] + \
        [D.Send(j % 32, INJECT, 0, 100 + j) for j in range(n_quiet)] + [D.WaitQuiescence()]


def bcast32_node_edge(extra):
    """bcast32, nine segments of one ttl-1 inject, 31 + extra ttl-0 injects in the first: 1 + 9 * 32 + 31 + extra
    DepTracker nodes on every schedule; 40 + extra Sends give pending_cap 128 and node_cap 2 * 128 + 64 = 320."""
    ev = list(BCAST32_START)
    for s in range(9):
        ev.append(D.Send(s + 1, INJECT, 1))
        if s == 0:
            ev += [D.Send(j % 32, INJECT, 0, 100 + j) for j in range(31 + extra)]
        ev.append(D.WaitQuiescence())
    return ev


def hard_kill_program(k):
    """pingpong3, actor 1 blocked: k Pings to it are all pending at the quiescent point, then HardKill(1) removes all k.
    k <= 119 gives pending_cap 128; k <= 111 also fits the send queue of the warp engine's shared-memory tier."""
    return [D.Start(a) for a in range(3)] + [D.Send(1, PING, i) for i in range(k)] + \
        [D.WaitQuiescence(), D.HardKill(1), D.Send(0, PING, 999), D.WaitQuiescence()]


def uniq_wrap_program(segments=34, per=1000):
    """pingpong3, unbounded: identical Sends reuse DepTracker nodes, so the execution issues ~2 Uniq ids per Send
    (68 000 here) on 3 nodes."""
    ev = [D.Start(a) for a in range(3)]
    for _ in range(segments):
        ev += [D.Send(0, PING, 5)] * per + [D.WaitQuiescence()]
    return ev


# (n_flood, n_quiet, pending_cap, {status: count} over seeds 1..400, prefixes with max_pending == pending_cap and status 0)
SMALL_CAPS = [(3, 0, 64, {0: 275, 1: 125}, 6),
              (5, 21, 128, {0: 380, 1: 20}, 3),
              (11, 79, 256, {0: 389, 1: 11}, 3)]
HARD_KILL_K = (64, 65, 70, 111, 112, 119, 120)


def pending_cap(model, max_messages, n_sends):
    """demi_pending_cap (include/demi_limits.h): the model's worst-case bound, rounded up to a power of two in
    [64, 8192]."""
    d = 0 if max_messages < 0 else min(max_messages, 100000)
    bound = n_sends + {N.MODEL_PINGPONG3: 8, N.MODEL_RAFT5: 16 + 4 * (d + 1), N.MODEL_BCAST32: 8 + 31 * (d + 1)}[model]
    c = 64
    while c < bound and c < 8192:
        c *= 2
    return c


def node_cap(pcap):
    return min(2 * pcap + 64, 65535)


def statuses(r):
    return dict(collections.Counter(int(s) for s in r["status"]))


def test_pending_cap_edges_on_bcast32(oracle):
    for n_flood, n_quiet, cap, counts, at_cap in SMALL_CAPS:
        ext = D.pack_externals(bcast32_small_cap(n_flood, n_quiet))
        assert pending_cap(N.MODEL_BCAST32, -1, n_flood + n_quiet) == cap
        r = oracle.fuzz_batch(N.MODEL_BCAST32, ext, 1, 400, -1, 0)
        ok = r["status"] == 0
        assert statuses(r) == counts
        assert int(r["max_pending"][ok].max()) == cap and int((r["max_pending"][ok] == cap).sum()) == at_cap


def test_pending_cap_clamp_on_bcast32(oracle):
    """bcast32_program(4) at depth 900 would need 27 939 entries: the cap is clamped to 8192."""
    assert pending_cap(N.MODEL_BCAST32, 900, 1) == 8192
    r = oracle.fuzz_batch(N.MODEL_BCAST32, D.pack_externals(D.bcast32_program(4)), 1, 500, 900, 0)
    assert statuses(r) == {0: 310, 1: 190}
    assert int(r["max_pending"][r["status"] == 0].max()) == 8190


def test_node_cap_edge_on_bcast32(oracle):
    assert node_cap(pending_cap(N.MODEL_BCAST32, -1, 41)) == 320
    r = oracle.fuzz_batch(N.MODEL_BCAST32, D.pack_externals(bcast32_node_edge(0)), 1, 300, -1, 0)
    assert statuses(r) == {0: 300} and (r["n_nodes"] == 320).all()
    r = oracle.fuzz_batch(N.MODEL_BCAST32, D.pack_externals(bcast32_node_edge(1)), 1, 300, -1, 0)
    assert statuses(r) == {PS_NODE_OVF: 300}


def run_micro_pingpong(prog, seed):
    actors = {str(i): M.PingPongActor(i) for i in range(3)}
    ex = M.Execution(actors, to_prog(prog), seed, -1, 0, M.pingpong_invariant(0), lambda m: m[0] == PING,
                     fresh_actor=lambda name: M.PingPongActor(int(name)))
    v = ex.run()
    return ex, v or 0


def same_execution(oracle, prog, seed, cap_events):
    ext = D.pack_externals(prog)
    r = oracle.fuzz_batch(N.MODEL_PINGPONG3, ext, seed, 1, -1, 0)[0]
    ev, par, _ = oracle.fuzz_trace(N.MODEL_PINGPONG3, ext, seed, -1, 0, cap_events=cap_events)
    ex, v = run_micro_pingpong(prog, seed)
    assert (int(r["violation"]), int(r["steps"]), int(r["n_nodes"]), int(r["max_pending"]), int(r["status"])) == \
        (v, ex.messagesScheduledSoFar, ex.depTracker.next_id, ex.max_pending, 0)
    assert int(r["n_events"]) == min(len(ex.events), 0xFFFF)                 # the result field saturates
    got = [(int(e["kind"]), int(e["src"]), int(e["dst"]), int(e["type"]), int(e["p0"]), int(e["p1"]), int(e["uniq"]),
            int(e["node"])) for e in ev]
    assert got == flat(ex.events)
    assert [int(x) for x in par] == [ex.depTracker.parent_of[i] for i in range(ex.depTracker.next_id)]
    return r, ev


def test_hard_kill_family(oracle):
    """HardKill(1) of the blocked actor removes its k pending Pings whatever k is, so every schedule makes one
    delivery (Ping 999 to actor 0, whose Pong to the killed actor is dropped), with status 0 and max_pending k."""
    for k in HARD_KILL_K:
        prog = hard_kill_program(k)
        r = oracle.fuzz_batch(N.MODEL_PINGPONG3, D.pack_externals(prog), 1, 50, -1, 0, blocked_mask=0b010)
        assert statuses(r) == {0: 50}
        assert (r["max_pending"] == k).all() and (r["steps"] == 1).all() and (r["n_events"] == k + 10).all()
        assert pending_cap(N.MODEL_PINGPONG3, -1, k + 1) == (128 if k <= 119 else 256)


def test_uniq_ids_wrap_at_65536(oracle):
    """Uniq ids are 16-bit (DESIGN.md §2): past 65 535 they wrap to 0, and the node field keeps the DepTracker node."""
    prog = uniq_wrap_program()
    r, ev = same_execution(oracle, prog, 1, cap_events=1 << 18)
    assert (int(r["status"]), int(r["n_nodes"]), int(r["n_events"]), int(r["steps"])) == (0, 3, 0xFFFF, 68000)
    sends = ev[ev["kind"] == N.EV_MSG_SEND]
    assert len(sends) == 68000 and int(sends["node"].max()) == 2
    assert np.array_equal(sends["uniq"], (np.arange(1, 68001) & 0xFFFF).astype(np.uint16))


# ---- K3 DPOR.  Each cap: the smallest value at which the search ends with status 0, and the status one below it
# (half of it for explored_slots, a power of two).  DPOR_BASE holds the other caps.
DPOR_BASE = dict(node_cap=4096, explored_slots=1 << 16, heap_cap=1 << 15)
# the first search of test_dpor_gpu's raft set, depth 24, 400 interleavings: default ordering, the bucket queue
DPOR_BUCKET_EDGES = [("node_cap", 32, 31, DS_NODE_OVF), ("heap_cap", 391, 390, DS_HEAP_OVF),
                     ("explored_slots", 128, 64, DS_EXPLORED_OVF)]
# ArvindDistanceOrdering + prioritizePendingUponDivergence seeded with a recorded raft5 execution: the binary heap
DPOR_HEAP_EDGES = [("node_cap", 158, 157, DS_NODE_OVF), ("heap_cap", 1682, 1681, DS_HEAP_OVF),
                   ("explored_slots", 1024, 512, DS_EXPLORED_OVF)]
DPOR_HEAP_BUDGET = 60


def dpor_bucket_program():
    return raft_programs(1, np.random.default_rng(1))[0]


def raft5_seed_world(oracle):
    """The DPOR externals of raft5_program() (Start / Send) and the recording of fuzz seed 2 at depth 40, the first
    execution there that shows violation 1."""
    ext_all = D.pack_externals(D.raft5_program())
    dext = ext_all[(ext_all["kind"] == N.EXT_SEND) | (ext_all["kind"] == N.EXT_START)]
    ev, par, r = oracle.fuzz_trace(N.MODEL_RAFT5, ext_all, 2, 40, 5, model_flags=1)
    assert int(r["violation"]) == 1 and int(r["steps"]) == 25 and len(par) == 46
    return dext, ev, par, int(r["steps"])


def dpor_heap_instance(oracle, dext, ev, par, steps, **caps):
    c = dict(DPOR_BASE, heap_cap=1 << 16); c.update(caps)
    inst = oracle.DporInstance(N.MODEL_RAFT5, dext[np.arange(len(dext)) != 7], steps, DPOR_HEAP_BUDGET,
                               seed=oracle.dpor_seed(ev, par), arvind=1, prioritize_pending=1, model_flags=1,
                               looking_for=0, stop_if_found=0, **c)
    r, h = inst.test(-1)
    inst.close()
    return r, h


def test_dpor_cap_edges(oracle):
    ext = D.pack_externals(dpor_bucket_program())
    for key, edge, below, status in DPOR_BUCKET_EDGES:
        for value, want in ((edge, 0), (below, status)):
            _, r, _, _ = oracle.dpor_search(N.MODEL_RAFT5, ext, 24, 400, 0, 0, -1, model_flags=1, **dict(DPOR_BASE, **{key: value}))
            assert int(r["status"]) == want, (key, value)
    world = raft5_seed_world(oracle)
    for key, edge, below, status in DPOR_HEAP_EDGES:
        for value, want in ((edge, 0), (below, status)):
            assert int(dpor_heap_instance(oracle, *world, **{key: value})[0]["status"]) == want, (key, value)


def dpor_queue_program(n):
    """n Sends to actor 0: n entries on the one FIFO (deadLetters, 0); DPOR_QCAP is 256."""
    return [D.Start(a) for a in range(3)] + [D.Send(0, PING, i) for i in range(n)]


def test_dpor_queue_edge(oracle):
    _, r, _, _ = oracle.dpor_search(N.MODEL_PINGPONG3, D.pack_externals(dpor_queue_program(256)), 4, 8)
    assert int(r["status"]) == 0 and int(r["n_nodes"]) == 259
    _, r, _, _ = oracle.dpor_search(N.MODEL_PINGPONG3, D.pack_externals(dpor_queue_program(257)), 4, 8)
    assert int(r["status"]) == DS_QUEUE_OVF


def long_seed_search(oracle, dext, ev, par, trace_len=None):
    """A seeded search whose initial trace (42 entries) is far longer than max_messages + 2 = 10: with
    prioritizePendingUponDivergence one scheduling step may skip many of its entries."""
    nodes, trace = oracle.dpor_seed(ev, par)
    keep = np.arange(len(dext)) != 5
    inst = oracle.DporInstance(N.MODEL_RAFT5, dext[keep], 8, 30, seed=(nodes, trace[:trace_len]), prioritize_pending=1,
                               model_flags=1, looking_for=1)
    r, h = inst.test(-1)
    inst.close()
    return r, h


def test_dpor_follows_the_whole_initial_trace(oracle):
    """nextTrace is not bounded in DPORwHeuristics: the search follows the whole initial trace.  Cut at
    max_messages + 2 entries (the longest trace an interleaving can record) it takes other schedules, so no engine
    may keep only that much of it."""
    ext_all = D.pack_externals(D.raft5_program())
    dext = ext_all[(ext_all["kind"] == N.EXT_SEND) | (ext_all["kind"] == N.EXT_START)]
    ev, par, _ = oracle.fuzz_trace(N.MODEL_RAFT5, ext_all, 1, 40, 5, model_flags=1)
    assert len(oracle.dpor_seed(ev, par)[1]) == 42
    whole, hw = long_seed_search(oracle, dext, ev, par)
    cut, hc = long_seed_search(oracle, dext, ev, par, trace_len=10)
    assert int(whole["status"]) == int(cut["status"]) == 0
    assert hw.tolist() != hc.tolist()
