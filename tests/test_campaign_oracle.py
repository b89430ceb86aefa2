"""The Fuzzer three ways and the CPU campaign: the oracle's C restatement of Fuzzer.generateFuzzTest equals the Python
restatement (demi_b200/fuzzer.py, message counter restarted per program) and the engine's demi_fuzzer_generate, and
record i of oracle_fuzz_campaign is oracle_fuzz_batch on program i."""
import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import fuzzer as F

FIELDS = ("kind", "a", "b", "type", "p0", "p1")


def _cfg(native, num_events, send_type, **kw):
    w = dict(kill=0.01, send=0.3, wait_quiescence=0.1, partition=0.1, unpartition=0.1)
    w.update(kw)
    return w, native.FuzzerConfig(w["kill"], w["send"], w["wait_quiescence"], w["partition"], w["unpartition"], num_events, send_type)


def _starts(n):
    return [D.Start(a) for a in range(n)]


# (name, prefix, postfix, num_events, send_type, weights)
CASES = [
    ("raft5_default", D.raft5_program(), [], 40, 2, {}),
    ("kill_heavy", _starts(5) + [D.Send(a, 1, 0x1F) for a in range(5)], [], 60, 2, dict(kill=0.5, send=0.2)),
    ("partition_heavy", _starts(16), [], 80, 1, dict(kill=0.0, partition=0.5, unpartition=0.4, wait_quiescence=0.05)),
    ("prefix_ends_wq_with_postfix", _starts(5) + [D.WaitQuiescence()], [D.Send(0, 2, 99), D.Kill(3)], 30, 2, {}),
    ("one_actor", _starts(1), [D.Send(0, 1, 7)], 25, 1, dict(partition=0.3)),
    ("bcast32", _starts(32) + [D.Send(0, 2, 3), D.WaitQuiescence()], [D.Partition(1, 2)], 50, 2, dict(partition=0.3, unpartition=0.2)),
]


def _python_program(prefix, postfix, num_events, send_type, w, seed):
    f = F.Fuzzer(num_events, F.FuzzerWeights(**w), F.ClientCommandGenerator(send_type), prefix, postfix, seed=seed)
    return D.pack_externals(f.generateFuzzTest())


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_c_fuzzer_equals_engine_and_python(native, case):
    from oracle import campaign_binding as CB
    name, prefix, postfix, num_events, send_type, kw = case
    w, cfg = _cfg(native, num_events, send_type, **kw)
    ocfg = CB.FuzzerConfig(w["kill"], w["send"], w["wait_quiescence"], w["partition"], w["unpartition"], num_events, send_type)
    pre, post = D.pack_externals(prefix), D.pack_externals(postfix)
    lengths, py_checked, py_raised = set(), 0, 0
    for seed in range(-5, 10000):
        got = CB.fuzzer_generate(ocfg, seed, pre, post)
        want = native.fuzzer_generate(cfg, seed, pre, post)
        assert np.array_equal(got, want), (name, seed)                 # every field, ids included
        lengths.add(len(got))
        if seed % 5 == 0:                                              # the Python restatement on 2000 seeds per case
            try:
                py = _python_program(prefix, postfix, num_events, send_type, w, seed)
            except ValueError:                                         # a Send drawn with everyone killed: nextInt(0)
                py_raised += 1
                continue
            assert len(py) == len(got), (name, seed)
            for f in FIELDS:
                assert (py[f] == got[f]).all(), (name, seed, f)
            py_checked += 1
    assert py_checked > 1000
    if name == "kill_heavy":
        full = len(pre) + num_events + 1
        assert min(lengths) < full                                     # generation ended early on a Kill with nobody alive


def test_early_end_has_no_postfix_and_counter_restarts(native):
    from oracle import campaign_binding as CB
    w, cfg = _cfg(native, 60, 2, kill=0.6, send=0.2)
    ocfg = CB.FuzzerConfig(w["kill"], w["send"], w["wait_quiescence"], w["partition"], w["unpartition"], 60, 2)
    pre, post = D.pack_externals(_starts(3)), D.pack_externals([D.Send(0, 1, 5)])
    early = 0
    for seed in range(200):
        p = CB.fuzzer_generate(ocfg, seed, pre, post)
        sends = p[len(pre):][(p[len(pre):]["kind"] == native.EXT_SEND) & (p[len(pre):]["type"] == 2)]
        assert list(sends["p0"]) == list(range(1, len(sends) + 1))     # message_gen's counter starts at 1 per program
        if len(p) < len(pre) + 60 + 2:
            early += 1
            assert not ((p["kind"] == native.EXT_SEND) & (p["p0"] == 5) & (p["type"] == 1)).any()   # no postfix
    assert early > 0
    ids = CB.fuzzer_generate(ocfg, 3, D.pack_externals([D.Start(0, _id=40)]), D.pack_externals([D.Send(0, 1, 5, _id=90)]))["id"]
    assert ids[0] == 40 and (ids[1:] > 90).all()                       # ids go on from the largest fixed id


def test_oracle_campaign_record_is_the_fixed_program_batch(oracle):
    from oracle import campaign_binding as CB
    ocfg = CB.FuzzerConfig(0.01, 0.3, 0.1, 0.1, 0.1, 20, 2)
    pre = D.pack_externals(D.raft5_program())
    n, sb, pb = 300, 1000, 77
    res = CB.fuzz_campaign(2, ocfg, pre, None, sb, n, 50, 5, pb, model_flags=1)
    for i in range(0, n, 7):
        prog = CB.fuzzer_generate(ocfg, pb + i, pre)
        want = oracle.fuzz_batch(2, prog, sb + i, 1, 50, 5, model_flags=1)[0]
        assert res[i].tobytes() == want.tobytes(), i
    assert (res["violation"] != 0).any() and (res["status"] == 0).all()
    # chunking does not matter: two halves with shifted bases
    a = CB.fuzz_campaign(2, ocfg, pre, None, sb, 150, 50, 5, pb, model_flags=1, threads=3)
    b = CB.fuzz_campaign(2, ocfg, pre, None, sb + 150, 150, 50, 5, pb + 150, model_flags=1)
    assert np.concatenate([a, b]).tobytes() == res.tobytes()
