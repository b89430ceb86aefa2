"""WildcardDriver (wildcard_driver.hpp) in lock-step rounds over many traces, with the CPU wildcard oracle as evaluator
and recorder, against oracle_wildcard_minimize (no GPU)."""
import os
import subprocess

import numpy as np

import demi_b200 as D
from demi_b200 import _native as N
import ir_gen
from test_cpp_intmin_driver import cases_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "wildcard_driver_test.cpp")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def write_cases(path, cases):
    """cases: (model, flags, code, blob, ext, trace, rules, increment_types)"""
    words = [len(cases)]
    for model, flags, code, blob, ext, ev, rules, incr in cases:
        b = bytes(blob) + b"\0" * (-len(blob) % 4)
        words += [model, flags, code, len(blob)] + list(np.frombuffer(b, dtype="<u4"))
        words += [len(ext)] + list(np.ascontiguousarray(ext).view("<u4"))
        words += [len(ev)] + list(np.ascontiguousarray(ev).view("<u4"))
        words += [len(rules)] + [int(r) for r in rules] + [int(w) for w in N.type_set(incr)]
    np.array(words, dtype="<u4").tofile(path)


def with_rules(cases, rules, incr):
    return [c + (list(rules), list(incr)) for c in cases]


def generated_cases(oracle, n_models, rng):
    """Violating traces of timer-free generated models, each model with random clock rules and incrementing types."""
    out, seed, models = [], 0, 0
    while models < n_models and seed < 400:
        seed += 1
        m = ir_gen.generate(seed)
        if m.uses_timers:
            continue
        try:
            cs = cases_of(oracle, N.MODEL_IR, m.flags, ir_gen.program(m, seed), [40, 60][seed % 2], seed % 4, 2, blob=m.blob,
                          seeds=80)
        except AssertionError:                       # fewer than two violating executions
            continue
        types = list(range(min(m.n_types, 256)))
        rules = [N.clock_rule(int(t), int(rng.integers(0, 2)), int(rng.integers(0, 8)), int(rng.choice([1, 2, 3, 8, 32])))
                 for t in rng.choice(types, size=min(len(types), int(rng.integers(1, 5))), replace=False)]
        incr = [int(t) for t in rng.choice(types, size=min(len(types), int(rng.integers(0, 3))), replace=False)]
        out += with_rules(cs, rules, incr)
        models += 1
    assert models == n_models
    return out


def test_wildcard_drivers_in_lock_step_match_the_oracle(oracle, tmp_path):
    from oracle import wildcard_binding as W
    from test_ir_timers_oracle import (ELECT, ELECTION_INTERVAL, ELECTION_MAXM, HB, REQ, VOTE, election_model,
                                       election_program)
    W.lib()                                           # builds liboracle_wildcard.so when needed
    pp = [D.Start(a) for a in range(3)] + [D.Send(k % 3, 1, k) for k in range(10)] + [D.WaitQuiescence()]
    rules, incr = D.raft5_clock_rules()
    cases = with_rules(cases_of(oracle, N.MODEL_RAFT5, 1, D.raft5_program(), 50, 5, 8, seeds=20000), rules, incr)
    cases += with_rules(cases_of(oracle, N.MODEL_RAFT5, 1, D.raft5_program(client_cmds=6), 50, 5, 5, seeds=20000), rules, incr)
    cases += with_rules(cases_of(oracle, N.MODEL_PINGPONG3, 1, pp, -1, 0, 5), [N.clock_rule(1, 0, 0, 2)], [])
    m = election_model()
    cases += with_rules(cases_of(oracle, N.MODEL_IR, m.flags, election_program(), ELECTION_MAXM, ELECTION_INTERVAL, 5,
                                 blob=m.blob, seeds=400), [N.clock_rule(t, 0, 0, 8) for t in (REQ, VOTE, HB)], [ELECT])
    cases += generated_cases(oracle, 4, np.random.default_rng(11))
    path = os.path.join(str(tmp_path), "cases.bin")
    write_cases(path, cases)
    exe = os.path.join(str(tmp_path), "wildcard_driver_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-I" + os.path.join(CUDA, "include"), SRC, "-o", exe,
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle_wildcard", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    out = subprocess.run([exe, path], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr[-4000:]
