"""IntMinDriver (intmin_driver.hpp) in lock-step rounds over many traces, with the CPU oracle as evaluator and recorder,
against oracle_internal_minimize (no GPU)."""
import os
import subprocess

import numpy as np

import demi_b200 as D
from demi_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "intmin_driver_test.cpp")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def cases_of(oracle, model, flags, prog, maxm, interval, n, blob=None, seeds=3000):
    """(model, flags, code, blob, externals, verified trace) of the first n violating executions: each trace is the
    recording of its execution's full externals, so the externals are its MCS."""
    ext = D.pack_externals(prog)
    if blob is not None:
        oracle.load_model(blob)
    res = oracle.fuzz_batch(model, ext, 1, seeds, maxm, interval, model_flags=flags)
    hits = np.nonzero((res["violation"] != 0) & (res["status"] == 0))[0][:n]
    assert len(hits) == n
    out = []
    for k in hits:
        ev, _, r = oracle.fuzz_trace(model, ext, 1 + int(k), maxm, interval, model_flags=flags)
        code = int(r["violation"])
        rr, vt = oracle.replay_trace(model, ev, ext, oracle.full_mask(ext, False), looking_for=code, model_flags=flags)
        assert rr["status"] == 0
        out.append((model, flags, code, blob or b"", ext, vt))
    return out


def write_cases(path, cases):
    words = [len(cases)]
    for model, flags, code, blob, ext, ev in cases:
        b = bytes(blob) + b"\0" * (-len(blob) % 4)
        words += [model, flags, code, len(blob)] + list(np.frombuffer(b, dtype="<u4"))
        words += [len(ext)] + list(np.ascontiguousarray(ext).view("<u4"))
        words += [len(ev)] + list(np.ascontiguousarray(ev).view("<u4"))
    np.array(words, dtype="<u4").tofile(path)


def test_intmin_drivers_in_lock_step_match_the_oracle(oracle, tmp_path):
    from test_ir_timers_oracle import ELECTION_INTERVAL, ELECTION_MAXM, election_model, election_program
    pp = [D.Start(a) for a in range(3)] + [D.Send(k % 3, 1, k) for k in range(10)] + [D.WaitQuiescence()]
    m = election_model()
    cases = cases_of(oracle, N.MODEL_RAFT5, 1, D.raft5_program(), 50, 5, 10, seeds=20000)
    cases += cases_of(oracle, N.MODEL_RAFT5, 1, D.raft5_program(client_cmds=6), 50, 5, 6, seeds=20000)
    cases += cases_of(oracle, N.MODEL_PINGPONG3, 1, pp, -1, 0, 6)
    cases += cases_of(oracle, N.MODEL_IR, m.flags, election_program(), ELECTION_MAXM, ELECTION_INTERVAL, 6, blob=m.blob,
                      seeds=400)
    path = os.path.join(str(tmp_path), "cases.bin")
    write_cases(path, cases)
    exe = os.path.join(str(tmp_path), "intmin_driver_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-I" + os.path.join(CUDA, "include"), SRC, "-o", exe,
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    out = subprocess.run([exe, path], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr[-4000:]
