"""IncDDMinDriver (incddmin_driver.hpp) behind the shared rendezvous (many_rendezvous.hpp) on host threads, under
AddressSanitizer, with the CPU oracle's DPOR instances as the evaluator: every trace equals oracle_incremental_ddmin and
its own solo run, at windows 1, 7 and 512 (no GPU)."""
import os
import subprocess

import numpy as np

import demi_b200 as D
from demi_b200 import _native as N
import ir_gen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "incddmin_many_driver_test.cpp")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
MAX_MAX_DISTANCE, STOP_AT_SIZE = 16, 1          # the constants of incddmin_many_driver_test.cpp


def dpor_ext(prog):
    ext = D.pack_externals(prog)
    return ext[(ext["kind"] == N.EXT_START) | (ext["kind"] == N.EXT_SEND)]


def raft5_cases(oracle, n, budget):
    ext = D.pack_externals(D.raft5_program())
    res = oracle.fuzz_batch(N.MODEL_RAFT5, ext, 1, 3000, 40, 5, model_flags=1)
    hits = np.nonzero((res["violation"] == 1) & (res["status"] == 0))[0][:n]
    assert len(hits) == n
    out = []
    for k in hits:
        ev, par, r = oracle.fuzz_trace(N.MODEL_RAFT5, ext, 1 + int(k), 40, 5, model_flags=1)
        out.append((N.MODEL_RAFT5, 1, 1, int(r["steps"]), budget, b"", dpor_ext(D.raft5_program()), oracle.dpor_seed(ev, par)))
    return out


def generated_cases(oracle, timers, n, budget):
    """Recordings of generated loaded models (with or without timer operations) whose oracle_incremental_ddmin finishes
    without a capacity status; each is its own group, since the oracle holds one loaded model at a time."""
    out = []
    for s in range(1, 400):
        m = ir_gen.generate(s)
        if m.uses_timers != timers:
            continue
        fprog = ir_gen.program(m, s, kills=False)
        dext = dpor_ext(fprog)[:m.n_actors + 4]
        oracle.load_model(m.blob)
        ev, par, r = oracle.fuzz_trace(N.MODEL_IR, D.pack_externals(fprog), s, 12, 3, model_flags=m.flags)
        if int(r["status"]) or int(r["steps"]) < 2:
            continue
        seed = oracle.dpor_seed(ev, par)
        rc, _, _ = oracle.incremental_ddmin(N.MODEL_IR, dext, int(r["steps"]), budget, seed, max_max_distance=MAX_MAX_DISTANCE,
                                            stop_at_size=STOP_AT_SIZE, model_flags=m.flags)
        if rc != 0:
            continue
        out.append((N.MODEL_IR, m.flags, 0, int(r["steps"]), budget, bytes(m.blob), dext, seed))
        if len(out) == n:
            return out
    raise AssertionError("not enough generated models (timers=%s)" % timers)


def write_cases(path, cases):
    words = [len(cases)]
    for model, flags, code, maxm, budget, blob, ext, (nodes, trace) in cases:
        b = bytes(blob) + b"\0" * (-len(blob) % 4)
        words += [model, flags, code, maxm, budget, len(blob)] + list(np.frombuffer(b, dtype="<u4"))
        words += [len(ext)] + list(np.ascontiguousarray(ext).view("<u4"))
        words += [len(nodes)] + list(np.ascontiguousarray(nodes, dtype="<u4").ravel())
        words += [len(trace)] + list(np.ascontiguousarray(trace, dtype="<u4"))
    np.array(words, dtype="<u4").tofile(path)


def test_incddmin_drivers_behind_the_rendezvous_match_the_oracle_asan(oracle, tmp_path):
    cases = raft5_cases(oracle, 5, 40)
    cases += generated_cases(oracle, True, 3, 20)
    cases += generated_cases(oracle, False, 2, 20)
    path = os.path.join(str(tmp_path), "cases.bin")
    write_cases(path, cases)
    exe = os.path.join(str(tmp_path), "incddmin_many_driver_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address", "-fno-omit-frame-pointer", "-pthread",
                           "-I" + os.path.join(CUDA, "include"), SRC, "-o", exe, "-L" + os.path.join(ROOT, "oracle"), "-loracle",
                           "-L" + os.path.join(CUDA, "lib64"), "-lcudart",
                           "-Wl,-rpath," + os.path.join(ROOT, "oracle") + ":" + os.path.join(CUDA, "lib64")])
    out = subprocess.run([exe, path], capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr[-4000:]
    assert "%d cases" % len(cases) in out.stdout
