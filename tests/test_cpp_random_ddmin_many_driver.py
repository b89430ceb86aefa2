"""RandomDDMinDriver (random_ddmin_driver.hpp) behind the shared rendezvous (many_rendezvous.hpp) on host threads, under
AddressSanitizer, with the C oracle's random-oracle tests as the evaluator: every trace equals oracle_random_ddmin and its
own solo run, at windows 1, 7 and 512 (no GPU)."""
import os
import subprocess

import numpy as np
import pytest

import demi_b200 as D
from demi_b200 import _native as N
from demi_b200.fuzzer import ClientCommandGenerator, Fuzzer, FuzzerWeights
import ir_gen
from test_random_ddmin_oracle import PP_FLAGS, RAFT_FLAGS, atoms_cover, bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "random_ddmin_many_driver_test.cpp")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")

PP_HK = D.pingpong3_program(n_sends=6)[:-1] + [D.WaitQuiescence(), D.HardKill(1), D.Send(0, 1, 50), D.Send(2, 1, 51),
                                               D.WaitQuiescence()]


@pytest.fixture(scope="module")
def rd():
    from demi_b200 import build
    build.build_oracle()
    from oracle import random_ddmin_binding
    random_ddmin_binding.lib()
    return random_ddmin_binding


def violation(rd, model, flags, prog, n, seed, maxm, interval):
    """The code of the whole program's first hit in n executions, 0 if none."""
    full = rd.random_test_batch(model, D.pack_externals(prog), bits(range(len(prog)), len(prog)), n, seed, maxm, interval,
                                model_flags=flags, threads=1)[0]
    return int(full["violation"]) if int(full["status"]) == 0 else 0


def raft5_cases(rd, want):
    """Fuzzer programs of a raft5 campaign (bench_random_ddmin.py's Fuzzer, 8 generated events) that violate, each with
    its own seed and max_messages"""
    out = []
    for s in range(1, 200):
        prog = Fuzzer(8, FuzzerWeights(), ClientCommandGenerator(2), D.raft5_program()[:-1], seed=1000 + s).generateFuzzTest()
        if not atoms_cover(prog):
            continue
        maxm = 40 + 5 * (s % 3)
        v = violation(rd, N.MODEL_RAFT5, RAFT_FLAGS, prog, 8, s, maxm, 5)
        if v:
            out.append((N.MODEL_RAFT5, RAFT_FLAGS, 8, s, maxm, 5, v, s % 2, b"", prog))
        if len(out) == want:
            return out
    raise AssertionError("not enough violating raft5 programs")


def pingpong_cases(rd):
    progs = [PP_HK, D.pingpong3_program(n_sends=6), PP_HK[:-3] + [D.WaitQuiescence()]]
    out = []
    for k, prog in enumerate(progs):
        v = violation(rd, N.MODEL_PINGPONG3, PP_FLAGS, prog, 16, 7 + k, 40, 0)
        assert v
        out.append((N.MODEL_PINGPONG3, PP_FLAGS, 16, 7 + k, 40, 0, v, k % 2, b"", prog))
    return out


def generated_cases(rd, groups):
    out = []
    from oracle import random_ddmin_binding
    for s in range(1, 60):
        m = ir_gen.generate(s)
        prog = ir_gen.program(m, s)
        if not atoms_cover(prog):
            continue
        random_ddmin_binding.load_model(m.blob)
        v = violation(rd, N.MODEL_IR, m.flags, prog, 16, s, 40, 2)
        if not v:
            continue
        out += [(N.MODEL_IR, m.flags, 16, s + k, 40, 2, v, 0, bytes(m.blob), prog) for k in range(2)]
        groups -= 1
        if not groups:
            return out
    raise AssertionError("not enough generated models")


def write_cases(path, cases):
    words = [len(cases)]
    for model, flags, n, seed, maxm, interval, looking, check, blob, prog in cases:
        b = bytes(blob) + b"\0" * (-len(blob) % 4)
        words += [model, flags, n, seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF, maxm, interval, looking, check, len(blob)]
        words += list(np.frombuffer(b, dtype="<u4"))
        ext = D.pack_externals(prog)
        words += [len(ext)] + list(np.ascontiguousarray(ext).view("<u4"))
    np.array(words, dtype="<u4").tofile(path)


def test_random_ddmin_drivers_behind_the_rendezvous_match_the_oracle_asan(rd, tmp_path):
    cases = raft5_cases(rd, 5) + pingpong_cases(rd) + generated_cases(rd, 3)
    path = os.path.join(str(tmp_path), "cases.bin")
    write_cases(path, cases)
    exe = os.path.join(str(tmp_path), "random_ddmin_many_driver_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address", "-fno-omit-frame-pointer", "-pthread",
                           "-I" + os.path.join(CUDA, "include"), SRC, "-o", exe, "-L" + os.path.join(ROOT, "oracle"),
                           "-loracle_random_ddmin", "-L" + os.path.join(CUDA, "lib64"), "-lcudart",
                           "-Wl,-rpath," + os.path.join(ROOT, "oracle") + ":" + os.path.join(CUDA, "lib64")])
    out = subprocess.run([exe, path], capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr[-4000:]
    assert "%d cases" % len(cases) in out.stdout
