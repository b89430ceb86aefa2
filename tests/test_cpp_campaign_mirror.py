"""The C++ host mirror's campaign driver (demi::fuzz in include/demi_b200.hpp) compiles against the C ABI, agrees with
a host loop of per-program calls, and finds the execution demi_b200.fuzz finds."""
import os
import re
import subprocess

import pytest

import demi_b200 as D
from demi_b200 import _native as N
from demi_b200 import fuzzer as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(native, out_dir):
    """Compiles the test into `out_dir` (the repository tree may be read-only) and returns the executable's path."""
    native.lib()
    exe = os.path.join(str(out_dir), "campaign_mirror_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "campaign_mirror_test.cpp"), "-o", exe,
                           "-L" + os.path.join(ROOT, "demi_b200"), "-ldemi_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "demi_b200")])
    return exe


def test_cpp_campaign_mirror_without_a_gpu(native, tmp_path):
    exe = build(native, tmp_path)
    if native.lib().demi_device_count() > 0:
        pytest.skip("a CUDA device is present (covered by the gpu test)")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "no-fallback contract" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_cpp_campaign_mirror_on_gpu(native, tmp_path):
    exe = build(native, tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr
    execution, violation = (int(x) for x in re.search(r"found (\d+) (\d+)", out.stdout).groups())
    fz = F.Fuzzer(40, F.FuzzerWeights(), F.ClientCommandGenerator(2), D.raft5_program())
    py = D.fuzz(fz, D.SchedulerConfig(N.MODEL_RAFT5, model_flags=3), maxMessages=50, invariant_check_interval=5,
                max_executions=2000)
    assert (py.execution, py.violation) == (execution, violation)
