"""The C++ host mirror's randomDDMin (demi::randomDDMin and DDMin over demi::RandomScheduler in include/demi_b200.hpp)
compiles against the C ABI, agrees with demi_random_ddmin called directly, and gives the MCS demi_b200.randomDDMin
gives."""
import os
import re
import subprocess

import pytest

import demi_b200 as D
from demi_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(native, out_dir):
    """Compiles the test into `out_dir` (the repository tree may be read-only) and returns the executable's path."""
    native.lib()
    exe = os.path.join(str(out_dir), "random_ddmin_mirror_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "random_ddmin_mirror_test.cpp"), "-o", exe,
                           "-L" + os.path.join(ROOT, "demi_b200"), "-ldemi_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "demi_b200")])
    return exe


def test_cpp_random_ddmin_mirror_without_a_gpu(native, tmp_path):
    exe = build(native, tmp_path)
    if native.lib().demi_device_count() > 0:
        pytest.skip("a CUDA device is present (covered by the gpu test)")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "no-fallback contract" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_cpp_random_ddmin_mirror_on_gpu(native, tmp_path):
    exe = build(native, tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr
    m = re.search(r"mcs((?: \d+)*) total (\d+) verified (\d) events (\d+)", out.stdout)
    mcs_idx = [int(x) for x in m.group(1).split()]
    prog = D.pingpong3_program(n_sends=6)[:-1] + [D.WaitQuiescence(), D.HardKill(1), D.Send(0, 1, 50), D.Send(2, 1, 51),
                                                  D.WaitQuiescence()]
    cfg = D.SchedulerConfig(N.MODEL_PINGPONG3, 1 | (2 << 8))
    sched = D.RandomScheduler(cfg, max_executions=64, invariant_check_interval=0, seed=7)
    trace, violation = sched.explore(prog)
    mcs, stats, verified, _ = D.randomDDMin(cfg, trace, prog, violation, max_executions=16, seed=7)
    assert [prog.index(e) for e in mcs] == mcs_idx
    assert stats.total_replays == int(m.group(2))
    assert (verified is not None) == bool(int(m.group(3)))
    if verified is not None:
        assert len(verified) == int(m.group(4))
