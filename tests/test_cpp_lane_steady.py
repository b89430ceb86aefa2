"""The rule that decides whether a fuzz batch may run the lane engine's steady instantiation
(demi_b200/csrc/lane_steady.hpp), unit-tested on the host: it is plain C++ over the snapshot's scalars."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_lane_steady_rule(tmp_path):
    exe = os.path.join(str(tmp_path), "lane_steady_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           "-I" + os.path.join(ROOT, "demi_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "lane_steady_test.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr
