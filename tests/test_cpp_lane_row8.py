"""The steady raft5 lane kernel's 8-byte pending rows (demi_b200/csrc/lane_steady.hpp): the layout and the per-launch
rule that admits it, unit-tested on the host."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_lane_row8_rule(tmp_path):
    exe = os.path.join(str(tmp_path), "lane_row8_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           "-I" + os.path.join(ROOT, "demi_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "lane_row8_test.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr
