"""The steady lane kernel's tree of first deliveries (demi_b200/csrc/lane_steady.hpp) on the host: record layout,
depth rule, which nodes get children, and the key the tree is cached under."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_lane_tree_rule(tmp_path):
    exe = os.path.join(str(tmp_path), "lane_tree_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           "-I" + os.path.join(ROOT, "demi_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "lane_tree_test.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr
