"""The C++ mirror's Engine::fuzz_traces_many (include/demi_b200.hpp) against the single-trace C ABI, on the GPU."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "fuzz_traces_many_mirror_test.cpp")

pytestmark = pytest.mark.gpu


def test_cpp_mirror_fuzz_traces_many(native, tmp_path):
    native.lib()
    exe = os.path.join(str(tmp_path), "fuzz_traces_many_mirror_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), SRC, "-o", exe,
                           "-L" + os.path.join(ROOT, "demi_b200"), "-ldemi_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "demi_b200")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip().endswith("traces OK"), out.stdout + out.stderr
