"""DDMinDriver on many host threads at once, under AddressSanitizer, against its solo runs (no GPU)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "ddmin_driver_threads_test.cpp")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def test_ddmin_drivers_on_threads_match_solo_runs_asan(tmp_path):
    exe = os.path.join(str(tmp_path), "ddmin_driver_threads_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address", "-fno-omit-frame-pointer", "-pthread",
                           "-I" + os.path.join(CUDA, "include"), SRC, "-o", exe, "-L" + os.path.join(CUDA, "lib64"),
                           "-lcudart", "-Wl,-rpath," + os.path.join(CUDA, "lib64")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr[-4000:]
