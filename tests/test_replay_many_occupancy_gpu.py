"""The multi-trace K2 kernel keeps the single-trace kernel's resident blocks per SM for every model: binding a trace per
warp must not cost the headline model a block."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cuda", "replay_many_occupancy.cu")

pytestmark = pytest.mark.gpu


def test_replay_many_kernel_keeps_blocks_per_sm(tmp_path):
    exe = os.path.join(str(tmp_path), "replay_many_occupancy")
    subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", SRC, "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    rows = {l.split()[0]: (int(l.split()[1]), int(l.split()[2])) for l in out.stdout.strip().splitlines()}
    assert set(rows) == {"pingpong3", "raft5", "bcast32", "ir"}
    for model, (single, many) in rows.items():
        assert many == single >= 1, (model, single, many)
    assert rows["raft5"][0] == 4
