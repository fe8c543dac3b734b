"""The exchange of a target map sharded across ranks (pcl_b200/csrc/shard_target_kernels.cuh, driven by icp.cu:
exchange_shard_matches and fitness_score_sharded), compiled for the host: no GPU needed."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"
HOST = os.path.join(ROOT, "tests", "host")


@pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")) or shutil.which("g++") is None,
                    reason="needs g++ and the CUDA headers (vector types only; nothing is run on a device)")
def test_sharded_target_table_sets_on_the_host(tmp_path):
    """1 / 2 / 3 / 5 / 8 simulated ranks, both exchange protocols: the gathered match and record of every query equal the
    brute-force (d2, id) argmin over the whole map — exact ties across ranks, ids near 2^31 - 1, a rank out of reach, a
    random partition, points held by two ranks — and the fitness reduction, reading the keys through peer_table_set, counts exactly."""
    exe = str(tmp_path / "shard_target_host_test")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-frounding-math", "-ffp-contract=off", "-fno-fast-math",
                           "-I" + CUDA_INC, "-I" + os.path.join(ROOT, "include"), "-I" + HOST,
                           os.path.join(HOST, "shard_target_host_test.cpp"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]
    assert any(l.startswith("a tile out of reach") and "R=8 nccl" in l for l in r.stdout.splitlines())
    assert "DIFFERS" not in r.stdout
