"""The correspondence rejector chain on a source sharded across ranks (reject.cu: apply_rejector_sharded, comm.cu: the u64
exchanges, reject_sharded_kernels.cuh): every rank must accept exactly what one process accepts over the concatenation
of the shards in rank order."""
import os
import shutil
import socket
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"
HOST = os.path.join(ROOT, "tests", "host")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _torchrun(nproc, script):
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                        "--master-addr", "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "tests", script)],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-4000:], r.stderr[-3000:])
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [2, 3])
def test_sharded_rejector_chains_share_one_gpu(nproc):
    """2 / 3 processes on cuda:0, peer exchange bootstrapped over gloo (comm_export / _import), uneven contiguous shards:
    each device rejector alone, the four-rejector chain (SVD, point-to-plane) and surface-normal + chain (point-to-plane).
    Iteration 1: the concatenated per-rank correspondences equal the single-process list exactly (smooth surface with
    outliers; a lattice scene with exact distance ties across shard boundaries).  Full align: bitwise the same transform
    on every rank; same iterations and correspondence counts as the single process, transform within 1e-6."""
    r = _torchrun(nproc, "_two_rank_one_gpu_rejectors.py")
    assert r.returncode == 0 and f"SHARDED_REJECTORS_OK export {nproc}" in r.stdout


@pytest.mark.gpu
def test_sharded_rejector_chains_two_gpus_nccl():
    """Needs 2 GPUs: the same checks with pclb200_comm_init and PCLB200_REDUCE_NCCL (histograms summed and the one-to-one
    tables min-reduced by ncclAllReduce)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (VISIBLE SKIP: the peer-mapped path runs on one GPU in test_sharded_rejector_chains_share_one_gpu)")
    r = _torchrun(2, "_two_gpu_rejectors_nccl.py")
    assert r.returncode == 0 and "SHARDED_REJECTORS_OK nccl 2" in r.stdout


@pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")) or shutil.which("g++") is None,
                    reason="needs g++ and the CUDA headers (vector types only; nothing is run on a device)")
def test_sharded_rejector_table_sets_on_the_host(tmp_path):
    """reject_sharded_kernels.cuh compiled for the host, 1 / 2 / 3 / 5 / 8 simulated ranks (the program sums the histograms
    and min-reduces the one-to-one tables itself, both one-to-one protocols, read through peer_table_set): the union of the survivors equals the oracle's
    rejector on the concatenation for every rejector, trimmed with keep = 0, 1, c - 1, c, and four chains; runs of exact
    ties, ranks with no accepted entry, array order unlike slot order."""
    import oracle
    oracle.build()
    odir = os.path.join(ROOT, "oracle")
    exe = str(tmp_path / "reject_sharded_host_test")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-frounding-math", "-ffp-contract=off", "-fno-fast-math",
                           "-I" + CUDA_INC, "-I" + os.path.join(ROOT, "include"), "-I" + HOST,
                           "-I" + os.path.join(ROOT, "pcl_b200", "pcl_compat"), os.path.join(HOST, "reject_sharded_host_test.cpp"),
                           "-o", exe, "-L" + odir, "-lpcl_oracle", "-Wl,-rpath," + odir])
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]
    assert "tiny                       R=8" in r.stdout and "DIFFERS" not in r.stdout
