"""The correspondence rejector chain on a source sharded across ranks (reject.cu: apply_rejector_sharded, comm.cu: the u64
exchanges, reject_sharded_kernels.cuh): every rank must accept exactly what one process accepts over the concatenation
of the shards in rank order."""
import os

import pytest

import _sharded as S


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [2, 3])
def test_sharded_rejector_chains_share_one_gpu(nproc):
    """2 / 3 processes on cuda:0, peer exchange bootstrapped over gloo (comm_export / _import), uneven contiguous shards:
    each device rejector alone, the four-rejector chain (SVD, point-to-plane) and surface-normal + chain (point-to-plane).
    Iteration 1: the concatenated per-rank correspondences equal the single-process list exactly (smooth surface with
    outliers; a lattice scene with exact distance ties across shard boundaries).  Full align: bitwise the same transform
    on every rank; same iterations and correspondence counts as the single process, transform within 1e-6."""
    r = S.torchrun("_two_rank_one_gpu_rejectors.py", nproc, timeout=900)
    assert r.returncode == 0 and f"SHARDED_REJECTORS_OK export {nproc}" in r.stdout


@pytest.mark.gpu
def test_sharded_rejector_chains_two_gpus_nccl():
    """Needs 2 GPUs: the same checks with pclb200_comm_init and PCLB200_REDUCE_NCCL (histograms summed and the one-to-one
    tables min-reduced by ncclAllReduce)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (VISIBLE SKIP: the peer-mapped path runs on one GPU in test_sharded_rejector_chains_share_one_gpu)")
    r = S.torchrun("_two_rank_one_gpu_rejectors.py", 2, nccl=True, timeout=900)
    assert r.returncode == 0 and "SHARDED_REJECTORS_OK nccl 2" in r.stdout


@S.needs_host_compiler
def test_sharded_rejector_table_sets_on_the_host(tmp_path):
    """reject_sharded_kernels.cuh compiled for the host, 1 / 2 / 3 / 5 / 8 simulated ranks (the program sums the histograms
    and min-reduces the one-to-one tables itself, both one-to-one protocols, read through peer_table_set): the union of the survivors equals the oracle's
    rejector on the concatenation for every rejector, trimmed with keep = 0, 1, c - 1, c, and four chains; runs of exact
    ties, ranks with no accepted entry, array order unlike slot order."""
    import oracle
    oracle.build()
    odir = os.path.join(S.ROOT, "oracle")
    out = S.host_program(tmp_path, "reject_sharded_host_test.cpp", link=["-L" + odir, "-lpcl_oracle", "-Wl,-rpath," + odir])
    assert "tiny                       R=8" in out and "DIFFERS" not in out
