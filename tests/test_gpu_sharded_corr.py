"""Correspondences, validation and inliers on a map sharded across ranks (pclb200_correspondences_sharded,
pclb200_validate_transformation_sharded, pclb200_inliers_sharded) under torchrun (tests/_sharded_corr_ranks.py): byte-equal
to one index of the whole map on every rank."""
import pytest

import _sharded as S


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [2, 3])
def test_sharded_corr_share_one_gpu(nproc):
    """2 / 3 processes on cuda:0, peer exchange bootstrapped over gloo: slabs, a random partition, ids shared near the cuts
    and a far tile; nearest lists (finite, zero and unbounded gates, src_indices, is_dense 0), reciprocal lists, the record
    rows, inliers byte for byte; validation to 1e-12 and equal on every rank; a hand-written ICP loop (rejector chain,
    SVD and point-to-plane over the record rows) byte-equal for 10 iterations; every refusal on every rank."""
    r = S.torchrun("_sharded_corr_ranks.py", nproc)
    assert r.returncode == 0 and f"SHARDED_CORR_OK export {nproc}" in r.stdout


@pytest.mark.gpu
def test_sharded_corr_two_gpus_nccl():
    """Needs 2 GPUs: the same comparison with pclb200_comm_init and PCLB200_REDUCE_NCCL (keys min-reduced, records
    max-reduced by ncclAllReduce)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (VISIBLE SKIP: the peer-mapped path runs on one GPU in test_sharded_corr_share_one_gpu)")
    r = S.torchrun("_sharded_corr_ranks.py", 2, nccl=True)
    assert r.returncode == 0 and "SHARDED_CORR_OK nccl 2" in r.stdout
