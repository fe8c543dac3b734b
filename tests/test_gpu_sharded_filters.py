"""k-NN queries, k-NN statistics and the outlier filters of a map sharded across ranks (pclb200_knn_sharded,
pclb200_knn_stats_sharded, pclb200_statistical_outlier_sharded, pclb200_radius_outlier_sharded) under torchrun
(tests/_sharded_filters_ranks.py): byte-equal to one process on an index of the whole map, the SOR threshold within fp64
round-off of one process's sequential threshold and the same on every rank."""
import pytest

import _sharded as S


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [2, 3])
def test_sharded_filters_share_one_gpu(nproc):
    """2 / 3 processes on cuda:0, peer exchange bootstrapped over gloo: a surface and a volume map with exact-tie lattices,
    slabs, a random partition, tiles sharing ids and a far tile of 2 points, k = 2 / 16 / 51, the tiles' own records and an
    indices subset: k-NN rows, k_eff, mean and kth byte-equal to one process on the whole map; ROR masks byte-equal (dense
    and not, negative both ways); the SOR threshold equal on every rank and within 1e-12 of the sequential one, its masks
    byte-equal; both masks equal the CPU oracle's; a map smaller than k; device arrays; every refusal on every rank."""
    r = S.torchrun("_sharded_filters_ranks.py", nproc)
    assert r.returncode == 0 and f"SHARDED_FILTERS_OK export {nproc}" in r.stdout


@pytest.mark.gpu
def test_sharded_filters_two_gpus_nccl():
    """Needs 2 GPUs: the same comparison with pclb200_comm_init and PCLB200_REDUCE_NCCL (the SOR partial sums travel
    through one u64 sum all-reduce of a zeroed table)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (VISIBLE SKIP: the peer-mapped path runs on one GPU in test_sharded_filters_share_one_gpu)")
    r = S.torchrun("_sharded_filters_ranks.py", 2, nccl=True)
    assert r.returncode == 0 and "SHARDED_FILTERS_OK nccl 2" in r.stdout
