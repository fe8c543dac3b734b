"""Radius search and GICP covariances of a map sharded across ranks (pclb200_radius_sharded, pclb200_radius_into_sharded,
pclb200_gicp_covariances_sharded) under torchrun (tests/_sharded_radius_ranks.py): byte-equal to one process on an index
of the whole map, and the collective capacity retry of pclb200_radius_into_sharded."""
import pytest

import _sharded as S


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [2, 3])
def test_sharded_radius_share_one_gpu(nproc):
    """2 / 3 processes on cuda:0, peer exchange bootstrapped over gloo: a surface and a volume map with exact-tie lattices
    and duplicated points, slabs, a random partition, tiles sharing ids and a far tile of 2 points; the tiles' records,
    arbitrary and NaN queries, a rank with no query; radii 0, NaN, ~10 and ~300 neighbours and one whose square overflows,
    max_nn 0 / 1 / 5 / 32 / 40 / more than the map, different radii on different ranks: offsets, ids and d2 of both calls,
    host and device buffers, byte-equal to one process on the whole map; the retry with one rank short of room (all_fit 0
    everywhere, then 1 with the same bytes); GICP covariances at k = 20, 64 and k above a tiny map's size, byte-equal as
    rows at the ids; every refusal on every rank, also when one rank alone passes the bad argument."""
    r = S.torchrun("_sharded_radius_ranks.py", nproc)
    assert r.returncode == 0 and f"SHARDED_RADIUS_OK export {nproc}" in r.stdout


@pytest.mark.gpu
def test_sharded_radius_two_gpus_nccl():
    """Needs 2 GPUs: the same comparison with pclb200_comm_init and PCLB200_REDUCE_NCCL."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (VISIBLE SKIP: the peer-mapped path runs on one GPU in test_sharded_radius_share_one_gpu)")
    r = S.torchrun("_sharded_radius_ranks.py", 2, nccl=True)
    assert r.returncode == 0 and "SHARDED_RADIUS_OK nccl 2" in r.stdout
