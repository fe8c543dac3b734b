"""VoxelGrid of a map sharded across ranks (pclb200_voxelgrid_sharded) under torchrun (tests/_sharded_voxel_ranks.py):
every rank's rows, sorted by voxel index, byte-equal to one process's VoxelGrid on the whole map, each voxel on one
rank."""
import pytest

import _sharded as S


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [2, 3])
def test_sharded_voxelgrid_share_one_gpu(nproc):
    """2 / 3 processes on cuda:0, peer exchange bootstrapped over gloo: slabs, a random partition, tiles sharing ids, a far
    tile, slabs cut on voxel faces and one rank empty; leaves giving 1 to 50 records per voxel, min_points_per_voxel 0 / 1
    / 3, with and without normals: the concatenated rows sorted by voxel byte-equal to one process's voxelgrid(_normals)
    with the sorted union of the ids, no voxel on two ranks, n_out <= n; a voxel only the whole map's count keeps; device
    arrays; ERR_LEAF_TOO_SMALL from the union grid alone; every refusal on every rank; k-NN on the output."""
    r = S.torchrun("_sharded_voxel_ranks.py", nproc)
    assert r.returncode == 0 and f"SHARDED_VOXEL_OK export {nproc}" in r.stdout


@pytest.mark.gpu
def test_sharded_voxelgrid_two_gpus_nccl():
    """Needs 2 GPUs: the same comparison with pclb200_comm_init and PCLB200_REDUCE_NCCL (the first exchange is a u64
    minimum all-reduce, the records travel through one u64 sum all-reduce of a zeroed table)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (VISIBLE SKIP: the peer-mapped path runs on one GPU in test_sharded_voxelgrid_share_one_gpu)")
    r = S.torchrun("_sharded_voxel_ranks.py", 2, nccl=True)
    assert r.returncode == 0 and "SHARDED_VOXEL_OK nccl 2" in r.stdout
