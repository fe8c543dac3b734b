"""Normals of a map sharded across ranks (pclb200_normals_knn_sharded / pclb200_normals_radius_sharded) under torchrun
(tests/_sharded_normals_ranks.py): byte-equal to one process's normals on an index of the whole map, and, fed to
set_target_sharded, point-to-plane and symmetric aligns byte-equal to one process that used the whole map's normals."""
import pytest

import _sharded as S


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [2, 3])
def test_sharded_normals_share_one_gpu(nproc):
    """2 / 3 processes on cuda:0, peer exchange bootstrapped over gloo: a surface and a volume map, slabs, a random
    partition, tiles sharing ids and a far tile of 2 points, k = 3 / 16 / 40 and a radius, the tiles' own records and an
    arbitrary query subset: out and is_dense byte-equal to one process on the whole map; the normals drive sharded
    point-to-plane and symmetric aligns byte-equal to one process; every refusal on every rank."""
    r = S.torchrun("_sharded_normals_ranks.py", nproc)
    assert r.returncode == 0 and f"SHARDED_NORMALS_OK export {nproc}" in r.stdout


@pytest.mark.gpu
def test_sharded_normals_two_gpus_nccl():
    """Needs 2 GPUs: the same comparison with pclb200_comm_init and PCLB200_REDUCE_NCCL (the halo travels through one u64
    sum all-reduce of a zeroed table)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (VISIBLE SKIP: the peer-mapped path runs on one GPU in test_sharded_normals_share_one_gpu)")
    r = S.torchrun("_sharded_normals_ranks.py", 2, nccl=True)
    assert r.returncode == 0 and "SHARDED_NORMALS_OK nccl 2" in r.stdout
