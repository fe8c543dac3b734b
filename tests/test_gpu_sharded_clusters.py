"""Euclidean clusters of a map sharded across ranks (pclb200_cluster_labels_sharded) under torchrun
(tests/_sharded_clusters_ranks.py): labels byte-equal to one process's cluster_labels on the whole map, sizes equal to its
component sizes, and euclidean_clusters_sharded's parts equal to the whole map's clusters."""
import pytest

import _sharded as S


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [2, 3])
def test_sharded_clusters_share_one_gpu(nproc):
    """2 / 3 processes on cuda:0, peer exchange bootstrapped over gloo: a zig-zag chain across every boundary, blobs with
    duplicates and non-finite records, a lattice at and just above the tolerance, tolerance 0 and a 1 M-point holed sheet;
    slabs, a random partition and shared ids with a 1-point tile: labels and sizes into host and device buffers, one label
    per shared id, the cluster lists, and every refusal on every rank."""
    r = S.torchrun("_sharded_clusters_ranks.py", nproc)
    assert r.returncode == 0 and f"SHARDED_CLUSTERS_OK export {nproc}" in r.stdout


@pytest.mark.gpu
def test_sharded_clusters_two_gpus_nccl():
    """Needs 2 GPUs: the same comparison with pclb200_comm_init and PCLB200_REDUCE_NCCL (every table travels through one
    u64 sum all-reduce of a zeroed table)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (VISIBLE SKIP: the peer-mapped path runs on one GPU in test_sharded_clusters_share_one_gpu)")
    r = S.torchrun("_sharded_clusters_ranks.py", 2, nccl=True)
    assert r.returncode == 0 and "SHARDED_CLUSTERS_OK nccl 2" in r.stdout
