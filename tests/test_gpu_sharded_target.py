"""A target map sharded across ranks: the labelled index (pclb200_index_build_ids) on one GPU, and the sharded-target ICP
session and fitness (pclb200_icp_set_target_sharded, pclb200_fitness_score_sharded) under torchrun
(tests/_sharded_target_ranks.py): byte-equal to one process on the whole map."""
import numpy as np
import pytest

import _sharded as S


@pytest.mark.gpu
def test_index_with_ids_equals_index_of_the_whole_cloud_with_subset():
    """Index(ctx, tile, ids=ids) answers k-NN and radius searches byte for byte like Index(ctx, whole, subset=ids) when
    tile[i] = whole[ids[i]]; negative, duplicate and reserved ids are refused, and so are the consumers that address the
    cloud an index was built from."""
    import pcl_b200 as P
    rng = np.random.default_rng(3)
    whole = P.xyz1(rng.random((60000, 3), dtype=np.float32))
    whole[::997, 1] = np.nan
    whole[1000:1100] = whole[2000:2100]  # equal points under different ids: ties
    ids = rng.permutation(60000)[:25000].astype(np.int32)
    ctx = P.Context(0)
    a = P.Index(ctx, np.ascontiguousarray(whole[ids]), ids=ids)
    b = P.Index(ctx, whole, subset=ids)
    assert a.size == b.size
    q = P.xyz1(rng.random((5000, 3), dtype=np.float32))
    for k in (1, 8, 40):
        ia, da, _ = a.knn(q, k)
        ib, db, _ = b.knn(q, k)
        assert ia.tobytes() == ib.tobytes() and da.tobytes() == db.tobytes(), k
    oa, xa, ra = a.radius(q, 0.03)
    ob, xb, rb = b.radius(q, 0.03)
    assert oa.tobytes() == ob.tobytes() and xa.tobytes() == xb.tobytes() and ra.tobytes() == rb.tobytes()
    assert np.array_equal(a.correspondences(q, 0.05), b.correspondences(q, 0.05))
    pts = np.ascontiguousarray(whole[:100])
    for bad in (np.r_[-1, np.arange(1, 100)], np.r_[5, np.arange(1, 100)], np.r_[2 ** 31 - 1, np.arange(1, 100)]):
        with pytest.raises(P.Pclb200Error) as e:
            P.Index(ctx, pts, ids=bad.astype(np.int32))
        assert e.value.code == P.ERR_INVALID
    ok = P.Index(ctx, pts, ids=np.arange(2 ** 31 - 101, 2 ** 31 - 1, dtype=np.int32))
    assert ok.knn(pts[1:4], 1)[0][:, 0].tolist() == [2 ** 31 - 100, 2 ** 31 - 99, 2 ** 31 - 98]
    with pytest.raises(P.Pclb200Error) as e:
        a.cluster_labels(0.01, out=np.empty(25000, np.int32))
    assert e.value.code == P.ERR_INVALID and "ids" in str(e.value)
    with pytest.raises(P.Pclb200Error) as e:
        a.gicp_covariances(np.ascontiguousarray(whole[ids]))
    assert e.value.code == P.ERR_INVALID and "ids" in str(e.value)
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [2, 3])
def test_sharded_target_share_one_gpu(nproc):
    """2 / 3 processes on cuda:0, peer exchange bootstrapped over gloo: slabs, a random partition, and slabs with duplicated
    points and a far 1-point tile; SVD (Umeyama and correlation), point-to-plane and symmetric, float and double, tracking
    off / on / auto, stepping and whole: every iteration's correspondences, the final stats and the aligned cloud
    byte-equal to one process on the whole map; fitness to 1e-12; every refusal on every rank."""
    r = S.torchrun("_sharded_target_ranks.py", nproc)
    assert r.returncode == 0 and f"SHARDED_TARGET_OK export {nproc}" in r.stdout


@pytest.mark.gpu
def test_sharded_target_two_gpus_nccl():
    """Needs 2 GPUs: the same comparison for point-to-plane with pclb200_comm_init and PCLB200_REDUCE_NCCL (keys
    min-reduced, records max-reduced by ncclAllReduce)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (VISIBLE SKIP: the peer-mapped path runs on one GPU in test_sharded_target_share_one_gpu)")
    r = S.torchrun("_sharded_target_ranks.py", 2, nccl=True)
    assert r.returncode == 0 and "SHARDED_TARGET_OK nccl 2" in r.stdout
