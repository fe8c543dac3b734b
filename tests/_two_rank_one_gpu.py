"""Helper for tests/test_multirank_gloo.py::test_two_ranks_share_one_gpu (launched under torchrun, gloo).

Two PROCESSES, both on cuda:0 (NCCL refuses duplicate devices; the library's fused exchange only needs CUDA IPC, which
the caller bootstraps with pclb200_comm_export / _import over gloo).  Each rank holds a replica of the target index and
one half of the source; every iteration's 40 accumulators cross between the two processes through the peer-mapped
exchange block inside the iteration kernel (comm.cu + peer_exchange.cuh).  The sharded result must equal the
single-process result on the whole cloud: same correspondence counts, same iterations, transform within 1e-6."""
import numpy as np
import torch.distributed as dist

import _sharded as S
import pcl_b200 as P

me = S.join()
rank, world, ctx = me.rank, me.world, me.ctx

rng = np.random.default_rng(5)
n = 120000
tgt = np.zeros((n, 12), dtype=np.float32)
tgt[:, :2] = rng.random((n, 2), dtype=np.float32) * 4
tgt[:, 2] = 0.3 * np.sin(tgt[:, 0]) * np.cos(tgt[:, 1])
tgt[:, 3] = 1
a = np.deg2rad(1.5)
R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
src = np.zeros((n, 12), dtype=np.float32)
src[:, :3] = (tgt[:, :3].astype(np.float64) @ R.T + [0.01, -0.01, 0.004]).astype(np.float32)
src[:, 3] = 1
idx = P.Index(ctx, tgt)
nrm, _ = idx.normals_knn(tgt, 12, viewpoint=(2, 2, 10))
results = {}
for name, est in (("svd", P.EST_SVD), ("lls", P.EST_POINT_TO_PLANE_LLS)):
    kw = dict(max_iterations=12, max_correspondence_distance=0.2, estimator=est, mse_threshold_absolute=0.0,
              with_normals_transform=1 if est != P.EST_SVD else 0)
    shard = np.ascontiguousarray(src[rank * n // world:(rank + 1) * n // world])
    r = P.icp_align(ctx, shard, idx, tgt_normals=nrm if est != P.EST_SVD else None,
                    src_normals=P.Field(shard, 4) if est != P.EST_SVD else None, **kw)
    results[name] = r
    got = S.gathered(r["final"].tobytes())
    assert all(g == got[0] for g in got), "ranks disagree on the transform (the fused fold is rank-ordered: must be bitwise equal)"
    # reciprocal correspondences need the whole source on every rank: refused, not silently different
    try:
        P.icp_align(ctx, shard, idx, use_reciprocal=1, **dict(kw, estimator=P.EST_SVD, with_normals_transform=0))
        raise SystemExit("reciprocal + communicator was accepted")
    except P.Pclb200Error as e:
        assert "reciprocal" in str(e), e
dist.barrier()
if rank == 0:
    ctx1 = me.ref  # no communicator: the whole cloud in one process
    idx1 = P.Index(ctx1, tgt)
    for name, est in (("svd", P.EST_SVD), ("lls", P.EST_POINT_TO_PLANE_LLS)):
        kw = dict(max_iterations=12, max_correspondence_distance=0.2, estimator=est, mse_threshold_absolute=0.0,
                  with_normals_transform=1 if est != P.EST_SVD else 0)
        r1 = P.icp_align(ctx1, src, idx1, tgt_normals=nrm if est != P.EST_SVD else None,
                         src_normals=P.Field(src, 4) if est != P.EST_SVD else None, **kw)
        r = results[name]
        err = float(np.linalg.norm(r1["final"] - r["final"]))
        assert r["n_correspondences"] == r1["n_correspondences"], (name, r["n_correspondences"], r1["n_correspondences"])
        assert r["total_correspondences"] == r1["total_correspondences"], name
        assert r["iterations"] == r1["iterations"] and err < 1e-6, (name, err, r["iterations"], r1["iterations"])
    print("TWO_RANK_ONE_GPU_OK")
dist.barrier()
dist.destroy_process_group()
