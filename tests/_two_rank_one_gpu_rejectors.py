"""Helper for tests/test_sharded_rejectors.py (launched under torchrun, gloo): the correspondence rejector chain on a
sharded source.

Every process holds a replica of the target index and one uneven contiguous range of the source (rank r holds the r-th
range, so global position = input order).  Bootstrap: two or three processes on cuda:0, the peer exchange made with
pclb200_comm_export / _import over gloo; with PCLB_SHARDED_NCCL=1, one process per GPU, pclb200_comm_init +
PCLB200_REDUCE_NCCL.
  * iteration 1, exact: the correspondences of every rank (query indices shifted by the shard offset), concatenated in
    rank order, equal the single-process list with the same chain, as arrays — on a smooth surface with outliers and on
    a lattice scene full of exact distance ties across shard boundaries (median, trimmed and one-to-one tie rules);
  * full align: every rank ends with the bitwise same transform; against the single process the same iterations,
    n_correspondences and total_correspondences, transforms within 1e-6 (the fp64 sums fold in another order)."""
import numpy as np

import _sharded as S
import pcl_b200 as P

CHAIN4 = [(P.REJ_MEDIAN, 3.0, 0), (P.REJ_ONE_TO_ONE, 0.0, 0), (P.REJ_TRIMMED, 0.9, 100), (P.REJ_DISTANCE, 0.2, 0)]
SVD, LLS = P.EST_SVD, P.EST_POINT_TO_PLANE_LLS
CASES = [  # (name, chain, estimator)
    ("median", [(P.REJ_MEDIAN, 3.0, 0)], SVD),
    ("median 1.0", [(P.REJ_MEDIAN, 1.0, 0)], SVD),
    ("one-to-one", [(P.REJ_ONE_TO_ONE, 0.0, 0)], SVD),
    ("trimmed", [(P.REJ_TRIMMED, 0.9, 100)], SVD),
    ("distance", [(P.REJ_DISTANCE, 0.2, 0)], SVD),
    ("chain of four", CHAIN4, SVD),
    ("chain of four, point-to-plane", CHAIN4, LLS),
    ("surface normal + chain, point-to-plane", [(P.REJ_SURFACE_NORMAL, 0.7, 0)] + CHAIN4, LLS),
]


def shard_bounds(n, world):
    """Uneven contiguous ranges: rank r gets a share proportional to r + 1."""
    w = np.arange(1, world + 1, dtype=np.float64)
    cuts = np.concatenate([[0], np.round(np.cumsum(w) / w.sum() * n)]).astype(int)
    return [(int(cuts[r]), int(cuts[r + 1])) for r in range(world)]


def with_normals(ctx, pts):
    """12-float records: xyz 1 | normal (from the cloud's own 12-NN) 0 | 4 pad."""
    rec = np.zeros((pts.shape[0], 12), dtype=np.float32)
    rec[:, :3] = pts
    rec[:, 3] = 1
    idx = P.Index(ctx, rec)
    nrm, _ = idx.normals_knn(rec, 12, viewpoint=(2, 2, 10))
    rec[:, 4:7] = nrm[:, :3]
    idx.close()
    return rec


def scenes(ctx):
    rng = np.random.default_rng(32)
    n = 40000
    tgt = rng.random((n, 3), dtype=np.float32)
    tgt[:, 2] = 0.2 * np.sin(3 * tgt[:, 0]) * np.cos(2 * tgt[:, 1])
    a = np.deg2rad(3.0)
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    src = (tgt.astype(np.float64)[: n // 2] @ R.T + [0.01, -0.01, 0.02] + rng.normal(0, 0.002, (n // 2, 3))).astype(np.float32)
    src[:500] += np.float32(0.3)  # gross outliers for the rejectors to remove
    yield "surface", with_normals(ctx, tgt), with_normals(ctx, src), True
    # lattice: target spacing 1/32, source on the lattice of spacing 1/64 shifted by one fine step — every distance is one of
    # a few exact values, many sources share a target at equal distance, and the runs cross every shard boundary
    h = 1.0 / 32
    g = np.stack(np.meshgrid(np.arange(40), np.arange(40), np.arange(6), indexing="ij"), -1).reshape(-1, 3)
    tl = (g * h).astype(np.float32)
    fg = np.stack(np.meshgrid(np.arange(4, 74), np.arange(4, 74), np.arange(2, 9), indexing="ij"), -1).reshape(-1, 3)
    sl = (fg * (h / 2) + [h / 2, 0, 0]).astype(np.float32)
    yield "lattice", with_normals(ctx, tl), with_normals(ctx, sl), False


def run_case(ctx, idx, tgt, src, lo, hi, chain, est, max_iterations):
    kw = dict(max_iterations=max_iterations, transformation_epsilon=1e-9, estimator=est,
              with_normals_transform=1 if est != SVD else 0)
    s = P.Icp(ctx, **kw)
    s.set_rejectors(chain)
    s.set_target(idx, normals=P.Field(tgt, 4) if est != SVD else None)
    part = np.ascontiguousarray(src[lo:hi])
    s.set_source(part, normals=P.Field(part, 4))
    st = s.iterate()
    corr = s.get_correspondences().copy()
    corr["index_query"] += lo
    s.close()
    return st, corr


def main(me):
    ctx, rank, world, single = me.ctx, me.rank, me.world, me.ref  # single: no communicator, the whole cloud
    for name, tgt, src, full in scenes(ctx):
        idx = P.Index(ctx, tgt)
        idx1 = P.Index(single, tgt) if rank == 0 else None
        lo, hi = shard_bounds(src.shape[0], world)[rank]
        for case, chain, est in CASES:
            # iteration 1: bit-identical inputs, so the lists must be equal
            st, corr = run_case(ctx, idx, tgt, src, lo, hi, chain, est, 1)
            got = S.gathered(corr.tobytes())
            if rank == 0:
                st1, corr1 = run_case(single, idx1, tgt, src, 0, src.shape[0], chain, est, 1)
                cat = np.frombuffer(b"".join(got), dtype=P.CORR_DTYPE)
                assert cat.shape == corr1.shape and np.array_equal(cat, corr1), (name, case, cat.shape, corr1.shape)
                assert st["n_correspondences"] == st1["n_correspondences"] == len(corr1), (name, case)
                print(f"{name:8s} {case:40s} iteration 1 equal: {len(corr1)} of {src.shape[0]} kept", flush=True)
            if not full:
                continue
            st, _ = run_case(ctx, idx, tgt, src, lo, hi, chain, est, 30)
            got = S.gathered(st["final"].tobytes())
            assert all(g == got[0] for g in got), (name, case, "ranks disagree on the transform")
            if rank == 0:
                st1, _ = run_case(single, idx1, tgt, src, 0, src.shape[0], chain, est, 30)
                err = float(np.linalg.norm(st1["final"] - st["final"]))
                assert st["iterations"] == st1["iterations"], (name, case, st["iterations"], st1["iterations"])
                assert st["n_correspondences"] == st1["n_correspondences"], (name, case)
                assert st["total_correspondences"] == st1["total_correspondences"], (name, case)
                assert err < 1e-6, (name, case, err)
                print(f"{name:8s} {case:40s} ok  iterations {st['iterations']:2d}  correspondences {st['n_correspondences']}"
                      f"  |dT| {err:.1e}", flush=True)
        idx.close()
        if idx1 is not None:
            idx1.close()


if __name__ == "__main__":
    me = S.join()
    main(me)
    me.finish("SHARDED_REJECTORS")
