"""Helper for tests/test_gpu_sharded_target.py (launched under torchrun, gloo): a map sharded across ranks, the whole source
on every rank (pclb200_index_build_ids + pclb200_icp_set_target_sharded).

Ranks on cuda:0 with the peer exchange bootstrapped over gloo (comm_export / _import), or, with PCLB_SHARDED_NCCL=1, one
GPU per rank with pclb200_comm_init and PCLB200_REDUCE_NCCL.  The map is a 200 k-point surface cut three ways (spatial
slabs; a random partition; slabs plus duplicated map points given to another rank under other ids and a far 1-point tile
no source point reaches within the gate).  For every estimator, Scalar and tracking mode, stepping one iteration at a
time and running whole, every iteration's correspondences, the final stats and the aligned cloud must be byte-equal to
one process on the whole map, on every rank.  Fitness agrees to 1e-12; every refusal is ERR_INVALID on every rank."""
import numpy as np

import _sharded as S
import pcl_b200 as P

me = S.join()
rank, world, ctx, ref_ctx = me.rank, me.world, me.ctx, me.ref

# ---- the map: a smooth surface, analytic normals; ids = row numbers of `whole` -------------------------------------------
rng = np.random.default_rng(11)
N = 200000
xy = rng.random((N, 2), dtype=np.float32) * 4
z = (0.3 * np.sin(xy[:, 0]) * np.cos(xy[:, 1])).astype(np.float32)
nrm = np.stack([-0.3 * np.cos(xy[:, 0]) * np.cos(xy[:, 1]), 0.3 * np.sin(xy[:, 0]) * np.sin(xy[:, 1]),
                np.ones(N)], 1)
nrm = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(np.float32)
dup_of = rng.choice(np.nonzero(xy[:, 0] >= 2)[0], 300, replace=False)   # duplicated under new ids, on another rank
far = np.array([[2.0, 2.0, 50.0]], np.float32)                           # beyond every source point's gate
whole = np.zeros((N + len(dup_of) + 1, 8), np.float32)
whole[:N, :2], whole[:N, 2], whole[:N, 4:7] = xy, z, nrm
whole[N:N + len(dup_of)] = whole[dup_of]
whole[-1, :3], whole[-1, 6] = far, 1.0
whole[:, 3] = 1
NW = len(whole)


def partitions():
    """Every partition covers the whole map: the union of the tiles' boxes is the frame of one index over it."""
    ids = np.arange(NW)
    slab = np.minimum((whole[:, 0] / 4 * world).astype(int), world - 1)
    yield "slabs", [ids[slab == r] for r in range(world)]
    perm = rng.permutation(NW)
    yield "random", [np.sort(perm[r::world]) for r in range(world)]
    ids, slab = ids[:N], slab[:N]
    parts = [ids[slab == r] for r in range(world)]
    parts[0] = np.r_[parts[0], np.arange(N, N + len(dup_of))]     # the copies of points another rank holds
    if world >= 3:
        parts[-1] = np.array([NW - 1])                              # a 1-point tile no source point reaches
        parts[-2] = np.r_[parts[-2], ids[slab == world - 1]]
    else:
        parts[-1] = np.r_[parts[-1], [NW - 1]]
    yield "special", [rng.permutation(p) for p in parts]            # ids in no particular order


# ---- the source: 40 k points of the surface, moved -----------------------------------------------------------------------
ns = 40000
sel = rng.choice(N, ns, replace=False)
a = np.deg2rad(2.0)
R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
src = np.zeros((ns, 8), np.float32)
src[:, :3] = (whole[sel, :3].astype(np.float64) @ R.T + [0.02, -0.015, 0.01]).astype(np.float32)
src[:, 3] = 1
src[:, 4:7] = (whole[sel, 4:7].astype(np.float64) @ R.T).astype(np.float32)
src[rng.choice(ns, 50, replace=False), 0] = np.nan                    # non-finite source points

ESTIMATORS = [("svd", P.EST_SVD, 0), ("svd_correlation", P.EST_SVD, 1), ("point_to_plane", P.EST_POINT_TO_PLANE_LLS, 0),
              ("symmetric", P.EST_SYMMETRIC_POINT_TO_PLANE_LLS, 0)]
if me.nccl:
    ESTIMATORS = ESTIMATORS[2:3]


def params(est, no_umeyama, dbl, track):
    return P.default_params(max_iterations=15, max_correspondence_distance=0.15, estimator=est, scalar_is_double=dbl,
                            svd_no_umeyama=no_umeyama, track_mode=track, mse_threshold_absolute=0.0,
                            transformation_epsilon=1e-12, with_normals_transform=0 if est == P.EST_SVD else 1)


def stats_bytes(st):
    return (st["iterations"], st["state"], st["converged"], st["n_correspondences"], st["total_correspondences"],
            np.float64(st["mse"]).tobytes(), st["final"].tobytes(), st["last"].tobytes())


def run(session_ctx, set_target, p, step):
    icp = P.Icp(session_ctx, p)
    set_target(icp)
    icp.set_source(src, normals=P.Field(src, 4), guess=None)
    corr = []
    if step:
        while True:
            st = icp.iterate(1)
            corr.append(icp.get_correspondences().tobytes())
            if st["state"] != 0 or st["iterations"] >= 15:
                break
    else:
        st = icp.iterate()
        corr.append(icp.get_correspondences().tobytes())
    cloud = icp.get_cloud(stride_floats=8, normals=None).tobytes()
    icp.close()
    return stats_bytes(st), corr, cloud


ref_index = P.Index(ref_ctx, whole)
ref_cache = {}
checked = 0
for pname, parts in partitions():
    ids = np.ascontiguousarray(parts[rank], dtype=np.int32)
    tile = np.ascontiguousarray(whole[ids])
    tindex = P.Index(ctx, tile, ids=ids)
    for ename, est, no_um in ESTIMATORS:
        for dbl in (0, 1):
            for track in (P.TRACK_OFF, P.TRACK_ON, P.TRACK_AUTO):
                p = params(est, no_um, dbl, track)
                for step in (True, False):
                    key = (ename, dbl, track, step)
                    if key not in ref_cache:
                        ref_cache[key] = run(ref_ctx, lambda icp: icp.set_target(ref_index, normals=P.Field(whole, 4)), p,
                                             step)
                    got = run(ctx, lambda icp: icp.set_target_sharded(tindex, normals=P.Field(tile, 4)), p, step)
                    ref = ref_cache[key]
                    what = f"{pname} {ename} double={dbl} track={track} step={step}"
                    first_diff = next((k for k, (g, r) in enumerate(zip(got[1], ref[1])) if g != r), None)
                    assert got[0] == ref[0], (what, "stats", got[0][:5], ref[0][:5], "mse", np.frombuffer(got[0][5]),
                                              np.frombuffer(ref[0][5]), "final", np.frombuffer(got[0][6]) -
                                              np.frombuffer(ref[0][6]), "first iteration with other pairs", first_diff)
                    assert len(got[1]) == len(ref[1]) and first_diff is None, (what, "corr", first_diff)
                    assert got[2] == ref[2], (what, "cloud")
                    checked += 1
    # fitness: same value on every rank, one process's to 1e-12
    T = np.eye(4)
    T[:3, :3] = R.T
    for max_range in (np.finfo(np.float64).max, 0.01):
        f = tindex.fitness_score_sharded(src, T, max_range=max_range)
        f1 = ref_index.fitness_score(src, T, max_range=max_range)
        allf = S.gathered(f)
        assert all(x == allf[0] for x in allf), (pname, allf)
        assert abs(f - f1) <= 1e-12 * abs(f1), (pname, f, f1)
    print(f"rank {rank}: {pname} ok ({checked} runs)", flush=True)


# ---- refusals: ERR_INVALID on every rank ---------------------------------------------------------------------------------
ids = np.ascontiguousarray(np.arange(rank, N, world), dtype=np.int32)
tile = np.ascontiguousarray(whole[ids])
tindex = P.Index(ctx, tile, ids=ids)


def session(**kw):
    icp = P.Icp(ctx, P.default_params(max_iterations=3, **kw))
    icp.set_target_sharded(tindex, normals=P.Field(tile, 4))
    return icp


def with_source(icp, s=src):
    icp.set_source(s, normals=P.Field(s, 4))
    icp.iterate()


S.refused(lambda: with_source(session(use_reciprocal=1)), "reciprocal")
S.refused(lambda: with_source(session(correspondence_kind=P.CORR_NORMAL_SHOOTING)), "normal-shooting")
S.refused(lambda: with_source(session(correspondence_kind=P.CORR_BACK_PROJECTION)), "back-projection")


def with_rejector():
    icp = session()
    icp.set_rejectors([(P.REJ_DISTANCE, 0.1, 0)])
    with_source(icp)


S.refused(with_rejector, "rejector")
short = np.ascontiguousarray(src[:ns - rank])  # rank 0 passes one point more than the others
S.refused(lambda: with_source(session(), short), "same whole source")
lone = P.Index(ref_ctx, tile, ids=ids)
S.refused(lambda: P.Icp(ref_ctx).set_target_sharded(lone), "communicator")
S.refused(lambda: lone.fitness_score_sharded(src, np.eye(4)), "communicator")
# the session still works after the refusals
with_source(session())
me.finish("SHARDED_TARGET", runs=checked)
