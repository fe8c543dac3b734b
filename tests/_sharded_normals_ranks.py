"""Helper for tests/test_gpu_sharded_normals.py (launched under torchrun, gloo): normals of a map sharded across ranks
(pclb200_normals_knn_sharded / pclb200_normals_radius_sharded).

Ranks on cuda:0 with the peer exchange bootstrapped over gloo (comm_export / _import), or, with PCLB_SHARDED_NCCL=1, one
GPU per rank with pclb200_comm_init and PCLB200_REDUCE_NCCL.  Two maps (a 200 k-point surface and a volume cloud, both
with non-finite rows and duplicated points under other ids), four partitions (spatial slabs; a random partition; slabs
whose points near a cut are held by both neighbours under one id; slabs plus a far tile of 2 points), k = 3 / 16 / 40
and radius 0.03.  Queries: each tile's own records (non-finite ones included), and an arbitrary point set through an
indices subset.  out and is_dense must be byte-equal to one process's normals on an index of the whole map.  Then the
pipeline: the tiles' normals from the new call feed set_target_sharded, and point-to-plane / symmetric aligns must be
byte-equal to one process that used the whole map's normals.  Last, the refusals (ERR_INVALID on every rank), after
which the communicator still works."""
import numpy as np

import _sharded as S
import pcl_b200 as P

me = S.join()
rank, world, ctx, ref_ctx = me.rank, me.world, me.ctx, me.ref

rng = np.random.default_rng(17)
SCENES = [("surface", S.with_extras(rng, S.surface(rng, 200000))), ("volume", S.with_extras(rng, S.volume(rng, 100000)))]


def tile_of(whole, ids):
    return np.ascontiguousarray(whole[ids]), np.ascontiguousarray(ids, dtype=np.int32)


def same(a, b):
    return a[0].tobytes() == b[0].tobytes() and a[1] == b[1]


checked = 0
for sname, whole0 in SCENES:
    for pname, parts, whole in S.partitions(rng, whole0, world):
        ref_index = P.Index(ref_ctx, whole)
        tile, ids = tile_of(whole, parts[rank])
        tindex = P.Index(ctx, tile, ids=ids)
        q_any, sub = S.arbitrary_queries(rng, whole)
        for k in (3, 16, 40):
            got = tindex.normals_knn_sharded(tile, k, viewpoint=(1, 2, 3))
            want = ref_index.normals_knn(tile, k, viewpoint=(1, 2, 3))
            assert same(got, want), (sname, pname, "k", k, rank)
            got = tindex.normals_knn_sharded(q_any, k, indices=sub)
            want = ref_index.normals_knn(q_any, k, indices=sub)
            assert same(got, want), (sname, pname, "k, arbitrary queries", k, rank)
            checked += 2
        got = tindex.normals_radius_sharded(tile, 0.03)
        want = ref_index.normals_radius(tile, 0.03)
        assert same(got, want), (sname, pname, "radius", rank)
        got = tindex.normals_radius_sharded(q_any, 0.03, indices=sub)
        want = ref_index.normals_radius(q_any, 0.03, indices=sub)
        assert same(got, want), (sname, pname, "radius, arbitrary queries", rank)
        checked += 2
        print(f"rank {rank}: {sname} {pname} ok", flush=True)

# ---- the pipeline: sharded normals -> set_target_sharded -> point-to-plane / symmetric ----------------------------------
whole = SCENES[0][1]
parts = next(S.partitions(rng, whole, world))[1]
ns = 40000
sel = rng.choice(len(whole), ns, replace=False)
a = np.deg2rad(2.0)
Rm = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
src = np.zeros((ns, 8), np.float32)
src[:, :3] = (np.nan_to_num(whole[sel, :3]).astype(np.float64) @ Rm.T + [0.02, -0.015, 0.01]).astype(np.float32)
src[:, 3] = 1
ref_index = P.Index(ref_ctx, whole)
src_n, _ = ref_index.normals_knn(src, 16)
src[:, 4:8] = src_n
whole_n, _ = ref_index.normals_knn(whole, 16)
tile, ids = tile_of(whole, parts[rank])
tindex = P.Index(ctx, tile, ids=ids)
tile_n, _ = tindex.normals_knn_sharded(tile, 16)
assert tile_n.tobytes() == np.ascontiguousarray(whole_n[ids]).tobytes()


def run(session_ctx, set_target, est):
    p = P.default_params(max_iterations=15, max_correspondence_distance=0.15, estimator=est, mse_threshold_absolute=0.0,
                         transformation_epsilon=1e-12, with_normals_transform=1)
    icp = P.Icp(session_ctx, p)
    set_target(icp)
    icp.set_source(src, normals=P.Field(src, 4), guess=None)
    st = icp.iterate()
    corr = icp.get_correspondences().tobytes()
    cloud = icp.get_cloud(stride_floats=8, normals=None).tobytes()
    icp.close()
    return (st["iterations"], st["state"], st["n_correspondences"], np.float64(st["mse"]).tobytes(),
            st["final"].tobytes()), corr, cloud


for est in (P.EST_POINT_TO_PLANE_LLS, P.EST_SYMMETRIC_POINT_TO_PLANE_LLS):
    want = run(ref_ctx, lambda icp: icp.set_target(ref_index, normals=whole_n), est)
    got = run(ctx, lambda icp: icp.set_target_sharded(tindex, normals=tile_n), est)
    assert got == want, ("pipeline", est, got[0], want[0])
    checked += 1
print(f"rank {rank}: pipeline ok", flush=True)


# ---- refusals: ERR_INVALID on every rank, and the communicator still works -------------------------------------------------
plain = P.Index(ctx, tile)
lone = P.Index(ref_ctx, tile, ids=ids)
S.refused(lambda: tindex.normals_knn_sharded(tile, 0), "k must be positive")
S.refused(lambda: tindex.normals_radius_sharded(tile, 0.0), "radius must be positive")
S.refused(lambda: plain.normals_knn_sharded(tile, 8), "pclb200_index_build_ids")
S.refused(lambda: plain.normals_radius_sharded(tile, 0.03), "pclb200_index_build_ids")
S.refused(lambda: lone.normals_knn_sharded(tile, 8), "communicator")
S.refused(lambda: lone.normals_radius_sharded(tile, 0.03), "communicator")
assert tindex.normals_knn_sharded(tile, 16)[0].tobytes() == tile_n.tobytes()
me.finish("SHARDED_NORMALS", checks=checked)
