"""Every device VoxelGrid, cluster label, normal-based correspondence, surface-normal rejection and fitness against the
references of tests/test_consumers_reference.py, on the map-scale scenes of tests/test_search_reference.py, every row
compared.  Host and torch device outputs; ERR_LEAF_TOO_SMALL exactly where the reference's guard fires; the normal-based
kinds both stand-alone and inside the ICP loop (a different instantiation of select_by_normals).  Needs an H100: run
with -m gpu."""
import os
import sys
import time
from collections import defaultdict

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_consumers_reference as CR  # noqa: E402
import test_search_reference as R  # noqa: E402

pytestmark = pytest.mark.gpu

SERVED = defaultdict(set)   # path -> scenes that went through it
ROWS = defaultdict(int)     # path -> rows compared
T0 = [0.0]


@pytest.fixture(scope="module")
def gpu():
    import pcl_b200
    pcl_b200.lib()
    ctx = pcl_b200.Context(0)
    T0[0] = time.time()
    yield pcl_b200, ctx
    ctx.close()
    print(f"\n{'path':48s} {'rows checked':>12s}  scenes")
    for path in sorted(ROWS):
        print(f"{path:48s} {ROWS[path]:12d}  {', '.join(sorted(SERVED[path]))}")
    print(f"test_gpu_consumers_reference.py: {time.time() - T0[0]:.1f} s")


def _served(path, scene, rows):
    SERVED[path].add(scene)
    ROWS[path] += int(rows)


def _same(got, want, label):
    ok, row = CR.equal_rows(np.ascontiguousarray(got), want)
    assert ok, (label, got.shape, want.shape, row, got[row:row + 2].tolist() if row >= 0 else None,
                want[row:row + 2].tolist() if row >= 0 else None)


@pytest.mark.parametrize("name", list(R.SCENES))
def test_voxelgrid(gpu, name):
    """VoxelGrid at every leaf, min_points_per_voxel 0 and 3, an index subset and NaN points, into host memory and into
    a torch device tensor; ERR_LEAF_TOO_SMALL where the guard fires; VoxelGrid<PointNormal>; tiles on the whole grid."""
    import torch
    P, ctx = gpu
    pts, spacing = R.SCENES[name]()
    S = type("S", (), dict(cloud=R.xyz1(pts), spacing=spacing))
    for label, cloud, leaf, mp, ind in CR.voxel_cases(name, S):
        want = CR.voxel_ref(cloud, leaf, mp, ind)
        if want is None:
            with pytest.raises(P.Pclb200Error) as e:
                ctx.voxelgrid(cloud, leaf, mp, indices=ind, is_dense=False)
            assert e.value.code == P.ERR_LEAF_TOO_SMALL, (name, label)
            _served("voxelgrid: guard", name, 1)
            continue
        _same(ctx.voxelgrid(cloud, leaf, mp, indices=ind, is_dense=False), want[0], (name, label))
        _served("voxelgrid", name, want[0].shape[0])
        out = torch.empty((cloud.shape[0] if ind is None else ind.size, 4), dtype=torch.float32, device="cuda")
        got = ctx.voxelgrid(cloud, leaf, mp, indices=ind, is_dense=False, out=out)
        torch.cuda.synchronize()
        _same(got.cpu().numpy(), want[0], (name, label, "torch"))
        _served("voxelgrid, torch device output", name, want[0].shape[0])
    pn = CR.voxel_normal_cloud(S)
    for leaf in CR.voxel_leaves(name, spacing):
        want = CR.voxel_ref(pn, leaf, 2, normal=True)
        if want is None:
            with pytest.raises(P.Pclb200Error) as e:
                ctx.voxelgrid_normals(pn, leaf, 2, is_dense=False)
            assert e.value.code == P.ERR_LEAF_TOO_SMALL, (name, leaf)
            continue
        got = ctx.voxelgrid_normals(pn, leaf, 2, is_dense=False)
        _same(got[0], want[0], (name, leaf, "normals xyz"))
        _same(got[1][:, :5], want[1][:, :5], (name, leaf, "normals"))
        _served("voxelgrid_normals", name, want[0].shape[0])
        tiles, (lo, hi) = CR.voxel_tiles(S.cloud, leaf)
        parts = []
        for t in tiles:
            w = CR.voxel_ref(S.cloud, leaf, indices=t, bounds=(lo, hi))[0]
            g = ctx.voxelgrid_tile(S.cloud[t], leaf, np.r_[lo, hi])
            _same(g, w, (name, leaf, "tile"))
            parts.append(g)
            _served("voxelgrid_tile", name, w.shape[0])
        _same(np.concatenate(parts), CR.voxel_ref(S.cloud, leaf)[0], (name, leaf, "tiles concatenated"))


@pytest.mark.parametrize("name", list(R.SCENES))
def test_cluster_labels(gpu, name):
    """Every label at every tolerance, over the whole cloud (host and torch device output) and over a subset with NaN
    points; euclidean_clusters with three size windows."""
    import torch
    P, ctx = gpu
    pts, spacing = R.SCENES[name]()
    cloud = R.xyz1(pts)
    S = CR.scene(name) if name == "map_1e5" else type("S", (), dict(cloud=cloud, spacing=spacing))
    nan = CR.with_nan_rows(cloud)
    sub = CR.cluster_subset(cloud.shape[0])
    gidx, gsub = P.Index(ctx, cloud), P.Index(ctx, nan, subset=sub)
    for tol in CR.cluster_tolerances(name, S):
        want = CR.cluster_ref(cloud, tol)
        got = gidx.cluster_labels(tol)
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, (name, tol, bad.size, bad[:5].tolist(), got[bad[:3]].tolist(), want[bad[:3]].tolist())
        _served("cluster_labels", name, cloud.shape[0])
        out = torch.empty(cloud.shape[0], dtype=torch.int32, device="cuda")
        gidx.cluster_labels(tol, out=out)
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), want), (name, tol, "torch")
        _served("cluster_labels, torch device output", name, cloud.shape[0])
        for mn, mx in ((1, 2 ** 32 - 1), (2, 50), (5, 10 ** 9)):
            a, b = gidx.euclidean_clusters(tol, mn, mx), CR.clusters_ref(want, mn, mx)
            assert len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b)), (name, tol, mn, mx)
        _served("euclidean_clusters", name, cloud.shape[0])
        want = CR.cluster_ref(nan, tol, subset=sub)
        assert np.array_equal(gsub.cluster_labels(tol), want), (name, tol, "subset + nan")
        _served("cluster_labels, subset + NaN", name, cloud.shape[0])


@pytest.mark.parametrize("name", list(R.SCENES))
def test_normal_correspondences(gpu, orc, name):
    """Normal shooting and back projection at every k (every k-NN kernel), three gates and an index subset,
    stand-alone; both kinds again inside the ICP loop (first iteration, no gate); the surface-normal rejector."""
    P, ctx = gpu
    S = CR.scene(name)
    sn, tn = CR.scene_normals(S, orc)
    src, tgt = CR.point_normal(S.q, sn), CR.point_normal(S.cloud, tn)
    gidx = P.Index(ctx, tgt)
    ind = np.random.default_rng(53).permutation(src.shape[0])[:20_000].astype(np.int32)
    for kind in (1, 2):
        kname = "normal shooting" if kind == 1 else "back projection"
        for k in CR.CORR_K:
            for md in CR.corr_gates(S):
                for sel in (None, ind):
                    if sel is not None and md != CR.corr_gates(S)[1]:
                        continue
                    want = CR.normals_corr_ref(kind, S.q, sn, S.cloud, tn, S.idx, S.d2, k, md, sel)
                    got = gidx.correspondences_normals(kind, src, P.Field(src, 4), P.Field(tgt, 4), k=k,
                                                       max_distance=md, indices=sel)
                    assert np.array_equal(got, want), (name, kind, k, md, sel is None, got.size, want.size)
                    _served(f"{kname}, k = {k}", name, src.shape[0] if sel is None else sel.size)
        for k in (3, 10, 40):
            want = CR.normals_corr_ref(kind, S.q, sn, S.cloud, tn, S.idx, S.d2, k)
            s = P.Icp(ctx, max_iterations=1, correspondence_kind=kind, correspondence_k=k, is_dense=0)
            s.set_target(gidx, P.Field(tgt, 4))
            s.set_source(src, normals=P.Field(src, 4))
            s.iterate(1)
            got = s.get_correspondences()
            assert np.array_equal(got, want), (name, kind, k, "in loop", got.size, want.size)
            _served(f"{kname} in the ICP loop", name, src.shape[0])
    corr = R.corr_ref(S.idx[:, 0], S.d2[:, 0])
    for thr in CR.surface_thresholds(CR.surface_dots(corr, sn, tn)):
        want = CR.surface_normal_ref(corr, sn, tn, thr)
        got = ctx.reject_surface_normal(corr, P.Field(src, 4), P.Field(tgt, 4), thr)
        assert np.array_equal(got, want), (name, thr, got.size, want.size)
        _served("surface-normal rejector", name, corr.size)


@pytest.mark.parametrize("name", list(R.SCENES))
def test_fitness_validation_inliers(gpu, name):
    """getFitnessScore and validateTransformation in float and double Scalar, an orthonormal and a non-orthonormal
    pose, four max_range: the count exact, the mean within count 2^-52; the inlier list and its float fitness bit for
    bit."""
    P, ctx = gpu
    S = CR.scene(name)
    gidx = P.Index(ctx, S.cloud)
    for ortho in (True, False):
        src, T = CR.pose_pair(name, S, ortho)
        for kind in ("fitness float", "fitness double", "validation float", "validation double"):
            dbl = kind.endswith("double")
            _, d2 = CR.moved_d2(S.cloud, src, T, kind)
            for mr in CR.fitness_ranges(d2):
                n, want = CR.fitness_ref(d2, mr)
                fn = gidx.fitness_score if kind.startswith("fitness") else gidx.validate_transformation
                got = fn(src, T, max_range=mr, scalar_is_double=dbl)
                assert CR.fitness_close(got, want, n), (name, kind, ortho, mr, got, want, n)
                _served(kind, name, src.shape[0])
        _, d2 = CR.moved_d2(S.cloud, src, T, "inliers")
        for thr in CR.inlier_thresholds(d2):
            keep, fit = CR.inliers_ref(d2, thr)
            gi, gf = gidx.inliers(src, T, thr)
            assert np.array_equal(gi, keep) and gf == fit, (name, ortho, thr, gi.size, keep.size, gf, fit)
            _served("inliers", name, src.shape[0])


def test_every_path_was_served_by_a_far_scene(gpu):
    """Each path went through at least one far scene (run after the scene tests; skipped when they were deselected)."""
    if len({s for v in SERVED.values() for s in v}) < len(R.SCENES):
        pytest.skip("needs every scene test of this file in the same run")
    paths = ["voxelgrid", "voxelgrid, torch device output", "voxelgrid: guard", "voxelgrid_normals", "voxelgrid_tile",
             "cluster_labels", "cluster_labels, torch device output", "euclidean_clusters",
             "cluster_labels, subset + NaN", "surface-normal rejector", "fitness float", "fitness double",
             "validation float", "validation double", "inliers"]
    for kname in ("normal shooting", "back projection"):
        paths += [f"{kname}, k = {k}" for k in CR.CORR_K] + [f"{kname} in the ICP loop"]
    for path in paths:
        assert SERVED[path] - {"outlier_frame"} or path == "voxelgrid: guard", path
