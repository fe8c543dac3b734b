"""Every device normal, curvature and GICP covariance against the extended-precision reference of its own
neighbourhood (tests/test_normals_reference.py), on every kernel that writes one, with the constants frozen on the
oracle.  Every query is checked; no percentiles.  Needs an H100: run with -m gpu."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_normals_reference as R  # noqa: E402

pytestmark = pytest.mark.gpu

WORST = {}


@pytest.fixture(scope="module")
def gpu():
    import pcl_b200
    pcl_b200.lib()
    ctx = pcl_b200.Context(0)
    yield pcl_b200, ctx
    ctx.close()
    for key, w in sorted(WORST.items()):
        print(f"device {key:40s} worst ratio: direction {w['dir']:.3g}  curvature {w['curv']:.3g}  Rayleigh {w['ray']:.3g}")


def _record(key, w):
    old = WORST.get(key, {"dir": 0.0, "curv": 0.0, "ray": 0.0})
    WORST[key] = {k: max(old[k], w[k]) for k in old}


def _xyz1(P, pts):
    return P.xyz1(np.asarray(pts, dtype=np.float32))


# k -> the kernel launch_normals picks (search.cu)
PATHS = {4: "k_normals<4>", 8: "k_normals<8>", 10: "k_normals<10>", 11: "k_normals<16>", 16: "k_knn_warp<true>",
         32: "k_knn_warp<true>", 33: "k_normals_from_lists", 64: "k_normals_from_lists"}


def _scenes():
    s, vp = R.sine_sheet()
    yield "sine_sheet", s, vp
    s, vp = R.noisy_plane()
    yield "noisy_plane", s, vp
    for off in (1e3, 1e4):
        s, vp = R.far_patch(off)
        yield f"far_{off:g}", s, vp
    s, vp = R.thin_strips()
    yield "thin_strips", s, vp
    s, vp = R.duplicated()
    yield "duplicates", s, vp


@pytest.mark.parametrize("k", sorted(PATHS))
def test_every_normal_within_the_bars(gpu, k):
    P, ctx = gpu
    for name, pts, vp in _scenes():
        cloud = _xyz1(P, pts)
        g, gd = P.Index(ctx, cloud).normals_knn(cloud, k, viewpoint=vp)
        ref = R.Reference(cloud, cloud, vp, k=k)
        assert gd == ref.is_dense, (name, k)
        _record(f"{PATHS[k]} k={k} {name}", ref.check(g, f"{name} k={k}"))
    s, vp = R.blobs()
    cloud = _xyz1(P, s)
    g, _ = P.Index(ctx, cloud).normals_knn(cloud, k, viewpoint=vp)
    _record(f"{PATHS[k]} k={k} blobs", R.Reference(cloud, cloud, vp, k=k).check(g, f"blobs k={k}", rayleigh_only=True))


@pytest.mark.parametrize("k", sorted(PATHS))
def test_exact_cases(gpu, k):
    """Lines along x, y, z, planes z = const (also 1e4 out) and identical points: the exact vectors, bit for bit."""
    P, ctx = gpu
    pts, vp, exp = R.exact_clusters(k)
    cloud = _xyz1(P, pts)
    g, gd = P.Index(ctx, cloud).normals_knn(cloud, k, viewpoint=vp)
    assert gd
    R.exact_check(g, exp, f"k={k}")


def test_nan_points_queries_subset_and_device_output(gpu):
    """NaN points and queries, an indices subset, torch output on the device; is_dense and the NaN rows exactly where
    the reference has fewer than 3 neighbours."""
    import torch
    P, ctx = gpu
    pts, vp = R.sine_sheet()
    cloud = _xyz1(P, pts)
    cloud[::301, 1] = np.nan
    rng = np.random.default_rng(4)
    sub = rng.permutation(cloud.shape[0])[:7000].astype(np.int32)
    idx = P.Index(ctx, cloud)
    for k in (5, 16, 33):
        for ind in (None, sub):
            q = cloud if ind is None else cloud[ind]
            g, gd = idx.normals_knn(cloud, k, viewpoint=vp, indices=ind, is_dense=False)
            ref = R.Reference(cloud, q, vp, k=k)
            assert gd == ref.is_dense and not gd
            _record(f"{PATHS.get(k, 'k_normals<8>')} k={k} nan/subset", ref.check(g, f"nan k={k} subset={ind is not None}"))
        out = torch.empty((cloud.shape[0], 4), dtype=torch.float32, device="cuda")
        idx.normals_knn(cloud, k, viewpoint=vp, is_dense=False, out=out)
        torch.cuda.synchronize()
        R.Reference(cloud, cloud, vp, k=k).check(out.cpu().numpy(), f"device out k={k}")


def test_per_thread_fallback_of_the_warp_kernel(gpu):
    """k 12..32 on queries the warp kernel hands back (off the cloud) and on a cloud under 256 points (no cell
    table): the per-thread kernel through `only`."""
    P, ctx = gpu
    pts, vp = R.sine_sheet()
    cloud = _xyz1(P, pts)
    rng = np.random.default_rng(6)
    off = _xyz1(P, (rng.random((3000, 3)) * 3 - 1).astype(np.float32))
    q = np.concatenate([cloud[:3000], off])
    small = cloud[:200]
    for k in (12, 16, 32):
        g, _ = P.Index(ctx, cloud).normals_knn(q, k, viewpoint=vp)
        _record(f"only k={k} off-cloud", R.Reference(cloud, q, vp, k=k).check(g, f"off-cloud k={k}"))
        g, _ = P.Index(ctx, small).normals_knn(small, k, viewpoint=vp)
        _record(f"only k={k} small cloud", R.Reference(small, small, vp, k=k).check(g, f"small k={k}"))


def test_radius_normals(gpu):
    """k_normals_from_csr: a small radius that leaves 3-5 neighbours (and many NaN rows), and a larger one."""
    P, ctx = gpu
    pts, vp = R.sine_sheet()
    cloud = _xyz1(P, pts)
    cloud[::501, 0] = np.nan
    sub = np.random.default_rng(8).permutation(cloud.shape[0])[:7000].astype(np.int32)
    for r, ind in ((0.004, None), (0.02, None), (0.02, sub)):
        q = cloud if ind is None else cloud[ind]
        g, gd = P.Index(ctx, cloud).normals_radius(cloud, r, viewpoint=vp, indices=ind, is_dense=False)
        ref = R.Reference(cloud, q, vp, radius=r)
        assert gd == ref.is_dense
        if r < 0.01:
            counts = np.array([s.size for s in ref.sets])
            assert np.mean((counts >= 3) & (counts <= 5)) > 0.3
        _record(f"k_normals_from_csr r={r}", ref.check(g, f"radius {r}"))
    pts, vp, exp = R.exact_clusters(8)
    cloud = _xyz1(P, pts)
    g, gd = P.Index(ctx, cloud).normals_radius(cloud, 100.0, viewpoint=vp)
    assert gd
    R.exact_check(g, exp, "radius exact")


@pytest.mark.parametrize("k", [5, 20])
def test_gicp_covariances(gpu, k):
    P, ctx = gpu
    for name, pts in R.gicp_scenes():
        cloud = _xyz1(P, pts)
        g = P.Index(ctx, cloud).gicp_covariances(cloud, k=k, gicp_epsilon=0.001)
        worst, n = R.gicp_check(cloud, g, k, 0.001, f"{name} k={k}")
        print(f"device gicp {name:12s} k={k:2d}  worst ratio {worst:.3g} over {n} rows")
    few = _xyz1(P, np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0]]))
    R.gicp_check(few, P.Index(ctx, few).gicp_covariances(few, k=k, gicp_epsilon=0.001), k, 0.001, "fewer than k")
