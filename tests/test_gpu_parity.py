"""Parity of the CUDA path (through the C-ABI) against the CPU oracle and the reference's golden vectors.
Bit-exact for indices and squared distances; transforms within the tolerance BASELINE.json states
(1e-5 Frobenius).  Needs an H100: run with -m gpu."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    import pcl_b200
    pcl_b200.lib()
    ctx = pcl_b200.Context(0)
    yield pcl_b200, ctx
    ctx.close()


def _reference(cloud, queries, vp, **kw):
    """The per-query extended-precision reference of tests/test_normals_reference.py."""
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import test_normals_reference
    return test_normals_reference.Reference(cloud, queries, vp, **kw)


def _clouds(rng):
    yield "uniform", rng.random((20000, 3), dtype=np.float32)
    g = np.stack(np.meshgrid(*[np.arange(13, dtype=np.float32)] * 3, indexing="ij"), -1).reshape(-1, 3)
    yield "grid_ties", g
    d = rng.random((700, 3), dtype=np.float32)
    yield "duplicates", np.concatenate([d, d, d[:300]])
    yield "collinear", np.stack([np.linspace(0, 1, 1777, dtype=np.float32)] * 3, 1)
    yield "tiny", rng.random((5, 3), dtype=np.float32)
    yield "single", rng.random((1, 3), dtype=np.float32)
    yield "all_same", np.ones((300, 3), dtype=np.float32) * np.float32(0.25)
    s = rng.normal(size=(30000, 3)).astype(np.float32)
    s[:, 2] = np.float32(0.3) * np.sin(s[:, 0]) * np.cos(s[:, 1])
    yield "surface", s


# ---------------------------------------------------------------------------------------------------------------------
# k-NN: bit-exact indices and distances
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 2, 3, 5, 8, 10, 16, 20, 32, 40])
def test_knn_bit_exact(gpu, orc, k):
    P, ctx = gpu
    rng = np.random.default_rng(11)
    for name, pts in _clouds(rng):
        cloud = orc.to_xyz1(pts)
        q = orc.to_xyz1(np.concatenate([pts[:300], (rng.random((300, 3), dtype=np.float32) - np.float32(0.2)) * (np.abs(pts).max() + 1)]))
        gi, gd, gk = P.Index(ctx, cloud).knn(q, k)
        oi, od, ok = orc.Index(cloud).knn(q, k, nthreads=4)
        assert gk == ok, name
        assert np.array_equal(gi, oi), (name, k, np.argwhere(gi != oi)[:5])
        assert np.array_equal(gd, od), (name, k)


def test_knn_golden_10_points(gpu, golden):
    # test/kdtree/test_kdtree.cpp:229-262
    P, ctx = gpu
    idx, d2, keff = P.Index(ctx, P.xyz1(golden["knn10_points"])).knn(P.xyz1(golden["knn10_query"][None]), 10)
    assert keff == 10
    assert np.array_equal(idx[0], golden["knn10_indices"])
    assert np.allclose(d2[0], golden["knn10_distances"], atol=0.1)
    idx, d2, keff = P.Index(ctx, P.xyz1(golden["knn10_points"])).knn(P.xyz1(golden["knn10_query"][None]), 15)
    assert keff == 10 and np.all(idx[0, 10:] == -1) and np.all(np.isinf(d2[0, 10:]))


def test_knn_and_normals_many_k(gpu, orc):
    """Exact k-NN lists for every compiled list size (and NaN queries); normals built on them agree with the oracle."""
    P, ctx = gpu
    walk = "default"
    rng = np.random.default_rng(12)
    for name, pts in _clouds(rng):
        cloud = orc.to_xyz1(pts)
        q = orc.to_xyz1(np.concatenate([pts[:257], (rng.random((100, 3), dtype=np.float32) - np.float32(0.2)) * (np.abs(pts).max() + 1)]))
        q[3::50, 2] = np.nan  # non-finite queries: empty rows
        for k in (1, 4, 10, 16, 20, 32):
            gi, gd, gk = P.Index(ctx, cloud).knn(q, k)
            oi, od, ok = orc.Index(cloud).knn(q, k, nthreads=4)
            fin = np.isfinite(q[:, 2])
            assert gk == ok and np.array_equal(gi[fin], oi[fin]) and np.array_equal(gd[fin], od[fin]), (name, k, walk)
            assert np.all(gi[~fin] == -1) and np.all(np.isinf(gd[~fin]))
    pts = rng.random((30000, 3), dtype=np.float32)
    pts[:, 2] = np.float32(0.1) * np.sin(np.float32(6) * pts[:, 0])
    cloud = orc.to_xyz1(pts)
    cloud[::301, 1] = np.nan
    for k in (5, 16, 32):
        g, gd = P.Index(ctx, cloud).normals_knn(cloud, k, viewpoint=(0.5, 0.5, 5), is_dense=False)
        o, od = orc.Index(cloud).normals_knn(cloud, k, viewpoint=(0.5, 0.5, 5), is_dense=False, nthreads=8)
        assert gd == od and np.array_equal(np.isnan(g[:, 0]), np.isnan(o[:, 0]))
        _reference(cloud, cloud, (0.5, 0.5, 5), k=k).check(g, f"k={k} {walk}")


def test_knn_warp_kernel_mixed_density_every_query(gpu, orc):
    """The warp-per-query kernel (12 <= k <= 32) on a cloud whose density changes by orders of magnitude — a dense sheet
    inside a sparse volume, so 8-point leaves span several of the cells a query gathers (a leaf shared by cells whose
    common nearer cell is empty must not be pruned by the bound of the wrong cell) — every point as a query plus
    queries off the cloud (empty home cell), all rows bit-exact against the oracle."""
    import os
    P, ctx = gpu
    rng = np.random.default_rng(77)
    n_sheet, n_vol = 340_000, 60_000
    sheet = rng.random((n_sheet, 3), dtype=np.float32) * np.float32(2.0)
    sheet[:, 2] = np.float32(0.3) * np.sin(np.float32(3) * sheet[:, 0]) * np.cos(np.float32(2) * sheet[:, 1]) + \
        np.float32(0.001) * rng.standard_normal(n_sheet).astype(np.float32)
    vol = (rng.random((n_vol, 3), dtype=np.float32) * np.float32(2.0))
    vol[:, 2] = vol[:, 2] - np.float32(1.0)
    pts = np.concatenate([sheet, vol])[rng.permutation(n_sheet + n_vol)]
    cloud = orc.to_xyz1(pts)
    off = orc.to_xyz1((rng.random((50_000, 3), dtype=np.float32) * np.float32(2.4) - np.float32(0.2)))
    q = np.concatenate([cloud, off])
    gidx, oidx = P.Index(ctx, cloud), orc.Index(cloud)
    nt = os.cpu_count() or 8
    for k in (12, 16, 24, 32):
        gi, gd, gk = gidx.knn(q, k)
        oi, od, ok = oidx.knn(q, k, nthreads=nt)
        bad = np.nonzero((gi != oi).any(axis=1) | (gd != od).any(axis=1))[0]
        assert gk == ok and bad.size == 0, (k, bad.size, bad[:5].tolist())


def test_knn_nan_points_subset_and_strides(gpu, orc):
    P, ctx = gpu
    rng = np.random.default_rng(12)
    pts = rng.random((5000, 3), dtype=np.float32)
    pts[::7, 1] = np.nan
    pts[5, 0] = np.inf
    cloud = orc.to_xyz1(pts)
    q = orc.to_xyz1(rng.random((500, 3), dtype=np.float32))
    gidx = P.Index(ctx, cloud)
    assert gidx.size == orc.Index(cloud).size == int(np.isfinite(pts).all(1).sum())
    gi, gd, _ = gidx.knn(q, 4)
    oi, od, _ = orc.Index(cloud).knn(q, 4)
    assert np.array_equal(gi, oi) and np.array_equal(gd, od)
    sub = np.arange(0, 5000, 3, dtype=np.int32)
    gi, gd, _ = P.Index(ctx, cloud, subset=sub).knn(q, 3)
    oi, od, _ = orc.Index(cloud, subset=sub).knn(q, 3)
    assert np.array_equal(gi, oi) and np.array_equal(gd, od)
    # pcl::PointNormal stride (48 B) and packed xyz (12 B)
    pn = np.zeros((5000, 12), np.float32)
    pn[:, :3] = pts
    gi2, gd2, _ = P.Index(ctx, pn).knn(np.ascontiguousarray(q[:, :3]), 4)
    oi2, od2, _ = orc.Index(cloud).knn(q, 4)
    assert np.array_equal(gi2, oi2) and np.array_equal(gd2, od2)
    with pytest.raises(P.Pclb200Error) as e:
        P.Index(ctx, np.full((10, 4), np.nan, np.float32))
    assert e.value.code == P.ERR_EMPTY


# ---------------------------------------------------------------------------------------------------------------------
# radius search
# ---------------------------------------------------------------------------------------------------------------------
def test_radius_golden_3283_lists(gpu, golden):
    # test/kdtree/test_kdtree.cpp:292-328: exact count and ORDER of every list
    P, ctx = gpu
    cloud = P.xyz1(golden["sac_plane"])
    offs, idx, d2 = P.Index(ctx, cloud).radius(cloud, float(golden["radius_r"]))
    assert np.array_equal(offs, golden["radius_offsets"])
    assert np.array_equal(idx, golden["radius_indices"])


def test_radius_vs_oracle(gpu, orc):
    P, ctx = gpu
    rng = np.random.default_rng(13)
    for name, pts in _clouds(rng):
        cloud = orc.to_xyz1(pts)
        q = cloud[:400]
        r = float(np.abs(pts).max()) * 0.08 + 1e-3
        go, gi, gd = P.Index(ctx, cloud).radius(q, r)
        oo, oi, od = orc.Index(cloud).radius(q, r, nthreads=4)
        assert np.array_equal(go, oo), name
        assert np.array_equal(gi, oi), name
        assert np.array_equal(gd, od), name
        go, gi, gd = P.Index(ctx, cloud).radius(q, r, max_nn=5)
        oo, oi, od = orc.Index(cloud).radius(q, r, max_nn=5, nthreads=4)
        assert np.array_equal(go, oo) and np.array_equal(gi, oi) and np.array_equal(gd, od), name


def test_radius_maxnn_dense_balls(gpu, orc):
    """Balls that hold far more than max_nn points are searched by the bounded k-NN kernel instead of being
    materialised (capi.cu: pclb200_radius); both strategies must return FLANN's KNNRadius answer."""
    P, ctx = gpu
    rng = np.random.default_rng(14)
    pts = rng.random((40000, 3), dtype=np.float32)
    pts[::9] = pts[1::9][: pts[::9].shape[0]]  # exact duplicates: distance ties inside the kept prefix
    cloud = orc.to_xyz1(pts)
    q = orc.to_xyz1(np.concatenate([pts[:500], rng.random((300, 3), dtype=np.float32) * 1.4 - 0.2]))
    gi, oi = P.Index(ctx, cloud), orc.Index(cloud)
    for r, max_nn in ((0.2, 4), (0.2, 32), (0.12, 10), (0.05, 3), (0.02, 32)):  # ~1300 / ~290 / ~20 / ~1.3 points per ball
        go, gidx, gd = gi.radius(q, r, max_nn=max_nn)
        oo, oidx, od = oi.radius(q, r, max_nn=max_nn, nthreads=8)
        assert np.array_equal(go, oo) and np.array_equal(gidx, oidx) and np.array_equal(gd, od), (r, max_nn)
        assert np.diff(go).max() <= max_nn


# ---------------------------------------------------------------------------------------------------------------------
# correspondences
# ---------------------------------------------------------------------------------------------------------------------
def test_correspondences_golden_397_and_53(gpu, golden):
    # test/registration/test_registration_api.cpp:83-128
    P, ctx = gpu
    src, tgt = P.xyz1(golden["bun0"]), P.xyz1(golden["bun4"])
    t = P.Index(ctx, tgt)
    c = t.correspondences(src)
    assert c.size == 397
    assert np.array_equal(c["index_query"], golden["corr_original"][:, 0])
    assert np.array_equal(c["index_match"], golden["corr_original"][:, 1])
    c = t.correspondences(src, src_index=P.Index(ctx, src))
    assert c.size == 53
    assert np.array_equal(c["index_query"], golden["corr_reciprocal"][:, 0])
    assert np.array_equal(c["index_match"], golden["corr_reciprocal"][:, 1])


def test_correspondences_vs_oracle(gpu, orc):
    P, ctx = gpu
    rng = np.random.default_rng(14)
    tgt = orc.to_xyz1(rng.random((50000, 3), dtype=np.float32))
    src = orc.to_xyz1(rng.random((40000, 3), dtype=np.float32))
    src[::11, 0] = np.nan
    gt, ot = P.Index(ctx, tgt), orc.Index(tgt)
    for md in (0.01, 0.02, 1e9):
        g = gt.correspondences(src, max_distance=md, is_dense=False)
        o = ot.correspondences(src, max_distance=md, is_dense=False, nthreads=4)
        assert np.array_equal(g, o), md
    ind = rng.permutation(40000)[:9000].astype(np.int32)
    g = gt.correspondences(src, max_distance=0.02, indices=ind, is_dense=False)
    o = ot.correspondences(src, max_distance=0.02, indices=ind, is_dense=False)
    assert np.array_equal(g, o)
    srcf = src.copy()
    srcf[::11, 0] = 0.5
    g = gt.correspondences(srcf, max_distance=0.03, src_index=P.Index(ctx, srcf))
    o = ot.correspondences_reciprocal(srcf, orc.Index(srcf), max_distance=0.03, nthreads=4)
    assert np.array_equal(g, o)


# ---------------------------------------------------------------------------------------------------------------------
# estimators
# ---------------------------------------------------------------------------------------------------------------------
def test_estimate_svd_golden(gpu, golden, orc):
    # test/registration/test_registration_api.cpp:383-423
    P, ctx = gpu
    src = P.xyz1(golden["bun4"])
    Tref = golden["svd_Tref"]
    tgt = orc.transform(src, Tref, mode=1)
    for dbl in (False, True):
        T = ctx.estimate_svd(src, tgt, scalar_is_double=dbl)
        assert np.allclose(T, Tref, atol=2e-6)
        T64 = orc.estimate_svd(src, tgt, scalar_is_double=True)
        assert np.linalg.norm(T - T64) < (1e-9 if dbl else 1e-6)
        corr = np.zeros(src.shape[0], dtype=P.CORR_DTYPE)
        corr["index_query"] = corr["index_match"] = np.arange(src.shape[0])
        assert np.array_equal(ctx.estimate_svd(src, tgt, corr=corr, scalar_is_double=dbl), T)


def test_estimate_point_to_plane_golden(gpu, orc):
    # test/registration/test_registration_api.cpp:469-518
    P, ctx = gpu
    xs = np.arange(-5.0, 5.0 + 1e-6, 0.5, dtype=np.float32)
    X, Y = np.meshgrid(xs, xs, indexing="ij")
    x, y = X.ravel(), Y.ravel()
    z = np.float32(0.1) * x ** 2 + np.float32(0.2) * x * y - np.float32(0.3) * y + np.float32(1.0)
    n = np.stack([-0.2 * x - 0.2, 0.6 * y - 0.2, np.ones_like(x)], 1).astype(np.float32)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    src = np.zeros((x.size, 12), np.float32)
    src[:, 0], src[:, 1], src[:, 2], src[:, 3] = x, y, z, 1
    src[:, 4:7] = n
    G = np.array([[0.9938, 0.0988, 0.0517, 0.1], [-0.0997, 0.9949, 0.0149, -0.2], [-0.05, -0.02, 0.9986, 0.3],
                  [0, 0, 0, 1]], np.float64)
    tgt = orc.transform(src, G, mode=1, normal_off=4)
    T = ctx.estimate_point_to_plane_lls(src, tgt)
    assert np.all(np.abs(T - G) < 1e-2)
    To, _ = orc.estimate_point_to_plane_lls(src, tgt)
    assert np.linalg.norm(T - To) < 1e-6
    Td = ctx.estimate_point_to_plane_lls(src, tgt, scalar_is_double=True)
    Tod, _ = orc.estimate_point_to_plane_lls(src, tgt, scalar_is_double=True)
    assert np.linalg.norm(Td - Tod) < 1e-10


# ---------------------------------------------------------------------------------------------------------------------
# ICP
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dbl", [False, True])
def test_icp_bun0_bun4_golden(gpu, golden, orc, dbl):
    # test/registration/test_registration.cpp:236-270 — config 1 of BASELINE.json
    P, ctx = gpu
    src, tgt = P.xyz1(golden["bun0"]), P.xyz1(golden["bun4"])
    out = np.zeros_like(src)
    r = P.icp_align(ctx, src, P.Index(ctx, tgt), out_cloud=out, max_iterations=50, transformation_epsilon=1e-8,
                    max_correspondence_distance=0.05, scalar_is_double=int(dbl))
    T, G = r["final"], golden["icp_bun0_bun4"]
    tol = np.full((4, 4), 1e-3)
    tol[0, 1] = 1e-2
    tol[3, :] = 0
    assert r["converged"] and np.all(np.abs(T - G) <= tol), (T, r)
    o = orc.icp_align(src, tgt, max_iterations=50, transformation_epsilon=1e-8, max_correspondence_distance=0.05,
                      scalar_is_double=dbl, want_cloud=True)
    assert r["iterations"] == o["iterations"] and r["state"] == o["state"], (r, o)
    assert np.linalg.norm(T - o["final"]) < 1e-5, np.linalg.norm(T - o["final"])
    o64 = orc.icp_align(src, tgt, max_iterations=50, transformation_epsilon=1e-8, max_correspondence_distance=0.05,
                        scalar_is_double=True)
    assert np.linalg.norm(T - o64["final"]) < 1e-5
    assert r["n_correspondences"] == o["n_correspondences"]
    assert np.allclose(out, o["cloud"], atol=1e-6)
    assert np.all(out[:, 3] == 1.0)


def test_icp_translated_and_fitness(gpu, golden, orc):
    # test/registration/test_registration.cpp:161-233
    P, ctx = gpu
    src = P.xyz1(golden["bun0"])
    tgt = src.copy()
    tgt[:, 2] += np.float32(0.2)
    t = P.Index(ctx, tgt)
    r = P.icp_align(ctx, src, t, max_iterations=50)
    assert r["converged"]
    assert t.fitness_score(src, r["final"]) < 1e-6
    assert np.allclose(np.diag(r["final"])[:3], 1.0, atol=2e-3) and np.allclose(r["final"][:3, 3], [0, 0, 0.2], atol=2e-3)
    o = orc.icp_align(src, tgt, max_iterations=50)
    assert r["iterations"] == o["iterations"] and np.linalg.norm(r["final"] - o["final"]) < 1e-5
    s4 = P.xyz1(np.array([[0, 0, 0], [0, 1, 0], [0, 0, 1], [10, 0, 0]], np.float32))
    t4 = P.Index(ctx, P.xyz1(np.array([[0, 0, 0], [0, 1, 0], [0, 0, 1], [10, 0, 0.5]], np.float32)))
    assert abs(t4.fitness_score(s4, np.eye(4), max_range=1.0) - 0.0625) < 1e-4
    assert abs(t4.fitness_score(s4, np.eye(4), max_range=1.0, indices=np.array([0, 1, 2], np.int32))) < 1e-4
    assert t4.fitness_score(s4 + 100, np.eye(4), max_range=1.0) == np.finfo(np.float64).max


def _synthetic_pair(rng, n, noise=0.001):
    tgt = rng.random((n, 3), dtype=np.float32)
    ang = np.deg2rad(5.0)
    ax = np.ones(3) / np.sqrt(3)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    R = np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K
    src = (tgt.astype(np.float64) @ R.T + np.array([0.01, -0.02, 0.015]) + rng.normal(0, noise, (n, 3))).astype(np.float32)
    return src, tgt


@pytest.mark.parametrize("recip", [False, True])
def test_icp_synthetic_vs_oracle(gpu, orc, recip):
    # config 2 shape at a size the oracle finishes in seconds
    P, ctx = gpu
    src, tgt = _synthetic_pair(np.random.default_rng(42), 60000)
    src, tgt = P.xyz1(src), P.xyz1(tgt)
    kw = dict(max_iterations=40, transformation_epsilon=1e-10, max_correspondence_distance=0.05)
    r = P.icp_align(ctx, src, P.Index(ctx, tgt), use_reciprocal=int(recip), **kw)
    o = orc.icp_align(src, tgt, use_reciprocal=recip, nthreads=8, **kw)
    o64 = orc.icp_align(src, tgt, use_reciprocal=recip, nthreads=8, scalar_is_double=True, **kw)
    assert r["converged"] == o["converged"]
    assert np.linalg.norm(r["final"] - o64["final"]) < 1e-5, (np.linalg.norm(r["final"] - o64["final"]), r, o64)
    assert abs(r["iterations"] - o["iterations"]) <= 1, (r["iterations"], o["iterations"])


def test_icp_guess_indices_and_stepwise(gpu, orc):
    P, ctx = gpu
    src, tgt = _synthetic_pair(np.random.default_rng(43), 20000)
    src, tgt = P.xyz1(src), P.xyz1(tgt)
    guess = np.eye(4)
    guess[:3, 3] = [-0.005, 0.01, -0.01]
    ind = np.arange(0, 20000, 2, dtype=np.int32)
    kw = dict(max_iterations=15, max_correspondence_distance=0.05)
    t = P.Index(ctx, tgt)
    r = P.icp_align(ctx, src, t, guess=guess, indices=ind, **kw)
    o = orc.icp_align(src, tgt, guess=guess, indices=ind, **kw)
    o64 = orc.icp_align(src, tgt, guess=guess, indices=ind, scalar_is_double=True, **kw)
    # the stop here is the |mse - prev_mse| < 1e-12 test on an mse of ~3e-6: it sits at fp32 round-off, so the
    # reference's own float and double instantiations may stop an iteration apart; the fixed point must agree.
    assert abs(r["iterations"] - o["iterations"]) <= 2 and abs(r["iterations"] - o64["iterations"]) <= 2
    assert np.linalg.norm(r["final"] - o["final"]) < 1e-5
    assert np.linalg.norm(r["final"] - o64["final"]) < 1e-5
    # the session API stepped one iteration at a time reaches the same state
    s = P.Icp(ctx, **kw)
    s.set_target(t)
    s.set_source(src, indices=ind, guess=guess)
    st = None
    for _ in range(100):
        st = s.iterate(1)
        if st["state"] != 0:
            break
    assert st["iterations"] == r["iterations"] and np.array_equal(st["final"], r["final"])
    # too few correspondences: NO_CORRESPONDENCES, not converged (icp.hpp:204-213)
    far = src.copy()
    far[:, :3] += 100
    r = P.icp_align(ctx, far, t, max_iterations=5, max_correspondence_distance=0.01)
    assert not r["converged"] and r["state"] == 5 and r["iterations"] == 0


def test_icp_point_to_plane_vs_oracle(gpu, orc):
    # config 3 shape (normals k=16 + TransformationEstimationPointToPlaneLLS), small
    P, ctx = gpu
    rng = np.random.default_rng(7)
    n = 40000

    def surf(m, seed):
        r = np.random.default_rng(seed)
        xy = r.random((m, 2)) * 10
        z = 0.5 * np.sin(xy[:, 0]) * np.cos(0.7 * xy[:, 1]) + r.normal(0, 0.002, m)
        return np.column_stack([xy, z])

    tgt_xyz = surf(n, 7).astype(np.float32)
    a = np.deg2rad(2.0)
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    src_xyz = (surf(n, 8) @ R.T + np.array([0.02, 0.01, -0.01])).astype(np.float32)
    tgt = np.zeros((n, 12), np.float32)
    tgt[:, :3], tgt[:, 3] = tgt_xyz, 1
    tidx = P.Index(ctx, tgt)
    normals, dense = tidx.normals_knn(tgt, 16, viewpoint=(5, 5, 10))
    on, odense = orc.Index(tgt).normals_knn(tgt, 16, viewpoint=(5, 5, 10), nthreads=8)
    assert dense == odense
    cosang = np.abs((normals[:, :3] * on[:, :3]).sum(1))
    assert np.percentile(cosang, 1) > 1 - 1e-4 and np.mean(cosang > 1 - 1e-6) > 0.95
    assert np.allclose(normals[:, 3], on[:, 3], atol=2e-3)
    tgt[:, 4:8] = on  # same normals on both sides so the ICP comparison isolates the registration path
    src = np.zeros((n, 12), np.float32)
    src[:, :3], src[:, 3] = src_xyz, 1
    kw = dict(max_iterations=30, max_correspondence_distance=0.05)
    r = P.icp_align(ctx, src, tidx, tgt_normals=P.Field(tgt, 4), estimator=P.EST_POINT_TO_PLANE_LLS,
                    with_normals_transform=1, **kw)
    o = orc.icp_align(src, tgt, estimator=1, with_normals_transform=True, nthreads=8, **kw)
    assert r["iterations"] == o["iterations"] and r["state"] == o["state"], (r, o)
    assert np.linalg.norm(r["final"] - o["final"]) < 1e-5, np.linalg.norm(r["final"] - o["final"])


# ---------------------------------------------------------------------------------------------------------------------
# normals and voxel grid
# ---------------------------------------------------------------------------------------------------------------------
def test_normal_bun0_golden(gpu, golden):
    # test/features/test_normal_estimation.cpp:98-163 with k = 32 < cloud: compare with the all-points plane instead
    P, ctx = gpu
    cloud = P.xyz1(golden["bun0"])
    normals, dense = P.Index(ctx, cloud).normals_knn(cloud, 10)
    assert dense and np.allclose(np.linalg.norm(normals[:, :3], axis=1), 1, atol=1e-4)
    # flipped toward the origin viewpoint (normal_3d.h:169-188)
    assert np.all((-(cloud[:, :3]) * normals[:, :3]).sum(1) >= -1e-6)


def test_normals_vs_oracle(gpu, orc):
    P, ctx = gpu
    rng = np.random.default_rng(15)
    pts = rng.random((30000, 3), dtype=np.float32)
    pts[:, 2] = np.float32(0.1) * np.sin(np.float32(6) * pts[:, 0])
    cloud = orc.to_xyz1(pts)
    for k in (5, 10, 16):
        g, gd = P.Index(ctx, cloud).normals_knn(cloud, k, viewpoint=(0.5, 0.5, 5))
        o, od = orc.Index(cloud).normals_knn(cloud, k, viewpoint=(0.5, 0.5, 5), nthreads=8)
        assert gd == od
        _reference(cloud, cloud, (0.5, 0.5, 5), k=k).check(g, f"k={k}")  # every normal and curvature
    few = orc.to_xyz1(pts[:2])
    g, gd = P.Index(ctx, few).normals_knn(few, 5)
    assert not gd and np.isnan(g).all()  # < 3 neighbours => NaN, is_dense false (normal_3d.hpp:62-69)


def test_voxelgrid_golden_and_oracle(gpu, golden, orc):
    # test/filters/test_filters.cpp:566-603
    P, ctx = gpu
    cloud = P.xyz1(golden["bun0"])
    out = ctx.voxelgrid(cloud, 0.02)
    assert out.shape[0] == 103
    assert np.array_equal(out, orc.voxelgrid(cloud, [0.02] * 3))
    z = cloud[:, 2]
    sel = np.nonzero(~((z > np.float32(0.1)) | (z < np.float32(0.05))))[0].astype(np.int32)
    out = ctx.voxelgrid(cloud, 0.02, indices=sel)
    assert out.shape[0] == 14
    assert np.allclose(out[0, :3], golden["voxel_z_first"], atol=1e-4) and np.allclose(out[13, :3], golden["voxel_z_last"], atol=1e-4)
    with pytest.raises(P.Pclb200Error) as e:
        ctx.voxelgrid(cloud, 1e-5)
    assert e.value.code == P.ERR_LEAF_TOO_SMALL
    rng = np.random.default_rng(16)
    big = orc.to_xyz1((rng.random((200000, 3), dtype=np.float32) - np.float32(0.3)) * np.float32(3))
    big[::13, 1] = np.nan
    for leaf, mp in (([0.01] * 3, 0), ([0.05, 0.1, 0.2], 0), ([0.1] * 3, 30)):
        g = ctx.voxelgrid(big, leaf, min_points_per_voxel=mp, is_dense=False)
        o = orc.voxelgrid(big, leaf, min_points_per_voxel=mp, is_dense=False)
        assert g.shape == o.shape and np.array_equal(g, o), (leaf, mp)


def _coherence_scenes():
    rng = np.random.default_rng(77)
    n = 50000
    xy = rng.random((n, 2)) * 4
    tgt = np.column_stack([xy, 0.3 * np.sin(xy[:, 0]) * np.cos(xy[:, 1]) + rng.normal(0, 0.002, n)]).astype(np.float32)
    a = np.deg2rad(1.0)
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    src = (tgt.astype(np.float64)[::2] @ R.T + [0.01, 0.005, -0.004]).astype(np.float32)
    src[5, 0] = np.nan
    yield "surface_subsample", tgt, src, 0.05
    # a different sample of the same surface (no exact mates), tiny motion: the regime where most walks are skipped
    xy2 = rng.random((30000, 2)) * 4
    src2 = np.column_stack([xy2 + 0.0005, 0.3 * np.sin(xy2[:, 0]) * np.cos(xy2[:, 1]) + rng.normal(0, 0.002, 30000)]).astype(np.float32)
    yield "surface_resample", tgt, src2, 0.05
    cube = rng.random((40000, 3), dtype=np.float32)
    yield "cube_gated", cube, (cube[:20000].astype(np.float64) * 1.0005 + 0.002).astype(np.float32), 0.02
    g = np.stack(np.meshgrid(*[np.arange(24, dtype=np.float32)] * 3, indexing="ij"), -1).reshape(-1, 3)
    yield "lattice_ties", g, (g[::3] + np.float32(0.26)).astype(np.float32), 1e9
    # every target point 12 times (more copies than a leaf holds: the tree has to cut INSIDE runs of equal Morton codes,
    # the cells a seeded walk must not start from) plus clusters far tighter than the quantisation step
    base = rng.random((1500, 3), dtype=np.float32)
    dup = np.concatenate([np.repeat(base, 12, axis=0), base[:200] + np.float32(1e-7) * rng.standard_normal((200, 3)).astype(np.float32)])
    dup = dup[rng.permutation(dup.shape[0])]
    yield "duplicates_x12", dup, (base[:900].astype(np.float64) * 1.001 + 0.0007).astype(np.float32), 1e9


def test_icp_per_iteration_correspondences_exact(gpu, orc):
    """The search kernel starts every walk at the candidate ball (cell table) and skips the walk altogether for queries
    whose previous match is provably still nearest (temporal coherence).  Neither may ever change a result: every
    iteration's correspondence list is compared, bit for bit, with a fresh exact search of the oracle on the same
    (re-transformed) cloud — with the lower-bound tracking forced on from the first iteration, forced off, and in the
    default automatic mode, on scenes with duplicates, exact ties, a gate and NaNs."""
    P, ctx = gpu
    total_skipped = 0
    for name, tgt, src, gate in _coherence_scenes():
        T, S = P.xyz1(tgt), P.xyz1(src)
        oidx = orc.Index(T)
        tidx = P.Index(ctx, T)
        for track in (P.TRACK_ON, P.TRACK_OFF, P.TRACK_AUTO):
            s = P.Icp(ctx, max_iterations=30, max_correspondence_distance=gate, is_dense=0, mse_threshold_absolute=0.0,
                      track_mode=track)
            s.set_target(tidx)
            s.set_source(S)
            cloud = S.copy()
            st = None
            for it in range(30):
                st = s.iterate(1)
                g = s.get_correspondences()
                o = oidx.correspondences(cloud, max_distance=gate, is_dense=False, nthreads=4)
                assert np.array_equal(g, o), (name, track, it, g.size, o.size)
                assert st["n_correspondences"] == o.size
                cloud = orc.transform(cloud, st["last"], mode=0)   # IterativeClosestPoint::transformCloud, fp32
                if st["state"] != 0:
                    break
            if track == P.TRACK_ON:
                total_skipped += st["total_skipped_walks"]
    assert total_skipped > 0, "the temporal-coherence path was never exercised"


def test_rejectors_golden_and_oracle(gpu, golden, orc):
    """The four correspondence rejectors (SURVEY.md §8f #1): PCL's golden pair lists
    (test/registration/test_registration_api.cpp:131-380) and bit-exact agreement with the oracle on random input."""
    P, ctx = gpu
    c = P.Index(ctx, P.xyz1(golden["bun4"])).correspondences(P.xyz1(golden["bun0"]))
    for kind, p, key in ((P.REJ_DISTANCE, 0.01, "corr_rej_dist"), (P.REJ_MEDIAN, 0.5, "corr_rej_median"),
                         (P.REJ_ONE_TO_ONE, 0.0, "corr_rej_one_to_one"), (P.REJ_TRIMMED, 0.5, "corr_rej_trimmed")):
        r, med = ctx.reject(c, kind, p=p)
        assert np.array_equal(np.stack([r["index_query"], r["index_match"]], 1), golden[key]), key
        if kind == P.REJ_MEDIAN:
            assert abs(med - 0.000465391) < 1e-4
    rng = np.random.default_rng(31)
    n = 200000
    big = np.zeros(n, dtype=P.CORR_DTYPE)
    big["index_query"] = np.arange(n)
    big["index_match"] = rng.integers(0, n // 3, n)
    big["distance"] = (rng.random(n, dtype=np.float32) ** 2).astype(np.float32)
    big["distance"][::97] = big["distance"][5]           # exact ties
    for kind, p, m in ((P.REJ_DISTANCE, 0.5, 0), (P.REJ_MEDIAN, 1.7, 0), (P.REJ_ONE_TO_ONE, 0.0, 0),
                       (P.REJ_TRIMMED, 0.37, 0), (P.REJ_TRIMMED, 0.01, 5000), (P.REJ_TRIMMED, 1.0, 0)):
        g, gm = ctx.reject(big, kind, p=p, min_correspondences=m)
        o, om = orc.reject(big, kind, p=p, min_correspondences=m)
        assert np.array_equal(g, o), (kind, p, m, g.size, o.size)
        assert gm == om
    e, _ = ctx.reject(big[:0], P.REJ_MEDIAN, p=1.0)
    assert e.size == 0


def test_icp_with_rejector_chain_vs_oracle(gpu, orc):
    """Rejectors inside the device loop (icp.hpp:187-201): per-iteration correspondence counts and the final
    transform agree with the oracle's loop (counts to 0.1 %: the float and double solves move borderline pairs)."""
    P, ctx = gpu
    rng = np.random.default_rng(32)
    n = 40000
    tgt = rng.random((n, 3), dtype=np.float32)
    a = np.deg2rad(3.0)
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    src = (tgt.astype(np.float64)[: n // 2] @ R.T + [0.01, -0.01, 0.02] + rng.normal(0, 0.002, (n // 2, 3))).astype(np.float32)
    src[:500] += np.float32(0.3)                          # gross outliers for the rejectors to remove
    S, T = P.xyz1(src), P.xyz1(tgt)
    chains = [[(P.REJ_MEDIAN, 3.0, 0)], [(P.REJ_ONE_TO_ONE, 0.0, 0)], [(P.REJ_TRIMMED, 0.9, 100)], [(P.REJ_DISTANCE, 0.2, 0)],
              [(P.REJ_MEDIAN, 3.0, 0), (P.REJ_ONE_TO_ONE, 0.0, 0), (P.REJ_TRIMMED, 0.9, 100), (P.REJ_DISTANCE, 0.2, 0)]]
    tidx = P.Index(ctx, T)
    for chain in chains:
        s = P.Icp(ctx, max_iterations=30, transformation_epsilon=1e-9)
        s.set_rejectors(chain)
        s.set_target(tidx)
        s.set_source(S)
        for k in range(1, 7):
            g = s.iterate(1)
            o = orc.icp_align_rejectors(S, T, chain, nthreads=4, max_iterations=k, transformation_epsilon=1e-9)
            assert abs(g["n_correspondences"] - o["n_correspondences"]) <= max(3, 0.001 * o["n_correspondences"]), (chain, k)
            # mid-trajectory: a handful of borderline pairs flip between the fp32 (oracle) and fp64 (device) solves
            assert np.linalg.norm(g["final"] - o["final"]) < 1e-4, (chain, k)
        if len(chain) == 4:
            assert g["n_correspondences"] < 0.8 * S.shape[0]
        g = s.iterate()                                      # run to convergence
        o64 = orc.icp_align_rejectors(S, T, chain, nthreads=4, max_iterations=30, transformation_epsilon=1e-9,
                                      scalar_is_double=True)
        assert g["converged"] and o64["converged"]
        assert np.linalg.norm(g["final"] - o64["final"]) < 5e-5, (chain, np.linalg.norm(g["final"] - o64["final"]))
    s = P.Icp(ctx, max_iterations=30, transformation_epsilon=1e-9)
    s.set_target(tidx)
    s.set_source(S)
    assert s.iterate(1)["n_correspondences"] == S.shape[0]   # no rejectors, no gate: every source point pairs up


@pytest.mark.parametrize("dbl", [False, True], ids=["float", "double"])
@pytest.mark.parametrize("track", ["on", "off", "auto"])
def test_icp_per_iteration_sync_matches_single_sync(gpu, track, dbl):
    """icp_iterate synchronises once per call, or after every iteration when a stage between search and solve needs the
    host (here a rejector chain).  A distance rejector far above the gate keeps every pair, so its only effect is the
    per-iteration synchronisation: stepped one iteration at a time and then run to the end, both modes go through the
    same states, counts and transforms, bit for bit, in every tracking mode."""
    P, ctx = gpu
    src, tgt = _synthetic_pair(np.random.default_rng(44), 30000)
    src, tgt = P.xyz1(src), P.xyz1(tgt)
    tidx = P.Index(ctx, tgt)
    gate = 0.05
    mode = {"on": P.TRACK_ON, "off": P.TRACK_OFF, "auto": P.TRACK_AUTO}[track]
    runs = []
    for chain in ([], [(P.REJ_DISTANCE, 100 * gate, 0)]):
        s = P.Icp(ctx, max_iterations=40, transformation_epsilon=1e-10, max_correspondence_distance=gate,
                  scalar_is_double=int(dbl), track_mode=mode)
        s.set_rejectors(chain)
        s.set_target(tidx)
        s.set_source(src)
        runs.append([s.iterate(1) for _ in range(3)] + [s.iterate()])
    keys = ("iterations", "state", "converged", "n_correspondences", "total_correspondences", "total_skipped_walks")
    for k, (a, b) in enumerate(zip(*runs)):
        assert [a[x] for x in keys] == [b[x] for x in keys], (k, a, b)
        assert np.array_equal(a["final"], b["final"]) and np.array_equal(a["last"], b["last"]), k
    assert runs[0][-1]["state"] != 0 and runs[0][-1]["iterations"] > 3


def test_symmetric_point_to_plane(gpu, orc):
    """TransformationEstimationSymmetricPointToPlaneLLS (SURVEY.md §8f #2): the reference's paraboloid test
    (test_registration_api.cpp:663-713), oracle parity, and ICP with setUseSymmetricObjective(true)."""
    P, ctx = gpu
    xs = np.arange(-5.0, 5.0 + 1e-6, 0.5, dtype=np.float32)
    X, Y = np.meshgrid(xs, xs, indexing="ij")
    x, y = X.ravel(), Y.ravel()
    z = np.float32(0.1) * x ** 2 + np.float32(0.2) * x * y - np.float32(0.3) * y + np.float32(1.0)
    nrm = np.stack([-0.2 * x - 0.2, 0.6 * y - 0.2, np.ones_like(x)], 1).astype(np.float32)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    src = np.zeros((x.size, 12), np.float32)
    src[:, 0], src[:, 1], src[:, 2], src[:, 3] = x, y, z, 1
    src[:, 4:7] = nrm
    G = np.array([[0.9938, 0.0988, 0.0517, 0.1], [-0.0997, 0.9949, 0.0149, -0.2], [-0.05, -0.02, 0.9986, 0.3],
                  [0, 0, 0, 1]], np.float64)
    tgt = orc.transform(src, G, mode=1, normal_off=4)
    for enforce in (True, False):
        T = ctx.estimate_symmetric_lls(src, tgt, enforce_same_direction=enforce, scalar_is_double=True)
        assert np.all(np.abs(T - G) < 1e-2)
        To, _ = orc.estimate_symmetric_lls(src, tgt, enforce_same_direction=enforce, scalar_is_double=True)
        assert np.linalg.norm(T - To) < 1e-9, np.linalg.norm(T - To)
        Tf = ctx.estimate_symmetric_lls(src, tgt, enforce_same_direction=enforce)
        Tof, _ = orc.estimate_symmetric_lls(src, tgt, enforce_same_direction=enforce)
        assert np.linalg.norm(Tf - Tof) < 2e-5          # the oracle (like PCL) accumulates in float here
    # ICP on a noisy surface, both clouds with normals
    rng = np.random.default_rng(41)
    n = 30000

    def surf(m):
        xy = rng.random((m, 2)) * 4
        zz = 0.3 * np.sin(xy[:, 0]) * np.cos(xy[:, 1])
        nn = np.stack([-0.3 * np.cos(xy[:, 0]) * np.cos(xy[:, 1]), 0.3 * np.sin(xy[:, 0]) * np.sin(xy[:, 1]), np.ones(m)], 1)
        nn /= np.linalg.norm(nn, axis=1, keepdims=True)
        c = np.zeros((m, 12), np.float32)
        c[:, :3] = np.column_stack([xy, zz + rng.normal(0, 0.001, m)])
        c[:, 3] = 1
        c[:, 4:7] = nn
        return c

    T0 = np.eye(4)
    a = np.deg2rad(1.5)
    T0[:3, :3] = [[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]
    T0[:3, 3] = [0.01, -0.005, 0.004]
    tgt_c = surf(n)
    src_c = orc.transform(surf(n), T0, mode=1, normal_off=4)
    kw = dict(max_iterations=30, max_correspondence_distance=0.05, transformation_epsilon=1e-10)
    r = P.icp_align(ctx, src_c, P.Index(ctx, tgt_c), src_normals=P.Field(src_c, 4), tgt_normals=P.Field(tgt_c, 4),
                    estimator=P.EST_SYMMETRIC_POINT_TO_PLANE_LLS, with_normals_transform=1, **kw)
    o64 = orc.icp_align(src_c, tgt_c, estimator=2, with_normals_transform=True, source_has_normals=True,
                        scalar_is_double=True, nthreads=8, **kw)
    assert r["converged"] and o64["converged"]
    assert np.linalg.norm(r["final"] - o64["final"]) < 5e-5, np.linalg.norm(r["final"] - o64["final"])
    assert np.linalg.norm(r["final"] @ T0 - np.eye(4)) < 5e-3     # undoes the applied motion
    with pytest.raises(P.Pclb200Error):                            # symmetric objective without source normals
        P.icp_align(ctx, src_c, P.Index(ctx, tgt_c), tgt_normals=P.Field(tgt_c, 4),
                    estimator=P.EST_SYMMETRIC_POINT_TO_PLANE_LLS, **kw)


def test_knn_stats_and_outlier_filters(gpu, golden, orc):
    """pclb200_knn_stats (what StatisticalOutlierRemoval / RadiusOutlierRemoval derive from nearestKSearch): bit-exact
    against the oracle for register (k <= 32) and list (k > 32) kernels, with NaN points and subsets; and the two
    filters' golden counts on bun0 (test/filters/test_filters.cpp:1494-1515, 1587-1613)."""
    P, ctx = gpu
    rng = np.random.default_rng(51)
    pts = rng.random((20000, 3), dtype=np.float32)
    pts[::53, 2] = np.nan
    cloud = orc.to_xyz1(pts)
    gi, oi = P.Index(ctx, cloud), orc.Index(cloud)
    for k in (2, 9, 15, 32, 51):
        gm, gk = gi.knn_stats(cloud, k)
        om, ok = oi.knn_stats(cloud, k, nthreads=4)
        assert np.array_equal(gm, om), k
        assert np.array_equal(gk, ok), k
    sub = np.arange(0, 20000, 7, dtype=np.int32)
    gm, gk = gi.knn_stats(cloud, 6, indices=sub)
    om, ok = oi.knn_stats(cloud, 6, nthreads=4)
    assert np.array_equal(gm, om[sub]) and np.array_equal(gk, ok[sub])
    bun = P.xyz1(golden["bun0"])
    bi = P.Index(ctx, bun)
    _, kth = bi.knn_stats(bun, 15)
    assert int((kth <= 0.02 * 0.02).sum()) == 307                       # RadiusOutlierRemoval(0.02, 14): dense rule
    mean, _ = bi.knn_stats(bun, 51)
    s = mean.astype(np.float64)
    mu = s.sum() / 397
    var = ((mean * mean).astype(np.float64).sum() - s.sum() ** 2 / 397) / 396
    assert int((mean <= mu + 1.0 * np.sqrt(var)).sum()) == 352          # StatisticalOutlierRemoval(50, 1.0)


def test_voxelgrid_point_normal_all_fields(gpu, orc):
    """VoxelGrid<PointNormal> with the reference's default downsample_all_data_ = true averages the normal (normalised
    4-vector sum) and the curvature per voxel as well (voxel_grid.hpp:796-806, accumulators.hpp:86-133); xyz stays
    bit-exact, the normalised sums agree to rounding of the square root / division."""
    P, ctx = gpu
    rng = np.random.default_rng(5)
    n = 60000
    rec = np.zeros((n, 12), dtype=np.float32)
    rec[:, :3] = rng.random((n, 3), dtype=np.float32) * np.float32(2.0)
    rec[:, 3] = 1.0
    nrm = rng.normal(size=(n, 3)).astype(np.float32)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    rec[:, 4:7] = nrm
    rec[:, 8] = rng.random(n, dtype=np.float32)
    rec[::97, 1] = np.nan
    idx = rng.permutation(n)[: n // 2].astype(np.int32)
    for leaf, mp, ind in (([0.05] * 3, 0, None), ([0.1, 0.2, 0.05], 3, idx)):
        gx, gn = ctx.voxelgrid_normals(rec, leaf, min_points_per_voxel=mp, indices=ind, is_dense=False)
        ox, on = orc.voxelgrid_normals(rec, leaf, min_points_per_voxel=mp, indices=ind, is_dense=False)
        assert gx.shape == ox.shape and np.array_equal(gx, ox)
        assert np.allclose(gn, on, rtol=0, atol=2e-7), float(np.abs(gn - on).max())
        assert np.allclose(np.linalg.norm(gn[:, :4], axis=1), 1.0, atol=1e-5)


def test_voxelgrid_tiles_equal_whole(gpu, orc):
    """Spatial tiles cut along voxel boundaries and filtered on the WHOLE cloud's grid (pclb200_voxelgrid_tile) give,
    concatenated, exactly the centroids of one VoxelGrid over the whole cloud (the multi-GPU front-end of config 5)."""
    P, ctx = gpu
    rng = np.random.default_rng(17)
    n = 200000
    pts = P.xyz1((rng.random((n, 3), dtype=np.float32) * np.array([40, 10, 3], np.float32)) - np.float32(7))
    leaf = np.float32(0.25)
    whole = ctx.voxelgrid(pts, leaf)
    lo, hi = pts[:, :3].min(0), pts[:, :3].max(0)
    inv = np.float32(1.0) / leaf
    i = (np.floor(pts[:, 0] * inv) - np.floor(lo[0] * inv)).astype(np.int64)   # voxel column of every point
    cuts = [0, int(i.max()) // 3, 2 * int(i.max()) // 3, int(i.max()) + 1]
    tiles = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        sel = pts[(i >= a) & (i < b)]
        tiles.append(ctx.voxelgrid_tile(sel, leaf, np.concatenate([lo, hi])))
    got = np.concatenate(tiles)
    assert got.shape == whole.shape

    def canon(a):
        return a[np.lexsort((a[:, 2], a[:, 1], a[:, 0]))]
    assert np.array_equal(canon(got), canon(whole))


def test_estimate_svd_correlation_path(gpu, orc):
    """TransformationEstimationSVD(use_umeyama = false): getTransformationFromCorrelation
    (transformation_estimation_svd.hpp:156-225) — stand-alone and inside the ICP loop (svd_no_umeyama)."""
    P, ctx = gpu
    rng = np.random.default_rng(3)
    n = 20000
    src = rng.random((n, 3), dtype=np.float32) * 3
    a = np.deg2rad(7.0)
    R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    tgt = (src.astype(np.float64) @ R.T + [0.3, -0.2, 0.1] + rng.normal(0, 1e-3, (n, 3))).astype(np.float32)
    S, T = P.xyz1(src), P.xyz1(tgt)
    corr = np.zeros(n // 2, dtype=P.CORR_DTYPE)
    corr["index_query"] = rng.permutation(n)[: n // 2]
    corr["index_match"] = corr["index_query"]
    for c in (None, corr):
        g = ctx.estimate_svd(S, T, c, scalar_is_double=True, use_umeyama=False)
        o = orc.estimate_svd(S, T, c, scalar_is_double=True, use_umeyama=False)
        u = ctx.estimate_svd(S, T, c, scalar_is_double=True, use_umeyama=True)
        assert np.linalg.norm(g - o) < 1e-9 and np.linalg.norm(g - u) < 1e-9   # same least-squares solution
        gf = ctx.estimate_svd(S, T, c, use_umeyama=False)
        of = orc.estimate_svd(S, T, c, use_umeyama=False)
        assert np.linalg.norm(gf - of) < 2e-5     # float Scalar: the reference sums in float, the device in fp64
    # inside the loop
    kw = dict(max_iterations=25, max_correspondence_distance=0.5, transformation_epsilon=1e-10)
    idx = P.Index(ctx, T)
    r0 = P.icp_align(ctx, S, idx, **kw)
    r1 = P.icp_align(ctx, S, idx, svd_no_umeyama=1, **kw)
    assert r0["converged"] and r1["converged"] and np.linalg.norm(r0["final"] - r1["final"]) < 1e-5
