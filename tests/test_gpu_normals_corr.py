"""Parity of the normal-based correspondence estimators, the surface-normal rejector and radius-search normals
(SURVEY.md §8f #1/#2, §8 a16) through the C-ABI against the CPU oracle and the reference's own tests.
Index lists are bit-exact; transforms within 1e-5 Frobenius.  Needs an H100: run with -m gpu."""
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


def _point_normal(xyz, normals=None):
    """(n,12) pcl::PointNormal rows."""
    out = np.zeros((xyz.shape[0], 12), np.float32)
    out[:, :3] = xyz[:, :3]
    out[:, 3] = 1
    if normals is not None:
        out[:, 4:4 + normals.shape[1]] = normals
    return out


def _unit(v):
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def _planes():
    # test/registration/test_correspondence_estimation.cpp:95-137: two parallel planes differing only in y
    ii, jj = np.meshgrid(np.arange(50), np.arange(25), indexing="ij")
    x = ii.ravel().astype(np.float32) * np.float32(0.2)
    z = jj.ravel().astype(np.float32) * np.float32(0.2)
    c1 = _point_normal(np.stack([x, np.zeros_like(x), z], 1))
    c2 = _point_normal(np.stack([x, np.full_like(x, 2), z], 1))
    return c1, c2


def test_normal_shooting_reference_planes(gpu, orc):
    P, ctx = gpu
    c1, c2 = _planes()
    nrm, dense = P.Index(ctx, c1).normals_knn(c1, 5)
    assert dense
    c1[:, 4:8] = nrm
    c2[:, 4:8] = nrm
    it = P.Index(ctx, c2)
    ot = orc.Index(c2)
    for kind in (P.CORR_NORMAL_SHOOTING, P.CORR_BACK_PROJECTION):
        g = it.correspondences_normals(kind, c1, P.Field(c1, 4), P.Field(c2, 4), k=10)
        assert len(g) == 1250 and np.array_equal(g["index_query"], g["index_match"])  # "1 <-> 1, 2 <-> 2, ..."
        o = ot.correspondences_normals(kind, c1, c2, k=10)
        assert np.array_equal(g, o)


@pytest.mark.parametrize("kind", [1, 2])
@pytest.mark.parametrize("k", [1, 3, 10, 16, 40])
def test_correspondences_normals_bit_exact(gpu, orc, kind, k):
    P, ctx = gpu
    rng = np.random.default_rng(100 + k)
    t = rng.normal(size=(20000, 3)).astype(np.float32)
    t[:, 2] = np.float32(0.3) * np.sin(t[:, 0]) * np.cos(t[:, 1])
    tgt = _point_normal(t, _unit(rng.normal(size=(20000, 3))))
    s = t[rng.permutation(20000)[:6000]] + rng.normal(scale=0.01, size=(6000, 3)).astype(np.float32)
    src = _point_normal(s, _unit(rng.normal(size=(6000, 3))))
    src[::97, 0] = np.nan          # non-finite source points: no correspondence
    src[5::211, 4:7] = np.nan      # NaN normals: every score is NaN
    tgt[7::301, 1] = np.inf        # dropped from the index, original ids kept
    it, ot = P.Index(ctx, tgt), orc.Index(tgt)
    sub = rng.permutation(6000)[:2500].astype(np.int32)
    for md in (np.sqrt(np.finfo(np.float64).max), 1e-3, 4e-5):
        for ind in (None, sub):
            g = it.correspondences_normals(kind, src, P.Field(src, 4), P.Field(tgt, 4), k=k, max_distance=md, indices=ind)
            o = ot.correspondences_normals(kind, src, tgt, k=k, max_distance=md, indices=ind, nthreads=8)
            assert len(g) == len(o), (kind, k, md, len(g), len(o))
            assert np.array_equal(g, o), (kind, k, md)
    small = _point_normal(t[:7], _unit(rng.normal(size=(7, 3))))  # k clamps to the 7 indexed points
    g = P.Index(ctx, small).correspondences_normals(kind, src, P.Field(src, 4), P.Field(small, 4), k=k)
    o = orc.Index(small).correspondences_normals(kind, src, small, k=k)
    assert np.array_equal(g, o)


def test_correspondences_normals_argument_errors(gpu):
    P, ctx = gpu
    c1, c2 = _planes()
    it = P.Index(ctx, c2)
    with pytest.raises(P.Pclb200Error) as e:
        it.correspondences_normals(P.CORR_NORMAL_SHOOTING, c1, None)
    assert e.value.code == P.ERR_INVALID
    with pytest.raises(P.Pclb200Error) as e:
        it.correspondences_normals(P.CORR_BACK_PROJECTION, c1, P.Field(c1, 4), None)
    assert e.value.code == P.ERR_INVALID
    with pytest.raises(P.Pclb200Error) as e:
        it.correspondences_normals(7, c1, P.Field(c1, 4))
    assert e.value.code == P.ERR_INVALID
    assert len(it.correspondences_normals(P.CORR_NORMAL_SHOOTING, c1, P.Field(c1, 4), k=0)) == 0


def test_reject_surface_normal(gpu, golden, orc):
    # test/registration/test_registration_api.cpp:266-317
    P, ctx = gpu
    b0, b4 = _point_normal(golden["bun0"]), _point_normal(golden["bun4"])
    i0, i4 = P.Index(ctx, b0), P.Index(ctx, b4)
    b0[:, 4:8] = i0.normals_knn(b0, 10)[0]
    b4[:, 4:8] = i4.normals_knn(b4, 10)[0]
    corr = i4.correspondences(b0)
    assert len(corr) == 397
    for thr in (0.5, 0.0, 0.95, -2.0, 2.0):
        g = ctx.reject_surface_normal(corr, P.Field(b0, 4), P.Field(b4, 4), thr)
        o = orc.reject_surface_normal(corr, b0[:, 4:], b4[:, 4:], thr)
        assert np.array_equal(g, o), thr
    assert len(ctx.reject_surface_normal(corr, P.Field(b0, 4), P.Field(b4, 4), -2.0)) == 397
    rng = np.random.default_rng(5)
    n = 200000
    sn, tn = _unit(rng.normal(size=(n, 3))), _unit(rng.normal(size=(n, 3)))
    sn[::31] = np.nan
    big = np.zeros(n, dtype=P.CORR_DTYPE)
    big["index_query"] = rng.integers(0, n, n)
    big["index_match"] = rng.integers(0, n, n)
    big["distance"] = rng.random(n, dtype=np.float32)
    g = ctx.reject_surface_normal(big, sn, tn, 0.25)
    assert np.array_equal(g, orc.reject_surface_normal(big, sn, tn, 0.25))
    assert len(ctx.reject_surface_normal(big[:0], sn, tn, 0.25)) == 0


def _reference(cloud, queries, vp, **kw):
    """The per-query extended-precision reference of tests/test_normals_reference.py."""
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import test_normals_reference
    return test_normals_reference.Reference(cloud, queries, vp, **kw)


def test_normals_radius_vs_oracle(gpu, golden, orc):
    P, ctx = gpu
    b0 = P.xyz1(golden["bun0"])
    g, gd = P.Index(ctx, b0).normals_radius(b0, 0.02)
    o, od = orc.Index(b0).normals_radius(b0, 0.02)
    assert gd == od
    assert np.array_equal(np.isnan(g[:, 0]), np.isnan(o[:, 0]))
    _reference(b0, b0, (0, 0, 0), radius=0.02).check(g, "bun0")
    rng = np.random.default_rng(15)
    pts = rng.random((30000, 3), dtype=np.float32)
    pts[:, 2] = np.float32(0.1) * np.sin(np.float32(6) * pts[:, 0])
    cloud = orc.to_xyz1(pts)
    cloud[::501, 0] = np.nan
    sub = rng.permutation(30000)[:7000].astype(np.int32)
    for r, ind in ((0.02, None), (0.05, sub), (0.004, None)):  # the small radius leaves many points with < 3 neighbours
        g, gd = P.Index(ctx, cloud).normals_radius(cloud, r, viewpoint=(0.5, 0.5, 5), indices=ind, is_dense=False)
        o, od = orc.Index(cloud).normals_radius(cloud, r, viewpoint=(0.5, 0.5, 5), indices=ind, is_dense=False, nthreads=8)
        assert gd == od and g.shape == o.shape
        assert np.array_equal(np.isnan(g[:, 0]), np.isnan(o[:, 0])), r
        ok = ~np.isnan(o[:, 0])
        assert ok.sum() > 100, r
        # every normal and curvature, also with 3-5 neighbours, against the reference of its own neighbourhood
        _reference(cloud, cloud if ind is None else cloud[ind], (0.5, 0.5, 5), radius=r).check(g, f"r={r}")
    with pytest.raises(P.Pclb200Error):
        P.Index(ctx, cloud).normals_radius(cloud, 0.0)


def _bunnies_with_normals(P, ctx, golden):
    b0, b4 = _point_normal(golden["bun0"]), _point_normal(golden["bun4"])
    b0[:, 4:8] = P.Index(ctx, b0).normals_knn(b0, 10)[0]
    b4[:, 4:8] = P.Index(ctx, b4).normals_knn(b4, 10)[0]
    return b0, b4


@pytest.mark.parametrize("double", [False, True])
@pytest.mark.parametrize("kind", [1, 2])
def test_icp_normal_based_estimators_in_loop(gpu, golden, orc, kind, double):
    """test/registration/test_registration.cpp:511-560: point-to-plane ICP whose correspondences come from
    CorrespondenceEstimationNormalShooting, filtered by CorrespondenceRejectorSurfaceNormal(threshold 0)."""
    P, ctx = gpu
    b0, b4 = _bunnies_with_normals(P, ctx, golden)
    it = P.Index(ctx, b4)
    rej = [(P.REJ_SURFACE_NORMAL, 0.0, 0)]
    common = dict(max_iterations=50, transformation_epsilon=1e-8)
    s = P.Icp(ctx, estimator=P.EST_POINT_TO_PLANE_LLS, scalar_is_double=int(double), with_normals_transform=1,
              correspondence_kind=kind, correspondence_k=10, **common)
    s.set_rejectors(rej)
    s.set_target(it, P.Field(b4, 4))
    s.set_source(b0, normals=P.Field(b0, 4))
    st = s.iterate()
    o = orc.icp_align_rejectors(b0, b4, rej, estimator=1, source_has_normals=True, scalar_is_double=double,
                                correspondence_kind=kind, correspondence_k=10, **common)
    assert st["converged"] and o["converged"]
    assert abs(st["iterations"] - o["iterations"]) <= 1
    assert np.linalg.norm(st["final"] - o["final"]) < (1e-5 if double else 5e-5)
    if st["iterations"] == o["iterations"]:
        assert st["n_correspondences"] == o["n_correspondences"]
    # the reference's acceptance criterion: the registration converges to a low fitness score
    assert it.fitness_score(b0, st["final"], scalar_is_double=double) < 0.005
    # first iteration's correspondences == the stand-alone estimator followed by the stand-alone rejector
    s.set_source(b0, normals=P.Field(b0, 4))
    s.iterate(1)
    c1 = s.get_correspondences()
    ref = it.correspondences_normals(kind, b0, P.Field(b0, 4), P.Field(b4, 4), k=10)
    ref = ctx.reject_surface_normal(ref, P.Field(b0, 4), P.Field(b4, 4), 0.0)
    assert np.array_equal(c1, ref)
    oref = orc.Index(b4).correspondences_normals(kind, b0, b4, k=10)
    assert np.array_equal(c1, orc.reject_surface_normal(oref, b0[:, 4:], b4[:, 4:], 0.0))


def test_icp_normal_based_argument_errors(gpu, golden):
    P, ctx = gpu
    b0, b4 = _bunnies_with_normals(P, ctx, golden)
    it = P.Index(ctx, b4)
    s = P.Icp(ctx, correspondence_kind=P.CORR_NORMAL_SHOOTING)
    s.set_target(it)
    with pytest.raises(P.Pclb200Error) as e:  # no source normals
        s.set_source(b0)
    assert e.value.code == P.ERR_INVALID
    s = P.Icp(ctx, correspondence_kind=P.CORR_BACK_PROJECTION)
    s.set_target(it)  # no target normals
    s.set_source(b0, normals=P.Field(b0, 4))
    with pytest.raises(P.Pclb200Error) as e:
        s.iterate()
    assert e.value.code == P.ERR_INVALID
    s = P.Icp(ctx, correspondence_kind=P.CORR_NORMAL_SHOOTING, use_reciprocal=1)
    s.set_target(it, P.Field(b4, 4))
    s.set_source(b0, normals=P.Field(b0, 4))
    with pytest.raises(P.Pclb200Error) as e:
        s.iterate()
    assert e.value.code == P.ERR_INVALID
    s = P.Icp(ctx)
    s.set_rejectors([(P.REJ_SURFACE_NORMAL, 0.0, 0)])
    s.set_target(it)
    with pytest.raises(P.Pclb200Error) as e:  # the rejector needs normals
        s.set_source(b0)
    assert e.value.code == P.ERR_INVALID


def test_icp_surface_normal_rejector_with_nearest_estimator(gpu, golden, orc):
    P, ctx = gpu
    b0, b4 = _bunnies_with_normals(P, ctx, golden)
    it = P.Index(ctx, b4)
    rej = [(P.REJ_SURFACE_NORMAL, 0.5, 0), (P.REJ_DISTANCE, 0.05, 0)]
    common = dict(max_iterations=30, transformation_epsilon=1e-8)
    s = P.Icp(ctx, estimator=P.EST_SVD, with_normals_transform=1, **common)
    s.set_rejectors(rej)
    s.set_target(it, P.Field(b4, 4))
    s.set_source(b0, normals=P.Field(b0, 4))
    st = s.iterate()
    o = orc.icp_align_rejectors(b0, b4, rej, estimator=0, source_has_normals=True, **common)
    assert abs(st["iterations"] - o["iterations"]) <= 1
    assert np.linalg.norm(st["final"] - o["final"]) < 5e-5
