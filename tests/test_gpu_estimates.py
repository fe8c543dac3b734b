"""Every transform estimate of the ICP kernels against an extended-precision reference of its own pairs.

The trajectory tests compare whole aligns with the oracle at 1e-5; a pair lost, counted twice or read from the wrong lane
moves T by ~1e-8 and passes them.  Here each estimate — k_accum_dmma (SVD, point-to-plane), k_accum (symmetric objective),
k_accum_pairs (the stand-alone estimators) and k_solve — is compared with a reference computed from the very pairs the
device used (get_correspondences of that iteration, or the caller's list): centroids and products summed with math.fsum
after demeaning in fp64, solved in fp64.  The bar is 1e-12 * max(1, kappa) in double and the float rounding of the
reference in float, and every scene first checks that removing its most influential pair moves the reference by more
than 100 times that bar, so a lost pair cannot pass.  Scenes: a bulk surface, small patches 500 m from the target map's
centre (the SVD sums must be taken about an origin near the pairs), degenerate point sets, and the tail shapes of every
grid (n around multiples of 32, 256 and the persistent grids).  The helpers are checked against the oracle's double
estimators without a GPU; the rest needs an H100: run with -m gpu."""
import math

import numpy as np
import pytest

TOL = 1e-12


# ---- references ---------------------------------------------------------------------------------------------------------
def _fsum_cols(M):
    return np.array([math.fsum(M[:, j]) for j in range(M.shape[1])])


def _centroids(p, q):
    n = p.shape[0]
    return _fsum_cols(p) / n, _fsum_cols(q) / n


def ref_svd(p, q):
    """Least-squares rigid motion p -> q (Umeyama without scale; the correlation formula gives the same R): centroids and
    the demeaned correlation H = sum (p - cp)(q - cq)^T by fsum, fp64 SVD, det(U) det(V) sign fix, t = cq - R cp.
    Returns (T, kappa = s0 / (s1 + s2), scale of the translation = 1 + |cq|)."""
    p, q = np.asarray(p, np.float64), np.asarray(q, np.float64)
    cp, cq = _centroids(p, q)
    P, Q = p - cp, q - cq
    H = np.array([[math.fsum(P[:, i] * Q[:, j]) for j in range(3)] for i in range(3)])
    U, s, Vt = np.linalg.svd(H)
    V = Vt.T
    if np.linalg.det(U) * np.linalg.det(V) < 0:
        V[:, 2] = -V[:, 2]
    R = V @ U.T
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, cq - R @ cp
    kappa = s[0] / (s[1] + s[2]) if s[1] + s[2] > 0 else np.inf
    return T, kappa, 1.0 + np.linalg.norm(cq)


def _euler_T(x):
    """k_solve's T of the point-to-plane solution x = (alpha, beta, gamma, tx, ty, tz)"""
    al, be, ga = x[:3]
    T = np.eye(4)
    T[0, 0] = math.cos(ga) * math.cos(be)
    T[0, 1] = -math.sin(ga) * math.cos(al) + math.cos(ga) * math.sin(be) * math.sin(al)
    T[0, 2] = math.sin(ga) * math.sin(al) + math.cos(ga) * math.sin(be) * math.cos(al)
    T[1, 0] = math.sin(ga) * math.cos(be)
    T[1, 1] = math.cos(ga) * math.cos(al) + math.sin(ga) * math.sin(be) * math.sin(al)
    T[1, 2] = -math.cos(ga) * math.sin(al) + math.sin(ga) * math.sin(be) * math.cos(al)
    T[2, 0] = -math.sin(be)
    T[2, 1] = math.cos(be) * math.sin(al)
    T[2, 2] = math.cos(be) * math.cos(al)
    T[:3, 3] = x[3:]
    return T


def _sym_T(x):
    """k_solve's T of the symmetric objective: [R R | R t], R = Rz(gamma) Ry(beta) Rx(alpha)"""
    al, be, ga = x[:3]
    ca, sa, cb, sb, cg, sg = math.cos(al), math.sin(al), math.cos(be), math.sin(be), math.cos(ga), math.sin(ga)
    Rm = np.array([[cg * cb, cg * sb * sa - sg * ca, cg * sb * ca + sg * sa],
                   [sg * cb, sg * sb * sa + cg * ca, sg * sb * ca - cg * sa],
                   [-sb, cb * sa, cb * ca]])
    T = np.eye(4)
    T[:3, :3] = Rm @ Rm
    T[:3, 3] = Rm @ x[3:]
    return T


def _lls_solve(V, b, nn_float=None):
    """A^T A and A^T b by fsum over the rows of V (6 columns) and b; the normal-normal block from nn_float (float products)
    when given.  Returns (x, kappa(A^T A))."""
    M = np.zeros((6, 6))
    for r in range(6):
        for c in range(r, 6):
            col = nn_float[r, c] if (nn_float is not None and r >= 3) else V[:, r] * V[:, c]
            M[r, c] = M[c, r] = math.fsum(col)
    rhs = np.array([math.fsum(V[:, r] * b) for r in range(6)])
    return np.linalg.solve(M, rhs), np.linalg.cond(M)


def _p2p_rows(p, q, nq):
    """point_to_plane_lls.hpp:202-204, 235 in float32 (numpy rounds every float32 operation: -fmad=false); rows with a
    non-finite normal dropped"""
    ok = np.isfinite(nq).all(1)
    f = np.float32
    p, q, nq = p[ok].astype(f), q[ok].astype(f), nq[ok].astype(f)
    sx, sy, sz = p.T
    dx, dy, dz = q.T
    nx, ny, nz = nq.T
    A = nz * sy - ny * sz
    B = nx * sz - nz * sx
    C = ny * sx - nx * sy
    D = nx * dx + ny * dy + nz * dz - nx * sx - ny * sy - nz * sz
    V = np.stack([A, B, C, nx, ny, nz], 1).astype(np.float64)
    nn = {}
    for r in range(3, 6):
        for c in range(r, 6):
            nn[r, c] = (nq[:, r - 3] * nq[:, c - 3]).astype(np.float64)
    return V, D.astype(np.float64), nn


def ref_p2p(p, q, nq):
    V, D, nn = _p2p_rows(p, q, nq)
    x, kappa = _lls_solve(V, D, nn)
    return _euler_T(x), kappa, 1.0


def _sym_rows(p, q, np_, nq, enforce_same_dir):
    """symmetric_point_to_plane_lls.hpp:166-193 with add_pair_terms' fp64 expressions"""
    d = np.float64
    p, q, n1, n2 = (np.asarray(a, d) for a in (p, q, np_, nq))
    d12 = n1[:, 0] * n2[:, 0] + n1[:, 1] * n2[:, 1] + n1[:, 2] * n2[:, 2]
    sg = np.where((not enforce_same_dir) | (d12 >= 0.0), 1.0, -1.0)
    n = n1 + sg[:, None] * n2
    with np.errstate(invalid="ignore"):
        ok = np.isfinite(n).all(1)
    p, q, n = p[ok], q[ok], n[ok]
    keep = np.nonzero(ok)[0]
    s = p + q
    nx, ny, nz = n.T
    sx, sy, sz = s.T
    V = np.stack([sy * nz - sz * ny, sz * nx - sx * nz, sx * ny - sy * nx, nx, ny, nz], 1)
    b = (q[:, 0] - p[:, 0]) * nx + (q[:, 1] - p[:, 1]) * ny + (q[:, 2] - p[:, 2]) * nz
    return V, b, keep


def ref_sym(p, q, np_, nq, enforce_same_dir=True):
    V, b, _ = _sym_rows(p, q, np_, nq, enforce_same_dir)
    x, kappa = _lls_solve(V, b)
    return _sym_T(x), kappa, 1.0


def reference(est, p, q, nq=None, np_=None):
    if est in ("svd", "svd_corr"):
        return ref_svd(p, q)
    if est == "p2p":
        return ref_p2p(p, q, nq)
    return ref_sym(p, q, np_, nq)


def _leverage_drop(est, p, q, nq, np_):
    """index of the pair whose removal moves the estimate most (largest leverage)"""
    if est in ("svd", "svd_corr"):
        c = np.mean(p, 0)
        return int(np.argmax(np.linalg.norm(np.asarray(p, np.float64) - c, axis=1)))
    if est == "p2p":
        ok = np.nonzero(np.isfinite(nq).all(1))[0]
        V, D, _ = _p2p_rows(p, q, nq)
    else:
        V, D, ok = _sym_rows(p, q, np_, nq, True)
    Minv = np.linalg.inv(V.T @ V)
    x = Minv @ (V.T @ D)
    g = V @ Minv                              # row i: the direction one pair moves the solution
    h = np.einsum("ij,ij->i", g, V)           # its leverage
    infl = np.linalg.norm(g, axis=1) * np.abs(D - V @ x) / (1.0 - np.minimum(h, 0.999))
    return int(ok[np.argmax(infl)])


def _dist(Ta, Tb, tscale):
    d = np.asarray(Ta, np.float64) - np.asarray(Tb, np.float64)
    d[:3, 3] /= tscale
    return float(np.linalg.norm(d))


def check_estimate(est, T_dev, dbl, p, q, nq=None, np_=None, sharp=True):
    """T_dev against the reference of the pairs (p_i, q_i); returns |T_dev - T_ref| / tol.  With sharp, first asserts
    that dropping the most influential pair moves the reference by more than 100 tol."""
    T_ref, kappa, tscale = reference(est, p, q, nq, np_)
    tol = TOL * max(1.0, kappa)
    if sharp:
        k = _leverage_drop(est, p, q, nq, np_)
        keep = np.ones(p.shape[0], bool)
        keep[k] = False
        sub = [None if a is None else a[keep] for a in (p, q, nq, np_)]
        T_drop = reference(est, *sub)[0]
        assert _dist(T_drop, T_ref, tscale) > 100 * tol, ("the bar does not see one lost pair", _dist(T_drop, T_ref, tscale), tol)
    if dbl:
        err = _dist(T_dev, T_ref, tscale)
        assert err <= tol, (est, err, tol, kappa, T_dev, T_ref)
        return err / tol
    # Scalar = float: k_solve rounds its fp64 solution once; it may land on the other side of a rounding boundary only
    # where the reference lies within the double bar of one
    f = T_ref.astype(np.float32)
    dev = np.asarray(T_dev).astype(np.float32)
    assert np.array_equal(dev.astype(np.float64), np.asarray(T_dev)), "a float estimate must be float-representable"
    bad = dev != f
    span = tol * np.where(np.arange(4)[None, :] == 3, tscale, 1.0) * np.ones((4, 4))
    lo, hi = (T_ref - span).astype(np.float32), (T_ref + span).astype(np.float32)
    ok = ~bad | (dev == lo) | (dev == hi)
    assert ok.all(), (est, T_dev[bad], T_ref[bad])
    return float(bad.sum())  # entries on the other side of a rounding boundary


# ---- scenes ---------------------------------------------------------------------------------------------------------------
def _rot(axis, deg):
    ax = np.asarray(axis, np.float64)
    ax = ax / np.linalg.norm(ax)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    a = np.deg2rad(deg)
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


def surface(rng, n, scale=1.0, center=(0.0, 0.0, 0.0)):
    """PointNormal rows (n, 8) on a bumpy sheet of side `scale` (bumps 10 % of it) with analytic normals"""
    xy = rng.random((n, 2))
    z = 0.1 * np.sin(3 * xy[:, 0]) + 0.1 * np.cos(4 * xy[:, 1])
    nrm = np.stack([-0.3 * np.cos(3 * xy[:, 0]), 0.4 * np.sin(4 * xy[:, 1]), np.ones(n)], 1)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    out = np.zeros((n, 8), np.float32)
    out[:, 0:3] = np.c_[xy, z] * scale + np.asarray(center)
    out[:, 3] = 1.0
    out[:, 4:7] = nrm
    return out


def moved(rng, tgt, deg, shift, noise, about=None):
    """source PointNormal rows: tgt rotated by deg about `about` (default its centroid), shifted, with noise"""
    c = np.mean(tgt[:, :3].astype(np.float64), 0) if about is None else np.asarray(about, np.float64)
    R = _rot((0.2, -0.3, 1.0), deg)
    src = tgt.copy()
    src[:, 0:3] = (tgt[:, :3].astype(np.float64) - c) @ R.T + c + np.asarray(shift) + rng.normal(0, noise, (tgt.shape[0], 3))
    src[:, 4:7] = tgt[:, 4:7].astype(np.float64) @ R.T
    return src


def bulk(n_src=60000, seed=3, deg=5.0, shift=(0.01, -0.02, 0.015)):
    rng = np.random.default_rng(seed)
    tgt = surface(rng, max(n_src, 60000))
    src = moved(rng, surface(rng, n_src), deg, shift, 0.001)
    return src, tgt


def far_patch(size, seed=5):
    """a sparse +-500 m map holding a dense object patch of side `size` near (400, -300, 5); the source is the patch,
    re-sampled, rotated 0.5 deg about its centre and shifted 1 mm"""
    rng = np.random.default_rng(seed)
    m = np.zeros((20000, 8), np.float32)
    m[:, 0:2] = rng.random((20000, 2)) * 1000 - 500
    m[:, 2] = rng.random(20000) * 20 - 10
    m[:, 3], m[:, 6] = 1.0, 1.0
    patch = surface(rng, 40000, size, (400.0, -300.0, 5.0))
    tgt = np.concatenate([m, patch])
    src = moved(rng, surface(rng, 20000, size, (400.0, -300.0, 5.0)), 0.5, (0.001, -0.0006, 0.0008), 0.0)
    return src, tgt


# ---- CPU: the references against the oracle's double estimators ----------------------------------------------------------
def test_references_match_the_oracle_double_estimators():
    import oracle as orc
    rng = np.random.default_rng(11)
    tgt = surface(rng, 3000)
    src = moved(rng, tgt, 3.0, (0.02, -0.01, 0.005), 0.001)
    corr = np.zeros(2000, orc.CORR_DTYPE)
    corr["index_query"] = rng.integers(0, 3000, 2000)
    corr["index_match"] = corr["index_query"]
    corr["index_match"][::7] = rng.integers(0, 3000, corr[::7].size)
    for c in (None, corr):
        iq = np.arange(3000) if c is None else c["index_query"]
        im = np.arange(3000) if c is None else c["index_match"]
        p, q = src[iq, :3], tgt[im, :3]
        T_ref = ref_svd(p, q)[0]
        assert np.linalg.norm(orc.estimate_svd(src, tgt, c, scalar_is_double=True) - T_ref) < TOL
        assert np.linalg.norm(orc.estimate_svd(src, tgt, c, scalar_is_double=True, use_umeyama=False) - T_ref) < TOL
        T_ref = ref_p2p(p, q, tgt[im, 4:7])[0]
        assert np.linalg.norm(orc.estimate_point_to_plane_lls(src, tgt, c, scalar_is_double=True)[0] - T_ref) < TOL
        T_ref = ref_sym(p, q, src[iq, 4:7], tgt[im, 4:7])[0]
        assert np.linalg.norm(orc.estimate_symmetric_lls(src, tgt, c, scalar_is_double=True)[0] - T_ref) < TOL


def test_far_patch_reference_is_exact_where_raw_moments_are_not():
    """The scene the SVD origin exists for: the reference does not depend on where the coordinates' origin lies (the same
    pairs moved by a float-exact 512 m give the same rotation to 1e-13), while raw moments about the map's centre lose
    most of the rotation's digits (the arithmetic k_solve had before its sums were taken about a point near the pairs)."""
    src, tgt = far_patch(0.02)
    import oracle as orc
    c = orc.Index(tgt).correspondences(src, 0.01)
    p, q = src[c["index_query"], :3].astype(np.float64), tgt[c["index_match"], :3].astype(np.float64)
    T = ref_svd(p, q)[0]
    T0 = ref_svd(p - 512.0, q - 512.0)[0]
    assert np.linalg.norm(T[:3, :3] - T0[:3, :3]) < 1e-13
    n = p.shape[0]
    mp, mq = p.sum(0) / n, q.sum(0) / n
    sig = (q.T @ p) / n - np.outer(mq, mp)
    U, s, Vt = np.linalg.svd(sig)
    S = np.diag([1, 1, np.sign(np.linalg.det(U) * np.linalg.det(Vt))])
    assert np.linalg.norm(U @ S @ Vt - T[:3, :3]) > 1e-8


# ---- GPU --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu():
    import pcl_b200
    pcl_b200.lib()
    ctx = pcl_b200.Context(0)
    yield pcl_b200, ctx
    ctx.close()


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sizes(k):
    """source sizes that end a warp, a block and the persistent grid of k blocks of 256 per SM on either side"""
    B = _sms() * k * 256
    return [3, 4, 31, 32, 33, 255, 256, 257, B - 1, B, B + 1, 2 * B + 37]


WORST = {}


def _note(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nlargest |T_dev - T_ref| / tol per estimator:", {k: f"{v:.3g}" for k, v in sorted(WORST.items())})


EST = {"svd": 0, "svd_corr": 0, "p2p": 1, "sym": 2}


def _session(P, ctx, src, tgt, est, dbl, gate, kind=0, recip=False, rejectors=(), is_dense=1, max_iterations=50):
    idx = P.Index(ctx, np.ascontiguousarray(tgt[:, :4]))
    normals_transform = est in ("p2p", "sym") or kind != 0
    s = P.Icp(ctx, max_iterations=max_iterations, estimator=EST[est], scalar_is_double=int(dbl),
              max_correspondence_distance=gate, use_reciprocal=int(recip), svd_no_umeyama=int(est == "svd_corr"),
              with_normals_transform=int(normals_transform), correspondence_kind=kind, correspondence_k=8,
              is_dense=is_dense, transformation_epsilon=0.0, euclidean_fitness_epsilon=-1.0)
    s.set_target(idx, normals=np.ascontiguousarray(tgt[:, 4:8]))
    if rejectors:
        s.set_rejectors(list(rejectors))
    s.set_source(np.ascontiguousarray(src[:, :4]), normals=np.ascontiguousarray(src[:, 4:8]) if normals_transform else None)
    return s, idx, normals_transform


def run_loop(P, ctx, src, tgt, est, dbl, gate, iterations=2, sharp=True, **kw):
    """`iterations` single steps of the loop; every step's estimate against the reference of its own pairs.  The source
    of step k is rebuilt from the caller's cloud and the device's earlier increments (the oracle's transform in the
    loop's operation order), and must reproduce every returned distance bit for bit."""
    import oracle as orc
    s, idx, nt = _session(P, ctx, src, tgt, est, dbl, gate, **kw)
    cur = np.ascontiguousarray(src.copy())
    ratios = []
    for it in range(iterations):
        st = s.iterate(1)
        if st["iterations"] != it + 1:
            break
        c = s.get_correspondences()
        assert st["n_correspondences"] == c.size
        d2 = c["distance"].astype(np.float64)
        assert abs(st["mse"] - math.fsum(d2) / c.size) <= 1e-15 * abs(st["mse"])
        p, q = cur[c["index_query"], :3], tgt[c["index_match"], :3]
        dd = (p - q).astype(np.float32)
        d2_host = (dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2]
        assert np.array_equal(d2_host.view(np.uint32), c["distance"].view(np.uint32)), "the rebuilt source is not the device's"
        r = check_estimate(est, st["last"], dbl, p, q, tgt[c["index_match"], 4:7], cur[c["index_query"], 4:7], sharp)
        _note(f"loop {est} {'double' if dbl else 'float'}", r)
        ratios.append(r)
        cur = orc.transform(cur, st["last"], scalar_is_double=dbl, mode=1 if nt else 0, normal_off=4 if nt else -1)
    return ratios, s


DBL = pytest.mark.parametrize("dbl", [False, True], ids=["float", "double"])


@pytest.mark.gpu
@DBL
@pytest.mark.parametrize("est", ["svd", "svd_corr", "p2p", "sym"])
@pytest.mark.parametrize("corr", ["nearest", "reciprocal", "normal_shooting", "median_one_to_one"])
def test_loop_bulk(gpu, est, dbl, corr):
    """the bulk surface (60 k pairs, 5 deg): two iterations of every estimator and correspondence mode"""
    P, ctx = gpu
    src, tgt = bulk()
    kw = {"reciprocal": dict(recip=True), "normal_shooting": dict(kind=P.CORR_NORMAL_SHOOTING),
          "median_one_to_one": dict(rejectors=[(P.REJ_MEDIAN, 1.5, 0), (P.REJ_ONE_TO_ONE, 0.0, 0)])}.get(corr, {})
    r, _ = run_loop(P, ctx, src, tgt, est, dbl, 0.05, **kw)
    assert len(r) == 2


@pytest.mark.gpu
@DBL
@pytest.mark.parametrize("est", ["svd", "svd_corr"])
@pytest.mark.parametrize("size", [0.02, 0.1, 1.0], ids=["2cm", "10cm", "1m"])
def test_loop_far_patch(gpu, est, dbl, size):
    """small patches 500 m from the map's centre: the SVD sums about an origin near the pairs, every iteration"""
    P, ctx = gpu
    src, tgt = far_patch(size)
    r, _ = run_loop(P, ctx, src, tgt, est, dbl, 0.01, iterations=3)
    assert len(r) == 3


@pytest.mark.gpu
@pytest.mark.parametrize("k_est", [(5, "svd"), (5, "p2p"), (8, "sym")], ids=["dmma-svd", "dmma-p2p", "accum-sym"])
@DBL
def test_loop_tail_shapes(gpu, k_est, dbl):
    """iteration 1 at every tail shape of the accumulating kernel's grid (k_accum_dmma: 5 blocks per SM, k_accum: 8); the
    normal equations need six pairs"""
    P, ctx = gpu
    k, est = k_est
    for n in _sizes(k):
        if est != "svd" and n < 6:
            continue
        src, tgt = bulk(n, seed=n % 97, deg=1.0, shift=(0.003, -0.002, 0.001))
        r, _ = run_loop(P, ctx, src, tgt, est, dbl, 0.05, iterations=1, sharp=n >= 31)
        assert len(r) == 1, n


@pytest.mark.gpu
@DBL
@pytest.mark.parametrize("est", ["svd", "p2p", "sym"])
def test_loop_holes_and_non_finite(gpu, est, dbl):
    """a gate that rejects about half the pairs at random, non-finite source points with is_dense = 0, non-finite target
    normals (the pair is counted and adds no terms)"""
    P, ctx = gpu
    rng = np.random.default_rng(8)
    src, tgt = bulk(100000)
    src = src[:100000].copy()
    far = rng.random(src.shape[0]) < 0.5
    src[far, 2] += 0.2
    src[rng.choice(src.shape[0], 500, replace=False), rng.integers(0, 3)] = np.nan
    src[rng.choice(src.shape[0], 20, replace=False), 1] = np.inf
    tgt = tgt.copy()
    tgt[rng.choice(tgt.shape[0], 3000, replace=False), 4 + rng.integers(0, 3)] = np.nan
    r, s = run_loop(P, ctx, src, tgt, est, dbl, 0.05, is_dense=0)
    assert len(r) == 2


@pytest.mark.gpu
@DBL
@pytest.mark.parametrize("est", ["svd", "svd_corr"])
def test_loop_exactly_three_pairs(gpu, est, dbl):
    """about 100 k queries of which exactly 3 (the loop's minimum) find a target point inside the gate"""
    P, ctx = gpu
    rng = np.random.default_rng(9)
    tgt = surface(rng, 100000)
    src = tgt.copy()
    src[:, 2] += 1.0
    pick = [10, 50000, 99990]
    src[pick, :3] = tgt[pick, :3] + np.array([[0.001, 0, 0], [0, -0.001, 0.0005], [0.0007, 0.0002, -0.001]], np.float32)
    r, s = run_loop(P, ctx, src, tgt, est, dbl, 0.01, iterations=1, sharp=False)
    assert len(r) == 1 and s.get_correspondences().size == 3


# ---- degenerate sets: stand-alone and iteration 1 ----------------------------------------------------------------------
def _degenerate(kind):
    rng = np.random.default_rng(12)
    n = 4000
    if kind == "planar":
        q = np.c_[rng.random((n, 2)), np.zeros(n)]
        p = (q - 0.5) @ _rot((0.1, 1.0, 0.3), 4.0).T + 0.5 + [0.01, 0.0, -0.02] + 1e-3 * rng.normal(size=(n, 3))
    elif kind == "collinear":
        tt = rng.random(n)
        q = np.c_[tt, 2 * tt, -tt] + [0.3, 0.1, 0.2]
        p = q + [0.002, -0.001, 0.003]
    elif kind == "identical":
        q = np.tile([[0.25, -0.5, 0.75]], (n, 1))
        p = np.tile([[0.5, 0.5, 0.5]], (n, 1))
    elif kind == "half_turn":
        q = rng.random((n, 3))
        p = (q - 0.5) @ _rot((1.0, 1.0, 0.0), 180.0).T + 0.5 + 1e-3 * rng.normal(size=(n, 3))
    else:  # near-planar: s2 ~ 0 with noise, where the sign fix decides
        q = np.c_[rng.random((n, 2)), 1e-6 * rng.normal(size=n)]
        p = (q - 0.5) @ _rot((0.0, 0.3, 1.0), 2.0).T + 0.5 + 1e-4 * rng.normal(size=(n, 3))
    src, tgt = np.zeros((n, 8), np.float32), np.zeros((n, 8), np.float32)
    src[:, :3], tgt[:, :3] = p, q
    src[:, 3] = tgt[:, 3] = 1.0
    return src, tgt


def _objective(T, p, q):
    r = np.asarray(p, np.float64) @ T[:3, :3].T + T[:3, 3] - np.asarray(q, np.float64)
    return math.fsum((r * r).ravel())


def _check_degenerate(kind, T, dbl, p, q):
    if kind in ("planar", "half_turn", "near_planar"):
        return check_estimate("svd", T, dbl, p, q)
    R = T[:3, :3]
    bar = 1e-12 if dbl else 1e-6
    assert abs(np.linalg.det(R) - 1) < bar and np.linalg.norm(R @ R.T - np.eye(3)) < bar
    if kind == "identical":
        assert np.array_equal(R, np.eye(3))
        assert np.array_equal(T[:3, 3], (q[0].astype(np.float64) - p[0]).astype(np.float32 if not dbl else np.float64))
        return 0.0
    # rank 1: the rotation about the line is free; the objective must equal the optimum
    f_ref = _objective(ref_svd(p, q)[0], p, q)
    assert abs(_objective(T, p, q) - f_ref) <= bar * max(1.0, f_ref) * p.shape[0]
    return 0.0


@pytest.mark.gpu
@DBL
@pytest.mark.parametrize("kind", ["planar", "collinear", "identical", "half_turn", "near_planar"])
def test_degenerate_sets(gpu, kind, dbl):
    """rank-2, rank-1 and rank-0 correlations, a 180 deg rotation and a noisy plane, through estimate_svd (both formulas,
    with and without a pair list) and through iteration 1 of the loop"""
    P, ctx = gpu
    src, tgt = _degenerate(kind)
    p, q = src[:, :3], tgt[:, :3]
    for um in (True, False):
        T = ctx.estimate_svd(np.ascontiguousarray(src[:, :4]), np.ascontiguousarray(tgt[:, :4]), scalar_is_double=dbl,
                             use_umeyama=um)
        _note(f"stand-alone degenerate {'double' if dbl else 'float'}", _check_degenerate(kind, T, dbl, p, q))
    if kind in ("planar", "half_turn", "near_planar"):
        corr = np.zeros(src.shape[0], P.CORR_DTYPE)
        corr["index_query"] = corr["index_match"] = np.arange(src.shape[0])
        T = ctx.estimate_svd(np.ascontiguousarray(src[:, :4]), np.ascontiguousarray(tgt[:, :4]), corr, scalar_is_double=dbl)
        _check_degenerate(kind, T, dbl, p, q)
    if kind in ("planar", "near_planar"):  # the nearest-neighbour pairs of the loop (a half turn pairs points differently)
        run_loop(P, ctx, src, tgt, "svd", dbl, 0.05, iterations=1)


# ---- the stand-alone estimators ----------------------------------------------------------------------------------------
def _standalone(P, ctx, est, src, tgt, corr, dbl):
    s4, t4 = np.ascontiguousarray(src[:, :4]), np.ascontiguousarray(tgt[:, :4])
    if est in ("svd", "svd_corr"):
        return ctx.estimate_svd(s4, t4, corr, scalar_is_double=dbl, use_umeyama=est == "svd")
    if est == "p2p":
        return ctx.estimate_point_to_plane_lls(s4, tgt, corr, scalar_is_double=dbl)
    return ctx.estimate_symmetric_lls(src, tgt, corr, scalar_is_double=dbl)


@pytest.mark.gpu
@DBL
@pytest.mark.parametrize("est", ["svd", "svd_corr", "p2p", "sym"])
@pytest.mark.parametrize("with_corr", [False, True], ids=["all_pairs", "pair_list"])
def test_standalone_tail_shapes(gpu, est, dbl, with_corr):
    """k_accum_pairs at every tail shape of its grid (4 blocks of 256 per SM), with a pair list that repeats indices; the
    normal equations need six pairs"""
    P, ctx = gpu
    for n in _sizes(4):
        if est in ("p2p", "sym") and n < 6:
            continue
        rng = np.random.default_rng(n)
        tgt = surface(rng, n)
        src = moved(rng, tgt, 3.0, (0.02, -0.01, 0.005), 0.001)
        corr = None
        iq = im = np.arange(n)
        if with_corr:
            corr = np.zeros(n, P.CORR_DTYPE)
            corr["index_query"] = rng.integers(0, n, n)
            corr["index_match"] = corr["index_query"]
            corr["index_match"][::5] = rng.integers(0, n, corr[::5].size)
            iq, im = corr["index_query"], corr["index_match"]
        T = _standalone(P, ctx, est, src, tgt, corr, dbl)
        r = check_estimate(est, T, dbl, src[iq, :3], tgt[im, :3], tgt[im, 4:7], src[iq, 4:7], sharp=n >= 31)
        _note(f"stand-alone {est} {'double' if dbl else 'float'}", r)


@pytest.mark.gpu
@DBL
@pytest.mark.parametrize("est", ["svd", "svd_corr"])
@pytest.mark.parametrize("size", [0.02, 0.1, 1.0], ids=["2cm", "10cm", "1m"])
def test_standalone_far_patch(gpu, est, dbl, size):
    """the far patch's pairs handed to estimate_svd as a list (the target's first point lies in the sparse map)"""
    P, ctx = gpu
    import oracle as orc
    src, tgt = far_patch(size)
    c = orc.Index(tgt).correspondences(src, 0.01)
    T = _standalone(P, ctx, est, src, tgt, c, dbl)
    r = check_estimate(est, T, dbl, src[c["index_query"], :3], tgt[c["index_match"], :3])
    _note(f"stand-alone far patch {est} {'double' if dbl else 'float'}", r)
