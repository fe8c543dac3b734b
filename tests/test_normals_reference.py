"""Every normal and curvature against an extended-precision reference of its own neighbourhood (CPU part).

The reference restates PCL's normal estimation (NormalEstimation::computePointNormal, normal_3d.h:308-322) in exact
arithmetic, query by query:

* the neighbour set by brute force over the fp32 points, with the library's squared distance
  ((dx*dx + dy*dy) + dz*dz) rounded to float at every step, ordered by (d2, original index);
* the covariance of those float points in long double (two passes: mean, then centred products) -- in exact
  arithmetic PCL's shifted single-pass moments (centroid.hpp:605-651) equal it for any shift K;
* the smallest eigenpair from fp64 eigh, with eigen33's branches (eigen.hpp:52-133, 273-326; knn_warp.cuh):
  |det S| < FLT_EPSILON (S = C / max|C_ij|) sets the root to 0 and takes the longest cross product of two rows of S,
  i.e. the dominant column of adj(S), with curvature exactly 0; a repeated smallest root leaves any unit vector of
  span(v0, v1); where a branch quantity is within its evaluation error of the threshold either branch is accepted;
* the viewpoint flip (normal_3d.h:169-188), either sign where (vp - q).n_ref is within the direction bar.

Each output is held to bars set by the conditioning of its own neighbourhood (eps = 2^-24, E the covariance budget
below, scale = max|C_ij|, gap = lambda1 - lambda0):

* direction  ||n - n_ref|| <= C_N eps E' / gap, where E' = E + scale min(scale / gap, eps^-1/2)
* curvature  |c - c_ref| trace <= C_C eps E'
* Rayleigh   n^T C n - lambda0 <= the curvature bar, everywhere
* unit length | ||n|| - 1 | <= 4 eps, and the float dot (vp - q).n of the output is >= 0.

E here is the budget of the float covariance: (sqrt(k) + 4) times the mean squared distance from the first neighbour
(the size of each summand of the shifted moments) plus scale; the squared diameter bounds that mean, and the k-times
bound the first form of these bars used left them more than 100 times wider than the oracle ever needed.  The term
scale min(scale / gap, eps^-1/2) is the closed-form cubic's error near a double root: a perturbation of the
characteristic polynomial by eps scale^3 moves a root by eps scale^3 / p'(lambda0) ~ eps scale^2 / gap, and never by
more than sqrt(eps) scale (the six points +-e_i give 0.33324 for 1/3 on the CPU); the direction inherits it through
the root the cross products use.  The constants were set once from
the oracle on the scenes below (the smallest power of two at least 4x its worst ratio, printed by these tests) and the
device is held to the same constants (tests/test_gpu_normals_reference.py).

GICP covariances (GeneralizedIterativeClosestPoint::computeCovariances, gicp.hpp:69-147) get the same treatment in
fp64: the exact covariance of the float differences fl(p - q), divided by the requested k, regularised to
I - (1 - eps_gicp) v0 v0^T, within C_G 2^-53 E / gap."""
import math

import numpy as np
import pytest
from scipy.spatial import cKDTree

EPS = 2.0 ** -24
FLT_EPSILON = float(np.finfo(np.float32).eps)
SQRT_EPS_INV = 2.0 ** 12
# frozen from the oracle on the scenes of this file (see the module docstring); never tuned to the device
C_N = 2.0 ** 2
C_C = 2.0 ** 4
C_G = 2.0 ** 0


# ---------------------------------------------------------------------------------------------------------------------
# neighbour sets
# ---------------------------------------------------------------------------------------------------------------------
def d2_fp32(q, P):
    """The library's squared distance of float points, rounded to float at every step: ((dx dx + dy dy) + dz dz)."""
    d = (P.astype(np.float32) - q.astype(np.float32)[..., None, :]).astype(np.float32)
    return ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).astype(np.float32)


def _valid(cloud):
    xyz = np.asarray(cloud, dtype=np.float32)[:, :3]
    ids = np.nonzero(np.isfinite(xyz).all(1))[0]
    return xyz, ids


def d2_fp64(q, P):
    """The squared distance of the same float points in double: what the fp32 rule must not be confused with."""
    d = P.astype(np.float64) - q.astype(np.float64)[..., None, :]
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def knn_sets(cloud, queries, k, return_d2=False, dist=d2_fp32, tie=1):
    """(nq, k) original indices of the k nearest finite points of every query by (fp32 d2, index), -1 past the number
    of finite points and for non-finite queries; with return_d2 also their d2 as float32 (+inf where the index is -1).
    A kd-tree proposes candidates; the fp32 rule selects them.  Smaller k are prefixes of the result.

    dist and tie replace the distance rule and the tie order (tie = -1: (d2, -index)); they exist to show that the
    scenes of tests/test_search_reference.py depend on both."""
    xyz, ids = _valid(cloud)
    q = np.asarray(queries, dtype=np.float32)[:, :3]
    nq = q.shape[0]
    out = np.full((nq, k), -1, dtype=np.int64)
    od = np.full((nq, k), np.inf, dtype=np.float32)
    keff = min(k, ids.size)
    if keff == 0:
        return (out, od) if return_d2 else out
    tree = cKDTree(xyz[ids].astype(np.float64))

    def take(rows, oi):
        d2 = dist(q[rows], xyz[oi])
        order = np.lexsort((tie * oi, d2), axis=-1)
        oi, d2 = np.take_along_axis(oi, order, 1), np.take_along_axis(d2, order, 1)
        out[rows, :keff] = oi[:, :keff]
        od[rows, :keff] = d2[:, :keff]

    todo = np.nonzero(np.isfinite(q).all(1))[0]
    m = min(keff + 8, ids.size)
    while todo.size:
        if 4 * m >= ids.size:
            # the rest against every point (queries far from a compact cloud, where all points are nearly equidistant)
            for a in range(0, todo.size, max(1, (1 << 22) // ids.size)):
                rows = todo[a:a + max(1, (1 << 22) // ids.size)]
                take(rows, np.broadcast_to(ids, (rows.size, ids.size)))
            break
        left = []
        for a in range(0, todo.size, max(1, (1 << 23) // m)):
            rows = todo[a:a + max(1, (1 << 23) // m)]
            dst, cand = tree.query(q[rows].astype(np.float64), m, workers=-1)
            dst, cand = dst.reshape(rows.size, m), cand.reshape(rows.size, m)
            oi = ids[cand]
            d2 = dist(q[rows], xyz[oi])
            # complete when every point outside the candidates is provably farther than the k-th (fp32 d2 is within a
            # few ulp of the exact squared distance)
            done = (m == ids.size) | (np.sort(d2, 1)[:, keff - 1].astype(np.float64) < dst[:, -1] ** 2 * (1 - 1e-5))
            # all m candidates coincide with the query (more than k + 8 exact duplicates): the k-th is at d2 = 0 and
            # the order among the duplicates is the index order, so gather every point at d2 = 0 and keep the first k
            dup = ~done & (dst[:, -1] == 0)
            if done.any():
                take(rows[done], oi[done])
            for i in np.nonzero(dup)[0]:
                z = ids[np.asarray(tree.query_ball_point(q[rows[i]].astype(np.float64), 1e-20), dtype=np.int64)]
                z = z[dist(q[rows[i]], xyz[z]) == 0]
                z = np.sort(tie * z) * tie
                out[rows[i], :keff] = z[:keff]
                od[rows[i], :keff] = 0
            left.append(rows[~(done | dup)])
        todo = np.concatenate(left)
        m = min(2 * m, ids.size)
    return (out, od) if return_d2 else out


def radius_csr(cloud, queries, radius, max_nn=0):
    """Every finite point with fp32 d2 < float(radius * radius) per query, by (d2, index), as CSR (offsets (nq + 1),
    original indices, d2); max_nn > 0 keeps the max_nn nearest of each row (KdTreeFLANN::radiusSearch)."""
    xyz, ids = _valid(cloud)
    q = np.asarray(queries, dtype=np.float32)[:, :3]
    nq = q.shape[0]
    r2 = np.float32(radius * radius)
    tree = cKDTree(xyz[ids].astype(np.float64))
    fin = np.nonzero(np.isfinite(q).all(1))[0]
    lists = tree.query_ball_point(q[fin].astype(np.float64), radius * (1 + 1e-5) + 1e-30, workers=-1,
                                  return_sorted=False) if fin.size else []
    lens = np.fromiter((len(x) for x in lists), dtype=np.int64, count=len(lists))
    row = np.repeat(fin, lens)
    oi = ids[np.concatenate([np.asarray(x, dtype=np.int64) for x in lists]) if lens.sum() else np.zeros(0, np.int64)]
    d2 = d2_fp32(q[row], xyz[oi][:, None, :])[:, 0] if row.size else np.zeros(0, np.float32)
    keep = d2 < r2
    row, oi, d2 = row[keep], oi[keep], d2[keep]
    order = np.lexsort((oi, d2, row))
    row, oi, d2 = row[order], oi[order], d2[order]
    if 0 < max_nn < ids.size:
        start = np.searchsorted(row, row, side="left")
        keep = np.arange(row.size) - start < max_nn
        row, oi, d2 = row[keep], oi[keep], d2[keep]
    offsets = np.zeros(nq + 1, dtype=np.int64)
    np.cumsum(np.bincount(row, minlength=nq), out=offsets[1:])
    return offsets, oi, d2


def radius_sets(cloud, queries, radius):
    """Per query, the original indices of every finite point with fp32 d2 < float(radius * radius), by (d2, index)."""
    offsets, oi, _ = radius_csr(cloud, queries, radius)
    return [oi[offsets[i]:offsets[i + 1]] for i in range(offsets.size - 1)]


# ---------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------
def _diameter2(X):
    """Squared diameter of every neighbourhood (m, k, 3) -> (m,)."""
    out = np.empty(X.shape[0])
    for a in range(0, X.shape[0], 512):
        Y = X[a:a + 512].astype(np.float64)
        d = Y[:, :, None, :] - Y[:, None, :, :]
        out[a:a + 512] = (d * d).sum(-1).max((1, 2))
    return out


def budget(X, scale):
    """E: what the float covariance of X can be off by, in units of eps: (sqrt(k) + 4) times the mean squared distance
    from the first neighbour (the shift of PCL's single-pass moments, so the size of every summand), plus scale for
    the solver.  The squared diameter bounds that mean; the rounding of k summands grows like sqrt(k)."""
    k = X.shape[1]
    d = (X[:, :, :].astype(np.float64) - X[:, :1, :].astype(np.float64))
    return (math.sqrt(k) + 4) * (d * d).sum(-1).mean(1) + scale


def _exact_cov(X, div=None):
    """Covariance of float points (m, k, 3) in long double, two passes, as fp64."""
    Xl = X.astype(np.longdouble)
    k = X.shape[1]
    mu = Xl.sum(1, keepdims=True) / k
    Y = Xl - mu
    C = np.einsum("mki,mkj->mij", Y, Y) / (k if div is None else div)
    return C.astype(np.float64)


def reference_batch(X, q, vp):
    """PCL's normal of every neighbourhood X (m, k, 3) float32 (all finite, k >= 3), queries q (m, 3), viewpoint vp:
    a dict of the quantities the acceptance needs."""
    m, k = X.shape[:2]
    C = _exact_cov(X)
    w, V = np.linalg.eigh(C)
    w = np.maximum(w, 0.0)
    scale = np.abs(C).reshape(m, 9).max(1)
    scale_s = np.where(scale <= np.finfo(np.float32).tiny, 1.0, scale)
    S = C / scale_s[:, None, None]
    det = np.linalg.det(S)
    E = budget(X, scale)
    gap = w[:, 1] - w[:, 0]
    tol = C_C * EPS * E / scale_s  # evaluation error of a branch quantity of S
    # eigen33's first branch: |det S| < FLT_EPSILON or a computed root <= 0 -> root 0, longest cross product of rows
    adj_possible = (np.abs(det) < FLT_EPSILON + 4 * tol) | (w[:, 0] / scale_s <= tol)
    cubic_possible = np.abs(det) >= FLT_EPSILON - 4 * tol
    rows = [(0, 1), (0, 2), (1, 2)]
    adj = np.stack([np.cross(S[:, a], S[:, b]) for a, b in rows], 1)  # (m, 3 candidates, 3)
    alen = np.linalg.norm(adj, axis=-1)
    adj_ok = alen >= alen.max(1, keepdims=True) - 4 * tol[:, None]
    adj = adj / np.where(alen > 0, alen, 1.0)[..., None]
    return dict(C=C, w=w, V=V, scale=scale, trace=np.trace(C, axis1=1, axis2=2), E=E, gap=gap, k=k,
                adj=adj, adj_ok=adj_ok & adj_possible[:, None] & (alen > 0), cubic=cubic_possible | ~adj_possible,
                adj_possible=adj_possible, q=np.asarray(q, np.float32)[:, :3], vp=np.asarray(vp, np.float32))


def bars(ref):
    """(direction bar, span(v0, v1) bar, curvature / Rayleigh bar) per query.  Every bar carries the budget E plus the
    closed-form cubic's root error near a double root, scale min(scale / gap, eps^-1/2); a direction is not checked
    where the neighbourhood is collinear in float (lambda1 < sqrt(eps) scale) or the gap it needs is lost."""
    gap, scale = ref["gap"], ref["scale"]
    gap2 = ref["w"][:, 2] - ref["w"][:, 1]
    with np.errstate(divide="ignore", invalid="ignore"):
        Ea = ref["E"] + scale * np.minimum(scale / gap, SQRT_EPS_INV)
        bar_n = np.where(gap > 0, C_N * EPS * Ea / gap, np.inf)
        bar_span = np.where((gap2 > 0) & (ref["w"][:, 1] >= scale / SQRT_EPS_INV), C_N * EPS * Ea / gap2, np.inf)
    bar_c = C_C * EPS * Ea
    return bar_n, bar_span, bar_c


def errors(ref, out):
    """Per query, (direction error, its bar), (curvature error, its bar), (Rayleigh residual, its bar), unit-length
    error, and whether the float flip test holds, for outputs out (m, 4) = (nx, ny, nz, curvature)."""
    out = np.asarray(out, dtype=np.float32)
    n = out[:, :3].astype(np.float64)
    nn = np.linalg.norm(n, axis=1)
    u = n / np.where(nn > 0, nn, 1.0)[:, None]
    bar_n, bar_span, bar_c = bars(ref)
    q, vp = ref["q"].astype(np.float64), ref["vp"].astype(np.float64)
    view = vp[None, :] - q
    vnorm = np.linalg.norm(view, axis=1)

    def oriented(c, bar):
        """chord distance from u to the candidate direction c (m, 3), with the sign the flip gives it"""
        s = np.sign((view * c).sum(1))
        either = np.abs((view * c).sum(1)) <= (bar + 8 * EPS) * vnorm
        s = np.where(s == 0, 1.0, s)
        d_fixed = np.linalg.norm(u - s[:, None] * c, axis=1)
        d_other = np.linalg.norm(u + s[:, None] * c, axis=1)
        return np.where(either, np.minimum(d_fixed, d_other), d_fixed)

    inf = np.full(len(u), np.inf)
    e_dir = np.where(ref["cubic"], oriented(ref["V"][:, :, 0], bar_n), inf)
    for j in range(3):
        e_dir = np.minimum(e_dir, np.where(ref["adj_ok"][:, j], oriented(ref["adj"][:, j], bar_n), inf))
    # where the first gap is lost in rounding (bar >= 1) only span(v0, v1) is determined
    span = bar_n >= 1
    e_span = np.abs((u * ref["V"][:, :, 2]).sum(1))
    e_dir = np.where(span, e_span, e_dir)
    b_dir = np.where(span, np.where(bar_span >= 1, np.inf, bar_span), bar_n)
    tr = ref["trace"]
    c_ref = np.where(tr > 0, ref["w"][:, 0] / np.where(tr > 0, tr, 1.0), 0.0)
    c = out[:, 3].astype(np.float64)
    e_c = np.where(ref["cubic"] | span, np.abs(c - c_ref) * tr, np.inf)
    e_c = np.minimum(e_c, np.where(ref["adj_possible"], np.abs(c) * tr, np.inf))
    e_ray = np.einsum("mi,mij,mj->m", u, ref["C"], u) - ref["w"][:, 0]
    e_unit = np.abs(nn - 1.0)
    vf = (ref["vp"][None, :] - ref["q"]).astype(np.float32)
    cos = ((vf[:, 0] * out[:, 0] + vf[:, 1] * out[:, 1]) + vf[:, 2] * out[:, 2]).astype(np.float32)
    return dict(dir=(e_dir, b_dir), curv=(e_c, bar_c), ray=(e_ray, bar_c), unit=e_unit, flip_ok=cos >= 0)


def check(ref, out, label="", rayleigh_only=False):
    """Asserts every query of `out` against the reference; returns the worst ratio of each error to its bar."""
    e = errors(ref, out)
    worst = {"dir": 0.0, "curv": 0.0}
    for key in ("ray",) if rayleigh_only else ("dir", "curv", "ray"):
        err, bar = e[key]
        r = np.where(np.isinf(bar), 0.0, err / np.maximum(bar, 1e-300))
        bad = np.nonzero(~(r <= 1.0))[0]
        assert bad.size == 0, (label, key, bad.size, bad[:5].tolist(), r[bad[:5]].tolist(), np.asarray(out)[bad[:3]].tolist())
        worst[key] = float(r.max()) if r.size else 0.0
    bad = np.nonzero(e["unit"] > 4 * EPS)[0]
    assert bad.size == 0, (label, "unit", bad[:5].tolist(), e["unit"][bad[:5]].tolist())
    bad = np.nonzero(~e["flip_ok"])[0]
    assert bad.size == 0, (label, "flip", bad[:5].tolist())
    return worst


class Reference:
    """Reference of every query of a normals call: rows[i] is None where PCL writes a NaN row (< 3 neighbours or a
    non-finite query), otherwise (group, position) into per-size batches."""

    def __init__(self, cloud, queries, vp, k=None, radius=None, sets=None):
        xyz, _ = _valid(cloud)
        q = np.asarray(queries, dtype=np.float32)[:, :3]
        if sets is None:
            sets = list(knn_sets(cloud, q, k)) if radius is None else radius_sets(cloud, q, radius)
        self.sets = [np.asarray(s)[np.asarray(s) >= 0] for s in sets]
        counts = np.array([s.size for s in self.sets])
        self.nan_rows = (counts < 3) | ~np.isfinite(q).all(1)
        self.groups = {}
        for c in np.unique(counts[~self.nan_rows]):
            rows = np.nonzero((counts == c) & ~self.nan_rows)[0]
            X = np.stack([xyz[self.sets[i]] for i in rows])
            self.groups[int(c)] = (rows, reference_batch(X, q[rows], vp))

    def check(self, out, label="", rayleigh_only=False):
        out = np.asarray(out, dtype=np.float32)
        assert np.array_equal(np.isnan(out).any(1), self.nan_rows), (label, np.nonzero(np.isnan(out).any(1) != self.nan_rows)[0][:5])
        assert np.isnan(out[self.nan_rows]).all(), label
        assert np.isfinite(out[~self.nan_rows]).all(), label
        worst = {"dir": 0.0, "curv": 0.0, "ray": 0.0}
        for c, (rows, ref) in self.groups.items():
            w = check(ref, out[rows], f"{label} n={c}", rayleigh_only)
            worst = {key: max(worst[key], w[key]) for key in worst}
        return worst

    @property
    def is_dense(self):
        return not self.nan_rows.any()


# ---------------------------------------------------------------------------------------------------------------------
# scenes (shared with tests/test_gpu_normals_reference.py)
# ---------------------------------------------------------------------------------------------------------------------
def sine_sheet(n=30000, seed=15):
    rng = np.random.default_rng(seed)
    pts = rng.random((n, 3), dtype=np.float32)
    pts[:, 2] = np.float32(0.1) * np.sin(np.float32(6) * pts[:, 0])
    return pts, (0.5, 0.5, 5.0)


def noisy_plane(n=20000, seed=3):
    rng = np.random.default_rng(seed)
    xy = rng.random((n, 2))
    z = 0.3 * xy[:, 0] - 0.2 * xy[:, 1] + 1e-4 * rng.standard_normal(n)
    return np.column_stack([xy, z]).astype(np.float32), (0.5, 0.5, 3.0)


def far_patch(offset, seed=5, side=70):
    """A curved patch `offset` from the origin on a jittered grid a few hundred ulp apart."""
    rng = np.random.default_rng(seed)
    h = 300 * float(np.spacing(np.float32(offset)))
    g = np.stack(np.meshgrid(np.arange(side), np.arange(side), indexing="ij"), -1).reshape(-1, 2).astype(np.float64)
    xy = (g + 0.3 * rng.random(g.shape)) * h
    ext = side * h
    z = 0.4 * ((xy[:, 0] - ext / 2) ** 2 - 0.5 * (xy[:, 1] - ext / 2) ** 2) / ext
    pts = (np.column_stack([xy, z]) + offset).astype(np.float32)
    return pts, tuple(float(v) for v in (offset + ext / 2, offset + ext / 2, offset + ext))


def thin_strips(seed=7, n_strips=12, per=400):
    """Strips whose k-neighbourhoods have lambda1 / lambda2 ~ 1e-2 and an out-of-plane spread ~1e-3 of the spacing:
    |det S| < FLT_EPSILON, eigen33's cross-product branch."""
    rng = np.random.default_rng(seed)
    out = []
    for s in range(n_strips):
        a = rng.normal(size=3)
        d = a / np.linalg.norm(a)
        b = np.cross(d, rng.normal(size=3))
        b /= np.linalg.norm(b)
        c = np.cross(d, b)
        t = np.arange(per) * 0.01
        pts = (np.array([s * 10.0, 0, 0]) + t[:, None] * d + (rng.random(per) - 0.5)[:, None] * 0.016 * b
               + 1e-5 * rng.standard_normal(per)[:, None] * c)
        out.append(pts)
    return np.concatenate(out).astype(np.float32), (0.0, 0.0, 50.0)


def blobs(seed=9, n_blobs=40, per=150):
    """Near-isotropic Gaussian blobs: the smallest eigenvalue is barely isolated, only the Rayleigh bar applies."""
    rng = np.random.default_rng(seed)
    centres = rng.random((n_blobs, 3)) * 100
    pts = centres[:, None, :] + rng.standard_normal((n_blobs, per, 3))
    return pts.reshape(-1, 3).astype(np.float32), (50.0, 50.0, 200.0)


def duplicated(seed=13, n=3000):
    """Every point three times (ties at the k-th distance, broken by index)."""
    rng = np.random.default_rng(seed)
    d = rng.random((n, 3), dtype=np.float32)
    d[:, 2] = np.float32(0.2) * np.sin(np.float32(4) * d[:, 0]) + np.float32(0.01) * d[:, 2]
    return np.concatenate([d, d, d]), (0.5, 0.5, 4.0)


# exact cases (no trigonometry is reached): the normal eigen33 returns before the viewpoint flip
EXACT_SHAPES = {"line_x": (0.0, 1.0, 0.0), "line_y": (1.0, 0.0, 0.0), "line_z": (0.0, -1.0, 0.0),
                "plane_z": (0.0, 0.0, 1.0), "plane_z_far": (0.0, 0.0, 1.0), "identical": (1.0, 0.0, 0.0)}


def exact_clusters(k, seed=21):
    """Separated clusters of exactly k points shaped as the exact cases, so that every k-NN list is one cluster.  Some
    clusters lie where (vp - q).n is exactly 0 (no flip), some on either side.  Returns (points, viewpoint, expected
    (n, 4) outputs, cluster radius bound)."""
    rng = np.random.default_rng(seed)
    vp = np.float32([0.0, 0.0, 0.0])
    pts, exp = [], []
    cl = 0
    for name, base in EXACT_SHAPES.items():
        for side in (0.0, 37.0, -37.0):
            # `side` is the coordinate along the expected normal: (vp - q).n is exactly 0 (no flip) when it is 0
            cl += 1
            far = cl * 1000.0  # keeps the clusters apart
            t = np.sort(rng.choice(np.arange(1, 4 * k + 1), size=k, replace=False)).astype(np.float64) * 0.125
            z = 0 * t
            if name == "line_x":
                P = np.column_stack([far + t, z + side, z])
            elif name == "line_y":
                P = np.column_stack([z + side, far + t, z])
            elif name == "line_z":
                P = np.column_stack([z + far, z + side, t])
            elif name.startswith("plane_z"):
                uv = rng.choice(np.arange(16), size=(k, 2)).astype(np.float64) * 0.25
                uv[:3] = [[0, 0], [1, 0], [0, 1]]  # never collinear
                uv[:, 0] += np.arange(k) * 4.0  # distinct points
                if name == "plane_z":
                    P = np.column_stack([far + uv[:, 0], uv[:, 1], z + side])
                else:
                    P = np.column_stack([1e4 + far + uv[:, 0], 1e4 + uv[:, 1], z + 1e4])
            else:
                P = np.column_stack([z + side, z + far, z])
            P = P.astype(np.float32)
            pts.append(P)
            for p in P:
                n = np.float32(base)
                v = (vp - p).astype(np.float32)
                if ((v[0] * n[0] + v[1] * n[1]) + v[2] * n[2]) < 0:
                    n = -n
                exp.append(np.r_[n, np.float32(0)])
    return np.concatenate(pts), tuple(float(v) for v in vp), np.array(exp, np.float32)


def exact_check(out, exp, label=""):
    out = np.asarray(out, dtype=np.float32)
    bad = np.nonzero((out != exp).any(1))[0]
    assert bad.size == 0, (label, bad.size, bad[:5].tolist(), out[bad[:3]].tolist(), exp[bad[:3]].tolist())


# ---------------------------------------------------------------------------------------------------------------------
# GICP covariances
# ---------------------------------------------------------------------------------------------------------------------
def gicp_reference(cloud, k, gicp_epsilon):
    """(n, 3, 3) reference, (n,) bar per row and the per-row kind: 'zero' (non-finite point), 'full'."""
    xyz, ids = _valid(cloud)
    n = xyz.shape[0]
    sets = knn_sets(cloud, xyz, k)
    keff = min(k, ids.size)
    fin = np.isfinite(xyz).all(1)
    ref = np.zeros((n, 3, 3))
    bar = np.zeros(n)
    rows = np.nonzero(fin)[0]
    if keff == 0 or rows.size == 0:
        return ref, bar, fin
    nb = sets[rows, :keff]
    d = (xyz[nb] - xyz[rows][:, None, :]).astype(np.float32)  # fl(p - q)
    dl = d.astype(np.longdouble)
    mean = dl.sum(1) / k
    M = (np.einsum("mki,mkj->mij", dl, dl) / k - mean[:, :, None] * mean[:, None, :]).astype(np.float64)
    w, V = np.linalg.eigh(M)
    v0 = V[:, :, 0]
    ref[rows] = np.eye(3)[None] - (1.0 - gicp_epsilon) * v0[:, :, None] * v0[:, None, :]
    scale = np.abs(M).reshape(-1, 9).max(1)
    E = (k + 4) * _diameter2(xyz[nb]) + scale
    gap = w[:, 1] - w[:, 0]
    bar[rows] = C_G * 2.0 ** -53 * E / np.maximum(gap, 1e-300)
    return ref, bar, fin


def gicp_check(cloud, got, k, gicp_epsilon, label=""):
    """Rows of non-finite points are 0; every other row is I - (1 - eps) u u^T with u a unit vector, within the bar of
    the reference where the bar is below 1.  Returns the worst ratio."""
    ref, bar, fin = gicp_reference(cloud, k, gicp_epsilon)
    got = np.asarray(got, dtype=np.float64)
    assert np.all(got[~fin] == 0), label
    w = np.linalg.eigvalsh(got[fin])
    assert np.allclose(w, [gicp_epsilon, 1.0, 1.0], atol=1e-12), (label, np.abs(w - [gicp_epsilon, 1, 1]).max())
    err = np.abs(got[fin] - ref[fin]).reshape(-1, 9).max(1)
    b = bar[fin]
    checked = b < 1
    r = np.where(checked, err / np.maximum(b, 1e-300), 0.0)
    bad = np.nonzero(r > 1)[0]
    assert bad.size == 0, (label, bad.size, bad[:5].tolist(), r[bad[:5]].tolist())
    return float(r.max()) if r.size else 0.0, int(checked.sum())


def gicp_scenes():
    rng = np.random.default_rng(31)
    n = 4000
    p = rng.random((n, 3), dtype=np.float32) * np.float32(3)
    p[:, 2] = np.float32(0.2) * np.sin(np.float32(4) * p[:, 0]) + np.float32(0.003) * rng.standard_normal(n).astype(np.float32)
    p[11, 1] = np.nan
    yield "surface", p
    pl = (rng.random((n, 3)) * [2, 2, 0] + [0, 0, 1.5]).astype(np.float32)
    yield "exact_plane", pl
    t = rng.random(n)
    yield "collinear", np.column_stack([t, 2 * t, -t]).astype(np.float32) + np.float32(0.25)
    d = rng.random((n // 4, 3), dtype=np.float32)
    dup = np.concatenate([d, d, d, d])
    dup[5, 0] = np.nan
    yield "duplicates", dup


# ---------------------------------------------------------------------------------------------------------------------
# CPU tests: the oracle against the reference, the bars' sharpness, the exact cases
# ---------------------------------------------------------------------------------------------------------------------
def _oracle_scenes():
    s, vp = sine_sheet()
    yield "sine_sheet", s, vp, (5, 16, 33)
    s, vp = noisy_plane()
    yield "noisy_plane", s, vp, (4, 16)
    for off in (1e3, 1e4):
        s, vp = far_patch(off)
        yield f"far_{off:g}", s, vp, (8, 16)
    s, vp = thin_strips()
    yield "thin_strips", s, vp, (10, 16)
    s, vp = duplicated()
    yield "duplicates", s, vp, (4, 16)


def test_neighbour_sets_match_the_oracle(orc):
    """The brute-force fp32 neighbour sets are the oracle's k-NN and radius lists."""
    rng = np.random.default_rng(1)
    for name, pts, vp, ks in _oracle_scenes():
        cloud = orc.to_xyz1(pts)
        sample = rng.choice(pts.shape[0], 500, replace=False)
        for k in ks:
            oi, _, _ = orc.Index(cloud).knn(cloud[sample], k, nthreads=4)
            assert np.array_equal(knn_sets(cloud, cloud[sample], k), oi), (name, k)
    pts, _ = sine_sheet()
    cloud = orc.to_xyz1(pts)
    cloud[::301, 1] = np.nan
    sample = rng.choice(pts.shape[0], 500, replace=False)
    offs, idx, _ = orc.Index(cloud).radius(cloud[sample], 0.004, nthreads=4)
    mine = radius_sets(cloud, cloud[sample], 0.004)
    for i in range(sample.size):
        assert np.array_equal(idx[offs[i]:offs[i + 1]], mine[i]), i


def test_oracle_normals_within_the_bars(orc):
    """Every oracle normal of every scene is inside the bars; prints the oracle's worst ratio to each bar."""
    for name, pts, vp, ks in _oracle_scenes():
        cloud = orc.to_xyz1(pts)
        for k in ks:
            o, od = orc.Index(cloud).normals_knn(cloud, k, viewpoint=vp, nthreads=8)
            ref = Reference(cloud, cloud, vp, k=k)
            worst = ref.check(o, f"{name} k={k}")
            assert od == ref.is_dense
            print(f"oracle {name:12s} k={k:2d}  worst ratio: direction {worst['dir']:.3g}  curvature {worst['curv']:.3g}"
                  f"  Rayleigh {worst['ray']:.3g}")
    s, vp = blobs()
    cloud = orc.to_xyz1(s)
    o, _ = orc.Index(cloud).normals_knn(cloud, 32, viewpoint=vp, nthreads=8)
    worst = Reference(cloud, cloud, vp, k=32).check(o, "blobs", rayleigh_only=True)
    print(f"oracle {'blobs':12s} k=32  worst ratio: Rayleigh {worst['ray']:.3g}")
    pts, vp = sine_sheet()
    cloud = orc.to_xyz1(pts)
    cloud[::501, 0] = np.nan
    for r in (0.004, 0.02):
        o, od = orc.Index(cloud).normals_radius(cloud, r, viewpoint=vp, is_dense=False, nthreads=8)
        ref = Reference(cloud, cloud, vp, radius=r)
        worst = ref.check(o, f"radius {r}")
        assert od == ref.is_dense
        print(f"oracle sine radius={r}  worst ratio: direction {worst['dir']:.3g}  curvature {worst['curv']:.3g}"
              f"  Rayleigh {worst['ray']:.3g}")


def _moved(ref, variant_n, variant_c):
    """How far a variant's (unit normal, curvature) lies outside the reference, in bars (max of direction, curvature)."""
    e = errors(ref, np.column_stack([variant_n, variant_c]).astype(np.float32))
    rd = e["dir"][0] / e["dir"][1]
    rc = e["curv"][0] / e["curv"][1]
    return np.maximum(np.nan_to_num(rd, posinf=np.inf), rc)


def _fp32_raw_moments(X):
    """PCL's single-pass moments with K = 0 in float32 (the unshifted variant), then the fp64 eigenpair."""
    X = X.astype(np.float32)
    k = X.shape[1]
    acc = np.zeros((X.shape[0], 9), np.float32)
    for j in range(k):
        x, y, z = X[:, j, 0], X[:, j, 1], X[:, j, 2]
        for t, v in enumerate((x * x, x * y, x * z, y * y, y * z, z * z, x, y, z)):
            acc[:, t] = acc[:, t] + v
    acc = acc / np.float32(k)
    C = np.empty((X.shape[0], 3, 3), np.float32)
    C[:, 0, 0] = acc[:, 0] - acc[:, 6] * acc[:, 6]
    C[:, 0, 1] = C[:, 1, 0] = acc[:, 1] - acc[:, 6] * acc[:, 7]
    C[:, 0, 2] = C[:, 2, 0] = acc[:, 2] - acc[:, 6] * acc[:, 8]
    C[:, 1, 1] = acc[:, 3] - acc[:, 7] * acc[:, 7]
    C[:, 1, 2] = C[:, 2, 1] = acc[:, 4] - acc[:, 7] * acc[:, 8]
    C[:, 2, 2] = acc[:, 5] - acc[:, 8] * acc[:, 8]
    w, V = np.linalg.eigh(C.astype(np.float64))
    tr = np.trace(C.astype(np.float64), axis1=1, axis2=2)
    return V[:, :, 0], np.abs(w[:, 0] / np.where(tr != 0, tr, 1.0))


def test_the_bars_have_teeth():
    """Each perturbed variant of the reference lies more than 100 bars away on at least 90 % of each scene's checked
    queries: unshifted fp32 moments (far scenes), the flip reversed, r1 in place of r0.  The last neighbour dropped
    does so on a third to nine tenths of the queries of the curved and noisy scenes (printed)."""
    shares = []
    for name, pts, vp, ks in _oracle_scenes():
        for k in ks:
            if name == "duplicates" and k == 4:
                continue  # three copies and one other point: collinear, only the Rayleigh bar applies
            xyz = pts[:, :3]
            sets = knn_sets(pts, xyz, k)
            X = xyz[sets]
            ref = reference_batch(X, xyz, vp)
            bar_n = bars(ref)[0]
            checked = bar_n < 1
            assert checked.mean() > 0.9, (name, k, checked.mean())

            def oriented(v):
                s = np.sign(((np.asarray(vp)[None, :] - xyz) * v).sum(1))
                return v * np.where(s == 0, 1, s)[:, None]

            tr = ref["trace"]
            variants = {}
            drop = reference_batch(X[:, :-1], xyz, vp)
            variants["drop last"] = (oriented(drop["V"][:, :, 0]), drop["w"][:, 0] / drop["trace"])
            if name.startswith("far"):
                v, c = _fp32_raw_moments(X)
                variants["K = 0 fp32"] = (oriented(v), c)
            n0 = oriented(ref["V"][:, :, 0])
            variants["flip reversed"] = (-n0, ref["w"][:, 0] / tr)
            variants["r1 for r0"] = (oriented(ref["V"][:, :, 1]), ref["w"][:, 1] / tr)
            for vname, (vn, vc) in variants.items():
                moved = _moved(ref, vn, vc)[checked]
                share = float(np.mean(moved > 100))
                print(f"sensitivity {name:12s} k={k:2d}  {vname:14s} moved > 100 bars on {100 * share:5.1f} % "
                      f"(median {np.median(moved):.3g} bars)")
                shares.append((name, k, vname, share))
    # a dropped neighbour moves a smooth fit by only ~100 bars: it must clear 100 bars on a third of the queries of
    # every curved or noisy scene (the strips are flat ribbons, where it does not move the plane at all)
    assert all(s >= (0.33 if v == "drop last" else 0.9) for n, _, v, s in shares if not (v == "drop last" and n == "thin_strips")), \
        [x for x in shares if x[-1] < 0.9]


@pytest.mark.parametrize("k", [4, 8, 10, 11, 16, 33])
def test_exact_cases_on_the_oracle(orc, k):
    """Axis-aligned lines, planes z = const (also 1e4 from the origin) and identical points: the oracle's normals are
    the exact vectors, signs by the viewpoint, curvature 0."""
    pts, vp, exp = exact_clusters(k)
    cloud = orc.to_xyz1(pts)
    o, od = orc.Index(cloud).normals_knn(cloud, k, viewpoint=vp, nthreads=4)
    assert od
    exact_check(o, exp, f"k={k}")


def test_six_axis_points_repeated_root(orc):
    """+-e_i: a triple root; the closed-form cubic loses half its digits (0.33324 for 1/3), the Rayleigh bar holds."""
    X = np.float32([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]])
    o, ok = orc.point_normal(orc.to_xyz1(X), np.arange(6))
    assert ok and abs(o[3] - 1 / 3) > 1e-5
    ref = reference_batch(X[None], X[:1], (0.0, 0.0, 0.0))
    vf = (np.float32(0) - X[0]).astype(np.float32)
    if ((vf[0] * o[0] + vf[1] * o[1]) + vf[2] * o[2]) < 0:
        o[:3] = -o[:3]
    check(ref, o[None], "six points")


def test_gicp_covariances_oracle_within_the_bar(orc):
    for name, pts in gicp_scenes():
        cloud = orc.to_xyz1(pts)
        for k in (5, 20):
            o = orc.Index(cloud).gicp_covariances(k=k, gicp_epsilon=0.001, nthreads=8)
            worst, n = gicp_check(cloud, o, k, 0.001, f"{name} k={k}")
            print(f"oracle gicp {name:12s} k={k:2d}  worst ratio {worst:.3g} over {n} rows with a bar below 1")
    few = orc.to_xyz1(np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0]]))
    o = orc.Index(few).gicp_covariances(k=5, gicp_epsilon=0.001)
    gicp_check(few, o, 5, 0.001, "fewer than k")
