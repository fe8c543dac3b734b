"""Every k-NN, radius and correspondence list against an fp32 brute-force reference on map-scale frames (CPU part).

The reference of one query is brute force under the library's rule (tests/test_normals_reference.py: d2_fp32,
knn_sets, radius_csr): d2 = ((dx dx + dy dy) + dz dz) rounded to float at every step, ordered by (d2, original index),
non-finite points dropped and non-finite queries given empty rows, as KdTreeFLANN does.  From it:

* k-NN: indices and d2, -1 / +inf past the number of finite points;
* radius: strict d2 < float(r * r), sorted; max_nn keeps the nearest prefix;
* 1-NN correspondences: the gate d2 > max_dist^2 evaluated in double; the reciprocal variant keeps a pair when the
  nearest source point of its match is the query itself, within the gate (correspondence_estimation.hpp:259-269);
* knn_stats: mean = float(sum_{j >= 1} sqrt(double(d2_j)) / (cnt - 1)), summed in list order; kth = d2 of neighbour
  k - 1, or +inf.

The scenes put the search where its exactness arguments depend on the frame: the size of an ulp against the point
spacing, a frame that straddles zero, a frame stretched by one outlier, a zero-extent axis, exact ties far out.  The
device paths are held to the same reference in tests/test_gpu_search_reference.py."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_normals_reference import d2_fp64, knn_sets, radius_csr  # noqa: E402

K_MAX = 64  # every k of these tests is a prefix of the lists at K_MAX
CORR_DTYPE = np.dtype([("index_query", np.int32), ("index_match", np.int32), ("distance", np.float32)])
NO_GATE = float(np.sqrt(np.finfo(np.float64).max))


# ---------------------------------------------------------------------------------------------------------------------
# scenes: seeded generators, (points (n, 3) float32, typical point spacing)
# ---------------------------------------------------------------------------------------------------------------------
def map_1e5(n=100_000, seed=101):
    """A wavy surface 200 m x 200 m at x, y ~ 1e5, every coordinate on the 1/128 m grid (the fp32 ulp there): many
    squared distances tie exactly."""
    rng = np.random.default_rng(seed)
    xy = rng.random((n, 2)) * 200
    z = 2.0 * np.sin(xy[:, 0] / 15) * np.cos(xy[:, 1] / 20)
    p = np.round(np.column_stack([xy + 1e5, z]) * 128) / 128
    return p.astype(np.float32), 200 / np.sqrt(n)


def straddle(n=100_000, seed=102):
    """A surface spanning -3e4 ... +3e4 along x: the frame straddles zero, so x - lo rounds."""
    rng = np.random.default_rng(seed)
    x = rng.random(n) * 6e4 - 3e4
    y = rng.random(n) * 20
    z = 3.0 * np.sin(x / 40) + 0.5 * np.cos(y / 3)
    return np.column_stack([x, y, z]).astype(np.float32), np.sqrt(6e4 * 20 / n)


def object_far_out(seed=103):
    """20 k points inside 2 cm at (500, 500, 0) plus 100 k sparse points across a 1 km map."""
    rng = np.random.default_rng(seed)
    obj = np.array([500.0, 500.0, 0.0]) + (rng.random((20_000, 3)) - 0.5) * 0.02
    xy = rng.random((100_000, 2)) * 1000
    mp = np.column_stack([xy, 5.0 * np.sin(xy[:, 0] / 50) * np.cos(xy[:, 1] / 70)])
    p = np.concatenate([mp, obj])[rng.permutation(120_000)]
    return p.astype(np.float32), 1000 / np.sqrt(100_000)


def outlier_frame(n=100_000, seed=104):
    """100 k points in a 1 m cube plus one point 1e6 away: the frame's finest cells are ~0.5 m, so runs of equal
    Morton codes far exceed a leaf, and only a handful of cells are occupied at any level."""
    rng = np.random.default_rng(seed)
    p = rng.random((n + 1, 3))
    p[n // 2] = [1e6, 0.5, 0.5]
    return p.astype(np.float32), n ** (-1 / 3)


def flat_far(n=100_000, seed=105):
    """The plane z = 1e4 exactly: one axis of the frame has zero extent."""
    rng = np.random.default_rng(seed)
    xy = rng.random((n, 2)) * 100 - 50
    return np.column_stack([xy, np.full(n, 1e4)]).astype(np.float32), 100 / np.sqrt(n)


def lattice_far(seed=106):
    """The 13^3 integer lattice shifted by 1e4, plus exact duplicates: 150 points 12 times, 3 points 91 times (more
    copies than a leaf holds, and more than k + 8 for every k checked)."""
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(*[np.arange(13.0)] * 3, indexing="ij"), -1).reshape(-1, 3) + 1e4
    extra = [np.repeat(g[rng.choice(g.shape[0], 150, replace=False)], 11, axis=0),
             np.repeat(g[rng.choice(g.shape[0], 3, replace=False)], 90, axis=0)]
    p = np.concatenate([g] + extra)
    return p[rng.permutation(p.shape[0])].astype(np.float32), 1.0


SCENES = {"map_1e5": map_1e5, "straddle": straddle, "object_far_out": object_far_out, "outlier_frame": outlier_frame,
          "flat_far": flat_far, "lattice_far": lattice_far}
TIE_SCENES = ("map_1e5", "lattice_far")


def morton_frame(pts):
    """lo (3,) and morton_scale as the index build forms them (lbvh.cu, morton_sort): float32 throughout."""
    p = pts[np.isfinite(pts).all(1)].astype(np.float32)
    lo, hi = p.min(0), p.max(0)
    ext = np.float32(max(np.float32(hi[d] - lo[d]) for d in range(3)))
    scale = np.float32(np.float32(2097152.0) / ext) if ext > 0 else np.float32(1.0)
    if not np.isfinite(scale):
        scale = np.float32(1.0)
    return lo, hi, scale


def make_queries(name, pts, spacing, n_jitter=20_000, n_boundary=8_000, n_beyond=600, seed=7):
    """Every point; jittered copies; points exactly on fp32 cell boundaries lo + K / scale of random levels (and one ulp
    either side); points beyond the frame on all six sides (the cells clamp there); NaN queries.  (nq, 3) float32 and
    the slices of each kind."""
    rng = np.random.default_rng(seed)
    n = pts.shape[0]
    parts = {"points": pts}
    j = pts[rng.integers(0, n, n_jitter)].astype(np.float64) + rng.normal(0, 0.5 * spacing, (n_jitter, 3))
    if name == "lattice_far":
        # cell centres, faces and edges of the lattice: 2-, 4- and 8-way ties
        j[::2] = np.round(j[::2] * 2) / 2
        # outside the lattice with x = z: lattice points mirrored across x = z tie exactly, but their fp32 d2 (>= 18,
        # where squares of 2^-10-grid differences no longer fit a float) add the same squares in another order and
        # round apart
        m = j[1::4]
        m[:, 0] = 1e4 - 3 - 10 * rng.random(m.shape[0])
        m[:, 1] = 1e4 + 12 * rng.random(m.shape[0])
        m[:, 2] = m[:, 0]
        j[1::4] = m
    parts["jittered"] = j.astype(np.float32)
    lo, hi, scale = morton_frame(pts)
    inv = np.float32(np.float32(1.0) / scale)
    b = pts[rng.integers(0, n, n_boundary)].copy()
    level = rng.integers(1, 22, n_boundary)
    step = (1 << (21 - level)).astype(np.float64)
    for d in range(3):
        snap = rng.random(n_boundary) < 0.6
        c = np.float64(np.float32((b[:, d] - lo[d])) * scale)
        K = np.clip(np.round(c / step) * step, 0, 2097152).astype(np.float32)
        x = (lo[d] + (K * inv).astype(np.float32)).astype(np.float32)
        side = rng.integers(-1, 2, n_boundary)
        x = np.where(side < 0, np.nextafter(x, np.float32(-np.inf)), np.where(side > 0, np.nextafter(x, np.float32(np.inf)), x))
        b[:, d] = np.where(snap, x, b[:, d])
    parts["boundary"] = b.astype(np.float32)
    e = pts[rng.integers(0, n, n_beyond)].astype(np.float64)
    axis, up = rng.integers(0, 3, n_beyond), rng.random(n_beyond) < 0.5
    off = spacing * (1 + 49 * rng.random(n_beyond))
    r = np.arange(n_beyond)
    e[r, axis] = np.where(up, hi[axis].astype(np.float64) + off, lo[axis].astype(np.float64) - off)
    parts["beyond"] = e.astype(np.float32)
    nan = pts[:7].copy()
    nan[[0, 1, 2], [0, 1, 2]] = np.nan
    nan[3] = np.nan
    nan[4, 0], nan[5, 1], nan[6, 2] = np.inf, -np.inf, np.nan
    parts["nan"] = nan
    q = np.concatenate(list(parts.values()))
    slices, a = {}, 0
    for key, v in parts.items():
        slices[key] = slice(a, a + v.shape[0])
        a += v.shape[0]
    return q, slices


def xyz1(a):
    out = np.ones((a.shape[0], 4), dtype=np.float32)
    out[:, :3] = a[:, :3]
    return out


class Scene:
    """One scene, its queries and the reference k-NN lists at K_MAX (computed once)."""

    def __init__(self, name):
        self.name = name
        pts, self.spacing = SCENES[name]()
        self.cloud = xyz1(pts)
        q, self.slices = make_queries(name, pts, self.spacing)
        self.q = xyz1(q)
        self.n_valid = int(np.isfinite(pts).all(1).sum())
        self.idx, self.d2 = knn_sets(self.cloud, self.q, K_MAX, return_d2=True)

    def knn(self, k):
        """Reference (idx int32, d2) at k <= K_MAX; -1 / +inf past the number of finite points."""
        assert k <= K_MAX
        return self.idx[:, :k].astype(np.int32), self.d2[:, :k]

    def radii(self):
        """Radii whose balls hold ~1, ~20 and ~300 points around the points of the scene."""
        pts = self.cloud[:, :3]
        rng = np.random.default_rng(3)
        s = pts[rng.choice(pts.shape[0], 2000, replace=False)]
        _, d2 = knn_sets(self.cloud, s, 300, return_d2=True)
        r = [0.5 * float(np.sqrt(np.median(self.d2[self.slices["points"], 1]))),
             float(np.sqrt(np.median(d2[:, 19]))), float(np.sqrt(np.median(d2[:, 299])))]
        return [max(x, 1e-3) for x in r]

    def radius_queries(self, r, budget=3_000_000):
        """The queries of a radius check at r: all of them where the balls hold <= budget points in all; otherwise
        a seeded random selection that fits the budget, plus every non-finite query (a dense object inside a sparse
        map puts ~20 k points in the map-scale balls of its 20 k points)."""
        from scipy.spatial import cKDTree
        fin = np.isfinite(self.q[:, :3]).all(1)
        tree = cKDTree(self.cloud[:, :3].astype(np.float64))
        cnt = np.zeros(self.q.shape[0], np.int64)
        cnt[fin] = tree.query_ball_point(self.q[fin, :3].astype(np.float64), r, return_length=True, workers=-1)
        if cnt.sum() <= budget:
            return self.q
        order = np.random.default_rng(9).permutation(self.q.shape[0])
        keep = order[np.cumsum(cnt[order]) <= budget]
        return self.q[np.sort(np.concatenate([keep, np.nonzero(~fin)[0]]))]


def knn_stats_ref(idx, d2, k, n_valid):
    """(mean, kth) of KdTreeFLANN-based StatisticalOutlierRemoval's first pass from the reference lists at >= k."""
    cnt = min(k, n_valid)
    nq = idx.shape[0]
    fin = idx[:, 0] >= 0
    s = np.zeros(nq)
    for j in range(1, cnt):
        s = s + np.sqrt(d2[:, j].astype(np.float64))
    mean = (s / (cnt - 1)).astype(np.float32) if cnt > 1 else np.zeros(nq, np.float32)
    kth = d2[:, k - 1].copy() if cnt == k else np.full(nq, np.inf, np.float32)
    mean[~fin] = 0
    kth[~fin] = np.inf
    return mean, kth


def corr_ref(nn, nn_d2, max_distance=NO_GATE, indices=None, back=None):
    """Correspondence list from the reference 1-NN of the source rows (nn, nn_d2: (n,) over every source row); indices
    selects the rows; back = (nearest source index, its d2) of every kept match's target point for the reciprocal
    variant, as a function of the match indices."""
    rows = np.arange(nn.size) if indices is None else np.asarray(indices, dtype=np.int64)
    m, d = nn[rows], nn_d2[rows]
    md2 = float(max_distance) * float(max_distance)
    keep = (m >= 0) & ~(d.astype(np.float64) > md2)
    if back is not None:
        bi, bd = back(m[keep])
        k2 = ~(bd.astype(np.float64) > md2) & (bi == rows[keep])
        keep[np.nonzero(keep)[0][~k2]] = False
    out = np.empty(int(keep.sum()), dtype=CORR_DTYPE)
    out["index_query"], out["index_match"], out["distance"] = rows[keep], m[keep], d[keep]
    return out


def reciprocal_back(src_cloud, tgt_cloud):
    def back(matches):
        i, d = knn_sets(src_cloud, tgt_cloud[matches], 1, return_d2=True)
        return i[:, 0], d[:, 0]
    return back


def csr_rows_equal(a, b):
    """(offsets, idx, d2) equal bit for bit; the first differing row otherwise."""
    if not np.array_equal(a[0], b[0]):
        return False, int(np.nonzero(a[0] != b[0])[0][0]) - 1
    for x, y in zip(a[1:], b[1:]):
        if not np.array_equal(x, y):
            i = int(np.nonzero(x != y)[0][0])
            return False, int(np.searchsorted(a[0], i, side="right")) - 1
    return True, -1


def first_bad_rows(got, want):
    return np.nonzero((np.asarray(got) != np.asarray(want)).reshape(len(want), -1).any(1))[0]


# ---------------------------------------------------------------------------------------------------------------------
# CPU tests: the oracle against the reference, and the scenes' teeth
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SCENES))
def test_oracle_lists_equal_the_reference(orc, name):
    """On every scene and every query kind: the oracle's k-NN (indices and d2), radius lists (with and without
    max_nn), correspondences (plain, gated, an index subset, reciprocal) and knn_stats equal the reference bit for
    bit."""
    S = Scene(name)
    nt = os.cpu_count() or 8
    oidx = orc.Index(S.cloud)
    assert oidx.size == S.n_valid
    # the oracle's nearestKSearch, like FLANN's, does not screen its queries: its rows for non-finite queries are not
    # defined (the device's are empty, tests/test_gpu_search_reference.py)
    fin = np.isfinite(S.q[:, :3]).all(1)
    for k in (1, 5, 16, K_MAX):
        oi, od, ok = oidx.knn(S.q[fin], k, nthreads=nt)
        ri, rd = S.knn(k)
        ri, rd = ri[fin], rd[fin]
        assert ok == min(k, S.n_valid)
        bad = first_bad_rows(np.concatenate([oi, od.view(np.int32)], 1), np.concatenate([ri, rd.view(np.int32)], 1))
        assert bad.size == 0, (name, k, bad.size, bad[:5].tolist(), oi[bad[:2]].tolist(), ri[bad[:2]].tolist())
    for r in S.radii():
        q = S.radius_queries(r)
        for max_nn in (0, 10):
            got = oidx.radius(q, r, max_nn=max_nn, nthreads=nt)
            ok, row = csr_rows_equal(got, radius_csr(S.cloud, q, r, max_nn=max_nn))
            assert ok, (name, r, max_nn, row)
    nn, nd = S.idx[:, 0], S.d2[:, 0]
    src = S.q
    for md in (NO_GATE, 3 * S.spacing, 0.3 * S.spacing):
        got = oidx.correspondences(src, max_distance=md, is_dense=False, nthreads=nt)
        want = corr_ref(nn, nd, md)
        assert np.array_equal(got, want), (name, md, got.size, want.size)
    ind = np.random.default_rng(5).permutation(src.shape[0])[:20_000].astype(np.int32)
    assert np.array_equal(oidx.correspondences(src, max_distance=S.spacing, indices=ind, is_dense=False, nthreads=nt),
                          corr_ref(nn, nd, S.spacing, indices=ind)), name
    got = oidx.correspondences_reciprocal(src, orc.Index(src), max_distance=3 * S.spacing, is_dense=False, nthreads=nt)
    want = corr_ref(nn, nd, 3 * S.spacing, back=reciprocal_back(src, S.cloud))
    assert want.size > 0 and np.array_equal(got, want), (name, got.size, want.size)
    for k in (2, 16, 51):
        om, ok_ = oidx.knn_stats(S.q, k, nthreads=nt)
        rm, rk = knn_stats_ref(S.idx, S.d2, k, S.n_valid)
        assert np.array_equal(om.view(np.int32), rm.view(np.int32)), (name, k, first_bad_rows(om, rm)[:5].tolist())
        assert np.array_equal(ok_.view(np.int32), rk.view(np.int32)), (name, k)


@pytest.mark.parametrize("name", TIE_SCENES)
def test_the_scenes_have_teeth(name):
    """The tie scenes really decide lists by the (d2, index) order and by fp32 rounding: swapping the tie order to
    (d2, -index) changes at least 1 % of the rows at K_MAX, and computing d2 in fp64 changes at least one row."""
    pts, spacing = SCENES[name]()
    cloud = xyz1(pts)
    q, _ = make_queries(name, pts, spacing)
    ref = knn_sets(cloud, q, K_MAX)
    swapped = knn_sets(cloud, q, K_MAX, tie=-1)
    fp64 = knn_sets(cloud, q, K_MAX, dist=d2_fp64)
    fin = np.isfinite(q).all(1)
    share = float(np.mean((ref != swapped).any(1)[fin]))
    n64 = int((ref != fp64).any(1).sum())
    print(f"teeth {name:12s}: (d2, -index) changes {100 * share:.2f} % of the rows, fp64 d2 changes {n64} rows")
    assert share >= 0.01, (name, share)
    assert n64 > 0, name
