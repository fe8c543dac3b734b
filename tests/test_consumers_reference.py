"""The operators built on the neighbour lists against a plain reference on map-scale frames (CPU part).

Each reference restates one operator in numpy, in the library's arithmetic, over the scenes of
tests/test_search_reference.py (their K_MAX reference k-NN lists included):

* VoxelGrid (voxel_grid.hpp:596-814, voxel.cu): min / max over the finite points; the guard
  int64((max - min) * inv) + 1 per axis in float, product > INT32_MAX -> no output (ERR_LEAF_TOO_SMALL on the device);
  inv = float(1 / leaf); min_b = floor(min * inv), div_b = floor(max * inv) - min_b + 1, both in float; the key
  int32(floor(x * inv) - float(min_b)) . (1, div_b0, div_b0 div_b1) with int32 wrap-around; a stable sort by key; runs
  shorter than min_points_per_voxel dropped; the centroid a sequential fp32 sum in input order, then one fp32 division.
  With normals (downsample_all_data_): the 4-vector normal sum in the same order, divided by its fp32 norm
  ((x x + y y) + (z z + w w)) unless that is 0, and the curvature sum / count.  A tile uses the whole cloud's min / max.
* Euclidean clusters (extract_clusters.hpp:124-223, cluster.cu:25-28): connected components of the graph with an edge
  wherever the fp32 d2 < float(double(float(tol))^2); label = smallest original index of the component, -1 for
  non-finite points and points outside the subset.
* Normal shooting (correspondence_estimation_normal_shooting.hpp:99-127, corr_select.cuh): over the k reference
  candidates, V = fp32 (target - source), then ((Cx^2 + Cy^2) + Cz^2) of the fp64 cross product N x V; the first strict
  minimum wins (start DBL_MAX); the row is dropped when that minimum > max_distance itself.
* Back projection (correspondence_estimation_backprojection.hpp:91-114): cos = fp32 ((n0 m0 + n1 m1) + n2 m2), score
  fp32 d2 (2 - cos^2), first strict minimum from FLT_MAX, dropped when double(score) > max_distance.  Both store the
  chosen candidate's d2; non-finite source points give no row; when no score compares (NaN normals) the first
  neighbour is taken with the start value as its score (pcl_oracle.cpp:1477-1479).
* Surface-normal rejector (correspondence_rejection.h:378-389): fp32 ((ax bx + ay by) + az bz), kept when
  double(dot) > threshold.
* Fitness, validation, inliers: the source transformed in the order its function uses (APPLY below), the reference
  1-NN d2 of each moved point; getFitnessScore / validateTransformation = the mean of the d2 <= max_range (count
  exact, mean within count 2^-52 relative of math.fsum); SampleConsensusPrerejective's inliers = the rows with
  d2 < float(thr)^2 (strict, float), fitness = their sequential fp32 sum / count.

The oracle is held to every reference here; the device is held to the same references in
tests/test_gpu_consumers_reference.py.  The teeth tests show that the scenes decide each rule: perturbing it changes
rows."""
import math
import os
import sys
import time

import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components
from scipy.spatial import cKDTree

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_search_reference as R  # noqa: E402
from test_normals_reference import d2_fp32, knn_sets  # noqa: E402

CORR_DTYPE = R.CORR_DTYPE
INT32_MAX = 2 ** 31 - 1
DBL_MAX = float(np.finfo(np.float64).max)
FLT_MAX = np.float32(np.finfo(np.float32).max)
CORR_K = (1, 3, 10, 16, 40)
SCENE_CACHE = {}


def scene(name):
    """One R.Scene per name and process: its reference k-NN lists are the expensive part."""
    if name not in SCENE_CACHE:
        SCENE_CACHE.clear()
        SCENE_CACHE[name] = R.Scene(name)
    return SCENE_CACHE[name]


def point_normal(xyz, normals=None, curvature=None):
    """(n, 12) pcl::PointNormal rows: x y z 1 | nx ny nz 0 | curvature 0 0 0."""
    out = np.zeros((xyz.shape[0], 12), np.float32)
    out[:, :3] = xyz[:, :3]
    out[:, 3] = 1
    if normals is not None:
        out[:, 4:4 + normals.shape[1]] = normals
    if curvature is not None:
        out[:, 8] = curvature
    return out


# ---------------------------------------------------------------------------------------------------------------------
# VoxelGrid
# ---------------------------------------------------------------------------------------------------------------------
def voxel_leaves(name, spacing):
    """The leaves of a scene: 0.7, 3 and 20 times the point spacing, plus the leaves where the key's rounding decides."""
    leaves = [0.7 * spacing, 3 * spacing, 20 * spacing]
    if name == "map_1e5":
        leaves += [1 / 16, 0.1]   # x * 16 exact, every point on a face; 1 / 0.1 inexact
    if name == "lattice_far":
        leaves += [1.0, 0.5]      # lattice points on faces
    return leaves


def voxel_grid(xyz, leaf, bounds=None):
    """(inv, min_b, mul) of the finite rows xyz, or None where the guard fires; bounds = (lo, hi) of the whole cloud."""
    inv = (np.float32(1) / np.broadcast_to(np.asarray(leaf, np.float32), (3,))).astype(np.float32)
    lo, hi = (xyz.min(0), xyz.max(0)) if bounds is None else bounds
    ext = ((hi - lo).astype(np.float32) * inv).astype(np.float32)
    if math.prod(int(e) + 1 for e in ext) > INT32_MAX:
        return None
    min_b = np.floor(lo * inv).astype(np.int64)
    div = np.floor(hi * inv).astype(np.int64) - min_b + 1
    mul = np.array([1, div[0], div[0] * div[1]], np.int64).astype(np.int32)  # int32 products wrap as in C
    return inv, min_b, mul


def voxel_keys(xyz, inv, min_b, mul, fp64=False):
    """uint32 key of every row: int(floor(x * inv) - float(min_b)) . mul, in float (fp64: the rule it must not be)."""
    if fp64:
        ijk = (np.floor(xyz.astype(np.float64) * inv.astype(np.float64)) - min_b).astype(np.int64)
    else:
        ijk = (np.floor((xyz * inv).astype(np.float32)) - min_b.astype(np.float32)).astype(np.int64)
    key = (ijk.astype(np.int32) * mul).astype(np.int32)
    return (key[:, 0] + key[:, 1] + key[:, 2]).astype(np.int32).view(np.uint32)


def sequential_sums(vals, order, starts, ends, fp64=False, reverse=False):
    """Sum of vals[order[b:e]] for every run, one fp32 addition after the other in run order (vectorised over runs)."""
    lens = ends - starts
    by_len = np.argsort(-lens, kind="stable")
    dt = np.float64 if fp64 else np.float32
    acc = np.zeros((starts.size, vals.shape[1]), dt)
    for t in range(int(lens.max()) if lens.size else 0):
        act = by_len[: int(np.searchsorted(-lens[by_len], -t, side="left"))]
        pos = ends[act] - 1 - t if reverse else starts[act] + t
        acc[act] = (acc[act] + vals[order[pos]].astype(dt)).astype(dt)
    return acc.astype(np.float32)


def voxel_ref(cloud, leaf, min_pts=0, indices=None, normal=False, bounds=None, fp64_key=False, fp64_sum=False,
              reverse=False):
    """VoxelGrid::applyFilter: (centroids (m, 4), normal / curvature rows (m, 8) or None), or None where the guard
    fires.  normal: the rows are PointNormal records (normal at float 4, curvature at float 8)."""
    rows = np.arange(cloud.shape[0]) if indices is None else np.asarray(indices, np.int64)
    xyz = cloud[rows, :3].astype(np.float32)
    fin = np.isfinite(xyz).all(1)
    rows, xyz = rows[fin], xyz[fin]
    if rows.size == 0:
        return np.zeros((0, 4), np.float32), (np.zeros((0, 8), np.float32) if normal else None)
    grid = voxel_grid(xyz, leaf, bounds)
    if grid is None:
        return None
    key = voxel_keys(xyz, *grid, fp64=fp64_key)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    starts = np.nonzero(np.r_[True, ks[1:] != ks[:-1]])[0]
    ends = np.r_[starts[1:], ks.size]
    keep = ends - starts >= min_pts
    starts, ends = starts[keep], ends[keep]
    fn = (ends - starts).astype(np.float32)[:, None]
    out = np.ones((starts.size, 4), np.float32)
    out[:, :3] = sequential_sums(xyz, order, starts, ends, fp64_sum, reverse) / fn
    if not normal:
        return out, None
    nc = np.zeros((starts.size, 8), np.float32)
    s = sequential_sums(cloud[rows, 4:9].astype(np.float32), order, starts, ends, fp64_sum, reverse)
    n4 = s[:, :4]
    sq = ((n4[:, 0] * n4[:, 0] + n4[:, 1] * n4[:, 1]) + (n4[:, 2] * n4[:, 2] + n4[:, 3] * n4[:, 3])).astype(np.float32)
    nrm = np.sqrt(sq)
    nc[:, :4] = np.where((sq > 0)[:, None], n4 / np.where(sq > 0, nrm, 1)[:, None], n4)
    nc[:, 4] = s[:, 4] / fn[:, 0]
    return out, nc


def voxel_tiles(cloud, leaf, n_tiles=3):
    """Row sets of tiles cut along voxel faces of the whole cloud's grid (in the reference's float arithmetic), and the
    whole cloud's bounds.  The cuts run across the slowest axis of the key that has more than one layer, in ascending
    order, so the tiles' VoxelGrids on the whole grid concatenate to the whole's."""
    xyz = cloud[:, :3].astype(np.float32)
    fin = np.nonzero(np.isfinite(xyz).all(1))[0]
    lo, hi = xyz[fin].min(0), xyz[fin].max(0)
    inv, min_b, mul = voxel_grid(xyz[fin], leaf)
    ijk = (np.floor((xyz[fin] * inv).astype(np.float32)) - min_b.astype(np.float32)).astype(np.int64)
    layered = [a for a in range(3) if ijk[:, a].max() > 0]
    if not layered:
        return [fin], (lo, hi)
    k = ijk[:, layered[-1]]
    cuts = np.unique(np.quantile(k, np.linspace(0, 1, n_tiles + 1)[1:-1]).astype(np.int64))
    tile = np.searchsorted(cuts, k, side="right")
    return [fin[tile == t] for t in range(cuts.size + 1) if (tile == t).any()], (lo, hi)


def with_nan_rows(cloud, every=997):
    c = cloud.copy()
    c[::every, 0] = np.nan
    c[5::every, 1] = np.inf
    c[9::every, :3] = np.nan
    return c


def voxel_cases(name, S):
    """(label, cloud, leaf, min_pts, indices) of every VoxelGrid check of a scene."""
    rng = np.random.default_rng(31)
    n = S.cloud.shape[0]
    sub = np.sort(rng.permutation(n)[: n // 2]).astype(np.int32)
    nan = with_nan_rows(S.cloud)
    out = []
    for leaf in voxel_leaves(name, S.spacing):
        for mp in (0, 3):
            out.append((f"leaf {leaf:.4g} min {mp}", S.cloud, leaf, mp, None))
        out.append((f"leaf {leaf:.4g} subset", S.cloud, leaf, 0, sub))
        out.append((f"leaf {leaf:.4g} nan", nan, leaf, 2, None))
    return out


def voxel_normal_cloud(S):
    """PointNormal records of a scene: unit-ish normals, a non-zero fourth component on some rows, a few opposite normals
    (zero sums), curvature."""
    rng = np.random.default_rng(37)
    n = S.cloud.shape[0]
    nv = rng.normal(size=(n, 3)).astype(np.float32)
    nv /= np.linalg.norm(nv, axis=1, keepdims=True)
    pn = point_normal(S.cloud, nv, rng.random(n).astype(np.float32))
    pn[::13, 7] = np.float32(0.25)
    return pn


def equal_rows(got, want):
    """(equal, first differing row) of two float arrays, bit for bit."""
    if got.shape != want.shape:
        return False, -1
    bad = np.nonzero((got.view(np.int32) != want.view(np.int32)).reshape(got.shape[0], -1).any(1))[0] if got.size else []
    return len(bad) == 0, int(bad[0]) if len(bad) else -1


# ---------------------------------------------------------------------------------------------------------------------
# Euclidean clusters
# ---------------------------------------------------------------------------------------------------------------------
def _edges_fp32(P, a, b, r2, le):
    d2 = d2_fp32(P[a], P[b][:, None, :])[:, 0]
    k = (d2 <= r2) if le else (d2 < r2)
    return a[k], b[k]


def cluster_ref(cloud, tol, subset=None, le=False, dense=2000, budget=4_000_000):
    """Labels of the connected components of fp32 d2 < float(double(float(tol))^2) (le: <=).  Edges are enumerated
    from the points whose ball holds at most `dense` points, in chunks of at most `budget`, keeping only a spanning
    forest between chunks.  The denser points are grouped into cells of diagonal < tol (all pairs in a cell are edges)
    and the cells are joined by their closest pairs, with every pair of the rounding band checked in fp32."""
    xyz = np.asarray(cloud, np.float32)[:, :3]
    ok = np.isfinite(xyz).all(1)
    if subset is not None:
        m = np.zeros(ok.size, bool)
        m[np.asarray(subset)] = True
        ok &= m
    ids = np.nonzero(ok)[0]
    labels = np.full(xyz.shape[0], -1, np.int32)
    if ids.size == 0:
        return labels
    P = xyz[ids]
    m = ids.size
    tolf = float(np.float32(tol))
    r2 = np.float32(tolf * tolf)
    hi_r, lo_r = tolf * (1 + 1e-5), tolf * (1 - 1e-5)   # fp32 d2 and float(tol^2) are within 1e-6 of the exact values
    tree = cKDTree(P.astype(np.float64))
    cnt = tree.query_ball_point(P.astype(np.float64), hi_r, return_length=True, workers=-1)
    forest = (np.zeros(0, np.int64), np.zeros(0, np.int64))

    def merge(ea, eb):
        nonlocal forest
        a = np.concatenate([forest[0], ea])
        b = np.concatenate([forest[1], eb])
        _, lab = connected_components(coo_matrix((np.ones(a.size, np.int8), (a, b)), shape=(m, m)), directed=False)
        first = np.full(m, m, np.int64)
        np.minimum.at(first, lab, np.arange(m))
        nz = np.nonzero(first[lab] != np.arange(m))[0]
        forest = (nz, first[lab[nz]])
        return lab

    sparse = np.nonzero(cnt <= dense)[0]
    pend_a, pend_b, pend = [], [], 0
    step = max(1, budget // max(1, int(cnt[sparse].max()) if sparse.size else 1))
    for s0 in range(0, sparse.size, step):
        rows = sparse[s0:s0 + step]
        lists = tree.query_ball_point(P[rows].astype(np.float64), hi_r, workers=-1, return_sorted=False)
        lens = np.fromiter((len(x) for x in lists), np.int64, count=len(lists))
        a = np.repeat(rows, lens)
        b = np.concatenate([np.asarray(x, np.int64) for x in lists]) if lens.sum() else np.zeros(0, np.int64)
        a, b = _edges_fp32(P, a[a != b], b[a != b], r2, le)
        pend_a.append(a)
        pend_b.append(b)
        pend += a.size
        if pend > budget:
            merge(np.concatenate(pend_a), np.concatenate(pend_b))
            pend_a, pend_b, pend = [], [], 0
    dpts = np.nonzero(cnt > dense)[0]
    ea, eb = [np.concatenate(pend_a) if pend_a else np.zeros(0, np.int64)], [np.concatenate(pend_b) if pend_b else np.zeros(0, np.int64)]
    if dpts.size:
        side = lo_r / math.sqrt(3)
        cell = np.floor(P[dpts].astype(np.float64) / side).astype(np.int64)
        ucell, inv = np.unique(cell, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        assert ucell.shape[0] <= 4000, ucell.shape   # the cell pairs below are a Python loop
        members = [dpts[inv == c] for c in range(ucell.shape[0])]
        for mem in members:                          # a cell is a clique
            ea.append(mem[1:])
            eb.append(np.full(mem.size - 1, mem[0]))
        croot = list(range(len(members)))

        def find(c):
            while croot[c] != c:
                croot[c] = croot[croot[c]]
                c = croot[c]
            return c
        ctrees = [cKDTree(P[mem].astype(np.float64)) for mem in members]
        for i in range(len(members)):
            near = np.nonzero((np.abs(ucell - ucell[i]) <= 2).all(1))[0]
            for j in near[near > i]:
                if find(i) == find(j):
                    continue
                dmin, _ = ctrees[j].query(P[members[i]].astype(np.float64), 1)
                if dmin.min() >= hi_r:
                    continue
                lists = ctrees[j].query_ball_point(P[members[i]].astype(np.float64), hi_r)
                lens = np.fromiter((len(x) for x in lists), np.int64, count=len(lists))
                a = np.repeat(members[i], lens)
                b = members[j][np.concatenate([np.asarray(x, np.int64) for x in lists])]
                a, b = _edges_fp32(P, a, b, r2, le)
                if a.size:
                    ea.append(a[:1])
                    eb.append(b[:1])
                    croot[find(i)] = find(j)
    lab = merge(np.concatenate(ea), np.concatenate(eb))
    first = np.full(m, np.iinfo(np.int64).max, np.int64)
    np.minimum.at(first, lab, ids)
    labels[ids] = first[lab].astype(np.int32)
    return labels


def clusters_ref(labels, min_size=1, max_size=2 ** 32 - 1):
    """EuclideanClusterExtraction::extract from labels (extract_clusters.hpp:196, 208, 249): each cluster's indices
    ascending, clusters by size descending, equal sizes by their smallest index, sizes outside the window dropped."""
    groups = {}
    for i, lab in enumerate(np.asarray(labels).tolist()):
        if lab >= 0:
            groups.setdefault(lab, []).append(i)
    out = [np.asarray(g, np.int32) for g in groups.values() if min_size <= len(g) <= max_size]
    return sorted(out, key=lambda g: (-g.size, int(g[0])))


def tie_tolerance(S):
    """A tolerance whose float square is a squared distance of the scene (a 1-NN d2 near (0.8 spacing)^2)."""
    d2 = np.unique(S.d2[S.slices["points"], 1])
    for v in d2[d2 >= np.float32((0.8 * S.spacing) ** 2)]:
        t = float(np.sqrt(np.float64(v)))
        for c in (t, float(np.nextafter(np.float32(t), np.float32(np.inf))), float(np.nextafter(np.float32(t), np.float32(0)))):
            tf = float(np.float32(c))
            if np.float32(tf * tf) == v:
                return tf
    raise AssertionError("no tie tolerance")


def cluster_tolerances(name, S):
    tols = [0.5 * S.spacing, 1.2 * S.spacing]
    if name == "map_1e5":
        t = tie_tolerance(S)
        tols += [t, float(np.nextafter(np.float32(t), np.float32(np.inf)))]
    if name == "lattice_far":
        tols += [1.0, 1.0001, 1.5]
    return tols


def cluster_subset(n):
    return np.sort(np.random.default_rng(41).permutation(n)[: (3 * n) // 4]).astype(np.int32)


# ---------------------------------------------------------------------------------------------------------------------
# normal-based correspondences and the surface-normal rejector
# ---------------------------------------------------------------------------------------------------------------------
def mixed_normals(normals, seed):
    """Estimated normals with every 9th row a random unit vector, every 53rd NaN and every 61st zero."""
    rng = np.random.default_rng(seed)
    n = normals[:, :3].astype(np.float32).copy()
    r = rng.normal(size=(n.shape[0], 3))
    n[::9] = (r / np.linalg.norm(r, axis=1, keepdims=True)).astype(np.float32)[::9]
    n[4::53] = np.nan
    n[7::61] = 0
    return np.ascontiguousarray(n)


def scene_normals(S, orc):
    """(source normals of S.q, target normals of S.cloud): the oracle's k = 10 normals of the cloud, mixed."""
    o = orc.Index(S.cloud)
    tn, _ = o.normals_knn(S.cloud, 10, nthreads=os.cpu_count() or 8)
    sn, _ = o.normals_knn(S.q, 10, nthreads=os.cpu_count() or 8)
    return mixed_normals(sn, 43), mixed_normals(tn, 47)


def corr_gates(S):
    return (R.NO_GATE, 3 * S.spacing ** 2, 1e-4 * S.spacing ** 2)


def normals_corr_ref(kind, src, sn, tgt, tn, idx, d2, k, max_distance=R.NO_GATE, indices=None, last=False,
                     fp64_diff=False):
    """Correspondence list of normal shooting (kind 1) or back projection (kind 2) from the reference k-NN lists
    (idx, d2: (n_src, >= k), -1 past the finite points) of every source row.  last: the last minimum wins;
    fp64_diff: target - source in fp64 (the rules the scenes must tell from the real ones)."""
    rows = np.arange(src.shape[0]) if indices is None else np.asarray(indices, np.int64)
    p = src[rows, :3].astype(np.float32)
    ok = np.isfinite(p).all(1) & (idx[rows, 0] >= 0)
    rows, p = rows[ok], p[ok]
    ci, cd = idx[rows, :k], d2[rows, :k]
    valid = ci >= 0
    safe = np.where(valid, ci, 0)
    n = sn[rows, :3].astype(np.float32)
    if kind == 1:
        q = tgt[safe, :3]
        V = (q.astype(np.float64) - p[:, None, :].astype(np.float64)) if fp64_diff else \
            (q.astype(np.float32) - p[:, None, :]).astype(np.float32).astype(np.float64)
        N = n.astype(np.float64)[:, None, :]
        Cx = N[..., 1] * V[..., 2] - N[..., 2] * V[..., 1]
        Cy = N[..., 2] * V[..., 0] - N[..., 0] * V[..., 2]
        Cz = N[..., 0] * V[..., 1] - N[..., 1] * V[..., 0]
        score = (Cx * Cx + Cy * Cy) + Cz * Cz
        start = DBL_MAX
    else:
        m = tn[safe, :3].astype(np.float32)
        cos = ((n[:, None, 0] * m[..., 0] + n[:, None, 1] * m[..., 1]) + n[:, None, 2] * m[..., 2]).astype(np.float32)
        score = (cd * (np.float32(2) - cos * cos)).astype(np.float32)
        start = FLT_MAX
    s = np.where(valid & ~np.isnan(score) & (score < start), score, np.inf)
    j = (k - 1 - np.argmin(s[:, ::-1], 1)) if last else np.argmin(s, 1)
    best = s[np.arange(rows.size), j]
    none = ~np.isfinite(best)
    j[none] = 0
    best = np.where(none, start, best).astype(np.float64)
    keep = ~(best > max_distance)
    out = np.empty(int(keep.sum()), CORR_DTYPE)
    out["index_query"] = rows[keep]
    out["index_match"] = ci[keep, j[keep]]
    out["distance"] = cd[keep, j[keep]]
    return out


def surface_normal_ref(corr, sn, tn, threshold):
    a, b = sn[corr["index_query"], :3].astype(np.float32), tn[corr["index_match"], :3].astype(np.float32)
    dot = ((a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]).astype(np.float32)
    return corr[dot.astype(np.float64) > threshold]


def surface_dots(corr, sn, tn):
    a, b = sn[corr["index_query"], :3].astype(np.float32), tn[corr["index_match"], :3].astype(np.float32)
    return ((a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]).astype(np.float32)


def surface_thresholds(dots):
    """0, -1 and dot values that occur in the input (kept only when strictly above)."""
    d = np.sort(dots[np.isfinite(dots)])
    return [0.0, -1.0] + [float(d[int(q * (d.size - 1))]) for q in (0.1, 0.5, 0.9)]


# ---------------------------------------------------------------------------------------------------------------------
# fitness, validation, inliers
# ---------------------------------------------------------------------------------------------------------------------
# the operation order of each consumer (icp_kernels.cuh apply_pending, pcl_oracle.cpp:561-568)
VALIDATION, SSE_FLOAT, TRANSFORMER_DOUBLE = "((T0 x + T1 y) + T2 z) + T3", "T0 x + (T1 y + (T2 z + T3))", \
    "((T3 + x T0) + y T1) + z T2"
APPLY = {"fitness float": (SSE_FLOAT, np.float32), "fitness double": (TRANSFORMER_DOUBLE, np.float64),
         "validation float": (VALIDATION, np.float32), "validation double": (VALIDATION, np.float64),
         "inliers": (SSE_FLOAT, np.float32)}


def apply_T(xyz, T, order, dt):
    """xyz (n, 3) float32 moved by rows 0..2 of T in Scalar dt, in the given operation order, rounded to float."""
    M = np.asarray(T, np.float64).astype(dt)
    x, y, z = (xyz[:, i].astype(dt) for i in range(3))
    out = np.empty_like(xyz, dtype=np.float32)
    for r in range(3):
        a, b, c, d = M[r]
        if order == VALIDATION:
            v = ((a * x + b * y) + c * z) + d
        elif order == SSE_FLOAT:
            v = a * x + (b * y + (c * z + d))
        else:
            v = ((d + x * a) + y * b) + z * c
        out[:, r] = v.astype(dt).astype(np.float32)
    return out


def pose_pair(name, S, orthonormal=True):
    """(source cloud, T): every third point of the scene turned by 1.5 degrees about a point of the map and shifted,
    and a pose close to the inverse motion (not orthonormal when asked)."""
    pts = S.cloud[:, :3]
    fin = np.nonzero(np.isfinite(pts).all(1))[0]
    c = pts[fin[fin.size // 2]].astype(np.float64)
    if name == "object_far_out":
        c = np.array([500.0, 500.0, 0.0])
    a = np.deg2rad(1.5)
    Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    t = np.array([0.4, -0.3, 0.2]) * S.spacing
    src = ((pts[::3].astype(np.float64) - c) @ Rz.T + c + t).astype(np.float32)
    Ri = Rz.T if orthonormal else Rz.T * 0.9999 + 1e-5
    T = np.eye(4)
    T[:3, :3] = Ri
    T[:3, 3] = c - Ri @ (c + t) + np.array([1e-3, -2e-3, 5e-4]) * S.spacing
    return R.xyz1(src), T


def moved_d2(tgt_cloud, src, T, kind):
    """The moved source of a consumer and the reference 1-NN d2 of every moved row (+inf for non-finite rows)."""
    order, dt = APPLY[kind]
    mv = apply_T(src[:, :3], T, order, dt)
    _, d2 = knn_sets(tgt_cloud, mv, 1, return_d2=True)
    return mv, d2[:, 0]


def fitness_ref(d2, max_range):
    """(count, mean) of the d2 <= max_range; DBL_MAX with no such row."""
    keep = np.isfinite(d2) & (d2.astype(np.float64) <= max_range)
    n = int(keep.sum())
    return n, (math.fsum(d2[keep].astype(np.float64).tolist()) / n if n else DBL_MAX)


def fitness_close(got, want, count):
    return got == want if count == 0 else abs(got - want) <= count * 2.0 ** -52 * abs(want)


def fitness_ranges(d2):
    f = d2[np.isfinite(d2)].astype(np.float64)
    return [DBL_MAX, float(np.percentile(f, 60)), float(np.sort(f)[f.size // 3]), 0.0]


def inliers_ref(d2, thr):
    mr = np.float32(np.float32(thr) * np.float32(thr))
    keep = np.nonzero(np.isfinite(d2) & (d2 < mr))[0].astype(np.int32)
    fit = np.float32(0)
    for d in d2[keep]:
        fit = np.float32(fit + d)
    return keep, (float(np.float32(fit / np.float32(keep.size))) if keep.size else float(FLT_MAX))


def inlier_thresholds(d2):
    f = np.sort(d2[np.isfinite(d2)])
    return [float(np.sqrt(f[f.size // 2])), float(np.sqrt(np.float64(f[f.size // 10]))), 1e-9]


# ---------------------------------------------------------------------------------------------------------------------
# CPU tests: the oracle against the references, and the scenes' teeth
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def clock():
    t0 = time.time()
    yield
    print(f" [{time.time() - t0:.1f} s]")


@pytest.mark.parametrize("name", list(R.SCENES))
def test_oracle_voxelgrid_equals_the_reference(orc, name, clock):
    """VoxelGrid and VoxelGrid<PointNormal> at every leaf, min_points_per_voxel 0 and 3, an index subset and NaN
    points: the oracle's centroids (and normals / curvature) equal the reference bit for bit, and its guard fires
    exactly where the reference's does; the tiles of the whole cloud's grid concatenate to the whole."""
    pts, spacing = R.SCENES[name]()
    S = type("S", (), dict(cloud=R.xyz1(pts), spacing=spacing))
    fired = []
    for label, cloud, leaf, mp, ind in voxel_cases(name, S):
        want = voxel_ref(cloud, leaf, mp, ind)
        got = orc.voxelgrid(cloud, [leaf] * 3, mp, indices=ind, is_dense=False)
        if want is None:
            fired.append(label)
            assert got is None, (name, label)
            continue
        ok, row = equal_rows(got, want[0])
        assert ok, (name, label, got.shape, want[0].shape, row)
    pn = voxel_normal_cloud(S)
    for leaf in voxel_leaves(name, spacing):
        want = voxel_ref(pn, leaf, 2, normal=True)
        got = orc.voxelgrid_normals(pn, [leaf] * 3, 2, is_dense=False)
        if want is None:
            assert got is None
            continue
        for g, w in zip(got, want):
            ok, row = equal_rows(g, w)
            assert ok, (name, leaf, row)
        tiles, bounds = voxel_tiles(S.cloud, leaf)
        whole = voxel_ref(S.cloud, leaf)[0]
        cat = np.concatenate([voxel_ref(S.cloud, leaf, indices=t, bounds=bounds)[0] for t in tiles])
        assert equal_rows(cat, whole)[0], (name, leaf, len(tiles))
    print(f"{name}: guard fired on {fired}")
    if name == "outlier_frame":
        assert len(fired) >= 2, fired


@pytest.mark.parametrize("name", ["map_1e5", "straddle", "lattice_far"])
def test_voxelgrid_scenes_have_teeth(name, clock):
    """The key in fp64 moves at least one point on map_1e5 and straddle (exact on the lattice, where it is only
    printed); an fp64 sum or the reversed within-voxel order changes at least one centroid."""
    pts, spacing = R.SCENES[name]()
    cloud = R.xyz1(pts)
    moved, changed = {}, {}
    for leaf in voxel_leaves(name, spacing):
        g = voxel_grid(pts, leaf)
        if g is None:
            continue
        moved[leaf] = int((voxel_keys(pts, *g) != voxel_keys(pts, *g, fp64=True)).sum())
        ref = voxel_ref(cloud, leaf)[0]
        for what, kw in (("fp64 sum", dict(fp64_sum=True)), ("reversed", dict(reverse=True))):
            alt = voxel_ref(cloud, leaf, **kw)[0]
            changed[(leaf, what)] = int((alt.view(np.int32) != ref.view(np.int32)).any(1).sum())
    print(f"teeth {name}: fp64 key moves {moved} points; centroids changed {changed}")
    if name != "lattice_far":
        assert sum(moved.values()) > 0, moved
    assert sum(v for (l, w), v in changed.items() if w == "fp64 sum") > 0, changed
    assert sum(v for (l, w), v in changed.items() if w == "reversed") > 0, changed


@pytest.mark.parametrize("name", list(R.SCENES))
def test_oracle_cluster_labels_equal_the_reference(orc, name, clock):
    """Every label at every tolerance, over the whole cloud and over a subset with NaN points; the ordering and the
    size window of euclidean_clusters restated from the labels."""
    S = scene(name) if name == "map_1e5" else None
    pts, spacing = R.SCENES[name]()
    cloud = R.xyz1(pts)
    if S is None:
        S = type("S", (), dict(cloud=cloud, spacing=spacing))
    import pcl_b200
    nan = with_nan_rows(cloud)
    sub = cluster_subset(cloud.shape[0])
    for tol in cluster_tolerances(name, S):
        want = cluster_ref(cloud, tol)
        got = orc.Index(cloud).cluster_labels(tol)
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, (name, tol, bad.size, bad[:5].tolist())
        for mn, mx in ((1, 2 ** 32 - 1), (2, 50), (5, 10 ** 9)):
            a, b = pcl_b200.clusters_from_labels(want, mn, mx), clusters_ref(want, mn, mx)
            assert len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b)), (name, tol, mn, mx)
        want = cluster_ref(nan, tol, subset=sub)
        got = orc.Index(nan, subset=sub).cluster_labels(tol)
        assert np.array_equal(got, want), (name, tol, "subset + nan")
        print(f"{name} tol {tol:.6g}: {np.unique(want[want >= 0]).size} clusters")


@pytest.mark.parametrize("name", ["map_1e5", "lattice_far"])
def test_cluster_scenes_have_teeth(name, clock):
    """<= in place of < changes labels at both exact-tie tolerances: the map_1e5 one and 1.0 on the lattice."""
    pts, spacing = R.SCENES[name]()
    cloud = R.xyz1(pts)
    tol = tie_tolerance(scene(name)) if name == "map_1e5" else 1.0
    n = int((cluster_ref(cloud, tol) != cluster_ref(cloud, tol, le=True)).sum())
    print(f"teeth {name}: <= at tolerance {tol!r} changes {n} labels")
    assert n > 0


@pytest.mark.parametrize("name", list(R.SCENES))
def test_oracle_normal_correspondences_equal_the_reference(orc, name, clock):
    """Normal shooting and back projection at every k, three gates and an index subset; the surface-normal rejector
    at thresholds that occur in its input."""
    S = scene(name)
    nt = os.cpu_count() or 8
    sn, tn = scene_normals(S, orc)
    src, tgt = point_normal(S.q, sn), point_normal(S.cloud, tn)
    oidx = orc.Index(tgt)
    ind = np.random.default_rng(53).permutation(src.shape[0])[:20_000].astype(np.int32)
    for kind in (1, 2):
        for k in CORR_K:
            for md in corr_gates(S):
                for sel in (None, ind):
                    if sel is not None and md != corr_gates(S)[1]:
                        continue
                    want = normals_corr_ref(kind, S.q, sn, S.cloud, tn, S.idx, S.d2, k, md, sel)
                    got = oidx.correspondences_normals(kind, src, tgt, k=k, max_distance=md, indices=sel, nthreads=nt)
                    assert np.array_equal(got, want), (name, kind, k, md, sel is None, got.size, want.size)
    corr = R.corr_ref(S.idx[:, 0], S.d2[:, 0])
    for thr in surface_thresholds(surface_dots(corr, sn, tn)):
        want = surface_normal_ref(corr, sn, tn, thr)
        assert want.size > 0 or thr != 0.0, (name, thr)
        assert np.array_equal(orc.reject_surface_normal(corr, sn, tn, thr), want), (name, thr)


@pytest.mark.parametrize("name", ["map_1e5", "flat_far", "lattice_far"])
def test_normal_correspondence_scenes_have_teeth(orc, name, clock):
    """Among the rows whose normal is finite and non-zero, the last minimum in place of the first changes rows on
    lattice_far (exact ties of the shooting score).  fp64 differences in place of fp32 ones are printed: the fp32
    difference of two nearby points is exact unless they straddle a power of two, and no scene here shows a change."""
    S = scene(name)
    sn, tn = scene_normals(S, orc)
    real = np.nonzero(np.isfinite(sn).all(1) & (sn != 0).any(1))[0].astype(np.int32)
    last, diff = {}, {}
    for kind in (1, 2):
        for k in (10, 40):
            ref = normals_corr_ref(kind, S.q, sn, S.cloud, tn, S.idx, S.d2, k, indices=real)
            alt = normals_corr_ref(kind, S.q, sn, S.cloud, tn, S.idx, S.d2, k, indices=real, last=True)
            last[(kind, k)] = int((ref != alt).sum())
            if kind == 1:
                alt = normals_corr_ref(kind, S.q, sn, S.cloud, tn, S.idx, S.d2, k, indices=real, fp64_diff=True)
                diff[k] = int((ref != alt).sum())
    print(f"teeth {name}: last minimum changes {last} rows (kind, k), fp64 differences change {diff} rows (k)")
    if name == "lattice_far":
        assert last[(1, 10)] > 0 and last[(1, 40)] > 0, last


@pytest.mark.parametrize("name", list(R.SCENES))
def test_oracle_fitness_equals_the_reference(orc, name, clock):
    """getFitnessScore (float and double Scalar, an orthonormal and a non-orthonormal pose, four max_range); the
    oracle's transforms equal the reference's operation orders bit for bit."""
    S = scene(name)
    for ortho in (True, False):
        src, T = pose_pair(name, S, ortho)
        oidx = orc.Index(S.cloud)
        for kind, dbl, mode in (("fitness float", False, 1), ("fitness double", True, 1), ("validation float", False, 0)):
            order, dt = APPLY[kind]
            Tm = T if dbl else T.astype(np.float32).astype(np.float64)
            assert np.array_equal(orc.transform(src, Tm, scalar_is_double=dbl, mode=mode)[:, :3],
                                  apply_T(src[:, :3], T, order, dt)), (name, kind)
            if kind.startswith("validation"):
                continue
            _, d2 = moved_d2(S.cloud, src, T, kind)
            for mr in fitness_ranges(d2):
                n, want = fitness_ref(d2, mr)
                got = oidx.fitness_score(src, T, max_range=mr, scalar_is_double=dbl)
                assert fitness_close(got, want, n), (name, kind, ortho, mr, got, want)


def test_transform_orders_have_teeth(clock):
    """On map_1e5, each transform order in float swapped for either of the other two moves at least one point and
    moves the fitness beyond the bar (the double orders are printed)."""
    S = scene("map_1e5")
    src, T = pose_pair("map_1e5", S, True)
    orders = (VALIDATION, SSE_FLOAT, TRANSFORMER_DOUBLE)
    for dt in (np.float32, np.float64):
        mv = {o: apply_T(src[:, :3], T, o, dt) for o in orders}
        fit = {}
        for o in orders:
            _, d2 = knn_sets(S.cloud, mv[o], 1, return_d2=True)
            fit[o] = fitness_ref(d2[:, 0], DBL_MAX)
        for a in orders:
            for b in orders:
                if a >= b:
                    continue
                n = int((mv[a] != mv[b]).any(1).sum())
                rel = abs(fit[a][1] - fit[b][1]) / fit[a][1]
                print(f"teeth {np.dtype(dt).name}: {a} vs {b}: {n} points moved, fitness {rel:.3g} relative")
                if dt == np.float32:
                    assert n > 0 and not fitness_close(fit[a][1], fit[b][1], fit[a][0]), (a, b, n, rel)
