"""Every device k-NN, radius, correspondence and knn_stats list against the fp32 brute-force reference of
tests/test_search_reference.py, on its map-scale scenes, on every search path, every query bit for bit.  Which kernel
served a call is proven, not assumed: the warp k-NN kernel adds one launch to a knn call, the bounded radius branch
records a "radius_knn" profile range.  Needs an H100: run with -m gpu."""
import os
import sys
import time
from collections import defaultdict

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_search_reference as R  # noqa: E402
from test_normals_reference import knn_sets, radius_csr  # noqa: E402

pytestmark = pytest.mark.gpu

# k -> the per-thread kernel launch_knn picks (search.cu); 12 <= k <= 32 first go through k_knn_warp where it applies,
# and the per-thread kernel then only redoes the rows the warp kernel handed back
KNN_PATHS = {1: "k_knn<1>", 2: "k_knn<2>", 3: "k_knn<4>", 4: "k_knn<4>", 5: "k_knn<8>", 8: "k_knn<8>", 10: "k_knn<10>",
             11: "k_knn<16>", 12: "k_knn<16>", 16: "k_knn<16>", 24: "k_knn<32>", 32: "k_knn<32>", 33: "k_knn_any",
             64: "k_knn_any"}
WARP_K = (12, 16, 24, 32)
STATS_PATHS = {2: "k_knn_stats<2>", 9: "k_knn_stats<10>", 16: "k_knn_stats<16>", 32: "k_knn_stats<32>",
               33: "knn_stats from lists", 51: "knn_stats from lists"}
MAX_NN = (0, 3, 10, 32, 64)

SERVED = defaultdict(set)   # path -> scenes that went through it
ROWS = defaultdict(int)     # path -> rows compared
SKIPPED = {}                # scene -> total_skipped_walks of the TRACK_ON loop
T0 = [0.0]


@pytest.fixture(scope="module")
def gpu():
    import pcl_b200
    pcl_b200.lib()
    ctx = pcl_b200.Context(0)
    T0[0] = time.time()
    yield pcl_b200, ctx
    ctx.close()
    print(f"\n{'path':56s} {'rows checked':>12s}  far scenes")
    for path in sorted(ROWS):
        print(f"{path:56s} {ROWS[path]:12d}  {', '.join(sorted(SERVED[path]))}")
    print(f"ICP skipped walks (TRACK_ON): {SKIPPED}")
    print(f"test_gpu_search_reference.py: {time.time() - T0[0]:.1f} s")


def _served(path, scene, rows):
    SERVED[path].add(scene)
    ROWS[path] += int(rows)


def _assert_rows(got_i, got_d, want_i, want_d, label):
    bad = np.nonzero((got_i != want_i).any(1) | (got_d.view(np.int32) != want_d.view(np.int32)).any(1))[0]
    assert bad.size == 0, (label, bad.size, bad[:5].tolist(), got_i[bad[:2]].tolist(), want_i[bad[:2]].tolist(),
                           got_d[bad[:2]].tolist(), want_d[bad[:2]].tolist())


def _truncate(csr, max_nn, n_valid):
    """The reference radius CSR cut to the max_nn nearest of every row (max_nn = 0 or >= n_valid: no cut)."""
    off, idx, d2 = csr
    if not 0 < max_nn < n_valid:
        return csr
    cnt = np.minimum(np.diff(off), max_nn)
    keep = np.concatenate([np.arange(off[i], off[i] + cnt[i]) for i in range(cnt.size)]) if cnt.sum() else np.zeros(0, np.int64)
    no = np.zeros_like(off)
    np.cumsum(cnt, out=no[1:])
    return no, idx[keep], d2[keep]


def _knn_all_k(ctx, gidx, q, ref_i, ref_d, n_valid, scene, label):
    """Every k of KNN_PATHS against the reference lists at K_MAX; returns the launches of each call."""
    launches = {}
    for k in sorted(KNN_PATHS):
        before = ctx.launches
        gi, gd, gk = gidx.knn(q, k)
        launches[k] = ctx.launches - before
        assert gk == min(k, n_valid), (scene, label, k, gk)
        _assert_rows(gi, gd, ref_i[:, :k].astype(np.int32), ref_d[:, :k], (scene, label, k))
    # the warp kernel is one launch more than the per-thread kernel alone (k = 11: k_knn<16> and nothing else)
    for k in sorted(KNN_PATHS):
        extra = launches[k] - launches[11]
        assert extra in (0, 1), (scene, label, k, launches)
        assert extra == 0 or k in WARP_K, (scene, label, k, launches)
        path = (f"k_knn_warp + {KNN_PATHS[k]} redo" if extra else KNN_PATHS[k]) + (f" ({label})" if label else "")
        _served(path, scene, q.shape[0])
    return launches


@pytest.mark.parametrize("name", list(R.SCENES))
def test_every_list_on_every_path(gpu, name):
    """k-NN at every k (every per-thread list size, the warp kernel and its redo, the any-k kernel), also through an
    index subset and 48-byte PointNormal records; knn_stats on both of its paths; radius search at three radii and
    five max_nn (the bounded k-NN branch and the count / fill / truncate branch), also into torch device buffers;
    correspondences plain, gated, with indices and reciprocal.  Every query of every kind, bit for bit."""
    import torch
    P, ctx = gpu
    S = R.Scene(name)
    gidx = P.Index(ctx, S.cloud)
    assert gidx.size == S.n_valid

    # ---- k-NN ----
    launches = _knn_all_k(ctx, gidx, S.q, S.idx, S.d2, S.n_valid, name, "")
    print(f"{name}: launches per knn call {launches}")
    rng = np.random.default_rng(17)
    n = S.cloud.shape[0]
    sub = np.sort(rng.permutation(n)[: (2 * n) // 3]).astype(np.int32)
    masked = S.cloud.copy()
    out = np.ones(n, bool)
    out[sub] = False
    masked[out, :3] = np.nan  # the reference of an index over `sub` keeps the original indices
    si, sd = knn_sets(masked, S.q, R.K_MAX, return_d2=True)
    pn = np.zeros((n, 12), np.float32)
    pn[:, :3] = S.cloud[:, :3]
    pn[:, 3] = 1
    qpn = np.zeros((S.q.shape[0], 12), np.float32)
    qpn[:, :3] = S.q[:, :3]
    _knn_all_k(ctx, P.Index(ctx, pn, subset=sub), qpn, si, sd, sub.size, name, "subset, 48-byte records")

    # ---- knn_stats ----
    for k, path in STATS_PATHS.items():
        gm, gk = gidx.knn_stats(S.q, k)
        rm, rk = R.knn_stats_ref(S.idx, S.d2, k, S.n_valid)
        bad = np.nonzero((gm.view(np.int32) != rm.view(np.int32)) | (gk.view(np.int32) != rk.view(np.int32)))[0]
        assert bad.size == 0, (name, k, bad.size, bad[:5].tolist(), gm[bad[:3]].tolist(), rm[bad[:3]].tolist(),
                               gk[bad[:3]].tolist(), rk[bad[:3]].tolist())
        _served(path, name, S.q.shape[0])

    # ---- radius ----
    ctx.profile(True)
    try:
        for r in S.radii():
            q = S.radius_queries(r)
            full = radius_csr(S.cloud, q, r)
            for max_nn in MAX_NN:
                ctx.profile_reset()
                got = gidx.radius(q, r, max_nn=max_nn)
                bounded = ctx.profile_get("radius_knn")[1] > 0
                ok, row = R.csr_rows_equal(got, _truncate(full, max_nn, S.n_valid))
                assert ok, (name, r, max_nn, bounded, row)
                path = ("radius: bounded k-NN" if bounded else
                        "radius: count / fill / truncate" if 0 < max_nn < S.n_valid else "radius: count / fill")
                _served(path, name, q.shape[0])
            for max_nn in (0, 10):
                want = _truncate(full, max_nn, S.n_valid)
                offs = torch.empty(q.shape[0] + 1, dtype=torch.int64, device="cuda")
                ti = torch.empty(max(int(want[0][-1]), 1), dtype=torch.int32, device="cuda")
                td = torch.empty(max(int(want[0][-1]), 1), dtype=torch.float32, device="cuda")
                total = gidx.radius_into(q, r, offs, ti, td, max_nn=max_nn)
                torch.cuda.synchronize()
                got = (offs.cpu().numpy(), ti.cpu().numpy()[:total], td.cpu().numpy()[:total])
                ok, row = R.csr_rows_equal(got, want)
                assert total == want[0][-1] and ok, (name, r, max_nn, row)
                _served("radius_into, torch device buffers", name, q.shape[0])
    finally:
        ctx.profile(False)

    # ---- correspondences ----
    nn, nd = S.idx[:, 0], S.d2[:, 0]
    src = S.q
    for md in (R.NO_GATE, 3 * S.spacing, S.spacing, 0.3 * S.spacing):
        g = gidx.correspondences(src, max_distance=md, is_dense=False)
        w = R.corr_ref(nn, nd, md)
        assert np.array_equal(g, w), (name, md, g.size, w.size)
        _served("correspondences" + (" gated" if md != R.NO_GATE else ""), name, src.shape[0])
    ind = rng.permutation(src.shape[0])[:30_000].astype(np.int32)
    g = gidx.correspondences(src, max_distance=S.spacing, indices=ind, is_dense=False)
    assert np.array_equal(g, R.corr_ref(nn, nd, S.spacing, indices=ind)), name
    _served("correspondences, indices", name, ind.size)
    g = gidx.correspondences(src, max_distance=3 * S.spacing, is_dense=False, src_index=P.Index(ctx, src))
    w = R.corr_ref(nn, nd, 3 * S.spacing, back=R.reciprocal_back(src, S.cloud))
    assert w.size > 0 and np.array_equal(g, w), (name, g.size, w.size)
    _served("correspondences, reciprocal", name, src.shape[0])


def _icp_pair(name):
    """(target points, source points, gate): the source is every third target point moved by a small rigid motion
    about the centre of the scene (so the motion is small where the points are)."""
    pts, spacing = R.SCENES[name]()
    rng = np.random.default_rng(23)
    src = pts[::3].astype(np.float64)
    c = src.mean(0)
    a = np.deg2rad(0.3)
    Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    t = rng.normal(0, 0.3 * spacing, 3)
    if name == "object_far_out":  # around the object, by a fraction of its own point spacing
        c = np.array([500.0, 500.0, 0.0])
        t = rng.normal(0, 5e-4, 3)
    src = (src - c) @ Rz.T + c + t
    return pts, src.astype(np.float32), 3 * spacing


@pytest.mark.parametrize("name", ["map_1e5", "object_far_out", "straddle"])
def test_icp_loop_lists_every_iteration(gpu, orc, name):
    """The ICP search (cell-table start, the TRACK skip) in every tracking mode: every iteration's correspondence list
    equals the reference on the cloud re-transformed in fp32 (IterativeClosestPoint::transformCloud)."""
    P, ctx = gpu
    tgt, src, gate = _icp_pair(name)
    T, Sx = R.xyz1(tgt), R.xyz1(src)
    tidx = P.Index(ctx, T)
    for track, tname in ((P.TRACK_ON, "on"), (P.TRACK_OFF, "off"), (P.TRACK_AUTO, "auto")):
        s = P.Icp(ctx, max_iterations=25, max_correspondence_distance=gate, is_dense=0, mse_threshold_absolute=0.0,
                  track_mode=track)
        s.set_target(tidx)
        s.set_source(Sx)
        cloud = Sx.copy()
        st = None
        for it in range(25):
            st = s.iterate(1)
            g = s.get_correspondences()
            ri, rd = knn_sets(T, cloud, 1, return_d2=True)
            w = R.corr_ref(ri[:, 0], rd[:, 0], gate)
            assert np.array_equal(g, w), (name, tname, it, g.size, w.size)
            assert st["n_correspondences"] == w.size
            _served(f"ICP nearest1, tracking {tname}", name, cloud.shape[0])
            cloud = orc.transform(cloud, st["last"], mode=0)
            if st["state"] != 0:
                break
        if track == P.TRACK_ON:
            SKIPPED[name] = st["total_skipped_walks"]


def test_every_path_was_served_by_a_far_scene(gpu):
    """Each named path went through at least one of the far scenes above (run after them; skipped when they were
    deselected)."""
    if len({s for v in SERVED.values() for s in v}) < len(R.SCENES) or len(SKIPPED) < 3:
        pytest.skip("needs every scene test of this file in the same run")
    knn = {KNN_PATHS[k] for k in KNN_PATHS if k not in WARP_K} | {f"k_knn_warp + {KNN_PATHS[k]} redo" for k in WARP_K}
    for path in knn | {p + " (subset, 48-byte records)" for p in knn} | set(STATS_PATHS.values()):
        assert SERVED[path], path
    for path in ("radius: bounded k-NN", "radius: count / fill / truncate", "radius: count / fill",
                 "radius_into, torch device buffers", "correspondences", "correspondences gated",
                 "correspondences, indices", "correspondences, reciprocal", "ICP nearest1, tracking on",
                 "ICP nearest1, tracking off", "ICP nearest1, tracking auto"):
        assert SERVED[path], path
    assert any(v > 0 for v in SKIPPED.values()), SKIPPED
