"""VoxelGrid of a batch of clouds in one call (include/pclb200_batch.h: pclb200_voxelgrid_batch) against one
pclb200_voxelgrid (pclb200_voxelgrid_normals) per cloud: every cloud's rows, normal rows and range byte for byte, for
fine, coarse and anisotropic leaves and min_points_per_voxel 0, 1 and 3; two clouds with identical coordinates, non-finite
records, empty ranges, far-out and degenerate clouds; strides 12, 16 and 48; host and device arrays; B = 1, 512 and a
1 M-record cloud among small ones; equal launch counts for B = 8 and 64; refusals that leave every output untouched; and
raw scans through voxel, build, normals and align batches equal to the loop of single calls.  Needs an H100: run with
-m gpu."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_index_batch import _chain

pytestmark = pytest.mark.gpu

LEAVES = {"fine": (0.125, 0.125, 0.125), "coarse": (0.5, 0.5, 0.5), "anisotropic": (0.25, 0.05, 0.125)}
MINS = (0, 1, 3)
SENTINEL = -7.5


@pytest.fixture(scope="module")
def gpu():
    import pcl_b200
    pcl_b200.lib()
    ctx = pcl_b200.Context(0)
    yield pcl_b200, ctx
    ctx.close()


def _scenes(seed):
    """(name, (n, 3) float32): the clouds a batch is made of"""
    r = np.random.default_rng(seed)
    box = lambda n, w, shift=(0, 0, 0): (r.random((n, 3)) * w + np.array(shift)).astype(np.float32)
    twin = box(2500, 3.0, (-1, 2, 0))
    c = box(3000, 4.0, (-7, 3, 11))
    c[::97, 0] = np.nan
    c[5::97, 2] = -np.inf
    c[11, 1] = np.inf
    out = [("twin a", twin), ("twin b", twin.copy()), ("NaN and Inf records", c),
           ("all NaN", np.full((40, 3), np.nan, np.float32)), ("one point", box(1, 1.0, (-7, 3, 11)))]
    sparse = np.zeros((60, 3), np.float32)
    sparse[:, 0] = 10.0 * np.arange(60)
    out.append(("emptied by the minimum", sparse))
    c = box(2000, 3.0)
    c[:, 2] = 0.75
    out.append(("zero-extent axis", c))
    g = np.stack(np.meshgrid(np.arange(12), np.arange(9), np.arange(5), indexing="ij"), -1).reshape(-1, 3)
    out.append(("on voxel faces", np.repeat(g * np.float32(0.125), 2, axis=0).astype(np.float32)))
    out.append(("1e4 away", box(2000, 6.0, (1e4, -1e4, 1e4))))
    out.append(("20 k points", box(20000, 10.0, (5, 5, 5))))
    return out


def _pn(xyz, r):
    """pcl::PointNormal records (12 floats): xyz 1 | unit normal 0 | curvature 0 0 0"""
    rec = np.zeros((len(xyz), 12), np.float32)
    rec[:, :3] = xyz
    rec[:, 3] = 1.0
    nrm = r.normal(0, 0.3, (len(xyz), 3)) + np.array([0, 0, 1.0])
    rec[:, 4:7] = nrm / np.linalg.norm(nrm, axis=1, keepdims=True)
    rec[:, 8] = r.random(len(xyz)) * 0.01
    return rec


def _records(xyz, stride, r):
    if stride == 48:
        return _pn(xyz, r)
    rec = np.full((len(xyz), stride // 4), 1.0, np.float32)
    rec[:, :3] = xyz
    return rec


def _batch(clouds, stride, seed=0):
    r = np.random.default_rng(seed)
    recs = [_records(c, stride, r) for c in clouds]
    off = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int64)
    return recs, np.concatenate(recs), off


def _check(P, ctx, recs, allr, off, leaf, mn, device_in, device_out):
    """the batch against one single call per cloud; device outputs pre-filled with a sentinel that no row past the last
    range may lose"""
    normals = allr.shape[1] == 12
    src = allr
    if device_in:
        import torch
        src = torch.from_numpy(allr).cuda()
    kw = dict(normal_offset=4) if normals else {}
    if device_out:
        import torch
        o = torch.full((len(allr), 4), SENTINEL, dtype=torch.float32, device="cuda")
        kw["out"] = o
        if normals:
            on = torch.full((len(allr), 8), SENTINEL, dtype=torch.float32, device="cuda")
            kw["out_normals"] = on
    res = ctx.voxelgrid_batch(src, off, leaf, mn, **kw)
    rows, oo = res[0], res[-1]
    nrows = res[1] if normals else None
    if device_out:
        m = int(oo[-1])
        assert (o[m:] == SENTINEL).all().item()
        rows = rows.cpu().numpy()
        if normals:
            assert (on[m:] == SENTINEL).all().item()
            nrows = nrows.cpu().numpy()
    assert oo[0] == 0 and len(rows) == oo[-1] and np.all(np.diff(oo) >= 0)
    for c, rec in enumerate(recs):
        a, b = int(oo[c]), int(oo[c + 1])
        if normals:
            ref, ref_n = ctx.voxelgrid_normals(rec, leaf, mn)
            assert nrows[a:b].tobytes() == ref_n.tobytes(), (c, leaf, mn)
        else:
            ref = ctx.voxelgrid(rec, leaf, mn)
        assert rows[a:b].tobytes() == ref.tobytes(), (c, leaf, mn, b - a, len(ref))
    return oo


@pytest.mark.parametrize("stride,device_in,device_out", [(12, False, False), (16, False, False), (48, False, False),
                                                         (16, True, False), (16, True, True), (48, True, True),
                                                         (12, False, True)])
def test_clouds_equal_single_calls(gpu, stride, device_in, device_out):
    """every cloud of a 37-cloud batch, every leaf and minimum, against its own single call"""
    if device_in or device_out:
        pytest.importorskip("torch")
    P, ctx = gpu
    kinds = _scenes(stride)
    r = np.random.default_rng(3 + stride)
    pick = list(range(len(kinds))) + list(r.integers(0, len(kinds), 37 - len(kinds)))
    r.shuffle(pick)
    clouds = [kinds[k][1] for k in pick]
    recs, allr, off = _batch(clouds, stride, stride)
    for leaf in LEAVES.values():
        for mn in MINS:
            oo = _check(P, ctx, recs, allr, off, leaf, mn, device_in, device_out)
            names = [kinds[k][0] for k in pick]
            assert oo[names.index("all NaN") + 1] == oo[names.index("all NaN")]
            if mn == 3:
                j = names.index("emptied by the minimum")
                assert oo[j + 1] == oo[j]


def test_twins_keep_their_own_rows(gpu):
    """two clouds with identical coordinates side by side: each gets all its voxels (a sort that ignored the cloud would
    merge the twins' runs into one cloud's rows)"""
    P, ctx = gpu
    twin = _scenes(1)[0][1]
    recs, allr, off = _batch([twin, twin], 16)
    rows, oo = ctx.voxelgrid_batch(allr, off, LEAVES["fine"])
    single = ctx.voxelgrid(recs[0], LEAVES["fine"])
    assert oo[1] - oo[0] == oo[2] - oo[1] == len(single) > 0
    assert rows[:oo[1]].tobytes() == rows[oo[1]:].tobytes() == single.tobytes()


def test_one_cloud_and_512_clouds(gpu):
    P, ctx = gpu
    kinds = _scenes(5)
    for clouds in ([kinds[2][1]], [kinds[k % len(kinds)][1][: 50 + 13 * (k % 40)] for k in range(512)]):
        recs, allr, off = _batch(clouds, 16)
        for leaf in LEAVES.values():
            for mn in (0, 3):
                _check(P, ctx, recs, allr, off, leaf, mn, False, False)


def test_million_record_cloud_among_small(gpu):
    P, ctx = gpu
    r = np.random.default_rng(4)
    clouds = [c for _, c in _scenes(9)]
    clouds.insert(3, (r.random((1 << 20, 3)) * np.array([50, 50, 4]) - 20).astype(np.float32))
    for stride in (16, 48):
        recs, allr, off = _batch(clouds, stride, 4)
        for mn in (0, 3):
            _check(P, ctx, recs, allr, off, LEAVES["fine"], mn, False, False)


def test_launches_independent_of_batch_size(gpu):
    P, ctx = gpu
    r = np.random.default_rng(9)
    for mn in (0, 3):
        for normals in (False, True):
            counts = []
            for B in (8, 64):
                clouds = [(r.random((500 + 37 * b, 3)) * 3).astype(np.float32) for b in range(B)]
                _, allr, off = _batch(clouds, 48 if normals else 16)
                kw = dict(normal_offset=4) if normals else {}
                ctx.voxelgrid_batch(allr, off, LEAVES["fine"], mn, **kw)
                before = ctx.launches
                ctx.voxelgrid_batch(allr, off, LEAVES["fine"], mn, **kw)
                counts.append(ctx.launches - before)
            assert counts[0] == counts[1], (mn, normals, counts)


def test_refusals_leave_outputs_untouched(gpu):
    P, ctx = gpu
    L = P.lib()
    r = np.random.default_rng(2)
    clouds = [(r.random((300, 3)) * 0.2).astype(np.float32) for _ in range(3)]
    recs, rec, off = _batch(clouds, 48)
    vp = lambda a: None if a is None else C.c_void_p(a.ctypes.data)
    leaf = lambda *x: (C.c_float * 3)(*x)
    good = leaf(0.1, 0.1, 0.1)
    nrm = C.c_void_p(rec.ctypes.data + 16)
    # (B, records, n, stride, offsets, leaf, normals, stride_n, with out_normal_curv, out_xyz1 given, out_offsets given)
    cases = [
        (0, rec, 900, 48, off, good, None, 0, False, True, True),
        (65537, rec, 900, 48, off, good, None, 0, False, True, True),
        (3, None, 900, 48, off, good, None, 0, False, True, True),
        (3, rec, 900, 48, None, good, None, 0, False, True, True),
        (3, rec, 900, 48, off, good, None, 0, False, False, True),
        (3, rec, 900, 48, off, good, None, 0, False, True, False),
        (3, rec, 900, 48, off, None, None, 0, False, True, True),
        (3, rec, 900, 48, np.array([1, 300, 600, 900], np.int64), good, None, 0, False, True, True),
        (3, rec, 900, 48, np.array([0, 300, 300, 900], np.int64), good, None, 0, False, True, True),
        (3, rec, 900, 48, np.array([0, 300, 600, 800], np.int64), good, None, 0, False, True, True),
        (3, rec, 2 ** 31 - 1, 48, np.array([0, 300, 600, 2 ** 31 - 1], np.int64), good, None, 0, False, True, True),
        (3, rec, 900, 10, off, good, None, 0, False, True, True),
        (3, rec, 900, 8, off, good, None, 0, False, True, True),
        (3, rec, 900, 48, off, leaf(0.1, 0.0, 0.1), None, 0, False, True, True),
        (3, rec, 900, 48, off, leaf(0.1, 0.1, -1.0), None, 0, False, True, True),
        (3, rec, 900, 48, off, leaf(float("nan"), 0.1, 0.1), None, 0, False, True, True),
        (3, rec, 900, 48, off, good, nrm, 48, False, True, True),
        (3, rec, 900, 48, off, good, None, 48, True, True, True),
        (3, rec, 900, 48, off, good, nrm, 16, True, True, True),
        (3, rec, 900, 48, off, good, nrm, 22, True, True, True),
    ]
    for j, (B, r_, n, stride, o, lf, nm, sn, with_nc, with_out, with_oo) in enumerate(cases):
        out = np.full((900, 4), SENTINEL, np.float32)
        out_nc = np.full((900, 8), SENTINEL, np.float32)
        oo = np.full(4, 5, np.int64)
        rc = L.pclb200_voxelgrid_batch(ctx.h, vp(r_), n, stride, vp(o), B, lf, 0, nm, sn,
                                       vp(out) if with_out else None, vp(out_nc) if with_nc else None,
                                       vp(oo) if with_oo else None)
        assert rc == P.ERR_INVALID, (j, rc, L.pclb200_last_error())
        assert L.pclb200_last_error()
        assert (out == SENTINEL).all() and (out_nc == SENTINEL).all() and (oo == 5).all(), j
    # the guard: clouds 1 and 2 span 1e3 units at a 1e-3 leaf (cloud 0, 0.2 units, does not); the error names cloud 1,
    # whose single call refuses too
    wide = [(r.random((300, 3)) * 1e3).astype(np.float32) for _ in range(2)]
    recs, rec, off = _batch([clouds[0], wide[0], wide[1], np.full((5, 3), np.nan, np.float32)], 48)
    tiny = (1e-3, 1e-3, 1e-3)
    out = np.full((len(rec), 4), SENTINEL, np.float32)
    out_nc = np.full((len(rec), 8), SENTINEL, np.float32)
    oo = np.full(5, 5, np.int64)
    for nm, onc in ((None, None), (C.c_void_p(rec.ctypes.data + 16), vp(out_nc))):
        rc = L.pclb200_voxelgrid_batch(ctx.h, vp(rec), len(rec), 48, vp(off), 4, leaf(*tiny), 0, nm, 48 if nm else 0,
                                       vp(out), onc, vp(oo))
        assert rc == P.ERR_LEAF_TOO_SMALL, rc
        assert "cloud 1" in L.pclb200_last_error().decode(), L.pclb200_last_error()
        assert (out == SENTINEL).all() and (out_nc == SENTINEL).all() and (oo == 5).all()
    with pytest.raises(Exception):
        ctx.voxelgrid(recs[1], tiny)
    assert ctx.voxelgrid(recs[0], tiny).shape[0] > 0
    # the context still works
    _check(P, ctx, recs[:1] + recs[3:], np.concatenate(recs[:1] + recs[3:]), np.array([0, 300, 305], np.int64),
           LEAVES["fine"], 0, False, False)


def _stats_equal(sa, sb, p):
    for key in sa:
        a, b = sa[key], sb[key]
        assert (a.tobytes() == b.tobytes()) if isinstance(a, np.ndarray) else (a == b or (a != a and b != b)), (p, key)


@pytest.mark.parametrize("est", [1, 0], ids=["point_to_plane", "svd"])
def test_raw_scans_to_aligned_pairs(gpu, est):
    """raw target and source windows through voxelgrid_batch, index_build_batch, normals_knn_batch and one batch align:
    every problem's stats, correspondences and aligned records equal the loop of single voxelgrid, Index, normals_knn and
    one session per pair"""
    P, ctx = gpu
    wins = _chain(16, 12000, 21)
    tg, src = wins[:-1], wins[1:]
    leaf = (0.06, 0.06, 0.06)
    params = P.default_params(max_iterations=30, transformation_epsilon=1e-9, max_correspondence_distance=0.3,
                              estimator=est, track_mode=P.TRACK_ON)
    B = len(tg)
    toff = np.concatenate([[0], np.cumsum([len(w) for w in tg])]).astype(np.int64)
    soff = np.concatenate([[0], np.cumsum([len(w) for w in src])]).astype(np.int64)
    # all batch
    trows, tro = ctx.voxelgrid_batch(np.concatenate(tg), toff, leaf)
    srows, sro = ctx.voxelgrid_batch(np.concatenate(src), soff, leaf)
    assert np.all(np.diff(tro) > 0) and np.all(np.diff(sro) > 0)
    tidx = ctx.index_build_batch(trows, tro)
    nrm = None
    if est == 1:
        bn, _ = ctx.normals_knn_batch(tidx, trows, tro, 16)
        nrm = [bn[tro[p]:tro[p + 1]] for p in range(B)]
    s = P.Icp(ctx, params)
    s.set_target_batch(tidx, normals=nrm)
    s.set_source_batch(srows, sro)
    st = s.iterate_batch()
    corr, cloud = s.get_correspondences_batch(), s.get_cloud()
    s.close()
    # a loop of single calls
    one = P.Icp(ctx, params)
    kept = []
    for p in range(B):
        t = ctx.voxelgrid(tg[p], leaf)
        q = ctx.voxelgrid(src[p], leaf)
        assert t.tobytes() == trows[tro[p]:tro[p + 1]].tobytes() and q.tobytes() == srows[sro[p]:sro[p + 1]].tobytes(), p
        idx = P.Index(ctx, t)
        kept.append(idx)
        n1 = idx.normals_knn(t, 16)[0] if est == 1 else None
        if est == 1:
            assert n1.tobytes() == nrm[p].tobytes(), p
        one.set_target(idx, normals=n1)
        one.set_source(q)
        st1 = one.iterate()
        _stats_equal(st[p], st1, p)
        assert corr[p].tobytes() == one.get_correspondences().tobytes(), p
        assert cloud[sro[p]:sro[p + 1]].tobytes() == one.get_cloud().tobytes(), p
    one.close()
    for i in tidx + kept:
        i.close()
