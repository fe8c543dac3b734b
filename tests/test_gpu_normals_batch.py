"""The k-NN normals of a batch of query sets in one call (include/pclb200_batch.h: pclb200_normals_knn_batch) against one
pclb200_normals_knn per set: every set's rows and is_dense byte for byte, for every k case (per-thread kernels, the warp
kernel, the materialised lists), handles from single and batch builds, repeated handles, query sets that are not the
handle's cloud, per-set viewpoints, strides, host and device arrays; equal launch counts for B = 8 and 64; refusals that
leave the output untouched; and batch aligns on these normals equal to aligns on per-handle normals.  Needs an H100: run
with -m gpu."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_index_batch import _batch_input, _chain, _kinds, _records

pytestmark = pytest.mark.gpu

KS = (3, 8, 10, 16, 20, 32, 40)


@pytest.fixture(scope="module")
def gpu():
    import pcl_b200
    pcl_b200.lib()
    ctx = pcl_b200.Context(0)
    yield pcl_b200, ctx
    ctx.close()


def _viewpoints(clouds, r):
    """per set: the origin, a point far above, or one far below the cloud (the flip matters)"""
    out = []
    for j, c in enumerate(clouds):
        fin = c[np.isfinite(c).all(1)]
        mid = fin.mean(0) if len(fin) else np.zeros(3)
        ext = float(np.max(fin.max(0) - fin.min(0))) if len(fin) else 1.0
        out.append([np.zeros(3), mid + np.array([0.1, -0.2, 3.0]) * (ext + 1), mid - np.array([0.3, 0.1, 5.0]) * (ext + 1)][j % 3])
    return np.array(out, np.float32) + r.normal(0, 0.01, (len(clouds), 3)).astype(np.float32)


def _setup(P, ctx, clouds, batch_built, seed):
    """handles for the query sets: set 1 repeats set 0's handle on another query set (a shifted copy of cloud 0), and
    the last set is searched in the handle of cloud 0"""
    r = np.random.default_rng(seed)
    qsets = list(clouds)
    if len(clouds) > 2:
        qsets[1] = (clouds[0] + r.normal(0, 0.01, clouds[0].shape)).astype(np.float32)
    if batch_built:
        src, off, _ = _batch_input(clouds, 16, False)
        built = ctx.index_build_batch(src, off)
    else:
        built = [P.Index(ctx, _records(c, 16)) for c in clouds]
    handles = list(built)
    if len(clouds) > 2:
        handles[1] = built[0]
        handles[-1] = built[0]
    return built, handles, qsets, _viewpoints(qsets, r)


def _compare(P, ctx, handles, qsets, vps, stride, device, ks=KS):
    allr, off, host = _batch_input(qsets, stride, device)
    for k in ks:
        out = None
        if device:
            import torch
            out = torch.full((len(host), 4), 7.0, device="cuda")
        got, dense = ctx.normals_knn_batch(handles, allr, off, k, viewpoints=vps, out=out)
        if device:
            got = got.cpu().numpy()
        assert got.shape == (len(host), 4) and dense.shape == (len(qsets),)
        for c, h in enumerate(handles):
            ref, d = h.normals_knn(host[off[c]:off[c + 1]], k, viewpoint=vps[c])
            assert got[off[c]:off[c + 1]].tobytes() == ref.tobytes(), (k, c)
            assert bool(dense[c]) == d, (k, c)


@pytest.mark.parametrize("stride,device,batch_built", [(16, False, False), (12, False, True), (48, False, False),
                                                       (16, True, True), (48, True, False)])
def test_sets_equal_single_calls(gpu, stride, device, batch_built):
    """a batch of the index-batch kinds of cloud (each twice) against one normals_knn per set, for every k"""
    if device:
        pytest.importorskip("torch")
    P, ctx = gpu
    clouds = [c for _, c in _kinds(stride)] * 2
    built, handles, qsets, vps = _setup(P, ctx, clouds, batch_built, stride)
    _compare(P, ctx, handles, qsets, vps, stride, device)
    for h in built:
        h.close()


def test_one_set_and_512_sets(gpu):
    P, ctx = gpu
    r = np.random.default_rng(3)
    one = [(r.random((5000, 3)) * [4, 4, 0.3]).astype(np.float32)]
    built, handles, qsets, vps = _setup(P, ctx, one, False, 1)
    _compare(P, ctx, handles, qsets, vps, 16, False)
    for h in built:
        h.close()
    kinds = [c for _, c in _kinds(5)]
    clouds = [kinds[j % len(kinds)] if j % 4 else (r.random((int(r.integers(20, 3000)), 3)) * 2).astype(np.float32)
              for j in range(512)]
    built, handles, qsets, vps = _setup(P, ctx, clouds, True, 2)
    _compare(P, ctx, handles, qsets, vps, 16, False, ks=(8, 16, 40))
    for h in built:
        h.close()


def test_million_point_set_among_small(gpu):
    P, ctx = gpu
    r = np.random.default_rng(4)
    clouds = [c for _, c in _kinds(9)]
    clouds.insert(3, (r.random((1 << 20, 3)) * np.array([50, 50, 4]) - 20).astype(np.float32))
    built, handles, qsets, vps = _setup(P, ctx, clouds, True, 4)
    _compare(P, ctx, handles, qsets, vps, 16, False, ks=(10, 16, 40))
    for h in built:
        h.close()


def test_launches_independent_of_batch_size(gpu):
    P, ctx = gpu
    r = np.random.default_rng(9)
    for k in (8, 16, 40):
        counts = []
        for B in (8, 64):
            clouds = [(r.random((500 + 37 * b, 3)) * 3).astype(np.float32) for b in range(B)]
            src, off, _ = _batch_input(clouds, 16, False)
            hs = ctx.index_build_batch(src, off)
            ctx.normals_knn_batch(hs, src, off, k)  # the lists path's lazy per-handle position table, made once
            before = ctx.launches
            ctx.normals_knn_batch(hs, src, off, k)
            counts.append(ctx.launches - before)
            for h in hs:
                h.close()
        assert counts[0] == counts[1], (k, counts)


def test_refusals_leave_output_untouched(gpu):
    P, ctx = gpu
    L = P.lib()
    clouds = [(np.random.default_rng(j).random((300, 3)) * 2).astype(np.float32) for j in range(3)]
    rec = np.concatenate([_records(c, 16) for c in clouds])
    off = np.array([0, 300, 600, 900], np.int64)
    hs = [P.Index(ctx, _records(c, 16)) for c in clouds]
    tagged = (C.c_void_p * 3)(*[h.h for h in hs])
    vp = lambda a: C.c_void_p(a.ctypes.data)
    lab, ids = C.c_void_p(), np.arange(300, dtype=np.int32) * 2
    assert L.pclb200_index_build_ids(ctx.h, vp(rec), 300, 16, vp(ids), C.byref(lab)) == P.OK
    with_lab = (C.c_void_p * 3)(hs[0].h, lab, hs[2].h)
    with_null = (C.c_void_p * 3)(hs[0].h, None, hs[2].h)
    cases = [  # (handles, B, records, n, stride, offsets, k)
        (tagged, 0, rec, 900, 16, off, 16),
        (tagged, 65537, rec, 900, 16, off, 16),
        (None, 3, rec, 900, 16, off, 16),
        (with_null, 3, rec, 900, 16, off, 16),
        (tagged, 3, None, 900, 16, off, 16),
        (tagged, 3, rec, 900, 16, None, 16),
        (tagged, 3, rec, 900, 16, np.array([1, 300, 600, 900], np.int64), 16),
        (tagged, 3, rec, 900, 16, np.array([0, 300, 300, 900], np.int64), 16),
        (tagged, 3, rec, 900, 16, np.array([0, 300, 600, 800], np.int64), 16),
        (tagged, 3, rec, 2 ** 31 - 1, 16, np.array([0, 300, 600, 2 ** 31 - 1], np.int64), 16),
        (tagged, 3, rec, 900, 10, off, 16),
        (tagged, 3, rec, 900, 16, off, 0),
        (tagged, 3, rec, 900, 16, off, -4),
        (with_lab, 3, rec, 900, 16, off, 40),  # the lists path needs the cloud the index was built from
    ]
    for j, (h, B, r_, n, stride, o, k) in enumerate(cases):
        out = np.full((900, 4), 7.0, np.float32)
        dense = np.full(3, 5, np.int32)
        rc = L.pclb200_normals_knn_batch(ctx.h, h, B, None if r_ is None else vp(r_), n, stride,
                                         None if o is None else vp(o), k, None, vp(out), vp(dense))
        assert rc == P.ERR_INVALID, (j, rc, L.pclb200_last_error())
        assert L.pclb200_last_error()
        assert (out == 7.0).all() and (dense == 5).all(), j
    out = np.full((900, 4), 7.0, np.float32)
    assert L.pclb200_normals_knn_batch(ctx.h, tagged, 3, vp(rec), 900, 16, vp(off), 16, None, None, None) == P.ERR_INVALID
    # the context still works
    got, dense = ctx.normals_knn_batch(hs, rec, off, 16)
    for c in range(3):
        ref, d = hs[c].normals_knn(rec[off[c]:off[c + 1]], 16)
        assert got[off[c]:off[c + 1]].tobytes() == ref.tobytes() and bool(dense[c]) == d
    L.pclb200_index_destroy(lab)
    for h in hs:
        h.close()


@pytest.mark.parametrize("est", [1, 2])
def test_batch_aligns_on_batch_normals(gpu, est):
    """point-to-plane and the symmetric objective: iterate_batch on the batch normals gives the stats, correspondences and
    aligned records it gives on per-handle normals"""
    P, ctx = gpu
    wins = _chain(24, 3000, 13)
    tg, src = wins[:-1], wins[1:]
    off = np.concatenate([[0], np.cumsum([len(w) for w in tg])]).astype(np.int64)
    all_tg = np.concatenate(tg)
    idx = ctx.index_build_batch(all_tg, off)
    bn, _ = ctx.normals_knn_batch(idx, all_tg, off, 16)
    nrm_batch = [bn[off[p]:off[p + 1]] for p in range(len(tg))]
    nrm_single = [i.normals_knn(w, 16)[0] for i, w in zip(idx, tg)]
    soff = np.concatenate([[0], np.cumsum([len(w) for w in src])]).astype(np.int64)
    all_src = np.concatenate(src)
    sidx = ctx.index_build_batch(all_src, soff)
    sn, _ = ctx.normals_knn_batch(sidx, all_src, soff, 16)
    srec = np.concatenate([all_src, sn], axis=1)
    params = P.default_params(max_iterations=30, transformation_epsilon=1e-9, max_correspondence_distance=0.3,
                              estimator=est, with_normals_transform=int(est == 2), track_mode=P.TRACK_ON)
    runs = []
    for nrm in (nrm_batch, nrm_single):
        s = P.Icp(ctx, params)
        s.set_target_batch(idx, normals=nrm)
        s.set_source_batch(srec, soff, normals=P.Field(srec, 4))
        st = s.iterate_batch()
        runs.append((st, s.get_correspondences_batch(), s.get_cloud(stride_floats=8)))
        s.close()
    (sa, ca, pa), (sb, cb, pb) = runs
    for p in range(len(src)):
        for key in sa[p]:
            a, b = sa[p][key], sb[p][key]
            assert (a.tobytes() == b.tobytes()) if isinstance(a, np.ndarray) else (a == b or (a != a and b != b)), (p, key)
        assert ca[p].tobytes() == cb[p].tobytes(), p
    assert pa.tobytes() == pb.tobytes()
    for i in idx + sidx:
        i.close()
