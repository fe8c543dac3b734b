"""C-ABI behaviour at the edges: device-resident buffers on every entry point, error statuses (never a crash, never
a CPU fallback), degenerate clouds, concurrent callers, session re-use.  Needs an H100: run with -m gpu."""
import threading

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


def _pair(n=30000, seed=3):
    rng = np.random.default_rng(seed)
    tgt = rng.random((n, 3), dtype=np.float32)
    a = np.deg2rad(2.0)
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    src = (tgt.astype(np.float64) @ R.T + [0.01, -0.01, 0.005]).astype(np.float32)
    return src, tgt


def test_device_pointers_everywhere(gpu):
    """Every point / index / output array may live in HBM (torch CUDA tensors): same results as host arrays."""
    import torch
    P, ctx = gpu
    src, tgt = _pair()
    S, T = P.xyz1(src), P.xyz1(tgt)
    dS, dT = torch.from_numpy(S).cuda(), torch.from_numpy(T).cuda()
    hi, di = P.Index(ctx, T), P.Index(ctx, dT)
    assert hi.size == di.size == T.shape[0]
    k = 5
    oi = torch.empty((S.shape[0], k), dtype=torch.int32, device="cuda")
    od = torch.empty((S.shape[0], k), dtype=torch.float32, device="cuda")
    di.knn(dS, k, out_idx=oi, out_d2=od)
    ri, rd, _ = hi.knn(S, k)
    assert np.array_equal(oi.cpu().numpy(), ri) and np.array_equal(od.cpu().numpy(), rd)
    assert np.array_equal(di.correspondences(dS, max_distance=0.05), hi.correspondences(S, max_distance=0.05))
    nd = torch.empty((T.shape[0], 4), dtype=torch.float32, device="cuda")
    di.normals_knn(dT, 10, viewpoint=(0.5, 0.5, 3.0), out=nd)
    nh, _ = hi.normals_knn(T, 10, viewpoint=(0.5, 0.5, 3.0))
    assert np.array_equal(nd.cpu().numpy(), nh, equal_nan=True)
    vd = torch.empty((T.shape[0], 4), dtype=torch.float32, device="cuda")
    vg = ctx.voxelgrid(dT, 0.05, out=vd)
    assert np.array_equal(vg.cpu().numpy(), ctx.voxelgrid(T, 0.05))
    out_d = torch.empty_like(dS)
    out_h = np.empty_like(S)
    rd_ = P.icp_align(ctx, dS, di, out_cloud=out_d, max_iterations=20, max_correspondence_distance=0.1)
    rh_ = P.icp_align(ctx, S, hi, out_cloud=out_h, max_iterations=20, max_correspondence_distance=0.1)
    assert np.array_equal(rd_["final"], rh_["final"]) and rd_["iterations"] == rh_["iterations"]
    assert np.array_equal(out_d.cpu().numpy(), out_h)
    idx_sub = np.arange(0, S.shape[0], 3, dtype=np.int32)
    d_sub = torch.from_numpy(idx_sub).cuda()
    a = P.icp_align(ctx, dS, di, indices=d_sub, max_iterations=5, max_correspondence_distance=0.1)
    b = P.icp_align(ctx, S, hi, indices=idx_sub, max_iterations=5, max_correspondence_distance=0.1)
    assert np.array_equal(a["final"], b["final"]) and a["n_correspondences"] == b["n_correspondences"]
    _device_pointers_other_entry_points(P, ctx, S, T, dS, dT, hi, di, nh, nd)


def _device_pointers_other_entry_points(P, ctx, S, T, dS, dT, hi, di, nh, nd):
    """The rest of the C-ABI with CUDA tensors for inputs and outputs.  Where the Python wrapper hands back NumPy
    arrays the C function is called directly with the tensors' pointers."""
    import ctypes as C
    import torch
    L = P.lib()
    ptr = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    n = S.shape[0]

    def dev_corr(c):
        return torch.from_numpy(np.ascontiguousarray(c).view(np.uint8).copy()).cuda()

    def corr_out(cap):
        return torch.empty(max(cap, 1) * P.CORR_DTYPE.itemsize, dtype=torch.uint8, device="cuda")

    def host_corr(t, m):
        return t.cpu().numpy().view(P.CORR_DTYPE)[:m]

    hm, hk = hi.knn_stats(T, 8)
    dm, dk = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
    P._check(L.pclb200_knn_stats(ctx.h, di.h, ptr(dT), n, 16, None, 0, 8, ptr(dm), ptr(dk)))
    assert np.array_equal(dm.cpu().numpy(), hm) and np.array_equal(dk.cpu().numpy(), hk)
    nr = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    di.normals_radius(dT, 0.05, viewpoint=(0.5, 0.5, 3.0), out=nr)
    assert np.array_equal(nr.cpu().numpy(), hi.normals_radius(T, 0.05, viewpoint=(0.5, 0.5, 3.0))[0], equal_nan=True)
    lab = torch.empty(n, dtype=torch.int32, device="cuda")
    di.cluster_labels(0.01, out=lab)
    assert np.array_equal(lab.cpu().numpy(), hi.cluster_labels(0.01))
    cov = torch.empty((n, 9), dtype=torch.float64, device="cuda")
    P._check(L.pclb200_gicp_covariances(ctx.h, di.h, ptr(dT), n, 16, 10, C.c_double(0.001), ptr(cov)))
    assert np.array_equal(cov.cpu().numpy().reshape(-1, 3, 3), hi.gicp_covariances(T, k=10))

    m = C.c_size_t()
    for kind in (P.CORR_NORMAL_SHOOTING, P.CORR_BACK_PROJECTION):
        want = hi.correspondences_normals(kind, S, nh, nh, k=10, max_distance=0.05)
        out = corr_out(n)
        P._check(L.pclb200_correspondences_normals(ctx.h, di.h, kind, ptr(dS), n, 16, ptr(nd), 16, ptr(nd), 16, None, 0,
                                                   10, C.c_double(0.05), ptr(out), C.byref(m)))
        assert want.size > 0 and np.array_equal(host_corr(out, m.value), want)

    corr = hi.correspondences(S, max_distance=0.05)
    dcorr = dev_corr(corr)
    for kind, p in ((P.REJ_DISTANCE, 0.02), (P.REJ_MEDIAN, 1.0), (P.REJ_ONE_TO_ONE, 0.0), (P.REJ_TRIMMED, 0.7)):
        want, want_med = ctx.reject(corr, kind, p)
        out, med = corr_out(corr.size), C.c_double()
        r = P.Rejector(kind, 0, float(p))
        P._check(L.pclb200_reject(ctx.h, C.byref(r), ptr(dcorr), corr.size, ptr(out), C.byref(m), C.byref(med)))
        assert np.array_equal(host_corr(out, m.value), want) and med.value == want_med
    want = ctx.reject_surface_normal(corr, nh, nh, 0.5)
    out = corr_out(corr.size)
    P._check(L.pclb200_reject_surface_normal(ctx.h, ptr(dcorr), corr.size, ptr(nd), n, 16, ptr(nd), n, 16,
                                             C.c_double(0.5), ptr(out), C.byref(m)))
    assert np.array_equal(host_corr(out, m.value), want)
    Tw = ctx.estimate_svd(S, T, corr=corr)
    Td = np.zeros(16)
    P._check(L.pclb200_estimate_svd(ctx.h, ptr(dS), 16, ptr(dT), 16, ptr(dcorr), corr.size, 0,
                                    Td.ctypes.data_as(C.POINTER(C.c_double))))
    assert np.array_equal(Td.reshape(4, 4), Tw)

    hs, ds = P.Icp(ctx, max_iterations=5, max_correspondence_distance=0.1), P.Icp(ctx, max_iterations=5,
                                                                                  max_correspondence_distance=0.1)
    hs.set_target(hi)
    hs.set_source(S)
    ds.set_target(di)
    ds.set_source(dS)
    hs.iterate()
    ds.iterate()
    want = hs.get_correspondences()
    out = corr_out(n)
    P._check(L.pclb200_icp_get_correspondences(ds.h, ptr(out), C.byref(m)))
    assert want.size > 0 and np.array_equal(host_corr(out, m.value), want)

    # pcl::PointNormal records (48 bytes): xyz1, normal, curvature
    PN = np.concatenate([T, nh, np.zeros((n, 4), np.float32)], axis=1)
    dPN = torch.from_numpy(PN).cuda()
    sub = np.arange(0, n, 2, dtype=np.int32)
    dsub = torch.from_numpy(sub).cuda()
    wx, wn = ctx.voxelgrid_normals(PN, 0.05, indices=sub)
    ox, on = torch.empty((sub.size, 4), device="cuda"), torch.empty((sub.size, 8), device="cuda")
    leaf = (C.c_float * 3)(0.05, 0.05, 0.05)
    P._check(L.pclb200_voxelgrid_normals(ctx.h, ptr(dPN), n, 48, C.c_void_p(dPN.data_ptr() + 16), 48, ptr(dsub),
                                         sub.size, 1, leaf, 0, ptr(ox), ptr(on), C.byref(m)))
    assert m.value == wx.shape[0] > 0
    assert np.array_equal(ox.cpu().numpy()[:m.value], wx) and np.array_equal(on.cpu().numpy()[:m.value], wn, equal_nan=True)


def test_error_statuses(gpu):
    P, ctx = gpu
    src, tgt = _pair(2000)
    T = P.xyz1(tgt)
    idx = P.Index(ctx, T)
    with pytest.raises(P.Pclb200Error) as e:
        P.Index(ctx, np.zeros((0, 4), np.float32))
    assert e.value.code == P.ERR_EMPTY
    with pytest.raises(P.Pclb200Error) as e:
        idx.knn(T[:10], -1)
    assert e.value.code == P.ERR_INVALID
    i, d, keff = idx.knn(T[:10], 0)        # k == 0 -> returns 0 neighbours (kdtree_flann.hpp:247-248)
    assert keff == 0 and i.shape == (10, 0)
    import torch
    bad = torch.zeros((10, 10), dtype=torch.uint8)   # records of 10 bytes: stride < 12 and not a multiple of 4
    with pytest.raises(P.Pclb200Error) as e:
        idx.knn(bad, 1)
    assert e.value.code == P.ERR_INVALID
    with pytest.raises(P.Pclb200Error) as e:
        ctx.voxelgrid(T, 0.0)
    assert e.value.code == P.ERR_INVALID
    with pytest.raises(P.Pclb200Error) as e:
        P.icp_align(ctx, T, idx, estimator=P.EST_POINT_TO_PLANE_LLS)   # no target normals
    assert e.value.code == P.ERR_INVALID
    assert "normals" in str(e.value)
    with pytest.raises(P.Pclb200Error):
        P.Context(99)


def test_degenerate_sources(gpu):
    P, ctx = gpu
    src, tgt = _pair(5000)
    idx = P.Index(ctx, P.xyz1(tgt))
    nan_src = np.full((100, 4), np.nan, np.float32)
    r = P.icp_align(ctx, nan_src, idx, max_iterations=5, is_dense=0)
    assert not r["converged"] and r["state"] == 5 and r["iterations"] == 0 and r["n_correspondences"] == 0
    assert np.array_equal(r["final"], np.eye(4))
    r = P.icp_align(ctx, P.xyz1(src[:2]), idx, max_iterations=5)      # < 3 correspondences (icp.hpp:204-213)
    assert r["state"] == 5 and r["n_correspondences"] == 2
    r = P.icp_align(ctx, P.xyz1(src[:3]), idx, max_iterations=5)      # exactly min_number_correspondences_
    assert r["iterations"] >= 1
    one = P.Index(ctx, P.xyz1(tgt[:1]))                                 # single-point target
    c = one.correspondences(P.xyz1(src[:50]))
    assert c.size == 50 and np.all(c["index_match"] == 0)
    s = P.Icp(ctx, max_iterations=3)
    s.set_target(idx)
    s.set_source(P.xyz1(src))
    assert s.get_correspondences().size == 0                           # nothing evaluated yet


def test_concurrent_callers_and_session_reuse(gpu, orc):
    """PCL's query methods are const and may be called from several threads (impl/search.hpp:126): calls on one
    context serialise and stay correct.  One registration object re-used for different sources == fresh objects."""
    P, ctx = gpu
    src, tgt = _pair(20000)
    T, S = P.xyz1(tgt), P.xyz1(src)
    idx = P.Index(ctx, T)
    want_i, want_d, _ = orc.Index(T).knn(S[:4000], 4, nthreads=4)
    errs = []

    def worker(lo):
        try:
            for _ in range(5):
                gi, gd, _ = idx.knn(S[lo:lo + 1000], 4)
                if not (np.array_equal(gi, want_i[lo:lo + 1000]) and np.array_equal(gd, want_d[lo:lo + 1000])):
                    errs.append(lo)
        except Exception as ex:  # noqa
            errs.append(repr(ex))

    th = [threading.Thread(target=worker, args=(i * 1000,)) for i in range(4)]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs, errs
    sess = P.Icp(ctx, max_iterations=12, max_correspondence_distance=0.1)
    sess.set_target(idx)
    for shift in (0.0, 0.004, -0.003):
        Sx = S.copy()
        Sx[:, 0] += np.float32(shift)
        sess.set_source(Sx)
        a = sess.iterate()
        b = P.icp_align(ctx, Sx, idx, max_iterations=12, max_correspondence_distance=0.1)
        assert np.array_equal(a["final"], b["final"]) and a["iterations"] == b["iterations"]


def test_radius_into_caller_buffers(gpu):
    """pclb200_radius_into: the same lists as pclb200_radius, written into caller buffers — host arrays, pinned host
    tensors and device tensors — without library-side allocation; a too-small capacity only reports the total."""
    import torch
    P, ctx = gpu
    rng = np.random.default_rng(8)
    cloud = P.xyz1(rng.random((50000, 3), dtype=np.float32))
    q = P.xyz1(rng.random((3000, 3), dtype=np.float32))
    idx = P.Index(ctx, cloud)
    for max_nn in (0, 7):
        offs, ii, dd = idx.radius(q, 0.05, max_nn=max_nn)
        total = int(offs[-1])
        o2 = np.zeros(q.shape[0] + 1, np.int64)
        assert idx.radius_into(q, 0.05, o2, np.empty(0, np.int32), np.empty(0, np.float32), max_nn=max_nn) == total
        assert np.array_equal(o2, offs)                     # sizing call: offsets + total, nothing else written
        i2, d2 = np.full(total + 5, -7, np.int32), np.full(total + 5, -7, np.float32)
        assert idx.radius_into(q, 0.05, o2, i2, d2, max_nn=max_nn) == total
        assert np.array_equal(i2[:total], ii) and np.array_equal(d2[:total], dd) and np.all(i2[total:] == -7)
        # device-resident result (queries, offsets and lists all in HBM)
        dq = torch.from_numpy(q).cuda()
        do = torch.zeros(q.shape[0] + 1, dtype=torch.int64, device="cuda")
        di = torch.empty(total, dtype=torch.int32, device="cuda")
        ddv = torch.empty(total, dtype=torch.float32, device="cuda")
        assert idx.radius_into(dq, 0.05, do, di, ddv, max_nn=max_nn) == total
        assert np.array_equal(do.cpu().numpy(), offs) and np.array_equal(di.cpu().numpy(), ii)
        assert np.array_equal(ddv.cpu().numpy(), dd)
        # pinned host buffers
        pi, pd = torch.empty(total, dtype=torch.int32).pin_memory(), torch.empty(total, dtype=torch.float32).pin_memory()
        po = torch.zeros(q.shape[0] + 1, dtype=torch.int64).pin_memory()
        assert idx.radius_into(q, 0.05, po, pi, pd, max_nn=max_nn) == total
        assert np.array_equal(pi.numpy(), ii) and np.array_equal(pd.numpy(), dd) and np.array_equal(po.numpy(), offs)
