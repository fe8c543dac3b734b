"""A batch of scan pairs in one session (include/pclb200_batch.h: pclb200_icp_set_target_batch), each problem against its
own target, against single sessions: per problem, every stats field, every iteration's correspondences and the aligned
records are byte-equal to a fresh session given set_target(its index, its normals) and set_source(its records, its
guess).  Needs an H100: run with -m gpu."""
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


def _surface(xy, scale=1.0, shift=(0.0, 0.0, 0.0)):
    """PointNormal records (n, 8) on z = 0.1 sin(3x) + 0.1 cos(4y), scaled and moved, with their analytic normals"""
    z = 0.1 * np.sin(3 * xy[:, 0]) + 0.1 * np.cos(4 * xy[:, 1])
    nrm = np.stack([-0.3 * np.cos(3 * xy[:, 0]), 0.4 * np.sin(4 * xy[:, 1]), np.ones(len(xy))], 1)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    out = np.zeros((len(xy), 8), np.float32)
    out[:, 0:2], out[:, 2], out[:, 3], out[:, 4:7] = xy * scale + shift[:2], z * scale + shift[2], 1.0, nrm
    return out


def _moved(rec, deg, t, centre, axis=2):
    """rec rotated by deg about `centre` and moved by t"""
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    R = np.array({2: [[c, -s, 0], [s, c, 0], [0, 0, 1]], 0: [[1, 0, 0], [0, c, -s], [0, s, c]]}[axis])
    out = rec.copy()
    out[:, 0:3] = (rec[:, 0:3].astype(np.float64) - centre) @ R.T + centre + t
    out[:, 4:7] = rec[:, 4:7].astype(np.float64) @ R.T
    return out


@pytest.fixture(scope="module")
def pairs(gpu):
    """12 problems over 10 targets (target 0 serves problems 0, 4 and 8): sizes 2 k to 20 k points, boxes from 1 to 100
    units wide, from the origin to 10^4 away; a target with NaN points, one with a NaN normal; problem 5 out of reach."""
    P, ctx = gpu
    r = np.random.default_rng(21)
    sizes = [20000, 2000, 8000, 5000, 12000, 3000, 16000, 2500, 6000, 10000]
    scales = [2.0, 1.0, 2.0, 40.0, 2.0, 2.0, 100.0, 1.0, 2.0, 2.0]
    shifts = [(0, 0, 0), (1000, -2000, 50), (-3, 4, 1), (10000, 10000, -300), (0.5, 0.5, 0), (7, -7, 2),
              (-5000, 300, 20), (0, 0, 0), (200, 100, -10), (-40, 80, 5)]
    tgts, idx, tnrm = [], [], []
    for k, (n, sc, sh) in enumerate(zip(sizes, scales, shifts)):
        t = _surface(r.random((n, 2)), sc, np.array(sh, np.float64))
        if k == 2:
            t[::50, 1] = np.nan   # NaN points: not indexed
        if k == 7:
            t[17:40, 5] = np.nan  # NaN normals: the LLS estimators skip those pairs
        tgts.append(t)
        idx.append(P.Index(ctx, np.ascontiguousarray(t[:, :4])))
        tnrm.append(np.ascontiguousarray(t[:, 4:8]))
    of = [0, 1, 2, 3, 0, 5, 6, 7, 0, 8, 9, 4]  # problem -> target
    motions = [(1.5, (0.004, -0.003, 0.002)), (0.2, (0.001, 0, 0)), (3.0, (0.01, 0.01, -0.005)), (0.5, (0.05, 0, 0)),
               (0.0, (0, 0, 0)), (2.0, (-0.006, 0.004, 0.001)), (0.3, (0.2, 0.1, 0)), (1.0, (0, 0.003, 0)),
               (4.0, (0.02, -0.01, 0.004)), (0.7, (0.003, 0.003, 0.003)), (2.5, (0.008, 0, -0.002)),
               (1.2, (0, -0.004, 0))]
    srcs = []
    for p, (k, (deg, t)) in enumerate(zip(of, motions)):
        m = max(1000, sizes[k] // 2)
        s = _surface(0.1 + r.random((m, 2)) * 0.8, scales[k], np.array(shifts[k], np.float64))
        centre = np.array(shifts[k], np.float64) + scales[k] * 0.5
        srcs.append(_moved(s, deg, np.array(t) * scales[k] / 2, centre, axis=2 if p % 2 == 0 else 0))
    srcs[5][:, 0:3] += np.float32(50.0)  # out of reach: NO_CORRESPONDENCES
    return P, ctx, [idx[k] for k in of], [tnrm[k] for k in of], srcs


ESTIMATORS = {"svd": dict(estimator=0), "svd_no_umeyama": dict(estimator=0, svd_no_umeyama=1),
              "point_to_plane": dict(estimator=1), "symmetric": dict(estimator=2, with_normals_transform=1)}


def _params(P, est, dbl, track, **kw):
    base = dict(max_iterations=40, transformation_epsilon=1e-9, max_correspondence_distance=0.5, is_dense=0,
                scalar_is_double=int(dbl), track_mode=track)
    base.update(ESTIMATORS[est])
    base.update(kw)
    return P.default_params(**base)


def _same_stats(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], np.ndarray):
            assert a[k].tobytes() == b[k].tobytes(), (k, a[k], b[k])
        else:
            assert a[k] == b[k] or (a[k] != a[k] and b[k] != b[k]), (k, a[k], b[k])


def _single(P, ctx, params, idx, tnrm, src, step):
    s = P.Icp(ctx, params)
    s.set_target(idx, normals=tnrm)
    s.set_source(src, normals=P.Field(src, 4))
    hist = []
    while True:
        st = s.iterate(1 if step else 2 ** 31 - 1)
        hist.append((st, s.get_correspondences()))
        if not step or st["state"] != 0:
            break
    cloud = s.get_cloud(stride_floats=8)
    s.close()
    return hist, cloud


def _run_batch(b, P, srcs, step, device=False):
    allr = np.concatenate(srcs)
    off = np.concatenate([[0], np.cumsum([len(x) for x in srcs])])
    if device:
        import torch
        t = torch.from_numpy(allr).cuda()
        b.set_source_batch(t, off, normals=P.Field(t, 4))
    else:
        b.set_source_batch(allr, off, normals=P.Field(allr, 4))
    hist = []
    while True:
        st = b.iterate_batch(1 if step else 2 ** 31 - 1)
        hist.append((st, b.get_correspondences_batch()))
        if not step or all(x["state"] != 0 for x in st):
            break
    return hist, b.get_cloud(stride_floats=8), off


def _batch(P, ctx, params, idx, tnrm, srcs, step, device=False):
    b = P.Icp(ctx, params)
    if device:
        import torch
        tnrm = None if tnrm is None else [torch.from_numpy(x).cuda() for x in tnrm]
    b.set_target_batch(idx, normals=tnrm)
    out = _run_batch(b, P, srcs, step, device)
    b.close()
    return out


def _check_equal(P, ctx, params, idx, tnrm, srcs, step):
    bh, bcloud, off = _batch(P, ctx, params, idx, tnrm, srcs, step)
    for p, src in enumerate(srcs):
        sh, scloud = _single(P, ctx, params, idx[p], None if tnrm is None else tnrm[p], src, step)
        # the batch keeps stepping until every problem is done; a finished problem's stats and lists stay put
        for k, (bst, bcorr) in enumerate(bh):
            sst, scorr = sh[min(k, len(sh) - 1)]
            _same_stats(bst[p], sst)
            assert bcorr[p].tobytes() == scorr.tobytes(), (p, k)
        assert bcloud[off[p]:off[p + 1]].tobytes() == scloud.tobytes(), p
    return bh


@pytest.mark.parametrize("est", list(ESTIMATORS))
@pytest.mark.parametrize("dbl", [False, True])
@pytest.mark.parametrize("track", [0, 1, 2])
@pytest.mark.parametrize("step", [False, True])
def test_pairs_batch_equals_single_sessions(pairs, est, dbl, track, step):
    P, ctx, idx, tnrm, srcs = pairs
    bh = _check_equal(P, ctx, _params(P, est, dbl, track), idx, tnrm, srcs, step)
    final = bh[-1][0]
    assert final[5]["state"] == 5  # NO_CORRESPONDENCES
    assert len({x["iterations"] for x in final}) > 2  # the problems stop after different numbers of iterations


def test_one_target_repeated_is_the_one_target_batch(pairs):
    """set_target_batch with one index B times gives the bytes of set_target + set_source_batch"""
    P, ctx, idx, tnrm, srcs = pairs
    params = _params(P, "point_to_plane", False, 2)
    same = [srcs[0], srcs[4], srcs[8]]  # the three problems of target 0
    a = P.Icp(ctx, params)
    a.set_target(idx[0], normals=tnrm[0])
    ha, ca, _ = _run_batch(a, P, same, False)
    b = P.Icp(ctx, params)
    b.set_target_batch([idx[0]] * 3, normals=[tnrm[0]] * 3)
    hb, cb, _ = _run_batch(b, P, same, False)
    for x, y in zip(ha[-1][0], hb[-1][0]):
        _same_stats(x, y)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(ha[-1][1], hb[-1][1]))
    assert ca.tobytes() == cb.tobytes()
    a.close()
    b.close()


@pytest.mark.parametrize("B", [1, 512])
def test_sizes(pairs, B):
    P, ctx, idx, tnrm, srcs = pairs
    r = np.random.default_rng(B)
    pick = r.integers(0, len(idx), B)
    pick[0] = 1
    sub = [srcs[k][r.choice(len(srcs[k]), 300, replace=False)] for k in pick]
    _check_equal(P, ctx, _params(P, "point_to_plane", False, 0), [idx[k] for k in pick], [tnrm[k] for k in pick], sub,
                 False)


def test_device_inputs(pairs):
    pytest.importorskip("torch")
    P, ctx, idx, tnrm, srcs = pairs
    params = _params(P, "point_to_plane", False, 0)
    host = _batch(P, ctx, params, idx, tnrm, srcs, False)
    dev = _batch(P, ctx, params, idx, tnrm, srcs, False, device=True)
    for (hs, hc), (ds, dc) in zip(host[0], dev[0]):
        for a, b in zip(hs, ds):
            _same_stats(a, b)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(hc, dc))
    assert host[1].tobytes() == dev[1].tobytes()


def test_launches_do_not_grow_with_the_targets(gpu):
    P, ctx = gpu
    r = np.random.default_rng(5)
    params = _params(P, "point_to_plane", False, 0, transformation_epsilon=0.0, euclidean_fitness_epsilon=-1.0,
                     max_iterations=100)
    tgts = [_surface(r.random((3000, 2)) * 2.0, 1.0, np.array([3.0 * k, 0.0, 0.0])) for k in range(64)]
    idx = [P.Index(ctx, np.ascontiguousarray(t[:, :4])) for t in tgts]
    nrm = [np.ascontiguousarray(t[:, 4:8]) for t in tgts]
    srcs = [_moved(t[:2000], 1.0, np.array([0.01, 0, 0]), t[:, :3].mean(0)) for t in tgts]
    counts = []
    for B in (1, 64):
        b = P.Icp(ctx, params)
        b.set_target_batch(idx[:B], normals=nrm[:B])
        allr = np.concatenate(srcs[:B])
        b.set_source_batch(allr, np.arange(B + 1) * 2000)
        b.iterate_batch(1)  # the first call also seeds; compare the steady calls
        before = ctx.launches
        st = b.iterate_batch(3)
        counts.append(ctx.launches - before)
        assert all(x["iterations"] == 4 for x in st)
        b.close()
    assert counts[0] == counts[1], counts


def test_refusals_and_recovery(pairs):
    P, ctx, idx, tnrm, srcs = pairs
    params = _params(P, "point_to_plane", False, 2)
    two = [srcs[1], srcs[2]]
    b = P.Icp(ctx, params)

    def refused(fn):
        with pytest.raises(P.Pclb200Error) as e:
            fn()
        assert e.value.code == P.ERR_INVALID

    b.set_target_batch(idx[1:3], normals=tnrm[1:3])
    allr = np.concatenate(two)
    off = [0, len(two[0]), len(allr)]
    b.set_source_batch(allr, off, normals=P.Field(allr, 4))  # every refusal below must leave this batch as it is
    refused(lambda: b.set_source_batch(allr, [0, 10, 20, len(allr)]))           # 3 problems for 2 targets
    refused(lambda: b.set_target_batch([]))                                      # no target
    set_tb = P.lib().pclb200_icp_set_target_batch
    h2 = (P.C.c_void_p * 2)(idx[1].h, None)
    assert set_tb(b.h, h2, None, 0, 2) == P.ERR_INVALID                          # a NULL handle
    assert set_tb(b.h, None, None, 0, 1) == P.ERR_INVALID                        # a NULL array
    assert set_tb(b.h, h2, None, 0, 65537) == P.ERR_INVALID                      # more than 65536
    refused(lambda: b.set_target_batch(idx[1:3], normals=[tnrm[1], None]))       # LLS without some problem's normals
    refused(lambda: b.set_target_batch(idx[1:3]))
    refused(lambda: b.set_source(two[0], normals=P.Field(two[0], 4)))             # a single source
    b.set_rejectors([(P.REJ_DISTANCE, 0.01, 0)])
    refused(lambda: b.set_target_batch(idx[1:3], normals=tnrm[1:3]))
    b.set_rejectors([])
    for kw in (dict(use_reciprocal=1), dict(correspondence_kind=P.CORR_NORMAL_SHOOTING)):
        P.lib().pclb200_icp_set_params(b.h, _params(P, "point_to_plane", False, 2, **kw))
        refused(lambda: b.set_target_batch(idx[1:3], normals=tnrm[1:3]))
        refused(lambda: b.iterate_batch())
    P.lib().pclb200_icp_set_params(b.h, params)
    # still usable: the batch set before the refusals, each problem as a fresh session
    got = b.iterate_batch()
    fresh, fresh_cloud, _ = _batch(P, ctx, params, idx[1:3], tnrm[1:3], two, False)
    for a, c in zip(got, fresh[-1][0]):
        _same_stats(a, c)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(b.get_correspondences_batch(), fresh[-1][1]))
    assert b.get_cloud(stride_floats=8).tobytes() == fresh_cloud.tobytes()
    # a new batch of targets drops the source: iterate_batch needs set_source_batch again
    b.set_target_batch(idx[1:3], normals=tnrm[1:3])
    refused(lambda: b.iterate_batch())
    refused(lambda: b.get_cloud())
    # set_target returns the session to one target: a single source, then a one-target batch
    b.set_target(idx[1], normals=tnrm[1])
    b.set_source(two[0], normals=P.Field(two[0], 4))
    st = b.iterate()
    sh, scloud = _single(P, ctx, params, idx[1], tnrm[1], two[0], False)
    _same_stats(st, sh[-1][0])
    assert b.get_correspondences().tobytes() == sh[-1][1].tobytes()
    assert b.get_cloud(stride_floats=8).tobytes() == scloud.tobytes()
    b.close()
