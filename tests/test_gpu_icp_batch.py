"""A batch of ICP problems in one session (include/pclb200_batch.h) against single sessions: per problem, every stats
field, every iteration's correspondences and the aligned records are byte-equal to a fresh session given the same
target and set_source(its records, its guess).  Needs an H100: run with -m gpu."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_MAP = 300_000


@pytest.fixture(scope="module")
def gpu():
    import pcl_b200
    pcl_b200.lib()
    ctx = pcl_b200.Context(0)
    yield pcl_b200, ctx
    ctx.close()


def _surface(xy):
    """PointNormal records (n, 8) on z = 0.1 sin(3x) + 0.1 cos(4y) with their analytic normals"""
    z = 0.1 * np.sin(3 * xy[:, 0]) + 0.1 * np.cos(4 * xy[:, 1])
    nrm = np.stack([-0.3 * np.cos(3 * xy[:, 0]), 0.4 * np.sin(4 * xy[:, 1]), np.ones(len(xy))], 1)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    out = np.zeros((len(xy), 8), np.float32)
    out[:, 0:2], out[:, 2], out[:, 3], out[:, 4:7] = xy, z, 1.0, nrm
    return out


def _moved(rec, deg, t, axis=2):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    R = {2: [[c, -s, 0], [s, c, 0], [0, 0, 1]], 0: [[1, 0, 0], [0, c, -s], [0, s, c]]}[axis]
    R = np.array(R)
    out = rec.copy()
    out[:, 0:3] = rec[:, 0:3].astype(np.float64) @ R.T + t
    out[:, 4:7] = rec[:, 4:7].astype(np.float64) @ R.T
    return out


@pytest.fixture(scope="module")
def scene(gpu):
    P, ctx = gpu
    r = np.random.default_rng(11)
    tgt = _surface(r.random((N_MAP, 2)) * 2.0)
    idx = P.Index(ctx, np.ascontiguousarray(tgt[:, :4]))
    sizes = [20000, 5000, 777, 12345, 2, 3001, 257, 8000, 1500, 33, 9999, 640]
    motions = [(1.5, (0.004, -0.003, 0.002)), (0.2, (0.001, 0, 0)), (3.0, (0.01, 0.01, -0.005)), (0.0, (0, 0, 0)),
               (0.5, (0.002, 0, 0)), (2.0, (-0.006, 0.004, 0.001)), (1.0, (0, 0.003, 0)), (4.0, (0.02, -0.01, 0.004)),
               (0.7, (0.003, 0.003, 0.003)), (0.1, (0, 0, 0.001)), (2.5, (0.008, 0, -0.002)), (1.2, (0, -0.004, 0))]
    srcs = []
    for i, (n, (deg, t)) in enumerate(zip(sizes, motions)):
        s = _moved(_surface(0.2 + r.random((n, 2)) * 1.6), deg, t, axis=2 if i % 2 == 0 else 0)
        srcs.append(s)
    srcs[5][:, 0:3] += np.float32(50.0)  # out of reach: NO_CORRESPONDENCES
    srcs[7][::97, 0] = np.nan             # NaN records, is_dense = 0
    srcs[7][5, 5] = np.nan                # and a NaN normal
    return P, ctx, tgt, idx, srcs


ESTIMATORS = {"svd": dict(estimator=0), "svd_no_umeyama": dict(estimator=0, svd_no_umeyama=1),
              "point_to_plane": dict(estimator=1), "symmetric": dict(estimator=2, with_normals_transform=1)}


def _params(P, est, dbl, track, **kw):
    base = dict(max_iterations=40, transformation_epsilon=1e-9, max_correspondence_distance=0.05, is_dense=0,
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


def _single(P, ctx, params, idx, tnrm, src, guess, step):
    s = P.Icp(ctx, params)
    s.set_target(idx, normals=tnrm)
    s.set_source(src, normals=P.Field(src, 4), guess=guess)
    hist = []
    while True:
        st = s.iterate(1 if step else 2 ** 31 - 1)
        hist.append((st, s.get_correspondences()))
        if not step or st["state"] != 0:
            break
    cloud = s.get_cloud(stride_floats=8)
    s.close()
    return hist, cloud


def _batch(P, ctx, params, idx, tnrm, srcs, guesses, step, device=False):
    allr = np.concatenate(srcs)
    off = np.concatenate([[0], np.cumsum([len(x) for x in srcs])])
    b = P.Icp(ctx, params)
    b.set_target(idx, normals=tnrm)
    if device:
        import torch
        t = torch.from_numpy(allr).cuda()
        b.set_source_batch(t, off, normals=P.Field(t, 4), guesses=guesses)
    else:
        b.set_source_batch(allr, off, normals=P.Field(allr, 4), guesses=guesses)
    hist = []
    while True:
        st = b.iterate_batch(1 if step else 2 ** 31 - 1)
        hist.append((st, b.get_correspondences_batch()))
        if not step or all(x["state"] != 0 for x in st):
            break
    cloud = b.get_cloud(stride_floats=8)
    b.close()
    return hist, cloud, off


def _check_equal(P, ctx, params, idx, tnrm, srcs, guesses, step, device=False):
    bh, bcloud, off = _batch(P, ctx, params, idx, tnrm, srcs, guesses, step, device)
    for p, src in enumerate(srcs):
        g = None if guesses is None else guesses[p]
        sh, scloud = _single(P, ctx, params, idx, tnrm, src, g, step)
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
def test_scan_to_map_batch_equals_single_sessions(scene, est, dbl, track, step):
    P, ctx, tgt, idx, srcs = scene
    params = _params(P, est, dbl, track)
    tnrm = np.ascontiguousarray(tgt[:, 4:8])
    bh = _check_equal(P, ctx, params, idx, tnrm, srcs, None, step)
    final = bh[-1][0]
    assert final[5]["state"] == 5  # NO_CORRESPONDENCES
    assert len({x["iterations"] for x in final}) > 2  # the problems stop after different numbers of iterations


def test_multi_hypothesis_bun0_bun4(gpu, golden):
    P, ctx = gpu
    src, tgt = P.xyz1(golden["bun0"]), P.xyz1(golden["bun4"])
    idx = P.Index(ctx, tgt)
    r = np.random.default_rng(3)
    guesses = np.tile(np.eye(4), (32, 1, 1))
    for g in guesses[1:]:
        a = np.deg2rad(r.uniform(-8, 8, 3))
        cx, cy, cz, sx, sy, sz = *np.cos(a), *np.sin(a)
        g[:3, :3] = (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
                     @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))
        g[:3, 3] = r.uniform(-0.01, 0.01, 3)
    params = P.default_params(max_iterations=50, transformation_epsilon=1e-8, max_correspondence_distance=0.05)
    b = P.Icp(ctx, params)
    b.set_target(idx)
    off = np.arange(33) * len(src)
    b.set_source_batch(np.tile(src, (32, 1)), off, guesses=guesses)
    st = b.iterate_batch()
    corr = b.get_correspondences_batch()
    cloud = b.get_cloud()
    for p in range(32):
        s = P.Icp(ctx, params)
        s.set_target(idx)
        s.set_source(src, guess=guesses[p])
        _same_stats(st[p], s.iterate())
        assert corr[p].tobytes() == s.get_correspondences().tobytes()
        assert cloud[off[p]:off[p + 1]].tobytes() == s.get_cloud().tobytes()
        s.close()
    T, G = st[0]["final"], golden["icp_bun0_bun4"]
    tol = np.full((4, 4), 1e-3)
    tol[0, 1] = 1e-2
    tol[3, :] = 0
    assert st[0]["converged"] and np.all(np.abs(T - G) <= tol), (T, st[0])


@pytest.mark.parametrize("B", [1, 512])
def test_sizes(scene, B):
    P, ctx, tgt, idx, _ = scene
    r = np.random.default_rng(B)
    srcs = [_moved(_surface(0.2 + r.random((500, 2)) * 1.6), r.uniform(0, 3), r.uniform(-0.005, 0.005, 3))
            for _ in range(B)]
    _check_equal(P, ctx, _params(P, "point_to_plane", False, 0), idx, np.ascontiguousarray(tgt[:, 4:8]), srcs, None,
                 False)


def test_device_inputs(scene):
    pytest.importorskip("torch")
    P, ctx, tgt, idx, srcs = scene
    params = _params(P, "svd", False, 0)
    host = _batch(P, ctx, params, idx, None, srcs, None, False)
    dev = _batch(P, ctx, params, idx, None, srcs, None, False, device=True)
    for (hs, hc), (ds, dc) in zip(host[0], dev[0]):
        for a, b in zip(hs, ds):
            _same_stats(a, b)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(hc, dc))
    assert host[1].tobytes() == dev[1].tobytes()


def test_launches_do_not_grow_with_the_batch(scene):
    P, ctx, tgt, idx, srcs = scene
    params = _params(P, "point_to_plane", False, 0, transformation_epsilon=0.0, euclidean_fitness_epsilon=-1.0,
                     max_iterations=100)
    tnrm = np.ascontiguousarray(tgt[:, 4:8])
    counts = []
    for B in (1, 64):
        allr = np.concatenate([srcs[0][:3000]] * B)
        b = P.Icp(ctx, params)
        b.set_target(idx, normals=tnrm)
        b.set_source_batch(allr, np.arange(B + 1) * 3000)
        b.iterate_batch(1)  # the first call also seeds; compare the steady calls
        before = ctx.launches
        st = b.iterate_batch(3)
        counts.append(ctx.launches - before)
        assert all(x["iterations"] == 4 for x in st)
        b.close()
    assert counts[0] == counts[1], counts


def test_refusals_and_recovery(scene):
    P, ctx, tgt, idx, srcs = scene
    params = _params(P, "svd", False, 2)
    src = srcs[2]
    b = P.Icp(ctx, params)
    b.set_target(idx)

    def refused(fn):
        with pytest.raises(P.Pclb200Error) as e:
            fn()
        assert e.value.code == P.ERR_INVALID

    n = len(src)
    b.set_source_batch(src, [0, 100, n])  # every refusal below must leave this batch as it is
    refused(lambda: b.set_source_batch(src, [0]))                       # B = 0
    refused(lambda: b.set_source_batch(np.zeros((65537, 4), np.float32), np.arange(65538)))  # B > 65536
    refused(lambda: b.set_source_batch(src, [1, n]))                    # does not start at 0
    refused(lambda: b.set_source_batch(src, [0, 10, 10, n]))            # an empty problem
    refused(lambda: b.set_source_batch(src, [0, 10, n - 1]))            # does not end at n
    big = P.lib().pclb200_icp_set_source_batch
    off = np.array([0, 2 ** 31 - 1], np.int64)
    assert big(b.h, src.ctypes.data, 2 ** 31 - 1, 32, None, 0, off.ctypes.data, 1, None) == P.ERR_INVALID
    b.set_rejectors([(P.REJ_DISTANCE, 0.01, 0)])
    refused(lambda: b.set_source_batch(src, [0, n]))
    b.set_rejectors([])
    for kw in (dict(use_reciprocal=1), dict(correspondence_kind=P.CORR_NORMAL_SHOOTING), dict(estimator=2)):
        bad = _session(P, ctx, idx, _params(P, "svd", False, 2, **kw))
        refused(lambda: bad.set_source_batch(src, [0, n]))
        bad.close()
    refused(lambda: b.iterate())
    refused(lambda: b.get_correspondences())
    P.lib().pclb200_icp_set_params(b.h, P.default_params(use_reciprocal=1))
    refused(lambda: b.iterate_batch())
    P.lib().pclb200_icp_set_params(b.h, params)
    # still usable: the batch set before the refusals, then a single source, each as a fresh session
    fresh, fresh_cloud, _ = _batch(P, ctx, params, idx, None, [src[:100], src[100:]], None, False)
    got = b.iterate_batch()
    for a, c in zip(got, fresh[-1][0]):
        _same_stats(a, c)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(b.get_correspondences_batch(), fresh[-1][1]))
    assert b.get_cloud(stride_floats=8).tobytes() == fresh_cloud.tobytes()
    b.set_source(src, normals=P.Field(src, 4))
    st = b.iterate()
    sh, scloud = _single(P, ctx, params, idx, None, src, None, False)
    _same_stats(st, sh[-1][0])
    assert b.get_correspondences().tobytes() == sh[-1][1].tobytes()
    assert b.get_cloud(stride_floats=8).tobytes() == scloud.tobytes()
    assert len(got) == 2
    b.close()


def _session(P, ctx, idx, params):
    s = P.Icp(ctx, params)
    s.set_target(idx)
    return s
