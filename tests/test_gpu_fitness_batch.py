"""The fitness score of a batch of registrations in one call (include/pclb200_batch.h: pclb200_fitness_score_batch,
pclb200_validate_transformation_batch, pclb200_icp_fitness_score_batch) against one pclb200_fitness_score /
pclb200_validate_transformation per problem: every score as raw bytes, for float and double Scalar and max_range = DBL_MAX,
a value that drops some pairs, and 0; handles from single and batch builds, a repeated handle, identity, random and
far-away transforms, an all-NaN problem, strides 12 / 16 / 48, host and device arrays, B = 1 and 512, a 1 M-point problem
among small ones.  The session form equals the single call on each problem's final transformation before, between and
after iterations, and leaves the next iterate_batch unchanged.  Equal launch counts for B = 8 and 64; refusals that leave
the scores untouched; raw scans through the voxel, build, normals, align and score batches equal the loop of single calls.
Needs an H100: run with -m gpu."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_index_batch import _batch_input, _chain, _kinds, _records

pytestmark = pytest.mark.gpu

DBL_MAX = np.finfo(np.float64).max
RANGES = (DBL_MAX, 1e-4, 0.0)


@pytest.fixture(scope="module")
def gpu():
    import pcl_b200
    pcl_b200.lib()
    ctx = pcl_b200.Context(0)
    yield pcl_b200, ctx
    ctx.close()


def _rigid(r, angle, shift):
    """a rotation of `angle` about a random axis, then a translation of length `shift` (row-major 4x4)"""
    ax = r.normal(size=3)
    ax /= np.linalg.norm(ax)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K
    d = r.normal(size=3)
    T[:3, 3] = shift * d / np.linalg.norm(d)
    return T


def _problems(targets, seed):
    """per target cloud: a source of noisy target points (NaN and Inf among them on some), and a transform that is the
    identity, a small random motion or a move 1e3 away; one problem holds NaN records only"""
    r = np.random.default_rng(seed)
    srcs, Ts = [], []
    for j, t in enumerate(targets):
        fin = t[np.isfinite(t).all(1)]
        m = int(min(len(fin) + 5, 2000))
        s = (fin[r.integers(0, len(fin), m)] + r.normal(0, 0.01, (m, 3))).astype(np.float32)
        if j % 4 == 1:
            s[::13, j % 3] = np.nan
            s[5::17, (j + 1) % 3] = np.inf
        if j == 2:
            s[:] = np.nan
        srcs.append(s)
        Ts.append([np.eye(4), _rigid(r, 0.02, 0.01), _rigid(r, 0.3, 1e3)][j % 3])
    return srcs, np.array(Ts)


def _handles(P, ctx, targets, batch_built):
    """the targets' handles; problem 1 repeats problem 0's handle"""
    if batch_built:
        allt, toff, _ = _batch_input(targets, 16, False)
        built = ctx.index_build_batch(allt, toff)
    else:
        built = [P.Index(ctx, _records(t, 16)) for t in targets]
    handles = list(built)
    if len(handles) > 2:
        handles[1] = built[0]
    return built, handles


def _compare(P, ctx, handles, srcs, Ts, stride, device, ranges=RANGES):
    allr, off, host = _batch_input(srcs, stride, device)
    for validate in (False, True):
        for dbl in (False, True):
            for mr in ranges:
                if validate:
                    got = ctx.validate_transformation_batch(handles, allr, off, Ts, max_range=mr, scalar_is_double=dbl)
                else:
                    got = ctx.fitness_score_batch(handles, allr, off, Ts.reshape(-1, 16), max_range=mr, scalar_is_double=dbl)
                assert got.dtype == np.float64 and got.shape == (len(srcs),)
                for p, h in enumerate(handles):
                    rec = host[off[p]:off[p + 1]]
                    single = (h.validate_transformation(rec, Ts[p], max_range=mr, scalar_is_double=dbl) if validate else
                              h.fitness_score(rec, Ts[p], max_range=mr, scalar_is_double=dbl))
                    assert got[p:p + 1].tobytes() == np.float64(single).tobytes(), (validate, dbl, mr, p, got[p], single)


@pytest.mark.parametrize("stride,device,batch_built", [(16, False, False), (12, False, True), (48, False, False),
                                                       (16, True, True), (48, True, False)])
def test_scores_equal_single_calls(gpu, stride, device, batch_built):
    """the index-batch kinds of cloud as targets (each twice), against one fitness_score / validate_transformation per
    problem"""
    if device:
        pytest.importorskip("torch")
    P, ctx = gpu
    targets = [c for _, c in _kinds(stride)] * 2
    built, handles = _handles(P, ctx, targets, batch_built)
    srcs, Ts = _problems(targets, stride)
    _compare(P, ctx, handles, srcs, Ts, stride, device)
    allr, off, _ = _batch_input(srcs, stride, False)
    got = ctx.fitness_score_batch(handles, allr, off, Ts)
    assert got[2] == DBL_MAX  # the all-NaN problem
    assert (got[np.arange(len(srcs)) != 2] < DBL_MAX).all()
    for h in built:
        h.close()


def test_one_problem_and_512_problems(gpu):
    P, ctx = gpu
    r = np.random.default_rng(3)
    one = [(r.random((5000, 3)) * [4, 4, 0.3]).astype(np.float32)]
    built, handles = _handles(P, ctx, one, False)
    srcs, Ts = _problems(one, 1)
    Ts[0] = _rigid(r, 0.05, 0.02)
    _compare(P, ctx, handles, srcs, Ts, 16, False)
    for h in built:
        h.close()
    kinds = [c for _, c in _kinds(5)]
    targets = [kinds[j % len(kinds)] if j % 4 else (r.random((int(r.integers(20, 3000)), 3)) * 2).astype(np.float32)
               for j in range(512)]
    built, handles = _handles(P, ctx, targets, True)
    srcs, Ts = _problems(targets, 2)
    _compare(P, ctx, handles, srcs, Ts, 16, False, ranges=(DBL_MAX, 1e-4))
    for h in built:
        h.close()


def test_million_point_problem_among_small(gpu):
    P, ctx = gpu
    r = np.random.default_rng(4)
    targets = [c for _, c in _kinds(9)]
    big = (r.random((1 << 20, 3)) * np.array([50, 50, 4]) - 20).astype(np.float32)
    targets.insert(3, big)
    built, handles = _handles(P, ctx, targets, True)
    srcs, Ts = _problems(targets, 4)
    srcs[3] = (big + r.normal(0, 0.01, big.shape)).astype(np.float32)
    _compare(P, ctx, handles, srcs, Ts, 16, False, ranges=(DBL_MAX, 1e-4))
    for h in built:
        h.close()


def _session(P, ctx, tg, src, est, per_target, dbl, guesses):
    """a batch session over the pairs (tg[p], src[p]): one target per problem, or tg[0] for every problem"""
    params = P.default_params(max_iterations=30, transformation_epsilon=1e-9, max_correspondence_distance=0.3,
                              estimator=est, track_mode=P.TRACK_AUTO, scalar_is_double=int(dbl))
    toff = np.concatenate([[0], np.cumsum([len(w) for w in tg])]).astype(np.int64)
    tidx = ctx.index_build_batch(np.concatenate(tg), toff)
    nrm = [i.normals_knn(w, 16)[0] for i, w in zip(tidx, tg)] if est == 1 else None
    s = P.Icp(ctx, params)
    if per_target:
        s.set_target_batch(tidx, normals=nrm)
    else:
        s.set_target(tidx[0], normals=None if nrm is None else nrm[0])
    soff = np.concatenate([[0], np.cumsum([len(w) for w in src])]).astype(np.int64)
    s.set_source_batch(np.concatenate(src), soff, guesses=guesses)
    return s, tidx, soff


def _check_session(ctx, s, tidx, src, soff, st, per_target, dbl):
    """the session's scores equal a single fitness_score and the free batch call on every final transformation"""
    finals = np.array([x["final"] for x in st])
    handles = list(tidx) if per_target else [tidx[0]] * len(src)
    allr = np.concatenate(src)
    for mr in (DBL_MAX, 1e-3, 0.0):
        got = s.fitness_score_batch(mr)
        free = ctx.fitness_score_batch(handles, allr, soff, finals, max_range=mr, scalar_is_double=dbl)
        assert got.tobytes() == free.tobytes(), mr
        for p in range(len(src)):
            one = handles[p].fitness_score(src[p], finals[p], max_range=mr, scalar_is_double=dbl)
            assert got[p:p + 1].tobytes() == np.float64(one).tobytes(), (mr, p)


def _same_stats(sa, sb):
    for p, (a, b) in enumerate(zip(sa, sb)):
        for key in a:
            x, y = a[key], b[key]
            assert (x.tobytes() == y.tobytes()) if isinstance(x, np.ndarray) else (x == y or (x != x and y != y)), (p, key)


@pytest.mark.parametrize("est,per_target,dbl", [(0, True, False), (1, True, True), (0, False, True), (1, False, False)],
                         ids=["svd-targets-float", "plane-targets-double", "svd-one-target-double", "plane-one-target-float"])
def test_session_scores(gpu, est, per_target, dbl):
    """before any iteration (the guesses), between steps of max_steps = 1 and after convergence, the session's scores are
    the single call's on stats[p].final_transformation; a session that scores between steps iterates, matches and moves
    its source exactly as one that does not"""
    P, ctx = gpu
    wins = _chain(12, 3000, 31)
    tg, src = wins[:-1], wins[1:]
    r = np.random.default_rng(5)
    guesses = np.array([_rigid(r, 0.01, 0.02) if p % 2 else np.eye(4) for p in range(len(src))])
    a, tidx, soff = _session(P, ctx, tg, src, est, per_target, dbl, guesses)
    b, tidx_b, _ = _session(P, ctx, tg, src, est, per_target, dbl, guesses)
    st0 = a.iterate_batch(0)
    _check_session(ctx, a, tidx, src, soff, st0, per_target, dbl)
    for _ in range(3):
        sa = a.iterate_batch(1)
        _check_session(ctx, a, tidx, src, soff, sa, per_target, dbl)
        sb = b.iterate_batch(1)
        _same_stats(sa, sb)
        for x, y in zip(a.get_correspondences_batch(), b.get_correspondences_batch()):
            assert x.tobytes() == y.tobytes()
        assert a.get_cloud().tobytes() == b.get_cloud().tobytes()
    a.fitness_score_batch()
    sa, sb = a.iterate_batch(), b.iterate_batch()
    _same_stats(sa, sb)
    for x, y in zip(a.get_correspondences_batch(), b.get_correspondences_batch()):
        assert x.tobytes() == y.tobytes()
    assert a.get_cloud().tobytes() == b.get_cloud().tobytes()
    _check_session(ctx, a, tidx, src, soff, sa, per_target, dbl)
    a.close()
    b.close()
    for i in tidx + tidx_b:
        i.close()


def test_launches_independent_of_batch_size(gpu):
    P, ctx = gpu
    r = np.random.default_rng(9)
    free, session = [], []
    for B in (8, 64):
        clouds = [(r.random((500 + 37 * b, 3)) * 3).astype(np.float32) for b in range(B)]
        src, off, _ = _batch_input(clouds, 16, False)
        hs = ctx.index_build_batch(src, off)
        Ts = np.array([_rigid(r, 0.01, 0.01) for _ in range(B)])
        before = ctx.launches
        ctx.fitness_score_batch(hs, src, off, Ts)
        free.append(ctx.launches - before)
        s = P.Icp(ctx, P.default_params(max_correspondence_distance=0.3))
        s.set_target_batch(hs)
        s.set_source_batch(src, off, guesses=Ts)
        before = ctx.launches
        s.fitness_score_batch()
        session.append(ctx.launches - before)
        s.close()
        for h in hs:
            h.close()
    assert free[0] == free[1] and session[0] == session[1], (free, session)


def test_refusals_leave_scores_untouched(gpu):
    P, ctx = gpu
    L = P.lib()
    clouds = [(np.random.default_rng(j).random((300, 3)) * 2).astype(np.float32) for j in range(3)]
    rec = np.concatenate([_records(c, 16) for c in clouds])
    off = np.array([0, 300, 600, 900], np.int64)
    hs = [P.Index(ctx, _records(c, 16)) for c in clouds]
    tagged = (C.c_void_p * 3)(*[h.h for h in hs])
    with_null = (C.c_void_p * 3)(hs[0].h, None, hs[2].h)
    T = np.tile(np.eye(4), (3, 1, 1))
    vp = lambda a: C.c_void_p(a.ctypes.data)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    cases = [  # (handles, B, records, n, stride, offsets, transforms)
        (tagged, 0, rec, 900, 16, off, T),
        (tagged, 65537, rec, 900, 16, off, T),
        (None, 3, rec, 900, 16, off, T),
        (with_null, 3, rec, 900, 16, off, T),
        (tagged, 3, None, 900, 16, off, T),
        (tagged, 3, rec, 900, 16, None, T),
        (tagged, 3, rec, 900, 16, off, None),
        (tagged, 3, rec, 900, 16, np.array([1, 300, 600, 900], np.int64), T),
        (tagged, 3, rec, 900, 16, np.array([0, 300, 300, 900], np.int64), T),
        (tagged, 3, rec, 900, 16, np.array([0, 300, 600, 800], np.int64), T),
        (tagged, 3, rec, 2 ** 31 - 1, 16, np.array([0, 300, 600, 2 ** 31 - 1], np.int64), T),
        (tagged, 3, rec, 900, 10, off, T),
        (tagged, 3, rec, 900, 8, off, T),
    ]
    for fn in (L.pclb200_fitness_score_batch, L.pclb200_validate_transformation_batch):
        for j, (h, B, r_, n, stride, o, t) in enumerate(cases):
            scores = np.full(3, 7.0)
            rc = fn(ctx.h, h, B, None if r_ is None else vp(r_), n, stride, None if o is None else vp(o),
                    None if t is None else dp(t), 0, DBL_MAX, dp(scores))
            assert rc == P.ERR_INVALID, (j, rc, L.pclb200_last_error())
            assert L.pclb200_last_error()
            assert (scores == 7.0).all(), j
        assert fn(ctx.h, tagged, 3, vp(rec), 900, 16, vp(off), dp(T), 0, DBL_MAX, None) == P.ERR_INVALID
    # the session form: no batch source (a fresh session; one whose source set_target_batch dropped), NULL scores
    s = P.Icp(ctx, P.default_params(max_correspondence_distance=0.3))
    scores = np.full(3, 7.0)
    assert L.pclb200_icp_fitness_score_batch(s.h, DBL_MAX, dp(scores)) == P.ERR_INVALID and (scores == 7.0).all()
    s.set_target_batch(hs)
    s.set_source_batch(rec, off)
    assert L.pclb200_icp_fitness_score_batch(s.h, DBL_MAX, None) == P.ERR_INVALID
    s.set_target_batch(hs)
    assert L.pclb200_icp_fitness_score_batch(s.h, DBL_MAX, dp(scores)) == P.ERR_INVALID and (scores == 7.0).all()
    assert L.pclb200_icp_fitness_score_batch(None, DBL_MAX, dp(scores)) == P.ERR_INVALID and (scores == 7.0).all()
    # the context and the session still work
    s.set_source_batch(rec, off)
    st = s.iterate_batch()
    got = s.fitness_score_batch()
    free = ctx.fitness_score_batch(hs, rec, off, np.array([x["final"] for x in st]))
    assert got.tobytes() == free.tobytes()
    for p in range(3):
        one = hs[p].fitness_score(rec[off[p]:off[p + 1]], st[p]["final"])
        assert got[p:p + 1].tobytes() == np.float64(one).tobytes(), p
    s.close()
    for h in hs:
        h.close()


@pytest.mark.parametrize("est", [1, 0], ids=["point_to_plane", "svd"])
def test_raw_scans_to_scored_pairs(gpu, est):
    """raw target and source windows through voxelgrid_batch, index_build_batch, normals_knn_batch, one batch align and
    one batch score: every problem's stats and score equal the loop of single voxelgrid, Index, normals_knn, one session
    per pair and fitness_score"""
    P, ctx = gpu
    wins = _chain(16, 12000, 21)
    tg, src = wins[:-1], wins[1:]
    leaf = (0.06, 0.06, 0.06)
    params = P.default_params(max_iterations=30, transformation_epsilon=1e-9, max_correspondence_distance=0.3,
                              estimator=est, track_mode=P.TRACK_ON)
    B = len(tg)
    toff = np.concatenate([[0], np.cumsum([len(w) for w in tg])]).astype(np.int64)
    soff = np.concatenate([[0], np.cumsum([len(w) for w in src])]).astype(np.int64)
    trows, tro = ctx.voxelgrid_batch(np.concatenate(tg), toff, leaf)
    srows, sro = ctx.voxelgrid_batch(np.concatenate(src), soff, leaf)
    tidx = ctx.index_build_batch(trows, tro)
    nrm = None
    if est == 1:
        bn, _ = ctx.normals_knn_batch(tidx, trows, tro, 16)
        nrm = [bn[tro[p]:tro[p + 1]] for p in range(B)]
    s = P.Icp(ctx, params)
    s.set_target_batch(tidx, normals=nrm)
    s.set_source_batch(srows, sro)
    st = s.iterate_batch()
    scores = s.fitness_score_batch()
    gated = s.fitness_score_batch(0.01)
    s.close()
    one = P.Icp(ctx, params)
    kept = []
    for p in range(B):
        t = ctx.voxelgrid(tg[p], leaf)
        q = ctx.voxelgrid(src[p], leaf)
        idx = P.Index(ctx, t)
        kept.append(idx)
        one.set_target(idx, normals=idx.normals_knn(t, 16)[0] if est == 1 else None)
        one.set_source(q)
        st1 = one.iterate()
        _same_stats([st[p]], [st1])
        assert scores[p:p + 1].tobytes() == np.float64(idx.fitness_score(q, st1["final"])).tobytes(), p
        assert gated[p:p + 1].tobytes() == np.float64(idx.fitness_score(q, st1["final"], max_range=0.01)).tobytes(), p
    one.close()
    for i in tidx + kept:
        i.close()
