"""A batch of clouds indexed in one build (include/pclb200_batch.h: pclb200_index_build_batch) against one
pclb200_index_build per cloud: every handle answers size, stats, k-NN (per-thread and warp kernels), radius and k = 16
normals byte for byte as its cloud's single build does, and scan pairs aligned against batch-built targets
(set_target_batch) give the stats, correspondences and aligned records of single-built targets.  Needs an H100: run with
-m gpu."""
import ctypes as C

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


def _kinds(seed):
    """(name, (n, 3) float32): the clouds a batch is made of"""
    r = np.random.default_rng(seed)
    box = lambda n, w, shift=(0, 0, 0): (r.random((n, 3)) * w + np.array(shift)).astype(np.float32)
    out = [("1 point", box(1, 1.0, (-7, 3, 11))), ("8 points", box(8, 1.0)), ("9 points", box(9, 1.0))]
    c = box(256, 2.0)
    c[77, 1] = np.nan
    out += [("255 finite of 256", c), ("256 points", box(256, 2.0))]
    c = box(3000, 5.0, (-7, 3, 11))
    c[::97, 0] = np.nan
    c[5::97, 2] = -np.inf
    c[11, 1] = np.inf
    out.append(("NaN and Inf records", c))
    c = box(600, 1.0)
    c[100:140] = c[99]
    out.append(("identical points", c))
    out.append(("zero extent", np.tile(np.array([[1.5, -2.0, 0.25]], np.float32), (300, 1))))
    c = box(2000, 3.0, (-7, 3, 11))
    c[:, 2] = 11.0
    out.append(("planar", c))
    out += [("1e-3 wide far out", box(1500, 1e-3, (1e5, -2e5, 3e4))), ("1e4 wide far out", box(1500, 1e4, (1e5, -2e5, 3e4))),
            ("20 k points", box(20000, 10.0, (5, 5, 5)))]
    return out


def _records(xyz, stride):
    """xyz as records of `stride` bytes (xyz at offset 0; w = 1 from 16 bytes on)"""
    rec = np.full((len(xyz), stride // 4), 1.0, np.float32)
    rec[:, :3] = xyz
    return rec


def _same(a, b, what):
    if isinstance(a, tuple):
        for x, y in zip(a, b):
            _same(x, y, what)
    elif isinstance(a, np.ndarray):
        assert a.tobytes() == b.tobytes(), what
    else:
        assert a == b, what


def _queries(xyz, r):
    """the cloud's own points (a sample of large clouds) and points around it"""
    q = xyz if len(xyz) <= 4000 else xyz[r.choice(len(xyz), 4000, replace=False)]
    fin = xyz[np.isfinite(xyz).all(1)]
    ext = float(np.max(fin.max(0) - fin.min(0))) or 1.0
    near = fin[r.integers(0, len(fin), 500)] + (r.random((500, 3)) - 0.5) * ext * 0.1
    return np.ascontiguousarray(np.concatenate([q, near.astype(np.float32)])), ext


def _check_handle(P, ctx, bi, xyz, rec, name, seed=0):
    si = P.Index(ctx, rec)
    _same(bi.size, si.size, name + ": size")
    _same(bi.stats, si.stats, name + ": stats")
    q, ext = _queries(xyz, np.random.default_rng(seed))
    qr = _records(q, 16)
    for k in (1, 8, 16, 32):
        _same(bi.knn(qr, k), si.knn(qr, k), f"{name}: knn k = {k}")
    _same(bi.radius(qr, 0.03 * ext), si.radius(qr, 0.03 * ext), name + ": radius")
    _same(bi.normals_knn(rec, 16, is_dense=False), si.normals_knn(rec, 16, is_dense=False), name + ": normals")
    si.close()


def _batch_input(clouds, stride, device):
    allr = np.concatenate([_records(c, stride) for c in clouds])
    off = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int64)
    if device:
        import torch
        return torch.from_numpy(allr).cuda(), off, allr
    return allr, off, allr


@pytest.mark.parametrize("stride,device,big", [(16, False, True), (12, False, False), (48, False, False), (16, True, False),
                                               (48, True, False)])
def test_handles_answer_as_single_builds(gpu, stride, device, big):
    """every handle of a 37-cloud batch (the 1 M-point cloud among small ones once) against its cloud's single build"""
    if device:
        pytest.importorskip("torch")
    P, ctx = gpu
    kinds = _kinds(stride)
    r = np.random.default_rng(7 + stride)
    pick = list(range(len(kinds))) + list(r.integers(0, len(kinds), 37 - len(kinds)))
    r.shuffle(pick)
    clouds = [kinds[k][1] for k in pick]
    names = [kinds[k][0] for k in pick]
    if big:
        clouds.insert(5, (r.random((1 << 20, 3)) * np.array([50, 50, 4]) - 20).astype(np.float32))
        names.insert(5, "1 M points")
    src, off, host = _batch_input(clouds, stride, device)
    handles = ctx.index_build_batch(src, off)
    assert len(handles) == len(clouds)
    for c, (h, xyz, name) in enumerate(zip(handles, clouds, names)):
        assert h.n_cloud == len(xyz)
        _check_handle(P, ctx, h, xyz, host[off[c]:off[c + 1]], f"cloud {c} ({name})", c)
    for h in handles:
        h.close()


def _chain(B, n, seed):
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from bench_icp_pairs import make_chain
    return make_chain(B, n, seed)


@pytest.mark.parametrize("est", [0, 1])
def test_aligns_against_batch_built_targets(gpu, est):
    """set_target_batch with batch-built targets: every problem's stats (total_skipped_walks included: the skips depend on
    the tree the walks visit), last correspondences and aligned records equal those against single-built targets"""
    P, ctx = gpu
    wins = _chain(24, 3000, 11)
    tg, src = wins[:-1], wins[1:]
    off = np.concatenate([[0], np.cumsum([len(w) for w in tg])]).astype(np.int64)
    bidx = ctx.index_build_batch(np.concatenate(tg), off)
    sidx = [P.Index(ctx, w) for w in tg]
    nrm = [i.normals_knn(w, 16)[0] for i, w in zip(sidx, tg)] if est == 1 else None
    params = P.default_params(max_iterations=30, transformation_epsilon=1e-9, max_correspondence_distance=0.3,
                              estimator=est, track_mode=P.TRACK_ON)
    soff = np.concatenate([[0], np.cumsum([len(w) for w in src])]).astype(np.int64)
    runs = []
    for idx in (bidx, sidx):
        s = P.Icp(ctx, params)
        s.set_target_batch(idx, normals=nrm)
        s.set_source_batch(np.concatenate(src), soff)
        st = s.iterate_batch()
        runs.append((st, s.get_correspondences_batch(), s.get_cloud()))
        s.close()
    (sa, ca, pa), (sb, cb, pb) = runs
    assert sum(x["total_skipped_walks"] for x in sa) > 0
    for p in range(len(src)):
        for k in sa[p]:
            a, b = sa[p][k], sb[p][k]
            assert (a.tobytes() == b.tobytes()) if isinstance(a, np.ndarray) else (a == b or (a != a and b != b)), (p, k)
        assert ca[p].tobytes() == cb[p].tobytes(), p
    assert pa.tobytes() == pb.tobytes()
    for i in bidx + sidx:
        i.close()


def test_handles_destroyed_in_any_order(gpu):
    """handles closed one by one in shuffled order, with builds and searches in between: the rest still answer as their
    single builds"""
    P, ctx = gpu
    kinds = _kinds(3)
    clouds = [k[1] for k in kinds] * 2
    src, off, host = _batch_input(clouds, 16, False)
    handles = ctx.index_build_batch(src, off)
    order = np.random.default_rng(5).permutation(len(handles))
    alive = set(range(len(handles)))
    for step, c in enumerate(order):
        handles[c].close()
        alive.discard(c)
        other = P.Index(ctx, _records(kinds[step % len(kinds)][1], 16))  # other work on the context
        other.knn(_records(kinds[-1][1][:100], 16), 4)
        if alive and step % 4 == 0:
            d = min(alive)
            _check_handle(P, ctx, handles[d], clouds[d], host[off[d]:off[d + 1]], f"cloud {d} after {step + 1} closed")
        other.close()


def test_launches_independent_of_batch_size(gpu):
    P, ctx = gpu
    r = np.random.default_rng(9)
    counts = []
    for B in (1, 64):
        clouds = [(r.random((500 + 37 * b, 3)) * 3).astype(np.float32) for b in range(B)]
        src, off, _ = _batch_input(clouds, 12, False)
        before = ctx.launches
        hs = ctx.index_build_batch(src, off)
        counts.append(ctx.launches - before)
        for h in hs:
            h.close()
    assert counts[0] == counts[1], counts


def test_refusals_leave_no_handle(gpu):
    P, ctx = gpu
    L = P.lib()
    good = [(np.random.default_rng(k).random((300, 3)) * 2).astype(np.float32) for k in range(5)]
    nan_mid = [g.copy() for g in good]
    nan_mid[2][:] = np.nan
    rec = np.concatenate([_records(c, 16) for c in good])
    rec_nan = np.concatenate([_records(c, 16) for c in nan_mid])
    off = np.array([0, 300, 600, 900, 1200, 1500], np.int64)
    vp = lambda a: C.c_void_p(a.ctypes.data)
    cases = [  # (records, n, stride, offsets, n_clouds, expected code)
        (rec, 1500, 16, off, 0, P.ERR_INVALID),
        (rec, 1500, 16, off, 65537, P.ERR_INVALID),
        (None, 1500, 16, off, 5, P.ERR_INVALID),
        (rec, 1500, 16, None, 5, P.ERR_INVALID),
        (rec, 1500, 16, np.array([1, 300, 600, 900, 1200, 1500], np.int64), 5, P.ERR_INVALID),
        (rec, 1500, 16, np.array([0, 300, 300, 900, 1200, 1500], np.int64), 5, P.ERR_INVALID),
        (rec, 1500, 16, np.array([0, 300, 600, 900, 1200, 1400], np.int64), 5, P.ERR_INVALID),
        (rec, 2 ** 31 - 1, 16, np.array([0, 300, 600, 900, 1200, 2 ** 31 - 1], np.int64), 5, P.ERR_INVALID),
        (rec, 1500, 10, off, 5, P.ERR_INVALID),
        (rec_nan, 1500, 16, off, 5, P.ERR_EMPTY),
    ]
    for rc_case, (r_, n, stride, o, B, code) in enumerate(cases):
        out = (C.c_void_p * 5)(*([C.c_void_p(0xdead)] * 5))
        rc = L.pclb200_index_build_batch(ctx.h, None if r_ is None else vp(r_), n, stride,
                                         None if o is None else vp(o), B, out)
        assert rc == code, (rc_case, rc, L.pclb200_last_error())
        if 1 <= B <= 65536:
            assert all(out[c] is None for c in range(5)), rc_case
        if code == P.ERR_EMPTY:
            assert b"cloud 2" in L.pclb200_last_error()
    # a NULL out array
    assert L.pclb200_index_build_batch(ctx.h, vp(rec), 1500, 16, vp(off), 5, None) == P.ERR_INVALID
    # the context builds again, correctly
    hs = ctx.index_build_batch(rec, off)
    for c, h in enumerate(hs):
        _check_handle(P, ctx, h, good[c], rec[off[c]:off[c + 1]], f"cloud {c} after the refusals")
        h.close()
