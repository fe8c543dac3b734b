"""The aligned cloud an ICP session hands back (icp.hpp:265-267: output = *input_, transformed by final_transformation_),
byte for byte, for every record layout and buffer kind get_cloud accepts: PointXYZ and PointNormal records, records with
extra fields, normals inside or outside the records, host / pinned / device outputs, host or device sources, an index
subset, non-finite points and normals, a non-identity guess; through the session and through one-call align.  The
expected bytes are computed here in float32 with the reference's operation order.  Needs an H100: run with -m gpu."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = 20000


@pytest.fixture(scope="module")
def gpu():
    import pcl_b200
    pcl_b200.lib()
    ctx = pcl_b200.Context(0)
    yield pcl_b200, ctx
    ctx.close()


def _scene(width):
    """target PointNormal records on z = 0.1 sin(3x) + 0.1 cos(4y), a source moved by a small rigid motion, `width` floats per record
    (words 8.. are extra fields that must pass through), one NaN point, one inf point, one NaN normal"""
    r = np.random.default_rng(4)
    xy = r.random((N, 2))
    z = 0.1 * np.sin(3 * xy[:, 0]) + 0.1 * np.cos(4 * xy[:, 1])
    nrm = np.stack([-0.3 * np.cos(3 * xy[:, 0]), 0.4 * np.sin(4 * xy[:, 1]), np.ones(N)], 1)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    tgt = np.zeros((N, width), np.float32)
    tgt[:, 0:2], tgt[:, 2], tgt[:, 3], tgt[:, 4:7] = xy, z, 1.0, nrm
    a = np.deg2rad(1.5)
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    src = tgt.copy()
    src[:, 0:3] = tgt[:, 0:3].astype(np.float64) @ R.T + [0.004, -0.003, 0.002]
    src[:, 4:7] = tgt[:, 4:7].astype(np.float64) @ R.T
    src[:, 3] = r.random(N)  # w: carried through where the output keeps the caller's records
    if width > 8:
        src[:, 8:] = r.random((N, width - 8))
    src[7, 0] = np.nan
    src[11, 1] = np.inf
    src[13, 5] = np.nan
    return tgt, src


GUESS = np.array([[1, 0, 0, 0.001], [0, 1, 0, 0], [0, 0, 1, -0.001], [0, 0, 0, 1]], np.float64)


def _tf(T, xyz, mode, normal):
    """one transform in float32 with the operation order of mode (0: icp.hpp transformCloud, 1: transformPointCloud)"""
    f = T.astype(np.float32)
    x, y, z = (xyz[:, i].astype(np.float32) for i in range(3))
    t = [np.float32(0) if normal else f[i, 3] for i in range(3)]
    if mode == 0:
        cols = [((f[i, 0] * x + f[i, 1] * y) + f[i, 2] * z) + t[i] for i in range(3)]
    elif normal:
        cols = [f[i, 0] * x + (f[i, 1] * y + f[i, 2] * z) for i in range(3)]
    else:
        cols = [f[i, 0] * x + (f[i, 1] * y + (f[i, 2] * z + t[i])) for i in range(3)]
    return np.stack(cols, 1).astype(np.float32)


def _expect(before, src, T, mode, nrm_word=None, w_one=False):
    """the output records: `before` with src's xyz (and its normals at float nrm_word, into the same word) written,
    transformed where the point is finite; a non-finite normal is left alone by mode 0; w = 1 when w_one"""
    out = before.copy()
    ok = np.isfinite(src[:, :3]).all(1)
    out[:, 0:3] = src[:, 0:3]
    out[ok, 0:3] = _tf(T, src[ok, 0:3], mode, False)
    if w_one:
        out[:, 3] = 1.0
    if nrm_word is not None:
        w = nrm_word
        okn = ok & np.isfinite(src[:, w:w + 3]).all(1) if mode == 0 else ok
        out[:, w:w + 3] = src[:, w:w + 3]
        out[okn, w:w + 3] = _tf(T, src[okn, w:w + 3], mode, True)
    return out


def _nrm_only(before, src, T, mode):
    """a separate normals array: the normals' xyz written (transformed as _expect does), their w left as it was"""
    out = before.copy()
    out[:, 0:3] = _expect(src, src, T, mode, 4)[:, 4:7]
    return out


def _same(a, b):
    """the same bytes; NaN only has to stay NaN (its payload after arithmetic is the hardware's choice)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(b)
    assert np.array_equal(np.isnan(a), nan)
    assert np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32))


def _session(P, ctx, tgt, with_normals_transform, src, normals=None, indices=None):
    import torch
    dt = torch.from_numpy(np.ascontiguousarray(tgt[:, :8])).cuda()
    idx = P.Index(ctx, dt)
    s = P.Icp(ctx, max_iterations=5, max_correspondence_distance=0.05, estimator=P.EST_POINT_TO_PLANE_LLS,
              with_normals_transform=with_normals_transform)
    s.set_target(idx, normals=P.Field(dt, 4))
    s.set_source(src, normals=normals, indices=indices, guess=GUESS)
    st = s.iterate()
    assert st["iterations"] >= 1 and np.isfinite(st["final"]).all()
    return s, st["final"], idx


@pytest.mark.parametrize("width", [8, 16])
@pytest.mark.parametrize("where", ["device_src", "host_src"])
@pytest.mark.parametrize("mode", [0, 1])
def test_records_with_normals_inside(gpu, width, where, mode):
    """PointNormal records (and records with extra fields): every output buffer kind gets the same bytes"""
    import torch
    P, ctx = gpu
    tgt, src = _scene(width)
    s_in = torch.from_numpy(src).cuda() if where == "device_src" else src
    s, T, _ = _session(P, ctx, tgt, mode, s_in, normals=P.Field(s_in, 4))
    exp = _expect(src, src, T, mode, 4)
    out_d = torch.full((N, width), -7.0, device="cuda")
    s.get_cloud(out_d, normals=P.Field(out_d, 4))
    _same(out_d.cpu().numpy(), exp)
    out_h = np.full((N, width), -7.0, np.float32)
    s.get_cloud(out_h, normals=P.Field(out_h, 4))
    _same(out_h, exp)
    out_p = torch.full((N, width), -7.0).pin_memory()
    s.get_cloud(out_p, normals=P.Field(out_p, 4))
    _same(out_p.numpy(), exp)
    # no normals asked for: the records' normals pass through untouched
    out_d.fill_(-7.0)
    s.get_cloud(out_d)
    _same(out_d.cpu().numpy(), _expect(src, src, T, mode))
    # normals into a separate array: xyz and w = 1 written into the records, the normals' xyz into the array
    out_r = torch.full((N, width), -7.0, device="cuda")
    out_n = torch.full((N, 4), -5.0, device="cuda")
    s.get_cloud(out_r, normals=out_n)
    before = np.full((N, width), -7.0, np.float32)
    _same(out_r.cpu().numpy(), _expect(before, src, T, mode, w_one=True))
    _same(out_n.cpu().numpy(), _nrm_only(np.full((N, 4), -5.0, np.float32), src, T, mode))


@pytest.mark.parametrize("where", ["device_src", "host_src"])
def test_pointxyz_and_separate_normals(gpu, where):
    """PointXYZ records (stride 16: the caller's w comes back) and normals kept in an array of their own"""
    import torch
    P, ctx = gpu
    tgt, src8 = _scene(8)
    xyz = np.ascontiguousarray(src8[:, :4])
    nrm = np.ascontiguousarray(src8[:, 4:8])
    s_in = torch.from_numpy(xyz).cuda() if where == "device_src" else xyz
    n_in = torch.from_numpy(nrm).cuda() if where == "device_src" else nrm
    s, T, _ = _session(P, ctx, tgt, 1, s_in, normals=n_in)
    exp = _expect(xyz, xyz, T, 1)
    for kind in ("cuda", "pinned"):
        out, out_n = torch.full((N, 4), -7.0), torch.full((N, 4), -5.0)
        out, out_n = (out.cuda(), out_n.cuda()) if kind == "cuda" else (out.pin_memory(), out_n.pin_memory())
        s.get_cloud(out, normals=out_n)
        _same(out.cpu().numpy(), exp)
        _same(out_n.cpu().numpy(), _nrm_only(np.full((N, 4), -5.0, np.float32), src8, T, 1))
    out_h = np.full((N, 4), -7.0, np.float32)
    s.get_cloud(out_h)
    _same(out_h, exp)


def test_index_subset_and_align(gpu):
    """an index subset aligns on its queries and still returns every record; one-call align gives the same bytes"""
    import torch
    P, ctx = gpu
    tgt, src = _scene(12)
    d_src = torch.from_numpy(src).cuda()
    sub = np.arange(0, N, 2, dtype=np.int32)
    s, T, idx = _session(P, ctx, tgt, 1, d_src, normals=P.Field(d_src, 4), indices=sub)
    out = torch.empty_like(d_src)
    s.get_cloud(out, normals=P.Field(out, 4))
    exp = _expect(src, src, T, 1, 4)
    _same(out.cpu().numpy(), exp)
    dt = torch.from_numpy(np.ascontiguousarray(tgt[:, :8])).cuda()
    out_a = torch.empty_like(d_src)
    r = P.icp_align(ctx, d_src, idx, src_normals=P.Field(d_src, 4), tgt_normals=P.Field(dt, 4), indices=sub,
                    guess=GUESS, out_cloud=out_a, max_iterations=5, max_correspondence_distance=0.05,
                    estimator=P.EST_POINT_TO_PLANE_LLS, with_normals_transform=1)
    assert np.array_equal(r["final"], T)
    _same(out_a.cpu().numpy(), exp)
