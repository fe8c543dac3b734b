"""Helper for tests/test_gpu_sharded_corr.py (launched under torchrun, gloo): the stand-alone consumers of the 1-NN search
on a map sharded across ranks (pclb200_correspondences_sharded, pclb200_validate_transformation_sharded,
pclb200_inliers_sharded), every rank holding one tile and the whole source.

Ranks on cuda:0 with the peer exchange bootstrapped over gloo, or, with PCLB_SHARDED_NCCL=1, one GPU per rank under NCCL.
The map is a 60 k-point surface with non-finite points and repeated points under other ids, cut four ways (tests/_sharded.py:
slabs, a random partition, ids shared by two ranks near the cuts, a far tile).  On every rank, against one index of the
whole map (pclb200_index_build with subset = the union of the ids): every list byte for byte (finite and unbounded gates,
with and without src_indices, is_dense 0 with NaN source points), reciprocal lists, inliers, the record rows against the
map's rows; validation to 1e-12 and the same on every rank; a hand-written ICP loop (correspondences with records, a
rejector chain, SVD / point-to-plane over the rows with corr = NULL) byte for byte for 10 iterations; every refusal on
every rank."""
import numpy as np

import _sharded as S
import pcl_b200 as P

me = S.join()
rank, world, ctx, ref_ctx = me.rank, me.world, me.ctx, me.ref

rng = np.random.default_rng(23)
base = S.with_extras(rng, S.surface(rng, 60000))
src0 = base[rng.choice(len(base), 12000, replace=False)].copy()
a = np.deg2rad(1.5)
Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
src = np.ones((len(src0), 4), np.float32)
src[:, :3] = (np.nan_to_num(src0[:, :3].astype(np.float64)) @ Rz.T + [0.01, -0.008, 0.004]).astype(np.float32)
src[rng.choice(len(src), 40, replace=False), 2] = np.nan                     # non-finite source points
sub = np.sort(rng.choice(len(src), 5000, replace=False)).astype(np.int32)
src_index = P.Index(ctx, src)
ref_src_index = P.Index(ref_ctx, src)


def unit_normals(n):
    v = rng.normal(size=(n, 3))
    out = np.zeros((n, 4), np.float32)
    out[:, :3] = v / np.linalg.norm(v, axis=1, keepdims=True)
    out[::997, 0] = np.nan                                                    # NaN normals travel as they are
    return out


def raw_inliers(index, T, thr, sharded):
    """the inlier list itself (Index.inliers returns only its query indices and fitness)"""
    b = P._Buf(src)
    T = np.ascontiguousarray(T, np.float64)
    out = np.empty(len(src), P.CORR_DTYPE)
    xyz = np.empty((len(src), 4), np.float32)
    m = P.C.c_size_t()
    Tp = T.ctypes.data_as(P.C.POINTER(P.C.c_double))
    if sharded:
        P._check(P.lib().pclb200_inliers_sharded(index.ctx.h, index.h, b.ptr, b.rows, b.stride, Tp, float(thr),
                                                 P.C.c_void_p(out.ctypes.data), P.C.c_void_p(xyz.ctypes.data),
                                                 P.C.byref(m)))
        return out[:m.value], xyz[:m.value]
    P._check(P.lib().pclb200_inliers(index.ctx.h, index.h, b.ptr, b.rows, b.stride, Tp, float(thr),
                                     P.C.c_void_p(out.ctypes.data), P.C.byref(m)))
    return out[:m.value], None


def same_everywhere(x):
    allx = S.gathered(x)
    assert all(v == allx[0] for v in allx), allx
    return x


def transform(pts, T):
    out = pts.copy()
    out[:, :3] = (pts[:, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    return out


REJECTORS = [(P.REJ_DISTANCE, 0.04), (P.REJ_MEDIAN, 3.0), (P.REJ_ONE_TO_ONE, 0.0), (P.REJ_TRIMMED, 0.9)]


def icp_loop(estimate, corr_of):
    """10 iterations of correspondences -> rejector chain -> estimate over gathered rows (corr = NULL) -> transform"""
    T, cur, Ts = np.eye(4), src.copy(), []
    for _ in range(10):
        corr, rows = corr_of(cur)
        for kind, p in REJECTORS:
            corr, _ = ctx.reject(corr, kind, p)
        at = {q: i for i, q in enumerate(rows[0]["index_query"])}
        pick = np.array([at[q] for q in corr["index_query"]], np.int64)
        s_rows = np.ascontiguousarray(cur[corr["index_query"]])
        t_rows = np.ascontiguousarray(np.c_[rows[1][pick], rows[2][pick]] if rows[2] is not None else rows[1][pick])
        step = estimate(s_rows, t_rows)
        T = step @ T
        cur = transform(src, T)
        Ts.append(T.tobytes())
    return Ts


snrm = unit_normals(len(src))                     # source normals, some NaN
lists = recip_lists = rows_checked = inliers_checked = loops = normal_lists = 0
for pname, parts, whole in S.partitions(rng, base, world):
    nrm = unit_normals(len(whole))
    union = np.unique(np.concatenate(parts)).astype(np.int32)
    ref = P.Index(ref_ctx, whole, subset=union)
    ids = np.ascontiguousarray(parts[rank], dtype=np.int32)
    tile, tnrm = np.ascontiguousarray(whole[ids]), np.ascontiguousarray(nrm[ids])
    tindex = P.Index(ctx, tile, ids=ids)
    for md in (np.sqrt(np.finfo(np.float64).max), 0.05, 0.0):
        for ind in (None, sub):
            for dense in (True, False):
                want = ref.correspondences(src, md, indices=ind, is_dense=dense)
                got = tindex.correspondences_sharded(src, md, indices=ind, is_dense=dense)
                assert got.tobytes() == want.tobytes(), (pname, md, ind is None, dense, len(got), len(want))
                lists += 1
            want = ref.correspondences(src, md, indices=ind, src_index=ref_src_index)
            got = tindex.correspondences_sharded(src, md, indices=ind, src_index=src_index)
            assert got.tobytes() == want.tobytes(), (pname, "reciprocal", md, ind is None, len(got), len(want))
            recip_lists += 1
            c, xyz, nr = tindex.correspondences_sharded(src, md, indices=ind, tgt_normals=tnrm, rows=True, normal_rows=True)
            assert c.tobytes() == ref.correspondences(src, md, indices=ind).tobytes(), (pname, "list with rows", md)
            w = whole[c["index_match"]].copy()
            w[:, 3] = 1
            n4 = nrm[c["index_match"]].copy()
            n4[:, 3] = 0
            assert xyz.tobytes() == w.tobytes() and nr.tobytes() == n4.tobytes(), (pname, "rows", md)
            rows_checked += len(c)
    T = np.eye(4)
    T[:3, :3] = Rz.T
    for thr in (0.02, 0.005, 0.0):
        got, xyz = raw_inliers(tindex, T, thr, True)
        want, _ = raw_inliers(ref, T, thr, False)
        assert got.tobytes() == want.tobytes(), (pname, "inliers", thr, len(got), len(want))
        w = whole[got["index_match"]].copy()
        w[:, 3] = 1
        assert xyz.tobytes() == w.tobytes(), (pname, "inlier rows", thr)
        inliers_checked += 1
    for dbl in (0, 1):
        for max_range in (np.finfo(np.float64).max, 0.001):
            v = same_everywhere(tindex.validate_transformation_sharded(src, T, max_range, scalar_is_double=dbl))
            v1 = ref.validate_transformation(src, T, max_range, scalar_is_double=dbl)
            assert abs(v - v1) <= 1e-12 * abs(v1), (pname, dbl, max_range, v, v1)
    # normal shooting and back projection: k = 1, 10, 40, finite and unbounded gates, with and without src_indices
    for kind in (P.CORR_NORMAL_SHOOTING, P.CORR_BACK_PROJECTION):
        for k in (1, 10, 40):
            for md, ind in ((np.sqrt(np.finfo(np.float64).max), None), (0.05, sub), (0.002, None)):
                want = ref.correspondences_normals(kind, src, snrm, tgt_normals=nrm, k=k, max_distance=md, indices=ind)
                c, xyz, nr = tindex.correspondences_normals_sharded(kind, src, snrm, tgt_normals=tnrm, k=k, max_distance=md,
                                                                    indices=ind, rows=True, normal_rows=True)
                assert c.tobytes() == want.tobytes(), (pname, "normals", kind, k, md, len(c), len(want))
                w = whole[c["index_match"]].copy()
                w[:, 3] = 1
                n4 = nrm[c["index_match"]].copy()
                n4[:, 3] = 0
                assert xyz.tobytes() == w.tobytes() and nr.tobytes() == n4.tobytes(), (pname, "normal rows", kind, k)
                normal_lists += 1
    # the hand-written loop: SVD and point-to-plane, sharded map vs one index of the whole map
    lnrm = np.nan_to_num(nrm)                 # point-to-plane over a NaN normal would end the loop after one step
    pn, ltnrm = np.ascontiguousarray(np.c_[whole, lnrm]), np.ascontiguousarray(lnrm[ids])
    for ename, est in (("svd", lambda s, t: ctx.estimate_svd(s, t)),
                       ("point_to_plane", lambda s, t: ctx.estimate_point_to_plane_lls(s, t))):
        with_n = ename != "svd"

        def sharded(cur):
            c, xyz, nr = tindex.correspondences_sharded(cur, 0.08, tgt_normals=ltnrm if with_n else None, rows=True,
                                                        normal_rows=with_n)
            return c, (c, xyz, nr)

        def single(cur):
            c = ref.correspondences(cur, 0.08)
            r = pn[c["index_match"]]
            xyz = r[:, :4].copy()
            xyz[:, 3] = 1
            return c, (c, xyz, r[:, 4:8].copy() if with_n else None)

        a_T, b_T = icp_loop(est, sharded), icp_loop(est, single)
        first = next((i for i, (x, y) in enumerate(zip(a_T, b_T)) if x != y), None)
        assert first is None, (pname, ename, "first iteration with another transform", first)
        same_everywhere(a_T[-1])
        loops += 1
    print(f"rank {rank}: {pname} ok", flush=True)

# a whole map with fewer than k points: k is clamped to its distinct finite ids (tiles hold fewer still)
tiny = P.xyz1(base[:30, :3])
tiny_nrm = unit_normals(30)
ids = np.arange(rank, 30, world, dtype=np.int32)
tref = P.Index(ref_ctx, tiny)
ttile = P.Index(ctx, np.ascontiguousarray(tiny[ids]), ids=ids)
for kind in (P.CORR_NORMAL_SHOOTING, P.CORR_BACK_PROJECTION):
    want = tref.correspondences_normals(kind, src, snrm, tgt_normals=tiny_nrm, k=40)
    got = ttile.correspondences_normals_sharded(kind, src, snrm, tgt_normals=np.ascontiguousarray(tiny_nrm[ids]), k=40)
    assert got.tobytes() == want.tobytes(), ("tiny map", kind, len(got), len(want))
    normal_lists += 1

# ---- refusals: ERR_INVALID on every rank, before any exchange --------------------------------------------------------------
ids = np.ascontiguousarray(np.arange(rank, len(base), world), dtype=np.int32)
tindex = P.Index(ctx, np.ascontiguousarray(base[ids]), ids=ids)
plain = P.Index(ctx, np.ascontiguousarray(base[ids]))
S.refused(lambda: plain.correspondences_sharded(src), "ids")
S.refused(lambda: tindex.correspondences_sharded(src, src_index=tindex), "without ids")
S.refused(lambda: tindex.correspondences_sharded(src, rows=True, normal_rows=True), "tgt_normals")
short = np.ascontiguousarray(src[:len(src) - rank])   # rank 0 passes one point more than the others
S.refused(lambda: tindex.correspondences_sharded(short), "same whole source")
S.refused(lambda: tindex.inliers_sharded(short, np.eye(4), 0.01), "same whole source")
S.refused(lambda: tindex.validate_transformation_sharded(short, np.eye(4)), "same source")
# one rank alone refuses its arguments: every rank refuses
if rank == 0:
    S.refused(lambda: tindex.correspondences_sharded(src, src_index=tindex), "without ids")
else:
    S.refused(lambda: tindex.correspondences_sharded(src, src_index=src_index), "another rank")
if rank == world - 1:
    S.refused(lambda: plain.validate_transformation_sharded(src, np.eye(4)), "ids")
else:
    S.refused(lambda: tindex.validate_transformation_sharded(src, np.eye(4)), "another rank")
tn = np.ascontiguousarray(unit_normals(len(ids)))
S.refused(lambda: tindex.correspondences_normals_sharded(P.CORR_NORMAL_SHOOTING, src, snrm, k=-1), "k < 0")
S.refused(lambda: tindex.correspondences_normals_sharded(7, src, snrm), "kind")
S.refused(lambda: tindex.correspondences_normals_sharded(P.CORR_NORMAL_SHOOTING, src, None), "source normals")
S.refused(lambda: tindex.correspondences_normals_sharded(P.CORR_NORMAL_SHOOTING, short, snrm[:len(short)]), "same whole")
S.refused(lambda: plain.correspondences_normals_sharded(P.CORR_NORMAL_SHOOTING, src, snrm), "ids")
if rank == 0:   # back projection without target normals on one rank only
    S.refused(lambda: tindex.correspondences_normals_sharded(P.CORR_BACK_PROJECTION, src, snrm), "target normals")
else:
    S.refused(lambda: tindex.correspondences_normals_sharded(P.CORR_BACK_PROJECTION, src, snrm, tgt_normals=tn),
              "another rank")
lone = P.Index(ref_ctx, np.ascontiguousarray(base[ids]), ids=ids)
S.refused(lambda: lone.correspondences_sharded(src), "communicator")
S.refused(lambda: lone.inliers_sharded(src, np.eye(4), 0.01), "communicator")
# the calls still work after the refusals
same_everywhere(tindex.correspondences_sharded(src, 0.05).tobytes())
me.finish("SHARDED_CORR", lists=lists, reciprocal=recip_lists, normal_lists=normal_lists, rows=rows_checked,
          inliers=inliers_checked, loops=loops)
