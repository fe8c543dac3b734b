"""ctypes binding of the CPU oracle (oracle/pcl_oracle.cpp).

TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  pcl_b200/ never imports this package.
Parity status: PINNED against the reference's golden vectors (tests/test_oracle_golden.py).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libpcl_oracle.so")


def build(force=False):
    src = os.path.join(_HERE, "pcl_oracle.cpp")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _SO


class Corr(C.Structure):
    _fields_ = [("index_query", C.c_int32), ("index_match", C.c_int32), ("distance", C.c_float)]


CORR_DTYPE = np.dtype([("index_query", np.int32), ("index_match", np.int32), ("distance", np.float32)])


class IcpParams(C.Structure):
    _fields_ = [("max_iterations", C.c_int32), ("use_reciprocal", C.c_int32),
                ("estimator", C.c_int32), ("scalar_is_double", C.c_int32),
                ("with_normals_transform", C.c_int32), ("source_has_normals", C.c_int32),
                ("is_dense", C.c_int32), ("nthreads", C.c_int32),
                ("max_correspondence_distance", C.c_double),
                ("transformation_epsilon", C.c_double),
                ("transformation_rotation_epsilon", C.c_double),
                ("euclidean_fitness_epsilon", C.c_double),
                ("correspondence_kind", C.c_int32), ("correspondence_k", C.c_int32)]


class IcpResult(C.Structure):
    _fields_ = [("final_transformation", C.c_double * 16), ("last_transformation", C.c_double * 16),
                ("converged", C.c_int32), ("state", C.c_int32), ("iterations", C.c_int32),
                ("n_correspondences", C.c_int32), ("mse", C.c_double), ("total_correspondences", C.c_longlong)]


class Rejector(C.Structure):
    _fields_ = [("kind", C.c_int32), ("min_correspondences", C.c_int32), ("p", C.c_double)]


REJ_DISTANCE, REJ_MEDIAN, REJ_ONE_TO_ONE, REJ_TRIMMED, REJ_SURFACE_NORMAL = 0, 1, 2, 3, 4
CORR_NEAREST, CORR_NORMAL_SHOOTING, CORR_BACK_PROJECTION = 0, 1, 2

_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        vp, sz, i32p, fp, dp = C.c_void_p, C.c_size_t, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_double)
        L.orc_index_build.restype = vp
        L.orc_index_build.argtypes = [fp, sz, sz, i32p, sz]
        L.orc_index_free.argtypes = [vp]
        L.orc_index_size.restype = sz
        L.orc_index_size.argtypes = [vp]
        L.orc_knn.argtypes = [vp, fp, sz, sz, C.c_int, i32p, fp, C.c_int]
        L.orc_knn_bruteforce.argtypes = [fp, sz, sz, fp, sz, sz, C.c_int, i32p, fp]
        L.orc_radius.argtypes = [vp, fp, sz, sz, C.c_double, C.c_uint, C.POINTER(C.c_int64), i32p, fp, C.c_int]
        L.orc_correspondences.restype = sz
        L.orc_correspondences.argtypes = [vp, fp, sz, sz, i32p, sz, C.c_int, C.c_double, C.POINTER(Corr), C.c_int]
        L.orc_correspondences_reciprocal.restype = sz
        L.orc_correspondences_reciprocal.argtypes = [vp, vp, fp, sz, sz, fp, sz, i32p, sz, C.c_int, C.c_double, C.POINTER(Corr), C.c_int]
        L.orc_estimate_svd.argtypes = [fp, sz, fp, sz, C.POINTER(Corr), sz, C.c_int, dp]
        L.orc_estimate_svd_correlation.argtypes = [fp, sz, fp, sz, C.POINTER(Corr), sz, C.c_int, dp]
        L.orc_estimate_point_to_plane_lls.argtypes = [fp, sz, fp, fp, sz, C.POINTER(Corr), sz, C.c_int, dp]
        L.orc_estimate_symmetric_lls.argtypes = [fp, fp, sz, fp, fp, sz, C.POINTER(Corr), sz, C.c_int, C.c_int, dp]
        L.orc_transform.argtypes = [fp, sz, sz, C.c_int, dp, C.c_int, C.c_int]
        L.orc_icp_align.argtypes = [C.POINTER(IcpParams), fp, sz, sz, i32p, sz, fp, sz, sz, dp, C.POINTER(IcpResult), fp]
        L.orc_icp_align_tree.argtypes = [C.POINTER(IcpParams), vp, fp, sz, sz, i32p, sz, fp, sz, sz, dp, C.POINTER(IcpResult), fp]
        L.orc_reject.restype = sz
        L.orc_reject.argtypes = [C.POINTER(Rejector), C.POINTER(Corr), sz, C.POINTER(Corr), dp]
        L.orc_reject_chain.restype = sz
        L.orc_reject_chain.argtypes = [C.POINTER(Rejector), C.c_int, C.POINTER(Corr), sz, C.POINTER(Corr), dp]
        L.orc_icp_align_full.argtypes = [C.POINTER(IcpParams), vp, C.POINTER(Rejector), C.c_int, vp, fp, sz, sz, i32p, sz,
                                         fp, sz, sz, dp, C.POINTER(IcpResult), fp, C.POINTER(Corr), C.POINTER(sz)]
        L.orc_icp_align_carry.argtypes = L.orc_icp_align_full.argtypes + [dp]
        L.orc_fitness_score.restype = C.c_double
        L.orc_fitness_score.argtypes = [vp, fp, sz, sz, i32p, sz, C.c_int, dp, C.c_int, C.c_double, C.c_int]
        L.orc_voxelgrid.restype = C.c_longlong
        L.orc_voxelgrid.argtypes = [fp, sz, sz, i32p, sz, C.c_int, fp, C.c_uint, fp]
        L.orc_gicp_covariances.restype = None
        L.orc_gicp_covariances.argtypes = [vp, fp, sz, sz, C.c_int, C.c_double, dp, C.c_int]
        L.orc_voxelgrid_normals.restype = C.c_longlong
        L.orc_voxelgrid_normals.argtypes = [fp, sz, sz, i32p, sz, C.c_int, fp, C.c_uint, fp, C.c_long, fp]
        L.orc_point_normal.argtypes = [fp, sz, C.c_int, i32p, sz, fp]
        L.orc_normals_knn.argtypes = [vp, fp, sz, sz, i32p, sz, C.c_int, C.c_int, fp, fp, C.c_int]
        u8p = C.POINTER(C.c_uint8)
        L.orc_knn_stats.argtypes = [vp, fp, sz, sz, i32p, sz, C.c_int, fp, fp, C.c_int]
        L.orc_sor.restype = sz
        L.orc_sor.argtypes = [vp, fp, sz, sz, i32p, sz, C.c_int, C.c_double, C.c_int, u8p, C.c_int]
        L.orc_ror.restype = sz
        L.orc_ror.argtypes = [vp, fp, sz, sz, i32p, sz, C.c_int, C.c_double, C.c_int, C.c_int, u8p, C.c_int]
        L.orc_correspondences_normals.restype = sz
        L.orc_correspondences_normals.argtypes = [vp, C.c_int, fp, sz, sz, fp, sz, fp, sz, fp, sz, i32p, sz, C.c_int,
                                                  C.c_double, C.POINTER(Corr), C.c_int]
        L.orc_reject_surface_normal.restype = sz
        L.orc_reject_surface_normal.argtypes = [C.POINTER(Corr), sz, fp, sz, fp, sz, C.c_double, C.POINTER(Corr)]
        L.orc_normals_radius.argtypes = [vp, fp, sz, sz, i32p, sz, C.c_int, C.c_double, fp, fp, C.c_int]
        L.orc_cluster_labels.argtypes = [vp, sz, C.c_double, i32p]
        L.orc_cluster_labels.restype = None
        L.orc_max_threads.restype = C.c_int
        _lib = L
    return _lib


def _f(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _i(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_int32))


def _d(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))


def as_cloud(a):
    """(n,>=3) float array -> C-contiguous float32 with row stride = a.shape[1] floats."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    assert a.ndim == 2 and a.shape[1] >= 3
    return a


def to_xyz1(xyz):
    """(n,3) -> (n,4) pcl::PointXYZ layout {x,y,z,1}."""
    xyz = np.asarray(xyz, dtype=np.float32)
    out = np.ones((xyz.shape[0], 4), dtype=np.float32)
    out[:, :3] = xyz[:, :3]
    return out


def max_threads():
    return int(lib().orc_max_threads())


class Index:
    """pcl::KdTreeFLANN restatement (exact, <=15-point leaves)."""

    def __init__(self, cloud, subset=None):
        self.cloud = as_cloud(cloud)
        self.subset = None if subset is None else np.ascontiguousarray(subset, dtype=np.int32)
        self.h = lib().orc_index_build(_f(self.cloud), self.cloud.shape[0], self.cloud.shape[1],
                                       _i(self.subset), 0 if self.subset is None else self.subset.size)

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_index_free(self.h)
            self.h = None

    @property
    def size(self):
        return int(lib().orc_index_size(self.h))

    def knn(self, q, k, nthreads=1):
        q = as_cloud(q)
        idx = np.empty((q.shape[0], k), dtype=np.int32)
        d2 = np.empty((q.shape[0], k), dtype=np.float32)
        keff = lib().orc_knn(self.h, _f(q), q.shape[0], q.shape[1], k, _i(idx), _f(d2), nthreads)
        return idx, d2, keff

    def radius(self, q, r, max_nn=0, nthreads=1):
        q = as_cloud(q)
        offs = np.zeros(q.shape[0] + 1, dtype=np.int64)
        lib().orc_radius(self.h, _f(q), q.shape[0], q.shape[1], float(r), max_nn,
                         offs.ctypes.data_as(C.POINTER(C.c_int64)), None, None, nthreads)
        idx = np.empty(max(int(offs[-1]), 1), dtype=np.int32)
        d2 = np.empty(max(int(offs[-1]), 1), dtype=np.float32)
        lib().orc_radius(self.h, _f(q), q.shape[0], q.shape[1], float(r), max_nn,
                         offs.ctypes.data_as(C.POINTER(C.c_int64)), _i(idx), _f(d2), nthreads)
        return offs, idx[:offs[-1]], d2[:offs[-1]]

    def correspondences(self, src, max_distance=np.sqrt(np.finfo(np.float64).max), indices=None,
                        is_dense=True, nthreads=1):
        src = as_cloud(src)
        indices = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
        n = src.shape[0] if indices is None else indices.size
        out = np.empty(max(n, 1), dtype=CORR_DTYPE)
        m = lib().orc_correspondences(self.h, _f(src), src.shape[0], src.shape[1], _i(indices),
                                      0 if indices is None else indices.size, int(is_dense),
                                      float(max_distance), out.ctypes.data_as(C.POINTER(Corr)), nthreads)
        return out[:m]

    def correspondences_reciprocal(self, src, src_index, max_distance=np.sqrt(np.finfo(np.float64).max),
                                   indices=None, is_dense=True, nthreads=1):
        src = as_cloud(src)
        indices = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
        n = src.shape[0] if indices is None else indices.size
        out = np.empty(max(n, 1), dtype=CORR_DTYPE)
        m = lib().orc_correspondences_reciprocal(
            self.h, src_index.h, _f(src), src.shape[0], src.shape[1], _f(self.cloud), self.cloud.shape[1],
            _i(indices), 0 if indices is None else indices.size, int(is_dense), float(max_distance),
            out.ctypes.data_as(C.POINTER(Corr)), nthreads)
        return out[:m]

    def fitness_score(self, src, final_T, max_range=np.finfo(np.float64).max, scalar_is_double=False,
                      indices=None, is_dense=True):
        src = as_cloud(src)
        T = np.ascontiguousarray(final_T, dtype=np.float64)
        indices = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
        return float(lib().orc_fitness_score(self.h, _f(src), src.shape[0], src.shape[1], _i(indices),
                                             0 if indices is None else indices.size, int(is_dense), _d(T),
                                             int(scalar_is_double), float(max_range), 1))

    def gicp_covariances(self, k=20, gicp_epsilon=0.001, nthreads=1):
        """GeneralizedIterativeClosestPoint::computeCovariances over the indexed cloud: (n, 3, 3) float64."""
        out = np.zeros((self.cloud.shape[0], 9), dtype=np.float64)
        lib().orc_gicp_covariances(self.h, _f(self.cloud), self.cloud.shape[0], self.cloud.shape[1], int(k),
                                   float(gicp_epsilon), _d(out), nthreads)
        return out.reshape(-1, 3, 3)

    def knn_stats(self, cloud, k, nthreads=1):
        cloud = as_cloud(cloud)
        mean = np.empty(cloud.shape[0], np.float32)
        kth = np.empty(cloud.shape[0], np.float32)
        lib().orc_knn_stats(self.h, _f(cloud), cloud.shape[0], cloud.shape[1], None, 0, k, _f(mean), _f(kth), nthreads)
        return mean, kth

    def statistical_outlier_removal(self, cloud, mean_k, std_mul, negative=False, nthreads=1):
        cloud = as_cloud(cloud)
        keep = np.empty(cloud.shape[0], np.uint8)
        lib().orc_sor(self.h, _f(cloud), cloud.shape[0], cloud.shape[1], None, 0, mean_k, float(std_mul), int(negative),
                      keep.ctypes.data_as(C.POINTER(C.c_uint8)), nthreads)
        return np.nonzero(keep)[0].astype(np.int32)

    def radius_outlier_removal(self, cloud, radius, min_pts, negative=False, is_dense=True, nthreads=1):
        cloud = as_cloud(cloud)
        keep = np.empty(cloud.shape[0], np.uint8)
        lib().orc_ror(self.h, _f(cloud), cloud.shape[0], cloud.shape[1], None, 0, int(is_dense), float(radius), min_pts,
                      int(negative), keep.ctypes.data_as(C.POINTER(C.c_uint8)), nthreads)
        return np.nonzero(keep)[0].astype(np.int32)

    def normals_knn(self, cloud, k, viewpoint=(0, 0, 0), indices=None, is_dense=True, nthreads=1):
        cloud = as_cloud(cloud)
        indices = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
        n = cloud.shape[0] if indices is None else indices.size
        out = np.empty((n, 4), dtype=np.float32)
        vp = np.asarray(viewpoint, dtype=np.float32)
        dense = lib().orc_normals_knn(self.h, _f(cloud), cloud.shape[0], cloud.shape[1], _i(indices),
                                      0 if indices is None else indices.size, int(is_dense), k, _f(vp),
                                      _f(out), nthreads)
        return out, bool(dense)


    def cluster_labels(self, tolerance):
        """extractEuclideanClusters over the indexed points: label = smallest index of the point's cluster, -1 = not held."""
        out = np.empty(self.cloud.shape[0], dtype=np.int32)
        lib().orc_cluster_labels(self.h, self.cloud.shape[0], float(tolerance), _i(out))
        return out

    def normals_radius(self, cloud, radius, viewpoint=(0, 0, 0), indices=None, is_dense=True, nthreads=1):
        """NormalEstimation with setRadiusSearch(radius)."""
        cloud = as_cloud(cloud)
        indices = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
        n = cloud.shape[0] if indices is None else indices.size
        out = np.empty((n, 4), dtype=np.float32)
        vp = np.asarray(viewpoint, dtype=np.float32)
        dense = lib().orc_normals_radius(self.h, _f(cloud), cloud.shape[0], cloud.shape[1], _i(indices),
                                         0 if indices is None else indices.size, int(is_dense), float(radius), _f(vp),
                                         _f(out), nthreads)
        return out, bool(dense)

    def correspondences_normals(self, kind, src_point_normal, tgt_point_normal, k=10,
                                max_distance=np.sqrt(np.finfo(np.float64).max), indices=None, nthreads=1):
        """CorrespondenceEstimationNormalShooting (kind 1) / ...BackProjection (kind 2); both clouds as rows with
        the normal at float offset 4 (pcl::PointNormal); the index must have been built over tgt_point_normal."""
        src, tgt = as_cloud(src_point_normal), as_cloud(tgt_point_normal)
        indices = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
        n = src.shape[0] if indices is None else indices.size
        out = np.empty(max(n, 1), dtype=CORR_DTYPE)
        fpt = C.POINTER(C.c_float)
        m = lib().orc_correspondences_normals(
            self.h, int(kind), _f(src), src.shape[0], src.shape[1], src[:, 4:].ctypes.data_as(fpt), src.shape[1],
            _f(tgt), tgt.shape[1], tgt[:, 4:].ctypes.data_as(fpt), tgt.shape[1], _i(indices),
            0 if indices is None else indices.size, int(k), float(max_distance), out.ctypes.data_as(C.POINTER(Corr)),
            nthreads)
        return out[:m].copy()


def reject_surface_normal(corr, src_normals, tgt_normals, threshold):
    """CorrespondenceRejectorSurfaceNormal; normals as (n,>=3) float rows indexed by index_query / index_match."""
    corr = np.ascontiguousarray(corr, dtype=CORR_DTYPE)
    sn, tn = as_cloud(src_normals), as_cloud(tgt_normals)
    out = np.empty(max(corr.size, 1), dtype=CORR_DTYPE)
    m = lib().orc_reject_surface_normal(corr.ctypes.data_as(C.POINTER(Corr)), corr.size, _f(sn), sn.shape[1], _f(tn),
                                        tn.shape[1], float(threshold), out.ctypes.data_as(C.POINTER(Corr)))
    return out[:m].copy()


def knn_bruteforce(cloud, q, k):
    cloud, q = as_cloud(cloud), as_cloud(q)
    idx = np.empty((q.shape[0], k), dtype=np.int32)
    d2 = np.empty((q.shape[0], k), dtype=np.float32)
    keff = lib().orc_knn_bruteforce(_f(cloud), cloud.shape[0], cloud.shape[1], _f(q), q.shape[0], q.shape[1],
                                    k, _i(idx), _f(d2))
    return idx, d2, keff


def _corr_ptr(corr):
    if corr is None:
        return None, 0
    corr = np.ascontiguousarray(corr, dtype=CORR_DTYPE)
    return corr, corr.size


def estimate_svd(src, tgt, corr=None, scalar_is_double=False, use_umeyama=True):
    src, tgt = as_cloud(src), as_cloud(tgt)
    corr, n = _corr_ptr(corr)
    T = np.zeros(16, dtype=np.float64)
    fn = lib().orc_estimate_svd if use_umeyama else lib().orc_estimate_svd_correlation
    fn(_f(src), src.shape[1], _f(tgt), tgt.shape[1],
                           None if corr is None else corr.ctypes.data_as(C.POINTER(Corr)),
                           n if corr is not None else src.shape[0], int(scalar_is_double), _d(T))
    return T.reshape(4, 4)


def estimate_point_to_plane_lls(src, tgt_point_normal, corr=None, scalar_is_double=False):
    """tgt_point_normal: (n,12) pcl::PointNormal rows (xyz1 | nx ny nz 0 | curv pad3) or (n,>=7) with
    normals at float offset 4."""
    src, tgt = as_cloud(src), as_cloud(tgt_point_normal)
    corr, n = _corr_ptr(corr)
    T = np.zeros(16, dtype=np.float64)
    tn = tgt[:, 4:]
    rc = lib().orc_estimate_point_to_plane_lls(
        _f(src), src.shape[1], _f(tgt), tn.ctypes.data_as(C.POINTER(C.c_float)), tgt.shape[1],
        None if corr is None else corr.ctypes.data_as(C.POINTER(Corr)),
        n if corr is not None else src.shape[0], int(scalar_is_double), _d(T))
    return T.reshape(4, 4), rc


def estimate_symmetric_lls(src_point_normal, tgt_point_normal, corr=None, enforce_same_direction=True, scalar_is_double=False):
    """Both clouds as pcl::PointNormal rows (normals at float offset 4)."""
    src, tgt = as_cloud(src_point_normal), as_cloud(tgt_point_normal)
    corr, n = _corr_ptr(corr)
    T = np.zeros(16, dtype=np.float64)
    rc = lib().orc_estimate_symmetric_lls(
        _f(src), src[:, 4:].ctypes.data_as(C.POINTER(C.c_float)), src.shape[1], _f(tgt),
        tgt[:, 4:].ctypes.data_as(C.POINTER(C.c_float)), tgt.shape[1],
        None if corr is None else corr.ctypes.data_as(C.POINTER(Corr)), n if corr is not None else src.shape[0],
        int(enforce_same_direction), int(scalar_is_double), _d(T))
    return T.reshape(4, 4), rc


def transform(cloud, T, scalar_is_double=False, mode=0, normal_off=-1):
    out = as_cloud(cloud).copy()
    T = np.ascontiguousarray(T, dtype=np.float64)
    lib().orc_transform(_f(out), out.shape[0], out.shape[1], normal_off, _d(T), int(scalar_is_double), mode)
    return out


def icp_align(src, tgt, max_iterations=10, max_correspondence_distance=np.sqrt(np.finfo(np.float64).max),
              transformation_epsilon=0.0, transformation_rotation_epsilon=0.0,
              euclidean_fitness_epsilon=-np.finfo(np.float64).max, use_reciprocal=False, estimator=0,
              scalar_is_double=False, with_normals_transform=False, source_has_normals=False,
              is_dense=True, guess=None, indices=None, nthreads=1, want_cloud=False, index=None, out=None,
              correspondence_kind=0, correspondence_k=10):
    src, tgt = as_cloud(src), as_cloud(tgt)
    P = IcpParams(max_iterations, int(use_reciprocal), estimator, int(scalar_is_double),
                  int(with_normals_transform), int(source_has_normals), int(is_dense), nthreads,
                  float(max_correspondence_distance), float(transformation_epsilon),
                  float(transformation_rotation_epsilon), float(euclidean_fitness_epsilon),
                  int(correspondence_kind), int(correspondence_k))
    R = IcpResult()
    g = None if guess is None else np.ascontiguousarray(guess, dtype=np.float64)
    indices = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
    if out is None:
        out = np.empty_like(src) if want_cloud else None
    if index is not None:
        lib().orc_icp_align_tree(C.byref(P), index.h, _f(src), src.shape[0], src.shape[1], _i(indices),
                                 0 if indices is None else indices.size, _f(tgt), tgt.shape[0], tgt.shape[1],
                                 _d(g), C.byref(R), None if out is None else _f(out))
    else:
        lib().orc_icp_align(C.byref(P), _f(src), src.shape[0], src.shape[1], _i(indices),
                            0 if indices is None else indices.size, _f(tgt), tgt.shape[0], tgt.shape[1], _d(g),
                            C.byref(R), None if out is None else _f(out))
    res = dict(final=np.array(R.final_transformation).reshape(4, 4),
               last=np.array(R.last_transformation).reshape(4, 4), converged=bool(R.converged),
               state=int(R.state), iterations=int(R.iterations), n_correspondences=int(R.n_correspondences),
               mse=float(R.mse), total_correspondences=int(R.total_correspondences))
    if want_cloud:
        res["cloud"] = out
    return res


def reject(corr, kind, p=0.0, min_correspondences=0):
    """Applies one correspondence rejector; returns (remaining, median) (median only meaningful for REJ_MEDIAN)."""
    corr = np.ascontiguousarray(corr, dtype=CORR_DTYPE)
    out = np.empty(max(corr.size, 1), dtype=CORR_DTYPE)
    r = Rejector(kind, min_correspondences, float(p))
    med = C.c_double(0.0)
    m = lib().orc_reject(C.byref(r), corr.ctypes.data_as(C.POINTER(Corr)), corr.size, out.ctypes.data_as(C.POINTER(Corr)),
                         C.byref(med))
    return out[:m].copy(), float(med.value)


def reject_chain(corr, rejectors):
    """The ICP loop's chain [(kind, p, min_correspondences), ...] on a list in position order: every rejector sees the
    survivors in that order (so breaks distance ties by position); returns (remaining in position order, median of the
    last MEDIAN stage)."""
    corr = np.ascontiguousarray(corr, dtype=CORR_DTYPE)
    out = np.empty(max(corr.size, 1), dtype=CORR_DTYPE)
    arr = (Rejector * max(len(rejectors), 1))(*[Rejector(k, m, float(p)) for (k, p, m) in rejectors])
    med = C.c_double(0.0)
    m = lib().orc_reject_chain(arr, len(rejectors), corr.ctypes.data_as(C.POINTER(Corr)), corr.size,
                               out.ctypes.data_as(C.POINTER(Corr)), C.byref(med))
    return out[:m].copy(), float(med.value)


def icp_align_rejectors(src, tgt, rejectors, **kw):
    """ICP with a chain of rejectors [(kind, p, min_correspondences), ...] (icp.hpp:187-201).  The result's
    "correspondences" are those of the last evaluated iteration, after the chain (Registration::correspondences_)."""
    src, tgt = as_cloud(src), as_cloud(tgt)
    has_n = int(kw.get("source_has_normals", False))
    P = IcpParams(kw.get("max_iterations", 10), int(kw.get("use_reciprocal", False)), int(kw.get("estimator", 0)),
                  int(kw.get("scalar_is_double", False)), has_n, has_n, int(kw.get("is_dense", True)),
                  kw.get("nthreads", 1), float(kw.get("max_correspondence_distance", np.sqrt(np.finfo(np.float64).max))),
                  float(kw.get("transformation_epsilon", 0.0)), 0.0, float(kw.get("euclidean_fitness_epsilon", -np.finfo(np.float64).max)),
                  int(kw.get("correspondence_kind", 0)), int(kw.get("correspondence_k", 10)))
    arr = (Rejector * len(rejectors))(*[Rejector(k, m, float(p)) for (k, p, m) in rejectors])
    R = IcpResult()
    indices = kw.get("indices")
    indices = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
    corr = np.empty(max(src.shape[0] if indices is None else indices.size, 1), dtype=CORR_DTYPE)
    nc = C.c_size_t(0)
    lib().orc_icp_align_full(C.byref(P), None, arr, len(rejectors), None, _f(src), src.shape[0], src.shape[1], _i(indices),
                             0 if indices is None else indices.size, _f(tgt), tgt.shape[0], tgt.shape[1], None,
                             C.byref(R), None, corr.ctypes.data_as(C.POINTER(Corr)), C.byref(nc))
    return dict(final=np.array(R.final_transformation).reshape(4, 4), converged=bool(R.converged), state=int(R.state),
                iterations=int(R.iterations), n_correspondences=int(R.n_correspondences), mse=float(R.mse),
                correspondences=corr[:nc.value].copy())


class IcpExt(C.Structure):
    _fields_ = [("failure_after_max_iter", C.c_int32), ("max_iterations_similar_transforms", C.c_int32),
                ("svd_no_umeyama", C.c_int32), ("enforce_same_direction_normals", C.c_int32),
                ("mse_threshold_absolute", C.c_double)]


def icp_align_criteria(src, tgt, max_iterations=10, max_correspondence_distance=np.sqrt(np.finfo(np.float64).max),
                       transformation_epsilon=0.0, transformation_rotation_epsilon=0.0,
                       euclidean_fitness_epsilon=-np.finfo(np.float64).max, mse_threshold_absolute=1e-12,
                       failure_after_max_iter=False, max_iterations_similar_transforms=0, estimator=0,
                       svd_no_umeyama=False, scalar_is_double=False, guess=None, prev_mse=None, nthreads=1):
    """One align with every DefaultConvergenceCriteria knob.  src / tgt: (n, 8) records, xyz 1 | normal 0 (the normals
    feed point-to-plane and the symmetric objective).  prev_mse: the criteria's previous MSE when the align starts (None
    = a new criteria object, DBL_MAX); the result's "prev_mse" is where the align leaves it."""
    src, tgt = as_cloud(src), as_cloud(tgt)
    P = IcpParams(max_iterations, 0, estimator, int(scalar_is_double), int(estimator != 0), int(estimator != 0), 1,
                  nthreads, float(max_correspondence_distance), float(transformation_epsilon),
                  float(transformation_rotation_epsilon), float(euclidean_fitness_epsilon), 0, 10)
    pm = C.c_double(np.finfo(np.float64).max if prev_mse is None else float(prev_mse))
    X = IcpExt(int(failure_after_max_iter), int(max_iterations_similar_transforms), int(svd_no_umeyama), 1,
               float(mse_threshold_absolute))
    R = IcpResult()
    g = None if guess is None else np.ascontiguousarray(guess, dtype=np.float64)
    corr = np.empty(max(src.shape[0], 1), dtype=CORR_DTYPE)
    nc = C.c_size_t(0)
    lib().orc_icp_align_carry(C.byref(P), C.byref(X), None, 0, None, _f(src), src.shape[0], src.shape[1], None, 0,
                              _f(tgt), tgt.shape[0], tgt.shape[1], _d(g), C.byref(R), None,
                              corr.ctypes.data_as(C.POINTER(Corr)), C.byref(nc), C.byref(pm))
    return dict(final=np.array(R.final_transformation).reshape(4, 4), last=np.array(R.last_transformation).reshape(4, 4),
                converged=bool(R.converged), state=int(R.state), iterations=int(R.iterations),
                n_correspondences=int(R.n_correspondences), mse=float(R.mse), prev_mse=float(pm.value),
                correspondences=corr[:nc.value].copy())


def voxelgrid(cloud, leaf, min_points_per_voxel=0, indices=None, is_dense=True):
    cloud = as_cloud(cloud)
    leaf = np.asarray(leaf, dtype=np.float32).reshape(3)
    indices = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
    out = np.empty((max(cloud.shape[0], 1), 4), dtype=np.float32)
    m = lib().orc_voxelgrid(_f(cloud), cloud.shape[0], cloud.shape[1], _i(indices),
                            0 if indices is None else indices.size, int(is_dense), _f(leaf),
                            min_points_per_voxel, _f(out))
    if m < 0:
        return None  # overflow guard: reference returns the input unfiltered
    return out[:m].copy()


def voxelgrid_normals(cloud, leaf, min_points_per_voxel=0, indices=None, is_dense=True, normal_offset=4):
    """VoxelGrid<PointNormal> with downsample_all_data_: (xyz1 rows, {nx,ny,nz,n4,curvature,0,0,0} rows)."""
    cloud = as_cloud(cloud)
    leaf = np.asarray(leaf, dtype=np.float32).reshape(3)
    indices = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
    out = np.empty((max(cloud.shape[0], 1), 4), dtype=np.float32)
    nc = np.empty((max(cloud.shape[0], 1), 8), dtype=np.float32)
    m = lib().orc_voxelgrid_normals(_f(cloud), cloud.shape[0], cloud.shape[1], _i(indices),
                                    0 if indices is None else indices.size, int(is_dense), _f(leaf),
                                    min_points_per_voxel, _f(out), normal_offset, _f(nc))
    if m < 0:
        return None
    return out[:m].copy(), nc[:m].copy()


def point_normal(cloud, indices, is_dense=True):
    cloud = as_cloud(cloud)
    indices = np.ascontiguousarray(indices, dtype=np.int32)
    out = np.empty(4, dtype=np.float32)
    ok = lib().orc_point_normal(_f(cloud), cloud.shape[1], int(is_dense), _i(indices), indices.size, _f(out))
    return out, bool(ok)
