"""pcl_b200 — H100-native ICP registration hot path behind PCL's API.

The product is `libpclb200.so` (CUDA, sm_90a) with the C-ABI in include/pclb200.h and the C++ facade in
pcl_b200/pcl_compat/ (pcl::IterativeClosestPoint, pcl::search::KdTree, ...).  This Python module is only
the ctypes harness that tests and bench.py use to reach the SAME C-ABI; it contains no compute and there
is no CPU fallback: importing works anywhere (the symbols are checked), but every call needs a CUDA device.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PCLB200_LIB", os.path.join(_HERE, "libpclb200.so"))  # override = experiments only

OK = 0
ERR_CUDA, ERR_INVALID, ERR_EMPTY, ERR_LEAF_TOO_SMALL, ERR_INTERNAL, ERR_NCCL = -1, -2, -3, -4, -5, -6
EST_SVD, EST_POINT_TO_PLANE_LLS, EST_SYMMETRIC_POINT_TO_PLANE_LLS = 0, 1, 2
TRACK_AUTO, TRACK_ON, TRACK_OFF = 0, 1, 2
REDUCE_FUSED, REDUCE_NCCL = 0, 1
CONV_NAMES = ["NOT_CONVERGED", "ITERATIONS", "TRANSFORM", "ABS_MSE", "REL_MSE", "NO_CORRESPONDENCES",
              "FAILURE_AFTER_MAX_ITERATIONS"]

CORR_DTYPE = np.dtype([("index_query", np.int32), ("index_match", np.int32), ("distance", np.float32)])


class Pclb200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"pclb200 error {code}: {msg}")
        self.code = code


class IcpParams(C.Structure):
    _fields_ = [("max_iterations", C.c_int32), ("use_reciprocal", C.c_int32), ("estimator", C.c_int32),
                ("scalar_is_double", C.c_int32), ("with_normals_transform", C.c_int32), ("is_dense", C.c_int32),
                ("failure_after_max_iter", C.c_int32), ("max_iterations_similar_transforms", C.c_int32),
                ("enforce_same_direction_normals", C.c_int32), ("correspondence_kind", C.c_int32),
                ("max_correspondence_distance", C.c_double), ("transformation_epsilon", C.c_double),
                ("transformation_rotation_epsilon", C.c_double), ("euclidean_fitness_epsilon", C.c_double),
                ("mse_threshold_absolute", C.c_double), ("correspondence_k", C.c_int32), ("track_mode", C.c_int32), ("svd_no_umeyama", C.c_int32), ("reserved2", C.c_int32)]


class IcpStats(C.Structure):
    _fields_ = [("converged", C.c_int32), ("state", C.c_int32), ("iterations", C.c_int32), ("reserved", C.c_int32),
                ("n_correspondences", C.c_int64), ("mse", C.c_double), ("final_transformation", C.c_double * 16),
                ("last_transformation", C.c_double * 16), ("total_correspondences", C.c_int64), ("total_skipped_walks", C.c_int64)]

    def as_dict(self):
        return dict(converged=bool(self.converged), state=int(self.state), iterations=int(self.iterations),
                    n_correspondences=int(self.n_correspondences), mse=float(self.mse),
                    total_correspondences=int(self.total_correspondences),
                    total_skipped_walks=int(self.total_skipped_walks),
                    final=np.array(self.final_transformation).reshape(4, 4),
                    last=np.array(self.last_transformation).reshape(4, 4))


class Rejector(C.Structure):
    _fields_ = [("kind", C.c_int32), ("min_correspondences", C.c_int32), ("p", C.c_double)]


REJ_DISTANCE, REJ_MEDIAN, REJ_ONE_TO_ONE, REJ_TRIMMED, REJ_SURFACE_NORMAL = 0, 1, 2, 3, 4
CORR_NEAREST, CORR_NORMAL_SHOOTING, CORR_BACK_PROJECTION = 0, 1, 2


# every symbol include/pclb200.h declares (tests/test_capi_symbols.py checks the two lists agree)
SYMBOLS = [
    "pclb200_version", "pclb200_last_error", "pclb200_create", "pclb200_destroy", "pclb200_synchronize",
    "pclb200_launch_count", "pclb200_stream", "pclb200_free", "pclb200_host_register", "pclb200_host_unregister",
    "pclb200_profile_enable", "pclb200_profile_get",
    "pclb200_profile_reset", "pclb200_index_build", "pclb200_index_destroy",
    "pclb200_index_size", "pclb200_index_stats", "pclb200_knn", "pclb200_knn_stats", "pclb200_radius", "pclb200_correspondences",
    "pclb200_estimate_svd", "pclb200_estimate_svd_correlation", "pclb200_estimate_point_to_plane_lls", "pclb200_estimate_symmetric_point_to_plane_lls", "pclb200_icp_default_params",
    "pclb200_icp_create", "pclb200_icp_destroy", "pclb200_icp_set_params", "pclb200_icp_set_target",
    "pclb200_icp_set_source", "pclb200_icp_iterate", "pclb200_icp_get_cloud", "pclb200_icp_get_correspondences",
    "pclb200_icp_align",
    "pclb200_fitness_score", "pclb200_reject", "pclb200_icp_set_rejectors", "pclb200_normals_knn", "pclb200_normals_radius",
    "pclb200_correspondences_normals", "pclb200_reject_surface_normal", "pclb200_cluster_labels", "pclb200_voxelgrid", "pclb200_voxelgrid_normals", "pclb200_voxelgrid_tile", "pclb200_validate_transformation", "pclb200_inliers", "pclb200_radius_into", "pclb200_gicp_covariances", "pclb200_comm_unique_id", "pclb200_comm_set_mode", "pclb200_comm_export", "pclb200_comm_import",
    "pclb200_comm_init",
]
# every symbol include/pclb200_sharded.h declares (the sharded-target extension; tests/test_sharded_target_symbols.py)
SHARDED_SYMBOLS = ["pclb200_index_build_ids", "pclb200_icp_set_target_sharded", "pclb200_fitness_score_sharded",
                   "pclb200_normals_knn_sharded", "pclb200_normals_radius_sharded", "pclb200_cluster_labels_sharded",
                   "pclb200_comm_allgather_u64", "pclb200_knn_sharded", "pclb200_knn_stats_sharded",
                   "pclb200_statistical_outlier_sharded", "pclb200_radius_outlier_sharded", "pclb200_voxelgrid_sharded",
                   "pclb200_correspondences_sharded", "pclb200_correspondences_normals_sharded",
                   "pclb200_validate_transformation_sharded", "pclb200_inliers_sharded", "pclb200_radius_sharded",
                   "pclb200_radius_into_sharded", "pclb200_gicp_covariances_sharded"]
# every symbol include/pclb200_batch.h declares (a batch of ICP problems in one session; tests/test_icp_batch_symbols.py)
BATCH_SYMBOLS = ["pclb200_icp_set_target_batch", "pclb200_icp_set_source_batch", "pclb200_icp_iterate_batch", "pclb200_icp_get_correspondences_batch",
                 "pclb200_index_build_batch", "pclb200_normals_knn_batch", "pclb200_voxelgrid_batch",
                 "pclb200_icp_fitness_score_batch", "pclb200_fitness_score_batch", "pclb200_validate_transformation_batch"]

_lib = None


def lib():
    """Loads libpclb200.so; raises (never falls back) if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: run `python -m pcl_b200.build` (nvcc, sm_90a). "
                          "There is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp, sz, i32p, fp, dp = C.c_void_p, C.c_size_t, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_double)
    L.pclb200_last_error.restype = C.c_char_p
    L.pclb200_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.pclb200_destroy.argtypes = [vp]
    L.pclb200_synchronize.argtypes = [vp]
    L.pclb200_launch_count.argtypes = [vp, C.POINTER(C.c_uint64)]
    L.pclb200_stream.argtypes = [vp, C.POINTER(vp)]
    L.pclb200_free.argtypes = [vp]
    L.pclb200_free.restype = None
    L.pclb200_host_register.argtypes = [vp, vp, C.c_size_t]
    L.pclb200_host_unregister.argtypes = [vp, vp]
    L.pclb200_profile_enable.argtypes = [vp, C.c_int]
    L.pclb200_profile_get.argtypes = [vp, C.c_char_p, dp, C.POINTER(C.c_uint64)]
    L.pclb200_profile_reset.argtypes = [vp]
    L.pclb200_index_build.argtypes = [vp, vp, sz, sz, vp, sz, C.POINTER(vp)]
    L.pclb200_index_build_ids.argtypes = [vp, vp, sz, sz, vp, C.POINTER(vp)]
    L.pclb200_index_destroy.argtypes = [vp]
    L.pclb200_index_size.argtypes = [vp, C.POINTER(sz)]
    L.pclb200_index_stats.argtypes = [vp, C.POINTER(C.c_uint64)]
    L.pclb200_knn.argtypes = [vp, vp, vp, sz, sz, C.c_int, vp, vp, C.POINTER(C.c_int)]
    L.pclb200_knn_stats.argtypes = [vp, vp, vp, sz, sz, vp, sz, C.c_int, vp, vp]
    L.pclb200_radius.argtypes = [vp, vp, vp, sz, sz, C.c_double, C.c_uint, C.c_int, C.POINTER(C.c_int64),
                                 C.POINTER(i32p), C.POINTER(fp)]
    L.pclb200_correspondences.argtypes = [vp, vp, vp, vp, sz, sz, vp, sz, C.c_int, C.c_double, vp, C.POINTER(sz)]
    L.pclb200_estimate_svd.argtypes = [vp, vp, sz, vp, sz, vp, sz, C.c_int, dp]
    L.pclb200_estimate_svd_correlation.argtypes = [vp, vp, sz, vp, sz, vp, sz, C.c_int, dp]
    L.pclb200_estimate_point_to_plane_lls.argtypes = [vp, vp, sz, vp, vp, sz, vp, sz, C.c_int, dp]
    L.pclb200_estimate_symmetric_point_to_plane_lls.argtypes = [vp, vp, vp, sz, vp, vp, sz, vp, sz, C.c_int, C.c_int, dp]
    L.pclb200_icp_default_params.argtypes = [C.POINTER(IcpParams)]
    L.pclb200_icp_default_params.restype = None
    L.pclb200_icp_create.argtypes = [vp, C.POINTER(IcpParams), C.POINTER(vp)]
    L.pclb200_icp_destroy.argtypes = [vp]
    L.pclb200_icp_set_params.argtypes = [vp, C.POINTER(IcpParams)]
    L.pclb200_icp_set_target.argtypes = [vp, vp, vp, sz]
    L.pclb200_icp_set_target_sharded.argtypes = [vp, vp, vp, sz]
    L.pclb200_icp_set_source.argtypes = [vp, vp, sz, sz, vp, sz, vp, sz, dp]
    L.pclb200_icp_iterate.argtypes = [vp, C.c_int, C.POINTER(IcpStats)]
    L.pclb200_icp_get_cloud.argtypes = [vp, vp, sz, vp, sz]
    L.pclb200_icp_get_correspondences.argtypes = [vp, vp, C.POINTER(sz)]
    L.pclb200_icp_align.argtypes = [vp, C.POINTER(IcpParams), vp, sz, sz, vp, sz, vp, sz, vp, vp, sz, dp, vp, sz,
                                    C.POINTER(IcpStats)]
    L.pclb200_reject.argtypes = [vp, C.POINTER(Rejector), vp, sz, vp, C.POINTER(sz), dp]
    L.pclb200_icp_set_rejectors.argtypes = [vp, C.POINTER(Rejector), C.c_int]
    L.pclb200_fitness_score.argtypes = [vp, vp, vp, sz, sz, vp, sz, C.c_int, dp, C.c_int, C.c_double, dp]
    L.pclb200_fitness_score_sharded.argtypes = [vp, vp, vp, sz, sz, vp, sz, C.c_int, dp, C.c_int, C.c_double, dp]
    L.pclb200_normals_knn.argtypes = [vp, vp, vp, sz, sz, vp, sz, C.c_int, C.c_int, fp, vp, C.POINTER(C.c_int)]
    L.pclb200_normals_radius.argtypes = [vp, vp, vp, sz, sz, vp, sz, C.c_int, C.c_double, fp, vp, C.POINTER(C.c_int)]
    L.pclb200_normals_knn_sharded.argtypes = L.pclb200_normals_knn.argtypes
    L.pclb200_normals_radius_sharded.argtypes = L.pclb200_normals_radius.argtypes
    L.pclb200_correspondences_normals.argtypes = [vp, vp, C.c_int, vp, sz, sz, vp, sz, vp, sz, vp, sz, C.c_int, C.c_double,
                                                  vp, C.POINTER(sz)]
    L.pclb200_reject_surface_normal.argtypes = [vp, vp, sz, vp, sz, sz, vp, sz, sz, C.c_double, vp, C.POINTER(sz)]
    L.pclb200_cluster_labels.argtypes = [vp, vp, C.c_double, vp, sz]
    L.pclb200_cluster_labels_sharded.argtypes = [vp, vp, C.c_double, vp, vp, sz]
    L.pclb200_comm_allgather_u64.argtypes = [vp, vp, sz, vp, sz, C.POINTER(sz)]
    L.pclb200_knn_sharded.argtypes = L.pclb200_knn.argtypes
    L.pclb200_knn_stats_sharded.argtypes = L.pclb200_knn_stats.argtypes
    L.pclb200_statistical_outlier_sharded.argtypes = [vp, vp, vp, sz, sz, vp, sz, C.c_int, C.c_double, C.c_int, vp, dp]
    L.pclb200_radius_outlier_sharded.argtypes = [vp, vp, vp, sz, sz, vp, sz, C.c_int, C.c_double, C.c_int, C.c_int, vp]
    L.pclb200_voxelgrid.argtypes = [vp, vp, sz, sz, vp, sz, C.c_int, fp, C.c_uint, vp, C.POINTER(sz)]
    L.pclb200_voxelgrid_tile.argtypes = [vp, vp, sz, sz, fp, fp, C.c_uint, vp, C.POINTER(sz)]
    L.pclb200_voxelgrid_normals.argtypes = [vp, vp, sz, sz, vp, sz, vp, sz, C.c_int, fp, C.c_uint, vp, vp, C.POINTER(sz)]
    L.pclb200_voxelgrid_sharded.argtypes = [vp, vp, sz, sz, vp, vp, sz, fp, C.c_uint, vp, vp, vp, C.POINTER(sz)]
    L.pclb200_validate_transformation.argtypes = [vp, vp, vp, sz, sz, dp, C.c_int, C.c_double, dp]
    L.pclb200_inliers.argtypes = [vp, vp, vp, sz, sz, dp, C.c_float, vp, C.POINTER(sz)]
    L.pclb200_correspondences_sharded.argtypes = [vp, vp, vp, vp, sz, sz, vp, sz, C.c_int, C.c_double, vp, sz, vp, vp, vp,
                                                  C.POINTER(sz)]
    L.pclb200_correspondences_normals_sharded.argtypes = [vp, vp, C.c_int, vp, sz, sz, vp, sz, vp, sz, vp, sz, C.c_int,
                                                          C.c_double, vp, vp, vp, C.POINTER(sz)]
    L.pclb200_validate_transformation_sharded.argtypes = L.pclb200_validate_transformation.argtypes
    L.pclb200_inliers_sharded.argtypes = [vp, vp, vp, sz, sz, dp, C.c_float, vp, vp, C.POINTER(sz)]
    L.pclb200_gicp_covariances.argtypes = [vp, vp, vp, sz, sz, C.c_int, C.c_double, vp]
    L.pclb200_radius_into.argtypes = [vp, vp, vp, sz, sz, C.c_double, C.c_uint, vp, vp, vp, sz, C.POINTER(sz)]
    L.pclb200_radius_sharded.argtypes = L.pclb200_radius.argtypes
    L.pclb200_radius_into_sharded.argtypes = L.pclb200_radius_into.argtypes + [C.POINTER(C.c_int)]
    L.pclb200_gicp_covariances_sharded.argtypes = L.pclb200_gicp_covariances.argtypes
    L.pclb200_comm_unique_id.argtypes = [vp]
    L.pclb200_comm_set_mode.argtypes = [vp, C.c_int]
    L.pclb200_comm_export.argtypes = [vp, vp]
    L.pclb200_comm_import.argtypes = [vp, C.c_int, C.c_int, vp]
    L.pclb200_comm_init.argtypes = [vp, C.c_int, C.c_int, vp]
    L.pclb200_icp_set_target_batch.argtypes = [vp, vp, vp, sz, C.c_int32]
    L.pclb200_icp_set_source_batch.argtypes = [vp, vp, sz, sz, vp, sz, vp, C.c_int32, dp]
    L.pclb200_icp_iterate_batch.argtypes = [vp, C.c_int, vp]
    L.pclb200_icp_get_correspondences_batch.argtypes = [vp, vp, vp]
    L.pclb200_index_build_batch.argtypes = [vp, vp, sz, sz, vp, C.c_int32, vp]
    L.pclb200_normals_knn_batch.argtypes = [vp, vp, C.c_int32, vp, sz, sz, vp, C.c_int, fp, vp, vp]
    L.pclb200_voxelgrid_batch.argtypes = [vp, vp, sz, sz, vp, C.c_int32, fp, C.c_uint, vp, sz, vp, vp, vp]
    L.pclb200_icp_fitness_score_batch.argtypes = [vp, C.c_double, dp]
    L.pclb200_fitness_score_batch.argtypes = [vp, vp, C.c_int32, vp, sz, sz, vp, dp, C.c_int, C.c_double, dp]
    L.pclb200_validate_transformation_batch.argtypes = L.pclb200_fitness_score_batch.argtypes
    for s in SYMBOLS + SHARDED_SYMBOLS + BATCH_SYMBOLS:
        getattr(L, s)  # AttributeError here == header and library disagree
    _lib = L
    return L


def _check(rc):
    if rc != OK:
        raise Pclb200Error(rc, lib().pclb200_last_error().decode("utf-8", "replace"))


def default_params(**kw):
    p = IcpParams()
    lib().pclb200_icp_default_params(C.byref(p))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


class Field:
    """A field inside strided records: e.g. Field(point_normal_array, 4) = the normals of pcl::PointNormal rows."""

    def __init__(self, base, float_offset):
        self.base = base
        self.float_offset = float_offset


class _Buf:
    """A point/normal/index array handed to the C-ABI: numpy (host) or torch (host or cuda)."""

    def __init__(self, a, dtype=np.float32):
        self.keep = a
        if a is None:
            self.ptr, self.rows, self.stride, self.nbytes = None, 0, 0, 0
            return
        if isinstance(a, Field):
            base = _Buf(a.base)
            self.keep = base
            self.ptr = C.c_void_p(base.ptr.value + 4 * a.float_offset)
            self.rows, self.stride = base.rows, base.stride
            return
        if hasattr(a, "data_ptr"):  # torch tensor
            assert a.is_contiguous()
            self.ptr = C.c_void_p(a.data_ptr())
            self.rows = a.shape[0]
            self.stride = a.stride(0) * a.element_size() if a.dim() > 1 else a.element_size()
        else:
            a = np.ascontiguousarray(a, dtype=dtype)
            self.keep = a
            self.ptr = C.c_void_p(a.ctypes.data)
            self.rows = a.shape[0]
            self.stride = a.strides[0]


def xyz1(a):
    """(n,3) -> (n,4) float32 {x,y,z,1} (pcl::PointXYZ records)."""
    a = np.asarray(a, dtype=np.float32)
    out = np.ones((a.shape[0], 4), dtype=np.float32)
    out[:, :3] = a[:, :3]
    return out


class Context:
    def __init__(self, device=0):
        self.h = C.c_void_p()
        _check(lib().pclb200_create(device, C.byref(self.h)))

    def close(self):
        if self.h:
            lib().pclb200_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def synchronize(self):
        _check(lib().pclb200_synchronize(self.h))

    def host_register(self, array):
        """Page-lock a host numpy array in place (cudaHostRegister): later calls move it by DMA.  Undo with
        host_unregister before the array is freed."""
        b = _Buf(array)
        _check(lib().pclb200_host_register(self.h, b.ptr, int(np.asarray(array).nbytes)))

    def host_unregister(self, array):
        _check(lib().pclb200_host_unregister(self.h, _Buf(array).ptr))

    @property
    def launches(self):
        v = C.c_uint64()
        _check(lib().pclb200_launch_count(self.h, C.byref(v)))
        return int(v.value)

    @property
    def stream(self):
        s = C.c_void_p()
        _check(lib().pclb200_stream(self.h, C.byref(s)))
        return s.value or 0

    def profile(self, enable=True):
        _check(lib().pclb200_profile_enable(self.h, int(enable)))

    def profile_reset(self):
        _check(lib().pclb200_profile_reset(self.h))

    def profile_get(self, name):
        ms, n = C.c_double(), C.c_uint64()
        _check(lib().pclb200_profile_get(self.h, name.encode(), C.byref(ms), C.byref(n)))
        return float(ms.value), int(n.value)

    def index_build_batch(self, cloud, offsets):
        """One Index per cloud, cloud c being the records [offsets[c], offsets[c+1]) of `cloud` (numpy, or a torch tensor on
        the host or the device), built in one batch: each is bit for bit Index(ctx, that cloud alone) and owns its handle."""
        b = _Buf(cloud)
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        nc = max(off.size - 1, 0)
        out = (C.c_void_p * max(nc, 1))()
        _check(lib().pclb200_index_build_batch(self.h, b.ptr, b.rows, b.stride, C.c_void_p(off.ctypes.data), nc, out))
        return [Index._adopt(self, out[c], off[c + 1] - off[c]) for c in range(nc)]

    def normals_knn_batch(self, indices, cloud, offsets, k, viewpoints=None, out=None):
        """The k-NN normals of B query sets in one call: set c = the records [offsets[c], offsets[c+1]) of `cloud` (numpy,
        or a torch tensor on the host or the device), searched in indices[c]; each set's rows and is_dense are bit for
        bit indices[c].normals_knn(its records, k, its viewpoint).  viewpoints: None (the origin), one xyz for every set
        or (B, 3).  Returns (out (n, 4), is_dense (B,) bool); out[offsets[c]:offsets[c+1]] are set c's normals, as
        Icp.set_target_batch takes them."""
        b = _Buf(cloud)
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        B = max(off.size - 1, 0)
        handles = (C.c_void_p * max(B, 1))(*[None if i is None else i.h for i in indices])
        vp = None
        if viewpoints is not None:
            v = np.asarray(viewpoints, dtype=np.float32)
            vp = np.ascontiguousarray(np.broadcast_to(v, (B, 3)) if v.ndim == 1 else v, dtype=np.float32)
            if vp.shape != (B, 3):
                raise ValueError("normals_knn_batch: viewpoints must be one xyz or one row of xyz per set")
        if out is None:
            out = np.empty((b.rows, 4), dtype=np.float32)
        ob = _Buf(out)
        dense = np.zeros(max(B, 1), dtype=np.int32)
        _check(lib().pclb200_normals_knn_batch(self.h, handles, B, b.ptr, b.rows, b.stride, C.c_void_p(off.ctypes.data),
                                               int(k), None if vp is None else vp.ctypes.data_as(C.POINTER(C.c_float)),
                                               ob.ptr, C.c_void_p(dense.ctypes.data)))
        return out, dense[:B].astype(bool)

    def voxelgrid_batch(self, cloud, offsets, leaf, min_points_per_voxel=0, normal_offset=None, out=None, out_normals=None):
        """VoxelGrid of B clouds in one call: cloud c = the records [offsets[c], offsets[c+1]) of `cloud` (numpy, or a torch
        tensor on the host or the device).  Returns (rows, out_offsets), or (rows, normal_rows, out_offsets) when
        normal_offset is given (pcl::PointNormal: 4): cloud c's rows are rows[out_offsets[c]:out_offsets[c+1]], bit for bit
        voxelgrid (voxelgrid_normals) of that cloud alone; rows and out_offsets go straight to index_build_batch once the
        empty ranges are dropped.  out / out_normals: caller buffers of (n, 4) / (n, 8) float32, returned as views; by
        default the rows come back as trimmed host copies."""
        b = _Buf(cloud)
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        B = max(off.size - 1, 0)
        leaf = (C.c_float * 3)(*[float(x) for x in np.broadcast_to(np.asarray(leaf, dtype=np.float32), (3,))])
        with_normals = normal_offset is not None
        nb = _Buf(Field(cloud, normal_offset) if with_normals else None)
        host_out, host_nout = out is None, out_normals is None
        if host_out:
            out = np.empty((max(b.rows, 1), 4), dtype=np.float32)
        if with_normals and host_nout:
            out_normals = np.empty((max(b.rows, 1), 8), dtype=np.float32)
        ob, onb = _Buf(out), _Buf(out_normals if with_normals else None)
        out_off = np.zeros(B + 1, dtype=np.int64)
        _check(lib().pclb200_voxelgrid_batch(self.h, b.ptr, b.rows, b.stride, C.c_void_p(off.ctypes.data), B, leaf,
                                             int(min_points_per_voxel), nb.ptr, nb.stride, ob.ptr, onb.ptr,
                                             C.c_void_p(out_off.ctypes.data)))
        m = int(out_off[B])
        rows = out[:m].copy() if host_out else out[:m]
        if not with_normals:
            return rows, out_off
        return rows, (out_normals[:m].copy() if host_nout else out_normals[:m]), out_off

    def fitness_score_batch(self, indices, cloud, offsets, transforms, max_range=np.finfo(np.float64).max,
                            scalar_is_double=False):
        """getFitnessScore of B problems in one call: problem p = the records [offsets[p], offsets[p+1]) of `cloud` (numpy,
        or a torch tensor on the host or the device) moved by transforms[p] ((B, 4, 4) or (B, 16)) and scored against
        indices[p].  Returns B float64 scores, each bit for bit indices[p].fitness_score(its records, transforms[p],
        max_range, scalar_is_double)."""
        return self._score_batch(lib().pclb200_fitness_score_batch, indices, cloud, offsets, transforms, max_range,
                                 scalar_is_double)

    def validate_transformation_batch(self, indices, cloud, offsets, transforms, max_range=np.finfo(np.float64).max,
                                      scalar_is_double=False):
        """TransformationValidationEuclidean of B problems in one call: as fitness_score_batch, each score bit for bit
        indices[p].validate_transformation(its records, transforms[p], max_range, scalar_is_double)."""
        return self._score_batch(lib().pclb200_validate_transformation_batch, indices, cloud, offsets, transforms,
                                 max_range, scalar_is_double)

    def _score_batch(self, fn, indices, cloud, offsets, transforms, max_range, scalar_is_double):
        b = _Buf(cloud)
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        B = max(off.size - 1, 0)
        handles = (C.c_void_p * max(B, 1))(*[None if i is None else i.h for i in indices])
        T = np.ascontiguousarray(transforms, dtype=np.float64).reshape(-1, 16)
        if T.shape[0] != B:
            raise ValueError("one 4x4 transform per problem")
        scores = np.empty(max(B, 1), dtype=np.float64)
        _check(fn(self.h, handles, B, b.ptr, b.rows, b.stride, C.c_void_p(off.ctypes.data),
                  T.ctypes.data_as(C.POINTER(C.c_double)), int(scalar_is_double), float(max_range),
                  scores.ctypes.data_as(C.POINTER(C.c_double))))
        return scores[:B]

    def comm_init(self, rank, nranks, unique_id_bytes):
        buf = C.create_string_buffer(bytes(unique_id_bytes), 128)
        _check(lib().pclb200_comm_init(self.h, rank, nranks, buf))

    def comm_set_mode(self, mode):
        _check(lib().pclb200_comm_set_mode(self.h, int(mode)))

    def allgather_u64(self, values):
        """Collective: every rank's uint64 values concatenated in rank order (the same array on every rank)."""
        v = np.ascontiguousarray(values, dtype=np.uint64)
        total = C.c_size_t()
        _check(lib().pclb200_comm_allgather_u64(self.h, C.c_void_p(v.ctypes.data), v.size, None, 0, C.byref(total)))
        out = np.empty(max(total.value, 1), dtype=np.uint64)
        _check(lib().pclb200_comm_allgather_u64(self.h, C.c_void_p(v.ctypes.data), v.size, C.c_void_p(out.ctypes.data),
                                                out.size, C.byref(total)))
        return out[:total.value]

    def comm_export(self):
        buf = C.create_string_buffer(64)
        _check(lib().pclb200_comm_export(self.h, buf))
        return buf.raw

    def comm_import(self, rank, nranks, handles):
        """handles: the nranks 64-byte blobs of comm_export, in rank order."""
        blob = b"".join(bytes(h) for h in handles)
        assert len(blob) == 64 * nranks
        buf = C.create_string_buffer(blob, len(blob))
        _check(lib().pclb200_comm_import(self.h, rank, nranks, buf))

    # ---- stand-alone operators -----------------------------------------------------------------
    def voxelgrid(self, cloud, leaf, min_points_per_voxel=0, indices=None, is_dense=True, out=None):
        b = _Buf(cloud)
        ib = _Buf(indices, np.int32)
        n = ib.rows if indices is not None else b.rows
        leaf = (C.c_float * 3)(*[float(x) for x in np.broadcast_to(np.asarray(leaf, dtype=np.float32), (3,))])
        host_out = out is None
        if host_out:
            out = np.empty((max(n, 1), 4), dtype=np.float32)
        ob = _Buf(out)
        m = C.c_size_t()
        _check(lib().pclb200_voxelgrid(self.h, b.ptr, b.rows, b.stride, ib.ptr, ib.rows, int(is_dense), leaf,
                                       int(min_points_per_voxel), ob.ptr, C.byref(m)))
        return out[:m.value].copy() if host_out else out[:m.value]

    def voxelgrid_tile(self, cloud, leaf, grid_bounds, min_points_per_voxel=0, out=None):
        """VoxelGrid of one spatial tile on the grid of the whole cloud (grid_bounds = its min xyz + max xyz)."""
        b = _Buf(cloud)
        leaf = (C.c_float * 3)(*[float(x) for x in np.broadcast_to(np.asarray(leaf, dtype=np.float32), (3,))])
        gb = (C.c_float * 6)(*[float(x) for x in np.asarray(grid_bounds, dtype=np.float32).reshape(6)])
        host_out = out is None
        if host_out:
            out = np.empty((max(b.rows, 1), 4), dtype=np.float32)
        ob = _Buf(out)
        m = C.c_size_t()
        _check(lib().pclb200_voxelgrid_tile(self.h, b.ptr, b.rows, b.stride, gb, leaf, int(min_points_per_voxel), ob.ptr,
                                            C.byref(m)))
        return out[:m.value].copy() if host_out else out[:m.value]

    def voxelgrid_normals(self, cloud, leaf, min_points_per_voxel=0, indices=None, is_dense=True, normal_offset=4):
        """VoxelGrid<PointNormal> with downsample_all_data_ = true: (xyz1 rows, {nx,ny,nz,n4,curvature,0,0,0} rows)."""
        b = _Buf(cloud)
        nb = _Buf(Field(cloud, normal_offset))
        ib = _Buf(indices, np.int32)
        n = ib.rows if indices is not None else b.rows
        leaf = (C.c_float * 3)(*[float(x) for x in np.broadcast_to(np.asarray(leaf, dtype=np.float32), (3,))])
        out = np.empty((max(n, 1), 4), dtype=np.float32)
        nc = np.empty((max(n, 1), 8), dtype=np.float32)
        m = C.c_size_t()
        _check(lib().pclb200_voxelgrid_normals(self.h, b.ptr, b.rows, b.stride, nb.ptr, nb.stride, ib.ptr, ib.rows,
                                               int(is_dense), leaf, int(min_points_per_voxel),
                                               C.c_void_p(out.ctypes.data), C.c_void_p(nc.ctypes.data), C.byref(m)))
        return out[:m.value].copy(), nc[:m.value].copy()

    def voxelgrid_sharded(self, cloud, ids, leaf, min_points_per_voxel=0, normal_offset=None):
        """Collective VoxelGrid of a map sharded across the communicator's ranks: this rank's records and their ids in,
        this rank's share of the whole map's output out, as (xyz1 rows, uint32 voxel indices) or, with the normal at float
        normal_offset of each record (PointNormal: 4), (xyz1 rows, voxel indices, {nx,ny,nz,n4,curvature,0,0,0} rows).
        Stable-sorting every rank's rows by voxel index gives pclb200_voxelgrid(_normals) of the whole map."""
        b = _Buf(cloud)
        ib = _Buf(ids, np.int32)
        nb = _Buf(Field(cloud, normal_offset) if normal_offset is not None else None)
        n = max(b.rows, 1)
        leaf = (C.c_float * 3)(*[float(x) for x in np.broadcast_to(np.asarray(leaf, dtype=np.float32), (3,))])
        out = np.empty((n, 4), dtype=np.float32)
        vox = np.empty(n, dtype=np.uint32)
        nc = np.empty((n, 8), dtype=np.float32) if normal_offset is not None else None
        m = C.c_size_t()
        _check(lib().pclb200_voxelgrid_sharded(self.h, b.ptr, b.rows, b.stride, ib.ptr, nb.ptr, nb.stride, leaf,
                                               int(min_points_per_voxel), C.c_void_p(out.ctypes.data),
                                               None if nc is None else C.c_void_p(nc.ctypes.data),
                                               C.c_void_p(vox.ctypes.data), C.byref(m)))
        got = (out[:m.value].copy(), vox[:m.value].copy())
        return got if nc is None else got + (nc[:m.value].copy(),)

    def reject(self, corr, kind, p=0.0, min_correspondences=0):
        """One correspondence rejector (getRemainingCorrespondences); returns (remaining, median)."""
        corr = np.ascontiguousarray(corr, dtype=CORR_DTYPE)
        out = np.empty(max(corr.size, 1), dtype=CORR_DTYPE)
        r = Rejector(kind, min_correspondences, float(p))
        m, med = C.c_size_t(), C.c_double()
        _check(lib().pclb200_reject(self.h, C.byref(r), C.c_void_p(corr.ctypes.data), corr.size,
                                    C.c_void_p(out.ctypes.data), C.byref(m), C.byref(med)))
        return out[:m.value].copy(), float(med.value)

    def reject_surface_normal(self, corr, src_normals, tgt_normals, threshold):
        """CorrespondenceRejectorSurfaceNormal; normals are arrays (or Fields) indexed by index_query / index_match."""
        corr = np.ascontiguousarray(corr, dtype=CORR_DTYPE)
        out = np.empty(max(corr.size, 1), dtype=CORR_DTYPE)
        sn, tn = _Buf(src_normals), _Buf(tgt_normals)
        m = C.c_size_t()
        _check(lib().pclb200_reject_surface_normal(self.h, C.c_void_p(corr.ctypes.data), corr.size, sn.ptr, sn.rows,
                                                   sn.stride, tn.ptr, tn.rows, tn.stride, float(threshold),
                                                   C.c_void_p(out.ctypes.data), C.byref(m)))
        return out[:m.value].copy()

    def estimate_svd(self, src, tgt, corr=None, scalar_is_double=False, use_umeyama=True):
        s, t = _Buf(src), _Buf(tgt)
        cb = None if corr is None else np.ascontiguousarray(corr, dtype=CORR_DTYPE)
        n = s.rows if cb is None else cb.size
        T = np.zeros(16)
        fn = lib().pclb200_estimate_svd if use_umeyama else lib().pclb200_estimate_svd_correlation
        _check(fn(self.h, s.ptr, s.stride, t.ptr, t.stride,
                                          None if cb is None else C.c_void_p(cb.ctypes.data), n, int(scalar_is_double),
                                          T.ctypes.data_as(C.POINTER(C.c_double))))
        return T.reshape(4, 4)

    def estimate_symmetric_lls(self, src_point_normal, tgt_point_normal, corr=None, enforce_same_direction=True,
                               scalar_is_double=False):
        src = np.ascontiguousarray(src_point_normal, dtype=np.float32)
        tgt = np.ascontiguousarray(tgt_point_normal, dtype=np.float32)
        cb = None if corr is None else np.ascontiguousarray(corr, dtype=CORR_DTYPE)
        n = src.shape[0] if cb is None else cb.size
        T = np.zeros(16)
        _check(lib().pclb200_estimate_symmetric_point_to_plane_lls(
            self.h, C.c_void_p(src.ctypes.data), C.c_void_p(src.ctypes.data + 16), src.strides[0],
            C.c_void_p(tgt.ctypes.data), C.c_void_p(tgt.ctypes.data + 16), tgt.strides[0],
            None if cb is None else C.c_void_p(cb.ctypes.data), n, int(enforce_same_direction), int(scalar_is_double),
            T.ctypes.data_as(C.POINTER(C.c_double))))
        return T.reshape(4, 4)

    def estimate_point_to_plane_lls(self, src, tgt_point_normal, corr=None, scalar_is_double=False):
        tgt = np.ascontiguousarray(tgt_point_normal, dtype=np.float32)
        s, t = _Buf(src), _Buf(tgt)
        cb = None if corr is None else np.ascontiguousarray(corr, dtype=CORR_DTYPE)
        n = s.rows if cb is None else cb.size
        T = np.zeros(16)
        _check(lib().pclb200_estimate_point_to_plane_lls(
            self.h, s.ptr, s.stride, t.ptr, C.c_void_p(tgt.ctypes.data + 16), t.stride,
            None if cb is None else C.c_void_p(cb.ctypes.data), n, int(scalar_is_double),
            T.ctypes.data_as(C.POINTER(C.c_double))))
        return T.reshape(4, 4)


class Index:
    """pcl::search::KdTree<PointT> / pcl::KdTreeFLANN replacement (LBVH in HBM).

    ids: label point i with ids[i] instead of i (one tile of a map sharded across ranks); exclusive with subset."""

    def __init__(self, ctx, cloud, subset=None, ids=None):
        self.ctx = ctx
        b = _Buf(cloud)
        self.n_cloud = b.rows
        self.h = C.c_void_p()
        if ids is not None:
            if subset is not None:
                raise ValueError("Index: subset and ids are exclusive")
            ib = _Buf(ids, np.int32)
            if ib.rows != b.rows:
                raise ValueError("Index: ids must have one entry per point")
            _check(lib().pclb200_index_build_ids(ctx.h, b.ptr, b.rows, b.stride, ib.ptr, C.byref(self.h)))
            return
        sb = _Buf(subset, np.int32)
        _check(lib().pclb200_index_build(ctx.h, b.ptr, b.rows, b.stride, sb.ptr, sb.rows, C.byref(self.h)))

    @classmethod
    def _adopt(cls, ctx, handle, n_cloud):
        """An Index that owns `handle`, an index of n_cloud records already built on ctx (nothing is rebuilt)."""
        self = cls.__new__(cls)
        self.ctx = ctx
        self.n_cloud = int(n_cloud)
        self.h = C.c_void_p(handle)
        return self

    def close(self):
        if getattr(self, "h", None):
            lib().pclb200_index_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def size(self):
        v = C.c_size_t()
        _check(lib().pclb200_index_size(self.h, C.byref(v)))
        return int(v.value)

    @property
    def stats(self):
        a = (C.c_uint64 * 4)()
        _check(lib().pclb200_index_stats(self.h, a))
        return dict(leaves=int(a[0]), nodes=int(a[1]), bytes=int(a[2]), leaf_size=int(a[3]))

    def knn(self, q, k, out_idx=None, out_d2=None):
        b = _Buf(q)
        if out_idx is None:
            out_idx = np.empty((b.rows, max(k, 0)), dtype=np.int32)
            out_d2 = np.empty((b.rows, max(k, 0)), dtype=np.float32)
        oi, od = _Buf(out_idx, np.int32), _Buf(out_d2)
        keff = C.c_int()
        _check(lib().pclb200_knn(self.ctx.h, self.h, b.ptr, b.rows, b.stride, k, oi.ptr, od.ptr, C.byref(keff)))
        return out_idx, out_d2, int(keff.value)

    def knn_stats(self, cloud, k, indices=None):
        """(mean distance to the k-1 nearest other points, squared distance of neighbour k-1) per point."""
        b, ib = _Buf(cloud), _Buf(indices, np.int32)
        n = ib.rows if indices is not None else b.rows
        mean, kth = np.empty(n, np.float32), np.empty(n, np.float32)
        _check(lib().pclb200_knn_stats(self.ctx.h, self.h, b.ptr, b.rows, b.stride, ib.ptr, ib.rows, k,
                                       C.c_void_p(mean.ctypes.data), C.c_void_p(kth.ctypes.data)))
        return mean, kth

    def radius(self, q, r, max_nn=0, sorted_results=True):
        b = _Buf(q)
        offs = np.zeros(b.rows + 1, dtype=np.int64)
        pi, pd = C.POINTER(C.c_int32)(), C.POINTER(C.c_float)()
        _check(lib().pclb200_radius(self.ctx.h, self.h, b.ptr, b.rows, b.stride, float(r), int(max_nn),
                                    int(sorted_results), offs.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(pi),
                                    C.byref(pd)))
        total = int(offs[-1])
        idx = np.ctypeslib.as_array(pi, shape=(max(total, 1),))[:total].copy()
        d2 = np.ctypeslib.as_array(pd, shape=(max(total, 1),))[:total].copy()
        lib().pclb200_free(pi)
        lib().pclb200_free(pd)
        return offs, idx, d2

    def radius_into(self, q, r, offsets, idx, d2, max_nn=0):
        """radiusSearch into caller buffers (numpy or torch, host or cuda); returns the total number of neighbours —
        when it exceeds the capacity of idx / d2 only `offsets` was written."""
        b = _Buf(q)
        ob, ib, db = _Buf(offsets, np.int64), _Buf(idx, np.int32), _Buf(d2)
        total = C.c_size_t()
        _check(lib().pclb200_radius_into(self.ctx.h, self.h, b.ptr, b.rows, b.stride, float(r), int(max_nn), ob.ptr,
                                         ib.ptr, db.ptr, min(ib.rows, db.rows), C.byref(total)))
        return int(total.value)

    def correspondences(self, src, max_distance=np.sqrt(np.finfo(np.float64).max), indices=None, is_dense=True,
                        src_index=None):
        b = _Buf(src)
        ib = _Buf(indices, np.int32)
        n = ib.rows if indices is not None else b.rows
        out = np.empty(max(n, 1), dtype=CORR_DTYPE)
        m = C.c_size_t()
        _check(lib().pclb200_correspondences(self.ctx.h, self.h, None if src_index is None else src_index.h, b.ptr,
                                             b.rows, b.stride, ib.ptr, ib.rows, int(is_dense), float(max_distance),
                                             C.c_void_p(out.ctypes.data), C.byref(m)))
        return out[:m.value]

    def correspondences_normals(self, kind, src, src_normals, tgt_normals=None, k=10,
                                max_distance=np.sqrt(np.finfo(np.float64).max), indices=None):
        """CorrespondenceEstimationNormalShooting (kind 1) / ...BackProjection (kind 2)."""
        b, sn, tn = _Buf(src), _Buf(src_normals), _Buf(tgt_normals)
        ib = _Buf(indices, np.int32)
        n = ib.rows if indices is not None else b.rows
        out = np.empty(max(n, 1), dtype=CORR_DTYPE)
        m = C.c_size_t()
        _check(lib().pclb200_correspondences_normals(self.ctx.h, self.h, int(kind), b.ptr, b.rows, b.stride, sn.ptr,
                                                     sn.stride, tn.ptr, tn.stride, ib.ptr, ib.rows, int(k),
                                                     float(max_distance), C.c_void_p(out.ctypes.data), C.byref(m)))
        return out[:m.value]

    def fitness_score(self, src, T, max_range=np.finfo(np.float64).max, scalar_is_double=False, indices=None,
                      is_dense=True):
        b = _Buf(src)
        ib = _Buf(indices, np.int32)
        T = np.ascontiguousarray(T, dtype=np.float64)
        out = C.c_double()
        _check(lib().pclb200_fitness_score(self.ctx.h, self.h, b.ptr, b.rows, b.stride, ib.ptr, ib.rows, int(is_dense),
                                           T.ctypes.data_as(C.POINTER(C.c_double)), int(scalar_is_double),
                                           float(max_range), C.byref(out)))
        return float(out.value)

    def fitness_score_sharded(self, src, T, max_range=np.finfo(np.float64).max, scalar_is_double=False, indices=None,
                              is_dense=True):
        """Collective getFitnessScore over a target sharded across the communicator's ranks (this index = this rank's
        tile, built with ids=...; every rank passes the same source)."""
        b = _Buf(src)
        ib = _Buf(indices, np.int32)
        T = np.ascontiguousarray(T, dtype=np.float64)
        out = C.c_double()
        _check(lib().pclb200_fitness_score_sharded(self.ctx.h, self.h, b.ptr, b.rows, b.stride, ib.ptr, ib.rows,
                                                   int(is_dense), T.ctypes.data_as(C.POINTER(C.c_double)),
                                                   int(scalar_is_double), float(max_range), C.byref(out)))
        return float(out.value)

    def gicp_covariances(self, cloud, k=20, gicp_epsilon=0.001):
        """GeneralizedIterativeClosestPoint::computeCovariances: (n, 3, 3) float64 for the indexed cloud."""
        b = _Buf(cloud)
        out = np.zeros((b.rows, 9), dtype=np.float64)
        _check(lib().pclb200_gicp_covariances(self.ctx.h, self.h, b.ptr, b.rows, b.stride, int(k), float(gicp_epsilon),
                                              C.c_void_p(out.ctypes.data)))
        return out.reshape(-1, 3, 3)

    def validate_transformation(self, src, T, max_range=np.finfo(np.float64).max, scalar_is_double=False):
        """TransformationValidationEuclidean::validateTransformation."""
        b = _Buf(src)
        T = np.ascontiguousarray(T, dtype=np.float64)
        out = C.c_double()
        _check(lib().pclb200_validate_transformation(self.ctx.h, self.h, b.ptr, b.rows, b.stride,
                                                     T.ctypes.data_as(C.POINTER(C.c_double)), int(scalar_is_double),
                                                     float(max_range), C.byref(out)))
        return float(out.value)

    def inliers(self, src, T, inlier_threshold):
        """SampleConsensusPrerejective::getFitness: (inlier indices, fitness = float mean of their squared distances)."""
        b = _Buf(src)
        T = np.ascontiguousarray(T, dtype=np.float64)
        out = np.empty(max(b.rows, 1), dtype=CORR_DTYPE)
        m = C.c_size_t()
        _check(lib().pclb200_inliers(self.ctx.h, self.h, b.ptr, b.rows, b.stride, T.ctypes.data_as(C.POINTER(C.c_double)),
                                     float(inlier_threshold), C.c_void_p(out.ctypes.data), C.byref(m)))
        c = out[:m.value]
        fit = np.float32(0.0)
        for d in c["distance"]:   # sequential float sum, like the reference's loop
            fit = np.float32(fit + d)
        fit = np.float32(fit / np.float32(m.value)) if m.value else np.finfo(np.float32).max
        return c["index_query"].copy(), float(fit)

    def correspondences_sharded(self, src, max_distance=np.sqrt(np.finfo(np.float64).max), indices=None, is_dense=True,
                                src_index=None, tgt_normals=None, rows=False, normal_rows=False):
        """Collective correspondences over a map sharded across the communicator's ranks (this index = this rank's tile,
        built with ids=...; every rank passes the same source, src_index = its own ordinary index of that source for the
        reciprocal variant).  Returns the list, or (list, xyz1 rows, normal rows) when rows / normal_rows: the matched map
        point {x, y, z, 1} and its normal {nx, ny, nz, 0} per correspondence (normal_rows needs tgt_normals, one per
        record of the tile), numpy float32 (m, 4), or None for the rows not asked for."""
        b, ib, tn = _Buf(src), _Buf(indices, np.int32), _Buf(tgt_normals)
        n = ib.rows if indices is not None else b.rows
        out = np.empty(max(n, 1), dtype=CORR_DTYPE)
        xyz = np.empty((max(n, 1), 4), np.float32) if rows else None
        nrm = np.empty((max(n, 1), 4), np.float32) if normal_rows else None
        m = C.c_size_t()
        _check(lib().pclb200_correspondences_sharded(
            self.ctx.h, self.h, None if src_index is None else src_index.h, b.ptr, b.rows, b.stride, ib.ptr, ib.rows,
            int(is_dense), float(max_distance), tn.ptr, tn.stride, C.c_void_p(out.ctypes.data),
            None if xyz is None else C.c_void_p(xyz.ctypes.data), None if nrm is None else C.c_void_p(nrm.ctypes.data),
            C.byref(m)))
        corr = out[:m.value]
        if not (rows or normal_rows):
            return corr
        return corr, None if xyz is None else xyz[:m.value], None if nrm is None else nrm[:m.value]

    def correspondences_normals_sharded(self, kind, src, src_normals, tgt_normals=None, k=10,
                                        max_distance=np.sqrt(np.finfo(np.float64).max), indices=None, rows=False,
                                        normal_rows=False):
        """Collective correspondences_normals over a map sharded across the communicator's ranks (this index = this
        rank's tile, built with ids=...; tgt_normals: one per record of the tile; every rank passes the same source).
        Returns the list, or (list, xyz1 rows, normal rows) as correspondences_sharded does."""
        b, sn, tn, ib = _Buf(src), _Buf(src_normals), _Buf(tgt_normals), _Buf(indices, np.int32)
        n = ib.rows if indices is not None else b.rows
        out = np.empty(max(n, 1), dtype=CORR_DTYPE)
        xyz = np.empty((max(n, 1), 4), np.float32) if rows else None
        nrm = np.empty((max(n, 1), 4), np.float32) if normal_rows else None
        m = C.c_size_t()
        _check(lib().pclb200_correspondences_normals_sharded(
            self.ctx.h, self.h, int(kind), b.ptr, b.rows, b.stride, sn.ptr, sn.stride, tn.ptr, tn.stride, ib.ptr, ib.rows,
            int(k), float(max_distance), C.c_void_p(out.ctypes.data), None if xyz is None else C.c_void_p(xyz.ctypes.data),
            None if nrm is None else C.c_void_p(nrm.ctypes.data), C.byref(m)))
        corr = out[:m.value]
        if not (rows or normal_rows):
            return corr
        return corr, None if xyz is None else xyz[:m.value], None if nrm is None else nrm[:m.value]

    def validate_transformation_sharded(self, src, T, max_range=np.finfo(np.float64).max, scalar_is_double=False):
        """Collective validate_transformation over a map sharded across the communicator's ranks (this index = this
        rank's tile; every rank passes the same source): the same value on every rank."""
        b = _Buf(src)
        T = np.ascontiguousarray(T, dtype=np.float64)
        out = C.c_double()
        _check(lib().pclb200_validate_transformation_sharded(self.ctx.h, self.h, b.ptr, b.rows, b.stride,
                                                             T.ctypes.data_as(C.POINTER(C.c_double)),
                                                             int(scalar_is_double), float(max_range), C.byref(out)))
        return float(out.value)

    def inliers_sharded(self, src, T, inlier_threshold, rows=False):
        """Collective pclb200_inliers over a map sharded across the communicator's ranks: the inlier correspondence list
        (and, with rows, the matched map points as {x, y, z, 1} rows), the same on every rank."""
        b = _Buf(src)
        T = np.ascontiguousarray(T, dtype=np.float64)
        out = np.empty(max(b.rows, 1), dtype=CORR_DTYPE)
        xyz = np.empty((max(b.rows, 1), 4), np.float32) if rows else None
        m = C.c_size_t()
        _check(lib().pclb200_inliers_sharded(self.ctx.h, self.h, b.ptr, b.rows, b.stride,
                                             T.ctypes.data_as(C.POINTER(C.c_double)), float(inlier_threshold),
                                             C.c_void_p(out.ctypes.data), None if xyz is None else C.c_void_p(xyz.ctypes.data),
                                             C.byref(m)))
        return (out[:m.value], xyz[:m.value]) if rows else out[:m.value]

    def normals_knn(self, cloud, k, viewpoint=(0, 0, 0), indices=None, is_dense=True, out=None):
        b = _Buf(cloud)
        ib = _Buf(indices, np.int32)
        n = ib.rows if indices is not None else b.rows
        if out is None:
            out = np.empty((n, 4), dtype=np.float32)
        ob = _Buf(out)
        vp = (C.c_float * 3)(*[float(v) for v in viewpoint])
        dense = C.c_int()
        _check(lib().pclb200_normals_knn(self.ctx.h, self.h, b.ptr, b.rows, b.stride, ib.ptr, ib.rows, int(is_dense), k,
                                         vp, ob.ptr, C.byref(dense)))
        return out, bool(dense.value)


    def cluster_labels(self, tolerance, out=None):
        """Connected components of d2 < tolerance^2 over the indexed points: label = smallest original index of the
        component, -1 for points the index does not hold."""
        if out is None:
            out = np.empty(self.n_cloud, dtype=np.int32)
        ob = _Buf(out, np.int32)
        _check(lib().pclb200_cluster_labels(self.ctx.h, self.h, float(tolerance), ob.ptr, self.n_cloud))
        return out

    def euclidean_clusters(self, tolerance, min_size=1, max_size=2 ** 32 - 1):
        """EuclideanClusterExtraction::extract: list of index arrays (ascending inside a cluster), largest first,
        equal sizes ordered by their smallest index."""
        return clusters_from_labels(self.cluster_labels(tolerance), min_size, max_size)

    def cluster_labels_sharded(self, tolerance, out=None, sizes=None):
        """Collective cluster_labels over a map sharded across the communicator's ranks (this index = this rank's tile,
        built with ids=...): (labels, sizes) per record of the tile.  labels[i] is the whole map's label of ids[i] (the
        smallest id of its component, -1 for a non-finite record); sizes[i] the number of distinct ids in that component
        (0 for a non-finite record).  out / sizes: numpy or torch, host or cuda."""
        if out is None:
            out = np.empty(self.n_cloud, dtype=np.int32)
        if sizes is None:
            sizes = np.empty(self.n_cloud, dtype=np.int64)
        ob, sb = _Buf(out, np.int32), _Buf(sizes, np.int64)
        _check(lib().pclb200_cluster_labels_sharded(self.ctx.h, self.h, float(tolerance), ob.ptr, sb.ptr, self.n_cloud))
        return out, sizes

    def euclidean_clusters_sharded(self, tolerance, ids, min_size=1, max_size=2 ** 32 - 1):
        """Collective euclidean_clusters over a sharded map (ids: the ids this tile was built with).  This rank's part of
        every whole-map cluster whose size is within [min_size, max_size], as ascending id arrays, in the order
        euclidean_clusters gives the whole map (size descending, then smallest id).  Every rank returns a list of the
        same length; a rank that holds no point of a cluster gets an empty array in its place, and an id held by two
        ranks is in both ranks' parts."""
        ids = np.asarray(ids, dtype=np.int64)
        labels, sizes = self.cluster_labels_sharded(tolerance)
        keep = (labels >= 0) & (sizes >= min_size) & (sizes <= max_size)
        # (size << 32) | label of every cluster in the window, from every rank (sizes and labels are below 2^31)
        mine = np.unique((sizes[keep].astype(np.uint64) << np.uint64(32)) | labels[keep].astype(np.uint64))
        every = np.unique(self.ctx.allgather_u64(mine))
        size, label = (every >> np.uint64(32)).astype(np.int64), (every & np.uint64(0xffffffff)).astype(np.int64)
        label = label[np.lexsort((label, -size))]
        order = np.lexsort((ids[keep], labels[keep]))  # this rank's records of the window by (label, id)
        lab_sorted, id_sorted = labels[keep][order], ids[keep][order]
        lo, hi = np.searchsorted(lab_sorted, label, "left"), np.searchsorted(lab_sorted, label, "right")
        return [id_sorted[a:b].astype(np.int32) for a, b in zip(lo, hi)]

    def normals_radius(self, cloud, radius, viewpoint=(0, 0, 0), indices=None, is_dense=True, out=None):
        """NormalEstimation with setRadiusSearch(radius)."""
        b = _Buf(cloud)
        ib = _Buf(indices, np.int32)
        n = ib.rows if indices is not None else b.rows
        if out is None:
            out = np.empty((n, 4), dtype=np.float32)
        ob = _Buf(out)
        vp = (C.c_float * 3)(*[float(v) for v in viewpoint])
        dense = C.c_int()
        _check(lib().pclb200_normals_radius(self.ctx.h, self.h, b.ptr, b.rows, b.stride, ib.ptr, ib.rows, int(is_dense),
                                            float(radius), vp, ob.ptr, C.byref(dense)))
        return out, bool(dense.value)

    def _normals_sharded(self, fn, cloud, param, viewpoint, indices, is_dense, out):
        b = _Buf(cloud)
        ib = _Buf(indices, np.int32)
        n = ib.rows if indices is not None else b.rows
        if out is None:
            out = np.empty((n, 4), dtype=np.float32)
        ob = _Buf(out)
        vp = (C.c_float * 3)(*[float(v) for v in viewpoint])
        dense = C.c_int()
        _check(fn(self.ctx.h, self.h, b.ptr, b.rows, b.stride, ib.ptr, ib.rows, int(is_dense), param, vp, ob.ptr,
                  C.byref(dense)))
        return out, bool(dense.value)

    def normals_knn_sharded(self, cloud, k, viewpoint=(0, 0, 0), indices=None, is_dense=True, out=None):
        """Collective normals_knn over a map sharded across the communicator's ranks (this index = this rank's tile,
        built with ids=...; cloud = this rank's own queries): bit for bit one index of the whole map's answer."""
        return self._normals_sharded(lib().pclb200_normals_knn_sharded, cloud, int(k), viewpoint, indices, is_dense, out)

    def normals_radius_sharded(self, cloud, radius, viewpoint=(0, 0, 0), indices=None, is_dense=True, out=None):
        """Collective normals_radius over a map sharded across the communicator's ranks (see normals_knn_sharded)."""
        return self._normals_sharded(lib().pclb200_normals_radius_sharded, cloud, float(radius), viewpoint, indices,
                                     is_dense, out)

    def knn_sharded(self, q, k, out_idx=None, out_d2=None):
        """Collective knn over a map sharded across the communicator's ranks (this index = this rank's tile, built with
        ids=...; q = this rank's own queries): (ids, d2, k_eff), bit for bit one index of the whole map's answer."""
        b = _Buf(q)
        if out_idx is None:
            out_idx = np.empty((b.rows, max(k, 0)), dtype=np.int32)
            out_d2 = np.empty((b.rows, max(k, 0)), dtype=np.float32)
        oi, od = _Buf(out_idx, np.int32), _Buf(out_d2)
        keff = C.c_int()
        _check(lib().pclb200_knn_sharded(self.ctx.h, self.h, b.ptr, b.rows, b.stride, k, oi.ptr, od.ptr, C.byref(keff)))
        return out_idx, out_d2, int(keff.value)

    def knn_stats_sharded(self, cloud, k, indices=None):
        """Collective knn_stats over a sharded map (see knn_sharded): bit for bit one index of the whole map's answer."""
        b, ib = _Buf(cloud), _Buf(indices, np.int32)
        n = ib.rows if indices is not None else b.rows
        mean, kth = np.empty(n, np.float32), np.empty(n, np.float32)
        _check(lib().pclb200_knn_stats_sharded(self.ctx.h, self.h, b.ptr, b.rows, b.stride, ib.ptr, ib.rows, k,
                                               C.c_void_p(mean.ctypes.data), C.c_void_p(kth.ctypes.data)))
        return mean, kth

    def statistical_outlier_removal_sharded(self, cloud, mean_k, std_mul, negative=False, indices=None):
        """Collective StatisticalOutlierRemoval over a sharded map, its statistics taken over every rank's queries:
        (keep mask of this rank's queries as uint8, dict(valid, mean, thr) the same on every rank)."""
        b, ib = _Buf(cloud), _Buf(indices, np.int32)
        n = ib.rows if indices is not None else b.rows
        keep = np.empty(n, np.uint8)
        stats = np.zeros(3)
        _check(lib().pclb200_statistical_outlier_sharded(self.ctx.h, self.h, b.ptr, b.rows, b.stride, ib.ptr, ib.rows,
                                                         int(mean_k), float(std_mul), int(negative),
                                                         C.c_void_p(keep.ctypes.data),
                                                         stats.ctypes.data_as(C.POINTER(C.c_double))))
        return keep, dict(valid=int(stats[0]), mean=float(stats[1]), thr=float(stats[2]))

    def radius_outlier_removal_sharded(self, cloud, radius, min_pts, negative=False, is_dense=True, indices=None):
        """Collective RadiusOutlierRemoval over a sharded map: the keep mask of this rank's queries as uint8 (the dense
        rule only when every rank passes is_dense)."""
        b, ib = _Buf(cloud), _Buf(indices, np.int32)
        n = ib.rows if indices is not None else b.rows
        keep = np.empty(n, np.uint8)
        _check(lib().pclb200_radius_outlier_sharded(self.ctx.h, self.h, b.ptr, b.rows, b.stride, ib.ptr, ib.rows,
                                                    int(is_dense), float(radius), int(min_pts), int(negative),
                                                    C.c_void_p(keep.ctypes.data)))
        return keep

    def radius_sharded(self, q, r, max_nn=0, sorted_results=True):
        """Collective radius over a map sharded across the communicator's ranks (this index = this rank's tile, built with
        ids=...; q = this rank's own queries, r and max_nn its own): (offsets, ids, d2), bit for bit one index of the whole
        map's answer."""
        b = _Buf(q)
        offs = np.zeros(b.rows + 1, dtype=np.int64)
        pi, pd = C.POINTER(C.c_int32)(), C.POINTER(C.c_float)()
        try:
            _check(lib().pclb200_radius_sharded(self.ctx.h, self.h, b.ptr, b.rows, b.stride, float(r), int(max_nn),
                                                int(sorted_results), offs.ctypes.data_as(C.POINTER(C.c_int64)),
                                                C.byref(pi), C.byref(pd)))
            total = int(offs[-1])
            idx = np.ctypeslib.as_array(pi, shape=(total,)).copy() if total else np.zeros(0, np.int32)
            d2 = np.ctypeslib.as_array(pd, shape=(total,)).copy() if total else np.zeros(0, np.float32)
        finally:
            lib().pclb200_free(pi)
            lib().pclb200_free(pd)
        return offs, idx, d2

    def radius_into_sharded(self, q, r, offsets, idx, d2, max_nn=0):
        """Collective radius_into over a sharded map (see radius_sharded) into caller buffers (numpy or torch, host or
        cuda): (total, all_fit).  total is this rank's number of neighbours; when it exceeds the capacity of idx / d2 only
        `offsets` was written.  all_fit, the same on every rank, says whether every rank's lists fit: while it is False,
        every rank grows its buffers to its total and calls again."""
        b = _Buf(q)
        ob, ib, db = _Buf(offsets, np.int64), _Buf(idx, np.int32), _Buf(d2)
        total, fit = C.c_size_t(), C.c_int()
        _check(lib().pclb200_radius_into_sharded(self.ctx.h, self.h, b.ptr, b.rows, b.stride, float(r), int(max_nn),
                                                 ob.ptr, ib.ptr, db.ptr, min(ib.rows, db.rows), C.byref(total),
                                                 C.byref(fit)))
        return int(total.value), bool(fit.value)

    def gicp_covariances_sharded(self, cloud, k=20, gicp_epsilon=0.001, out=None):
        """Collective gicp_covariances over a sharded map (cloud = the records this tile was built from): (n, 3, 3)
        float64, row i bit for bit row ids[i] of one index of the whole map's answer.  out: (n, 9) float64, numpy or
        torch, host or cuda (returned as given)."""
        b = _Buf(cloud)
        ret = out
        if out is None:
            out = np.zeros((b.rows, 9), dtype=np.float64)
            ret = out.reshape(-1, 3, 3)
        ob = _Buf(out, np.float64)
        _check(lib().pclb200_gicp_covariances_sharded(self.ctx.h, self.h, b.ptr, b.rows, b.stride, int(k),
                                                      float(gicp_epsilon), ob.ptr))
        return ret


def clusters_from_labels(labels, min_size=1, max_size=2 ** 32 - 1):
    """Groups component labels into clusters the way EuclideanClusterExtraction::extract returns them
    (extract_clusters.hpp:98-113, 249): indices ascending inside a cluster, clusters by size descending."""
    labels = np.asarray(labels)
    valid = np.nonzero(labels >= 0)[0]
    order = valid[np.argsort(labels[valid], kind="stable")]
    lab_sorted = labels[order]
    starts = np.nonzero(np.r_[True, lab_sorted[1:] != lab_sorted[:-1]])[0] if order.size else np.zeros(0, np.int64)
    ends = np.r_[starts[1:], order.size] if order.size else starts
    out = [order[b:e].astype(np.int32) for b, e in zip(starts, ends) if min_size <= e - b <= max_size]
    out.sort(key=lambda a: (-a.size, int(a[0])))
    return out


class Icp:
    """Session form of pcl::IterativeClosestPoint[WithNormals] (set_target / set_source / iterate)."""

    def __init__(self, ctx, params=None, **kw):
        self.ctx = ctx
        self.params = params if params is not None else default_params(**kw)
        self.h = C.c_void_p()
        _check(lib().pclb200_icp_create(ctx.h, C.byref(self.params), C.byref(self.h)))
        self._keep = []

    def close(self):
        if getattr(self, "h", None):
            lib().pclb200_icp_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_rejectors(self, rejectors):
        """rejectors: [(kind, p, min_correspondences), ...] applied in order every iteration; [] clears."""
        arr = (Rejector * max(len(rejectors), 1))(*[Rejector(k, m, float(p)) for (k, p, m) in rejectors])
        _check(lib().pclb200_icp_set_rejectors(self.h, arr, len(rejectors)))

    def set_target(self, index, normals=None):
        nb = _Buf(normals)
        self._keep = [index]
        _check(lib().pclb200_icp_set_target(self.h, index.h, nb.ptr, nb.stride))

    def set_target_sharded(self, tile_index, normals=None):
        """Collective: this rank's tile of a map sharded across the communicator's ranks (an Index built with ids=...);
        normals: one per point of the tile.  Every rank then passes the same whole source to set_source."""
        nb = _Buf(normals)
        self._keep = [tile_index]
        _check(lib().pclb200_icp_set_target_sharded(self.h, tile_index.h, nb.ptr, nb.stride))

    def set_source(self, src, normals=None, indices=None, guess=None):
        b, nb, ib = _Buf(src), _Buf(normals), _Buf(indices, np.int32)
        g = None if guess is None else np.ascontiguousarray(guess, dtype=np.float64)
        _check(lib().pclb200_icp_set_source(self.h, b.ptr, b.rows, b.stride, nb.ptr, nb.stride, ib.ptr, ib.rows,
                                            None if g is None else g.ctypes.data_as(C.POINTER(C.c_double))))
        self.n_src = b.rows
        self.n_queries = ib.rows if indices is not None else b.rows

    def iterate(self, max_steps=2 ** 31 - 1):
        st = IcpStats()
        _check(lib().pclb200_icp_iterate(self.h, int(max_steps), C.byref(st)))
        return st.as_dict()

    def get_correspondences(self):
        out = np.empty(max(self.n_queries, 1), dtype=CORR_DTYPE)
        m = C.c_size_t()
        _check(lib().pclb200_icp_get_correspondences(self.h, C.c_void_p(out.ctypes.data), C.byref(m)))
        return out[:m.value]

    def set_target_batch(self, indices, normals=None):
        """One target per problem of the next set_source_batch: problem p runs as a session after set_target(indices[p],
        normals[p]) would, bit for bit.  normals: None or a list of B arrays (or None entries) of one stride."""
        B = len(indices)
        handles = (C.c_void_p * max(B, 1))(*[None if i is None else i.h for i in indices])
        bufs = [None if x is None else _Buf(x) for x in normals] if normals is not None else []
        strides = {b.stride for b in bufs if b is not None}
        if len(strides) > 1:
            raise ValueError("set_target_batch: every normals array must have the same row stride")
        nptr = (C.c_void_p * max(B, 1))(*[None if b is None else b.ptr for b in bufs]) if normals is not None else None
        _check(lib().pclb200_icp_set_target_batch(self.h, handles, nptr, strides.pop() if strides else 0, B))
        self._keep = [list(indices), bufs]

    def set_source_batch(self, src, offsets, normals=None, guesses=None):
        """B problems against the session's target, problem p = records offsets[p]:offsets[p+1] of src (B + 1 offsets);
        guesses: (B, 4, 4) or None.  Each problem then runs as its own set_source session would, bit for bit."""
        b, nb = _Buf(src), _Buf(normals)
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        g = None if guesses is None else np.ascontiguousarray(guesses, dtype=np.float64)
        _check(lib().pclb200_icp_set_source_batch(self.h, b.ptr, b.rows, b.stride, nb.ptr, nb.stride,
                                                  off.ctypes.data_as(C.c_void_p), len(off) - 1,
                                                  None if g is None else g.ctypes.data_as(C.POINTER(C.c_double))))
        self.n_src = self.n_queries = b.rows
        self.n_problems = len(off) - 1

    def iterate_batch(self, max_steps=2 ** 31 - 1):
        """one list entry per problem: the dict iterate() returns"""
        st = (IcpStats * self.n_problems)()
        _check(lib().pclb200_icp_iterate_batch(self.h, int(max_steps), C.cast(st, C.c_void_p)))
        return [x.as_dict() for x in st]

    def get_correspondences_batch(self):
        """one array per problem: what get_correspondences() of its own session returns"""
        out = np.empty(max(self.n_queries, 1), dtype=CORR_DTYPE)
        counts = np.zeros(self.n_problems, dtype=np.int64)
        _check(lib().pclb200_icp_get_correspondences_batch(self.h, C.c_void_p(out.ctypes.data),
                                                           C.c_void_p(counts.ctypes.data)))
        ends = np.cumsum(counts)
        return [out[e - c:e].copy() for c, e in zip(counts, ends)]

    def fitness_score_batch(self, max_range=np.finfo(np.float64).max):
        """getFitnessScore(max_range) of every problem under its current final transformation: B float64 scores, each bit
        for bit Context.fitness_score_batch of the session's source, offsets, targets and final transformations.  The
        session's loop state is left as it was."""
        scores = np.empty(max(getattr(self, "n_problems", 0), 1), dtype=np.float64)
        _check(lib().pclb200_icp_fitness_score_batch(self.h, float(max_range),
                                                     scores.ctypes.data_as(C.POINTER(C.c_double))))
        return scores[:getattr(self, "n_problems", 0)]

    def get_cloud(self, out=None, stride_floats=4, normals=None):
        if out is None:
            out = np.zeros((self.n_src, stride_floats), dtype=np.float32)
        ob, nb = _Buf(out), _Buf(normals)
        _check(lib().pclb200_icp_get_cloud(self.h, ob.ptr, ob.stride, nb.ptr, nb.stride))
        return out


def icp_align(ctx, src, index_tgt, params=None, src_normals=None, tgt_normals=None, indices=None, guess=None,
              out_cloud=None, **kw):
    """One-call Registration::align."""
    p = params if params is not None else default_params(**kw)
    b, sn, tn, ib, ob = _Buf(src), _Buf(src_normals), _Buf(tgt_normals), _Buf(indices, np.int32), _Buf(out_cloud)
    g = None if guess is None else np.ascontiguousarray(guess, dtype=np.float64)
    st = IcpStats()
    _check(lib().pclb200_icp_align(ctx.h, C.byref(p), b.ptr, b.rows, b.stride, sn.ptr, sn.stride, ib.ptr, ib.rows,
                                   index_tgt.h, tn.ptr, tn.stride,
                                   None if g is None else g.ctypes.data_as(C.POINTER(C.c_double)), ob.ptr, ob.stride,
                                   C.byref(st)))
    return st.as_dict()


def comm_unique_id():
    buf = C.create_string_buffer(128)
    _check(lib().pclb200_comm_unique_id(buf))
    return buf.raw
