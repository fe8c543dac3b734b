/* pclb200.h — C-ABI of libpclb200.so: an H100-native (sm_90a) replacement for the ICP registration
 * hot path of PointCloudLibrary/pcl 1.15.
 *
 * PCL has no C plugin ABI; its extension points are C++ virtual classes injected by shared_ptr
 * (pcl::search::KdTree<PointT>, pcl::registration::CorrespondenceEstimationBase,
 * pcl::registration::TransformationEstimation, pcl::Registration).  This header is what an FFI for
 * that path binds: every entry point names the reference interface it replaces (file:line relative
 * to the PCL source root).  The C++ facade in pcl_b200/pcl_compat/ re-creates the PCL classes on
 * top of it; INTEGRATION.md shows the subclass a PCL maintainer would add.
 *
 * Conventions
 *   - every function returns an int status: 0 = OK, < 0 = error (text via pclb200_last_error(),
 *     thread-local); nothing throws across the boundary; there is NO CPU fallback — without a
 *     CUDA device pclb200_create fails.
 *   - point arrays are raw bytes + a stride: pcl::PointXYZ = 16, pcl::PointNormal = 48, packed
 *     xyz = 12.  x,y,z are the first three floats of each record
 *     (common/include/pcl/impl/point_types.hpp:205-322).  Normals, where needed, are passed as a
 *     separate pointer to the first nx with their own stride (PointNormal: base + 16, stride 48).
 *   - every `const void*` point/normal/index array may be HOST memory (pageable or pinned) or
 *     DEVICE memory on the ctx's GPU; the library detects which (cudaPointerGetAttributes) and
 *     skips the staging copy for device-resident data.  Output arrays follow the same rule.
 *   - indices are int32 == pcl::index_t (common/include/pcl/types.h:112); distances are SQUARED,
 *     fp32, computed as ((dx*dx)+dy*dy)+dz*dz without fma (flann::L2_Simple order); exact ties are
 *     broken by the smaller original index.
 *   - 4x4 transforms cross the boundary as 16 doubles, ROW-major (a float result is widened).
 */
#ifndef PCLB200_H_
#define PCLB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define PCLB200_API __attribute__((visibility("default")))
#else
#define PCLB200_API
#endif

#define PCLB200_VERSION 100 /* 0.1.0 */

/* status codes */
#define PCLB200_OK 0
#define PCLB200_ERR_CUDA -1          /* CUDA runtime error (no device, OOM, launch failure) */
#define PCLB200_ERR_INVALID -2       /* bad argument (NULL, k < 0, stride < 12, ...) */
#define PCLB200_ERR_EMPTY -3         /* empty cloud / no finite point: kdtree_flann.hpp:118-129 */
#define PCLB200_ERR_LEAF_TOO_SMALL -4 /* VoxelGrid int32 overflow guard: voxel_grid.hpp:620-629 */
#define PCLB200_ERR_INTERNAL -5      /* traversal stack overflow or other invariant violation */
#define PCLB200_ERR_NCCL -6

typedef struct pclb200_ctx pclb200_ctx;     /* one per GPU: stream, memory pool, optional NCCL comm */
typedef struct pclb200_index pclb200_index; /* Morton-sorted LBVH over one cloud, resident in HBM */
typedef struct pclb200_icp pclb200_icp;     /* one registration session (device-resident state) */

/* pcl::Correspondence — common/include/pcl/correspondence.h:60-71 */
typedef struct pclb200_corr {
  int32_t index_query;
  int32_t index_match;
  float distance; /* squared */
} pclb200_corr;

PCLB200_API int pclb200_version(void);
PCLB200_API const char* pclb200_last_error(void);

/* ---- context ------------------------------------------------------------------------------- */
PCLB200_API int pclb200_create(int device, pclb200_ctx** out);
PCLB200_API int pclb200_destroy(pclb200_ctx* ctx);
/* blocks until all work queued on the ctx's stream has finished */
PCLB200_API int pclb200_synchronize(pclb200_ctx* ctx);
/* number of kernels this library has launched on ctx since creation (bench.py's gpu_launches) */
PCLB200_API int pclb200_launch_count(pclb200_ctx* ctx, uint64_t* out);
/* raw cudaStream_t of the ctx (so callers can record CUDA events on the launching stream) */
PCLB200_API int pclb200_stream(pclb200_ctx* ctx, void** out_stream);
PCLB200_API void pclb200_free(void* host_ptr); /* frees arrays returned by pclb200_radius */
/* Page-lock a host buffer the caller owns (a std::vector's storage, an mmap'ed PCD body) so that every later call that
 * takes it as an input or output moves it by DMA at PCIe rate instead of through the driver's pageable staging path —
 * the "pinned reader" of SURVEY.md §8f #3: read the file into the buffer, register it once, hand it to
 * pclb200_index_build / pclb200_icp_set_source.  Unregister before the buffer is freed or reallocated.  Registering a
 * buffer twice, or a device pointer, is PCLB200_ERR_INVALID. */
PCLB200_API int pclb200_host_register(pclb200_ctx* ctx, void* host_ptr, size_t bytes);
PCLB200_API int pclb200_host_unregister(pclb200_ctx* ctx, void* host_ptr);
/* measurement hooks (bench.py's roofline leg): when enabled, the library brackets its named kernels
 * ("icp_iter", "solve", "query_sort", "index_build", "normals", "knn", "voxelgrid", "transform_out") with
 * CUDA events on the ctx stream; profile_get synchronises, returns the summed device time and the number of
 * bracketed launches of that name since the last reset, and profile_reset drops the records. */
PCLB200_API int pclb200_profile_enable(pclb200_ctx* ctx, int enable);
PCLB200_API int pclb200_profile_get(pclb200_ctx* ctx, const char* name, double* total_ms, uint64_t* count);
PCLB200_API int pclb200_profile_reset(pclb200_ctx* ctx);

/* ---- index: replaces pcl::KdTreeFLANN<PointT>::setInputCloud(cloud, indices) ------------------
 * kdtree/include/pcl/kdtree/impl/kdtree_flann.hpp:100-136, 429-498 (reached through
 * pcl::search::KdTree::setInputCloud, search/include/pcl/search/impl/kdtree.hpp:89-98).
 * Non-finite points are dropped; results carry ORIGINAL cloud indices (index_mapping_).
 * subset == NULL indexes the whole cloud.  Empty / all-NaN input => PCLB200_ERR_EMPTY. */
PCLB200_API int pclb200_index_build(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride,
                                    const int32_t* subset, size_t n_subset, pclb200_index** out);
PCLB200_API int pclb200_index_destroy(pclb200_index* idx);
PCLB200_API int pclb200_index_size(const pclb200_index* idx, size_t* n_valid);
/* build statistics: [0] leaves, [1] internal nodes, [2] bytes resident in HBM, [3] leaf size */
PCLB200_API int pclb200_index_stats(const pclb200_index* idx, uint64_t out[4]);

/* ---- k-NN: replaces pcl::KdTreeFLANN::nearestKSearch and the batch overload of
 * pcl::search::Search (kdtree_flann.hpp:234-274; search/include/pcl/search/impl/search.hpp:111-137).
 * Exact.  k is clamped to the number of indexed points (returned in *k_eff); outputs are nq rows
 * of pitch k, ascending (d2, index); unused slots are (-1, +inf). */
PCLB200_API int pclb200_knn(pclb200_ctx* ctx, const pclb200_index* idx, const void* queries,
                            size_t nq, size_t stride, int k, int32_t* out_idx, float* out_d2,
                            int* k_eff);

/* ---- k-NN statistics: the per-point quantities pcl::StatisticalOutlierRemoval and pcl::RadiusOutlierRemoval derive
 * from nearestKSearch (filters/include/pcl/filters/impl/statistical_outlier_removal.hpp:72-97,
 * radius_outlier_removal.hpp:74-118), computed on the device so only 4-8 bytes per point come back (SURVEY.md §8f #4).
 * out_mean (nullable): mean distance to neighbours 1..k'-1 (neighbour 0 = the query itself), k' = min(k, indexed points);
 *   0 for non-finite queries.  out_kth (nullable): squared distance of neighbour k-1, +inf if fewer than k points. */
PCLB200_API int pclb200_knn_stats(pclb200_ctx* ctx, const pclb200_index* idx, const void* pts, size_t n, size_t stride,
                                  const int32_t* indices, size_t n_idx, int k, float* out_mean, float* out_kth);

/* ---- radius: replaces pcl::KdTreeFLANN::radiusSearch (kdtree_flann.hpp:372-414) and the batch
 * overload search.hpp:157-194.  Neighbours with d2 < float(radius*radius) (strict, FLANN
 * RadiusResultSet); max_nn == 0 or > N => unlimited, else the max_nn nearest; always returned
 * ascending by (d2, index) (a sorted list is a valid answer for sorted == 0 too).
 * out_offsets: caller array of nq+1; *out_idx / *out_d2: malloc'd host arrays of
 * out_offsets[nq] entries, release with pclb200_free. */
PCLB200_API int pclb200_radius(pclb200_ctx* ctx, const pclb200_index* idx, const void* queries,
                               size_t nq, size_t stride, double radius, unsigned max_nn, int sorted,
                               int64_t* out_offsets, int32_t** out_idx, float** out_d2);
/* The same search into CALLER buffers (host — preferably pinned — or device): no allocation, no pageable staging.
 * out_offsets: nq + 1 entries; out_idx / out_d2: `capacity` entries each; *total = number of neighbours found.  If
 * *total > capacity nothing is written to out_idx / out_d2 (offsets and *total are valid): call again with larger
 * buffers, or first with capacity = 0 to size them.  With device buffers the lists never leave HBM. */
PCLB200_API int pclb200_radius_into(pclb200_ctx* ctx, const pclb200_index* idx, const void* queries, size_t nq,
                                    size_t stride, double radius, unsigned max_nn, int64_t* out_offsets,
                                    int32_t* out_idx, float* out_d2, size_t capacity, size_t* total);

/* ---- correspondences: replaces CorrespondenceEstimation::determineCorrespondences and
 * ::determineReciprocalCorrespondences (registration/include/pcl/registration/impl/
 * correspondence_estimation.hpp:145-218, 220-311).
 * src_indices == NULL => all points (PCLBase::initCompute identity indices).  is_dense == 0 skips
 * non-finite source points (:173-174).  Pairs with d2 > max_dist*max_dist are dropped (:176).
 * idx_src != NULL selects the reciprocal variant: idx_src must index the same `src` array and
 * `tgt` must be the cloud idx_tgt was built from.  out: capacity n_idx (or n) records, ordered by
 * index_query; *n_out receives the count. */
PCLB200_API int pclb200_correspondences(pclb200_ctx* ctx, const pclb200_index* idx_tgt,
                                        const pclb200_index* idx_src, const void* src, size_t n,
                                        size_t stride, const int32_t* src_indices, size_t n_idx,
                                        int is_dense, double max_dist, pclb200_corr* out,
                                        size_t* n_out);

/* ---- correspondences from the k nearest + normals (SURVEY.md §8f #2): replaces
 * CorrespondenceEstimationNormalShooting::determineCorrespondences
 *   (registration/include/pcl/registration/impl/correspondence_estimation_normal_shooting.hpp:66-131): among the k
 *   nearest target points, the one closest to the line through the source point along its normal (|N x V|^2 in
 *   double); that squared line distance is gated against max_dist itself (:121, as in the reference); the stored
 *   distance is the squared point distance (:126) — kind = PCLB200_CORR_NORMAL_SHOOTING, tgt_normals unused;
 * CorrespondenceEstimationBackProjection::determineCorrespondences
 *   (impl/correspondence_estimation_backprojection.hpp:66-118): minimises d2 * (2 - cos^2(n_src, n_tgt)) in float —
 *   kind = PCLB200_CORR_BACK_PROJECTION.
 * src_normals: n records (same indexing as src); tgt_normals: one record per point of the cloud idx_tgt was built
 * from.  Non-finite source points produce no pair.  out: capacity n_idx (or n), ordered by index_query. */
#define PCLB200_CORR_NEAREST 0
#define PCLB200_CORR_NORMAL_SHOOTING 1
#define PCLB200_CORR_BACK_PROJECTION 2
PCLB200_API int pclb200_correspondences_normals(pclb200_ctx* ctx, const pclb200_index* idx_tgt, int kind,
                                                const void* src, size_t n, size_t stride, const void* src_normals,
                                                size_t stride_sn, const void* tgt_normals, size_t stride_tn,
                                                const int32_t* src_indices, size_t n_idx, int k, double max_dist,
                                                pclb200_corr* out, size_t* n_out);

/* ---- correspondence rejectors (SURVEY.md §8f #1): the stage between estimation and solve, icp.hpp:187-201 -------
 * DISTANCE   CorrespondenceRejectorDistance        registration/src/correspondence_rejection_distance.cpp:44-68
 *            p = maximum distance (NOT squared, as setMaximumDistance takes it); keeps distance < p*p
 * MEDIAN     CorrespondenceRejectorMedianDistance  .../correspondence_rejection_median_distance.cpp:44-70
 *            p = median factor; keeps distance <= median * p; *median_out = the median (squared) distance
 * ONE_TO_ONE CorrespondenceRejectorOneToOne        .../correspondence_rejection_one_to_one.cpp:44-71
 *            the closest query of every index_match; output ordered by index_match
 * TRIMMED    CorrespondenceRejectorTrimmed         .../correspondence_rejection_trimmed.cpp:44-63
 *            p = overlap ratio, clamped like setOverlapRatio: min(1, max(0, float(p))), NaN gives 0;
 *            min_correspondences is read as the unsigned int of setMinCorrespondences (-1 is 2^32 - 1);
 *            keep = max(floor(p * float(n)) in float, min): when keep < n the keep smallest distances (sorted output),
 *            otherwise the input unchanged
 * Exact-distance ties (std::sort in the reference is unstable) resolve to the entry that comes first in the input.
 * Distances may be any float but NaN (NaN is outside the contract): -0.0 compares equal to +0.0 and is reported as
 * +0.0 when it is the median, negatives come before zero, +inf after FLT_MAX. */
#define PCLB200_REJ_DISTANCE 0
#define PCLB200_REJ_MEDIAN 1
#define PCLB200_REJ_ONE_TO_ONE 2
#define PCLB200_REJ_TRIMMED 3
/* SURFACE_NORMAL CorrespondenceRejectorSurfaceNormal .../correspondence_rejection_surface_normal.cpp:43-66
 *            p = threshold; keeps pairs whose normals' float dot product, as double, is > p (correspondence_rejection.h
 *            :378-389).  Inside an ICP session it sees the rotated source normals and the target normals given to
 *            set_source / set_target; stand-alone use goes through pclb200_reject_surface_normal (it needs the normals). */
#define PCLB200_REJ_SURFACE_NORMAL 4
typedef struct pclb200_rejector {
  int32_t kind;
  int32_t min_correspondences; /* TRIMMED only (nr_min_correspondences_) */
  double p;
} pclb200_rejector;
/* getRemainingCorrespondences: in/out may be host or device arrays; out capacity n */
PCLB200_API int pclb200_reject(pclb200_ctx* ctx, const pclb200_rejector* rejector, const pclb200_corr* in, size_t n,
                               pclb200_corr* out, size_t* n_out, double* median_out);

PCLB200_API int pclb200_reject_surface_normal(pclb200_ctx* ctx, const pclb200_corr* in, size_t n,
                                              const void* src_normals, size_t n_src, size_t stride_sn,
                                              const void* tgt_normals, size_t n_tgt, size_t stride_tn, double threshold,
                                              pclb200_corr* out, size_t* n_out);

/* ---- transformation estimation: replaces TransformationEstimationSVD::estimateRigidTransformation
 * (impl/transformation_estimation_svd.hpp:50-181, Umeyama path, common/impl/eigen.hpp:675-734) and
 * TransformationEstimationPointToPlaneLLS (impl/transformation_estimation_point_to_plane_lls.hpp
 * :50-268).  corr == NULL pairs point i with point i.  Sums are accumulated in fp64 on the device;
 * scalar_is_double selects the Scalar the 4x4 is rounded to. */
PCLB200_API int pclb200_estimate_svd(pclb200_ctx* ctx, const void* src, size_t stride_s,
                                     const void* tgt, size_t stride_t, const pclb200_corr* corr,
                                     size_t n, int scalar_is_double, double T_out[16]);
/* TransformationEstimationSVD(use_umeyama = false): compute3DCentroid + demeanPointCloud + getTransformationFromCorrelation
 * (impl/transformation_estimation_svd.hpp:156-225; common/impl/centroid.hpp:55-85, 933-964): H = sum (p - cp)(q - cq)^T,
 * SVD, R = V U^T (last column of V negated when det(U) det(V) < 0), t = cq - R cp. */
PCLB200_API int pclb200_estimate_svd_correlation(pclb200_ctx* ctx, const void* src, size_t stride_s,
                                                 const void* tgt, size_t stride_t, const pclb200_corr* corr,
                                                 size_t n, int scalar_is_double, double T_out[16]);
PCLB200_API int pclb200_estimate_point_to_plane_lls(pclb200_ctx* ctx, const void* src,
                                                    size_t stride_s, const void* tgt,
                                                    const void* tgt_normals, size_t stride_t,
                                                    const pclb200_corr* corr, size_t n,
                                                    int scalar_is_double, double T_out[16]);

PCLB200_API int pclb200_estimate_symmetric_point_to_plane_lls(pclb200_ctx* ctx, const void* src,
                                                              const void* src_normals, size_t stride_s,
                                                              const void* tgt, const void* tgt_normals,
                                                              size_t stride_t, const pclb200_corr* corr, size_t n,
                                                              int enforce_same_direction_normals,
                                                              int scalar_is_double, double T_out[16]);

/* ---- ICP: replaces pcl::IterativeClosestPoint[WithNormals]::computeTransformation and the
 * pcl::Registration state around it (impl/icp.hpp:113-268; impl/registration.hpp:45-221;
 * default_convergence_criteria.h:64-326). */
#define PCLB200_EST_SVD 0            /* TransformationEstimationSVD (default of IterativeClosestPoint) */
#define PCLB200_EST_POINT_TO_PLANE_LLS 1 /* IterativeClosestPointWithNormals, non-symmetric */
#define PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS 2 /* setUseSymmetricObjective(true): needs source AND target normals
    (impl/transformation_estimation_symmetric_point_to_plane_lls.hpp:128-200; SURVEY.md §8f #2) */

/* DefaultConvergenceCriteria::ConvergenceState — default_convergence_criteria.h:75-83 */
#define PCLB200_CONV_NOT_CONVERGED 0
#define PCLB200_CONV_ITERATIONS 1
#define PCLB200_CONV_TRANSFORM 2
#define PCLB200_CONV_ABS_MSE 3
#define PCLB200_CONV_REL_MSE 4
#define PCLB200_CONV_NO_CORRESPONDENCES 5
#define PCLB200_CONV_FAILURE_AFTER_MAX_ITERATIONS 6

/* Temporal coherence of the per-iteration 1-NN search: a query whose previous match is PROVABLY still its unique nearest
 * neighbour (triangle inequality on a tracked lower bound) skips the tree walk.  Results are identical in every mode;
 * AUTO (default) switches the tracking on once an iteration moves the cloud by less than half the RMS residual. */
#define PCLB200_TRACK_AUTO 0
#define PCLB200_TRACK_ON 1
#define PCLB200_TRACK_OFF 2

typedef struct pclb200_icp_params {
  int32_t max_iterations;         /* registration.h:566, default 10 */
  int32_t use_reciprocal;         /* icp.h:265-280 setUseReciprocalCorrespondences */
  int32_t estimator;              /* PCLB200_EST_* */
  int32_t scalar_is_double;       /* the Scalar template argument */
  int32_t with_normals_transform; /* 0: IterativeClosestPoint::transformCloud (icp.hpp:49-111);
                                     1: ...WithNormals -> transformPointCloudWithNormals */
  int32_t is_dense;               /* input_->is_dense: 0 => skip non-finite source points */
  int32_t failure_after_max_iter; /* default_convergence_criteria.h:148-152 */
  int32_t max_iterations_similar_transforms; /* :310, default 0 */
  int32_t enforce_same_direction_normals;    /* symmetric estimator: n = n1 - n2 when n1.n2 < 0 (icp.h:402-418), default 1 */
  int32_t correspondence_kind;    /* PCLB200_CORR_*: which CorrespondenceEstimation runs inside the loop, default NEAREST */
  double max_correspondence_distance;     /* registration.h:117, default sqrt(DBL_MAX) */
  double transformation_epsilon;          /* registration.h:588, default 0 */
  double transformation_rotation_epsilon; /* default 0 = keep criteria default 0.99999 */
  double euclidean_fitness_epsilon;       /* registration.h:116, default -DBL_MAX */
  double mse_threshold_absolute;          /* default_convergence_criteria.h:307, default 1e-12 */
  int32_t correspondence_k;       /* k_ of the normal-shooting / back-projection estimators (setKSearch, default 10) */
  int32_t track_mode;             /* PCLB200_TRACK_*: temporal-coherence skip test of the 1-NN search (exact either way) */
  int32_t svd_no_umeyama;         /* TransformationEstimationSVD(use_umeyama = false): getTransformationFromCorrelation
                                     (transformation_estimation_svd.hpp:156-225) instead of Eigen::umeyama; default 0 */
  int32_t reserved2;
} pclb200_icp_params;

typedef struct pclb200_icp_stats {
  int32_t converged;          /* Registration::hasConverged */
  int32_t state;              /* PCLB200_CONV_* */
  int32_t iterations;         /* nr_iterations_ */
  int32_t reserved;
  int64_t n_correspondences;  /* accepted pairs in the last evaluated iteration (all ranks) */
  double mse;                 /* mean squared correspondence distance of that iteration */
  double final_transformation[16];  /* row-major, rounded to Scalar */
  double last_transformation[16];   /* getLastIncrementalTransformation */
  int64_t total_correspondences;    /* sum of accepted pairs over all iterations since set_source */
  int64_t total_skipped_walks;      /* queries (this rank) whose tree walk was skipped by the temporal-coherence test */
} pclb200_icp_stats;

PCLB200_API void pclb200_icp_default_params(pclb200_icp_params* p);

/* session API (the facade's IterativeClosestPoint holds one).
 * set_target  : Registration::setInputTarget + initCompute's tree hand-over (registration.hpp:61-101);
 *               tgt_normals (nullable) = first nx of the target normals, device copy kept for LLS.
 * set_source  : Registration::setInputSource + align()'s prologue (registration.hpp:172-216,
 *               icp.hpp:120-161): uploads the (indexed) source, applies `guess` (NULL = identity),
 *               resets the iteration state.  The convergence criteria's previous MSE is the one thing it
 *               keeps: as in the reference, whose DefaultConvergenceCriteria lives as long as the
 *               IterativeClosestPoint object (icp.h:155), the first iteration after set_source is compared
 *               with the last MSE the criteria recorded in this session (DBL_MAX in a new session).  So a
 *               tracking loop that aligns again from its last result can stop at iteration 1 on the MSE
 *               tests.  pclb200_icp_align and every problem of pclb200_icp_set_source_batch start from a
 *               new criteria object (DBL_MAX).
 * iterate     : runs up to max_steps iterations of the do-while at icp.hpp:164-241, stopping early
 *               when the convergence criteria fire; *stats is refreshed after every call.
 * get_cloud   : output = *input_ transformed by final_transformation_ (icp.hpp:265-267), written
 *               with stride_out; normals (if the source had them) rotated into out_normals. */
PCLB200_API int pclb200_icp_create(pclb200_ctx* ctx, const pclb200_icp_params* params,
                                   pclb200_icp** out);
PCLB200_API int pclb200_icp_destroy(pclb200_icp* icp);
PCLB200_API int pclb200_icp_set_params(pclb200_icp* icp, const pclb200_icp_params* params);
/* Registration::addCorrespondenceRejector / clearCorrespondenceRejectors (registration.h:373-416): the chain is
 * applied on the device, in order, to every iteration's correspondences (n == 0 clears it).  Every rejector sees the
 * survivors of the one before in source-position order (the order of the source index list), so exact-distance ties
 * break by position at every stage, also after a ONE_TO_ONE (whose stand-alone output is in index_match order); the
 * list get_correspondences returns is in that order too.  With a multi-GPU communicator every rank accepts what one
 * process accepts running the chain over the shards concatenated in rank order (see the communicator section below). */
PCLB200_API int pclb200_icp_set_rejectors(pclb200_icp* icp, const pclb200_rejector* list, int n);
PCLB200_API int pclb200_icp_set_target(pclb200_icp* icp, const pclb200_index* idx_tgt,
                                       const void* tgt_normals, size_t stride_n);
PCLB200_API int pclb200_icp_set_source(pclb200_icp* icp, const void* src, size_t n, size_t stride,
                                       const void* src_normals, size_t stride_n,
                                       const int32_t* src_indices, size_t n_idx,
                                       const double guess[16]);
PCLB200_API int pclb200_icp_iterate(pclb200_icp* icp, int max_steps, pclb200_icp_stats* stats);
PCLB200_API int pclb200_icp_get_cloud(pclb200_icp* icp, void* out_pts, size_t stride_out,
                                      void* out_normals, size_t stride_n);
/* correspondences of the last evaluated iteration (Registration::correspondences_, what icp.hpp:228-236 hands to
 * the visualisation callback): capacity = number of indexed source points, ordered like the source index list.  A
 * loop that stopped with NO_CORRESPONDENCES returns the list (fewer than 3 pairs) that stopped it. */
PCLB200_API int pclb200_icp_get_correspondences(pclb200_icp* icp, pclb200_corr* out, size_t* n_out);

/* one-call form: Registration::align(output, guess) (registration.hpp:172-221) of a new IterativeClosestPoint object,
 * so its criteria start with a previous MSE of DBL_MAX */
PCLB200_API int pclb200_icp_align(pclb200_ctx* ctx, const pclb200_icp_params* params,
                                  const void* src, size_t n, size_t stride, const void* src_normals,
                                  size_t stride_sn, const int32_t* src_indices, size_t n_idx,
                                  const pclb200_index* idx_tgt, const void* tgt_normals,
                                  size_t stride_tn, const double guess[16], void* out_cloud,
                                  size_t stride_out, pclb200_icp_stats* stats);

/* Registration::getFitnessScore(max_range, use_indices) — registration.hpp:134-168.
 * Returns DBL_MAX in *score when no point is within max_range. */
PCLB200_API int pclb200_fitness_score(pclb200_ctx* ctx, const pclb200_index* idx_tgt,
                                      const void* src, size_t n, size_t stride,
                                      const int32_t* src_indices, size_t n_idx, int is_dense,
                                      const double T[16], int scalar_is_double, double max_range,
                                      double* score);

/* GeneralizedIterativeClosestPoint::computeCovariances — registration/include/pcl/registration/impl/gicp.hpp:69-147
 * (SURVEY.md §8f #2): for every point of `pts` (the cloud idx was built over, so neighbours and queries are the same
 * cloud) the covariance of its k nearest neighbours relative to the point, mean removed, singular values replaced by
 * (1, 1, gicp_epsilon) (:136-147).  out_cov: n x 9 doubles, row-major 3x3 (host or device); zeros for non-finite points.
 * k = k_correspondences_ (default 20), gicp_epsilon default 0.001 (gicp.h:127-129). */
PCLB200_API int pclb200_gicp_covariances(pclb200_ctx* ctx, const pclb200_index* idx, const void* pts, size_t n,
                                         size_t stride, int k, double gicp_epsilon, double* out_cov);

/* TransformationValidationEuclidean::validateTransformation — registration/include/pcl/registration/impl/
 * transformation_validation_euclidean.hpp:50-109: the source transformed by T (products and sums in Scalar, left to right,
 * cast to float: :62-75), 1-NN into the target, mean of the squared distances that are <= max_range (the reference compares
 * the squared distance with max_range_ as given); DBL_MAX when none is. */
PCLB200_API int pclb200_validate_transformation(pclb200_ctx* ctx, const pclb200_index* idx_tgt, const void* src, size_t n,
                                                size_t stride, const double T[16], int scalar_is_double,
                                                double max_range, double* score);

/* SampleConsensusPrerejective::getFitness — impl/sample_consensus_prerejective.hpp:308-347: the source transformed by T
 * (pcl::transformPointCloud, float), 1-NN into the target, inliers = points whose squared distance is STRICTLY below
 * inlier_threshold^2 (float).  out (capacity n): one pclb200_corr per inlier {source index, nearest target index, d2},
 * ascending source index — the caller sums `distance` in that order (float) to reproduce the reference's fitness. */
PCLB200_API int pclb200_inliers(pclb200_ctx* ctx, const pclb200_index* idx_tgt, const void* src, size_t n, size_t stride,
                                const double T[16], float inlier_threshold, pclb200_corr* out, size_t* n_out);

/* ---- normals: replaces NormalEstimation[OMP]::computeFeature with setKSearch(k)
 * (features/include/pcl/features/impl/normal_3d.hpp:47-96; normal_3d.h:169-188,308-322;
 * common/impl/centroid.hpp:578-652; features/impl/feature.hpp:65-92; common/impl/eigen.hpp:68-326).
 * idx is the search surface; pts/indices are the query points.  out: n (or n_idx) records of
 * 4 floats (nx, ny, nz, curvature); NaN rows where the reference writes NaN; *is_dense_out = 0
 * if any. */
PCLB200_API int pclb200_normals_knn(pclb200_ctx* ctx, const pclb200_index* idx, const void* pts,
                                    size_t n, size_t stride, const int32_t* indices, size_t n_idx,
                                    int is_dense, int k, const float viewpoint[3], float* out,
                                    int* is_dense_out);
/* setRadiusSearch(radius) variant: the neighbourhood is radiusSearch(point, radius) with max_nn = 0
 * (features/include/pcl/features/impl/feature.hpp:149-166), i.e. every indexed point with d2 < float(radius^2) in
 * ascending (d2, index) order; everything after the search is the k-NN path's arithmetic. */
PCLB200_API int pclb200_normals_radius(pclb200_ctx* ctx, const pclb200_index* idx, const void* pts,
                                       size_t n, size_t stride, const int32_t* indices, size_t n_idx,
                                       int is_dense, double radius, const float viewpoint[3], float* out,
                                       int* is_dense_out);

/* ---- Euclidean clustering: replaces the flood fill of pcl::extractEuclideanClusters /
 * EuclideanClusterExtraction<PointT>::extract (segmentation/include/pcl/segmentation/impl/extract_clusters.hpp:45-257),
 * one radiusSearch per point on one thread, by the connected components of the graph "d2 < float(tolerance)^2" over
 * the points of idx (the cloud, or cloud + indices, the tree would be built from) — the same sets, because the fp32
 * squared distance is symmetric and the radius test is the searcher's own (SURVEY.md §8f #4).
 * out_labels: one entry per point of the cloud idx was built from (n_labels must equal that count; host or device):
 * the SMALLEST ORIGINAL INDEX of the point's component, -1 for points idx does not hold (non-finite / outside the subset;
 * the reference never clusters those either, since the tree cannot return them).  Grouping by label, the size window
 * [min, max] and the final ordering by size (extract_clusters.hpp:249) stay with the caller: they touch 4 bytes/point. */
PCLB200_API int pclb200_cluster_labels(pclb200_ctx* ctx, const pclb200_index* idx, double tolerance,
                                       int32_t* out_labels, size_t n_labels);

/* ---- VoxelGrid: replaces pcl::VoxelGrid<PointT>::applyFilter (no filter field)
 * (filters/include/pcl/filters/impl/voxel_grid.hpp:596-814).  out_xyz1: capacity n records
 * {x,y,z,1}; ordered by voxel linear index.  PCLB200_ERR_LEAF_TOO_SMALL mirrors :620-629 (the
 * caller then copies the input unfiltered, as the reference does). */
PCLB200_API int pclb200_voxelgrid(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride,
                                  const int32_t* indices, size_t n_idx, int is_dense,
                                  const float leaf[3], unsigned min_points_per_voxel,
                                  float* out_xyz1, size_t* n_out);

/* One SPATIAL TILE of a VoxelGrid over a larger cloud (multi-GPU front-end, SURVEY.md §8e): grid_bounds = {min x,y,z,
 * max x,y,z} of the WHOLE cloud fix the grid (min_b, div_b: voxel_grid.hpp:632-644), so a tile cut along voxel boundaries
 * yields exactly the centroids a single VoxelGrid over the whole cloud yields for those voxels; the tiles' outputs,
 * concatenated, are the whole output as a set.  The INT32 guard (:620-629) applies to the whole grid. */
PCLB200_API int pclb200_voxelgrid_tile(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride,
                                       const float grid_bounds[6], const float leaf[3], unsigned min_points_per_voxel,
                                       float* out_xyz1, size_t* n_out);

/* The same filter for records that carry a normal and a curvature (pcl::PointNormal, pcl::Normal), with the
 * reference's default downsample_all_data_ = true (voxel_grid.hpp:796-806, CentroidPoint): per voxel the normals are
 * summed as 4-vectors and normalised (accumulators.hpp:86-116), the curvature is averaged (:118-133).
 * normals: pointer to the first normal_x (PointNormal: base + 16); the 5 floats {nx, ny, nz, n4, curvature} are read at
 * stride_n.  out_normal_curv: capacity n records of 8 floats {nx, ny, nz, n4, curvature, 0, 0, 0} — bytes 16..47 of a
 * pcl::PointNormal. */
PCLB200_API int pclb200_voxelgrid_normals(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const void* normals,
                                          size_t stride_n, const int32_t* indices, size_t n_idx, int is_dense,
                                          const float leaf[3], unsigned min_points_per_voxel, float* out_xyz1,
                                          float* out_normal_curv, size_t* n_out);

/* ---- multi-GPU: one process per GPU, in one of two layouts.
 * Sharded source (pclb200_icp_set_target): every rank holds a replica of the target index and a shard of the source;
 *   pclb200_icp_iterate all-reduces the 40 fp64 accumulators of each iteration across ranks, so every rank computes the
 *   identical transform.
 * Sharded target (include/pclb200_sharded.h: tiles indexed with caller ids, a collective set-target of the session, a
 *   collective fitness score): every rank holds one tile of the map and the whole source; each iteration exchanges one
 *   8-byte key per query and the winning target records, and every rank computes the single-process result on the whole
 *   map.  The largest map is then the sum of the tiles, not one GPU's memory.
 * unique_id: 128 bytes from pclb200_comm_unique_id on rank 0, broadcast by the caller. */
PCLB200_API int pclb200_comm_unique_id(void* out_128_bytes);
PCLB200_API int pclb200_comm_init(pclb200_ctx* ctx, int rank, int nranks, const void* unique_id);
/* The per-iteration exchange: FUSED (default) = the last block of the iteration kernel stores its 40 sums into every
 * peer's memory over NVLink and folds all ranks' sums in rank order (no collective launch, bitwise identical on all
 * ranks); NCCL = a separate ncclAllReduce after the kernel (kept for comparison and as the fallback when peer mappings
 * cannot be made). */
#define PCLB200_REDUCE_FUSED 0
#define PCLB200_REDUCE_NCCL 1
PCLB200_API int pclb200_comm_set_mode(pclb200_ctx* ctx, int mode);
/* NCCL-free bootstrap of the FUSED exchange, for launchers that can all-gather 64 bytes per rank themselves (MPI, gloo,
 * a shared file) and for ranks that share one GPU: comm_export returns this rank's 64-byte cudaIpcMemHandle_t;
 * comm_import takes the nranks handles in rank order.
 * Rejector chains (pclb200_icp_set_rejectors) on a sharded source: distance and surface-normal run per rank; median,
 * trimmed and one-to-one decide over all ranks' correspondences through small exchanges (DESIGN.md §5), so every rank
 * accepts exactly the correspondences one process accepts on the concatenation of the shards in rank order.  A query's
 * position is the queries of the lower ranks plus its position in its rank's source list: distance ties break in
 * (rank, position) order, which is the input order when rank r holds the r-th contiguous range.  All ranks must set the
 * same chain and run the same iterations (the exchanges are collective); more than 2^32 queries in all is
 * PCLB200_ERR_INVALID.  Reciprocal correspondences stay PCLB200_ERR_INVALID with a communicator. */
PCLB200_API int pclb200_comm_export(pclb200_ctx* ctx, void* out_handle_64_bytes);
PCLB200_API int pclb200_comm_import(pclb200_ctx* ctx, int rank, int nranks, const void* handles);

#ifdef __cplusplus
}
#endif
#endif /* PCLB200_H_ */
