/* pclb200_sharded.h — C-ABI of libpclb200.so for a target map sharded across the ranks of a multi-GPU communicator
 * (the second multi-GPU layout of include/pclb200.h): every rank holds one tile of the map, indexed with the caller's
 * ids, and the whole source; the registration is the single-process registration on the whole map, bit for bit.
 *
 * The entry points follow every convention of include/pclb200.h (status codes, host-or-device arrays, strides, squared
 * fp32 distances, smaller-id tie rule, row-major transforms).  They live in their own header because they have no
 * counterpart in the reference's API and the PCL facade (pcl_b200/pcl_compat/) does not reach them: pclb200.h stays the
 * contract of the facade, this header is the multi-GPU extension on top of it. */
#ifndef PCLB200_SHARDED_H_
#define PCLB200_SHARDED_H_

#include "pclb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The same index with point i labelled ids[i] instead of i: every search returns the caller's ids, and exact ties are
 * broken by the smaller id.  Built over one tile of a larger map whose point ids[i] is pts[i], it is byte for byte the
 * index pclb200_index_build makes of that map with subset = ids.  Non-finite points are dropped as by pclb200_index_build.  ids (host or
 * device, n entries) must be distinct and lie in [0, 2^31 - 2], else PCLB200_ERR_INVALID.  What maps ids back to
 * records of the cloud an index was built from refuses a labelled index (PCLB200_ERR_INVALID): the normal-based
 * correspondence estimators, normal estimation with k > 32 or a radius, GICP covariances, pclb200_cluster_labels.
 * The normals of a sharded map come from pclb200_normals_knn_sharded / pclb200_normals_radius_sharded, and the clusters
 * of a sharded map come from pclb200_cluster_labels_sharded, its k-NN lists and outlier filters from pclb200_knn_sharded,
 * pclb200_knn_stats_sharded, pclb200_statistical_outlier_sharded and pclb200_radius_outlier_sharded, its VoxelGrid from
 * pclb200_voxelgrid_sharded, its nearest and reciprocal correspondences, validation and inliers from
 * pclb200_correspondences_sharded, pclb200_correspondences_normals_sharded, pclb200_validate_transformation_sharded
 * and pclb200_inliers_sharded, its radius neighbourhoods from pclb200_radius_sharded and pclb200_radius_into_sharded,
 * and its GICP covariances from pclb200_gicp_covariances_sharded. */
PCLB200_API int pclb200_index_build_ids(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride,
                                        const int32_t* ids, pclb200_index** out);

/* Target sharded across the ranks of the context's communicator (collective: every rank calls it with its tile).  idx_tile
 * is this rank's tile of the map, built with pclb200_index_build_ids (the union of the tiles' ids is the map; an id held
 * by two ranks must name the same point and normal, the lowest rank's record is used); tgt_normals (nullable) has one
 * record per point of the tile.  Every rank then passes the SAME whole source to set_source (array, indices, is_dense,
 * guess) and runs the same iterate calls: each rank searches its tile, the per-query minimum of (d2, id) over the ranks
 * is the whole map's nearest neighbour, and every rank solves on those pairs.  get_cloud, get_correspondences and the
 * stats equal one process's on the whole map, bit for bit, on every rank (total_skipped_walks stays per rank).
 * The first iterate after set_source checks that every rank staged the same number of queries.  Nearest-neighbour
 * correspondences only: reciprocal correspondences, the normal-shooting / back-projection estimators, rejector chains,
 * and a context without an active communicator are PCLB200_ERR_INVALID. */
PCLB200_API int pclb200_icp_set_target_sharded(pclb200_icp* icp, const pclb200_index* idx_tile,
                                               const void* tgt_normals, size_t stride_n);

/* The same score over a target sharded across the ranks of the context's communicator (collective: every rank passes its
 * tile, built with pclb200_index_build_ids, and the same source).  Every rank returns the same value; the count of points
 * within max_range is one process's count on the whole map, the score agrees with one process's to fp64 round-off (the
 * sum runs in another order).  Arguments one rank refuses (a tile without ids, a source count other ranks do not pass)
 * are PCLB200_ERR_INVALID on every rank. */
PCLB200_API int pclb200_fitness_score_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile,
                                              const void* src, size_t n, size_t stride,
                                              const int32_t* src_indices, size_t n_idx, int is_dense,
                                              const double T[16], int scalar_is_double, double max_range,
                                              double* score);

/* The stand-alone consumers of the 1-NN search over a target sharded across the ranks of the context's communicator, so
 * that any registration loop of correspondence estimation, pclb200_reject chains and pclb200_estimate_* runs against a map
 * larger than one GPU.  Collective, in the layout of pclb200_icp_set_target_sharded and pclb200_fitness_score_sharded:
 * every rank passes its tile (built with pclb200_index_build_ids; the map is the union of the ids, an id held by two ranks
 * names the same point and normal) and the SAME whole source (array, src_indices, is_dense, transform), and every rank
 * returns the same result.  "One index of the whole map" below is pclb200_index_build over the map with subset = the
 * union of the ids; index_match holds map ids.  Arrays may be host or device memory.
 *
 * pclb200_correspondences_sharded: the list pclb200_correspondences returns on one index of the whole map, byte for
 * byte.  idx_src != NULL selects the reciprocal variant; it is an ordinary index (pclb200_index_build) each rank builds
 * over the same source.  out_xyz1 (nullable) receives one {x, y, z, 1} row per output correspondence, the matched map
 * point; out_normals (nullable, needs tgt_normals: one record per record of the tile, stride stride_tn) receives its
 * {nx, ny, nz, 0}.  Rows have a stride of 16 bytes (device rows 16-byte aligned), so they pass straight to
 * pclb200_estimate_* with corr = NULL.
 * pclb200_validate_transformation_sharded: pclb200_validate_transformation's score on one index of the whole map, as
 * pclb200_fitness_score_sharded states it: the same value on every rank, the count exact, the score within fp64
 * round-off of one process's (the sum runs in another order).
 * pclb200_correspondences_normals_sharded: the list pclb200_correspondences_normals returns on one index of the whole
 * map, byte for byte, with the same record outputs; k is clamped to the whole map's number of distinct finite ids, as
 * pclb200_knn_sharded clamps k_eff.  tgt_normals (back projection, out_normals) has one record per record of the tile.
 * Each rank's k nearest of its tile (as keys) are merged per source point into the whole map's row: every member of the
 * whole map's k nearest that lies in a tile is among that tile's k nearest.  Every rank scores the candidates its tile
 * holds; one u64 minimum of the n_q x k_eff score table gives every rank every score.  Memory per rank at the peak: its
 * published rows (n_q k_eff 8 B), the other ranks' rows where they must be resident to merge (none on the peer path,
 * which reads them in place; (R - 1) n_q k_eff 8 B under NCCL, an all-gather), the merged rows and the score table
 * (2 n_q k_eff 8 B).
 * pclb200_inliers_sharded: the inlier list of pclb200_inliers (float transform, strict d2 < threshold^2) on one index of
 * the whole map, byte for byte; out_xyz1 as above.
 *
 * Each rank searches its tile; per source point the smallest key (d2 bits << 32 | id) over the ranks is the whole map's
 * nearest neighbour (one u64-minimum exchange of n_q keys, 2 n_q for the reciprocal variant: the second key carries the
 * verdict of the reverse search of whichever rank holds the winning point).  The record rows take a second exchange of
 * n_q keys and n_q (n_q more with normals) 16-byte records, the one the sharded ICP session runs every iteration; both
 * exchanges of a call draw one scratch table of the larger size, and under NCCL each reduces only its own words.
 * PCLB200_ERR_INVALID on every rank, before any exchange, without an active communicator, and when any rank passes a
 * tile built without ids, a NULL argument (a NULL tile included), k < 0, an unknown kind, missing source normals, back
 * projection without target normals, a labelled idx_src, out_normals without tgt_normals, misaligned device rows, a query
 * count other ranks do not pass, or a different choice of variant, kind, k and rows. */
PCLB200_API int pclb200_correspondences_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile,
                                                const pclb200_index* idx_src /*nullable*/, const void* src, size_t n,
                                                size_t stride, const int32_t* src_indices, size_t n_idx, int is_dense,
                                                double max_dist, const void* tgt_normals /*nullable*/, size_t stride_tn,
                                                pclb200_corr* out, float* out_xyz1 /*nullable*/,
                                                float* out_normals /*nullable*/, size_t* n_out);
PCLB200_API int pclb200_correspondences_normals_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, int kind,
                                                        const void* src, size_t n, size_t stride, const void* src_normals,
                                                        size_t stride_sn, const void* tgt_normals /*nullable*/,
                                                        size_t stride_tn, const int32_t* src_indices, size_t n_idx, int k,
                                                        double max_dist, pclb200_corr* out, float* out_xyz1 /*nullable*/,
                                                        float* out_normals /*nullable*/, size_t* n_out);
PCLB200_API int pclb200_validate_transformation_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* src,
                                                        size_t n, size_t stride, const double T[16], int scalar_is_double,
                                                        double max_range, double* score);
PCLB200_API int pclb200_inliers_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* src, size_t n,
                                        size_t stride, const double T[16], float inlier_threshold, pclb200_corr* out,
                                        float* out_xyz1 /*nullable*/, size_t* n_out);

/* Collective over the context's communicator: every rank passes its tile (built with pclb200_index_build_ids) and its
 * OWN queries (any points; typically the tile's records).  out[i] is, bit for bit, what pclb200_normals_knn /
 * pclb200_normals_radius returns for query i against one index of the whole map (the union of the tiles' ids),
 * including NaN rows; *is_dense_out covers this rank's queries.  Arrays, strides, indices and out follow
 * pclb200_normals_knn; a rank with no queries still takes part.  Each rank fetches, from the other ranks' tiles, the
 * points within its queries' k-th nearest distance in its own tile (or the radius) and indexes its tile plus those points:
 * both are resident at the peak.  An id held by two ranks must name the same point.  PCLB200_ERR_INVALID on every rank,
 * before any exchange, without an active communicator, for a tile built without ids, and for k <= 0 / radius <= 0. */
PCLB200_API int pclb200_normals_knn_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* pts, size_t n,
                                            size_t stride, const int32_t* indices, size_t n_idx, int is_dense, int k,
                                            const float viewpoint[3], float* out, int* is_dense_out);
PCLB200_API int pclb200_normals_radius_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* pts,
                                               size_t n, size_t stride, const int32_t* indices, size_t n_idx,
                                               int is_dense, double radius, const float viewpoint[3], float* out,
                                               int* is_dense_out);

/* k-NN queries, k-NN statistics and the two outlier filters of a map sharded across the ranks of the context's
 * communicator.  Collective: every rank passes its tile (built with pclb200_index_build_ids; the whole map is the union
 * of the tiles' ids) and its OWN queries (any points; typically the tile's records, through an optional indices subset).
 * Arrays may be host or device memory; a rank with no query still takes part.  Each rank fetches, from the other ranks'
 * tiles, the points within its queries' k-th nearest distance in its own tile and indexes its tile plus those points:
 * both are resident at the peak.  An id held by two ranks must name the same point.  PCLB200_ERR_INVALID on every rank,
 * before any exchange, without an active communicator, for a tile built without ids, and for k <= 0 / mean_k <= 0 /
 * min_pts < 0 / radius <= 0.
 *
 * pclb200_knn_sharded: row i (k entries of out_idx / out_d2) is, byte for byte, what pclb200_knn returns for query i
 * against one index of the whole map (pclb200_index_build over the map with subset = the union of the ids): the ids, the
 * d2, the (d2, id) order, the (-1, +inf) padding and the rows of non-finite queries.  *k_eff (nullable) is the whole
 * map's clamp min(k, number of distinct finite ids), the same on every rank.
 * pclb200_knn_stats_sharded: out_mean / out_kth (either nullable) are, byte for byte, pclb200_knn_stats on one index of
 * the whole map. */
PCLB200_API int pclb200_knn_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* queries, size_t nq,
                                    size_t stride, int k, int32_t* out_idx, float* out_d2, int* k_eff);
PCLB200_API int pclb200_knn_stats_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* pts, size_t n,
                                          size_t stride, const int32_t* indices, size_t n_idx, int k, float* out_mean,
                                          float* out_kth);

/* StatisticalOutlierRemoval (setMeanK(mean_k), setStddevMulThresh(std_mul), setNegative(negative)) over the concatenation
 * of every rank's queries in rank order.  keep[i] (1 = kept) covers this rank's queries; stats (nullable) receives the
 * number of finite queries, the mean and the threshold, the same on every rank.  The per-query mean distances are
 * pclb200_knn_stats's with k = mean_k + 1 on the whole map, bit for bit.  The threshold is not bit for bit: the reference
 * sums the means one after the other in record order, and here every rank sums its own in a fixed order, the ranks'
 * partial sums travel exactly and every rank adds them up in rank order.  So every rank holds the same threshold, within
 * fp64 round-off of one process's, and keep differs from one process's only for a query whose mean lies within that
 * round-off of the threshold.  The statistics run over the queries as passed: a point two ranks hold under one id counts
 * once only if just one of them passes it as a query. */
PCLB200_API int pclb200_statistical_outlier_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* pts,
                                                    size_t n, size_t stride, const int32_t* indices, size_t n_idx,
                                                    int mean_k, double std_mul, int negative, uint8_t* keep,
                                                    double stats[3]);

/* RadiusOutlierRemoval (setRadiusSearch(radius), setMinNeighborsInRadius(min_pts), setNegative(negative)) of this rank's
 * queries on the whole map: keep[i] (1 = kept) is, byte for byte, the reference's rule on pclb200_knn_stats with
 * k = min_pts + 1.  The dense rule (the k-NN comparison) applies when every rank passes is_dense, else the radius rule
 * (strict d2 < radius^2, non-finite queries removed) applies on every rank. */
PCLB200_API int pclb200_radius_outlier_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* pts,
                                               size_t n, size_t stride, const int32_t* indices, size_t n_idx,
                                               int is_dense, double radius, int min_pts, int negative, uint8_t* keep);

/* Radius search and GICP covariances of a map sharded across the ranks of the context's communicator.  Collective: every
 * rank passes its tile (built with pclb200_index_build_ids; the map is the union of the ids, an id held by two ranks names
 * the same point and counts once).  "One index of the whole map" is pclb200_index_build over the map with subset = the
 * union of the ids in ascending order.  Arrays may be host or device memory, as for the single-index calls.
 *
 * pclb200_radius_sharded / pclb200_radius_into_sharded: every rank passes its OWN queries (any points; a rank may pass
 * none), and its own radius and max_nn (they serve only its queries; the ranks need not agree).  Each query's row of
 * out_offsets / out_idx / out_d2 is, byte for byte, what pclb200_radius / pclb200_radius_into return for it on one index
 * of the whole map: the ids, the d2, the (d2, id) order, strict d2 < float(radius * radius), max_nn keeping the nearest,
 * empty rows for non-finite queries.  A radius of 0 or NaN gives empty lists, a radius whose square overflows the whole
 * map.  A rank with nq == 0 takes part in every exchange and gets out_offsets[0] = 0 (and, from pclb200_radius_sharded,
 * *out_idx = *out_d2 = NULL).  pclb200_radius_sharded takes host out_offsets and allocates the lists (pclb200_free).
 * pclb200_radius_into_sharded keeps pclb200_radius_into's rule on each rank: when *total > capacity only out_offsets and
 * *total are written, else the lists too.  Once every rank has counted, one u64 minimum sets *all_fit (nullable; the
 * exchange runs either way) to the same value on every rank: 1 exactly when every rank's lists fit.  So every rank runs the
 * same loop, while (!all_fit) { grow to *total; call again }, and a rank whose lists already fit may pass the same
 * buffers again and gets the same bytes.  Each call rebuilds the halo.  A rank's lists share pclb200_radius's limit of
 * 2^31 neighbours (max_nn <= 32 materialises only the kept ones).
 * Each rank fetches, from the other ranks' tiles, every point within the radius of its queries' box, and indexes its tile
 * plus those points: both are resident at the peak, and on a random partition the halo is nearly the whole map.
 *
 * pclb200_gicp_covariances_sharded: pts, n, stride are the records the tile was built from (n = its record count).
 * Row i of out_cov (9 doubles) is, byte for byte, row ids[i] of pclb200_gicp_covariances on one index of the whole map
 * called with the whole map's array: zero rows for non-finite records, k clamped to the whole map's distinct finite ids,
 * the division by k.  Each rank fetches the points within its records' k-th nearest distance in its tile, as
 * pclb200_knn_sharded does.
 *
 * PCLB200_ERR_INVALID on every rank, before any halo moves, when any rank has no active communicator, a NULL or
 * unlabelled tile, a NULL argument where one is not allowed, device out_offsets given to pclb200_radius_sharded,
 * capacity > 0 with NULL output buffers, k < 1, or (covariances) n other than its tile's record count.  Each rank's
 * verdict on its own arguments travels in one u64 minimum. */
PCLB200_API int pclb200_radius_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* queries, size_t nq,
                                       size_t stride, double radius, unsigned max_nn, int sorted,
                                       int64_t* out_offsets, int32_t** out_idx, float** out_d2);
PCLB200_API int pclb200_radius_into_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* queries,
                                            size_t nq, size_t stride, double radius, unsigned max_nn,
                                            int64_t* out_offsets, int32_t* out_idx, float* out_d2, size_t capacity,
                                            size_t* total, int* all_fit /*nullable*/);
PCLB200_API int pclb200_gicp_covariances_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* pts,
                                                 size_t n, size_t stride, int k, double gicp_epsilon, double* out_cov);

/* Euclidean clustering of a map sharded across the ranks of the context's communicator (collective: every rank passes its
 * tile, built with pclb200_index_build_ids; the whole map is the union of the tiles' ids).  n_labels is the number of
 * records the tile was built from.  out_labels[i] is, byte for byte, what pclb200_cluster_labels returns at ids[i] for one
 * index of the whole map: the smallest id of the record's component of the d2 < tolerance^2 graph (tolerance narrowed to
 * float as there), -1 for a non-finite record.  out_sizes (nullable) receives the number of distinct ids in that
 * component on the whole map (what EuclideanClusterExtraction's min / max cluster size compare), 0 for a non-finite
 * record.  Both may be host or device memory.  An id held by two ranks must name the same point; it gets the same label
 * on both and counts once.  Each rank fetches the other tiles' points within the tolerance of its tile's box, clusters
 * its tile plus those points, and one exchange of labels along that halo stitches components across any number of tiles;
 * tile and halo are resident at the peak.  PCLB200_ERR_INVALID on every rank, before any exchange, without an active
 * communicator, for a tile built without ids, for a negative tolerance and for n_labels other than the tile's records. */
PCLB200_API int pclb200_cluster_labels_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, double tolerance,
                                               int32_t* out_labels, int64_t* out_sizes, size_t n_labels);

/* VoxelGrid of a map sharded across the ranks of the context's communicator.  Collective: every rank passes its own
 * records pts[0..n) and their ids (the map is the union of the ids; on one rank they are distinct and lie in
 * [0, 2^31 - 2]; an id held by two ranks must name the same record, and it counts once).  The output is pclb200_voxelgrid
 * (pclb200_voxelgrid_normals when normals is given) of the whole map with indices = the union of the ids in ascending
 * order, byte for byte, split across the ranks:
 * - each voxel of that output is returned by exactly one rank;
 * - each rank returns its voxels ordered by voxel linear index;
 * - out_voxel[i] is the linear index of row i (ijk . (1, div_b0, div_b0 div_b1) on the whole map's grid).
 * Stable-sorting the concatenation of every rank's rows by out_voxel gives the whole output.  Every voxel a rank returns
 * holds at least one of its own finite records, so *n_out <= n and a capacity of n rows always suffices.
 * Arrays may be host or device memory; normals and out_normal_curv (both or neither) use the layouts of
 * pclb200_voxelgrid_normals.  A rank with no finite record still takes part; when no rank has one, *n_out = 0 everywhere.
 * Each rank receives, from the other ranks, every record whose voxel lies in the voxel range of its own records' box, and
 * sorts its records plus those: both are resident at the peak (on a random partition that is nearly the whole map).
 * PCLB200_ERR_INVALID on every rank, before any record moves, without an active communicator, for a NULL argument, a leaf
 * <= 0 or non-finite, invalid ids on any rank, ranks that disagree on leaf or min_points_per_voxel, and normals given on
 * some ranks and not on others.  PCLB200_ERR_LEAF_TOO_SMALL on every rank exactly when the whole map's grid trips
 * pclb200_voxelgrid's integer guard. */
PCLB200_API int pclb200_voxelgrid_sharded(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride,
                                          const int32_t* ids, const void* normals /*nullable*/, size_t stride_n,
                                          const float leaf[3], unsigned min_points_per_voxel,
                                          float* out_xyz1, float* out_normal_curv /*nullable*/,
                                          uint32_t* out_voxel, size_t* n_out);

/* Collective over the context's communicator: every rank's send[0..n) concatenated in rank order, the same on every
 * rank.  *n_total is the total; recv (host or device, nullable) receives it when capacity >= *n_total, else nothing is
 * written there (every rank sees the same total, so all of them can call again with room).  It lets every rank learn,
 * for instance, the (size, label) pairs of every cluster pclb200_cluster_labels_sharded found on the other ranks.
 * PCLB200_ERR_INVALID on every rank without an active communicator. */
PCLB200_API int pclb200_comm_allgather_u64(pclb200_ctx* ctx, const uint64_t* send, size_t n, uint64_t* recv,
                                           size_t capacity, size_t* n_total);

#ifdef __cplusplus
}
#endif
#endif /* PCLB200_SHARDED_H_ */
