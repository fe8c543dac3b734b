/* pclb200_batch.h — C-ABI of libpclb200.so for a batch of ICP problems in one session: a queue of scans against one
 * prior map, one scan from many initial guesses (one target for all problems), or many independent scan pairs such as
 * the consecutive scans of an odometry sequence or the edges of a pose graph (pclb200_icp_set_target_batch: one target
 * per problem).  Every stage of an iteration is one launch for the whole batch, however many problems and targets it
 * holds, and the loop state of every problem comes back in one read.
 *
 * The entry points follow every convention of include/pclb200.h (status codes, host-or-device arrays, strides, squared
 * fp32 distances, row-major transforms).  They live in their own header because they have no counterpart in the
 * reference's API and the PCL facade (pcl_b200/pcl_compat/) does not reach them.  The target is the session's
 * (pclb200_icp_set_target), or one per problem (pclb200_icp_set_target_batch).
 *
 * Problem p is bit for bit what a fresh session with the same parameters, target and target normals would do after
 * pclb200_icp_set_source(its records, its guess) and the same sequence of max_steps: every pclb200_icp_stats field
 * (total_skipped_walks included), every iteration's correspondences and the aligned records.  Every problem starts
 * with a new criteria state, previous MSE DBL_MAX: unlike pclb200_icp_set_source, set_source_batch carries nothing
 * over from the session's earlier aligns.
 *
 * A batch takes nearest-neighbour correspondences; SVD (Umeyama or not), point-to-plane LLS or the symmetric objective;
 * float or double Scalar; with_normals_transform; is_dense = 0; every convergence criterion; tracking OFF / ON / AUTO
 * (AUTO decides per problem); host or device source arrays.  PCLB200_ERR_INVALID, with the session left as it was, for a
 * rejector chain, use_reciprocal, a correspondence_kind other than NEAREST, an active communicator or a sharded target,
 * and the symmetric objective without source normals.
 *
 * The clouds of such a batch can themselves be down-sampled as one batch (pclb200_voxelgrid_batch), the targets built as
 * one batch (pclb200_index_build_batch), their normals for point-to-plane or the symmetric objective estimated as one
 * batch (pclb200_normals_knn_batch), and the aligned pairs scored as one batch (pclb200_icp_fitness_score_batch,
 * pclb200_fitness_score_batch, pclb200_validate_transformation_batch). */
#ifndef PCLB200_BATCH_H_
#define PCLB200_BATCH_H_

#include "pclb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Problem p of the next set_source_batch is registered against targets[p] (and tgt_normals[p]) instead of the session's
 * single target: problem p is bit for bit a fresh session after pclb200_icp_set_target(targets[p], tgt_normals[p],
 * stride_n) + pclb200_icp_set_source(its records, its guess) and the same max_steps.  A handle may repeat.
 *
 * targets: host, n_targets handles, kept alive by the caller as with pclb200_icp_set_target.  tgt_normals (host, nullable;
 * entries nullable): one array per problem, one normal per point of the cloud its index was built from, host or device,
 * all with stride stride_n.  set_target_batch drops whatever source the session held, so iterate_batch refuses until
 * set_source_batch runs again (the query order depends on the targets' frames); set_source_batch then refuses unless
 * n_problems == n_targets.  pclb200_icp_set_source refuses while the session holds a target batch;
 * pclb200_icp_set_target puts the session back to one target (and drops a source staged for the batch).
 * PCLB200_ERR_INVALID, with the session left as it was, for n_targets outside 1 to 65536, a NULL array or NULL handle,
 * an index on another device than the session, point-to-plane or the symmetric objective when some problem has no
 * target normals, and the refusals in the header comment. */
PCLB200_API int pclb200_icp_set_target_batch(pclb200_icp* icp, const pclb200_index* const* targets,
                                             const void* const* tgt_normals /* nullable; entries nullable */,
                                             size_t stride_n, int32_t n_targets);

/* B = n_problems problems, problem p being the records [offsets[p], offsets[p+1]) of src (offsets: host, B + 1 entries,
 * offsets[0] = 0, strictly increasing, offsets[B] = n); src_normals (nullable) as in pclb200_icp_set_source.  guesses
 * (host, nullable = identity for every problem): B row-major 4x4 matrices.  Replaces whatever source the session held;
 * pclb200_icp_set_source puts the session back into single-problem mode.  PCLB200_ERR_INVALID for B < 1 or B > 65536,
 * bad offsets (an empty problem included), n >= 2^31 - 1, and the refusals in the header comment.
 * pclb200_icp_get_cloud on a batch session writes all n records, each moved by its own problem's final transform. */
PCLB200_API int pclb200_icp_set_source_batch(pclb200_icp* icp, const void* src, size_t n, size_t stride,
                                             const void* src_normals, size_t stride_n, const int64_t* offsets,
                                             int32_t n_problems, const double* guesses);

/* Advances every problem still NOT_CONVERGED by up to max_steps iterations (pclb200_icp_iterate of each problem's own
 * session).  stats (host, nullable): B entries.  pclb200_icp_iterate and pclb200_icp_get_correspondences refuse a batch
 * session (PCLB200_ERR_INVALID). */
PCLB200_API int pclb200_icp_iterate_batch(pclb200_icp* icp, int max_steps, pclb200_icp_stats* stats);

/* The last evaluated iteration's correspondences of every problem, concatenated in problem order (each problem's list
 * is what its own session's pclb200_icp_get_correspondences returns: index_query relative to the problem's first
 * record).  out: host or device, capacity n (the batch's records); counts: host, B entries. */
PCLB200_API int pclb200_icp_get_correspondences_batch(pclb200_icp* icp, pclb200_corr* out, int64_t* counts);

/* getFitnessScore(max_range) of every problem of a batch session: problem p's own records under its current
 * final_transformation, against its own target (or the session's one target).  scores (host, B entries): scores[p] is bit
 * for bit pclb200_fitness_score_batch on the session's source, offsets, targets and stats[p].final_transformation with
 * the session's scalar_is_double, in any state, before the first pclb200_icp_iterate_batch (the guess) included.  The
 * call works on scratch of its own: the loop state, the correspondences and the moved source stay as they were, so the
 * next pclb200_icp_iterate_batch continues as if it had not run.  PCLB200_ERR_INVALID, with scores untouched, for a NULL
 * scores and a session without a batch source. */
PCLB200_API int pclb200_icp_fitness_score_batch(pclb200_icp* icp, double max_range, double* scores);

/* Registration::getFitnessScore of a batch of problems in one call: problem p = records [offsets[p], offsets[p+1]) of
 * src, moved by transforms[16p..16p+16) (row-major) and scored against targets[p].  scores[p] is bit for bit what
 * pclb200_fitness_score(ctx, targets[p], its first record, its record count, stride, NULL, 0, 1, T_p, scalar_is_double,
 * max_range, &s) gives: the mean squared distance of the nearest-neighbour pairs with d2 <= max_range, or DBL_MAX for a
 * problem with no finite point or no such pair.  A handle may repeat; every handle pclb200_fitness_score accepts is
 * accepted, from single builds or from pclb200_index_build_batch.  There is no per-problem index subset, and max_range is
 * one value for every problem.
 *
 * src: host or device, with the stride rules of pclb200_fitness_score.  targets, offsets (n_problems + 1 entries),
 * transforms (16 n_problems) and scores (n_problems): host.  Each stage is one launch for the whole batch, whatever
 * n_problems is, and the call reads the sums back and synchronises the context's stream once.  PCLB200_ERR_INVALID, with
 * scores untouched, for n_problems outside 1 to 65536, a NULL array or NULL handle, offsets[0] != 0, a problem with no
 * records, offsets[n_problems] != n, n >= 2^31 - 1, a bad stride and a handle on another device than the context. */
PCLB200_API int pclb200_fitness_score_batch(pclb200_ctx* ctx, const pclb200_index* const* targets, int32_t n_problems,
                                            const void* src, size_t n, size_t stride, const int64_t* offsets,
                                            const double* transforms, int scalar_is_double, double max_range,
                                            double* scores);

/* The same for TransformationValidationEuclidean::validateTransformation: scores[p] is bit for bit
 * pclb200_validate_transformation(ctx, targets[p], its first record, its record count, stride, T_p, scalar_is_double,
 * max_range, &s).  Arguments and refusals as pclb200_fitness_score_batch. */
PCLB200_API int pclb200_validate_transformation_batch(pclb200_ctx* ctx, const pclb200_index* const* targets,
                                                      int32_t n_problems, const void* src, size_t n, size_t stride,
                                                      const int64_t* offsets, const double* transforms,
                                                      int scalar_is_double, double max_range, double* scores);

/* A batch of independent indices in one build: cloud c = records [offsets[c], offsets[c+1]) of pts.  out[c] is bit for
 * bit the handle pclb200_index_build(ctx, its first record, its record count, stride, NULL, 0, &h) would give.  Its result
 * indices are relative to the cloud's first record.  Each handle is independent: it can be destroyed alone and in any
 * order, and it is accepted by every entry point that takes an index, pclb200_icp_set_target_batch included.
 *
 * pts: host or device, with the stride rules of pclb200_index_build.  offsets: host, n_clouds + 1 entries.  out: host,
 * n_clouds entries.  Every stage of the build is one launch for the whole batch, and the call synchronises the context's
 * stream three times, as one single build does.  All or nothing: on any error no handle exists afterwards and every
 * out[c] is NULL.  PCLB200_ERR_INVALID for n_clouds outside 1 to 65536, a NULL pts, offsets or out, offsets[0] != 0, a
 * cloud with no records, offsets[n_clouds] != n, n >= 2^31 - 1 or a bad stride; PCLB200_ERR_EMPTY when some cloud has no
 * finite point (pclb200_last_error names it). */
PCLB200_API int pclb200_index_build_batch(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride,
                                          const int64_t* offsets, int32_t n_clouds, pclb200_index** out);

/* The k-NN normals of a batch of query sets, each against its own index, in one call: query set c = records
 * [offsets[c], offsets[c+1]) of pts, searched in indices[c].  Row i of out (n rows of {nx, ny, nz, curvature}) belongs to
 * record i and is bit for bit what pclb200_normals_knn(ctx, indices[c], pts + offsets[c] * stride, its record count,
 * stride, NULL, 0, 1, k, viewpoint c, out + 4 offsets[c], &d_c) writes, and is_dense_out[c] (host, nullable, n_clouds
 * entries) is that call's d_c.  A query set need not be the cloud its index was built from, and a handle may repeat; every
 * handle pclb200_normals_knn accepts is accepted, from single builds or from pclb200_index_build_batch.
 *
 * pts and out: host or device, with the stride rules of pclb200_normals_knn.  offsets: host, n_clouds + 1 entries.
 * viewpoints: host, nullable, n_clouds rows of xyz; NULL = (0, 0, 0) for every set, PCL's default.  Every k the single call
 * takes is taken.  Each stage is one launch for the whole batch, whatever n_clouds is, and the call reads the flags back
 * and synchronises the context's stream once.  PCLB200_ERR_INVALID, with out and is_dense_out untouched, for n_clouds
 * outside 1 to 65536, a NULL indices, handle, pts, offsets or out, offsets[0] != 0, a query set with no records,
 * offsets[n_clouds] != n, n >= 2^31 - 1, a bad stride, k <= 0, a handle on another device than the context, and what
 * pclb200_normals_knn refuses of a handle (k > 32 on an index built with caller ids). */
PCLB200_API int pclb200_normals_knn_batch(pclb200_ctx* ctx, const pclb200_index* const* indices, int32_t n_clouds,
                                          const void* pts, size_t n, size_t stride, const int64_t* offsets, int k,
                                          const float* viewpoints /* nullable: n_clouds x 3 */, float* out,
                                          int32_t* is_dense_out /* nullable: n_clouds */);

/* VoxelGrid of a batch of clouds in one call: cloud c = records [offsets[c], offsets[c+1]) of pts, down-sampled with one
 * leaf and one minimum for every cloud.  Cloud c's rows are rows [out_offsets[c], out_offsets[c+1]) of out_xyz1, packed
 * in cloud order; they and their count are bit for bit what pclb200_voxelgrid(ctx, its first record, its record count,
 * stride, NULL, 0, 1, leaf, min_points_per_voxel, out, &m) gives, and with normals the same rows of out_normal_curv are
 * what pclb200_voxelgrid_normals gives.  No row past out_offsets[n_clouds] is written, so out_xyz1 and out_offsets go
 * straight to pclb200_index_build_batch and pclb200_icp_set_source_batch.  A cloud with no finite point, or whose voxels
 * all hold fewer than min_points_per_voxel points, gets an empty range, as the single call returns 0 for it; the caller
 * drops such a cloud before pclb200_index_build_batch, which refuses it.
 *
 * pts, normals, out_xyz1 and out_normal_curv: host or device, with the stride rules of pclb200_voxelgrid and
 * pclb200_voxelgrid_normals; normals and out_normal_curv are both given or both NULL.  out_xyz1 (and out_normal_curv):
 * capacity n rows.  offsets: host, n_clouds + 1 entries.  out_offsets: host, n_clouds + 1 entries.  Each stage is one
 * launch (or one sort or select) for the whole batch, and the call synchronises the context's stream as often as one
 * pclb200_voxelgrid does.  PCLB200_ERR_INVALID for n_clouds outside 1 to 65536, a NULL pts, offsets, leaf, out_xyz1 or
 * out_offsets, offsets[0] != 0, a cloud with no records, offsets[n_clouds] != n, n >= 2^31 - 1, a bad stride, a normal
 * stride below 20 or not a multiple of 4, a leaf that is not positive, and only one of normals and out_normal_curv;
 * PCLB200_ERR_LEAF_TOO_SMALL when the grid of some cloud trips pclb200_voxelgrid's integer guard (pclb200_last_error
 * names the first such cloud), with no result for any cloud.  Every refusal leaves the outputs and out_offsets
 * untouched. */
PCLB200_API int pclb200_voxelgrid_batch(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride,
                                        const int64_t* offsets, int32_t n_clouds, const float leaf[3],
                                        unsigned min_points_per_voxel,
                                        const void* normals /* nullable */, size_t stride_n,
                                        float* out_xyz1, float* out_normal_curv /* nullable */,
                                        int64_t* out_offsets /* host, n_clouds + 1 */);

#ifdef __cplusplus
}
#endif
#endif /* PCLB200_BATCH_H_ */
