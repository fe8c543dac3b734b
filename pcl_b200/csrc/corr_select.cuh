// corr_select.cuh — choosing one of the k nearest target points with the help of normals.
//
// Device restatement of the inner loops of
//   CorrespondenceEstimationNormalShooting::determineCorrespondences
//     (registration/include/pcl/registration/impl/correspondence_estimation_normal_shooting.hpp:99-127)
//   CorrespondenceEstimationBackProjection::determineCorrespondences
//     (registration/include/pcl/registration/impl/correspondence_estimation_backprojection.hpp:91-114)
// and of the score of CorrespondenceRejectorSurfaceNormal
//     (registration/include/pcl/registration/correspondence_rejection.h:378-389).
// The k candidates come from the exact k-NN kernels (search.cu) as rows of (original index, d2) in ascending
// (d2, index) order; every operation is a single correctly rounded fp32 / fp64 op in the reference's order, so the
// chosen index is the one the CPU path picks.
#pragma once
#include <cfloat>

#include "internal.cuh"
#include "traverse.cuh"

namespace pclb200 {

// The score of one candidate, the per-candidate arithmetic of both loops below (and of their form on a sharded map,
// shard_target_kernels.cuh).  Normal shooting: pt = target - source in float (:106-108), then the squared norm of its
// cross product with the source normal in double (:110-116).  Back projection: d2 (2 - cos^2) in float (:99-108).
__device__ __forceinline__ double shooting_score(const float4 q, float px, float py, float pz, double Nx, double Ny,
                                                 double Nz)
{
  const double Vx = (double)__fsub_rn(q.x, px), Vy = (double)__fsub_rn(q.y, py), Vz = (double)__fsub_rn(q.z, pz);
  const double Cx = __dsub_rn(__dmul_rn(Ny, Vz), __dmul_rn(Nz, Vy));
  const double Cy = __dsub_rn(__dmul_rn(Nz, Vx), __dmul_rn(Nx, Vz));
  const double Cz = __dsub_rn(__dmul_rn(Nx, Vy), __dmul_rn(Ny, Vx));
  return __dadd_rn(__dadd_rn(__dmul_rn(Cx, Cx), __dmul_rn(Cy, Cy)), __dmul_rn(Cz, Cz));
}
__device__ __forceinline__ float backprojection_score(float d2, float nx, float ny, float nz, const float4 m)
{
  const float cos_angle = __fadd_rn(__fadd_rn(__fmul_rn(nx, m.x), __fmul_rn(ny, m.y)), __fmul_rn(nz, m.z));
  return __fmul_rn(d2, __fsub_rn(2.0f, __fmul_rn(cos_angle, cos_angle)));
}

// Returns the column of the chosen candidate, or -1 when the gate rejects the point.
//   row_idx / row_d2 : this query's k candidates (k >= 1, all valid)
//   (px,py,pz), (nx,ny,nz) : source point and its normal
//   pos_of_orig : original target index -> position in tgt_pts
//   tgt_nrm     : target normals (back projection only), indexed by position when NRM_BY_POS, else by original index
template <bool NRM_BY_POS>
__device__ __forceinline__ int select_by_normals(int kind, int k, const int32_t* __restrict__ row_idx,
                                                 const float* __restrict__ row_d2, float px, float py, float pz,
                                                 float nx, float ny, float nz, const float4* __restrict__ tgt_pts,
                                                 const int32_t* __restrict__ pos_of_orig,
                                                 const float4* __restrict__ tgt_nrm, double max_dist)
{
  int min_j = 0;
  if (kind == PCLB200_CORR_NORMAL_SHOOTING) {
    double min_dist = DBL_MAX;
    const double Nx = (double)nx, Ny = (double)ny, Nz = (double)nz;
    for (int j = 0; j < k; ++j) {
      const int oi = row_idx[j];
      if (oi < 0)
        break;
      const float4 q = ldg4(tgt_pts + pos_of_orig[oi]);
      const double dist = shooting_score(q, px, py, pz, Nx, Ny, Nz);
      if (dist < min_dist) {
        min_dist = dist;
        min_j = j;
      }
    }
    if (min_dist > max_dist)  // :121 — the squared line distance against max_distance itself, as the reference does
      return -1;
  }
  else {
    float min_dist = FLT_MAX;
    for (int j = 0; j < k; ++j) {
      const int oi = row_idx[j];
      if (oi < 0)
        break;
      const float4 m = ldg4(tgt_nrm + (NRM_BY_POS ? pos_of_orig[oi] : oi));
      const float dist = backprojection_score(row_d2[j], nx, ny, nz, m);
      if (dist < min_dist) {
        min_dist = dist;
        min_j = j;
      }
    }
    if ((double)min_dist > max_dist)
      return -1;
  }
  return min_j;
}

// float dot product of two normals, promoted to double, against the threshold (correspondence_rejection.h:386-388,
// correspondence_rejection_surface_normal.cpp:60-62).  NaN normals fail the test, as `NaN > t` does on the host.
__device__ __forceinline__ bool surface_normal_keeps(const float4 a, const float4 b, double threshold)
{
  const float dot = __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z));
  return (double)dot > threshold;
}

}  // namespace pclb200
