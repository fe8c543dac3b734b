// knn_warp.cuh — device code of the normals epilogue (eigen33 in fp32, the single-pass moments) and of the
// warp-per-query k-NN kernel.  A header so that search.cu's kernels share it and so that tests/host/knn_warp_host_test.cpp
// can compile the SAME source for the host (a lock-step emulation of one warp) and check it against brute force.
#pragma once
#include "internal.cuh"
#include "traverse.cuh"

namespace pclb200 {

// ---- normals ---------------------------------------------------------------------------------------
// pcl::eigen33 smallest eigenpair in fp32 — common/include/pcl/common/impl/eigen.hpp:52-133 (roots),
// :273-288 (largest cross product), :293-326 (eigen33); m = row-major symmetric 3x3.
__device__ __forceinline__ void roots2_dev(float b, float c, float* r)
{
  r[0] = 0.f;
  float d = (float)((double)(b * b) - 4.0 * (double)c);
  if (d < 0.f)
    d = 0.f;
  float sd = sqrtf(d);
  r[2] = 0.5f * (b + sd);
  r[1] = 0.5f * (b - sd);
}

__device__ void roots3_dev(const float* m, float* r)
{
  float c0 = m[0] * m[4] * m[8] + 2.f * m[1] * m[2] * m[5] - m[0] * m[5] * m[5] - m[4] * m[2] * m[2] -
             m[8] * m[1] * m[1];
  float c1 = m[0] * m[4] - m[1] * m[1] + m[0] * m[8] - m[2] * m[2] + m[4] * m[8] - m[5] * m[5];
  float c2 = m[0] + m[4] + m[8];
  if (fabsf(c0) < FLT_EPSILON) {
    roots2_dev(c2, c1, r);
    return;
  }
  const float s_inv3 = (float)(1.0 / 3.0);
  const float s_sqrt3 = sqrtf(3.f);
  float c2_over_3 = c2 * s_inv3;
  float a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
  if (a_over_3 > 0.f)
    a_over_3 = 0.f;
  float half_b = 0.5f * (c0 + c2_over_3 * (2.f * c2_over_3 * c2_over_3 - c1));
  float q = half_b * half_b + a_over_3 * a_over_3 * a_over_3;
  if (q > 0.f)
    q = 0.f;
  float rho = sqrtf(-a_over_3);
  float theta = atan2f(sqrtf(-q), half_b) * s_inv3;
  float cos_theta = cosf(theta), sin_theta = sinf(theta);
  r[0] = c2_over_3 + 2.f * rho * cos_theta;
  r[1] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
  r[2] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
  float t;
  if (r[0] >= r[1]) { t = r[0]; r[0] = r[1]; r[1] = t; }
  if (r[1] >= r[2]) {
    t = r[1]; r[1] = r[2]; r[2] = t;
    if (r[0] >= r[1]) { t = r[0]; r[0] = r[1]; r[1] = t; }
  }
  if (r[0] <= 0.f)
    roots2_dev(c2, c1, r);
}

__device__ void largest_eigvec_dev(const float* s, float* v)
{
  float c[3][3] = {{s[1] * s[5] - s[2] * s[4], s[2] * s[3] - s[0] * s[5], s[0] * s[4] - s[1] * s[3]},
                   {s[1] * s[8] - s[2] * s[7], s[2] * s[6] - s[0] * s[8], s[0] * s[7] - s[1] * s[6]},
                   {s[4] * s[8] - s[5] * s[7], s[5] * s[6] - s[3] * s[8], s[3] * s[7] - s[4] * s[6]}};
  float len[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
    len[i] = sqrtf(c[i][0] * c[i][0] + c[i][1] * c[i][1] + c[i][2] * c[i][2]);
  int idx = 0;
  if (len[1] > len[idx]) idx = 1;
  if (len[2] > len[idx]) idx = 2;
  float l = idx == 0 ? len[0] : (idx == 1 ? len[1] : len[2]);
#pragma unroll
  for (int d = 0; d < 3; ++d)
    v[d] = (idx == 0 ? c[0][d] : (idx == 1 ? c[1][d] : c[2][d])) / l;
}

__device__ void eigen33_smallest_dev(const float* mat, float& eigenvalue, float* ev)
{
  float scale = 0.f;
#pragma unroll
  for (int i = 0; i < 9; ++i)
    scale = fmaxf(scale, fabsf(mat[i]));
  if (scale <= FLT_MIN)
    scale = 1.f;
  float s[9];
#pragma unroll
  for (int i = 0; i < 9; ++i)
    s[i] = __fdiv_rn(mat[i], scale);
  float r[3];
  roots3_dev(s, r);
  eigenvalue = r[0] * scale;
  if ((r[1] - r[0]) > FLT_EPSILON) {
    s[0] -= r[0]; s[4] -= r[0]; s[8] -= r[0];
    largest_eigvec_dev(s, ev);
  }
  else if ((r[2] - r[0]) > FLT_EPSILON) {
    s[0] -= r[2]; s[4] -= r[2]; s[8] -= r[2];
    float v[3];
    largest_eigvec_dev(s, v);
    // Eigen unitOrthogonal()
    bool a = fabsf(v[0]) <= fabsf(v[2]) * FLT_EPSILON, b = fabsf(v[1]) <= fabsf(v[2]) * FLT_EPSILON;
    if (!a || !b) {
      float inv = 1.f / sqrtf(v[0] * v[0] + v[1] * v[1]);
      ev[0] = -v[1] * inv; ev[1] = v[0] * inv; ev[2] = 0.f;
    }
    else {
      float inv = 1.f / sqrtf(v[1] * v[1] + v[2] * v[2]);
      ev[0] = 0.f; ev[1] = -v[2] * inv; ev[2] = v[1] * inv;
    }
  }
  else {
    ev[0] = 1.f; ev[1] = 0.f; ev[2] = 0.f;
  }
}

// shifted single-pass moments (centroid.hpp:605-640): one neighbour, K = the first neighbour of the list
__device__ __forceinline__ void moments_add(float (&accu)[9], float Kx, float Ky, float Kz, const float4 p)
{
  const float x = __fsub_rn(p.x, Kx), y = __fsub_rn(p.y, Ky), z = __fsub_rn(p.z, Kz);
  accu[0] = __fadd_rn(accu[0], __fmul_rn(x, x));
  accu[1] = __fadd_rn(accu[1], __fmul_rn(x, y));
  accu[2] = __fadd_rn(accu[2], __fmul_rn(x, z));
  accu[3] = __fadd_rn(accu[3], __fmul_rn(y, y));
  accu[4] = __fadd_rn(accu[4], __fmul_rn(y, z));
  accu[5] = __fadd_rn(accu[5], __fmul_rn(z, z));
  accu[6] = __fadd_rn(accu[6], x);
  accu[7] = __fadd_rn(accu[7], y);
  accu[8] = __fadd_rn(accu[8], z);
}

// moments -> covariance (centroid.hpp:641-651) -> solvePlaneParameters (feature.hpp:65-92) ->
// flipNormalTowardsViewpoint (normal_3d.h:169-188); returns {nx, ny, nz, curvature}
__device__ __forceinline__ float4 normal_from_moments(float (&accu)[9], int cnt, const float4 qq, float vpx, float vpy,
                                                      float vpz, int* __restrict__ not_dense)
{
  const float fc = (float)cnt;
#pragma unroll
  for (int t = 0; t < 9; ++t)
    accu[t] = __fdiv_rn(accu[t], fc);
  float cov[9];
  cov[0] = __fsub_rn(accu[0], __fmul_rn(accu[6], accu[6]));
  cov[1] = __fsub_rn(accu[1], __fmul_rn(accu[6], accu[7]));
  cov[2] = __fsub_rn(accu[2], __fmul_rn(accu[6], accu[8]));
  cov[4] = __fsub_rn(accu[3], __fmul_rn(accu[7], accu[7]));
  cov[5] = __fsub_rn(accu[4], __fmul_rn(accu[7], accu[8]));
  cov[8] = __fsub_rn(accu[5], __fmul_rn(accu[8], accu[8]));
  cov[3] = cov[1]; cov[6] = cov[2]; cov[7] = cov[5];
  float ev, n[3];
  eigen33_smallest_dev(cov, ev, n);
  const float eig_sum = __fadd_rn(__fadd_rn(cov[0], cov[4]), cov[8]);
  const float curv = eig_sum != 0.f ? fabsf(__fdiv_rn(ev, eig_sum)) : 0.f;
  const float vx = vpx - qq.x, vy = vpy - qq.y, vz = vpz - qq.z;
  const float cos_theta = vx * n[0] + vy * n[1] + vz * n[2];
  if (cos_theta < 0.f) { n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2]; }
  if (!(isfinite(n[0]) && isfinite(n[1]) && isfinite(n[2]) && isfinite(curv)))
    *not_dense = 1;
  return make_float4(n[0], n[1], n[2], curv);
}

// =============================================================================================================
// Warp-cooperative k-NN (k <= 32): one WARP per query, brute force over the cells that hold the answer
// =============================================================================================================
// The per-thread kernels above keep a k-deep sorted list in registers: at k = 16 every accepted candidate costs a
// ~100-instruction dependent bubble pass executed under divergence, with a fraction of the lanes active.  Here the list
// is ONE ENTRY PER LANE, sorted
// across the warp, and candidates arrive 32 at a time from CONTIGUOUS memory:
//   * the cell table (traverse.cuh) maps a cell of level b to the subtree holding exactly its points; a subtree's leaves
//     are consecutive in the Morton array, so "all points of a cell" is one coalesced range;
//   * a ball of radius R = half a level-b cell reaches at most 2 x 2 x 2 cells.  The warp gathers those cells, keeps the k
//     smallest (d2, index) — a bitonic sort / merge by shuffles when many candidates beat the current k-th, a ranked
//     insertion (ballot + shuffle-up) when few do — and the result is EXACT iff the k-th distance is below R: every
//     point outside the gathered cells lies outside [q - R, q + R]^3.  Otherwise the next coarser level (R doubles).
//   * the start level comes from the index's density (cells that hold ~2k points on average), so one attempt is the norm.
// Queries the scheme does not fit (far outside the cloud, > kWarpKnnMaxLeaves leaves in reach, no level certifies) are
// flagged and redone by the per-thread kernel — same results, the exact walk is the fallback, never an approximation.
constexpr int kWarpKnnMaxLeaves = 1024;

__device__ __forceinline__ bool lex_less(float da, int ia, float db, int ib) { return da < db || (da == db && ia < ib); }

// ascending bitonic sort of one (d, i, p) triple per lane
__device__ __forceinline__ void warp_sort32(float& d, int& i, int& p, int lane)
{
  const unsigned full = 0xffffffffu;
#pragma unroll
  for (int k2 = 2; k2 <= 32; k2 <<= 1)
#pragma unroll
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      const float pd = __shfl_xor_sync(full, d, j);
      const int pi = __shfl_xor_sync(full, i, j);
      const int pp = __shfl_xor_sync(full, p, j);
      const bool asc = (lane & k2) == 0, lower = (lane & j) == 0;
      const bool mine_first = lex_less(d, i, pd, pi);
      const bool keep = (lower == asc) ? mine_first : !mine_first;
      if (!keep) {
        d = pd; i = pi; p = pp;
      }
    }
}

// list (sorted ascending across lanes) <- the 32 smallest of list U cand (cand sorted ascending across lanes)
__device__ __forceinline__ void warp_merge32(float& ld, int& li, int& lp, float cd, int ci, int cp, int lane)
{
  const unsigned full = 0xffffffffu;
  const float rd = __shfl_sync(full, cd, 31 - lane);
  const int ri = __shfl_sync(full, ci, 31 - lane);
  const int rp = __shfl_sync(full, cp, 31 - lane);
  if (lex_less(rd, ri, ld, li)) {  // elementwise min of an ascending and a descending sequence: bitonic, the 32 smallest
    ld = rd; li = ri; lp = rp;
  }
#pragma unroll
  for (int j = 16; j > 0; j >>= 1) {
    const float pd = __shfl_xor_sync(full, ld, j);
    const int pi = __shfl_xor_sync(full, li, j);
    const int pp = __shfl_xor_sync(full, lp, j);
    const bool lower = (lane & j) == 0;
    const bool mine_first = lex_less(ld, li, pd, pi);
    if (lower != mine_first) {
      ld = pd; li = pi; lp = pp;
    }
  }
}

template <bool NORMALS>
__global__ void __launch_bounds__(256)
k_knn_warp(const TreeView T, const int2* __restrict__ node_leaves, int b_start, float r_first, const float4* __restrict__ q, size_t nq,
           int k, int32_t* __restrict__ out_idx, float* __restrict__ out_d2, float vpx, float vpy, float vpz,
           float4* __restrict__ out_n, int* __restrict__ not_dense, unsigned char* __restrict__ redo)
{
#define PCLB_KNN_WARP_QUERY(qi)
#define PCLB_KNN_WARP_LANE(qi)
#include "knn_warp_body.inc"
#undef PCLB_KNN_WARP_QUERY
#undef PCLB_KNN_WARP_LANE
}

// ---- the k-NN normals of a batch of query sets, each against its own index (search.cu: launch_normals_batch) ----------
// One entry per query set: what the single normals kernels take as parameters.
struct NormalsCloud {
  TreeView tree;
  const int2* node_leaves;
  const int32_t* pos_of_orig;  // the lists path (k > 32) only
  int level;                   // start level of the warp kernel; 0 = every query goes to the per-thread kernel
  float r_first;
  float vp[3];
  int* not_dense;              // this set's own flag
};

// k_knn_warp<true> over queries sorted by set (q[offsets[c] .. offsets[c+1]) belong to set c): each query is searched
// in its own set's index (one lookup, the same for the whole warp), and each lane's epilogue reads its own set's points,
// viewpoint and flag.  A set with level 0 hands every finite query to the per-thread kernel.
__global__ void __launch_bounds__(256)
k_knn_warp_batch(const NormalsCloud* __restrict__ clouds, const long long* __restrict__ offsets, int n_clouds,
                 const float4* __restrict__ q, size_t nq, int k, float4* __restrict__ out_n,
                 unsigned char* __restrict__ redo)
{
  constexpr bool NORMALS = true;
  int32_t* const out_idx = nullptr;
  float* const out_d2 = nullptr;
#define PCLB_KNN_WARP_QUERY(qi)                                          \
  const NormalsCloud& Q = clouds[problem_of(offsets, n_clouds, (long long)(qi))]; \
  const TreeView T = Q.tree;                                             \
  const int2* __restrict__ node_leaves = Q.node_leaves;                  \
  const int b_start = Q.level;                                           \
  const float r_first = Q.r_first;
#define PCLB_KNN_WARP_LANE(qi)                                           \
  const NormalsCloud& L = clouds[problem_of(offsets, n_clouds, (long long)(qi))]; \
  const TreeView T = L.tree;                                             \
  const float vpx = L.vp[0], vpy = L.vp[1], vpz = L.vp[2];               \
  int* const not_dense = L.not_dense;
#include "knn_warp_body.inc"
#undef PCLB_KNN_WARP_QUERY
#undef PCLB_KNN_WARP_LANE
}

}  // namespace pclb200
