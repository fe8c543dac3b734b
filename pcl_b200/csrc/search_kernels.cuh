// search_kernels.cuh — the per-thread search kernels: exact k-NN with a register list (k <= 32) or with the list in the
// output rows (any k), k-NN statistics for the outlier filters, radius count / fill, and the per-thread normals kernels.
// A header so that tests/host/search_host_test.cpp can compile the SAME source for the host and check it against brute
// force; search.cu holds the launches.
#pragma once
#include "internal.cuh"
#include "traverse.cuh"
#include "knn_warp.cuh"

namespace pclb200 {

// ---- k nearest, k <= K (compile-time), ascending (d2, original index) ------------------------------
template <int K>
struct NearestK {
  float qx, qy, qz;
  const float4* pts;
  float d[K];
  int pos[K];
  __device__ __forceinline__ void init(float bound)
  {
#pragma unroll
    for (int j = 0; j < K; ++j) {
      d[j] = bound;
      pos[j] = -1;
    }
  }
  __device__ __forceinline__ int orig(int p) const
  {
    return p < 0 ? kSentinelIndex : __float_as_int(__ldg(&pts[p].w));
  }
  __device__ __forceinline__ float bound() const { return d[K - 1]; }
  __device__ __forceinline__ void prune(float) {}
  __device__ __forceinline__ void leaf(const float4* lp, int first_pos)
  {
    float4 p[kLeafSize];
#pragma unroll
    for (int j = 0; j < kLeafSize; ++j)
      p[j] = ldg4(lp + j);
#pragma unroll
    for (int j = 0; j < kLeafSize; ++j) {
      float dd = dist2_rn(qx, qy, qz, p[j].x, p[j].y, p[j].z);
      int oi = __float_as_int(p[j].w);
      if (dd < d[K - 1] || (dd == d[K - 1] && oi < orig(pos[K - 1]))) {
        d[K - 1] = dd;
        pos[K - 1] = first_pos + j;
        // one bubble pass keeps the list sorted; exact-distance ties compare original indices
#pragma unroll
        for (int t = K - 1; t > 0; --t) {
          bool lt = d[t] < d[t - 1] || (d[t] == d[t - 1] && orig(pos[t]) < orig(pos[t - 1]));
          if (lt) {
            float td = d[t]; d[t] = d[t - 1]; d[t - 1] = td;
            int tp = pos[t]; pos[t] = pos[t - 1]; pos[t - 1] = tp;
          }
        }
      }
    }
  }
};

template <int K>
__global__ void __launch_bounds__(128)
k_knn(const BvhNode* __restrict__ nodes, const float4* __restrict__ pts, int root,
      const float4* __restrict__ q, size_t nq, int k_out, float init_bound,
      int32_t* __restrict__ out_idx, float* __restrict__ out_d2, int* __restrict__ d_error,
      const unsigned char* __restrict__ only = nullptr)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq || (only && !only[i]))  // fix-up pass: only the queries the warp kernel handed back
    return;
  const float4 qq = __ldg(q + i);
  const size_t slot = (size_t)(unsigned)__float_as_int(qq.w);
  NearestK<K> v;
  v.qx = qq.x; v.qy = qq.y; v.qz = qq.z;
  v.pts = pts;
  v.init(init_bound);
  // a non-finite query has no neighbours (every comparison with NaN fails; rows stay (-1, +inf)) — without the guard
  // it would walk the whole tree, because a NaN box bound never prunes
  if (isfinite(qq.x) && isfinite(qq.y) && isfinite(qq.z) && !traverse(nodes, pts, root, qq.x, qq.y, qq.z, v))
    atomicExch(d_error, kErrStackOverflow);
#pragma unroll
  for (int j = 0; j < K; ++j)
    if (j < k_out) {
      const bool have = v.pos[j] >= 0;
      out_idx[slot * k_out + j] = have ? v.orig(v.pos[j]) : -1;
      out_d2[slot * k_out + j] = have ? v.d[j] : __int_as_float(0x7f800000);
    }
}

// ---- any k: the candidate list lives in the output rows themselves (global memory) -----------------
struct NearestAny {
  float qx, qy, qz;
  const float4* pts;
  float* d;   // k entries, ascending
  int* pos;   // k entries (positions; converted to original indices afterwards)
  int k;
  __device__ __forceinline__ int orig(int p) const
  {
    return p < 0 ? kSentinelIndex : __float_as_int(__ldg(&pts[p].w));
  }
  __device__ __forceinline__ float bound() const { return d[k - 1]; }
  __device__ __forceinline__ void prune(float) {}
  __device__ __forceinline__ void leaf(const float4* lp, int first_pos)
  {
    for (int j = 0; j < kLeafSize; ++j) {
      float4 p = ldg4(lp + j);
      float dd = dist2_rn(qx, qy, qz, p.x, p.y, p.z);
      int oi = __float_as_int(p.w);
      if (dd < d[k - 1] || (dd == d[k - 1] && oi < orig(pos[k - 1]))) {
        int t = k - 1;
        while (t > 0 && (dd < d[t - 1] || (dd == d[t - 1] && oi < orig(pos[t - 1])))) {
          d[t] = d[t - 1];
          pos[t] = pos[t - 1];
          --t;
        }
        d[t] = dd;
        pos[t] = first_pos + j;
      }
    }
  }
};

__global__ void __launch_bounds__(128)
k_knn_any(const BvhNode* __restrict__ nodes, const float4* __restrict__ pts, int root,
          const float4* __restrict__ q, size_t nq, int k, float init_bound, int32_t* out_idx, float* out_d2,
          int* __restrict__ d_error)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
#include "knn_any_body.inc"
}

// ---- per-query statistics of the k nearest neighbours (outlier filters) -------------------------------------------
// mean[slot] = float( sum_{j=1..k'-1} sqrt(double(d2_j)) / (k'-1) )   (statistical_outlier_removal.hpp:88-97; j = 0 is
//              the query itself when it belongs to the cloud), 0 for non-finite queries
// kth[slot]  = d2 of neighbour k-1, +inf when fewer than k points are indexed (radius_outlier_removal.hpp:86-118)
template <int K>
__global__ void __launch_bounds__(128)
k_knn_stats(const BvhNode* __restrict__ nodes, const float4* __restrict__ pts, int root, const float4* __restrict__ q,
            size_t nq, int k, float* __restrict__ out_mean, float* __restrict__ out_kth, int* __restrict__ d_error)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  const float4 qq = __ldg(q + i);
  const size_t slot = (size_t)(unsigned)__float_as_int(qq.w);
  float mean = 0.f, kth = __int_as_float(0x7f800000);
  if (isfinite(qq.x) && isfinite(qq.y) && isfinite(qq.z)) {
    NearestK<K> v;
    v.qx = qq.x; v.qy = qq.y; v.qz = qq.z;
    v.pts = pts;
    v.init(__int_as_float(0x7f800000));
    if (!traverse(nodes, pts, root, qq.x, qq.y, qq.z, v))
      atomicExch(d_error, kErrStackOverflow);
    double sum = 0.0;
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < K; ++j)
      if (j < k && v.pos[j] >= 0) {
        if (j >= 1)
          sum += sqrt((double)v.d[j]);
        ++cnt;
        if (j == k - 1)
          kth = v.d[j];
      }
    if (cnt > 1)
      mean = (float)(sum / (double)(cnt - 1));
  }
  if (out_mean)
    out_mean[slot] = mean;
  if (out_kth)
    out_kth[slot] = kth;
}

// same from materialised lists (k > 32): rows of pitch k by slot
__global__ void k_stats_from_lists(const float4* __restrict__ q, size_t nq, int k, const int32_t* __restrict__ li,
                                   const float* __restrict__ ld, float* __restrict__ out_mean, float* __restrict__ out_kth)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  const float4 qq = __ldg(q + i);
  const size_t slot = (size_t)(unsigned)__float_as_int(qq.w);
  float mean = 0.f, kth = __int_as_float(0x7f800000);
  if (isfinite(qq.x) && isfinite(qq.y) && isfinite(qq.z)) {
    double sum = 0.0;
    int cnt = 0;
    for (int j = 0; j < k; ++j)
      if (li[slot * k + j] >= 0) {
        if (j >= 1)
          sum += sqrt((double)ld[slot * k + j]);
        ++cnt;
        if (j == k - 1)
          kth = ld[slot * k + j];
      }
    if (cnt > 1)
      mean = (float)(sum / (double)(cnt - 1));
  }
  if (out_mean)
    out_mean[slot] = mean;
  if (out_kth)
    out_kth[slot] = kth;
}

// ---- radius search: count, then fill keys (d2 bits << 32 | original index) -------------------------
struct RadiusCount {
  float qx, qy, qz, r2;
  float r2_below;  // largest float < r2: subtrees with bound > r2_below hold no d2 < r2
  unsigned long long n;
  __device__ __forceinline__ float bound() const { return r2_below; }
  __device__ __forceinline__ void prune(float) {}
  __device__ __forceinline__ void leaf(const float4* lp, int)
  {
#pragma unroll
    for (int j = 0; j < kLeafSize; ++j) {
      float4 p = ldg4(lp + j);
      if (dist2_rn(qx, qy, qz, p.x, p.y, p.z) < r2)
        ++n;
    }
  }
};

struct RadiusFill {
  float qx, qy, qz, r2;
  float r2_below;
  unsigned long long* out;
  __device__ __forceinline__ float bound() const { return r2_below; }
  __device__ __forceinline__ void prune(float) {}
  __device__ __forceinline__ void leaf(const float4* lp, int)
  {
#pragma unroll
    for (int j = 0; j < kLeafSize; ++j) {
      float4 p = ldg4(lp + j);
      float dd = dist2_rn(qx, qy, qz, p.x, p.y, p.z);
      if (dd < r2)
        *out++ = ((unsigned long long)__float_as_uint(dd) << 32) | (unsigned)__float_as_int(p.w);
    }
  }
};

__global__ void __launch_bounds__(128)
k_radius_count(const BvhNode* __restrict__ nodes, const float4* __restrict__ pts, int root,
               const float4* __restrict__ q, size_t nq, float r2, float r2_below,
               unsigned long long* __restrict__ counts, int* __restrict__ d_error)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  const float4 qq = __ldg(q + i);
  RadiusCount v{qq.x, qq.y, qq.z, r2, r2_below, 0ULL};
  // a non-finite query has no neighbour (every comparison with NaN fails) — and would otherwise walk the whole tree
  if (isfinite(qq.x) && isfinite(qq.y) && isfinite(qq.z) && !traverse(nodes, pts, root, qq.x, qq.y, qq.z, v))
    atomicExch(d_error, kErrStackOverflow);
  counts[(size_t)(unsigned)__float_as_int(qq.w)] = v.n;
}

__global__ void __launch_bounds__(128)
k_radius_fill(const BvhNode* __restrict__ nodes, const float4* __restrict__ pts, int root,
              const float4* __restrict__ q, size_t nq, float r2, float r2_below,
              const unsigned long long* __restrict__ offsets, unsigned long long* __restrict__ keys,
              int* __restrict__ d_error)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  const float4 qq = __ldg(q + i);
  RadiusFill v{qq.x, qq.y, qq.z, r2, r2_below, keys + offsets[(size_t)(unsigned)__float_as_int(qq.w)]};
  if (isfinite(qq.x) && isfinite(qq.y) && isfinite(qq.z) && !traverse(nodes, pts, root, qq.x, qq.y, qq.z, v))
    atomicExch(d_error, kErrStackOverflow);
}

// k-NN -> shifted single-pass covariance in the neighbour order the search returns
// (common/include/pcl/common/impl/centroid.hpp:578-652, Scalar = float, same operation order, no fma)
// -> solvePlaneParameters (features/impl/feature.hpp:65-92) -> flipNormalTowardsViewpoint
// (features/normal_3d.h:169-188).  The neighbour list is never materialised in HBM.
template <int K>
__global__ void __launch_bounds__(128)
k_normals(const BvhNode* __restrict__ nodes, const float4* __restrict__ pts, int root,
          const float4* __restrict__ q, size_t nq, int k_req, float vpx, float vpy, float vpz,
          float4* __restrict__ out, int* __restrict__ not_dense, int* __restrict__ d_error,
          const unsigned char* __restrict__ only = nullptr)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq || (only && !only[i]))
    return;
#include "normals_body.inc"
}

// normals from materialised neighbour lists (k > 32): same arithmetic as k_normals, neighbours fetched through
// pos_of_orig.  lists are rows of pitch k indexed by the query's slot.
__global__ void __launch_bounds__(128)
k_normals_from_lists(const float4* __restrict__ pts, const int32_t* __restrict__ pos_of_orig,
                     const float4* __restrict__ q, size_t nq, int k, const int32_t* __restrict__ lists, size_t slot0,
                     float vpx, float vpy, float vpz, float4* __restrict__ out, int* __restrict__ not_dense)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
#include "normals_from_lists_body.inc"
}

// normals from radius neighbourhoods (setRadiusSearch): rows of a CSR of packed keys (radius_csr), addressed by the
// query's slot; same arithmetic as k_normals over a variable-length, (d2, index)-ascending neighbour list.
__global__ void __launch_bounds__(128)
k_normals_from_csr(const float4* __restrict__ pts, const int32_t* __restrict__ pos_of_orig,
                   const float4* __restrict__ q, size_t nq, const unsigned long long* __restrict__ offsets,
                   const unsigned long long* __restrict__ keys, float vpx, float vpy, float vpz,
                   float4* __restrict__ out, int* __restrict__ not_dense)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  const float4 qq = __ldg(q + i);
  const size_t slot = (size_t)(unsigned)__float_as_int(qq.w);
  const unsigned long long b = offsets[slot], e = offsets[slot + 1];
  const float qnan = __int_as_float(0x7fc00000);
  if (!(isfinite(qq.x) && isfinite(qq.y) && isfinite(qq.z)) || e - b < 3ULL) {  // normal_3d.h:308-312
    out[slot] = make_float4(qnan, qnan, qnan, qnan);
    *not_dense = 1;
    return;
  }
  float accu[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float Kx = 0.f, Ky = 0.f, Kz = 0.f;
  for (unsigned long long j = b; j < e; ++j) {
    const int oi = (int)(unsigned)(keys[j] & 0xffffffffULL);
    const float4 p = ldg4(pts + pos_of_orig[oi]);
    if (j == b) { Kx = p.x; Ky = p.y; Kz = p.z; }
    moments_add(accu, Kx, Ky, Kz, p);
  }
  out[slot] = normal_from_moments(accu, (int)(e - b), qq, vpx, vpy, vpz, not_dense);
}

// ---- batch forms of the k-NN normals kernels (search.cu: launch_normals_batch) -----------------------------------------
// The queries of every set, sorted by set (q[offsets[c] .. offsets[c+1]) belong to set c, w = the record's row in the
// whole batch); each thread runs the single kernel's body on its own set's entry of the table (knn_warp.cuh: NormalsCloud).
template <int K>
__global__ void __launch_bounds__(128)
k_normals_batch(const NormalsCloud* __restrict__ clouds, const long long* __restrict__ offsets, int n_clouds,
                const float4* __restrict__ q, size_t nq, int k_req, float4* __restrict__ out, int* __restrict__ d_error,
                const unsigned char* __restrict__ only)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq || (only && !only[i]))
    return;
  const NormalsCloud& Q = clouds[problem_of(offsets, n_clouds, (long long)i)];
  const BvhNode* __restrict__ nodes = Q.tree.nodes;
  const float4* __restrict__ pts = Q.tree.pts;
  const int root = Q.tree.root;
  const float vpx = Q.vp[0], vpy = Q.vp[1], vpz = Q.vp[2];
  int* const not_dense = Q.not_dense;
#include "normals_body.inc"
}

// k_knn_any over every set's tree: rows of pitch k by the query's row in the batch
__global__ void __launch_bounds__(128)
k_knn_any_batch(const NormalsCloud* __restrict__ clouds, const long long* __restrict__ offsets, int n_clouds,
                const float4* __restrict__ q, size_t nq, int k, float init_bound, int32_t* out_idx, float* out_d2,
                int* __restrict__ d_error)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  const NormalsCloud& Q = clouds[problem_of(offsets, n_clouds, (long long)i)];
  const BvhNode* __restrict__ nodes = Q.tree.nodes;
  const float4* __restrict__ pts = Q.tree.pts;
  const int root = Q.tree.root;
#include "knn_any_body.inc"
}

__global__ void __launch_bounds__(128)
k_normals_from_lists_batch(const NormalsCloud* __restrict__ clouds, const long long* __restrict__ offsets, int n_clouds,
                           const float4* __restrict__ q, size_t nq, int k, const int32_t* __restrict__ lists,
                           float4* __restrict__ out)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  const NormalsCloud& Q = clouds[problem_of(offsets, n_clouds, (long long)i)];
  const float4* __restrict__ pts = Q.tree.pts;
  const int32_t* __restrict__ pos_of_orig = Q.pos_of_orig;
  const float vpx = Q.vp[0], vpy = Q.vp[1], vpz = Q.vp[2];
  int* const not_dense = Q.not_dense;
  const size_t slot0 = 0;
#include "normals_from_lists_body.inc"
}

}  // namespace pclb200
