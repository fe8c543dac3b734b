// shard_filter_kernels.cuh — the device side of k-NN queries and the two outlier filters over a map sharded across ranks
// (driver: shard_filter.cu, called by pclb200_knn_sharded, pclb200_knn_stats_sharded, pclb200_statistical_outlier_sharded
// and pclb200_radius_outlier_sharded).  The searches run unchanged on the rank's local map (shard_normals.cu:
// sharded_local_map), whose records are its ids in ascending order; what is new is
//   k_sf_row_ids       the local map's record numbers of k-NN rows -> the whole map's ids (padding -1 stays)
//   k_sf_tile_ids      the ids of a tile's indexed points (the count of distinct ids behind k_eff on a small map)
//   k_sf_sor_partials  this rank's (valid, sum d, sum d*d) over its queries in slot order, a fixed-order grid sum, written
//                      as u64 bit patterns into this rank's exchange table
//   k_sf_sor_fold      every rank's partials folded in rank order -> (valid, mean, thr), the same on every rank
//   k_sf_sor_mask      StatisticalOutlierRemoval's rule (statistical_outlier_removal.hpp:100-135)
//   k_sf_ror_mask      RadiusOutlierRemoval's rule (radius_outlier_removal.hpp:86-150)
// A header of its own so that tests/host/shard_filter_host_test.cpp can compile the kernels for the host and simulate
// several ranks.
#pragma once
#include "grid_sum.cuh"
#include "peer_tables.cuh"

namespace pclb200 {

constexpr int kSorWords = 3;  // per rank: number of finite queries, sum of the means, sum of their float squares

// out[i] >= 0 is a record of the local map, whose records are its ids in ascending order: local_ids[out[i]] is the id
__global__ void __launch_bounds__(256)
k_sf_row_ids(int32_t* __restrict__ out, size_t n, const unsigned* __restrict__ local_ids)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int32_t r = out[i];
    if (r >= 0)
      out[i] = (int32_t)local_ids[r];
  }
}

// the id of every slot of a labelled index's Morton array (padding: kSentinelIndex) as u64
__global__ void __launch_bounds__(256)
k_sf_tile_ids(const float4* __restrict__ pts, size_t n, unsigned long long* __restrict__ ids)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    ids[i] = (unsigned)__float_as_int(pts[i].w);
}

// StatisticalOutlierRemoval's sums over this rank's queries: valid counts the finite ones, and every mean (0 for a
// non-finite query) adds d and float(d * d), as the reference's loop does.  The last block writes the three totals' bit
// patterns into table[0..3) (this rank's exchange table).  Launched with 256 threads per block.
__global__ void __launch_bounds__(256)
k_sf_sor_partials(const float4* __restrict__ q, const float* __restrict__ mean, size_t nq, GridSum g,
                  unsigned long long* __restrict__ table)
{
  double acc[kSorWords] = {0.0, 0.0, 0.0};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nq; i += (size_t)gridDim.x * blockDim.x) {
    const float4 p = q[i];
    const float d = mean[i];
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z))
      acc[0] += 1.0;
    acc[1] += (double)d;
    acc[2] += (double)__fmul_rn(d, d);
  }
  if (block_reduce_and_publish<kSorWords>(acc, g) && threadIdx.x < kSorWords)
    table[threadIdx.x] = (unsigned long long)__double_as_longlong(g.accum[threadIdx.x]);
}

// The partials of every rank (parts.t[s][0..3), read through to memory) folded in rank order, then the reference's
// arithmetic (statistical_outlier_removal.hpp:108-112; no fused multiply-add): stats = {valid, mean, thr}.  One thread.
__global__ void k_sf_sor_fold(const __grid_constant__ PeerTableSet<unsigned long long> parts, double std_mul, double* __restrict__ stats)
{
  if (blockIdx.x != 0 || threadIdx.x != 0)
    return;
  double s[kSorWords] = {0.0, 0.0, 0.0};
  for (int r = 0; r < parts.n; ++r)
    for (int w = 0; w < kSorWords; ++w)
      s[w] = __dadd_rn(s[w], __longlong_as_double((long long)__ldcv(parts.t[r] + w)));
  const double valid = s[0], sum = s[1], sq_sum = s[2];
  const double mean = sum / valid;
  const double variance = (sq_sum - __dmul_rn(sum, sum) / valid) / (valid - 1.0);
  stats[0] = valid;
  stats[1] = mean;
  stats[2] = __dadd_rn(mean, __dmul_rn(std_mul, sqrt(variance)));
}

// keep[i] = 0 when the query's mean distance is above thr (negative: at most thr)
__global__ void __launch_bounds__(256)
k_sf_sor_mask(const float* __restrict__ mean, size_t nq, const double* __restrict__ stats, int negative,
              unsigned char* __restrict__ keep)
{
  const double thr = stats[2];
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nq; i += (size_t)gridDim.x * blockDim.x) {
    const double d = (double)mean[i];
    const bool removed = negative ? d <= thr : d > thr;
    keep[i] = removed ? 0 : 1;
  }
}

// RadiusOutlierRemoval on the squared distance of neighbour min_pts (kth, +inf when the map holds fewer points).  *dense
// (every rank's is_dense, folded with a u64 minimum) selects the rule: dense, the k-NN rule against nn_dists_max = r * r in
// double; else the radius rule, d2 < float(r * r) strictly, and a non-finite query is removed.
__global__ void __launch_bounds__(256)
k_sf_ror_mask(const float4* __restrict__ q, const float* __restrict__ kth, size_t nq,
              const unsigned long long* __restrict__ dense, double nn_dists_max, float r2f, int negative,
              unsigned char* __restrict__ keep)
{
  const bool is_dense = *dense != 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nq; i += (size_t)gridDim.x * blockDim.x) {
    const float d2 = kth[i];
    bool k = true;
    if (is_dense) {
      if (isfinite(d2))
        k = negative ? !(nn_dists_max >= (double)d2) : !(nn_dists_max < (double)d2);
      else
        k = negative != 0;
    }
    else {
      const float4 p = q[i];
      if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z)))
        k = false;
      else {
        const bool enough = d2 < r2f;
        k = negative ? !enough : enough;
      }
    }
    keep[i] = k ? 1 : 0;
  }
}

}  // namespace pclb200
