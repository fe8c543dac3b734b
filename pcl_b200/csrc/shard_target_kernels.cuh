// shard_target_kernels.cuh — the device side of a target map sharded across ranks (drivers: icp.cu, icp_iterate with
// icp_set_target_sharded, and fitness_score_sharded).  Every rank holds one tile of the map, built with caller ids
// (lbvh.cu: build_index_ids), and the whole source.  Each rank searches its tile; per query the nearest neighbour of the
// whole map is the smallest key
//     (d2 bits << 32) | (uint32) id          (~0: no point of the tile within the gate)
// over the ranks — d2 >= 0, so its bit pattern orders like its value, and ties go to the smaller id, the rule of a single
// index over the whole map.  k_shard_publish writes the key and the tile's record of the match into this rank's exchange
// arrays, k_shard_gather picks the winner per query from every rank's arrays (peer-mapped) or from their NCCL reduction,
// and writes the match the accumulate kernels read: {pos = i, d2} against the gathered records.  A header of its own so
// that tests/host/shard_target_host_test.cpp can compile the kernels for the host and simulate several ranks.
#pragma once
#include "icp_kernels.cuh"
#include "peer_tables.cuh"

namespace pclb200 {

constexpr unsigned long long kNoShardMatch = ~0ull;

__device__ __forceinline__ unsigned long long shard_key(float d2, int id)
{
  return ((unsigned long long)(unsigned)__float_as_int(d2) << 32) | (unsigned)id;
}

// one rank's exchange arrays: per query the key and the tile's record of its match (point with w = id; normal)
struct ShardRecords {
  unsigned long long* key;
  float4* pts;
  float4* nrm;  // nullable: the estimator reads no target normal
};

// the arrays a rank reads the winners from: every rank's (peer path, n = nranks) or their reduction (NCCL, n = 1)
struct ShardReadSet {
  int n;
  const unsigned long long* key[kMaxRanks];
  const float4* pts[kMaxRanks];
  const float4* nrm[kMaxRanks];
};

// match[i] of this rank's tile search -> key and record of query i.  Queries without a match write zero records (the
// NCCL path takes the maximum of the records' bit patterns).
__global__ void __launch_bounds__(256)
k_shard_publish(const Match* __restrict__ match, size_t n, const float4* __restrict__ tile_pts,
                const float4* __restrict__ tile_nrm, const LoopCtrl* ctrl, ShardRecords out)
{
  if (ctrl && ctrl->done)
    return;
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const Match m = match[i];
  unsigned long long k = kNoShardMatch;
  float4 p = make_float4(0.f, 0.f, 0.f, 0.f), q = p;
  if (match_accepted(m)) {
    p = tile_pts[m.pos];
    k = shard_key(m.d2, __float_as_int(p.w));
    if (tile_nrm)
      q = tile_nrm[m.pos];
  }
  out.key[i] = k;
  out.pts[i] = p;
  if (out.nrm)
    out.nrm[i] = q;
}

// NCCL path, after the min reduction of the keys (gkey): this rank's records of the queries another rank won become
// zeros, so that the max reduction of the records' bit patterns copies the winner's record exactly
__global__ void __launch_bounds__(256)
k_shard_keep_winners(const unsigned long long* __restrict__ gkey, size_t n, const LoopCtrl* ctrl, ShardRecords mine)
{
  if (ctrl && ctrl->done)
    return;
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n || mine.key[i] == gkey[i])
    return;
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  mine.pts[i] = z;
  if (mine.nrm)
    mine.nrm[i] = z;
}

// per query the smallest key over the read set (equal keys: the lowest rank) -> the global match {pos = i, d2}, with
// kNotAccepted set when no rank matched, and the winner's record in gpts / gnrm
__global__ void __launch_bounds__(256)
k_shard_gather(const ShardReadSet rs, size_t n, const LoopCtrl* ctrl, Match* __restrict__ gmatch, float4* __restrict__ gpts,
               float4* __restrict__ gnrm)
{
  if (ctrl && ctrl->done)
    return;
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  unsigned long long best = kNoShardMatch;
  int w = -1;
  for (int r = 0; r < rs.n; ++r) {
    const unsigned long long k = __ldcv(rs.key[r] + i);
    if (k < best) {
      best = k;
      w = r;
    }
  }
  Match m;
  if (w < 0) {
    m.pos = (int)i | kNotAccepted;
    m.d2 = 0.f;
  }
  else {
    m.pos = (int)i;
    m.d2 = __int_as_float((int)(best >> 32));
    gpts[i] = __ldcv(rs.pts[w] + i);
    if (gnrm)
      gnrm[i] = __ldcv(rs.nrm[w] + i);
  }
  gmatch[i] = m;
}

// getFitnessScore over a sharded target, step 1: the key of every query's nearest point of this tile (no gate), by slot
__global__ void __launch_bounds__(256)
k_fitness_keys(const TreeView T, const float4* __restrict__ q, size_t nq, unsigned long long* __restrict__ key,
               int* d_error)
{
  bool overflow = false;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nq; i += (size_t)gridDim.x * blockDim.x) {
    const float4 p = __ldg(q + i);
    unsigned long long k = kNoShardMatch;
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
      Nearest1 v{p.x, p.y, p.z, __int_as_float(0x7f800000), kSentinelIndex, -1};
      WalkStats ws{};
      if (!nearest1<false>(T, p.x, p.y, p.z, v, -1, 1.00001f, ws))
        overflow = true;
      if (v.best_pos >= 0)
        k = shard_key(v.best, v.best_idx);
    }
    key[__float_as_int(p.w)] = k;
  }
  if (overflow)
    atomicExch(d_error, kErrStackOverflow);
}

// step 2: per slot the smallest key over the tables (every rank's, or their NCCL minimum), then k_fitness's sums (count
// and sum of d2 <= max_range) in slot order: the same value on every rank
__global__ void __launch_bounds__(256)
k_fitness_reduce(const __grid_constant__ PeerTableSet<unsigned long long> keys, size_t n, double max_range, GridSum sum)
{
  double acc[2] = {0.0, 0.0};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    unsigned long long best = kNoShardMatch;
    for (int r = 0; r < keys.n; ++r) {
      const unsigned long long k = __ldcv(keys.t[r] + i);
      best = k < best ? k : best;
    }
    if (best != kNoShardMatch) {
      const float d2 = __int_as_float((int)(best >> 32));
      if ((double)d2 <= max_range) {
        acc[0] += 1.0;
        acc[1] += (double)d2;
      }
    }
  }
  block_reduce_and_publish<2>(acc, sum);
}

}  // namespace pclb200
