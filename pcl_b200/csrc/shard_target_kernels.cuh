// shard_target_kernels.cuh — the device side of a target map sharded across ranks (drivers: icp.cu, icp_iterate with
// icp_set_target_sharded, and fitness_score_sharded).  Every rank holds one tile of the map, built with caller ids
// (lbvh.cu: build_index_ids), and the whole source.  Each rank searches its tile; per query the nearest neighbour of the
// whole map is the smallest key
//     (d2 bits << 32) | (uint32) id          (~0: no point of the tile within the gate)
// over the ranks — d2 >= 0, so its bit pattern orders like its value, and ties go to the smaller id, the rule of a single
// index over the whole map.  k_shard_publish writes the key and the tile's record of the match into this rank's exchange
// arrays, k_shard_gather picks the winner per query from every rank's arrays (peer-mapped) or from their NCCL reduction,
// and writes the match the accumulate kernels read: {pos = i, d2} against the gathered records.  The stand-alone
// correspondence lists, inliers and validation of a sharded map (icp.cu: correspondences_sharded) reduce the same keys.
// A header of its own so that tests/host/shard_target_host_test.cpp and shard_corr_host_test.cpp can compile the kernels
// for the host and simulate several ranks.
#pragma once
#include "corr_select.cuh"
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

// Step 1 of getFitnessScore and of the correspondence lists over a sharded target: the key of every query's nearest point
// of this tile within the gate (k_corr's walk), by slot.  RECIP (reciprocal lists): key[nq + slot] is the same key when
// the reverse search from that tile point onto the source (s_nodes / s_pts / s_root, every rank's own index of the whole
// source) returns the query's own index, with k_corr<true>'s gate and rule, else kNoShardMatch.  Equal keys name the same
// point, hence the same verdict, so after the minimum over the ranks the pair is reciprocal iff both halves agree.
// match (nullable) receives the tile match by slot, for the record exchange (k_shard_publish).
template <bool RECIP>
__global__ void __launch_bounds__(256)
k_tile_keys(const TreeView T, const float4* __restrict__ q, size_t nq, float gate, const BvhNode* __restrict__ s_nodes,
            const float4* __restrict__ s_pts, int s_root, const int32_t* __restrict__ src_orig,
            unsigned long long* __restrict__ key, Match* __restrict__ match, int* d_error)
{
  bool overflow = false;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nq; i += (size_t)gridDim.x * blockDim.x) {
    const float4 p = __ldg(q + i);
    const int slot = __float_as_int(p.w);
    unsigned long long k = kNoShardMatch, kr = kNoShardMatch;
    Match m{-1, 0.f};
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
      Nearest1 v{p.x, p.y, p.z, gate, kSentinelIndex, -1};
      WalkStats ws{};
      if (!nearest1<false>(T, p.x, p.y, p.z, v, -1, 1.00001f, ws))
        overflow = true;
      if (v.best_pos >= 0) {
        k = shard_key(v.best, v.best_idx);
        m = Match{v.best_pos, v.best};
        if (RECIP) {
          const float4 t = ldg4(T.pts + v.best_pos);
          Nearest1 b{t.x, t.y, t.z, gate, kSentinelIndex, -1};
          if (!traverse(s_nodes, s_pts, s_root, t.x, t.y, t.z, b))
            overflow = true;
          if (b.best_pos >= 0 && b.best_idx == (src_orig ? src_orig[slot] : slot))
            kr = k;
        }
      }
    }
    key[slot] = k;
    if (RECIP)
      key[nq + slot] = kr;
    if (match)
      match[slot] = m;
  }
  if (overflow)
    atomicExch(d_error, kErrStackOverflow);
}

// Step 2 of the correspondence lists: per slot the smallest key over the tables -> the whole map's correspondence of the
// query (k_corr's record: index_query = the caller's index, index_match = the id, distance = d2; index_match = -1 when no
// point of the map lies within the gate, or, reciprocal, when the winning point's reverse search does not return the query)
__global__ void __launch_bounds__(256)
k_keys_to_corr(const __grid_constant__ PeerTableSet<unsigned long long> keys, size_t nq, int recip,
               const int32_t* __restrict__ src_orig, pclb200_corr* __restrict__ by_slot)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  unsigned long long a = kNoShardMatch, b = kNoShardMatch;
  for (int r = 0; r < keys.n; ++r) {
    const unsigned long long ka = __ldcv(keys.t[r] + i);
    a = ka < a ? ka : a;
    if (recip) {
      const unsigned long long kb = __ldcv(keys.t[r] + nq + i);
      b = kb < b ? kb : b;
    }
  }
  pclb200_corr c;
  c.index_query = src_orig ? src_orig[i] : (int)i;
  c.index_match = -1;
  c.distance = 0.f;
  if (a != kNoShardMatch && (!recip || b == a)) {
    c.index_match = (int)(unsigned)a;
    c.distance = __int_as_float((int)(a >> 32));
  }
  by_slot[i] = c;
}

// The gathered records of the correspondences (k_shard_gather's gpts / gnrm by slot) as the rows the estimators read:
// {x, y, z, 1} and {nx, ny, nz, 0}, flagged where the slot holds a correspondence (the order compact_corr_to keeps)
__global__ void __launch_bounds__(256)
k_corr_rows(const pclb200_corr* __restrict__ by_slot, const float4* __restrict__ gpts, const float4* __restrict__ gnrm,
            size_t n, float4* __restrict__ rows, float4* __restrict__ nrows, unsigned char* __restrict__ flag)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const bool on = by_slot[i].index_match >= 0;
  flag[i] = on ? 1 : 0;
  if (!on)
    return;
  if (rows) {
    const float4 p = gpts[i];
    rows[i] = make_float4(p.x, p.y, p.z, 1.f);
  }
  if (nrows) {
    const float4 m = gnrm[i];
    nrows[i] = make_float4(m.x, m.y, m.z, 0.f);
  }
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

// ---- normal shooting / back projection over a sharded map (driver: icp.cu, correspondences_normals_sharded) ----------
// Exactness: launch_knn on a labelled tile returns its k nearest in (d2, id) order, and every member of the whole map's
// k nearest that lies in tile T_r is among T_r's k nearest.  So merging the R rows of a query, dropping equal keys (one id
// held twice), and keeping the first keff gives the row one index of the whole map returns.  Candidates' records never
// move: every rank scores the merged candidates it holds and the others' scores arrive through one u64 minimum.

// a k-NN row entry of this tile -> its key (padding: kNoShardMatch)
__global__ void __launch_bounds__(256)
k_knn_keys(const int32_t* __restrict__ idx, const float* __restrict__ d2, size_t n, unsigned long long* __restrict__ key)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    key[i] = idx[i] < 0 ? kNoShardMatch : shard_key(d2[i], idx[i]);
}

// per query the merge of every rank's row (rows[r] + i keff, ascending) without repeated keys: the first keff
__global__ void __launch_bounds__(256)
k_merge_rows(const __grid_constant__ PeerTableSet<unsigned long long> rows, size_t nq, int keff,
             unsigned long long* __restrict__ merged)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  int head[kMaxRanks];
  for (int r = 0; r < rows.n; ++r)
    head[r] = 0;
  unsigned long long last = kNoShardMatch;
  for (int j = 0; j < keff;) {
    unsigned long long best = kNoShardMatch;
    int w = -1;
    for (int r = 0; r < rows.n; ++r) {
      if (head[r] >= keff)
        continue;
      const unsigned long long k = __ldcv(rows.t[r] + i * (size_t)keff + head[r]);
      if (k < best) {
        best = k;
        w = r;
      }
    }
    if (w < 0) {  // every row exhausted: a non-finite query (its rows are padding)
      for (; j < keff; ++j)
        merged[i * (size_t)keff + j] = kNoShardMatch;
      break;
    }
    ++head[w];
    if (best == last)
      continue;
    merged[i * (size_t)keff + j++] = best;
    last = best;
  }
}

// the position in the tile of id (sorted ids sid[0..n) with their positions spos), or -1 when the tile holds no such id
__device__ __forceinline__ int tile_pos_of(const unsigned* __restrict__ sid, const int* __restrict__ spos, size_t n, unsigned id)
{
  size_t lo = 0, hi = n;
  while (lo < hi) {
    const size_t mid = (lo + hi) / 2;
    if (sid[mid] < id)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo < n && sid[lo] == id ? spos[lo] : -1;
}

// per merged candidate the bit pattern of its score (corr_select.cuh: shooting_score in double, backprojection_score in
// float widened exactly) when this rank holds it, else kNoShardMatch (no score has that pattern: the arithmetic yields
// the canonical NaN).  dense: the queries by slot; src_nrm: the source normals by the caller's index.
__global__ void __launch_bounds__(256)
k_candidate_scores(const unsigned long long* __restrict__ merged, size_t nq, int keff, int kind,
                   const float4* __restrict__ dense, const int32_t* __restrict__ src_orig, const float4* __restrict__ src_nrm,
                   const unsigned* __restrict__ sid, const int* __restrict__ spos, size_t n_sorted,
                   const float4* __restrict__ tile_pts, const float4* __restrict__ tile_nrm, unsigned long long* __restrict__ score)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  const float4 p = dense[i];
  const float4 n = src_nrm[src_orig ? src_orig[i] : (int)i];
  const bool finite = isfinite(p.x) && isfinite(p.y) && isfinite(p.z);
  for (int j = 0; j < keff; ++j) {
    const unsigned long long key = merged[i * (size_t)keff + j];
    unsigned long long s = kNoShardMatch;
    const int pos = finite && key != kNoShardMatch ? tile_pos_of(sid, spos, n_sorted, (unsigned)key) : -1;
    if (pos >= 0) {
      const double v = kind == PCLB200_CORR_NORMAL_SHOOTING
                           ? shooting_score(ldg4(tile_pts + pos), p.x, p.y, p.z, (double)n.x, (double)n.y, (double)n.z)
                           : (double)backprojection_score(__int_as_float((int)(key >> 32)), n.x, n.y, n.z,
                                                          ldg4(tile_nrm + pos));
      s = (unsigned long long)__double_as_longlong(v);
    }
    score[i * (size_t)keff + j] = s;
  }
}

// the choice of select_by_normals over the merged row and the reduced scores (strict <, the first column wins, the gate
// on the minimum) -> the correspondence by slot; match (nullable): this tile's record of the chosen point, for the rows
__global__ void __launch_bounds__(256)
k_select_sharded(const unsigned long long* __restrict__ merged, const __grid_constant__ PeerTableSet<unsigned long long> scores,
                 size_t nq, int keff, int kind, const float4* __restrict__ dense, const int32_t* __restrict__ src_orig,
                 double max_dist, const unsigned* __restrict__ sid, const int* __restrict__ spos, size_t n_sorted,
                 pclb200_corr* __restrict__ by_slot, Match* __restrict__ match)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  const float4 p = dense[i];
  pclb200_corr r;
  r.index_query = src_orig ? src_orig[i] : (int)i;
  r.index_match = -1;
  r.distance = 0.f;
  Match m{-1, 0.f};
  if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
    int min_j = 0;
    bool gated = false;
    double dmin = DBL_MAX;
    float fmin = FLT_MAX;
    for (int j = 0; j < keff; ++j) {
      if (merged[i * (size_t)keff + j] == kNoShardMatch)
        break;
      unsigned long long s = kNoShardMatch;
      for (int t = 0; t < scores.n; ++t) {
        const unsigned long long v = __ldcv(scores.t[t] + i * (size_t)keff + j);
        s = v < s ? v : s;
      }
      const double dist = __longlong_as_double((long long)s);
      if (kind == PCLB200_CORR_NORMAL_SHOOTING) {
        if (dist < dmin) {
          dmin = dist;
          min_j = j;
        }
      }
      else if ((float)dist < fmin) {
        fmin = (float)dist;
        min_j = j;
      }
    }
    gated = kind == PCLB200_CORR_NORMAL_SHOOTING ? dmin > max_dist : (double)fmin > max_dist;
    const unsigned long long key = merged[i * (size_t)keff + min_j];
    if (!gated && key != kNoShardMatch) {
      r.index_match = (int)(unsigned)key;
      r.distance = __int_as_float((int)(key >> 32));
      if (match) {
        const int pos = tile_pos_of(sid, spos, n_sorted, (unsigned)key);
        if (pos >= 0)
          m = Match{pos, r.distance};
      }
    }
  }
  by_slot[i] = r;
  if (match)
    match[i] = m;
}

}  // namespace pclb200
