// shard_normals_kernels.cuh — the device side of normal estimation over a map sharded across ranks (driver:
// shard_normals.cu, called by pclb200_normals_knn_sharded / _radius_sharded).  Every rank holds one tile of the map,
// indexed with the caller's ids (lbvh.cu: build_index_ids), and its own queries.  Rank r gathers a halo: every point of
// the other tiles that can belong to the whole map's neighbour list of one of its queries.
//   k_halo_box     per finite query q a reach rho_q (the k-th nearest squared distance in the tile, or the radius) ->
//                  the box [q - reach, q + reach] rounded outward, folded into this rank's 6 box keys (u64 minimum)
//   k_halo_select  per tile point and per rank r: inside r's box?  Counts (dst == nullptr) or writes the point, a float4
//                  whose w is its id, to the rank's segment (warp-aggregated cursors: the order inside a segment is free,
//                  the local map is sorted by id afterwards)
//   k_halo_ids     the id of every point (w bits): the sort key of the local map
// The segments travel through comm_segment_tables and are read back with k_gather_segments (peer_tables.cuh).
// A header of its own so that tests/host/shard_normals_host_test.cpp can compile the kernels for the host and simulate
// several ranks.
#pragma once
#include "internal.cuh"

namespace pclb200 {

// Box of rank r in the exchange array: keys[6 r + a] = halo_key(lo_a) and keys[6 r + 3 + a] = 0xffffffff - halo_key(hi_a),
// so that both fold with a u64 minimum; kNoHaloBox (every word) = the rank has no finite query.
constexpr unsigned long long kNoHaloBox = ~0ull;
constexpr int kHaloBoxWords = 6;

// float -> u32 whose unsigned order is the float order (-0 < +0), and back
__device__ __forceinline__ unsigned halo_key(float f)
{
  const unsigned u = (unsigned)__float_as_int(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float halo_key_value(unsigned k)
{
  const unsigned u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __int_as_float((int)u);
}

// Half-width of a query's box for a reach of rho2 (squared, fp32): every p whose canonical d2 (traverse.cuh: dist2_rn,
// fp32 round-to-nearest, possibly flushing tiny differences and squares to zero) is <= rho2 has |p_a - q_a| <= the
// returned value on each axis.  d2 >= fl(dx * dx) (every term is >= 0 and rounding is monotone), fl(dx * dx) <= rho2 gives
// |fl(dx)| <= rho (1 + 2^-23) unless dx * dx underflows (|fl(dx)| < 2^-63), and |dx| <= |fl(dx)| (1 + 2^-23) unless the
// difference itself flushes (|dx| < 2^-126).  sqrt, scale and the 2^-60 floor all round up: rho (1 + 2^-20) + 2^-60 covers
// both bounds.  +inf stays +inf (a tile with fewer than k points bounds nothing).
__device__ __forceinline__ float halo_reach(float rho2)
{
  return __fadd_ru(__fmul_ru(__fsqrt_ru(rho2), 1.00000095367431640625f), 8.67361737988403547e-19f /* 2^-60 */);
}

// is p inside the box of keys[0..6)?  (p finite; an empty box holds nothing)
__device__ __forceinline__ bool in_halo_box(const unsigned long long* __restrict__ keys, const float4& p)
{
  if (keys[0] == kNoHaloBox)
    return false;
  const float v[3] = {p.x, p.y, p.z};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float lo = halo_key_value((unsigned)keys[a]);
    const float hi = halo_key_value((unsigned)(0xffffffffull - keys[3 + a]));
    if (!(v[a] >= lo && v[a] <= hi))
      return false;
  }
  return true;
}

// The box of the finite queries q[0..nq), each widened by halo_reach(rho2[i]) (rho2 == nullptr: r2 for every query),
// lower faces rounded down and upper faces up, folded into box[0..6) (initially kNoHaloBox) with a u64 minimum.
// Launched with a multiple of 32 threads per block.
__global__ void __launch_bounds__(256)
k_halo_box(const float4* __restrict__ q, const float* __restrict__ rho2, float r2, size_t nq,
           unsigned long long* __restrict__ box)
{
  unsigned long long acc[kHaloBoxWords];
#pragma unroll
  for (int a = 0; a < kHaloBoxWords; ++a)
    acc[a] = kNoHaloBox;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nq; i += (size_t)gridDim.x * blockDim.x) {
    const float4 p = q[i];
    if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z)))
      continue;
    const float h = halo_reach(rho2 ? rho2[i] : r2);
    const float v[3] = {p.x, p.y, p.z};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const unsigned long long lo = halo_key(__fsub_rd(v[a], h));
      const unsigned long long hi = 0xffffffffull - halo_key(__fadd_ru(v[a], h));
      acc[a] = lo < acc[a] ? lo : acc[a];
      acc[3 + a] = hi < acc[3 + a] ? hi : acc[3 + a];
    }
  }
#pragma unroll
  for (int a = 0; a < kHaloBoxWords; ++a) {
    unsigned long long m = acc[a];
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long x = __shfl_xor_sync(0xffffffffu, m, o);
      m = x < m ? x : m;
    }
    if ((threadIdx.x & 31) == 0 && m != kNoHaloBox)
      atomicMin(box + a, m);
  }
}

// Where k_halo_select sends the points: per rank a cursor (counts when dst is null) and a destination segment.
struct HaloOut {
  unsigned long long* count;       // [nranks]: points sent to each rank (atomically advanced)
  float4* dst[kMaxRanks];          // nullptr: count only
};

// Every indexed point of this rank's tile (pts: a labelled index's Morton array, padding w = kSentinelIndex) that lies in
// rank r's box goes to rank r; every one goes to this rank (self: the tile part of the local map).  Launched with a
// multiple of 32 threads per block; a warp advances each cursor once per step.
__global__ void __launch_bounds__(256)
k_halo_select(const float4* __restrict__ pts, size_t n, const unsigned long long* __restrict__ boxes, int nranks, int self,
              HaloOut out)
{
  const unsigned lane = threadIdx.x & 31;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t base = blockIdx.x * (size_t)blockDim.x + (threadIdx.x & ~31u); base < n; base += stride) {
    const size_t j = base + lane;
    float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
    bool real = false;
    if (j < n) {
      p = pts[j];
      real = __float_as_int(p.w) != kSentinelIndex;
    }
    for (int r = 0; r < nranks; ++r) {
      const bool in = real && (r == self || in_halo_box(boxes + (size_t)kHaloBoxWords * r, p));
      const unsigned m = __ballot_sync(0xffffffffu, in);
      if (!m)
        continue;
      unsigned long long at = 0;
      if (lane == 0)
        at = atomicAdd(out.count + r, (unsigned long long)__popc(m));
      at = __shfl_sync(0xffffffffu, at, 0);
      if (in && out.dst[r])
        out.dst[r][at + __popc(m & ((1u << lane) - 1u))] = p;
    }
  }
}

// id of every point of the local map (w bits, non-negative): the key it is sorted by
__global__ void __launch_bounds__(256)
k_halo_ids(const float4* __restrict__ pts, size_t n, unsigned* __restrict__ ids)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n)
    ids[i] = (unsigned)__float_as_int(pts[i].w);
}

}  // namespace pclb200
