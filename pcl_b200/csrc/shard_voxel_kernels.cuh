// shard_voxel_kernels.cuh — the device side of VoxelGrid over a map sharded across ranks (driver: shard_voxel.cu, called
// by pclb200_voxelgrid_sharded).  Every rank holds some records of the map under the caller's ids; the grid is the one of
// the union of every rank's box (voxel_grid.cuh: vg_grid, from one u64 minimum of the ranks' box keys).
//   k_sv_ranges   per rank s, the voxel coordinates of its box's faces: I_s, which holds the voxel of every record of s
//                 (vg_ijk is non-decreasing on each axis)
//   k_sv_select   per finite record and per rank s: its voxel inside I_s?  Counts (dst == nullptr) or writes the record
//                 (a float4 whose w is its id, then its two normal / curvature float4s when normals travel) to the rank's
//                 segment; every finite record also goes to this rank itself
//   k_sv_keys     per record of the local array (own records, then the received ones by sender): the 64-bit key
//                 (voxel << 32) | id, its position, the rank it came from; with normals, the points and the normal planes
//                 split out of the records for k_vg_centroids / k_vg_normals
//   k_sv_heads    run heads of the voxels of sorted keys
//   k_sv_holders  per voxel run of the sorted keys (duplicate ids included): the mask of the ranks that hold a record of it
//   k_sv_own      per voxel run of the deduplicated keys: kept when this rank holds a record of it, is its owner (sv_owner)
//                 and the run has min_pts records; its linear index
// The segments travel through comm_segment_tables and are read back with k_gather_segments (peer_tables.cuh).  A header
// of its own so that tests/host/shard_voxel_host_test.cpp can compile the kernels for the host and simulate several ranks.
#pragma once
#include "internal.cuh"
#include "voxel_grid.cuh"

namespace pclb200 {

// The first exchange of pclb200_voxelgrid_sharded: one u64 minimum over kSvHeadWords + kSvBoxWords * R words, every rank
// writing its own verdict, its parameters (p and ~p: the minimum of both says whether the ranks agree) and its box at
// kSvHeadWords + kSvBoxWords * rank, every other word ~0.  Box keys: lo_a as the order-preserving u32 of its float,
// hi_a as 0xffffffff minus that, so that both fold with a u64 minimum; every word ~0 = no finite record.
enum { kSvVerdict = 0, kSvParams = 1, kSvNotParams = 4, kSvHeadWords = 7 };
constexpr int kSvBoxWords = 6;
// Bits of the local sort key (voxel << 32) | id that the sort compares: all of them.  The voxel index can reach 2^31 and
// beyond (the guard bounds int(extent / leaf) + 1 per axis, div_b can be one more), so its top bit counts too.
constexpr int kSvKeyBits = 64;
constexpr unsigned long long kSvNoBox = ~0ull;

// order-preserving u32 of a float (-0 < +0) from the ordered int of k_vg_minmax, and back
inline unsigned long long sv_box_key(int ord) { return (unsigned)ord ^ 0x80000000u; }
inline float sv_key_value(unsigned long long key) { return vord2f((int)((unsigned)key ^ 0x80000000u)); }

// this rank's box keys (kSvBoxWords) from the min / max of k_vg_minmax over its records
inline void sv_fold_box(const MinMaxAcc& acc, unsigned long long* w)
{
  for (int a = 0; a < 3; ++a) {
    w[a] = acc.count ? sv_box_key(acc.lo[a]) : kSvNoBox;
    w[3 + a] = acc.count ? 0xffffffffull - sv_box_key(acc.hi[a]) : kSvNoBox;
  }
}
// the box of keys w (false: no finite record)
inline bool sv_box(const unsigned long long* w, float lo[3], float hi[3])
{
  if (w[0] == kSvNoBox)
    return false;
  for (int a = 0; a < 3; ++a) {
    lo[a] = sv_key_value(w[a]);
    hi[a] = sv_key_value(0xffffffffull - w[3 + a]);
  }
  return true;
}

// The owner of voxel v among the ranks of mask (bit r = rank r holds a record of v): member v mod |mask| in rank order,
// so that the voxels shared by several ranks spread over them.
__host__ __device__ inline int sv_owner(unsigned v, unsigned mask)
{
  unsigned n = 0;
  for (int r = 0; r < kMaxRanks; ++r)
    n += (mask >> r) & 1u;
  unsigned k = v % n;
  for (int r = 0; r < kMaxRanks; ++r)
    if ((mask >> r) & 1u) {
      if (k == 0)
        return r;
      --k;
    }
  return -1;
}

// every rank's box, as read back from the first exchange (sv_box)
struct SvBoxes {
  int n;
  bool any[kMaxRanks];  // false: the rank has no finite record
  float lo[kMaxRanks][3], hi[kMaxRanks][3];
};
// I_s of every rank s: lo[s][a] .. hi[s][a] (lo > hi: the rank has no finite record)
struct SvRanges {
  int lo[kMaxRanks][3];
  int hi[kMaxRanks][3];
};

// One thread per rank: the voxel coordinates of its box's faces.
__global__ void k_sv_ranges(SvBoxes b, VgParams g, SvRanges* __restrict__ out)
{
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= b.n)
    return;
  for (int a = 0; a < 3; ++a) {
    out->lo[s][a] = b.any[s] ? vg_ijk(b.lo[s][a], g.inv[a], g.min_b[a]) : 1;
    out->hi[s][a] = b.any[s] ? vg_ijk(b.hi[s][a], g.inv[a], g.min_b[a]) : 0;
  }
}

// Where k_sv_select sends the records: per rank a cursor (counts when dst is null) and a destination segment of float4s,
// sv_units(normals) per record.
struct SvOut {
  unsigned long long* count;  // [nranks]: records sent to each rank (atomically advanced)
  float4* dst[kMaxRanks];     // nullptr: count only
};
__host__ __device__ inline int sv_units(bool normals) { return normals ? 3 : 1; }

// p: this rank's records (xyz, w ignored), ids: their ids, nc (nullable): their normal planes (k_vg_load_nc's layout).
// Launched with a multiple of 32 threads per block; a warp advances each cursor once per step.
__global__ void __launch_bounds__(256)
k_sv_select(const float4* __restrict__ p, const int32_t* __restrict__ ids, const float4* __restrict__ nc, size_t n,
            VgParams g, const SvRanges* __restrict__ rg, int nranks, int self, SvOut out)
{
  const unsigned lane = threadIdx.x & 31;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const int per = sv_units(nc != nullptr);
  for (size_t base = blockIdx.x * (size_t)blockDim.x + (threadIdx.x & ~31u); base < n; base += stride) {
    const size_t j = base + lane;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    bool real = false;
    int ijk[3] = {0, 0, 0};
    if (j < n) {
      v = p[j];
      real = isfinite(v.x) && isfinite(v.y) && isfinite(v.z);
      if (real) {
        ijk[0] = vg_ijk(v.x, g.inv[0], g.min_b[0]);
        ijk[1] = vg_ijk(v.y, g.inv[1], g.min_b[1]);
        ijk[2] = vg_ijk(v.z, g.inv[2], g.min_b[2]);
      }
    }
    for (int r = 0; r < nranks; ++r) {
      bool in = real;
      if (in && r != self)
        for (int a = 0; a < 3; ++a)
          in = in && ijk[a] >= rg->lo[r][a] && ijk[a] <= rg->hi[r][a];
      const unsigned m = __ballot_sync(0xffffffffu, in);
      if (!m)
        continue;
      unsigned long long at = 0;
      if (lane == 0)
        at = atomicAdd(out.count + r, (unsigned long long)__popc(m));
      at = __shfl_sync(0xffffffffu, at, 0);
      if (in && out.dst[r]) {
        float4* d = out.dst[r] + (at + __popc(m & ((1u << lane) - 1u))) * per;
        d[0] = make_float4(v.x, v.y, v.z, __int_as_float(ids[j]));
        if (nc) {
          d[1] = nc[2 * j];
          d[2] = nc[2 * j + 1];
        }
      }
    }
  }
}

// The senders of the local array: records [begin[t], begin[t + 1]) came from rank[t] (t = 0: this rank's own).
struct SvSenders {
  int n;
  int rank[kMaxRanks];
  unsigned long long begin[kMaxRanks + 1];
};

// local: n records of sv_units(nc != nullptr) float4s.  keys[i] = (voxel << 32) | id, vals[i] = i, holder[i] = the rank
// record i came from; with normals, pts[i] = its point and nc[2 i], nc[2 i + 1] = its normal planes.
__global__ void __launch_bounds__(256)
k_sv_keys(const float4* __restrict__ local, size_t n, VgParams g, SvSenders s, unsigned long long* __restrict__ keys,
          int32_t* __restrict__ vals, unsigned char* __restrict__ holder, float4* __restrict__ pts, float4* __restrict__ nc)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const int per = sv_units(nc != nullptr);
  const float4 v = local[i * per];
  const unsigned vox =
      vg_linear(vg_ijk(v.x, g.inv[0], g.min_b[0]), vg_ijk(v.y, g.inv[1], g.min_b[1]), vg_ijk(v.z, g.inv[2], g.min_b[2]), g);
  keys[i] = ((unsigned long long)vox << 32) | (unsigned)__float_as_int(v.w);
  vals[i] = (int32_t)i;
  int t = 0;
  while (i >= s.begin[t + 1])
    ++t;
  holder[i] = (unsigned char)s.rank[t];
  if (nc) {
    pts[i] = v;
    nc[2 * i] = local[i * per + 1];
    nc[2 * i + 1] = local[i * per + 2];
  }
}

// head[j] = sorted key j starts a voxel
__global__ void k_sv_heads(const unsigned long long* __restrict__ keys, size_t n, unsigned char* __restrict__ head)
{
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j < n)
    head[j] = (j == 0 || (keys[j] >> 32) != (keys[j - 1] >> 32)) ? 1 : 0;
}

// mask[m] = the ranks holding a record of voxel run m of the sorted keys (runs start at starts[], n entries in all)
__global__ void k_sv_holders(const unsigned* __restrict__ starts, size_t n_runs, size_t n, const int32_t* __restrict__ vals,
                             const unsigned char* __restrict__ holder, unsigned char* __restrict__ mask)
{
  const size_t m = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (m >= n_runs)
    return;
  const size_t b = starts[m], e = (m + 1 < n_runs) ? starts[m + 1] : n;
  unsigned acc = 0;
  for (size_t j = b; j < e; ++j)
    acc |= 1u << holder[vals[j]];
  mask[m] = (unsigned char)acc;
}

// keep[m]: voxel run m (over the deduplicated keys ukeys) is this rank's to return; voxel[m] = its linear index.  mask[m]
// is the holder mask of the same voxel (the runs of the sorted and of the deduplicated keys are the same voxels in the
// same order).
__global__ void k_sv_own(const RunRef* __restrict__ runs, const unsigned long long* __restrict__ ukeys,
                         const unsigned char* __restrict__ mask, size_t n_runs, int self, unsigned min_pts,
                         unsigned char* __restrict__ keep, unsigned* __restrict__ voxel)
{
  const size_t m = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (m >= n_runs)
    return;
  const RunRef r = runs[m];
  const unsigned v = (unsigned)(ukeys[r.begin] >> 32);
  const unsigned mk = mask[m];
  voxel[m] = v;
  keep[m] = (((mk >> self) & 1u) && sv_owner(v, mk) == self && r.end - r.begin >= min_pts) ? 1 : 0;
}

}  // namespace pclb200
