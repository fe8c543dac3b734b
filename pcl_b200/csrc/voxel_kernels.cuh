// voxel_kernels.cuh — the device side of VoxelGrid::applyFilter: min / max, voxel keys in the reference's float arithmetic,
// run heads, runs, the minimum-points filter, centroids in input order, and the normal / curvature planes of a PointNormal.
// A header so that voxel.cu stays the host-side driver (CUB sort / select between the kernels) and
// tests/host/voxel_host_test.cpp can compile the SAME kernels for the host and compare with the oracle bit for bit.
#pragma once
#include "voxel_grid.cuh"

namespace pclb200 {

__global__ void k_vg_minmax(const float4* __restrict__ p, size_t n, MinMaxAcc* acc)
{
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  unsigned cnt = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float4 v = __ldg(p + i);
    if (isfinite(v.x) && isfinite(v.y) && isfinite(v.z)) {
      lo[0] = fminf(lo[0], v.x); hi[0] = fmaxf(hi[0], v.x);
      lo[1] = fminf(lo[1], v.y); hi[1] = fmaxf(hi[1], v.y);
      lo[2] = fminf(lo[2], v.z); hi[2] = fmaxf(hi[2], v.z);
      ++cnt;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if ((threadIdx.x & 31) == 0 && cnt) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      atomicMin(&acc->lo[d], vf2ord(lo[d]));
      atomicMax(&acc->hi[d], vf2ord(hi[d]));
    }
    atomicAdd(&acc->count, (unsigned long long)cnt);
  }
}

__global__ void k_vg_keys(const float4* __restrict__ p, size_t n, VgParams g, unsigned* __restrict__ keys,
                          int32_t* __restrict__ vals)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  float4 v = __ldg(p + i);
  unsigned key = 0xffffffffu;  // non-finite points sort to the tail and are cut off
  if (isfinite(v.x) && isfinite(v.y) && isfinite(v.z))
    key = vg_linear(vg_ijk(v.x, g.inv[0], g.min_b[0]), vg_ijk(v.y, g.inv[1], g.min_b[1]), vg_ijk(v.z, g.inv[2], g.min_b[2]), g);
  keys[i] = key;
  vals[i] = (int32_t)i;
}

__global__ void k_vg_heads(const unsigned* __restrict__ keys, size_t n, unsigned char* __restrict__ head)
{
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j < n)
    head[j] = (j == 0 || keys[j] != keys[j - 1]) ? 1 : 0;
}

// keep[m] = run m has >= min_pts points
__global__ void k_vg_keep(const unsigned* __restrict__ starts, size_t n_runs, size_t n_valid, unsigned min_pts,
                          unsigned char* __restrict__ keep)
{
  size_t m = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (m >= n_runs)
    return;
  size_t b = starts[m], e = (m + 1 < n_runs) ? starts[m + 1] : n_valid;
  keep[m] = (e - b) >= min_pts ? 1 : 0;
}

__global__ void k_vg_runs(const unsigned* __restrict__ starts, size_t n_runs, size_t n_valid, RunRef* __restrict__ runs)
{
  size_t m = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (m >= n_runs)
    return;
  runs[m].begin = starts[m];
  runs[m].end = (m + 1 < n_runs) ? starts[m + 1] : (unsigned)n_valid;
}

__global__ void k_vg_centroids(const float4* __restrict__ p, const int32_t* __restrict__ vals,
                               const RunRef* __restrict__ runs, size_t n_runs, float4* __restrict__ out)
{
  size_t m = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (m >= n_runs)
    return;
  const RunRef r = runs[m];
  float cx = 0.f, cy = 0.f, cz = 0.f;
  for (unsigned j = r.begin; j < r.end; ++j) {
    const float4 v = __ldg(p + vals[j]);
    cx = __fadd_rn(cx, v.x);
    cy = __fadd_rn(cy, v.y);
    cz = __fadd_rn(cz, v.z);
  }
  const float fn = (float)(r.end - r.begin);
  out[m] = make_float4(__fdiv_rn(cx, fn), __fdiv_rn(cy, fn), __fdiv_rn(cz, fn), 1.0f);
}

// downsample_all_data_ (voxel_grid.hpp:796-806, CentroidPoint): normals are summed as 4-vectors and normalised
// (AccumulatorNormal, accumulators.hpp:86-116), the curvature is averaged (AccumulatorCurvature, :118-133).
// nc: two float4 per selected point {nx,ny,nz,n4} {curvature,-,-,-}; out: two float4 per voxel, same layout
__global__ void k_vg_load_nc(const unsigned char* __restrict__ src, size_t stride, const int32_t* __restrict__ subset,
                             size_t n, float4* __restrict__ out)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const size_t r = subset ? (size_t)subset[i] : i;
  const float* f = reinterpret_cast<const float*>(src + r * stride);
  out[2 * i] = make_float4(f[0], f[1], f[2], f[3]);
  out[2 * i + 1] = make_float4(f[4], 0.f, 0.f, 0.f);
}

__global__ void k_vg_normals(const float4* __restrict__ nc, const int32_t* __restrict__ vals, const RunRef* __restrict__ runs,
                             size_t n_runs, float4* __restrict__ out)
{
  size_t m = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (m >= n_runs)
    return;
  const RunRef r = runs[m];
  float nx = 0.f, ny = 0.f, nz = 0.f, nw = 0.f, cv = 0.f;
  for (unsigned j = r.begin; j < r.end; ++j) {
    const float4 a = __ldg(nc + 2 * (size_t)vals[j]);
    const float4 b = __ldg(nc + 2 * (size_t)vals[j] + 1);
    nx = __fadd_rn(nx, a.x); ny = __fadd_rn(ny, a.y); nz = __fadd_rn(nz, a.z); nw = __fadd_rn(nw, a.w);
    cv = __fadd_rn(cv, b.x);
  }
  const float sq = __fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fadd_rn(__fmul_rn(nz, nz), __fmul_rn(nw, nw)));
  if (sq > 0.f) {  // Eigen's normalized(): the zero vector stays zero
    const float nrm = __fsqrt_rn(sq);
    nx = __fdiv_rn(nx, nrm); ny = __fdiv_rn(ny, nrm); nz = __fdiv_rn(nz, nrm); nw = __fdiv_rn(nw, nrm);
  }
  out[2 * m] = make_float4(nx, ny, nz, nw);
  out[2 * m + 1] = make_float4(__fdiv_rn(cv, (float)(r.end - r.begin)), 0.f, 0.f, 0.f);
}

// ---- a batch of clouds in one call (voxelgrid_batch) ------------------------------------------------------------------
// Cloud c is the records [offsets[c], offsets[c + 1]) of one dense array.  Record i's key is (c << 32) | its voxel's linear
// index in cloud c's own grid, or B << 32 when it is not finite.  One stable sort by key then puts every cloud's voxels in
// its single call's order, one cloud after another, with each voxel's records in ascending record order, and every
// non-finite record at the tail; no run crosses a cloud.  The runs, the minimum-points filter and the reductions are the
// single call's kernels over the whole batch.
__global__ void k_vg_keys_batch(const float4* __restrict__ p, size_t n, const long long* __restrict__ offsets, int n_clouds,
                                const VgParams* __restrict__ grids, unsigned long long* __restrict__ keys,
                                int32_t* __restrict__ vals)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const float4 v = __ldg(p + i);
  unsigned long long key = (unsigned long long)n_clouds << 32;
  if (isfinite(v.x) && isfinite(v.y) && isfinite(v.z)) {
    const int c = problem_of(offsets, n_clouds, (long long)i);
    const VgParams g = grids[c];
    key = ((unsigned long long)c << 32) |
          vg_linear(vg_ijk(v.x, g.inv[0], g.min_b[0]), vg_ijk(v.y, g.inv[1], g.min_b[1]), vg_ijk(v.z, g.inv[2], g.min_b[2]), g);
  }
  keys[i] = key;
  vals[i] = (int32_t)i;
}

__global__ void k_vg_heads_batch(const unsigned long long* __restrict__ keys, size_t n, unsigned char* __restrict__ head)
{
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j < n)
    head[j] = (j == 0 || keys[j] != keys[j - 1]) ? 1 : 0;
}

// out[c], c = 0..B: the first of the *n_runs runs whose cloud is >= c, so that cloud c's rows are [out[c], out[c + 1]).
// Run m starts at sorted position begins[m * step]: step 1 over the run heads, step 2 over RunRef {begin, end}.
__global__ void k_vg_offsets_batch(const unsigned long long* __restrict__ keys, const unsigned* __restrict__ begins,
                                   size_t step, const size_t* __restrict__ n_runs, int n_clouds, long long* __restrict__ out)
{
  const int c = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (c > n_clouds)
    return;
  size_t lo = 0, hi = *n_runs;
  while (lo < hi) {
    const size_t mid = (lo + hi) >> 1;
    if ((keys[begins[mid * step]] >> 32) < (unsigned long long)c)
      lo = mid + 1;
    else
      hi = mid;
  }
  out[c] = (long long)lo;
}

}  // namespace pclb200
