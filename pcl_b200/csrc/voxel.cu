// voxel.cu — pcl::VoxelGrid<PointT>::applyFilter on the device (downsample front-end of configs 2 and 5).
//
// Reference: filters/include/pcl/filters/impl/voxel_grid.hpp:596-814
//   getMinMax3D (:617) -> int32 overflow guard (:620-629) -> min_b/max_b/div_b/divb_mul (:632-644)
//   -> per point ijk = floor(p*inv_leaf) - min_b, idx = ijk . divb_mul (:705-719)
//   -> sort by idx (:724-725) -> runs of equal idx, drop runs < min_points_per_voxel (:737-748)
//   -> per run centroid = float sum / count (:779-812, accumulators.hpp:68-85)
// The reference sorts with an UNSTABLE spreadsort, so its within-voxel summation order is unspecified;
// here (and in the oracle) the sort is stable => the order is ascending position in `indices`, and one
// thread sums its voxel's points in that order, so device and oracle agree bit for bit.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <limits>

#include "internal.cuh"
#include "voxel_kernels.cuh"

namespace pclb200 {

struct IsSet {
  __host__ __device__ bool operator()(unsigned char v) const { return v != 0; }
};

size_t voxelgrid(Ctx& c, const void* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int is_dense,
                 const float leaf[3], unsigned min_pts, float* out_xyz1, const void* normals, size_t stride_n,
                 float* out_normal_curv, const float* grid_bounds)
{
  (void)is_dense;  // non-finite points are skipped on either setting (a dense cloud has none)
  cudaStream_t st = c.stream;
  const size_t cnt = indices ? n_idx : n;
  if (cnt == 0)
    return 0;
  PCLB_REQUIRE(leaf[0] > 0 && leaf[1] > 0 && leaf[2] > 0, PCLB200_ERR_INVALID, "leaf size must be positive");
  DevBuf<float4> dense;
  dense.alloc(cnt, st);
  load_xyz_as_float4(c, pts, n, stride, indices, n_idx, dense.p, st);
  // pass 1: min/max
  DevBuf<MinMaxAcc> acc;
  acc.alloc(1, st);
  MinMaxAcc init;
  for (int d = 0; d < 3; ++d) {
    init.lo[d] = 0x7fffffff;
    init.hi[d] = (int)0x80000000;
  }
  init.count = 0;
  PCLB_CUDA(cudaMemcpyAsync(acc.p, &init, sizeof(init), cudaMemcpyHostToDevice, st));
  unsigned g = (unsigned)std::min<size_t>((cnt + 255) / 256, (size_t)c.sm_count * 8);
  k_vg_minmax<<<g, 256, 0, st>>>(dense.p, cnt, acc.p);
  ++c.launches;
  MinMaxAcc h;
  PCLB_CUDA(cudaMemcpyAsync(&h, acc.p, sizeof(h), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  const size_t n_valid = (size_t)h.count;
  if (n_valid == 0)
    return 0;
  float mn[3], mx[3], inv[3];
  for (int d = 0; d < 3; ++d) {
    mn[d] = vord2f(h.lo[d]);
    mx[d] = vord2f(h.hi[d]);
    inv[d] = 1.0f / leaf[d];  // inverse_leaf_size_ = 1 / leaf_size_ (voxel_grid.h:266,282)
  }
  if (grid_bounds) {
    // a spatial tile of a larger cloud: the grid (min_b, div_b) is the WHOLE cloud's, so that the tiles' voxels are the
    // voxels a single VoxelGrid over the whole cloud would form (the caller cuts tiles along voxel boundaries)
    for (int d = 0; d < 3; ++d) {
      PCLB_REQUIRE(grid_bounds[d] <= mn[d] && grid_bounds[3 + d] >= mx[d], PCLB200_ERR_INVALID,
                   "voxelgrid: the given grid bounds do not contain the points");
      mn[d] = grid_bounds[d];
      mx[d] = grid_bounds[3 + d];
    }
  }
  // guard, in the reference's float arithmetic (voxel_grid.hpp:620-629)
  volatile float e0 = (mx[0] - mn[0]) * inv[0], e1 = (mx[1] - mn[1]) * inv[1], e2 = (mx[2] - mn[2]) * inv[2];
  const int64_t dx = (int64_t)e0 + 1, dy = (int64_t)e1 + 1, dz = (int64_t)e2 + 1;
  if (dx * dy * dz > (int64_t)std::numeric_limits<int32_t>::max())
    throw Error(PCLB200_ERR_LEAF_TOO_SMALL,
                "VoxelGrid: leaf size is too small for the input dataset, integer indices would overflow "
                "(voxel_grid.hpp:620-629)");
  VgParams gp;
  int max_b[3], div_b[3];
  for (int d = 0; d < 3; ++d) {
    volatile float lo_s = mn[d] * inv[d], hi_s = mx[d] * inv[d];
    gp.inv[d] = inv[d];
    gp.min_b[d] = (int)std::floor(lo_s);
    max_b[d] = (int)std::floor(hi_s);
    div_b[d] = max_b[d] - gp.min_b[d] + 1;
  }
  gp.mul[0] = 1;
  gp.mul[1] = div_b[0];
  gp.mul[2] = div_b[0] * div_b[1];
  // pass 2: keys ; pass 3: stable radix sort
  DevBuf<unsigned> keys_in, keys;
  DevBuf<int32_t> vals_in, vals;
  keys_in.alloc(cnt, st);
  keys.alloc(cnt, st);
  vals_in.alloc(cnt, st);
  vals.alloc(cnt, st);
  k_vg_keys<<<grid_for(cnt, 256), 256, 0, st>>>(dense.p, cnt, gp, keys_in.p, vals_in.p);
  ++c.launches;
  size_t tmp_bytes = 0;
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys_in.p, keys.p, vals_in.p, vals.p, (int)cnt, 0, 32, st));
  DevBuf<unsigned char> tmp;
  tmp.alloc(tmp_bytes, st);
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, keys_in.p, keys.p, vals_in.p, vals.p, (int)cnt, 0, 32, st));
  c.launches += 5;
  // pass 4: run starts
  DevBuf<unsigned char> head;
  head.alloc(n_valid, st);
  k_vg_heads<<<grid_for(n_valid, 256), 256, 0, st>>>(keys.p, n_valid, head.p);
  ++c.launches;
  DevBuf<unsigned> starts;
  DevBuf<size_t> d_num;
  starts.alloc(n_valid, st);
  d_num.alloc(1, st);
  cub::CountingInputIterator<unsigned> counting(0);
  size_t tb2 = 0;
  PCLB_CUDA(cub::DeviceSelect::Flagged(nullptr, tb2, counting, head.p, starts.p, d_num.p, (int)n_valid, st));
  DevBuf<unsigned char> tmp2;
  tmp2.alloc(tb2, st);
  PCLB_CUDA(cub::DeviceSelect::Flagged(tmp2.p, tb2, counting, head.p, starts.p, d_num.p, (int)n_valid, st));
  c.launches += 2;
  size_t n_runs = 0;
  PCLB_CUDA(cudaMemcpyAsync(&n_runs, d_num.p, sizeof(size_t), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  DevBuf<RunRef> runs_all, runs;
  runs_all.alloc(n_runs, st);
  k_vg_runs<<<grid_for(n_runs, 256), 256, 0, st>>>(starts.p, n_runs, n_valid, runs_all.p);
  ++c.launches;
  size_t n_out = n_runs;
  const RunRef* d_runs = runs_all.p;
  if (min_pts > 1) {
    DevBuf<unsigned char> keep;
    keep.alloc(n_runs, st);
    k_vg_keep<<<grid_for(n_runs, 256), 256, 0, st>>>(starts.p, n_runs, n_valid, min_pts, keep.p);
    runs.alloc(n_runs, st);
    size_t tb3 = 0;
    PCLB_CUDA(cub::DeviceSelect::Flagged(nullptr, tb3, runs_all.p, keep.p, runs.p, d_num.p, (int)n_runs, st));
    DevBuf<unsigned char> tmp3;
    tmp3.alloc(tb3, st);
    PCLB_CUDA(cub::DeviceSelect::Flagged(tmp3.p, tb3, runs_all.p, keep.p, runs.p, d_num.p, (int)n_runs, st));
    c.launches += 3;
    PCLB_CUDA(cudaMemcpyAsync(&n_out, d_num.p, sizeof(size_t), cudaMemcpyDeviceToHost, st));
    PCLB_CUDA(cudaStreamSynchronize(st));
    d_runs = runs.p;
  }
  if (n_out == 0)
    return 0;
  // pass 5: centroids
  DevBuf<float4> out;
  float4* const caller_out = reinterpret_cast<float4*>(out_xyz1);
  k_vg_centroids<<<grid_for(n_out, 128), 128, 0, st>>>(dense.p, vals.p, d_runs, n_out, out_on_device(c, caller_out, n_out, out));
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  copy_out(c, caller_out, out, n_out);
  if (normals && out_normal_curv) {
    // the remaining fields of a PointNormal / Normal record, averaged over the same runs in the same order
    PCLB_REQUIRE(stride_n >= 20 && stride_n % 4 == 0, PCLB200_ERR_INVALID, "normal stride must be a multiple of 4 and >= 20");
    // the upload stops at the last byte of the last record's fields (as in strided_to_float4)
    DevBuf<unsigned char> staged;
    DevBuf<int32_t> staged_sub;
    const unsigned char* d_src = on_device(c, static_cast<const unsigned char*>(normals), (n - 1) * stride_n + 20, staged);
    const int32_t* d_sub = on_device(c, indices, n_idx, staged_sub);
    DevBuf<float4> nc, nout;
    nc.alloc(2 * cnt, st);
    k_vg_load_nc<<<grid_for(cnt, 256), 256, 0, st>>>(d_src, stride_n, d_sub, cnt, nc.p);
    float4* const caller_nout = reinterpret_cast<float4*>(out_normal_curv);
    k_vg_normals<<<grid_for(n_out, 128), 128, 0, st>>>(nc.p, vals.p, d_runs, n_out,
                                                       out_on_device(c, caller_nout, 2 * n_out, nout));
    c.launches += 2;
    PCLB_CUDA(cudaGetLastError());
    copy_out(c, caller_nout, nout, 2 * n_out);
    PCLB_CUDA(cudaStreamSynchronize(st));
    return n_out;
  }
  PCLB_CUDA(cudaStreamSynchronize(st));
  return n_out;
}

}  // namespace pclb200
