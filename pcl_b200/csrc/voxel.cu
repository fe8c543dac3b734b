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

MinMaxAcc vg_minmax(Ctx& c, const float4* d_pts, size_t n)
{
  cudaStream_t st = c.stream;
  MinMaxAcc h;
  for (int d = 0; d < 3; ++d) {
    h.lo[d] = 0x7fffffff;
    h.hi[d] = (int)0x80000000;
  }
  h.count = 0;
  if (!n)
    return h;
  DevBuf<MinMaxAcc> acc;
  acc.alloc(1, st);
  PCLB_CUDA(cudaMemcpyAsync(acc.p, &h, sizeof(h), cudaMemcpyHostToDevice, st));
  unsigned g = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)c.sm_count * 8);
  k_vg_minmax<<<g, 256, 0, st>>>(d_pts, n, acc.p);
  ++c.launches;
  PCLB_CUDA(cudaMemcpyAsync(&h, acc.p, sizeof(h), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  return h;
}

void vg_load_normals(Ctx& c, const void* normals, size_t n, size_t stride_n, const int32_t* indices, size_t n_idx,
                     float4* d_nc)
{
  // the remaining fields of a PointNormal / Normal record; the upload stops at the last byte of the last record's fields
  // (as in strided_to_float4).  The staging buffers go back to the stream's cache after the launch: stream-ordered.
  DevBuf<unsigned char> staged;
  DevBuf<int32_t> staged_sub;
  const unsigned char* d_src = on_device(c, static_cast<const unsigned char*>(normals), (n - 1) * stride_n + 20, staged);
  const int32_t* d_sub = on_device(c, indices, n_idx, staged_sub);
  const size_t cnt = indices ? n_idx : n;
  k_vg_load_nc<<<grid_for(cnt, 256), 256, 0, c.stream>>>(d_src, stride_n, d_sub, cnt, d_nc);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

void vg_runs(Ctx& c, const unsigned* starts, size_t n_runs, size_t n_valid, RunRef* runs)
{
  k_vg_runs<<<grid_for(n_runs, 256), 256, 0, c.stream>>>(starts, n_runs, n_valid, runs);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

void vg_reduce(Ctx& c, const float4* pts, const float4* nc, const int32_t* vals, const RunRef* runs, size_t n_runs,
               float4* out, float4* out_nc)
{
  k_vg_centroids<<<grid_for(n_runs, 128), 128, 0, c.stream>>>(pts, vals, runs, n_runs, out);
  ++c.launches;
  if (nc) {
    k_vg_normals<<<grid_for(n_runs, 128), 128, 0, c.stream>>>(nc, vals, runs, n_runs, out_nc);
    ++c.launches;
  }
  PCLB_CUDA(cudaGetLastError());
}

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
  const MinMaxAcc h = vg_minmax(c, dense.p, cnt);
  const size_t n_valid = (size_t)h.count;
  if (n_valid == 0)
    return 0;
  float mn[3], mx[3];
  for (int d = 0; d < 3; ++d) {
    mn[d] = vord2f(h.lo[d]);
    mx[d] = vord2f(h.hi[d]);
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
  VgParams gp;
  if (!vg_grid(mn, mx, leaf, gp))
    throw Error(PCLB200_ERR_LEAF_TOO_SMALL, kVgLeafTooSmall);
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
  vg_runs(c, starts.p, n_runs, n_valid, runs_all.p);
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
  // pass 5: centroids, and with normals the remaining fields averaged over the same runs in the same order
  const bool with_nc = normals && out_normal_curv;
  DevBuf<float4> nc, out, nout;
  if (with_nc) {
    PCLB_REQUIRE(stride_n >= 20 && stride_n % 4 == 0, PCLB200_ERR_INVALID, "normal stride must be a multiple of 4 and >= 20");
    nc.alloc(2 * cnt, st);
    vg_load_normals(c, normals, n, stride_n, indices, n_idx, nc.p);
  }
  float4* const caller_out = reinterpret_cast<float4*>(out_xyz1);
  float4* const caller_nout = reinterpret_cast<float4*>(out_normal_curv);
  vg_reduce(c, dense.p, with_nc ? nc.p : nullptr, vals.p, d_runs, n_out, out_on_device(c, caller_out, n_out, out),
            with_nc ? out_on_device(c, caller_nout, 2 * n_out, nout) : nullptr);
  copy_out(c, caller_out, out, n_out);
  if (with_nc)
    copy_out(c, caller_nout, nout, 2 * n_out);
  PCLB_CUDA(cudaStreamSynchronize(st));
  return n_out;
}

// ---- a batch of clouds in one call ------------------------------------------------------------------------------------
// Cloud k = records [offsets[k], offsets[k + 1]) of pts; its rows are what voxelgrid() makes of it alone.  voxelgrid()'s
// stages in its order, each one launch (or one CUB call) for the whole batch, and the host synchronises as often as one
// single call does: for the boxes, for the run count, for the kept-run count when min_pts > 1, and at the end.  Every
// refusal comes before the first write to an output.
size_t voxelgrid_batch(Ctx& c, const void* pts, size_t n, size_t stride, const int64_t* offsets, int n_clouds,
                       const float leaf[3], unsigned min_pts, const void* normals, size_t stride_n, float* out_xyz1,
                       float* out_normal_curv, int64_t* out_offsets)
{
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(n_clouds >= 1 && n_clouds <= 65536, PCLB200_ERR_INVALID, "voxelgrid_batch: a batch holds 1 to 65536 clouds");
  PCLB_REQUIRE(pts && offsets && leaf && out_xyz1 && out_offsets, PCLB200_ERR_INVALID, "voxelgrid_batch: NULL argument");
  PCLB_REQUIRE(offsets[0] == 0 && offsets[n_clouds] == (int64_t)n, PCLB200_ERR_INVALID,
               "voxelgrid_batch: offsets must run from 0 to n");
  for (int k = 0; k < n_clouds; ++k)
    PCLB_REQUIRE(offsets[k + 1] > offsets[k], PCLB200_ERR_INVALID,
                 "voxelgrid_batch: offsets must increase strictly (every cloud holds a record)");
  PCLB_REQUIRE(n < (size_t)0x7fffffff, PCLB200_ERR_INVALID, "voxelgrid_batch: a batch holds fewer than 2^31 - 1 records");
  PCLB_REQUIRE(stride >= 12 && stride % 4 == 0, PCLB200_ERR_INVALID, "stride must be a multiple of 4 and >= 12");
  PCLB_REQUIRE(leaf[0] > 0 && leaf[1] > 0 && leaf[2] > 0, PCLB200_ERR_INVALID, "leaf size must be positive");
  PCLB_REQUIRE(!normals == !out_normal_curv, PCLB200_ERR_INVALID,
               "voxelgrid_batch: normals and out_normal_curv are both given or both NULL");
  const bool with_nc = normals != nullptr;
  if (with_nc)
    PCLB_REQUIRE(stride_n >= 20 && stride_n % 4 == 0, PCLB200_ERR_INVALID, "normal stride must be a multiple of 4 and >= 20");
  const int B = n_clouds;
  DevBuf<float4> dense;
  dense.alloc(n, st);
  load_xyz_as_float4(c, pts, n, stride, nullptr, 0, dense.p, st);

  // pass 1: every cloud's box (synchronisation 1) -> its grid, or the guard
  std::vector<MinMaxAcc> box(B);
  cloud_boxes(c, dense.p, offsets, B, box.data());
  std::vector<VgParams> grid(B);
  size_t n_valid = 0;
  for (int k = 0; k < B; ++k) {
    n_valid += (size_t)box[k].count;
    if (!box[k].count)
      continue;  // no key uses this cloud's grid
    float mn[3], mx[3];
    for (int d = 0; d < 3; ++d) {
      mn[d] = vord2f(box[k].lo[d]);
      mx[d] = vord2f(box[k].hi[d]);
    }
    if (!vg_grid(mn, mx, leaf, grid[k]))
      throw Error(PCLB200_ERR_LEAF_TOO_SMALL, "voxelgrid_batch: cloud " + std::to_string(k) + ": " + kVgLeafTooSmall);
  }
  std::vector<int64_t> h_off(B + 1, 0);
  if (n_valid == 0) {
    std::copy(h_off.begin(), h_off.end(), out_offsets);
    return 0;
  }
  DevBuf<long long> d_off, d_out_off;
  DevBuf<VgParams> d_grid;
  d_off.alloc(B + 1, st);
  d_out_off.alloc(B + 1, st);
  d_grid.alloc(B, st);
  PCLB_CUDA(cudaMemcpyAsync(d_off.p, offsets, (B + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
  PCLB_CUDA(cudaMemcpyAsync(d_grid.p, grid.data(), B * sizeof(VgParams), cudaMemcpyHostToDevice, st));

  // pass 2: keys (cloud, voxel) ; pass 3: one stable radix sort over the 32 voxel bits and the bits of B
  DevBuf<unsigned long long> keys_in, keys;
  DevBuf<int32_t> vals_in, vals;
  keys_in.alloc(n, st);
  keys.alloc(n, st);
  vals_in.alloc(n, st);
  vals.alloc(n, st);
  k_vg_keys_batch<<<grid_for(n, 256), 256, 0, st>>>(dense.p, n, d_off.p, B, d_grid.p, keys_in.p, vals_in.p);
  ++c.launches;
  int cloud_bits = 0;
  while ((1 << cloud_bits) <= B)
    ++cloud_bits;
  const int end_bit = 32 + cloud_bits;
  size_t tmp_bytes = 0;
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys_in.p, keys.p, vals_in.p, vals.p, (int)n, 0, end_bit, st));
  DevBuf<unsigned char> tmp;
  tmp.alloc(tmp_bytes, st);
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, keys_in.p, keys.p, vals_in.p, vals.p, (int)n, 0, end_bit, st));
  c.launches += 1 + (end_bit + 7) / 8;  // onesweep: histogram + one pass per 8-bit digit

  // pass 4: run starts over the finite records (synchronisation 2: the run count, and the rows of every cloud when every
  // run is kept)
  DevBuf<unsigned char> head;
  head.alloc(n_valid, st);
  k_vg_heads_batch<<<grid_for(n_valid, 256), 256, 0, st>>>(keys.p, n_valid, head.p);
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
  const unsigned off_grid = grid_for((size_t)B + 1, 256);
  if (min_pts <= 1) {
    k_vg_offsets_batch<<<off_grid, 256, 0, st>>>(keys.p, starts.p, 1, d_num.p, B, d_out_off.p);
    ++c.launches;
    PCLB_CUDA(cudaMemcpyAsync(h_off.data(), d_out_off.p, (B + 1) * sizeof(long long), cudaMemcpyDeviceToHost, st));
  }
  size_t n_runs = 0;
  PCLB_CUDA(cudaMemcpyAsync(&n_runs, d_num.p, sizeof(size_t), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  DevBuf<RunRef> runs_all, runs;
  runs_all.alloc(n_runs, st);
  vg_runs(c, starts.p, n_runs, n_valid, runs_all.p);
  size_t n_out = n_runs;
  const RunRef* d_runs = runs_all.p;
  if (min_pts > 1) {  // synchronisation 3: the kept runs and the rows of every cloud
    DevBuf<unsigned char> keep;
    keep.alloc(n_runs, st);
    k_vg_keep<<<grid_for(n_runs, 256), 256, 0, st>>>(starts.p, n_runs, n_valid, min_pts, keep.p);
    runs.alloc(n_runs, st);
    size_t tb3 = 0;
    PCLB_CUDA(cub::DeviceSelect::Flagged(nullptr, tb3, runs_all.p, keep.p, runs.p, d_num.p, (int)n_runs, st));
    DevBuf<unsigned char> tmp3;
    tmp3.alloc(tb3, st);
    PCLB_CUDA(cub::DeviceSelect::Flagged(tmp3.p, tb3, runs_all.p, keep.p, runs.p, d_num.p, (int)n_runs, st));
    static_assert(sizeof(RunRef) == 2 * sizeof(unsigned) && offsetof(RunRef, begin) == 0, "RunRef = {begin, end}");
    k_vg_offsets_batch<<<off_grid, 256, 0, st>>>(keys.p, reinterpret_cast<const unsigned*>(runs.p), 2, d_num.p, B,
                                                 d_out_off.p);
    c.launches += 4;
    PCLB_CUDA(cudaMemcpyAsync(h_off.data(), d_out_off.p, (B + 1) * sizeof(long long), cudaMemcpyDeviceToHost, st));
    PCLB_CUDA(cudaMemcpyAsync(&n_out, d_num.p, sizeof(size_t), cudaMemcpyDeviceToHost, st));
    PCLB_CUDA(cudaStreamSynchronize(st));
    d_runs = runs.p;
  }
  if (n_out == 0) {
    std::copy(h_off.begin(), h_off.end(), out_offsets);
    return 0;
  }
  // pass 5: centroids, and with normals the remaining fields, of every kept run: run m is row m
  DevBuf<float4> nc, out, nout;
  if (with_nc) {
    nc.alloc(2 * n, st);
    vg_load_normals(c, normals, n, stride_n, nullptr, 0, nc.p);
  }
  float4* const caller_out = reinterpret_cast<float4*>(out_xyz1);
  float4* const caller_nout = reinterpret_cast<float4*>(out_normal_curv);
  vg_reduce(c, dense.p, with_nc ? nc.p : nullptr, vals.p, d_runs, n_out, out_on_device(c, caller_out, n_out, out),
            with_nc ? out_on_device(c, caller_nout, 2 * n_out, nout) : nullptr);
  copy_out(c, caller_out, out, n_out);
  if (with_nc)
    copy_out(c, caller_nout, nout, 2 * n_out);
  PCLB_CUDA(cudaStreamSynchronize(st));
  std::copy(h_off.begin(), h_off.end(), out_offsets);
  return n_out;
}

}  // namespace pclb200
