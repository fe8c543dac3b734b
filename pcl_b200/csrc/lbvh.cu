// lbvh.cu — target-side data layout: Morton-sorted linear BVH in HBM.
//
// Replaces what pcl::KdTreeFLANN::setInputCloud builds on the CPU
// (kdtree/include/pcl/kdtree/impl/kdtree_flann.hpp:100-136, 429-498: drop non-finite points, keep
// index_mapping_, build a FLANN KDTreeSingleIndex with <=15-point leaves).  Here:
//   1. bbox + finite count (one streaming pass, block reduce + atomics on ordered-int floats)
//   2. 63-bit Morton key per point (21 bits/axis, ONE isotropic scale so cells are cubes);
//      non-finite points get key ~0 and sort to the tail
//   3. cub::DeviceRadixSort (key64, value = original index) — stable, so equal keys keep index order
//   4. Karras 2012 binary radix tree over the POINTS (ties by index), cut where a cell holds <= 8 points: every leaf is a
//      whole radix-tree cell, stored as one 128-byte line of float4 {x,y,z, original-index bits} padded with +inf
//   5. bottom-up refit (atomic arrival flags), then both children's boxes are packed into the parent's 64-byte node so
//      one node visit = four independent 128-bit loads
//   6. cell table: every occupied cell of the levels 1..bmax of the Morton grid -> the deepest node / leaf that holds all
//      its points (open-addressing hash, 8 B per slot), so that walks start at the candidate ball instead of the root
//      (traverse.cuh: CellTable, nearest1)
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <memory>

#include "internal.cuh"
#include "traverse.cuh"
#include "lbvh_kernels.cuh"
#include "voxel_grid.cuh"

namespace pclb200 {

bool is_device_ptr(const void* p)
{
  if (!p)
    return false;
  cudaPointerAttributes at;
  cudaError_t e = cudaPointerGetAttributes(&at, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

// ---- strided record -> dense float4 ------------------------------------------------------------
__global__ void k_strided_to_float4(const unsigned char* __restrict__ src, size_t stride,
                                    const int32_t* __restrict__ subset, size_t n, float w_fill,
                                    float4* __restrict__ out)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  size_t r = subset ? (size_t)subset[i] : i;
  const float* p = reinterpret_cast<const float*>(src + r * stride);
  out[i] = make_float4(p[0], p[1], p[2], w_fill);
}

static void strided_to_float4(Ctx& c, const void* src, size_t n_records, size_t stride, const int32_t* subset,
                              size_t n_subset, float w_fill, float4* d_out, cudaStream_t s)
{
  const size_t n = subset ? n_subset : n_records;
  if (n == 0)
    return;
  PCLB_REQUIRE(src != nullptr, PCLB200_ERR_INVALID, "null point array");
  PCLB_REQUIRE(stride >= 12 && stride % 4 == 0, PCLB200_ERR_INVALID, "stride must be a multiple of 4 and >= 12");
  if (!subset && stride == 16) {
    // pcl::PointXYZ records already are float4: one straight copy (w is never read by the kernels)
    PCLB_CUDA(cudaMemcpyAsync(d_out, src, n * 16, is_device_ptr(src) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                              s));
    return;
  }
  // only up to the last byte a record's xyz can occupy: `src` may point INSIDE the caller's records (normals at offset 16
  // of a PointNormal), so n_records * stride bytes would run past the end of the caller's array
  DevBuf<unsigned char> staged;
  DevBuf<int32_t> staged_sub;
  const unsigned char* d_src = on_device(c, static_cast<const unsigned char*>(src), (n_records - 1) * stride + 12, staged);
  const int32_t* d_sub = on_device(c, subset, n_subset, staged_sub);
  k_strided_to_float4<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(d_src, stride, d_sub, n, w_fill, d_out);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

void load_xyz_as_float4(Ctx& c, const void* src, size_t n_records, size_t stride, const int32_t* subset,
                        size_t n_subset, float4* d_out, cudaStream_t s)
{
  strided_to_float4(c, src, n_records, stride, subset, n_subset, 1.f, d_out, s);
}

void load_vec3_as_float4(Ctx& c, const void* src, size_t n_records, size_t stride, float4* d_out, cudaStream_t s)
{
  strided_to_float4(c, src, n_records, stride, nullptr, 0, 0.f, d_out, s);
}

struct SortedCloud {
  DevBuf<unsigned long long> keys;  // sorted
  DevBuf<int32_t> vals;             // sorted slots
  size_t n_valid = 0;
  float lo[3], hi[3];
  float scale = 1.f;
};

// bbox + 63-bit Morton keys + radix sort of n dense float4 points (the index's order)
static void morton_sort(Ctx& c, const float4* d_pts, size_t n, SortedCloud& out)
{
  cudaStream_t s = c.stream;
  {
    DevBuf<BBoxAcc> acc;
    acc.alloc(1, s);
    BBoxAcc init;
    for (int d = 0; d < 3; ++d) {
      init.lo[d] = 0x7fffffff;
      init.hi[d] = (int)0x80000000;
    }
    init.count = 0;
    PCLB_CUDA(cudaMemcpyAsync(acc.p, &init, sizeof(init), cudaMemcpyHostToDevice, s));
    unsigned g = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)c.sm_count * 8);
    k_bbox<<<g ? g : 1, 256, 0, s>>>(d_pts, n, acc.p);
    ++c.launches;
    BBoxAcc h;
    PCLB_CUDA(cudaMemcpyAsync(&h, acc.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    PCLB_CUDA(cudaStreamSynchronize(s));
    out.n_valid = (size_t)h.count;
    if (out.n_valid == 0)
      return;
    morton_frame(h, out.lo, out.hi, out.scale);
  }
  DevBuf<unsigned long long> keys_in;
  DevBuf<int32_t> vals_in;
  keys_in.alloc(n, s);
  vals_in.alloc(n, s);
  out.keys.alloc(n, s);
  out.vals.alloc(n, s);
  k_morton<false><<<grid_for(n, 256), 256, 0, s>>>(d_pts, n, out.lo[0], out.lo[1], out.lo[2], out.scale, keys_in.p,
                                                  vals_in.p);
  ++c.launches;
  size_t tmp_bytes = 0;
  // the index needs the full 63-bit order (leaves are radix-tree cells)
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys_in.p, out.keys.p, vals_in.p, out.vals.p,
                                            (int)n, 0, 64, s));
  DevBuf<unsigned char> tmp;
  tmp.alloc(tmp_bytes, s);
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, keys_in.p, out.keys.p, vals_in.p, out.vals.p, (int)n,
                                            0, 64, s));
  c.launches += 9;  // onesweep: histogram + one pass per 8-bit digit
  PCLB_CUDA(cudaGetLastError());
}

static Index* build_from_dense(Ctx& c, const float4* d_pts, size_t n, const int32_t* d_orig_of_slot, size_t n_cloud,
                                bool build_cell_table)
{
  cudaStream_t s = c.stream;
  PCLB_REQUIRE(n > 0, PCLB200_ERR_EMPTY, "cannot index an empty cloud (kdtree_flann.hpp:118-129)");
  PCLB_REQUIRE(n < (size_t)0x7fffffff, PCLB200_ERR_INVALID, "cloud too large for int32 indices");
  SortedCloud sc;
  morton_sort(c, d_pts, n, sc);
  PCLB_REQUIRE(sc.n_valid > 0, PCLB200_ERR_EMPTY, "no finite point in the cloud (kdtree_flann.hpp:124-129)");
  std::unique_ptr<Index> idx(new Index());
  idx->ctx = &c;
  idx->device = c.device;
  idx->n_cloud = n_cloud;
  idx->n_valid = sc.n_valid;
  for (int d = 0; d < 3; ++d) {
    idx->lo[d] = sc.lo[d];
    idx->hi[d] = sc.hi[d];
  }
  idx->morton_scale = sc.scale;
  const int nv = (int)sc.n_valid;
  if (nv <= kLeafSize) {
    // the whole cloud is one leaf
    idx->n_leaves = 1;
    idx->root = ~0;
    idx->pts.alloc(kLeafSize, s);
    k_gather_sorted<<<1, 256, 0, s>>>(d_pts, sc.vals.p, d_orig_of_slot, sc.n_valid, kLeafSize, idx->pts.p);
    ++c.launches;
  }
  else {
    // 1. radix tree over the points, 2. cut it where a cell holds <= kLeafSize points, 3. renumber, 4. refit + pack
    const int ni = nv - 1;
    DevBuf<int2> kchildren, krange;
    DevBuf<int> knode_parent, kpoint_parent, keep, new_id, leaf_flag, leaf_incl;
    kchildren.alloc(ni, s);
    krange.alloc(ni, s);
    knode_parent.alloc(ni, s);
    kpoint_parent.alloc(nv, s);
    keep.alloc(ni, s);
    new_id.alloc(ni, s);
    leaf_flag.alloc(nv, s);
    leaf_incl.alloc(nv, s);
    PCLB_CUDA(cudaMemsetAsync(leaf_flag.p, 0, leaf_flag.bytes(), s));
    k_karras_points<<<grid_for(ni, 256), 256, 0, s>>>(sc.keys.p, nv, kchildren.p, knode_parent.p, kpoint_parent.p,
                                                      krange.p);
    k_mark_cells<<<grid_for(nv, 256), 256, 0, s>>>(nv, krange.p, knode_parent.p, kpoint_parent.p, keep.p, leaf_flag.p);
    size_t tb = 0, tb2 = 0;
    PCLB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tb, leaf_flag.p, leaf_incl.p, nv, s));
    PCLB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb2, keep.p, new_id.p, ni, s));
    DevBuf<unsigned char> tmp;
    tmp.alloc(std::max(tb, tb2), s);
    PCLB_CUDA(cub::DeviceScan::InclusiveSum(tmp.p, tb, leaf_flag.p, leaf_incl.p, nv, s));
    PCLB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb2, keep.p, new_id.p, ni, s));
    c.launches += 4;
    DevBuf<unsigned> hist;
    unsigned h_hist[64] = {0};
    const bool want_cells = build_cell_table && nv >= 256;
    if (want_cells) {
      hist.alloc(64, s);
      PCLB_CUDA(cudaMemsetAsync(hist.p, 0, 64 * sizeof(unsigned), s));
      k_prefix_hist<<<std::min<unsigned>(grid_for(nv, 256), (unsigned)c.sm_count * 8), 256, 0, s>>>(sc.keys.p, nv, hist.p);
      ++c.launches;
      PCLB_CUDA(cudaMemcpyAsync(h_hist, hist.p, sizeof(h_hist), cudaMemcpyDeviceToHost, s));
    }
    int h_leaves = 0, h_last_id = 0, h_last_keep = 0;
    PCLB_CUDA(cudaMemcpyAsync(&h_leaves, leaf_incl.p + (nv - 1), sizeof(int), cudaMemcpyDeviceToHost, s));
    PCLB_CUDA(cudaMemcpyAsync(&h_last_id, new_id.p + (ni - 1), sizeof(int), cudaMemcpyDeviceToHost, s));
    PCLB_CUDA(cudaMemcpyAsync(&h_last_keep, keep.p + (ni - 1), sizeof(int), cudaMemcpyDeviceToHost, s));
    PCLB_CUDA(cudaStreamSynchronize(s));
    const int n_leaves = h_leaves;
    const int n_int = h_last_id + h_last_keep;
    PCLB_REQUIRE(n_leaves >= 2 && n_int == n_leaves - 1, PCLB200_ERR_INTERNAL, "LBVH build: inconsistent cell cut");
    idx->n_leaves = n_leaves;
    idx->root = 0;
    const size_t n_padded = (size_t)n_leaves * kLeafSize;
    idx->pts.alloc(n_padded, s);
    idx->nodes.alloc(n_int, s);
    DevBuf<int> leaf_start;
    DevBuf<int> node_parent, leaf_parent;  // build-time only (bottom-up refit)
    DevBuf<int2> children;
    DevBuf<float4> leaf_lo, leaf_hi, node_lo, node_hi;
    DevBuf<unsigned> flags;
    leaf_start.alloc(n_leaves, s);
    node_parent.alloc(n_int, s);
    leaf_parent.alloc(n_leaves, s);
    children.alloc(n_int, s);
    idx->node_leaves.alloc(n_int, s);
    leaf_lo.alloc(n_leaves, s);
    leaf_hi.alloc(n_leaves, s);
    node_lo.alloc(n_int, s);
    node_hi.alloc(n_int, s);
    flags.alloc(n_int, s);
    PCLB_CUDA(cudaMemsetAsync(flags.p, 0, flags.bytes(), s));
    k_leaf_starts<<<grid_for(nv, 256), 256, 0, s>>>(nv, leaf_flag.p, leaf_incl.p, leaf_start.p);
    k_fill_sentinels<<<grid_for(n_padded, 256), 256, 0, s>>>(idx->pts.p, n_padded);
    k_scatter_cells<<<grid_for(nv, 256), 256, 0, s>>>(d_pts, sc.vals.p, d_orig_of_slot, nv, leaf_incl.p, leaf_start.p,
                                                      idx->pts.p);
    // cell table (traverse.cuh: CellTable), sized by the prefix-length histogram (cell_table_plan)
    CellTableW cellw{nullptr, 0, 0, 0};
    if (want_cells) {
      idx->cells = cell_table_plan(h_hist, nv, idx->lo, idx->hi, idx->morton_scale);
      if (idx->cells.log2_slots) {
        idx->cell_slots.alloc((size_t)1 << idx->cells.log2_slots, s);
        PCLB_CUDA(cudaMemsetAsync(idx->cell_slots.p, 0, idx->cell_slots.bytes(), s));
        cellw = cell_table_view(idx->cell_slots.p, idx->cells);
      }
    }
    k_link_cells<<<grid_for(ni, 256), 256, 0, s>>>(nv, kchildren.p, krange.p, keep.p, new_id.p, leaf_incl.p, sc.keys.p,
                                                   children.p, node_parent.p, leaf_parent.p, idx->node_leaves.p, cellw);
    k_refit<<<grid_for(n_leaves, 256), 256, 0, s>>>(idx->pts.p, n_leaves, children.p, node_parent.p, leaf_parent.p,
                                                    leaf_lo.p, leaf_hi.p, node_lo.p, node_hi.p, flags.p);
    k_pack_nodes<<<grid_for(n_int, 256), 256, 0, s>>>(n_int, children.p, leaf_lo.p, leaf_hi.p, node_lo.p, node_hi.p,
                                                     idx->nodes.p);
    c.launches += 8;
    PCLB_CUDA(cudaGetLastError());
  }
  PCLB_CUDA(cudaStreamSynchronize(s));  // temporaries are released stream-ordered; surface build errors here
  return idx.release();
}

Index* build_index(Ctx& c, const void* pts, size_t n, size_t stride, const int32_t* subset, size_t n_subset)
{
  cudaStream_t s = c.stream;
  const size_t cnt = subset ? n_subset : n;
  PCLB_REQUIRE(pts != nullptr && cnt > 0, PCLB200_ERR_EMPTY, "cannot index an empty cloud (kdtree_flann.hpp:118-129)");
  DevBuf<float4> dense;
  dense.alloc(cnt, s);
  load_xyz_as_float4(c, pts, n, stride, subset, n_subset, dense.p, s);
  DevBuf<int32_t> d_sub;
  return build_from_dense(c, dense.p, cnt, on_device(c, subset, n_subset, d_sub), n, true);
}

Index* build_index_from_device(Ctx& c, const float4* d_pts, size_t n, const int32_t* d_orig, bool cell_table)
{
  return build_from_dense(c, d_pts, n, d_orig, n, cell_table);
}

// ---- a batch of clouds in one build ------------------------------------------------------------------------------
// Cloud c = records [offsets[c], offsets[c + 1]) of one array; each Index is what build_index makes of the cloud alone.
// Every stage is one launch for the whole batch (lbvh_kernels.cuh: the *_batch kernels run the single build's bodies on
// each cloud's base pointers), and the host synchronises three times, as one single build does: for the clouds' boxes,
// for their cuts, and at the end.
std::vector<std::unique_ptr<Index>> build_index_batch(Ctx& c, const void* pts, size_t n, size_t stride,
                                                      const int64_t* offsets, int n_clouds)
{
  cudaStream_t s = c.stream;
  PCLB_REQUIRE(n_clouds >= 1 && n_clouds <= 65536, PCLB200_ERR_INVALID, "index_build_batch: a batch holds 1 to 65536 clouds");
  PCLB_REQUIRE(pts && offsets, PCLB200_ERR_INVALID, "index_build_batch: NULL argument");
  PCLB_REQUIRE(offsets[0] == 0 && offsets[n_clouds] == (int64_t)n, PCLB200_ERR_INVALID,
               "index_build_batch: offsets must run from 0 to n");
  for (int k = 0; k < n_clouds; ++k)
    PCLB_REQUIRE(offsets[k + 1] > offsets[k], PCLB200_ERR_INVALID,
                 "index_build_batch: offsets must increase strictly (every cloud holds a record)");
  PCLB_REQUIRE(n < (size_t)0x7fffffff, PCLB200_ERR_INVALID, "cloud too large for int32 indices");
  const int B = n_clouds;
  DevBuf<float4> dense;
  dense.alloc(n, s);
  load_xyz_as_float4(c, pts, n, stride, nullptr, 0, dense.p, s);

  // prefix tables of the launches' work spaces, B + 1 entries each: records, tiles, leaves, final nodes, cell-table slots
  enum { kRecords, kTiles, kLeaves, kNodes, kSlots, kSpaces };
  std::vector<long long> pre((size_t)kSpaces * (B + 1), 0);
  auto P = [&](int space) { return pre.data() + (size_t)space * (B + 1); };
  std::vector<BuildCloud> cl(B);
  for (int k = 0; k < B; ++k) {
    cl[k].first = offsets[k];
    cl[k].n = offsets[k + 1] - offsets[k];
    P(kRecords)[k + 1] = offsets[k + 1];
    P(kTiles)[k + 1] = P(kTiles)[k] + (cl[k].n + kBatchTile - 1) / kBatchTile;
  }
  DevBuf<long long> d_pre;
  DevBuf<BuildCloud> d_cl;
  d_pre.alloc(pre.size(), s);
  d_cl.alloc(B, s);
  const long long* d_off = d_pre.p + (size_t)kRecords * (B + 1);
  const long long* d_tiles = d_pre.p + (size_t)kTiles * (B + 1);
  PCLB_CUDA(cudaMemcpyAsync(d_pre.p, pre.data(), pre.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
  PCLB_CUDA(cudaMemcpyAsync(d_cl.p, cl.data(), B * sizeof(BuildCloud), cudaMemcpyHostToDevice, s));

  // 1. per cloud: box and finite count -> frame (synchronisation 1)
  std::vector<BBoxAcc> acc(B);
  for (auto& a : acc) {
    for (int d = 0; d < 3; ++d) {
      a.lo[d] = 0x7fffffff;
      a.hi[d] = (int)0x80000000;
    }
    a.count = 0;
  }
  {
    DevBuf<BBoxAcc> d_acc;
    d_acc.alloc(B, s);
    PCLB_CUDA(cudaMemcpyAsync(d_acc.p, acc.data(), B * sizeof(BBoxAcc), cudaMemcpyHostToDevice, s));
    k_bbox_batch<<<(unsigned)P(kTiles)[B], 256, 0, s>>>(dense.p, d_cl.p, d_tiles, B, d_acc.p);
    ++c.launches;
    PCLB_CUDA(cudaMemcpyAsync(acc.data(), d_acc.p, B * sizeof(BBoxAcc), cudaMemcpyDeviceToHost, s));
    PCLB_CUDA(cudaStreamSynchronize(s));
  }
  for (int k = 0; k < B; ++k) {
    PCLB_REQUIRE(acc[k].count > 0, PCLB200_ERR_EMPTY,
                 "index_build_batch: cloud " + std::to_string(k) + " has no finite point (kdtree_flann.hpp:124-129)");
    cl[k].nv = (int)acc[k].count;
    float hi[3];  // the handle's, filled in step 4
    morton_frame(acc[k], cl[k].lo, hi, cl[k].scale);
  }
  PCLB_CUDA(cudaMemcpyAsync(d_cl.p, cl.data(), B * sizeof(BuildCloud), cudaMemcpyHostToDevice, s));

  // 2. keys in each cloud's frame; sorted by key, then stably by cloud: each cloud's range in its single build's order
  DevBuf<unsigned long long> keys;
  DevBuf<int32_t> vals;
  keys.alloc(n, s);
  vals.alloc(n, s);
  DevBuf<unsigned> cloud_of;  // the cloud of each sorted position (the key of the per-cloud scans)
  cloud_of.alloc(n, s);
  {
    DevBuf<unsigned long long> keys_in, keys1;
    DevBuf<int32_t> vals_in, vals1, pos, perm;
    DevBuf<unsigned> cloud_in;
    keys_in.alloc(n, s);
    keys1.alloc(n, s);
    vals_in.alloc(n, s);
    vals1.alloc(n, s);
    pos.alloc(n, s);
    perm.alloc(n, s);
    cloud_in.alloc(n, s);
    k_morton_batch<<<grid_for(n, 256), 256, 0, s>>>(dense.p, n, d_off, B, d_cl.p, keys_in.p, vals_in.p);
    size_t tb1 = 0, tb2 = 0;
    PCLB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb1, keys_in.p, keys1.p, vals_in.p, vals1.p, (int)n, 0, 64, s));
    PCLB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb2, cloud_in.p, cloud_of.p, pos.p, perm.p, (int)n, 0, 16, s));
    DevBuf<unsigned char> tmp;
    tmp.alloc(std::max(tb1, tb2), s);
    PCLB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb1, keys_in.p, keys1.p, vals_in.p, vals1.p, (int)n, 0, 64, s));
    k_cloud_of_sorted<<<grid_for(n, 256), 256, 0, s>>>(vals1.p, n, d_off, B, cloud_in.p, pos.p);
    PCLB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb2, cloud_in.p, cloud_of.p, pos.p, perm.p, (int)n, 0, 16, s));
    k_permute_sorted<<<grid_for(n, 256), 256, 0, s>>>(keys1.p, vals1.p, perm.p, n, d_off, B, keys.p, vals.p);
    c.launches += 3 + 9 + 3;  // onesweep: histogram + one pass per 8-bit digit
    PCLB_CUDA(cudaGetLastError());
  }

  // 3. radix trees, cuts, scans by cloud, prefix histograms -> leaf and node counts (synchronisation 2)
  const size_t n_tree = n - (size_t)B;  // node scratch: cloud c's at first - c (a cloud of m records has <= m - 1 nodes)
  DevBuf<int2> kchildren, krange;
  DevBuf<int> knode_parent, kpoint_parent, keep, new_id, leaf_flag, leaf_incl;
  DevBuf<unsigned> node_cloud;
  kchildren.alloc(n_tree, s);
  krange.alloc(n_tree, s);
  knode_parent.alloc(n_tree, s);
  keep.alloc(n_tree, s);
  new_id.alloc(n_tree, s);
  node_cloud.alloc(n_tree, s);
  kpoint_parent.alloc(n, s);
  leaf_flag.alloc(n, s);
  leaf_incl.alloc(n, s);
  PCLB_CUDA(cudaMemsetAsync(leaf_flag.p, 0, leaf_flag.bytes(), s));
  if (n_tree)
    PCLB_CUDA(cudaMemsetAsync(keep.p, 0, keep.bytes(), s));
  k_karras_points_batch<<<grid_for(n, 256), 256, 0, s>>>(keys.p, n, d_off, B, d_cl.p, kchildren.p, knode_parent.p,
                                                         kpoint_parent.p, krange.p, node_cloud.p);
  k_mark_cells_batch<<<grid_for(n, 256), 256, 0, s>>>(n, d_off, B, d_cl.p, krange.p, knode_parent.p, kpoint_parent.p,
                                                      keep.p, leaf_flag.p);
  {
    size_t tb = 0, tb2 = 0;
    PCLB_CUDA(cub::DeviceScan::InclusiveSumByKey(nullptr, tb, cloud_of.p, leaf_flag.p, leaf_incl.p, (int)n, cub::Equality(), s));
    PCLB_CUDA(cub::DeviceScan::ExclusiveSumByKey(nullptr, tb2, node_cloud.p, keep.p, new_id.p, (int)n_tree, cub::Equality(), s));
    DevBuf<unsigned char> tmp;
    tmp.alloc(std::max(tb, tb2), s);
    PCLB_CUDA(cub::DeviceScan::InclusiveSumByKey(tmp.p, tb, cloud_of.p, leaf_flag.p, leaf_incl.p, (int)n, cub::Equality(), s));
    if (n_tree)
      PCLB_CUDA(cub::DeviceScan::ExclusiveSumByKey(tmp.p, tb2, node_cloud.p, keep.p, new_id.p, (int)n_tree, cub::Equality(), s));
    c.launches += 2 + (n_tree ? 2 : 0);  // init + scan pass of each scan
  }
  std::vector<CloudSummary> sum(B);
  {
    DevBuf<CloudSummary> d_sum;
    d_sum.alloc(B, s);
    PCLB_CUDA(cudaMemsetAsync(d_sum.p, 0, d_sum.bytes(), s));
    k_prefix_hist_batch<<<(unsigned)P(kTiles)[B], 256, 0, s>>>(keys.p, d_cl.p, d_tiles, B, d_sum.p);
    k_cut_summary<<<grid_for(B, 256), 256, 0, s>>>(d_cl.p, B, leaf_incl.p, new_id.p, keep.p, d_sum.p);
    c.launches += 2;
    PCLB_CUDA(cudaGetLastError());
    PCLB_CUDA(cudaMemcpyAsync(sum.data(), d_sum.p, B * sizeof(CloudSummary), cudaMemcpyDeviceToHost, s));
    PCLB_CUDA(cudaStreamSynchronize(s));
  }

  // 4. the handles: sized and planned by the single build's rules, allocated from the block cache, written in place
  std::vector<std::unique_ptr<Index>> out(B);
  for (int k = 0; k < B; ++k) {
    BuildCloud& C = cl[k];
    const CloudSummary& S = sum[k];
    std::unique_ptr<Index> idx(new Index());
    idx->ctx = &c;
    idx->device = c.device;
    idx->n_cloud = (size_t)C.n;
    idx->n_valid = (size_t)C.nv;
    morton_frame(acc[k], idx->lo, idx->hi, idx->morton_scale);
    if (C.nv <= kLeafSize) {
      idx->n_leaves = 1;
      idx->root = ~0;
    }
    else {
      PCLB_REQUIRE(S.n_leaves >= 2 && S.n_int == S.n_leaves - 1, PCLB200_ERR_INTERNAL, "LBVH build: inconsistent cell cut");
      idx->n_leaves = S.n_leaves;
      idx->root = 0;
      idx->nodes.alloc(S.n_int, s);
      idx->node_leaves.alloc(S.n_int, s);
      if (C.nv >= 256) {
        idx->cells = cell_table_plan(S.hist, C.nv, idx->lo, idx->hi, idx->morton_scale);
        if (idx->cells.log2_slots) {
          idx->cell_slots.alloc((size_t)1 << idx->cells.log2_slots, s);
          C.cells = cell_table_view(idx->cell_slots.p, idx->cells);
        }
      }
    }
    idx->pts.alloc((size_t)idx->n_leaves * kLeafSize, s);
    C.n_leaves = idx->n_leaves;
    C.n_int = C.nv <= kLeafSize ? 0 : S.n_int;
    C.pts = idx->pts.p;
    C.nodes = idx->nodes.p;
    C.node_leaves = idx->node_leaves.p;
    C.leaf_first = P(kLeaves)[k];
    C.node_first = P(kNodes)[k];
    P(kLeaves)[k + 1] = P(kLeaves)[k] + C.n_leaves;
    P(kNodes)[k + 1] = P(kNodes)[k] + C.n_int;
    P(kSlots)[k + 1] = P(kSlots)[k] + (long long)idx->cell_slots.n;
    out[k] = std::move(idx);
  }
  PCLB_CUDA(cudaMemcpyAsync(d_pre.p, pre.data(), pre.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
  PCLB_CUDA(cudaMemcpyAsync(d_cl.p, cl.data(), B * sizeof(BuildCloud), cudaMemcpyHostToDevice, s));
  const long long* d_leaves = d_pre.p + (size_t)kLeaves * (B + 1);
  const long long* d_nodes = d_pre.p + (size_t)kNodes * (B + 1);
  const long long* d_slots = d_pre.p + (size_t)kSlots * (B + 1);
  const size_t n_leaves = (size_t)P(kLeaves)[B], n_int = (size_t)P(kNodes)[B];
  DevBuf<int> leaf_start, node_parent, leaf_parent;
  DevBuf<int2> children;
  DevBuf<float4> leaf_lo, leaf_hi, node_lo, node_hi;
  DevBuf<unsigned> flags;
  leaf_start.alloc(n_leaves, s);
  leaf_parent.alloc(n_leaves, s);
  leaf_lo.alloc(n_leaves, s);
  leaf_hi.alloc(n_leaves, s);
  node_parent.alloc(n_int, s);
  children.alloc(n_int, s);
  node_lo.alloc(n_int, s);
  node_hi.alloc(n_int, s);
  flags.alloc(n_int, s);
  if (n_int)
    PCLB_CUDA(cudaMemsetAsync(flags.p, 0, flags.bytes(), s));
  const size_t n_clear = std::max<size_t>(n_leaves * kLeafSize, (size_t)P(kSlots)[B]);
  k_clear_outputs_batch<<<grid_for(n_clear, 256), 256, 0, s>>>(d_cl.p, B, d_leaves, d_slots);
  k_gather_small_batch<<<grid_for((size_t)B * kLeafSize, 256), 256, 0, s>>>(dense.p, vals.p, d_cl.p, B);
  k_leaf_starts_batch<<<grid_for(n, 256), 256, 0, s>>>(n, d_off, B, d_cl.p, leaf_flag.p, leaf_incl.p, leaf_start.p);
  k_scatter_cells_batch<<<grid_for(n, 256), 256, 0, s>>>(dense.p, vals.p, n, d_off, B, d_cl.p, leaf_incl.p,
                                                         leaf_start.p);
  k_link_cells_batch<<<grid_for(n, 256), 256, 0, s>>>(n, d_off, B, d_cl.p, kchildren.p, krange.p, keep.p, new_id.p,
                                                      leaf_incl.p, keys.p, children.p, node_parent.p, leaf_parent.p);
  k_refit_batch<<<grid_for(n_leaves, 256), 256, 0, s>>>(d_cl.p, B, d_leaves, children.p, node_parent.p, leaf_parent.p,
                                                        leaf_lo.p, leaf_hi.p, node_lo.p, node_hi.p, flags.p);
  if (n_int)
    k_pack_nodes_batch<<<grid_for(n_int, 256), 256, 0, s>>>(d_cl.p, B, d_nodes, children.p, leaf_lo.p, leaf_hi.p,
                                                            node_lo.p, node_hi.p);
  c.launches += 6 + (n_int ? 1 : 0);
  PCLB_CUDA(cudaGetLastError());
  PCLB_CUDA(cudaStreamSynchronize(s));  // temporaries are released stream-ordered; surface build errors here
  return out;
}

// the boxes of a batch of clouds (every cloud holds a record), as build_index_batch's step 1 reduces them
// (voxel.cu: voxelgrid_batch)
void cloud_boxes(Ctx& c, const float4* d_pts, const int64_t* offsets, int n_clouds, MinMaxAcc* out)
{
  cudaStream_t s = c.stream;
  const int B = n_clouds;
  std::vector<long long> tiles(B + 1, 0);
  std::vector<BuildCloud> cl(B);
  std::vector<BBoxAcc> acc(B);
  for (int k = 0; k < B; ++k) {
    cl[k].first = offsets[k];
    cl[k].n = offsets[k + 1] - offsets[k];
    tiles[k + 1] = tiles[k] + (cl[k].n + kBatchTile - 1) / kBatchTile;
    for (int d = 0; d < 3; ++d) {
      acc[k].lo[d] = 0x7fffffff;
      acc[k].hi[d] = (int)0x80000000;
    }
    acc[k].count = 0;
  }
  DevBuf<long long> d_tiles;
  DevBuf<BuildCloud> d_cl;
  DevBuf<BBoxAcc> d_acc;
  d_tiles.alloc(B + 1, s);
  d_cl.alloc(B, s);
  d_acc.alloc(B, s);
  PCLB_CUDA(cudaMemcpyAsync(d_tiles.p, tiles.data(), (B + 1) * sizeof(long long), cudaMemcpyHostToDevice, s));
  PCLB_CUDA(cudaMemcpyAsync(d_cl.p, cl.data(), B * sizeof(BuildCloud), cudaMemcpyHostToDevice, s));
  PCLB_CUDA(cudaMemcpyAsync(d_acc.p, acc.data(), B * sizeof(BBoxAcc), cudaMemcpyHostToDevice, s));
  k_bbox_batch<<<(unsigned)tiles[B], 256, 0, s>>>(d_pts, d_cl.p, d_tiles.p, B, d_acc.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  PCLB_CUDA(cudaMemcpyAsync(acc.data(), d_acc.p, B * sizeof(BBoxAcc), cudaMemcpyDeviceToHost, s));
  PCLB_CUDA(cudaStreamSynchronize(s));
  for (int k = 0; k < B; ++k) {
    for (int d = 0; d < 3; ++d) {
      out[k].lo[d] = acc[k].lo[d];
      out[k].hi[d] = acc[k].hi[d];
    }
    out[k].count = acc[k].count;
  }
}

// ---- labelled index: one tile of a map, its points carrying the caller's ids -------------------------------------
// sorted ids: kIdOutOfRange = an id outside [0, 2^31 - 2] (2^31 - 1 marks padding), kIdRepeated = two equal ids
__global__ void k_check_sorted_ids(const int32_t* __restrict__ sorted, size_t n, int* __restrict__ flag)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const int32_t v = sorted[i];
  if (v < 0 || v == kSentinelIndex)
    atomicOr(flag, kIdOutOfRange);
  if (i > 0 && sorted[i - 1] == v)
    atomicOr(flag, kIdRepeated);
}

int id_faults(Ctx& c, const int32_t* d_ids, size_t n)
{
  cudaStream_t s = c.stream;
  if (!n)
    return 0;
  DevBuf<int32_t> sorted;
  sorted.alloc(n, s);
  size_t tb = 0;
  PCLB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, d_ids, sorted.p, (int)n, 0, 32, s));
  DevBuf<unsigned char> tmp;
  tmp.alloc(tb, s);
  PCLB_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, tb, d_ids, sorted.p, (int)n, 0, 32, s));
  c.launches += 5;
  DevBuf<int> flag;
  flag.alloc(1, s);
  PCLB_CUDA(cudaMemsetAsync(flag.p, 0, sizeof(int), s));
  k_check_sorted_ids<<<grid_for(n, 256), 256, 0, s>>>(sorted.p, n, flag.p);
  ++c.launches;
  int h = 0;
  PCLB_CUDA(cudaMemcpyAsync(&h, flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  PCLB_CUDA(cudaStreamSynchronize(s));
  return h;
}

// w = record number (as built) -> w = ids[record], the record number kept in slot_of_pos
__global__ void k_label_points(float4* __restrict__ pts, size_t n_padded, const int32_t* __restrict__ ids,
                               int32_t* __restrict__ slot_of_pos)
{
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n_padded)
    return;
  const int slot = __float_as_int(pts[j].w);
  if (slot == kSentinelIndex) {
    slot_of_pos[j] = -1;
    return;
  }
  slot_of_pos[j] = slot;
  pts[j].w = __int_as_float(ids[slot]);
}

// The tree of build_index over the same points in the same order (the labels never enter the build), with w relabelled:
// byte for byte the index build_index makes of a whole cloud with subset = ids, when point i of this tile is point ids[i]
// of that cloud.
Index* build_index_ids(Ctx& c, const void* pts, size_t n, size_t stride, const int32_t* ids)
{
  cudaStream_t s = c.stream;
  PCLB_REQUIRE(pts != nullptr && n > 0, PCLB200_ERR_EMPTY, "cannot index an empty cloud (kdtree_flann.hpp:118-129)");
  PCLB_REQUIRE(ids != nullptr, PCLB200_ERR_INVALID, "index_build_ids: NULL ids");
  PCLB_REQUIRE(n < (size_t)0x7fffffff, PCLB200_ERR_INVALID, "cloud too large for int32 indices");
  DevBuf<int32_t> d_ids;
  d_ids.alloc(n, s);
  PCLB_CUDA(cudaMemcpyAsync(d_ids.p, ids, n * sizeof(int32_t), cudaMemcpyDefault, s));
  const int h = id_faults(c, d_ids.p, n);
  PCLB_REQUIRE(!(h & kIdOutOfRange), PCLB200_ERR_INVALID, "index_build_ids: every id must lie in [0, 2^31 - 2]");
  PCLB_REQUIRE(!(h & kIdRepeated), PCLB200_ERR_INVALID, "index_build_ids: two points of the cloud carry the same id");
  DevBuf<float4> dense;
  dense.alloc(n, s);
  load_xyz_as_float4(c, pts, n, stride, nullptr, 0, dense.p, s);
  std::unique_ptr<Index> idx(build_from_dense(c, dense.p, n, nullptr, n, true));
  idx->labelled = true;
  idx->slot_of_pos.alloc(idx->pts.n, s);
  k_label_points<<<grid_for(idx->pts.n, 256), 256, 0, s>>>(idx->pts.p, idx->pts.n, d_ids.p, idx->slot_of_pos.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  PCLB_CUDA(cudaStreamSynchronize(s));
  return idx.release();
}

// ---- position of each original index in the Morton array (for gathers by index_match) -------------
__global__ void k_pos_of_orig(const float4* __restrict__ pts, size_t n_padded, int32_t* __restrict__ pos)
{
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n_padded)
    return;
  int oi = __float_as_int(pts[j].w);
  if (oi != kSentinelIndex)
    pos[oi] = (int32_t)j;
}

void ensure_pos_of_orig(Ctx& c, Index& idx)
{
  if (idx.pos_of_orig.p)
    return;
  PCLB_REQUIRE(!idx.labelled, PCLB200_ERR_INVALID,
               "an index built with caller ids (pclb200_index_build_ids) cannot serve the normal-based estimators, normal "
               "estimation with k > 32 or a radius, or GICP covariances: they address the cloud the index was built from");
  cudaStream_t s = c.stream;
  idx.pos_of_orig.alloc(idx.n_cloud, s);
  PCLB_CUDA(cudaMemsetAsync(idx.pos_of_orig.p, 0xff, idx.pos_of_orig.bytes(), s));
  k_pos_of_orig<<<grid_for(idx.pts.n, 256), 256, 0, s>>>(idx.pts.p, idx.pts.n, idx.pos_of_orig.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

// ---- query batches ------------------------------------------------------------------------------
__global__ void k_gather_queries(const float4* __restrict__ q, const int32_t* __restrict__ vals, size_t n,
                                 float4* __restrict__ out)
{
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n)
    return;
  int32_t slot = vals[j];
  float4 v = __ldg(q + slot);
  out[j] = make_float4(v.x, v.y, v.z, __int_as_float(slot));
}

// the queries pts[vals_in[j]] by keys_in (stable: the points of one key cell keep their input order), w = slot
static void sort_queries(Ctx& c, DevBuf<unsigned>& keys_in, DevBuf<int32_t>& vals_in, const float4* pts, size_t n,
                         QueryBatch& qb)
{
  cudaStream_t s = c.stream;
  DevBuf<unsigned> keys;
  DevBuf<int32_t> vals;
  keys.alloc(n, s);
  vals.alloc(n, s);
  size_t tmp_bytes = 0;
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys_in.p, keys.p, vals_in.p, vals.p, (int)n, 0, 32, s));
  DevBuf<unsigned char> tmp;
  tmp.alloc(tmp_bytes, s);
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, keys_in.p, keys.p, vals_in.p, vals.p, (int)n, 0, 32, s));
  c.launches += 5;  // onesweep: histogram + one pass per 8-bit digit
  qb.q.alloc(n, s);
  k_gather_queries<<<grid_for(n, 256), 256, 0, s>>>(pts, vals.p, n, qb.q.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

void stage_records(Ctx& c, const Index& frame, const unsigned char* recs, size_t n, size_t stride, unsigned char* copy,
                   float4* dense, QueryBatch* qb)
{
  cudaStream_t s = c.stream;
  if (qb)
    qb->n = n;
  if (n == 0 || !(copy || dense || qb))
    return;
  DevBuf<unsigned> keys_in;
  DevBuf<int32_t> vals_in;
  if (qb) {
    keys_in.alloc(n, s);
    vals_in.alloc(n, s);
  }
  const bool vec = stride % 16 == 0 && reinterpret_cast<uintptr_t>(recs) % 16 == 0 &&
                   reinterpret_cast<uintptr_t>(copy) % 16 == 0;
  if (vec)
    k_stage_records<<<grid_for(n, 256), 256, 0, s>>>(reinterpret_cast<const float4*>(recs), n, (unsigned)(stride / 16),
                                                      reinterpret_cast<float4*>(copy), dense, frame.lo[0], frame.lo[1],
                                                      frame.lo[2], frame.morton_scale, keys_in.p, vals_in.p);
  else
    k_stage_records<<<grid_for(n, 256), 256, 0, s>>>(reinterpret_cast<const float*>(recs), n, (unsigned)(stride / 4),
                                                      reinterpret_cast<float*>(copy), dense, frame.lo[0], frame.lo[1],
                                                      frame.lo[2], frame.morton_scale, keys_in.p, vals_in.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  if (!qb)
    return;
  sort_queries(c, keys_in, vals_in, dense ? dense : reinterpret_cast<const float4*>(recs), n, *qb);
}

void make_query_batch_framed(Ctx& c, const float4* d_frames, const long long* d_offsets, int n_problems,
                             const float4* d_q, size_t n, QueryBatch& out)
{
  cudaStream_t s = c.stream;
  out.n = n;
  if (n == 0)
    return;
  DevBuf<unsigned> keys_in;
  DevBuf<int32_t> vals_in;
  keys_in.alloc(n, s);
  vals_in.alloc(n, s);
  k_problem_frame_keys<<<grid_for(n, 256), 256, 0, s>>>(d_q, n, d_offsets, n_problems, d_frames, keys_in.p, vals_in.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  sort_queries(c, keys_in, vals_in, d_q, n, out);
}

void make_query_batch(Ctx& c, const Index& frame, const float4* d_q, size_t n, QueryBatch& out)
{
  stage_records(c, frame, reinterpret_cast<const unsigned char*>(d_q), n, 16, nullptr, nullptr, &out);
}

QueryBatch load_queries(Ctx& c, const Index& frame, const void* pts, size_t n, size_t stride, const int32_t* subset,
                        size_t n_subset, DevBuf<float4>& dense)
{
  const size_t nq = subset ? n_subset : n;
  dense.alloc(nq, c.stream);
  load_xyz_as_float4(c, pts, n, stride, subset, n_subset, dense.p, c.stream);
  QueryBatch qb;
  make_query_batch(c, frame, dense.p, nq, qb);
  return qb;
}

// ---- correspondence lists to the caller ---------------------------------------------------------------------------
struct CorrValid {
  __host__ __device__ bool operator()(const pclb200_corr& c) const { return c.index_match >= 0; }
};

// select(temp, temp_bytes, d_out, d_count): one cub::DeviceSelect call of the two-phase protocol
template <typename Select>
static size_t compact_with(Ctx& c, size_t n, pclb200_corr* out, Select&& select)
{
  cudaStream_t st = c.stream;
  DevBuf<pclb200_corr> staged;
  DevBuf<size_t> d_count;
  pclb200_corr* d_out = out_on_device(c, out, n, staged);
  d_count.alloc(1, st);
  size_t tmp_bytes = 0;
  PCLB_CUDA(select(nullptr, tmp_bytes, d_out, d_count.p));
  DevBuf<unsigned char> tmp;
  tmp.alloc(tmp_bytes, st);
  PCLB_CUDA(select(tmp.p, tmp_bytes, d_out, d_count.p));
  c.launches += 2;
  size_t m = 0;
  PCLB_CUDA(cudaMemcpyAsync(&m, d_count.p, sizeof(size_t), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  copy_out(c, out, staged, m);
  return m;
}

size_t compact_corr_to(Ctx& c, const pclb200_corr* d_in, size_t n, pclb200_corr* out)
{
  return compact_with(c, n, out, [&](void* tmp, size_t& tb, pclb200_corr* d_out, size_t* d_count) {
    return cub::DeviceSelect::If(tmp, tb, d_in, d_out, d_count, (int)n, CorrValid(), c.stream);
  });
}

size_t compact_corr_to(Ctx& c, const pclb200_corr* d_in, const unsigned char* d_flags, size_t n, pclb200_corr* out)
{
  return compact_with(c, n, out, [&](void* tmp, size_t& tb, pclb200_corr* d_out, size_t* d_count) {
    return cub::DeviceSelect::Flagged(tmp, tb, d_in, d_flags, d_out, d_count, (int)n, c.stream);
  });
}

}  // namespace pclb200
