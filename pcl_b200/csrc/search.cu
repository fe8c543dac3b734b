// search.cu — batch k-NN, radius search and k-NN normals over the LBVH.
//
// Replaces pcl::KdTreeFLANN::nearestKSearch / radiusSearch (kdtree/include/pcl/kdtree/impl/
// kdtree_flann.hpp:234-274, 372-414), the OpenMP batch loops of pcl::search::Search
// (search/include/pcl/search/impl/search.hpp:111-194) and NormalEstimation::computeFeature
// (features/include/pcl/features/impl/normal_3d.hpp:47-96).
// One query per thread, queries in Morton order so a warp walks one neighbourhood of the tree
// (node lines are shared through L1/L2); candidate lists live in registers (k <= 32).
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <limits>

#include "internal.cuh"
#include "traverse.cuh"
#include "knn_warp.cuh"
#include "search_kernels.cuh"

namespace pclb200 {

// warp-cooperative path (defined below): returns the per-query "redo" flags of the queries it handed back, or an empty
// buffer when it does not apply (no cell table, k outside 8..32)
static bool warp_knn_lists(Ctx& c, const Index& idx, const float4* d_q, size_t nq, int k, int32_t* d_out_idx,
                           float* d_out_d2, DevBuf<unsigned char>& redo);

void launch_knn(Ctx& c, const Index& idx, const float4* d_q, size_t nq, int k, float init_bound, int32_t* d_out_idx,
                float* d_out_d2)
{
  if (nq == 0 || k <= 0)
    return;
  cudaStream_t s = c.stream;
  const unsigned g = grid_for(nq, 128);
  DevBuf<unsigned char> redo;
  const unsigned char* only = nullptr;
  if (init_bound == std::numeric_limits<float>::infinity() && warp_knn_lists(c, idx, d_q, nq, k, d_out_idx, d_out_d2, redo))
    only = redo.p;  // the per-thread kernel below only redoes what the warp kernel handed back
#define PCLB_KNN_CASE(KK)                                                                                            \
  k_knn<KK><<<g, 128, 0, s>>>(idx.nodes.p, idx.pts.p, idx.root, d_q, nq, k, init_bound, d_out_idx, d_out_d2, c.d_error, only)
  if (k == 1) PCLB_KNN_CASE(1);
  else if (k == 2) PCLB_KNN_CASE(2);
  else if (k <= 4) PCLB_KNN_CASE(4);
  else if (k <= 8) PCLB_KNN_CASE(8);
  else if (k <= 10) PCLB_KNN_CASE(10);
  else if (k <= 16) PCLB_KNN_CASE(16);
  else if (k <= 20) PCLB_KNN_CASE(20);
  else if (k <= 32) PCLB_KNN_CASE(32);
  else
    k_knn_any<<<g, 128, 0, s>>>(idx.nodes.p, idx.pts.p, idx.root, d_q, nq, k, init_bound, d_out_idx, d_out_d2,
                                c.d_error);
#undef PCLB_KNN_CASE
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

// exact lists first (launch_knn: the warp-cooperative search where it applies), folded afterwards.  NaN queries get empty
// rows from the walk (no box is ever within a NaN bound) and are zeroed by the fold.
static void knn_stats_from_lists(Ctx& c, const Index& idx, const float4* d_q, size_t nq, int k, float* d_mean, float* d_kth)
{
  cudaStream_t s = c.stream;
  DevBuf<int32_t> li;
  DevBuf<float> ld;
  li.alloc(nq * (size_t)k, s);
  ld.alloc(nq * (size_t)k, s);
  launch_knn(c, idx, d_q, nq, k, __builtin_inff(), li.p, ld.p);
  k_stats_from_lists<<<grid_for(nq, 256), 256, 0, s>>>(d_q, nq, k, li.p, ld.p, d_mean, d_kth);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

void launch_knn_kth(Ctx& c, const Index& idx, const float4* d_q, size_t nq, int k, float* d_kth)
{
  if (nq && k > 0)
    knn_stats_from_lists(c, idx, d_q, nq, k, nullptr, d_kth);
}

void launch_knn_stats(Ctx& c, const Index& idx, const float4* d_q, size_t nq, int k, float* d_mean, float* d_kth)
{
  if (!nq || k <= 0)
    return;
  cudaStream_t s = c.stream;
  const unsigned g = grid_for(nq, 128);
  if (k > 32) {  // large neighbourhoods (StatisticalOutlierRemoval's usual mean_k = 50)
    knn_stats_from_lists(c, idx, d_q, nq, k, d_mean, d_kth);
    return;
  }
#define PCLB_STAT_CASE(KK) \
  k_knn_stats<KK><<<g, 128, 0, s>>>(idx.nodes.p, idx.pts.p, idx.root, d_q, nq, k, d_mean, d_kth, c.d_error)
  if (k <= 2) PCLB_STAT_CASE(2);
  else if (k <= 4) PCLB_STAT_CASE(4);
  else if (k <= 8) PCLB_STAT_CASE(8);
  else if (k <= 10) PCLB_STAT_CASE(10);
  else if (k <= 16) PCLB_STAT_CASE(16);
  else if (k <= 20) PCLB_STAT_CASE(20);
  else PCLB_STAT_CASE(32);
#undef PCLB_STAT_CASE
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

static float float_below(float x) { return std::nextafter(x, -INFINITY); }

void launch_radius_count(Ctx& c, const Index& idx, const float4* d_q, size_t nq, float r2,
                         unsigned long long* d_counts)
{
  if (!nq)
    return;
  k_radius_count<<<grid_for(nq, 128), 128, 0, c.stream>>>(idx.nodes.p, idx.pts.p, idx.root, d_q, nq, r2,
                                                         float_below(r2), d_counts, c.d_error);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

void launch_radius_fill(Ctx& c, const Index& idx, const float4* d_q, size_t nq, float r2,
                        const unsigned long long* d_offsets, unsigned long long* d_keys)
{
  if (!nq)
    return;
  k_radius_fill<<<grid_for(nq, 128), 128, 0, c.stream>>>(idx.nodes.p, idx.pts.p, idx.root, d_q, nq, r2,
                                                        float_below(r2), d_offsets, d_keys, c.d_error);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

// Radius neighbourhoods of a query batch as CSR rows addressed by the query's slot, in two steps so the caller can look
// at the total before materialising anything:
//   radius_count       counts / offsets (nq + 1 entries, offsets[nq] = total); synchronises once to read the total
//   radius_fill_sorted keys = (d2 bits << 32) | original index, ascending inside every row (= ascending (d2, index))
void radius_count(Ctx& c, const Index& idx, const float4* d_q, size_t nq, float r2, DevBuf<unsigned long long>& counts,
                  DevBuf<unsigned long long>& offsets, unsigned long long& total)
{
  cudaStream_t st = c.stream;
  counts.alloc(nq + 1, st);
  offsets.alloc(nq + 1, st);
  PCLB_CUDA(cudaMemsetAsync(counts.p, 0, (nq + 1) * sizeof(unsigned long long), st));
  launch_radius_count(c, idx, d_q, nq, r2, counts.p);
  size_t tb = 0;
  PCLB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, counts.p, offsets.p, (int)(nq + 1), st));
  DevBuf<unsigned char> tmp;
  tmp.alloc(tb, st);
  PCLB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, counts.p, offsets.p, (int)(nq + 1), st));
  ++c.launches;
  total = 0;
  PCLB_CUDA(cudaMemcpyAsync(&total, offsets.p + nq, sizeof(total), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
}

void radius_fill_sorted(Ctx& c, const Index& idx, const float4* d_q, size_t nq, float r2,
                        const DevBuf<unsigned long long>& offsets, unsigned long long total,
                        DevBuf<unsigned long long>& keys_sorted)
{
  if (total == 0)
    return;
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(total < (unsigned long long)std::numeric_limits<int>::max(), PCLB200_ERR_INVALID,
               "radius search result exceeds 2^31 neighbours; lower the radius or set max_nn (<= 32 is searched without "
               "materialising the whole ball)");
  DevBuf<unsigned long long> keys;
  keys.alloc(total, st);
  keys_sorted.alloc(total, st);
  launch_radius_fill(c, idx, d_q, nq, r2, offsets.p, keys.p);
  size_t tb2 = 0;
  PCLB_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, tb2, keys.p, keys_sorted.p, (int)total, (int)nq, offsets.p,
                                               offsets.p + 1, st));
  DevBuf<unsigned char> tmp2;
  tmp2.alloc(tb2, st);
  PCLB_CUDA(cub::DeviceSegmentedSort::SortKeys(tmp2.p, tb2, keys.p, keys_sorted.p, (int)total, (int)nq, offsets.p,
                                               offsets.p + 1, st));
  c.launches += 3;
}

void radius_csr(Ctx& c, const Index& idx, const float4* d_q, size_t nq, float r2, DevBuf<unsigned long long>& counts,
                DevBuf<unsigned long long>& offsets, DevBuf<unsigned long long>& keys_sorted, unsigned long long& total)
{
  radius_count(c, idx, d_q, nq, r2, counts, offsets, total);
  radius_fill_sorted(c, idx, d_q, nq, r2, offsets, total, keys_sorted);
}

// ---- radius search of a caller's queries ------------------------------------------------------------------------------
__global__ void k_unpack_keys(const unsigned long long* __restrict__ keys, size_t n, int32_t* __restrict__ idx,
                              float* __restrict__ d2)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) {
    unsigned long long k = keys[i];
    idx[i] = (int32_t)(unsigned)(k & 0xffffffffULL);
    d2[i] = __uint_as_float((unsigned)(k >> 32));
  }
}

// keep only the first max_nn entries of every (sorted) segment
__global__ void k_truncate_segments(const unsigned long long* __restrict__ keys,
                                    const unsigned long long* __restrict__ off_in,
                                    const unsigned long long* __restrict__ off_out, size_t nq,
                                    unsigned long long* __restrict__ out)
{
  size_t q = blockIdx.x;
  if (q >= nq)
    return;
  const unsigned long long b = off_in[q], bo = off_out[q], len = off_out[q + 1] - off_out[q];
  for (unsigned long long j = threadIdx.x; j < len; j += blockDim.x)
    out[bo + j] = keys[b + j];
}

// max_nn <= 32 radius search = "the max_nn nearest inside the ball": k-NN rows (-1 padded) -> CSR
__global__ void k_count_row_entries(const int32_t* __restrict__ rows, size_t nq, int k, unsigned long long* __restrict__ counts)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  unsigned long long c = 0;
  for (int j = 0; j < k; ++j)
    if (rows[i * (size_t)k + j] >= 0)
      ++c;
  counts[i] = c;
}

__global__ void k_pack_rows(const int32_t* __restrict__ rows, const float* __restrict__ rows_d2, size_t nq, int k,
                            const unsigned long long* __restrict__ offsets, int32_t* __restrict__ idx,
                            float* __restrict__ d2)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  unsigned long long o = offsets[i];
  for (int j = 0; j < k; ++j) {
    const int32_t v = rows[i * (size_t)k + j];
    if (v < 0)
      break;  // rows are filled from the front
    idx[o] = v;
    d2[o] = rows_d2[i * (size_t)k + j];
    ++o;
  }
}

__global__ void k_clamp_counts(const unsigned long long* __restrict__ in, size_t n, unsigned long long cap,
                               unsigned long long* __restrict__ out)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n)
    out[i] = in[i] < cap ? in[i] : cap;
}

__global__ void k_offsets_to_i64(const unsigned long long* __restrict__ in, size_t n, int64_t* __restrict__ out)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n)
    out[i] = (int64_t)in[i];
}

void radius_search(Ctx& c, const Index& idx, const void* queries, size_t nq, size_t stride, double radius, unsigned max_nn,
                 int64_t* out_offsets, const std::function<RadiusSinkBuffers(unsigned long long)>& sink)
{
  cudaStream_t st = c.stream;
  auto write_offsets = [&](const unsigned long long* d_off) {
    if (is_device_ptr(out_offsets)) {
      k_offsets_to_i64<<<grid_for(nq + 1, 256), 256, 0, st>>>(d_off, nq + 1, out_offsets);
      ++c.launches;
    }
    else {
      static_assert(sizeof(unsigned long long) == sizeof(int64_t), "offset width");
      PCLB_CUDA(cudaMemcpyAsync(out_offsets, d_off, (nq + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    }
  };
  const float r2 = (float)(radius * radius);  // kdtree_flann.hpp:398
  if (max_nn == 0 || (size_t)max_nn > idx.n_valid)
    max_nn = (unsigned)idx.n_valid;            // :382-383
  DevBuf<float4> dense;
  QueryBatch qb = load_queries(c, idx, queries, nq, stride, nullptr, 0, dense);
  DevBuf<unsigned long long> counts, offsets, keys_sorted;
  unsigned long long total = 0;
  {
    ProfScope ps(c, "radius_count");
    radius_count(c, idx, qb.q.p, nq, r2, counts, offsets, total);
  }
  // KNNRadiusResultSet semantics (kdtree_flann.hpp:382-391): the max_nn nearest among those with d2 < r2.  Normally
  // the whole ball is materialised, sorted and cut (the passes below: ~3 ms per million queries at ~30 neighbours).
  // When the balls hold far more than max_nn points that would move (or overflow on) data that is thrown away, so
  // for max_nn <= 32 the register k-NN kernel runs instead, started with the pruning bound just below r2 (every
  // d2 < r2 is <= that bound; a candidate AT the bound still enters through the index tie rule).
  if ((size_t)max_nn < idx.n_valid && max_nn <= 32 && total > 16ULL * (unsigned long long)nq * max_nn) {
    const int k = (int)max_nn;
    DevBuf<int32_t> rows;
    DevBuf<float> rows_d2;
    rows.alloc(nq * (size_t)k, st);
    rows_d2.alloc(nq * (size_t)k, st);
    {
      ProfScope ps(c, "radius_knn");
      launch_knn(c, idx, qb.q.p, nq, k, std::nextafter(r2, -std::numeric_limits<float>::infinity()), rows.p, rows_d2.p);
    }
    DevBuf<unsigned long long> cnt, off;
    cnt.alloc(nq + 1, st);
    off.alloc(nq + 1, st);
    PCLB_CUDA(cudaMemsetAsync(cnt.p, 0, (nq + 1) * sizeof(unsigned long long), st));
    k_count_row_entries<<<grid_for(nq, 256), 256, 0, st>>>(rows.p, nq, k, cnt.p);
    size_t tb = 0;
    PCLB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt.p, off.p, (int)(nq + 1), st));
    DevBuf<unsigned char> tmp;
    tmp.alloc(tb, st);
    PCLB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, cnt.p, off.p, (int)(nq + 1), st));
    c.launches += 2;
    unsigned long long kept = 0;
    PCLB_CUDA(cudaMemcpyAsync(&kept, off.p + nq, sizeof(kept), cudaMemcpyDeviceToHost, st));
    write_offsets(off.p);
    PCLB_CUDA(cudaStreamSynchronize(st));
    const RadiusSinkBuffers o = sink(kept);
    if (kept > 0 && o.idx && o.d2) {
      DevBuf<int32_t> di;
      DevBuf<float> dd;
      k_pack_rows<<<grid_for(nq, 256), 256, 0, st>>>(rows.p, rows_d2.p, nq, k, off.p, out_on_device(c, o.idx, kept, di),
                                                     out_on_device(c, o.d2, kept, dd));
      ++c.launches;
      copy_out(c, o.idx, di, kept);
      copy_out(c, o.d2, dd, kept);
      PCLB_CUDA(cudaStreamSynchronize(st));
    }
    check_device_error(c);
    return;
  }
  {
    ProfScope ps(c, "radius");
    radius_fill_sorted(c, idx, qb.q.p, nq, r2, offsets, total, keys_sorted);
  }
  const unsigned long long* d_final_keys = nullptr;
  const unsigned long long* d_final_off = offsets.p;
  unsigned long long final_total = total;
  DevBuf<unsigned long long> counts2, offsets2, keys_trunc;
  if (total > 0) {
    d_final_keys = keys_sorted.p;
    if ((size_t)max_nn < idx.n_valid) {  // KNNRadius semantics: the max_nn nearest inside the ball
      counts2.alloc(nq + 1, st);
      offsets2.alloc(nq + 1, st);
      PCLB_CUDA(cudaMemsetAsync(counts2.p, 0, (nq + 1) * sizeof(unsigned long long), st));
      k_clamp_counts<<<grid_for(nq, 256), 256, 0, st>>>(counts.p, nq, (unsigned long long)max_nn, counts2.p);
      size_t tb = 0;
      PCLB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, counts2.p, offsets2.p, (int)(nq + 1), st));
      DevBuf<unsigned char> tmp;
      tmp.alloc(tb, st);
      PCLB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, counts2.p, offsets2.p, (int)(nq + 1), st));
      PCLB_CUDA(cudaMemcpyAsync(&final_total, offsets2.p + nq, sizeof(final_total), cudaMemcpyDeviceToHost, st));
      PCLB_CUDA(cudaStreamSynchronize(st));
      keys_trunc.alloc(std::max<unsigned long long>(final_total, 1), st);
      k_truncate_segments<<<(unsigned)nq, 64, 0, st>>>(keys_sorted.p, offsets.p, offsets2.p, nq, keys_trunc.p);
      c.launches += 3;
      d_final_keys = keys_trunc.p;
      d_final_off = offsets2.p;
    }
  }
  write_offsets(d_final_off);
  PCLB_CUDA(cudaStreamSynchronize(st));
  const RadiusSinkBuffers o = sink(final_total);
  if (final_total > 0 && o.idx && o.d2) {
    DevBuf<int32_t> di;
    DevBuf<float> dd;
    k_unpack_keys<<<grid_for(final_total, 256), 256, 0, st>>>(d_final_keys, final_total,
                                                              out_on_device(c, o.idx, final_total, di),
                                                              out_on_device(c, o.d2, final_total, dd));
    ++c.launches;
    copy_out(c, o.idx, di, final_total);
    copy_out(c, o.d2, dd, final_total);
    PCLB_CUDA(cudaStreamSynchronize(st));
  }
  check_device_error(c);
}

// ---- normals: eigen33 / moments (knn_warp.cuh) ------------------------------------------------------------------
#ifndef PCLB_KNN_TARGET_X10
#define PCLB_KNN_TARGET_X10 12
#endif
#ifndef PCLB_KNN_LEVEL_X10
#define PCLB_KNN_LEVEL_X10 10
#endif

// Where the warp kernel starts.  The ball it certifies should hold a little more than k points: from the occupancy of
// the cell levels, n / occupied(l) points per cell and the ratio of two levels give the cloud's local density and
// intrinsic dimension (4 per level = a surface, 8 = a volume), hence the radius of a ball of ~1.2 k + 4 points.  The
// start level is the finest whose half cell holds ~k points by that estimate (the ball's box must span <= 2 cells per axis); the
// first attempt uses the sized ball when it is well inside half a cell, later attempts half a cell of ever coarser
// levels.  Only speed depends on this estimate: an attempt counts only if the k-th distance certifies it.
struct WarpKnnStart {
  int level = 0;      // 0: no level fits (tiny cloud) -> per-thread kernels
  float r_first = 0;  // 0: start with half a cell
};
static WarpKnnStart warp_knn_start(const Index& idx, int k)
{
  WarpKnnStart w;
  const CellTableHost& c = idx.cells;
  auto avg = [&](int l) { return (double)idx.n_valid / (double)std::max<unsigned long long>(1, c.occupied[l]); };
  int ref = 0;
  for (int l = 2; l <= c.bmax; ++l)
    if (c.occupied[l] > 0 && c.occupied[l - 1] > 0 && avg(l) >= 8.0)
      ref = l;
  if (ref < 2)
    return w;
  const double dim = std::min(3.0, std::max(1.0, std::log2(avg(ref - 1) / avg(ref))));
  const double unit_ball = std::pow(M_PI, 0.5 * dim) / std::tgamma(0.5 * dim + 1.0);
  const double width = (double)(1u << (21 - ref)) / (double)idx.morton_scale;
  auto ball_of = [&](double points) { return width * std::pow(points / (avg(ref) * unit_ball), 1.0 / dim); };
  const double radius = ball_of(PCLB_KNN_TARGET_X10 * 0.1 * k + 4.0);
  // the level: the finest whose half cell still holds ~k points by the estimate, which runs ~15 % large on tilted
  // surfaces (a level finer gathers 2-3 times fewer candidates,
  // measured 16 vs 20 ms at k = 16, and its half-cell ball certifies most queries)
  const double need = ball_of(PCLB_KNN_LEVEL_X10 * 0.1 * k);
  for (int l = 1; l <= c.bmax; ++l) {
    const double half = 0.5 * 0.999 * (double)(1u << (21 - l)) / (double)idx.morton_scale;
    if (c.occupied[l] > 0 && half >= need)
      w.level = l;
  }
  if (w.level >= 1) {
    const double half = 0.5 * 0.999 * (double)(1u << (21 - w.level)) / (double)idx.morton_scale;
    if (radius < 0.85 * half)
      w.r_first = (float)radius;
  }
  return w;
}

static bool warp_knn_lists(Ctx& c, const Index& idx, const float4* d_q, size_t nq, int k, int32_t* d_out_idx,
                           float* d_out_d2, DevBuf<unsigned char>& redo)
{
  if (!(idx.cell_slots.p && idx.node_leaves.p) || k < 12 || k > 32 || (size_t)k > idx.n_valid)
    return false;
  const WarpKnnStart w0 = warp_knn_start(idx, k);
  if (w0.level < 1)
    return false;
  cudaStream_t s = c.stream;
  redo.alloc(nq, s);
  PCLB_CUDA(cudaMemsetAsync(redo.p, 0, nq, s));
  const unsigned wg = (unsigned)std::min<size_t>((nq + 255) / 256, (size_t)c.sm_count * 8);
  k_knn_warp<false><<<wg, 256, 0, s>>>(tree_view(idx), idx.node_leaves.p, w0.level, w0.r_first, d_q, nq, k, d_out_idx, d_out_d2, 0.f, 0.f, 0.f,
                                      nullptr, nullptr, redo.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  return true;
}

void launch_normals_radius(Ctx& c, Index& idx, const float4* d_q, size_t nq, float r2, const float vp[3], float4* d_out,
                           int* d_not_dense)
{
  if (!nq)
    return;
  cudaStream_t s = c.stream;
  DevBuf<unsigned long long> counts, offsets, keys;
  unsigned long long total = 0;
  radius_csr(c, idx, d_q, nq, r2, counts, offsets, keys, total);
  ensure_pos_of_orig(c, idx);
  k_normals_from_csr<<<grid_for(nq, 128), 128, 0, s>>>(idx.pts.p, idx.pos_of_orig.p, d_q, nq, offsets.p, keys.p, vp[0],
                                                      vp[1], vp[2], d_out, d_not_dense);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

void launch_normals(Ctx& c, Index& idx, const float4* d_q, size_t nq, int k, const float vp[3], float4* d_out,
                    int* d_not_dense)
{
  if (!nq)
    return;
  cudaStream_t s = c.stream;
  const unsigned g = grid_for(nq, 128);
  if (k > 32) {
    // large neighbourhoods: materialise the exact k-NN lists (any-k kernel), then fold them
    ensure_pos_of_orig(c, idx);
    DevBuf<int32_t> li;
    DevBuf<float> ld;
    li.alloc(nq * (size_t)k, s);
    ld.alloc(nq * (size_t)k, s);
    launch_knn(c, idx, d_q, nq, k, __builtin_inff(), li.p, ld.p);
    k_normals_from_lists<<<g, 128, 0, s>>>(idx.pts.p, idx.pos_of_orig.p, d_q, nq, k, li.p, 0, vp[0], vp[1], vp[2], d_out,
                                           d_not_dense);
    ++c.launches;
    PCLB_CUDA(cudaGetLastError());
    return;
  }
  DevBuf<unsigned char> redo;
  const unsigned char* only = nullptr;
  {
    const WarpKnnStart w0 = (idx.cell_slots.p && idx.node_leaves.p && k >= 12) ? warp_knn_start(idx, k) : WarpKnnStart{};
    if (w0.level >= 1 && (size_t)k <= idx.n_valid) {
      redo.alloc(nq, s);
      PCLB_CUDA(cudaMemsetAsync(redo.p, 0, nq, s));
      const unsigned wg = (unsigned)std::min<size_t>((nq + 255) / 256, (size_t)c.sm_count * 8);
      k_knn_warp<true><<<wg, 256, 0, s>>>(tree_view(idx), idx.node_leaves.p, w0.level, w0.r_first, d_q, nq, k, nullptr, nullptr, vp[0], vp[1],
                                         vp[2], d_out, d_not_dense, redo.p);
      ++c.launches;
      only = redo.p;
    }
  }
#define PCLB_NRM_CASE(KK)                                                                                              \
  k_normals<KK><<<g, 128, 0, s>>>(idx.nodes.p, idx.pts.p, idx.root, d_q, nq, k, vp[0], vp[1], vp[2], d_out, d_not_dense, \
                                  c.d_error, only)
  if (k <= 4) PCLB_NRM_CASE(4);
  else if (k <= 8) PCLB_NRM_CASE(8);
  else if (k <= 10) PCLB_NRM_CASE(10);
  else if (k <= 16) PCLB_NRM_CASE(16);
  else if (k <= 20) PCLB_NRM_CASE(20);
  else PCLB_NRM_CASE(32);
#undef PCLB_NRM_CASE
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

// launch_normals of every set of a batch in one sequence: each set takes the path its single call would (the lists for
// k > 32, else the warp kernel where launch_normals runs it, then the per-thread kernel over what is left), so every row
// is the single call's.  The queries are already sorted by set, and each set's in the order of its own index's frame.
void launch_normals_batch(Ctx& c, Index* const* idx, int B, const long long* d_offsets, const float4* d_q, size_t nq, int k,
                          const float* vps, float4* d_out, int* d_flags)
{
  cudaStream_t s = c.stream;
  const unsigned g = grid_for(nq, 128);
  if (k > 32)
    for (int b = 0; b < B; ++b)
      ensure_pos_of_orig(c, *idx[b]);
  std::vector<NormalsCloud> h(B);
  bool any_warp = false;
  for (int b = 0; b < B; ++b) {
    const Index& I = *idx[b];
    NormalsCloud& e = h[b];
    e.tree = tree_view(I);
    e.node_leaves = I.node_leaves.p;
    e.pos_of_orig = k > 32 ? I.pos_of_orig.p : nullptr;
    const WarpKnnStart w =
        (k <= 32 && I.cell_slots.p && I.node_leaves.p && k >= 12) ? warp_knn_start(I, k) : WarpKnnStart{};
    const bool warp = w.level >= 1 && (size_t)k <= I.n_valid;
    e.level = warp ? w.level : 0;
    e.r_first = warp ? w.r_first : 0.f;
    for (int d = 0; d < 3; ++d)
      e.vp[d] = vps[3 * b + d];
    e.not_dense = d_flags + b;
    any_warp = any_warp || warp;
  }
  DevBuf<NormalsCloud> table;
  table.alloc(B, s);
  PCLB_CUDA(cudaMemcpyAsync(table.p, h.data(), B * sizeof(NormalsCloud), cudaMemcpyHostToDevice, s));
  if (k > 32) {
    DevBuf<int32_t> li;
    DevBuf<float> ld;
    li.alloc(nq * (size_t)k, s);
    ld.alloc(nq * (size_t)k, s);
    k_knn_any_batch<<<g, 128, 0, s>>>(table.p, d_offsets, B, d_q, nq, k, __builtin_inff(), li.p, ld.p, c.d_error);
    k_normals_from_lists_batch<<<g, 128, 0, s>>>(table.p, d_offsets, B, d_q, nq, k, li.p, d_out);
    c.launches += 2;
    PCLB_CUDA(cudaGetLastError());
    return;
  }
  DevBuf<unsigned char> redo;
  const unsigned char* only = nullptr;
  if (any_warp) {
    redo.alloc(nq, s);
    PCLB_CUDA(cudaMemsetAsync(redo.p, 0, nq, s));
    const unsigned wg = (unsigned)std::min<size_t>((nq + 255) / 256, (size_t)c.sm_count * 8);
    k_knn_warp_batch<<<wg, 256, 0, s>>>(table.p, d_offsets, B, d_q, nq, k, d_out, redo.p);
    ++c.launches;
    only = redo.p;
  }
#define PCLB_NRM_CASE(KK) \
  k_normals_batch<KK><<<g, 128, 0, s>>>(table.p, d_offsets, B, d_q, nq, k, d_out, c.d_error, only)
  if (k <= 4) PCLB_NRM_CASE(4);
  else if (k <= 8) PCLB_NRM_CASE(8);
  else if (k <= 10) PCLB_NRM_CASE(10);
  else if (k <= 16) PCLB_NRM_CASE(16);
  else if (k <= 20) PCLB_NRM_CASE(20);
  else PCLB_NRM_CASE(32);
#undef PCLB_NRM_CASE
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

}  // namespace pclb200
