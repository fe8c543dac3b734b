// shard_filter.cu — k-NN queries, k-NN statistics and the two outlier filters over a map sharded across the ranks of a
// communicator (pclb200_knn_sharded, pclb200_knn_stats_sharded, pclb200_statistical_outlier_sharded,
// pclb200_radius_outlier_sharded; capi.cu).  Each rank builds the local map of its own queries with the k of the call
// (shard_normals.cu: sharded_local_map, the argument of DESIGN.md §5, "Normals of a sharded map"): its tile plus every
// point of the other tiles within the tile's k-th distance of a query, sorted by id.  Every whole-map k-NN list of a query
// lies in it, and record order is id order, so the unchanged launch_knn / launch_knn_stats on it return the whole map's
// lists and statistics; k_sf_row_ids turns the rows' records back into ids (DESIGN.md §5, "Filters of a sharded map").
//
//   k_eff     min(k, distinct finite ids of the map): k when some tile alone holds k points (one u64 minimum over the
//             ranks' ~n_valid); else every tile is smaller than k, and the ranks all-gather their ids and count them.
//   SOR       each rank sums (valid, d, float(d * d)) over its queries in slot order (a fixed-grid sum) into its table of
//             comm_segment_tables, three words; publish; every rank folds every rank's words in rank order and applies
//             the reference's mean / variance / threshold; release; the mask on the device.
//   ROR       one u64 minimum of the ranks' is_dense flags picks the rule on every rank; the mask on the device.
// Radius search (pclb200_radius_sharded, pclb200_radius_into_sharded) and GICP covariances (pclb200_gicp_covariances_sharded)
// run the unchanged radius_search / gicp_covariances on the local map of the radius, or of k for the tile's own records
// (DESIGN.md §5, "Radius search and GICP covariances of a sharded map").  Their refusals travel in one u64 minimum of
// the ranks' verdicts before any halo moves.
#include <limits>
#include <memory>
#include <vector>

#include "internal.cuh"
#include "shard_filter_kernels.cuh"

namespace pclb200 {

bool comm_active(const Ctx& c);
int comm_nranks(const Ctx& c);
int comm_rank(const Ctx& c);
template <typename K>
size_t sort_unique(Ctx& c, const K* keys, size_t n, DevBuf<K>& out);  // shard_cluster.cu
void gicp_covariances(Ctx& c, Index& idx, const void* pts, size_t n, size_t stride, int k, double gicp_epsilon,
                      double* out);  // icp.cu

static const ShardedMapStages kFilterStages{"sharded_filter_bound", "sharded_filter_halo", "sharded_filter_build"};

// The caller's queries staged densely (kept: the masks read them in input order) and the local map of this rank for
// neighbourhoods of k, with its ids by record.
struct FilterMap {
  DevBuf<float4> dense;
  std::unique_ptr<Index> local;
  HaloTrace trace;
  QueryBatch qb;  // the queries in the local map's frame
};

static void filter_map(Ctx& c, const Index& tile, const void* pts, size_t n, size_t stride, const int32_t* indices,
                       size_t n_idx, int k, FilterMap& fm)
{
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID,
               "sharded k-NN and filters need an active communicator (pclb200_comm_init or pclb200_comm_export / _import)");
  PCLB_REQUIRE(tile.labelled, PCLB200_ERR_INVALID,
               "sharded k-NN and filters: every rank's tile must be built with pclb200_index_build_ids");
  PCLB_REQUIRE(k > 0, PCLB200_ERR_INVALID, "sharded k-NN and filters: k must be positive");
  const size_t nq = indices ? n_idx : n;
  fm.dense.alloc(nq, c.stream);
  if (nq)
    load_xyz_as_float4(c, pts, n, stride, indices, n_idx, fm.dense.p, c.stream);
  fm.local.reset(sharded_local_map(c, tile, fm.dense.p, nq, k, 0.f, kFilterStages, &fm.trace));
  if (nq)
    make_query_batch(c, *fm.local, fm.dense.p, nq, fm.qb);
}

// mean and kth (each nullable) of every query, by input position, as launch_knn_stats on one index of the whole map
static void local_stats(Ctx& c, FilterMap& fm, size_t nq, int k, float* d_mean, float* d_kth)
{
  ProfScope ps(c, "sharded_filter_stats");
  if (nq)
    launch_knn_stats(c, *fm.local, fm.qb.q.p, nq, k, d_mean, d_kth);
}

int knn_sharded(Ctx& c, const Index& tile, const void* queries, size_t nq, size_t stride, int k, int32_t* d_idx,
                float* d_d2)
{
  cudaStream_t st = c.stream;
  FilterMap fm;
  filter_map(c, tile, queries, nq, stride, nullptr, 0, k, fm);
  {
    ProfScope ps(c, "sharded_filter_knn");
    if (nq) {
      const size_t n_out = nq * (size_t)k;
      launch_knn(c, *fm.local, fm.qb.q.p, nq, k, std::numeric_limits<float>::infinity(), d_idx, d_d2);
      k_sf_row_ids<<<persistent_blocks(c, n_out), 256, 0, st>>>(d_idx, n_out, fm.trace.local_ids.p);
      ++c.launches;
      PCLB_CUDA(cudaGetLastError());
    }
  }
  fm.local.reset();
  return sharded_keff(c, tile, k);
}

// Collective: the minimum of one word over the ranks, the same on every rank
unsigned long long ranks_min(Ctx& c, unsigned long long word)
{
  cudaStream_t st = c.stream;
  DevBuf<unsigned long long> w;
  w.alloc(1, st);
  PCLB_CUDA(cudaMemcpyAsync(w.p, &word, sizeof(word), cudaMemcpyHostToDevice, st));
  comm_allreduce_u64(c, w.p, w.p, 1, kU64Min);
  PCLB_CUDA(cudaMemcpyAsync(&word, w.p, sizeof(word), cudaMemcpyDeviceToHost, st));
  check_device_error(c);
  return word;
}

// Collective: every rank's verdict on its own arguments (fault: this rank's reason to refuse, or null) in one u64
// minimum, so that a refusal happens on every rank before anything moves.  The ranks' query counts may differ, so unlike
// the ICP session's check (icp.cu: require_same_count) no count travels with it.
static void require_every_rank_accepts(Ctx& c, const char* fault)
{
  const unsigned long long all = ranks_min(c, fault ? 0 : 1);
  PCLB_REQUIRE(!fault, PCLB200_ERR_INVALID, fault);
  PCLB_REQUIRE(all, PCLB200_ERR_INVALID, "another rank refused its arguments");
}

// Radius search of this rank's queries on the whole map (DESIGN.md §5, "Radius search and GICP covariances of a sharded
// map"): the local map of every point of the other tiles within r2 of the queries' box, then the unchanged radius_search
// on it.  Its lists go to device buffers, whichever the caller's are, so that the local record numbers become ids
// (k_sf_row_ids) before they leave the device; both paths of radius_search (sorted keys, register k-NN rows) unpack to
// such lists.  sink(total) is called once on every rank, a rank with no query included (total 0), so that it can hold a
// collective exchange.  Returns the total delivered (0 when the sink declined the lists).
unsigned long long radius_sharded(Ctx& c, const Index* tile, const void* queries, size_t nq, size_t stride, double radius,
                                  unsigned max_nn, int64_t* out_offsets,
                                  const std::function<RadiusSinkBuffers(unsigned long long)>& sink, const char* fault)
{
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID,
               "sharded radius search needs an active communicator (pclb200_comm_init or pclb200_comm_export / _import)");
  if (!fault && !tile->labelled)
    fault = "sharded radius search: every rank's tile must be built with pclb200_index_build_ids";
  require_every_rank_accepts(c, fault);
  const float r2 = (float)(radius * radius);  // what radius_search compares against: d2 < r2
  DevBuf<float4> dense;
  dense.alloc(nq, st);
  if (nq)
    load_xyz_as_float4(c, queries, nq, stride, nullptr, 0, dense.p, st);
  // r2 of 0 or NaN holds no point: no halo (a query box of its own would still fetch the points that coincide with it)
  static const ShardedMapStages stages{"sharded_radius_halo", "sharded_radius_halo", "sharded_radius_build"};
  HaloTrace trace;
  std::unique_ptr<Index> local(sharded_local_map(c, *tile, dense.p, r2 > 0.f ? nq : 0, 0, r2, stages, &trace));
  RadiusSinkBuffers to{nullptr, nullptr};
  DevBuf<int32_t> di;
  DevBuf<float> dd;
  unsigned long long n = 0;
  auto on_device = [&](unsigned long long total) {
    to = sink(total);
    if (!to.idx || !to.d2 || !total)
      return RadiusSinkBuffers{nullptr, nullptr};
    n = total;
    return RadiusSinkBuffers{out_on_device(c, to.idx, n, di), out_on_device(c, to.d2, n, dd)};
  };
  if (nq) {
    ProfScope ps(c, "sharded_radius_search");
    radius_search(c, *local, dense.p, nq, sizeof(float4), radius, max_nn, out_offsets, on_device);
  }
  else {
    const int64_t zero = 0;
    PCLB_CUDA(cudaMemcpy(out_offsets, &zero, sizeof(zero), cudaMemcpyDefault));
    on_device(0);
  }
  if (n) {
    int32_t* d_idx = di.p ? di.p : to.idx;
    k_sf_row_ids<<<persistent_blocks(c, n), 256, 0, st>>>(d_idx, n, trace.local_ids.p);
    ++c.launches;
    PCLB_CUDA(cudaGetLastError());
    copy_out(c, to.idx, di, n);
    copy_out(c, to.d2, dd, n);
  }
  check_device_error(c);
  return n;
}

// GICP covariances of this rank's tile records on the whole map: the local map of their k nearest (the argument of the
// filters), then the unchanged gicp_covariances on it, an ordinary index, with the staged records as its queries.
void gicp_covariances_sharded(Ctx& c, const Index* tile, const void* pts, size_t n, size_t stride, int k,
                              double gicp_epsilon, double* out, const char* fault)
{
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID,
               "sharded GICP covariances need an active communicator (pclb200_comm_init or pclb200_comm_export / _import)");
  if (!fault && !tile->labelled)
    fault = "sharded GICP covariances: every rank's tile must be built with pclb200_index_build_ids";
  else if (!fault && k < 1)
    fault = "sharded GICP covariances: k must be positive";
  else if (!fault && n != tile->n_cloud)
    fault = "sharded GICP covariances: pts must be the records the tile was built from (n = its record count)";
  require_every_rank_accepts(c, fault);
  DevBuf<float4> dense;
  dense.alloc(n, st);
  if (n)
    load_xyz_as_float4(c, pts, n, stride, nullptr, 0, dense.p, st);
  static const ShardedMapStages stages{"sharded_gicp_bound", "sharded_gicp_halo", "sharded_gicp_build"};
  std::unique_ptr<Index> local(sharded_local_map(c, *tile, dense.p, n, k, 0.f, stages));
  ProfScope ps(c, "sharded_gicp_covariances");
  gicp_covariances(c, *local, dense.p, n, sizeof(float4), k, gicp_epsilon, out);
}

// k_eff: the whole map's clamp (kdtree_flann.hpp:241-242), the same on every rank (collective)
int sharded_keff(Ctx& c, const Index& tile, int k)
{
  cudaStream_t st = c.stream;
  DevBuf<unsigned long long> w;
  w.alloc(1, st);
  const unsigned long long not_n = ~(unsigned long long)tile.n_valid;
  PCLB_CUDA(cudaMemcpyAsync(w.p, &not_n, sizeof(not_n), cudaMemcpyHostToDevice, st));
  comm_allreduce_u64(c, w.p, w.p, 1, kU64Min);
  unsigned long long largest = 0;
  PCLB_CUDA(cudaMemcpyAsync(&largest, w.p, sizeof(largest), cudaMemcpyDeviceToHost, st));
  check_device_error(c);
  largest = ~largest;
  if (largest >= (unsigned long long)k)
    return k;
  // every tile holds fewer than k points: count the distinct ids of the map (padding ids, kSentinelIndex, excluded)
  DevBuf<unsigned long long> ids, all, uniq;
  ids.alloc(tile.pts.n, st);
  if (tile.pts.n) {
    k_sf_tile_ids<<<persistent_blocks(c, tile.pts.n), 256, 0, st>>>(tile.pts.p, tile.pts.n, ids.p);
    ++c.launches;
    PCLB_CUDA(cudaGetLastError());
  }
  const size_t total = allgather_u64(c, ids.p, ids.n, all);
  size_t m = sort_unique(c, all.p, total, uniq);
  if (m) {
    unsigned long long last = 0;
    PCLB_CUDA(cudaMemcpyAsync(&last, uniq.p + (m - 1), sizeof(last), cudaMemcpyDeviceToHost, st));
    check_device_error(c);
    m -= last == (unsigned long long)kSentinelIndex;
  }
  return (int)m;
}

void knn_stats_sharded(Ctx& c, const Index& tile, const void* pts, size_t n, size_t stride, const int32_t* indices,
                       size_t n_idx, int k, float* d_mean, float* d_kth)
{
  FilterMap fm;
  filter_map(c, tile, pts, n, stride, indices, n_idx, k, fm);
  local_stats(c, fm, indices ? n_idx : n, k, d_mean, d_kth);
}

void statistical_outlier_sharded(Ctx& c, const Index& tile, const void* pts, size_t n, size_t stride,
                                 const int32_t* indices, size_t n_idx, int mean_k, double std_mul, int negative,
                                 unsigned char* d_keep, double* d_stats)
{
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(mean_k > 0, PCLB200_ERR_INVALID, "sharded statistical outlier removal: mean_k must be positive");
  const size_t nq = indices ? n_idx : n;
  FilterMap fm;
  filter_map(c, tile, pts, n, stride, indices, n_idx, mean_k + 1, fm);  // statistical_outlier_removal.hpp:84: mean_k + 1
  DevBuf<float> mean;
  mean.alloc(nq, st);
  local_stats(c, fm, nq, mean_k + 1, mean.p, nullptr);
  fm.local.reset();

  ProfScope ps(c, "sharded_filter_sor");
  const int R = comm_nranks(c);
  std::vector<unsigned long long> words(R, kSorWords);
  const PeerTables t = comm_segment_tables(c, words.data(), sizeof(unsigned long long));
  const unsigned grid = persistent_blocks(c, nq);
  DevBuf<double> partials, accum;
  DevBuf<unsigned> counter;
  partials.alloc((size_t)grid * kAccum, st);
  accum.alloc(kAccum, st);
  counter.alloc(1, st);
  PCLB_CUDA(cudaMemsetAsync(counter.p, 0, sizeof(unsigned), st));
  k_sf_sor_partials<<<grid, 256, 0, st>>>(fm.dense.p, mean.p, nq, GridSum{partials.p, counter.p, accum.p}, t.local);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  comm_tables_publish(c, t, kU64Sum);  // NCCL: the tables lie end to end in one zeroed table, one writer per word
  k_sf_sor_fold<<<1, 32, 0, st>>>(peer_table_set(t), std_mul, d_stats);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  comm_tables_release(c, t);
  if (nq) {
    k_sf_sor_mask<<<persistent_blocks(c, nq), 256, 0, st>>>(mean.p, nq, d_stats, negative, d_keep);
    ++c.launches;
    PCLB_CUDA(cudaGetLastError());
  }
}

void radius_outlier_sharded(Ctx& c, const Index& tile, const void* pts, size_t n, size_t stride, const int32_t* indices,
                            size_t n_idx, int is_dense, double radius, int min_pts, int negative, unsigned char* d_keep)
{
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(radius > 0.0, PCLB200_ERR_INVALID, "sharded radius outlier removal: radius must be positive");
  PCLB_REQUIRE(min_pts >= 0, PCLB200_ERR_INVALID, "sharded radius outlier removal: min_pts must not be negative");
  const size_t nq = indices ? n_idx : n;
  FilterMap fm;
  filter_map(c, tile, pts, n, stride, indices, n_idx, min_pts + 1, fm);  // radius_outlier_removal.hpp:86: min_pts + 1
  DevBuf<float> kth;
  kth.alloc(nq, st);
  local_stats(c, fm, nq, min_pts + 1, nullptr, kth.p);
  fm.local.reset();

  ProfScope ps(c, "sharded_filter_ror");
  DevBuf<unsigned long long> dense;  // the dense rule only when every rank's cloud is dense
  dense.alloc(1, st);
  const unsigned long long mine = is_dense ? 1 : 0;
  PCLB_CUDA(cudaMemcpyAsync(dense.p, &mine, sizeof(mine), cudaMemcpyHostToDevice, st));
  comm_allreduce_u64(c, dense.p, dense.p, 1, kU64Min);
  if (nq) {
    k_sf_ror_mask<<<persistent_blocks(c, nq), 256, 0, st>>>(fm.dense.p, kth.p, nq, dense.p, radius * radius,
                                                             (float)(radius * radius), negative, d_keep);
    ++c.launches;
    PCLB_CUDA(cudaGetLastError());
  }
}

}  // namespace pclb200
