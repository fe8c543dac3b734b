// shard_normals.cu — normal estimation over a map sharded across the ranks of a communicator (pclb200_normals_knn_sharded /
// _radius_sharded, capi.cu).  Each rank gathers, for its own queries, a halo out of the other ranks' tiles that provably
// holds every whole-map neighbour of every query, indexes its tile plus that halo as an ordinary index sorted by id, and
// runs the unchanged single-GPU normals on it (DESIGN.md §5, "Normals of a sharded map").  Clustering a sharded map
// (shard_cluster.cu) builds its local map here too, with the tile's points as the queries and the tolerance as the radius,
// and takes a HaloTrace of the exchange so that it can answer every received point back to its sender: the ids it
// received, and the ids it sent, read from its own table, where its segments are one run.
//
//   bound   rho_q^2 = the k-th nearest squared distance of q in this rank's tile (launch_knn_kth; +inf when the tile
//           holds fewer than k points), or r^2.  The tile is part of the map, so every member of q's whole-map list,
//           ties at the k-th distance included, lies within rho_q.
//   boxes   this rank's box = the union of [q - reach(rho_q), q + reach(rho_q)] over its finite queries, rounded outward;
//           one u64 minimum over every rank's 6 keys (the discipline of icp.cu: union_frame).
//   halo    every rank counts its tile points inside every other rank's box (one u64 sum of the R x R counts), writes
//           them into its table of comm_segment_tables, one segment per destination (peer_tables.cuh: the layout);
//           publish; every rank copies its segments out of every rank's table; release.  The peer path's tables are
//           peer-mapped and both steps are barriers; under PCLB200_REDUCE_NCCL they lie end to end in one zeroed table
//           and one u64 sum all-reduce, with one contributor per word, copies them exactly.
//   map     tile + halo sorted by id, duplicate ids (one point held by two ranks) dropped, indexed with
//           build_index_from_device: record numbers increase with the id, so the index's (d2, index) tie rule is the
//           whole map's (d2, id) rule and every list it returns is the whole map's, in the same order.
#include <cub/cub.cuh>

#include <algorithm>
#include <limits>
#include <memory>
#include <vector>

#include "internal.cuh"
#include "peer_tables.cuh"
#include "shard_normals_kernels.cuh"

namespace pclb200 {

bool comm_active(const Ctx& c);
int comm_nranks(const Ctx& c);
int comm_rank(const Ctx& c);

// Steps bound and boxes: every rank's box, on the device (kHaloBoxWords keys per rank, folded over the ranks)
static void exchange_boxes(Ctx& c, const Index& tile, const float4* d_q, size_t nq, int k, float r2, int R, int me,
                           const ShardedMapStages& stages, DevBuf<unsigned long long>& boxes)
{
  cudaStream_t st = c.stream;
  DevBuf<float> rho2;
  if (k > 0 && nq) {
    ProfScope ps(c, stages.bound);
    QueryBatch qb;
    make_query_batch(c, tile, d_q, nq, qb);
    rho2.alloc(nq, st);
    launch_knn_kth(c, tile, qb.q.p, nq, k, rho2.p);  // by slot = by dense position
  }
  ProfScope ps(c, stages.halo);
  boxes.alloc((size_t)kHaloBoxWords * R, st);
  PCLB_CUDA(cudaMemsetAsync(boxes.p, 0xff, boxes.bytes(), st));
  if (nq) {
    k_halo_box<<<persistent_blocks(c, nq), 256, 0, st>>>(d_q, rho2.p, r2, nq, boxes.p + (size_t)kHaloBoxWords * me);
    ++c.launches;
    PCLB_CUDA(cudaGetLastError());
  }
  comm_allreduce_u64(c, boxes.p, boxes.p, boxes.n, kU64Min);
}

Index* sharded_local_map(Ctx& c, const Index& tile, const float4* d_q, size_t nq, int k, float r2,
                         const ShardedMapStages& stages, HaloTrace* trace)
{
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID, "the local map of a sharded map needs an active communicator");
  const int R = comm_nranks(c), me = comm_rank(c);
  DevBuf<unsigned long long> boxes;
  exchange_boxes(c, tile, d_q, nq, k, r2, R, me, stages, boxes);

  // the halo: counts of every (source, destination) pair on every rank, then the points
  DevBuf<float4> local;  // tile, then halo
  size_t n_local = 0;
  {
    ProfScope ps(c, stages.halo);
    const size_t np = tile.pts.n;
    DevBuf<unsigned long long> d_cnt, cursor;
    d_cnt.alloc((size_t)R * R, st);
    PCLB_CUDA(cudaMemsetAsync(d_cnt.p, 0, d_cnt.bytes(), st));
    HaloOut count_only;
    memset(&count_only, 0, sizeof(count_only));
    count_only.count = d_cnt.p + (size_t)R * me;  // row `me`: what this rank sends to each rank
    k_halo_select<<<persistent_blocks(c, np), 256, 0, st>>>(tile.pts.p, np, boxes.p, R, me, count_only);
    ++c.launches;
    PCLB_CUDA(cudaGetLastError());
    comm_allreduce_u64(c, d_cnt.p, d_cnt.p, d_cnt.n, kU64Sum);
    std::vector<unsigned long long> cnt((size_t)R * R);
    PCLB_CUDA(cudaMemcpyAsync(cnt.data(), d_cnt.p, d_cnt.bytes(), cudaMemcpyDeviceToHost, st));
    check_device_error(c);
    const std::vector<unsigned long long> n_table = segment_table_sizes(cnt.data(), R);  // (s, s) is the tile itself
    unsigned long long halo = 0, all = 0;
    for (int s = 0; s < R; ++s) {
      all += n_table[s];
      if (s != me)
        halo += cnt[(size_t)s * R + me];
    }
    const size_t n_tile = cnt[(size_t)me * R + me];
    PCLB_REQUIRE(n_tile == tile.n_valid, PCLB200_ERR_INTERNAL, "sharded normals: the tile's points were miscounted");
    n_local = n_tile + halo;
    PCLB_REQUIRE(n_local < (size_t)0x7fffffff, PCLB200_ERR_INVALID,
                 "sharded normals: the tile and its halo exceed 2^31 - 1 points");
    local.alloc(n_local, st);
    HaloOut out;
    memset(&out, 0, sizeof(out));
    cursor.alloc(R, st);
    PCLB_CUDA(cudaMemsetAsync(cursor.p, 0, cursor.bytes(), st));
    out.count = cursor.p;
    out.dst[me] = local.p;
    PeerTables t;
    if (all) {  // every rank knows every count: all of them take this branch or none
      t = comm_segment_tables(c, n_table.data(), sizeof(float4));
      segment_writes(reinterpret_cast<float4*>(t.local), cnt.data(), R, me, out.dst);
    }
    k_halo_select<<<persistent_blocks(c, np), 256, 0, st>>>(tile.pts.p, np, boxes.p, R, me, out);
    ++c.launches;
    PCLB_CUDA(cudaGetLastError());
    if (trace) {  // this rank's segments are the first n_table[me] points of its table, by destination
      trace->cnt = cnt;
      trace->sent_ids.alloc(n_table[me], st);
      if (n_table[me]) {
        k_halo_ids<<<grid_for(n_table[me], 256), 256, 0, st>>>(reinterpret_cast<const float4*>(t.local), n_table[me],
                                                               trace->sent_ids.p);
        ++c.launches;
        PCLB_CUDA(cudaGetLastError());
      }
    }
    if (all) {
      comm_tables_publish(c, t, kU64Sum);
      gather_segments(c, segment_reads<float4>(t, cnt.data(), R, me), local.p + n_tile);
      comm_tables_release(c, t);
    }
  }

  // the local map: sorted by id, each id once, indexed
  ProfScope ps(c, stages.build);
  DevBuf<unsigned> ids, ids_sorted, ids_unique;
  DevBuf<float4> sorted, uniq;
  DevBuf<int> d_m;
  ids.alloc(n_local, st);
  ids_sorted.alloc(n_local, st);
  ids_unique.alloc(n_local, st);
  sorted.alloc(n_local, st);
  uniq.alloc(n_local, st);
  d_m.alloc(1, st);
  k_halo_ids<<<grid_for(n_local, 256), 256, 0, st>>>(local.p, n_local, ids.p);
  ++c.launches;
  const size_t n_tile = tile.n_valid;
  if (trace) {
    trace->recv_ids.alloc(n_local - n_tile, st);
    if (n_local > n_tile)
      PCLB_CUDA(cudaMemcpyAsync(trace->recv_ids.p, ids.p + n_tile, (n_local - n_tile) * sizeof(unsigned),
                                cudaMemcpyDeviceToDevice, st));
  }
  size_t tb = 0, tb2 = 0;
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, ids.p, ids_sorted.p, local.p, sorted.p, (int)n_local, 0, 31, st));
  PCLB_CUDA(cub::DeviceSelect::UniqueByKey(nullptr, tb2, ids_sorted.p, sorted.p, ids_unique.p, uniq.p, d_m.p, (int)n_local,
                                           st));
  DevBuf<unsigned char> tmp;
  tmp.alloc(std::max(tb, tb2), st);
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, ids.p, ids_sorted.p, local.p, sorted.p, (int)n_local, 0, 31, st));
  PCLB_CUDA(cub::DeviceSelect::UniqueByKey(tmp.p, tb2, ids_sorted.p, sorted.p, ids_unique.p, uniq.p, d_m.p, (int)n_local,
                                           st));
  c.launches += 6;
  int m = 0;
  PCLB_CUDA(cudaMemcpyAsync(&m, d_m.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  local.release();
  sorted.release();
  Index* built = build_index_from_device(c, uniq.p, (size_t)m, nullptr, true);
  if (trace)
    trace->local_ids = std::move(ids_unique);
  return built;
}

}  // namespace pclb200
