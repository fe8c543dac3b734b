// shard_cluster.cu — Euclidean clustering over a map sharded across the ranks of a communicator
// (pclb200_cluster_labels_sharded, capi.cu).  A component can cross any number of tile boundaries, so no halo alone holds
// it; each rank clusters its tile plus a halo, and one round of label exchange stitches the local components into the
// whole map's (DESIGN.md §5, "Clusters of a sharded map").
//
//   halo    C_r = this rank's tile T_r plus every point of the other tiles inside T_r's box widened by halo_reach(r2),
//           sorted by id, each id once (shard_normals.cu: sharded_local_map with the tile's points as the queries).  Every
//           edge d2 < r2 with an end in T_r lies in C_r, because halo_reach covers d2 <= r2.
//   local   the unchanged cluster_labels on the index of C_r; records increase with the id, so the smallest record of a
//           local component names its smallest id: the local label L_r(x).  Every edge of C_r is an edge of the whole map,
//           so a local component lies inside one whole-map component.
//   stitch  every receiver answers L_r(x) for every point x it received, aligned with the segment its sender wrote; the
//           sender pairs it with its own L_s(x): the edge (L_s(x), L_r(x)).  A whole-map path x_0 .. x_n is covered by
//           local components of the ranks that own the x_i (each edge lies in its owner's C), and two of them meeting at
//           x_i both hold x_i, which its owner sent to the other: they are linked by an edge.  Every rank sort-uniques its
//           edges, all of them are gathered on every rank, and one union-find over the sorted unique labels (the nodes)
//           gives, identically on every rank, the smallest label linked to each node: the smallest id of the whole-map
//           component.  A label on no edge is a component no other rank holds a point of, and stays as it is.
//   labels  each tile record's final label; its size is counted by the lowest rank that holds its id in its tile (a
//           higher rank received the id from it in the halo): local components locally, graph nodes in one dense array,
//           the same on every rank, summed over the ranks and folded onto the roots.
// Every exchange moves a count known to every rank, so all ranks take the same branches.  The answers and the edges move
// through comm_segment_tables in the layout of peer_tables.cuh, the node counts through comm_scratch_tables; each
// exchange is comm_tables_publish before the reads and comm_tables_release after them.
#include <cub/cub.cuh>

#include <algorithm>
#include <memory>
#include <vector>

#include "internal.cuh"
#include "peer_tables.cuh"
#include "shard_cluster_kernels.cuh"

namespace pclb200 {

int comm_nranks(const Ctx& c);
int comm_rank(const Ctx& c);

// sorted unique copy of keys[0..n) (u32 or u64) into out; returns how many (shard_filter.cu counts a map's ids with it)
template <typename K>
size_t sort_unique(Ctx& c, const K* keys, size_t n, DevBuf<K>& out)
{
  cudaStream_t st = c.stream;
  out.alloc(n, st);
  if (!n)
    return 0;
  DevBuf<K> sorted;
  DevBuf<int> d_m;
  sorted.alloc(n, st);
  d_m.alloc(1, st);
  size_t tb = 0, tb2 = 0;
  PCLB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, keys, sorted.p, (int)n, 0, (int)(8 * sizeof(K)), st));
  PCLB_CUDA(cub::DeviceSelect::Unique(nullptr, tb2, sorted.p, out.p, d_m.p, (int)n, st));
  DevBuf<unsigned char> tmp;
  tmp.alloc(std::max(tb, tb2), st);
  PCLB_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, tb, keys, sorted.p, (int)n, 0, (int)(8 * sizeof(K)), st));
  PCLB_CUDA(cub::DeviceSelect::Unique(tmp.p, tb2, sorted.p, out.p, d_m.p, (int)n, st));
  c.launches += 2 * sizeof(K) + 3;
  int m = 0;
  PCLB_CUDA(cudaMemcpyAsync(&m, d_m.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  return (size_t)m;
}
template size_t sort_unique<unsigned long long>(Ctx&, const unsigned long long*, size_t, DevBuf<unsigned long long>&);

void cluster_labels_sharded(Ctx& c, const Index& tile, double tolerance, int32_t* d_labels, int64_t* d_sizes)
{
  cudaStream_t st = c.stream;
  const int R = comm_nranks(c), me = comm_rank(c);
  // cluster.cu: the tolerance narrowed to float, squared in double, narrowed again
  const double tol = (double)(float)tolerance;
  const float r2 = (float)(tol * tol);
  PCLB_CUDA(cudaMemsetAsync(d_labels, 0xff, tile.n_cloud * sizeof(int32_t), st));
  if (d_sizes)
    PCLB_CUDA(cudaMemsetAsync(d_sizes, 0, tile.n_cloud * sizeof(int64_t), st));

  HaloTrace tr;
  std::unique_ptr<Index> local;
  {
    static const ShardedMapStages stages{"sharded_cluster_halo", "sharded_cluster_halo", "sharded_cluster_halo"};
    local.reset(sharded_local_map(c, tile, tile.pts.p, tile.pts.n, 0, r2, stages, &tr));
  }
  const size_t m = local->n_cloud;
  // the answers go back along the halo: rank r sends sender s one u32 per point it received from s (transposed counts)
  const std::vector<unsigned long long> ans = segment_answers(tr.cnt, R);
  const std::vector<unsigned long long> n_ans = segment_table_sizes(ans.data(), R);
  unsigned long long all = 0;
  for (int r = 0; r < R; ++r)
    all += n_ans[r];
  const unsigned long long lower = segment_start(ans.data(), R, me, me);  // received from the ranks below
  const size_t n_recv = tr.recv_ids.n, n_sent = tr.sent_ids.n;

  DevBuf<int32_t> lab;
  DevBuf<unsigned> lab_id;
  {
    ProfScope ps(c, "sharded_cluster_local");
    lab.alloc(m, st);
    lab_id.alloc(m, st);
    cluster_labels(c, *local, tolerance, lab.p);
    k_sc_label_ids<<<persistent_blocks(c, m), 256, 0, st>>>(lab.p, tr.local_ids.p, m, lab_id.p);
    ++c.launches;
    PCLB_CUDA(cudaGetLastError());
    local.reset();
  }

  DevBuf<unsigned> nodes;
  DevBuf<int> parent, root;
  size_t n_nodes = 0;
  {
    ProfScope ps(c, "sharded_cluster_stitch");
    DevBuf<unsigned long long> edges;
    edges.alloc(n_sent, st);
    if (all) {
      const PeerTables t = comm_segment_tables(c, n_ans.data(), sizeof(unsigned));
      if (n_recv) {
        k_sc_answer<<<persistent_blocks(c, n_recv), 256, 0, st>>>(tr.recv_ids.p, n_recv, tr.local_ids.p, m, lab_id.p,
                                                                  reinterpret_cast<unsigned*>(t.local));
        ++c.launches;
        PCLB_CUDA(cudaGetLastError());
      }
      comm_tables_publish(c, t, kU64Sum);  // NCCL: every word has one writer, so the u64 sum copies it
      if (n_sent) {
        k_sc_edges<<<persistent_blocks(c, n_sent), 256, 0, st>>>(tr.sent_ids.p, n_sent, tr.local_ids.p, m, lab_id.p,
                                                                 segment_reads<unsigned>(t, ans.data(), R, me), edges.p);
        ++c.launches;
        PCLB_CUDA(cudaGetLastError());
      }
      comm_tables_release(c, t);
    }
    DevBuf<unsigned long long> uniq;
    const size_t n_uniq = sort_unique(c, edges.p, n_sent, uniq);
    edges.release();

    DevBuf<unsigned long long> edges_all;
    const size_t n_edges = allgather_u64(c, uniq.p, n_uniq, edges_all);
    if (n_edges) {
      // the graph: the same edges, the same nodes and the same roots on every rank
      DevBuf<unsigned> ends;
      ends.alloc(2 * n_edges, st);
      k_sc_split<<<persistent_blocks(c, n_edges), 256, 0, st>>>(edges_all.p, n_edges, ends.p);
      ++c.launches;
      n_nodes = sort_unique(c, ends.p, 2 * n_edges, nodes);
      parent.alloc(n_nodes, st);
      root.alloc(n_nodes, st);
      k_sc_init<<<persistent_blocks(c, n_nodes), 256, 0, st>>>(parent.p, n_nodes);
      k_sc_unite<<<persistent_blocks(c, n_edges), 256, 0, st>>>(edges_all.p, n_edges, nodes.p, n_nodes, parent.p);
      k_sc_roots<<<persistent_blocks(c, n_nodes), 256, 0, st>>>(n_nodes, parent.p, root.p);
      c.launches += 3;
      PCLB_CUDA(cudaGetLastError());
    }
  }

  ProfScope ps(c, "sharded_cluster_labels");
  DevBuf<unsigned char> dup;
  DevBuf<unsigned long long> local_cnt, node_cnt, comp;
  dup.alloc(m, st);
  local_cnt.alloc(m, st);
  node_cnt.alloc(n_nodes, st);
  comp.alloc(n_nodes, st);
  PCLB_CUDA(cudaMemsetAsync(dup.p, 0, dup.bytes(), st));
  PCLB_CUDA(cudaMemsetAsync(local_cnt.p, 0, local_cnt.bytes(), st));
  if (n_nodes) {
    PCLB_CUDA(cudaMemsetAsync(node_cnt.p, 0, node_cnt.bytes(), st));
    PCLB_CUDA(cudaMemsetAsync(comp.p, 0, comp.bytes(), st));
  }
  if (lower) {
    k_sc_mark_lower<<<persistent_blocks(c, lower), 256, 0, st>>>(tr.recv_ids.p, lower, tr.local_ids.p, m, dup.p);
    ++c.launches;
  }
  const size_t np = tile.pts.n;
  k_sc_count<<<persistent_blocks(c, np), 256, 0, st>>>(tile.pts.p, np, tr.local_ids.p, m, lab.p, lab_id.p, dup.p, nodes.p,
                                                       n_nodes, node_cnt.p, local_cnt.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  if (n_nodes) {  // the node counts summed over the ranks, then folded onto the roots
    const PeerTables t = comm_scratch_tables(c, n_nodes);
    gather_segments(c, one_segment(node_cnt.p, n_nodes), t.local);  // the write a peer reads after the barrier: a kernel
    comm_tables_publish(c, t, kU64Sum);
    k_sc_sum<<<persistent_blocks(c, n_nodes), 256, 0, st>>>(peer_table_set(t), n_nodes, node_cnt.p);
    ++c.launches;
    comm_tables_release(c, t);
    k_sc_fold<<<persistent_blocks(c, n_nodes), 256, 0, st>>>(node_cnt.p, n_nodes, root.p, comp.p);
    ++c.launches;
    PCLB_CUDA(cudaGetLastError());
  }
  k_sc_output<<<persistent_blocks(c, np), 256, 0, st>>>(tile.pts.p, tile.slot_of_pos.p, np, tr.local_ids.p, m, lab.p,
                                                        lab_id.p, nodes.p, n_nodes, root.p, comp.p, local_cnt.p, d_labels,
                                                        d_sizes);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

}  // namespace pclb200
