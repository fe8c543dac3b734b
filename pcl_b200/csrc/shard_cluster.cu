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
// Every exchange moves a count known to every rank, so all ranks take the same branches; a table moves through
// comm_scratch_tables: peer path, each rank's table with a barrier before the reads and one after them; NCCL path, a
// zeroed table with one contributor per entry and one u64 sum all-reduce.
#include <cub/cub.cuh>

#include <algorithm>
#include <memory>
#include <vector>

#include "internal.cuh"
#include "shard_cluster_kernels.cuh"

namespace pclb200 {

bool comm_active(const Ctx& c);
bool comm_peer_fused(const Ctx& c);
int comm_nranks(const Ctx& c);
int comm_rank(const Ctx& c);

static unsigned persistent_blocks(const Ctx& c, size_t n)
{
  return (unsigned)std::max<size_t>(1, std::min<size_t>(grid_for(n, 256), (size_t)c.sm_count * 8));
}

// sorted unique copy of keys[0..n) (u32 or u64) into out; returns how many
template <typename K>
static size_t sort_unique(Ctx& c, const K* keys, size_t n, DevBuf<K>& out)
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

// n u64 words from `from` into `to` with a kernel (the write a peer may read after the next barrier)
static void copy_u64(Ctx& c, const unsigned long long* from, size_t n, unsigned long long* to)
{
  if (!n)
    return;
  ScReadSet<unsigned long long> one;
  memset(&one, 0, sizeof(one));
  one.n = 1;
  one.src[0] = from;
  one.begin[1] = n;
  k_sc_gather<<<persistent_blocks(c, n), 256, 0, c.stream>>>(one, to);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

size_t allgather_u64(Ctx& c, const unsigned long long* d_send, size_t n, DevBuf<unsigned long long>& out)
{
  cudaStream_t st = c.stream;
  const int R = comm_nranks(c), me = comm_rank(c);
  std::vector<unsigned long long> cnt(R, 0);  // every rank's count
  {
    DevBuf<unsigned long long> d_cnt;
    d_cnt.alloc(R, st);
    cnt[me] = n;
    PCLB_CUDA(cudaMemcpyAsync(d_cnt.p, cnt.data(), R * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
    comm_allreduce_u64(c, d_cnt.p, d_cnt.p, R, kU64Sum);
    PCLB_CUDA(cudaMemcpyAsync(cnt.data(), d_cnt.p, R * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    check_device_error(c);
  }
  unsigned long long total = 0, most = 0, below = 0;
  for (int s = 0; s < R; ++s) {
    if (s < me)
      below += cnt[s];
    total += cnt[s];
    most = std::max(most, cnt[s]);
  }
  out.alloc(total, st);
  if (!total)
    return 0;
  const bool peer = comm_peer_fused(c);
  const size_t words = (size_t)(peer ? most : total);
  OneToOneTables t = comm_scratch_tables(c, words);
  if (!t.peer)
    PCLB_CUDA(cudaMemsetAsync(t.local, 0, words * sizeof(unsigned long long), st));
  copy_u64(c, d_send, n, t.local + (t.peer ? 0 : below));
  ScReadSet<unsigned long long> rs;
  memset(&rs, 0, sizeof(rs));
  if (t.peer) {
    comm_barrier(c);
    for (int s = 0; s < R; ++s) {
      rs.src[s] = t.read[s];
      rs.begin[s + 1] = rs.begin[s] + cnt[s];
    }
    rs.n = R;
  }
  else {
    comm_allreduce_u64(c, t.local, const_cast<unsigned long long*>(t.read[0]), words, kU64Sum);
    rs.n = 1;
    rs.src[0] = t.read[0];
    rs.begin[1] = total;
  }
  k_sc_gather<<<persistent_blocks(c, total), 256, 0, st>>>(rs, out.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  if (t.peer)
    comm_barrier(c);
  return (size_t)total;
}

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
  auto sent = [&](int s, int r) { return s == r ? 0ull : tr.cnt[(size_t)s * R + r]; };
  unsigned long long all = 0, most_in = 0, lower = 0;
  for (int r = 0; r < R; ++r) {
    unsigned long long in = 0;
    for (int s = 0; s < R; ++s)
      in += sent(s, r);
    most_in = std::max(most_in, in);
    all += in;
  }
  for (int s = 0; s < me; ++s)
    lower += sent(s, me);
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
    // the answers: u32 per received point; peer path, in the receiver's table in the order it received them (by sender);
    // NCCL path, in one table of runs by receiver, each run by sender
    DevBuf<unsigned long long> edges;
    edges.alloc(n_sent, st);
    if (all) {
      const bool peer = comm_peer_fused(c);
      const size_t words = (size_t)((peer ? most_in : all) + 1) / 2;
      OneToOneTables t = comm_scratch_tables(c, words);
      auto run_of = [&](int r) {  // NCCL layout: the answers of the ranks below r come first
        unsigned long long off = 0;
        for (int x = 0; x < r; ++x)
          for (int s = 0; s < R; ++s)
            off += sent(s, x);
        return off;
      };
      unsigned* mine = reinterpret_cast<unsigned*>(t.local);
      if (!t.peer)
        PCLB_CUDA(cudaMemsetAsync(t.local, 0, words * sizeof(unsigned long long), st));
      if (n_recv) {
        k_sc_answer<<<persistent_blocks(c, n_recv), 256, 0, st>>>(tr.recv_ids.p, n_recv, tr.local_ids.p, m, lab_id.p,
                                                                  t.peer ? mine : mine + run_of(me));
        ++c.launches;
        PCLB_CUDA(cudaGetLastError());
      }
      if (t.peer)
        comm_barrier(c);
      else  // each u32 has one writer and is zero elsewhere: the u64 sum carries nothing between the halves
        comm_allreduce_u64(c, t.local, const_cast<unsigned long long*>(t.read[0]), words, kU64Sum);
      ScReadSet<unsigned> rs;  // the answers to this rank's segments, by destination
      memset(&rs, 0, sizeof(rs));
      for (int r = 0; r < R; ++r) {
        if (r == me)
          continue;
        unsigned long long off = t.peer ? 0 : run_of(r);
        for (int s = 0; s < me; ++s)
          off += sent(s, r);
        rs.src[rs.n] = reinterpret_cast<const unsigned*>(t.read[t.peer ? r : 0]) + off;
        rs.begin[rs.n + 1] = rs.begin[rs.n] + sent(me, r);
        ++rs.n;
      }
      if (n_sent) {
        k_sc_edges<<<persistent_blocks(c, n_sent), 256, 0, st>>>(tr.sent_ids.p, n_sent, tr.local_ids.p, m, lab_id.p, rs,
                                                                 edges.p);
        ++c.launches;
        PCLB_CUDA(cudaGetLastError());
      }
      if (t.peer)
        comm_barrier(c);
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
    OneToOneTables t = comm_scratch_tables(c, n_nodes);
    copy_u64(c, node_cnt.p, n_nodes, t.local);
    ScReadSet<unsigned long long> tables;
    memset(&tables, 0, sizeof(tables));
    if (t.peer) {
      comm_barrier(c);
      tables.n = R;
      for (int s = 0; s < R; ++s)
        tables.src[s] = t.read[s];
    }
    else {
      comm_allreduce_u64(c, t.local, const_cast<unsigned long long*>(t.read[0]), n_nodes, kU64Sum);
      tables.n = 1;
      tables.src[0] = t.read[0];
    }
    k_sc_sum<<<persistent_blocks(c, n_nodes), 256, 0, st>>>(tables, n_nodes, node_cnt.p);
    ++c.launches;
    if (t.peer)
      comm_barrier(c);
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
