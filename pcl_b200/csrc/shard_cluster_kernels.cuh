// shard_cluster_kernels.cuh — the device side of Euclidean clustering over a map sharded across ranks (driver:
// shard_cluster.cu, called by pclb200_cluster_labels_sharded).  Every rank has clustered its local map C_r (its tile plus
// the halo of shard_normals_kernels.cuh, sorted by id) with the unchanged kernels of cluster_kernels.cuh; these kernels
// stitch the local components of all ranks into the whole map's.
//   k_sc_label_ids   local label of every record of C_r as an id (the smallest id of its local component)
//   k_sc_answer      per received halo point, its local label on this rank: the answer its sender reads back
//   k_sc_mark_lower  records of C_r that a lower rank also holds in its tile (counted there, not here)
//   k_sc_edges       per point this rank sent, the edge (its label here, the label its receiver answered) as one u64
//   k_sc_split       both ends of every edge: the node list is their sorted unique set
//   k_sc_init        parent = identity over the dense node numbers
//   k_sc_unite       union-find over them (cc_unite of union_find.cuh, as cluster_kernels.cuh)
//   k_sc_roots       per node its root, whose node carries the smallest label of the stitched component
//   k_sc_count       per owned tile record, +1 to its graph node or to its local component
//   k_sc_sum         element-wise u64 sum of the tables (the node counts: every rank's, or their NCCL sum)
//   k_sc_fold        per node, its summed count added to its root
//   k_sc_output      per tile record, the final label and the whole-map size of its component
// A header of its own so that tests/host/shard_cluster_host_test.cpp can compile the kernels for the host and simulate
// several ranks.
#pragma once
#include "internal.cuh"
#include "peer_tables.cuh"
#include "union_find.cuh"

namespace pclb200 {

// position of v in the ascending array a[0..n), or -1
__device__ __forceinline__ int sc_find(const unsigned* __restrict__ a, size_t n, unsigned v)
{
  size_t lo = 0, hi = n;
  while (lo < hi) {
    const size_t mid = (lo + hi) >> 1;
    if (a[mid] < v)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo < n && a[lo] == v ? (int)lo : -1;
}

// lab_id[i] = local_ids[lab[i]]: cluster_labels labels record i of C_r with the smallest record of its component, and
// records increase with the id
__global__ void __launch_bounds__(256)
k_sc_label_ids(const int32_t* __restrict__ lab, const unsigned* __restrict__ local_ids, size_t m, unsigned* __restrict__ lab_id)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < m; i += (size_t)gridDim.x * blockDim.x)
    lab_id[i] = local_ids[lab[i]];
}

// out[i] = the local label of received point i (every received id is a record of C_r)
__global__ void __launch_bounds__(256)
k_sc_answer(const unsigned* __restrict__ recv_ids, size_t n, const unsigned* __restrict__ local_ids, size_t m,
            const unsigned* __restrict__ lab_id, unsigned* __restrict__ out)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = lab_id[sc_find(local_ids, m, recv_ids[i])];
}

// dup[record] = 1 for the first n received points (those of the ranks below this one)
__global__ void __launch_bounds__(256)
k_sc_mark_lower(const unsigned* __restrict__ recv_ids, size_t n, const unsigned* __restrict__ local_ids, size_t m,
                unsigned char* __restrict__ dup)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    dup[sc_find(local_ids, m, recv_ids[i])] = 1;
}

// edges[i] = (min << 32) | max of (the local label of sent point i here, the label its receiver answered for it); the
// answers are aligned with sent_ids (by destination, each segment in the order this rank wrote it)
__global__ void __launch_bounds__(256)
k_sc_edges(const unsigned* __restrict__ sent_ids, size_t n, const unsigned* __restrict__ local_ids, size_t m,
           const unsigned* __restrict__ lab_id, const PeerSegments<unsigned> answers, unsigned long long* __restrict__ edges)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned a = lab_id[sc_find(local_ids, m, sent_ids[i])];
    const unsigned b = peer_segment_read(answers, i);
    edges[i] = a < b ? ((unsigned long long)a << 32) | b : ((unsigned long long)b << 32) | a;
  }
}

__global__ void __launch_bounds__(256)
k_sc_split(const unsigned long long* __restrict__ edges, size_t n, unsigned* __restrict__ ends)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    ends[2 * i] = (unsigned)(edges[i] >> 32);
    ends[2 * i + 1] = (unsigned)edges[i];
  }
}

__global__ void __launch_bounds__(256)
k_sc_init(int* __restrict__ parent, size_t n)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    parent[i] = (int)i;
}

// parent[] starts as the identity (k_sc_init); cc_unite hooks the larger root under the smaller, so every root ends as
// the smallest node of its component, whatever the order of the unions
__global__ void __launch_bounds__(256)
k_sc_unite(const unsigned long long* __restrict__ edges, size_t n, const unsigned* __restrict__ nodes, size_t n_nodes,
           int* parent)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int a = sc_find(nodes, n_nodes, (unsigned)(edges[i] >> 32));
    const int b = sc_find(nodes, n_nodes, (unsigned)edges[i]);
    cc_unite(parent, a, b);
  }
}

// root[i] = the root of node i: nodes ascend, so nodes[root[i]] is the smallest label linked to nodes[i]
__global__ void __launch_bounds__(256)
k_sc_roots(size_t n_nodes, int* parent, int* __restrict__ root)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n_nodes; i += (size_t)gridDim.x * blockDim.x)
    root[i] = cc_find(parent, (int)i);
}

// Every tile record (pts: the tile index's Morton array, w = id, padding w = kSentinelIndex) that no lower rank holds
// counts once: to node_cnt of its local label when that label is a graph node, else to local_cnt at its local
// component's record (lab).
__global__ void __launch_bounds__(256)
k_sc_count(const float4* __restrict__ pts, size_t np, const unsigned* __restrict__ local_ids, size_t m,
           const int32_t* __restrict__ lab, const unsigned* __restrict__ lab_id, const unsigned char* __restrict__ dup,
           const unsigned* __restrict__ nodes, size_t n_nodes, unsigned long long* __restrict__ node_cnt,
           unsigned long long* __restrict__ local_cnt)
{
  for (size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x; j < np; j += (size_t)gridDim.x * blockDim.x) {
    const int id = __float_as_int(pts[j].w);
    if (id == kSentinelIndex)
      continue;
    const int rec = sc_find(local_ids, m, (unsigned)id);
    if (dup[rec])
      continue;
    const int node = sc_find(nodes, n_nodes, lab_id[rec]);
    if (node >= 0)
      atomicAdd(node_cnt + node, 1ull);
    else
      atomicAdd(local_cnt + lab[rec], 1ull);
  }
}

// out[i] = the sum over the tables of word i
__global__ void __launch_bounds__(256)
k_sc_sum(const __grid_constant__ PeerTableSet<unsigned long long> tables, size_t n, unsigned long long* __restrict__ out)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    unsigned long long s = 0;
    for (int t = 0; t < tables.n; ++t)
      s += __ldcv(tables.t[t] + i);
    out[i] = s;
  }
}

// comp[root[i]] += node_sum[i] (comp zeroed)
__global__ void __launch_bounds__(256)
k_sc_fold(const unsigned long long* __restrict__ node_sum, size_t n_nodes, const int* __restrict__ root,
          unsigned long long* __restrict__ comp)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n_nodes; i += (size_t)gridDim.x * blockDim.x)
    atomicAdd(comp + root[i], node_sum[i]);
}

// labels[slot] = the smallest id of the record's whole-map component and, when sizes is not null, sizes[slot] = the
// number of distinct ids in it (slot_of_pos: position in pts -> the tile's record)
__global__ void __launch_bounds__(256)
k_sc_output(const float4* __restrict__ pts, const int32_t* __restrict__ slot_of_pos, size_t np,
            const unsigned* __restrict__ local_ids, size_t m, const int32_t* __restrict__ lab,
            const unsigned* __restrict__ lab_id, const unsigned* __restrict__ nodes, size_t n_nodes,
            const int* __restrict__ root, const unsigned long long* __restrict__ comp,
            const unsigned long long* __restrict__ local_cnt, int32_t* __restrict__ labels, int64_t* __restrict__ sizes)
{
  for (size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x; j < np; j += (size_t)gridDim.x * blockDim.x) {
    const int id = __float_as_int(pts[j].w);
    if (id == kSentinelIndex)
      continue;
    const int rec = sc_find(local_ids, m, (unsigned)id);
    const unsigned l = lab_id[rec];
    const int node = sc_find(nodes, n_nodes, l);
    const int slot = slot_of_pos[j];
    labels[slot] = node >= 0 ? (int32_t)nodes[root[node]] : (int32_t)l;
    if (sizes)
      sizes[slot] = (int64_t)(node >= 0 ? comp[root[node]] : local_cnt[lab[rec]]);
  }
}

}  // namespace pclb200
