// cluster_kernels.cuh — the device side of cluster.cu (lock-free union-find over the "closer than the tolerance" graph), in a
// header of its own so that tests/host/consumers_host_test.cpp can compile it for the host and compare with the oracle.
#pragma once
#include "internal.cuh"
#include "traverse.cuh"
#include "union_find.cuh"

namespace pclb200 {

struct UnionVisitor {
  float qx, qy, qz, r2, r2_below;
  int self_pos;
  int* parent;
  __device__ __forceinline__ float bound() const { return r2_below; }
  __device__ __forceinline__ void prune(float) {}
  __device__ __forceinline__ void leaf(const float4* lp, int first_pos)
  {
#pragma unroll
    for (int j = 0; j < kLeafSize; ++j) {
      const float4 p = ldg4(lp + j);
      // padding slots hold +inf and never pass; every edge is handled once, from its larger end
      if (first_pos + j < self_pos && dist2_rn(qx, qy, qz, p.x, p.y, p.z) < r2)
        cc_unite(parent, self_pos, first_pos + j);
    }
  }
};

__global__ void k_cc_init(int* __restrict__ parent, int* __restrict__ min_orig, size_t n_padded)
{
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j < n_padded) {
    parent[j] = (int)j;
    min_orig[j] = kSentinelIndex;
  }
}

__global__ void __launch_bounds__(128)
k_cc_union(const BvhNode* __restrict__ nodes, const float4* __restrict__ pts, int root, size_t n_padded, float r2,
           float r2_below, int* parent, int* __restrict__ d_error)
{
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n_padded)
    return;
  const float4 q = ldg4(pts + j);
  if (__float_as_int(q.w) == kSentinelIndex)
    return;  // padding slot
  UnionVisitor v{q.x, q.y, q.z, r2, r2_below, (int)j, parent};
  if (!traverse(nodes, pts, root, q.x, q.y, q.z, v))
    atomicExch(d_error, kErrStackOverflow);
}

// smallest original index of every component, kept at the component's root
__global__ void k_cc_min_orig(const float4* __restrict__ pts, size_t n_padded, int* parent, int* __restrict__ min_orig)
{
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n_padded)
    return;
  const int oi = __float_as_int(pts[j].w);
  if (oi == kSentinelIndex)
    return;
  atomicMin(min_orig + cc_find(parent, (int)j), oi);
}

__global__ void k_cc_labels(const float4* __restrict__ pts, size_t n_padded, int* parent, const int* __restrict__ min_orig,
                            int32_t* __restrict__ labels)
{
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n_padded)
    return;
  const int oi = __float_as_int(pts[j].w);
  if (oi == kSentinelIndex)
    return;
  labels[oi] = min_orig[cc_find(parent, (int)j)];
}

}  // namespace pclb200
