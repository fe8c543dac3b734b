// union_find.cuh — the lock-free union-find of cluster_kernels.cuh (Euclidean clustering) and shard_cluster_kernels.cuh
// (the stitching graph of a sharded map): atomicCAS hooks the larger root under the smaller, so parents only ever
// decrease, no cycle can form, and every root ends as the smallest element of its set whatever the order of the unions.
// Device functions only, so that any number of translation units may include it.
#pragma once

namespace pclb200 {

__device__ __forceinline__ int cc_find(int* parent, int x)
{
  volatile int* vp = parent;
  int cur = x;
  while (true) {
    const int p = vp[cur];
    if (p == cur)
      return cur;
    const int gp = vp[p];
    if (gp != p)
      vp[cur] = gp;  // path halving: gp was an ancestor of cur and stays one (roots never become roots again)
    cur = p;
  }
}

__device__ __forceinline__ void cc_unite(int* parent, int a, int b)
{
  while (true) {
    a = cc_find(parent, a);
    b = cc_find(parent, b);
    if (a == b)
      return;
    const int hi = a > b ? a : b, lo = a > b ? b : a;
    if (atomicCAS(parent + hi, hi, lo) == hi)
      return;
    a = hi;  // somebody hooked `hi` first: start again from the new roots
    b = lo;
  }
}

}  // namespace pclb200
