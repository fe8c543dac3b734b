// grid_sum.cuh — the fixed-order grid sum of fp64 accumulators (the ICP kernels' normal equations and fitness score,
// icp_kernels.cuh; the sharded statistical outlier removal's partial sums, shard_filter_kernels.cuh): bitwise reproducible
// for a given grid.  A header of its own so that more than one translation unit can use it.
#pragma once
#include "internal.cuh"

namespace pclb200 {

// scratch of a grid sum (grid_fold): per-block partials, the ticket counter (zero between launches), the totals
struct GridSum {
  double* partials;
  unsigned* counter;
  double* accum;
};

// Where a block sits in the grid whose sum it takes part in: the launch's grid (HwGrid), or the grid of one problem of a
// batch that lies inside a larger launch (VirtualGrid, icp_kernels.cuh: BatchBlock).  The sums of a virtual grid are
// those of a launch of vgrid blocks, bit for bit.
struct HwGrid {
  __device__ __forceinline__ unsigned block() const { return blockIdx.x; }
  __device__ __forceinline__ unsigned blocks() const { return gridDim.x; }
};
struct VirtualGrid {
  unsigned vblock, vgrid;
  __device__ __forceinline__ unsigned block() const { return vblock; }
  __device__ __forceinline__ unsigned blocks() const { return vgrid; }
};

// The fixed-order grid sum of WIDTH slots.  rows[w * WIDTH + t]: the sums of slot t over the pairs of warp w of this
// block, w < nwarps, in shared memory.  Thread t < WIDTH adds them up over the warps into partials[block * STRIDE + t];
// the LAST block to take a ticket adds those up over the blocks, in block order (bitwise reproducible), into out[t] and
// returns true, and the caller's last block then publishes the totals and resets the counter.  Must be called by every
// thread of every block.  is_last: a __shared__ flag declared by the caller, so that it keeps its place in the caller's
// shared memory.  The pointers are taken by reference, so that a kernel reads them from its parameters where they are
// used.
template <int WIDTH, int STRIDE, class G = HwGrid>
__device__ __forceinline__ bool grid_fold(const double* rows, int nwarps, double* const& partials,
                                          unsigned* const& counter, bool& is_last, double* out, const G& grid = G())
{
  if (threadIdx.x < WIDTH) {
    double v = 0.0;
    for (int w = 0; w < nwarps; ++w)
      v += rows[w * WIDTH + threadIdx.x];
    partials[(size_t)grid.block() * STRIDE + threadIdx.x] = v;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned tk = atomicAdd(counter, 1u);
    is_last = (tk == grid.blocks() - 1);
  }
  __syncthreads();
  const bool last = is_last;
  if (last) {
    __threadfence();
    if (threadIdx.x < WIDTH) {
      double v = 0.0;
      for (unsigned b = 0; b < grid.blocks(); ++b)
        v += __ldcg(&partials[(size_t)b * STRIDE + threadIdx.x]);
      out[threadIdx.x] = v;
    }
  }
  return last;
}

// per-thread accumulators acc[0..NACC) -> block (fixed order) -> grid (grid_fold) -> g.accum[0..kAccum), zero beyond
// NACC.  Returns true in the last block.
template <int NACC, class G = HwGrid>
__device__ __forceinline__ bool block_reduce_and_publish(const double* acc, const GridSum& g, const G& grid = G())
{
  __shared__ double sm[8][NACC];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int t = 0; t < NACC; ++t) {
    double v = acc[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0)
      sm[warp][t] = v;
  }
  __syncthreads();
  if (!grid_fold<NACC, kAccum>(&sm[0][0], blockDim.x >> 5, g.partials, g.counter, is_last, g.accum, grid))
    return false;
  if (threadIdx.x >= NACC && threadIdx.x < kAccum)
    g.accum[threadIdx.x] = 0.0;
  if (threadIdx.x == 0)
    *g.counter = 0;
  return true;
}

}  // namespace pclb200
