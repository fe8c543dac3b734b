// cluster.cu — Euclidean clustering = connected components of the "closer than the tolerance" graph (SURVEY.md §8f #4).
//
// Replaces the breadth-first flood fill of pcl::extractEuclideanClusters
// (segmentation/include/pcl/segmentation/impl/extract_clusters.hpp:45-119, 124-223), which issues one radiusSearch per
// point from a single thread.  The squared distance is symmetric in fp32 (dist2_rn squares the same differences), so the
// sets the flood fill produces are exactly the connected components of the undirected graph with an edge wherever
// d2 < float(tolerance^2) (the strict FLANN radius test, kdtree_flann.hpp:398); they do not depend on the seed order.
// One thread per point walks the LBVH once and merges itself with every neighbour at a smaller position through a
// lock-free union-find (atomicCAS hooks the larger root under the smaller one, so parents only ever decrease and no cycle
// can form; path halving writes are benign races).  The label of a component is the smallest ORIGINAL index in it.
#include <limits>

#include "internal.cuh"
#include "cluster_kernels.cuh"

namespace pclb200 {

// labels: idx.n_cloud entries on the device; -1 for points the index does not hold (non-finite, outside the subset)
void cluster_labels(Ctx& c, const Index& idx, double tolerance, int32_t* d_labels)
{
  cudaStream_t st = c.stream;
  PCLB_CUDA(cudaMemsetAsync(d_labels, 0xff, idx.n_cloud * sizeof(int32_t), st));
  if (idx.n_valid == 0)
    return;
  // extract_clusters.hpp:246: the tolerance is narrowed to float before it reaches radiusSearch(point, double radius),
  // which squares it in double and narrows again (kdtree_flann.hpp:398)
  const double tol = (double)(float)tolerance;
  const float r2 = (float)(tol * tol);
  const float r2_below = std::nextafter(r2, -std::numeric_limits<float>::infinity());
  const size_t np = idx.pts.n;
  DevBuf<int> parent, min_orig;
  parent.alloc(np, st);
  min_orig.alloc(np, st);
  k_cc_init<<<grid_for(np, 256), 256, 0, st>>>(parent.p, min_orig.p, np);
  {
    ProfScope ps(c, "cluster_union");
    k_cc_union<<<grid_for(np, 128), 128, 0, st>>>(idx.nodes.p, idx.pts.p, idx.root, np, r2, r2_below, parent.p, c.d_error);
  }
  k_cc_min_orig<<<grid_for(np, 256), 256, 0, st>>>(idx.pts.p, np, parent.p, min_orig.p);
  k_cc_labels<<<grid_for(np, 256), 256, 0, st>>>(idx.pts.p, np, parent.p, min_orig.p, d_labels);
  c.launches += 4;
  PCLB_CUDA(cudaGetLastError());
}

}  // namespace pclb200
