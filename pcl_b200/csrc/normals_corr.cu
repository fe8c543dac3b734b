// normals_corr.cu — correspondence estimation and rejection that use surface normals (SURVEY.md §8f #1/#2).
//
// Replaces CorrespondenceEstimationNormalShooting / CorrespondenceEstimationBackProjection
// (registration/include/pcl/registration/impl/correspondence_estimation_normal_shooting.hpp:66-131,
//  impl/correspondence_estimation_backprojection.hpp:66-118) and CorrespondenceRejectorSurfaceNormal
// (registration/src/correspondence_rejection_surface_normal.cpp:43-66).
// The k candidates of every source point come from the exact k-NN kernels of search.cu (one batch launch), the
// choice among them is one thread per source point over its candidate row (corr_select.cuh).
#include <cub/cub.cuh>

#include <algorithm>
#include <limits>

#include "internal.cuh"
#include "normals_corr_kernels.cuh"

namespace pclb200 {

size_t correspondences_by_normals(Ctx& c, Index& tgt, int kind, const void* src, size_t n, size_t stride,
                                  const void* src_normals, size_t stride_sn, const void* tgt_normals, size_t stride_tn,
                                  const int32_t* indices, size_t n_idx, int k, double max_dist, pclb200_corr* out)
{
  cudaStream_t st = c.stream;
  const size_t nq = indices ? n_idx : n;
  const int keff = (int)std::min<size_t>((size_t)std::max(k, 0), tgt.n_valid);  // kdtree_flann.hpp:241-242
  if (nq == 0 || keff <= 0)
    return 0;
  DevBuf<float4> dense, sn, tn;
  QueryBatch qb = load_queries(c, tgt, src, n, stride, indices, n_idx, dense);
  sn.alloc(n, st);
  load_vec3_as_float4(c, src_normals, n, stride_sn, sn.p, st);
  if (kind == PCLB200_CORR_BACK_PROJECTION) {
    tn.alloc(tgt.n_cloud, st);
    load_vec3_as_float4(c, tgt_normals, tgt.n_cloud, stride_tn, tn.p, st);
  }
  DevBuf<int32_t> staged_ind;
  const int32_t* d_ind = on_device(c, indices, n_idx, staged_ind);
  DevBuf<int32_t> nn_idx;
  DevBuf<float> nn_d2;
  nn_idx.alloc(nq * (size_t)keff, st);
  nn_d2.alloc(nq * (size_t)keff, st);
  {
    ProfScope ps(c, "knn");
    launch_knn(c, tgt, qb.q.p, nq, keff, std::numeric_limits<float>::infinity(), nn_idx.p, nn_d2.p);
  }
  ensure_pos_of_orig(c, tgt);
  DevBuf<pclb200_corr> by_slot;
  by_slot.alloc(nq, st);
  k_corr_by_normals<<<grid_for(nq, 128), 128, 0, st>>>(dense.p, nq, d_ind, sn.p, kind, keff, nn_idx.p, nn_d2.p,
                                                      tgt.pts.p, tgt.pos_of_orig.p, tn.p, max_dist, by_slot.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  const size_t m = compact_corr_to(c, by_slot.p, nq, out);
  PCLB_CUDA(cudaStreamSynchronize(st));
  return m;
}

// ---- CorrespondenceRejectorSurfaceNormal, stand-alone ---------------------------------------------------------------
size_t reject_surface_normal(Ctx& c, const pclb200_corr* in, size_t n, const void* src_normals, size_t n_src,
                             size_t stride_sn, const void* tgt_normals, size_t n_tgt, size_t stride_tn,
                             double threshold, pclb200_corr* out)
{
  cudaStream_t st = c.stream;
  if (n == 0)
    return 0;
  DevBuf<float4> sn, tn;
  sn.alloc(n_src, st);
  tn.alloc(n_tgt, st);
  load_vec3_as_float4(c, src_normals, n_src, stride_sn, sn.p, st);
  load_vec3_as_float4(c, tgt_normals, n_tgt, stride_tn, tn.p, st);
  DevBuf<pclb200_corr> staged, marked;
  const pclb200_corr* pin = on_device(c, in, n, staged);
  marked.alloc(n, st);
  k_mark_surface_normal<<<grid_for(n, 256), 256, 0, st>>>(pin, n, sn.p, n_src, tn.p, n_tgt, threshold, marked.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  const size_t m = compact_corr_to(c, marked.p, n, out);
  PCLB_CUDA(cudaStreamSynchronize(st));
  return m;
}

}  // namespace pclb200
