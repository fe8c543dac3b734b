// capi.cu — the C boundary of libpclb200.so (include/pclb200.h).  No exception crosses it; there is no CPU
// fallback: every entry point either runs the CUDA path or returns an error status.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <limits>
#include <memory>

#include "internal.cuh"
#include "../../include/pclb200_batch.h"

namespace pclb200 {
// icp.cu
struct Icp;
Icp* icp_create(Ctx& c, const pclb200_icp_params& P);
void icp_destroy(Icp* s);
void icp_set_params(Icp& s, const pclb200_icp_params& P);
void icp_set_rejectors(Icp& s, const pclb200_rejector* list, int n);
size_t reject_standalone(Ctx& c, const pclb200_rejector& r, const pclb200_corr* in, size_t n, pclb200_corr* out,
                         double* median_out);
void icp_set_target(Icp& s, const Index* idx, const void* tgt_normals, size_t stride_n);
void icp_set_target_sharded(Icp& s, const Index* tile, const void* tgt_normals, size_t stride_n);
void icp_set_source(Icp& s, const void* src, size_t n, size_t stride, const void* src_normals, size_t stride_n,
                    const int32_t* indices, size_t n_idx, const double* guess);
void icp_iterate(Icp& s, int max_steps, pclb200_icp_stats* stats);
void icp_set_source_batch(Icp& s, const void* src, size_t n, size_t stride, const void* src_normals, size_t stride_n,
                          const int64_t* offsets, int n_problems, const double* guesses);
void icp_iterate_batch(Icp& s, int max_steps, pclb200_icp_stats* stats);
void icp_set_target_batch(Icp& s, const Index* const* targets, const void* const* tgt_normals, size_t stride_n,
                          int n_targets);
void icp_get_correspondences_batch(Icp& s, pclb200_corr* out, int64_t* counts);
void icp_get_cloud(Icp& s, void* out_pts, size_t stride_out, void* out_normals, size_t stride_n);
size_t icp_get_correspondences(Icp& s, pclb200_corr* out);
void estimate_pairs(Ctx& c, int est, const void* src, size_t stride_s, const void* tgt, const void* tgt_normals,
                    size_t stride_t, const pclb200_corr* corr, size_t n, int scalar_is_double, double* T_out,
                    const void* src_normals = nullptr, int enforce_same_dir = 1, int svd_correlation = 0);
size_t correspondences(Ctx& c, const Index& tgt, const Index* src_index, const void* src, size_t n, size_t stride,
                       const int32_t* indices, size_t n_idx, int is_dense, double max_dist, pclb200_corr* out,
                       const double* pre_T = nullptr, int pre_mode = kApplyIcp, const float* gate_override = nullptr);
double fitness_score(Ctx& c, const Index& tgt, const void* src, size_t n, size_t stride, const int32_t* indices,
                     size_t n_idx, const double* T, int scalar_is_double, double max_range, int mode_override = -1);
void fitness_score_batch(Ctx& c, const Index* const* tgt, int B, const void* src, size_t n, size_t stride,
                         const int64_t* offsets, const double* transforms, int mode, double max_range, double* scores);
void icp_fitness_score_batch(Icp& s, double max_range, double* scores);
double fitness_score_sharded(Ctx& c, const Index* tile, const void* src, size_t n, size_t stride, const int32_t* indices,
                             size_t n_idx, const double* T, int scalar_is_double, double max_range, int mode_override = -1,
                             const char* fault = nullptr);
size_t correspondences_normals_sharded(Ctx& c, const Index* tile, int kind, const void* src, size_t n, size_t stride,
                                       const void* src_normals, size_t stride_sn, const void* tgt_normals,
                                       size_t stride_tn, const int32_t* indices, size_t n_idx, int k, double max_dist,
                                       pclb200_corr* out, float* out_xyz1, float* out_normals, const char* fault);
size_t correspondences_sharded(Ctx& c, const Index* tile, const Index* src_index, const void* src, size_t n, size_t stride,
                               const int32_t* indices, size_t n_idx, double max_dist, const void* tgt_normals,
                               size_t stride_tn, pclb200_corr* out, float* out_xyz1, float* out_normals, const char* fault,
                               const double* pre_T = nullptr, int pre_mode = kApplyIcp,
                               const float* gate_override = nullptr);
void gicp_covariances(Ctx& c, Index& idx, const void* pts, size_t n, size_t stride, int k, double gicp_epsilon,
                      double* out);
// shard_filter.cu
int knn_sharded(Ctx& c, const Index& tile, const void* queries, size_t nq, size_t stride, int k, int32_t* d_idx,
                float* d_d2);
void knn_stats_sharded(Ctx& c, const Index& tile, const void* pts, size_t n, size_t stride, const int32_t* indices,
                       size_t n_idx, int k, float* d_mean, float* d_kth);
void statistical_outlier_sharded(Ctx& c, const Index& tile, const void* pts, size_t n, size_t stride,
                                 const int32_t* indices, size_t n_idx, int mean_k, double std_mul, int negative,
                                 unsigned char* d_keep, double* d_stats);
void radius_outlier_sharded(Ctx& c, const Index& tile, const void* pts, size_t n, size_t stride, const int32_t* indices,
                            size_t n_idx, int is_dense, double radius, int min_pts, int negative, unsigned char* d_keep);
unsigned long long radius_sharded(Ctx& c, const Index* tile, const void* queries, size_t nq, size_t stride, double radius,
                                  unsigned max_nn, int64_t* out_offsets,
                                  const std::function<RadiusSinkBuffers(unsigned long long)>& sink, const char* fault);
void gicp_covariances_sharded(Ctx& c, const Index* tile, const void* pts, size_t n, size_t stride, int k,
                              double gicp_epsilon, double* out, const char* fault);
unsigned long long ranks_min(Ctx& c, unsigned long long word);
// voxel.cu
size_t voxelgrid(Ctx& c, const void* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int is_dense,
                 const float leaf[3], unsigned min_pts, float* out_xyz1, const void* normals, size_t stride_n,
                 float* out_normal_curv, const float* grid_bounds = nullptr);
size_t voxelgrid_batch(Ctx& c, const void* pts, size_t n, size_t stride, const int64_t* offsets, int n_clouds,
                       const float leaf[3], unsigned min_pts, const void* normals, size_t stride_n, float* out_xyz1,
                       float* out_normal_curv, int64_t* out_offsets);
// shard_voxel.cu
size_t voxelgrid_sharded(Ctx& c, const void* pts, size_t n, size_t stride, const int32_t* ids, const void* normals,
                         size_t stride_n, const float leaf[3], unsigned min_pts, float* out_xyz1, float* out_normal_curv,
                         uint32_t* out_voxel, size_t* n_out);
// comm.cu
void comm_unique_id(void* out128);
void comm_export(Ctx& c, void* out64);
void comm_import(Ctx& c, int rank, int nranks, const void* handles);
void comm_set_mode(Ctx& c, int mode);
void comm_init(Ctx& c, int rank, int nranks, const void* unique_id);
void comm_destroy(Ctx& c);
bool comm_active(const Ctx& c);

static thread_local std::string g_last_error;

template <typename F>
static int guarded(F&& f)
{
  try {
    f();
    return PCLB200_OK;
  }
  catch (const Error& e) {
    g_last_error = e.what();
    return e.code;
  }
  catch (const std::bad_alloc&) {
    g_last_error = "host allocation failed";
    return PCLB200_ERR_INTERNAL;
  }
  catch (const std::exception& e) {
    g_last_error = e.what();
    return PCLB200_ERR_INTERNAL;
  }
}

void raise_device_error(Ctx& c, int code)
{
  PCLB_CUDA(cudaMemsetAsync(c.d_error, 0, sizeof(int), c.stream));
  if (code == kErrPeerTimeout)
    throw Error(PCLB200_ERR_NCCL, "fused cross-GPU reduce timed out waiting for a peer rank");
  throw Error(PCLB200_ERR_INTERNAL, "LBVH traversal stack overflow (tree deeper than the per-query stack)");
}

void check_device_error(Ctx& c)
{
  int h = 0;
  PCLB_CUDA(cudaMemcpyAsync(&h, c.d_error, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
  PCLB_CUDA(cudaStreamSynchronize(c.stream));
  if (h)
    raise_device_error(c, h);
}

}  // namespace pclb200

using namespace pclb200;

struct pclb200_ctx {
  Ctx c;
};
struct pclb200_index {
  Index* idx;
};
struct pclb200_icp {
  Icp* s;
  pclb200_ctx* ctx;
  int device;
};

// Binds an entry point to its context: errors become a status (guarded), calls on one context serialise on Ctx::mu, and
// the work runs on the context's device.  `body` checks its other arguments.
template <typename F>
static int on_ctx(pclb200_ctx* ctx, F&& body, const char* if_null = "NULL argument")
{
  return guarded([&] {
    PCLB_REQUIRE(ctx, PCLB200_ERR_INVALID, if_null);
    Ctx& c = ctx->c;
    std::lock_guard<std::recursive_mutex> lk(c.mu);
    PCLB_CUDA(cudaSetDevice(c.device));
    body(c);
  });
}

// the same for a session, through the context it was created on
template <typename F>
static int on_ctx(pclb200_icp* icp, F&& body)
{
  return on_ctx(icp ? icp->ctx : nullptr, [&](Ctx&) { body(*icp->s); });
}

// Shared body of pclb200_normals_knn / pclb200_normals_radius: `launch(d_q, nq, d_out, d_not_dense)` runs the estimator
// over the query batch.
template <typename Launch>
static void normals(Ctx& c, const Index& idx, const void* pts, size_t n, size_t stride, const int32_t* indices,
                    size_t n_idx, float* out, int* is_dense_out, Launch&& launch)
{
  cudaStream_t st = c.stream;
  const size_t nq = indices ? n_idx : n;
  if (is_dense_out)
    *is_dense_out = 1;
  if (!nq)
    return;
  DevBuf<float4> dense;
  QueryBatch qb = load_queries(c, idx, pts, n, stride, indices, n_idx, dense);
  DevBuf<float4> tmp;
  DevBuf<int> d_flag;
  d_flag.alloc(1, st);
  PCLB_CUDA(cudaMemsetAsync(d_flag.p, 0, sizeof(int), st));
  float4* const caller_out = reinterpret_cast<float4*>(out);
  {
    ProfScope ps(c, "normals");
    launch(qb.q.p, nq, out_on_device(c, caller_out, nq, tmp), d_flag.p);
  }
  int flag = 0;
  PCLB_CUDA(cudaMemcpyAsync(&flag, d_flag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  copy_out(c, caller_out, tmp, nq);
  check_device_error(c);
  if (is_dense_out)
    *is_dense_out = flag ? 0 : 1;
}

// Shared body of pclb200_normals_knn_sharded / _radius_sharded (collective): the caller's queries staged once, the local
// map of this rank (shard_normals.cu: its tile plus the halo its queries need), then the single-GPU normals on that map.
template <typename Launch>
static void normals_sharded(Ctx& c, const Index& tile, const void* pts, size_t n, size_t stride, const int32_t* indices,
                            size_t n_idx, int k, float r2, float* out, int* is_dense_out, Launch&& launch)
{
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID,
               "sharded normals need an active communicator (pclb200_comm_init or pclb200_comm_export / _import)");
  PCLB_REQUIRE(tile.labelled, PCLB200_ERR_INVALID,
               "sharded normals: every rank's tile must be built with pclb200_index_build_ids");
  const size_t nq = indices ? n_idx : n;
  DevBuf<float4> dense;
  dense.alloc(nq, c.stream);
  load_xyz_as_float4(c, pts, n, stride, indices, n_idx, dense.p, c.stream);
  static const ShardedMapStages stages{"sharded_normals_bound", "sharded_normals_halo", "sharded_normals_build"};
  std::unique_ptr<Index> local(sharded_local_map(c, tile, dense.p, nq, k, r2, stages));
  normals(c, *local, dense.p, nq, sizeof(float4), nullptr, 0, out, is_dense_out,
          [&](const float4* d_q, size_t m, float4* d_out, int* d_flag) { launch(*local, d_q, m, d_out, d_flag); });
}

extern "C" {

int pclb200_version(void) { return PCLB200_VERSION; }
const char* pclb200_last_error(void) { return g_last_error.c_str(); }

int pclb200_create(int device, pclb200_ctx** out)
{
  return guarded([&] {
    PCLB_REQUIRE(out != nullptr, PCLB200_ERR_INVALID, "out == NULL");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
      cudaGetLastError();
      throw Error(PCLB200_ERR_CUDA, "no CUDA device available: libpclb200 has no CPU fallback");
    }
    PCLB_REQUIRE(device >= 0 && device < ndev, PCLB200_ERR_INVALID, "bad device ordinal");
    PCLB_CUDA(cudaSetDevice(device));
    std::unique_ptr<pclb200_ctx> h(new pclb200_ctx());
    Ctx& c = h->c;
    c.device = device;
    cudaDeviceProp prop;
    PCLB_CUDA(cudaGetDeviceProperties(&prop, device));
    c.sm_count = prop.multiProcessorCount;
    PCLB_CUDA(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
    c.pinned_bytes = 4096;
    PCLB_CUDA(cudaMallocHost(&c.pinned, c.pinned_bytes));
    PCLB_CUDA(cudaMalloc(reinterpret_cast<void**>(&c.d_error), sizeof(int)));
    PCLB_CUDA(cudaMemsetAsync(c.d_error, 0, sizeof(int), c.stream));
    PCLB_CUDA(cudaStreamSynchronize(c.stream));
    *out = h.release();
  });
}

int pclb200_destroy(pclb200_ctx* ctx)
{
  return guarded([&] {
    if (!ctx)
      return;
    Ctx& c = ctx->c;
    cudaSetDevice(c.device);
    comm_destroy(c);
    if (c.stream)
      cudaStreamSynchronize(c.stream);
    for (auto& e : c.prof) {
      cudaEventDestroy(e.a);
      cudaEventDestroy(e.b);
    }
    if (c.pinned)
      cudaFreeHost(c.pinned);
    if (c.d_error)
      cudaFree(c.d_error);
    if (c.stream) {
      cached_release_all(c.stream);  // every DevBuf of this ctx is gone or orphaned by now
      cudaStreamDestroy(c.stream);
    }
    delete ctx;
  });
}

int pclb200_synchronize(pclb200_ctx* ctx)
{
  return on_ctx(ctx, [&](Ctx& c) { PCLB_CUDA(cudaStreamSynchronize(c.stream)); }, "ctx == NULL");
}

int pclb200_launch_count(pclb200_ctx* ctx, uint64_t* out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(out, PCLB200_ERR_INVALID, "NULL argument");
    *out = c.launches;
  });
}

int pclb200_stream(pclb200_ctx* ctx, void** out_stream)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(out_stream, PCLB200_ERR_INVALID, "NULL argument");
    *out_stream = (void*)c.stream;
  });
}

void pclb200_free(void* p) { free(p); }

int pclb200_host_register(pclb200_ctx* ctx, void* host_ptr, size_t bytes)
{
  return on_ctx(ctx, [&](Ctx&) {
    PCLB_REQUIRE(host_ptr && bytes, PCLB200_ERR_INVALID, "NULL argument or empty buffer");
    PCLB_REQUIRE(!is_device_ptr(host_ptr), PCLB200_ERR_INVALID, "pclb200_host_register: not a host pointer");
    const cudaError_t e = cudaHostRegister(host_ptr, bytes, cudaHostRegisterPortable);
    if (e == cudaErrorHostMemoryAlreadyRegistered) {
      cudaGetLastError();
      throw Error(PCLB200_ERR_INVALID, "pclb200_host_register: the buffer (or a part of it) is already registered");
    }
    PCLB_CUDA(e);
  }, "NULL argument or empty buffer");
}

int pclb200_host_unregister(pclb200_ctx* ctx, void* host_ptr)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(host_ptr, PCLB200_ERR_INVALID, "NULL argument");
    // nothing may still be copying out of it: wait for this context's stream
    PCLB_CUDA(cudaStreamSynchronize(c.stream));
    const cudaError_t e = cudaHostUnregister(host_ptr);
    if (e == cudaErrorHostMemoryNotRegistered) {
      cudaGetLastError();
      throw Error(PCLB200_ERR_INVALID, "pclb200_host_unregister: the buffer is not registered");
    }
    PCLB_CUDA(e);
  });
}

int pclb200_profile_enable(pclb200_ctx* ctx, int enable)
{
  return on_ctx(ctx, [&](Ctx& c) { c.profiling = enable != 0; }, "ctx == NULL");
}

int pclb200_profile_reset(pclb200_ctx* ctx)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_CUDA(cudaStreamSynchronize(c.stream));
    for (auto& e : c.prof) {
      cudaEventDestroy(e.a);
      cudaEventDestroy(e.b);
    }
    c.prof.clear();
  }, "ctx == NULL");
}

int pclb200_profile_get(pclb200_ctx* ctx, const char* name, double* total_ms, uint64_t* count)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(name && total_ms && count, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_CUDA(cudaStreamSynchronize(c.stream));
    double t = 0.0;
    uint64_t n = 0;
    for (auto& e : c.prof)
      if (strcmp(e.name, name) == 0) {
        float ms = 0.f;
        PCLB_CUDA(cudaEventElapsedTime(&ms, e.a, e.b));
        t += ms;
        ++n;
      }
    *total_ms = t;
    *count = n;
  });
}

// ---- index -----------------------------------------------------------------------------------------------------
int pclb200_index_build(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const int32_t* subset,
                        size_t n_subset, pclb200_index** out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(out, PCLB200_ERR_INVALID, "NULL argument");
    Index* idx = nullptr;
    {
      ProfScope ps(c, "index_build");
      idx = build_index(c, pts, n, stride, subset, n_subset);
    }
    *out = new pclb200_index{idx};
  });
}

int pclb200_index_build_ids(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const int32_t* ids,
                            pclb200_index** out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(out, PCLB200_ERR_INVALID, "NULL argument");
    Index* idx = nullptr;
    {
      ProfScope ps(c, "index_build");
      idx = build_index_ids(c, pts, n, stride, ids);
    }
    *out = new pclb200_index{idx};
  });
}

int pclb200_index_build_batch(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const int64_t* offsets,
                              int32_t n_clouds, pclb200_index** out)
{
  if (out && n_clouds > 0 && n_clouds <= 65536)
    std::fill(out, out + n_clouds, nullptr);
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(out, PCLB200_ERR_INVALID, "NULL argument");
    std::vector<std::unique_ptr<Index>> idx;
    {
      ProfScope ps(c, "index_build_batch");
      idx = build_index_batch(c, pts, n, stride, offsets, n_clouds);
    }
    std::vector<std::unique_ptr<pclb200_index>> h(n_clouds);
    for (int k = 0; k < n_clouds; ++k)
      h[k].reset(new pclb200_index{nullptr});
    for (int k = 0; k < n_clouds; ++k) {
      h[k]->idx = idx[k].release();
      out[k] = h[k].release();
    }
  });
}

int pclb200_index_destroy(pclb200_index* h)
{
  return guarded([&] {
    if (!h)
      return;
    if (h->idx) {
      cudaSetDevice(h->idx->device);
      delete h->idx;
    }
    delete h;
  });
}

int pclb200_index_size(const pclb200_index* h, size_t* n_valid)
{
  return guarded([&] {
    PCLB_REQUIRE(h && h->idx && n_valid, PCLB200_ERR_INVALID, "NULL argument");
    *n_valid = h->idx->n_valid;
  });
}

int pclb200_index_stats(const pclb200_index* h, uint64_t out[4])
{
  return guarded([&] {
    PCLB_REQUIRE(h && h->idx && out, PCLB200_ERR_INVALID, "NULL argument");
    out[0] = (uint64_t)h->idx->n_leaves;
    out[1] = (uint64_t)(h->idx->n_leaves > 0 ? h->idx->n_leaves - 1 : 0);
    out[2] = (uint64_t)h->idx->bytes();
    out[3] = (uint64_t)kLeafSize;
  });
}

// ---- k-NN ---------------------------------------------------------------------------------------------------------
int pclb200_knn(pclb200_ctx* ctx, const pclb200_index* h, const void* queries, size_t nq, size_t stride, int k,
                int32_t* out_idx, float* out_d2, int* k_eff)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(h && h->idx, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(k >= 0, PCLB200_ERR_INVALID, "k < 0");
    const Index& idx = *h->idx;
    const int keff = (int)std::min<size_t>((size_t)k, idx.n_valid);  // kdtree_flann.hpp:241-242
    if (k_eff)
      *k_eff = keff;
    if (k == 0 || nq == 0)
      return;
    PCLB_REQUIRE(queries && out_idx && out_d2, PCLB200_ERR_INVALID, "NULL argument");
    DevBuf<float4> dense;
    QueryBatch qb = load_queries(c, idx, queries, nq, stride, nullptr, 0, dense);
    DevBuf<int32_t> ti;
    DevBuf<float> td;
    const size_t n_out = nq * (size_t)k;
    {
      ProfScope ps(c, "knn");
      launch_knn(c, idx, qb.q.p, nq, k, std::numeric_limits<float>::infinity(), out_on_device(c, out_idx, n_out, ti),
                 out_on_device(c, out_d2, n_out, td));
    }
    copy_out(c, out_idx, ti, n_out);
    copy_out(c, out_d2, td, n_out);
    check_device_error(c);
  });
}

int pclb200_knn_stats(pclb200_ctx* ctx, const pclb200_index* h, const void* pts, size_t n, size_t stride,
                      const int32_t* indices, size_t n_idx, int k, float* out_mean, float* out_kth)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(h && h->idx && (out_mean || out_kth), PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(k > 0, PCLB200_ERR_INVALID, "k must be positive");
    const size_t nq = indices ? n_idx : n;
    if (!nq)
      return;
    DevBuf<float4> dense;
    QueryBatch qb = load_queries(c, *h->idx, pts, n, stride, indices, n_idx, dense);
    DevBuf<float> tm, tk;
    {
      ProfScope ps(c, "knn_stats");
      launch_knn_stats(c, *h->idx, qb.q.p, nq, k, out_on_device(c, out_mean, nq, tm), out_on_device(c, out_kth, nq, tk));
    }
    copy_out(c, out_mean, tm, nq);
    copy_out(c, out_kth, tk, nq);
    check_device_error(c);
  });
}

// ---- radius -------------------------------------------------------------------------------------------------------
int pclb200_radius(pclb200_ctx* ctx, const pclb200_index* h, const void* queries, size_t nq, size_t stride,
                   double radius, unsigned max_nn, int sorted, int64_t* out_offsets, int32_t** out_idx, float** out_d2)
{
  (void)sorted;
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(h && h->idx && out_offsets && out_idx && out_d2, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(!is_device_ptr(out_offsets), PCLB200_ERR_INVALID, "pclb200_radius returns host arrays: out_offsets must be host memory");
    *out_idx = nullptr;
    *out_d2 = nullptr;
    out_offsets[0] = 0;
    if (nq == 0)
      return;
    radius_search(c, *h->idx, queries, nq, stride, radius, max_nn, out_offsets, [&](unsigned long long total) {
      int32_t* hi = static_cast<int32_t*>(malloc(std::max<size_t>(total, 1) * sizeof(int32_t)));
      float* hd = static_cast<float*>(malloc(std::max<size_t>(total, 1) * sizeof(float)));
      *out_idx = hi;  // owned by the caller from here on (pclb200_free), also on the error paths
      *out_d2 = hd;
      PCLB_REQUIRE(hi && hd, PCLB200_ERR_INTERNAL, "host allocation failed");
      return RadiusSinkBuffers{hi, hd};
    });
  });
}

int pclb200_radius_into(pclb200_ctx* ctx, const pclb200_index* h, const void* queries, size_t nq, size_t stride,
                        double radius, unsigned max_nn, int64_t* out_offsets, int32_t* out_idx, float* out_d2,
                        size_t capacity, size_t* total)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(h && h->idx && out_offsets && total, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(capacity == 0 || (out_idx && out_d2), PCLB200_ERR_INVALID, "NULL output buffers with a non-zero capacity");
    *total = 0;
    if (nq == 0) {
      const int64_t zero = 0;
      PCLB_CUDA(cudaMemcpy(out_offsets, &zero, sizeof(zero), cudaMemcpyDefault));
      return;
    }
    radius_search(c, *h->idx, queries, nq, stride, radius, max_nn, out_offsets, [&](unsigned long long n) {
      *total = (size_t)n;
      if ((size_t)n > capacity)
        return RadiusSinkBuffers{nullptr, nullptr};  // offsets and *total are valid; call again with larger buffers
      return RadiusSinkBuffers{out_idx, out_d2};
    });
  });
}

// ---- correspondences -------------------------------------------------------------------------------------------------
int pclb200_correspondences(pclb200_ctx* ctx, const pclb200_index* idx_tgt, const pclb200_index* idx_src,
                            const void* src, size_t n, size_t stride, const int32_t* src_indices, size_t n_idx,
                            int is_dense, double max_dist, pclb200_corr* out, size_t* n_out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(idx_tgt && idx_tgt->idx && n_out, PCLB200_ERR_INVALID, "NULL argument");
    *n_out = correspondences(c, *idx_tgt->idx, idx_src ? idx_src->idx : nullptr, src, n, stride, src_indices, n_idx,
                             is_dense, max_dist, out);
  });
}

int pclb200_correspondences_normals(pclb200_ctx* ctx, const pclb200_index* idx_tgt, int kind, const void* src, size_t n,
                                    size_t stride, const void* src_normals, size_t stride_sn, const void* tgt_normals,
                                    size_t stride_tn, const int32_t* src_indices, size_t n_idx, int k, double max_dist,
                                    pclb200_corr* out, size_t* n_out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(idx_tgt && idx_tgt->idx && n_out, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(kind == PCLB200_CORR_NORMAL_SHOOTING || kind == PCLB200_CORR_BACK_PROJECTION, PCLB200_ERR_INVALID,
                 "kind must be PCLB200_CORR_NORMAL_SHOOTING or PCLB200_CORR_BACK_PROJECTION");
    PCLB_REQUIRE(k >= 0, PCLB200_ERR_INVALID, "k < 0");
    *n_out = 0;
    const size_t nq = src_indices ? n_idx : n;
    if (nq == 0 || k == 0)
      return;
    PCLB_REQUIRE(src && out, PCLB200_ERR_INVALID, "NULL argument");
    // correspondence_estimation_normal_shooting.hpp:51-57 / backprojection.hpp:51-57: normals are mandatory
    PCLB_REQUIRE(src_normals, PCLB200_ERR_INVALID, "source normals are required");
    PCLB_REQUIRE(kind != PCLB200_CORR_BACK_PROJECTION || tgt_normals, PCLB200_ERR_INVALID,
                 "back projection needs target normals");
    *n_out = correspondences_by_normals(c, *idx_tgt->idx, kind, src, n, stride, src_normals, stride_sn, tgt_normals,
                                        stride_tn, src_indices, n_idx, k, max_dist, out);
    check_device_error(c);
  });
}

int pclb200_reject_surface_normal(pclb200_ctx* ctx, const pclb200_corr* in, size_t n, const void* src_normals, size_t n_src,
                                  size_t stride_sn, const void* tgt_normals, size_t n_tgt, size_t stride_tn,
                                  double threshold, pclb200_corr* out, size_t* n_out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(n_out, PCLB200_ERR_INVALID, "NULL argument");
    *n_out = 0;
    if (n == 0)
      return;
    PCLB_REQUIRE(in && out && src_normals && tgt_normals && n_src && n_tgt, PCLB200_ERR_INVALID,
                 "NULL argument (correspondence_rejection_surface_normal.cpp:49-54: the normals must be set)");
    *n_out = reject_surface_normal(c, in, n, src_normals, n_src, stride_sn, tgt_normals, n_tgt, stride_tn, threshold, out);
  });
}

// ---- estimators ---------------------------------------------------------------------------------------------------------
int pclb200_estimate_svd(pclb200_ctx* ctx, const void* src, size_t stride_s, const void* tgt, size_t stride_t,
                         const pclb200_corr* corr, size_t n, int scalar_is_double, double T_out[16])
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(T_out, PCLB200_ERR_INVALID, "NULL argument");
    estimate_pairs(c, PCLB200_EST_SVD, src, stride_s, tgt, nullptr, stride_t, corr, n, scalar_is_double, T_out);
  });
}

int pclb200_estimate_svd_correlation(pclb200_ctx* ctx, const void* src, size_t stride_s, const void* tgt, size_t stride_t,
                                     const pclb200_corr* corr, size_t n, int scalar_is_double, double T_out[16])
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(T_out, PCLB200_ERR_INVALID, "NULL argument");
    estimate_pairs(c, PCLB200_EST_SVD, src, stride_s, tgt, nullptr, stride_t, corr, n, scalar_is_double, T_out, nullptr, 1,
                   1);
  });
}

int pclb200_estimate_point_to_plane_lls(pclb200_ctx* ctx, const void* src, size_t stride_s, const void* tgt,
                                        const void* tgt_normals, size_t stride_t, const pclb200_corr* corr, size_t n,
                                        int scalar_is_double, double T_out[16])
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(T_out, PCLB200_ERR_INVALID, "NULL argument");
    estimate_pairs(c, PCLB200_EST_POINT_TO_PLANE_LLS, src, stride_s, tgt, tgt_normals, stride_t, corr, n,
                   scalar_is_double, T_out);
  });
}

int pclb200_estimate_symmetric_point_to_plane_lls(pclb200_ctx* ctx, const void* src, const void* src_normals,
                                                  size_t stride_s, const void* tgt, const void* tgt_normals,
                                                  size_t stride_t, const pclb200_corr* corr, size_t n,
                                                  int enforce_same_direction_normals, int scalar_is_double,
                                                  double T_out[16])
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(T_out, PCLB200_ERR_INVALID, "NULL argument");
    estimate_pairs(c, PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS, src, stride_s, tgt, tgt_normals, stride_t, corr, n,
                   scalar_is_double, T_out, src_normals, enforce_same_direction_normals);
  });
}

// ---- ICP ------------------------------------------------------------------------------------------------------------------
void pclb200_icp_default_params(pclb200_icp_params* p)
{
  if (!p)
    return;
  memset(p, 0, sizeof(*p));
  p->max_iterations = 10;
  p->estimator = PCLB200_EST_SVD;
  p->is_dense = 1;
  p->enforce_same_direction_normals = 1;
  p->correspondence_kind = PCLB200_CORR_NEAREST;
  p->correspondence_k = 10;  // k_{10}: correspondence_estimation_normal_shooting.h:251, ..._backprojection.h:251
  p->max_correspondence_distance = std::sqrt(std::numeric_limits<double>::max());
  p->transformation_epsilon = 0.0;
  p->transformation_rotation_epsilon = 0.0;
  p->euclidean_fitness_epsilon = -std::numeric_limits<double>::max();
  p->mse_threshold_absolute = 1e-12;
}

int pclb200_icp_create(pclb200_ctx* ctx, const pclb200_icp_params* params, pclb200_icp** out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(out, PCLB200_ERR_INVALID, "NULL argument");
    pclb200_icp_params P;
    if (params)
      P = *params;
    else
      pclb200_icp_default_params(&P);
    *out = new pclb200_icp{icp_create(c, P), ctx, c.device};
  });
}

int pclb200_icp_destroy(pclb200_icp* icp)
{
  return guarded([&] {
    if (!icp)
      return;
    cudaSetDevice(icp->device);
    icp_destroy(icp->s);
    delete icp;
  });
}

int pclb200_icp_set_params(pclb200_icp* icp, const pclb200_icp_params* params)
{
  return on_ctx(icp, [&](Icp& s) {
    PCLB_REQUIRE(params, PCLB200_ERR_INVALID, "NULL argument");
    icp_set_params(s, *params);
  });
}

int pclb200_icp_set_rejectors(pclb200_icp* icp, const pclb200_rejector* list, int n)
{
  return on_ctx(icp, [&](Icp& s) {
    PCLB_REQUIRE(n <= 0 || list, PCLB200_ERR_INVALID, "NULL argument");
    icp_set_rejectors(s, list, n);
  });
}

int pclb200_reject(pclb200_ctx* ctx, const pclb200_rejector* rejector, const pclb200_corr* in, size_t n,
                   pclb200_corr* out, size_t* n_out, double* median_out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(rejector && n_out && (n == 0 || (in && out)), PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(rejector->kind >= PCLB200_REJ_DISTANCE && rejector->kind <= PCLB200_REJ_TRIMMED, PCLB200_ERR_INVALID,
                 "unknown rejector kind");
    *n_out = reject_standalone(c, *rejector, in, n, out, median_out);
  });
}

int pclb200_icp_set_target(pclb200_icp* icp, const pclb200_index* idx_tgt, const void* tgt_normals, size_t stride_n)
{
  return on_ctx(icp, [&](Icp& s) {
    PCLB_REQUIRE(idx_tgt && idx_tgt->idx, PCLB200_ERR_INVALID, "NULL argument");
    icp_set_target(s, idx_tgt->idx, tgt_normals, stride_n);
  });
}

int pclb200_icp_set_target_sharded(pclb200_icp* icp, const pclb200_index* idx_tile, const void* tgt_normals,
                                   size_t stride_n)
{
  return on_ctx(icp, [&](Icp& s) {
    PCLB_REQUIRE(idx_tile && idx_tile->idx, PCLB200_ERR_INVALID, "NULL argument");
    icp_set_target_sharded(s, idx_tile->idx, tgt_normals, stride_n);
  });
}

int pclb200_icp_set_source(pclb200_icp* icp, const void* src, size_t n, size_t stride, const void* src_normals,
                           size_t stride_n, const int32_t* src_indices, size_t n_idx, const double guess[16])
{
  return on_ctx(icp, [&](Icp& s) {
    icp_set_source(s, src, n, stride, src_normals, stride_n, src_indices, n_idx, guess);
  });
}

int pclb200_icp_iterate(pclb200_icp* icp, int max_steps, pclb200_icp_stats* stats)
{
  return on_ctx(icp, [&](Icp& s) { icp_iterate(s, max_steps, stats); });
}

int pclb200_icp_set_source_batch(pclb200_icp* icp, const void* src, size_t n, size_t stride, const void* src_normals,
                                 size_t stride_n, const int64_t* offsets, int32_t n_problems, const double* guesses)
{
  return on_ctx(icp, [&](Icp& s) {
    icp_set_source_batch(s, src, n, stride, src_normals, stride_n, offsets, n_problems, guesses);
  });
}

int pclb200_icp_set_target_batch(pclb200_icp* icp, const pclb200_index* const* targets, const void* const* tgt_normals,
                                 size_t stride_n, int32_t n_targets)
{
  return on_ctx(icp, [&](Icp& s) {
    PCLB_REQUIRE(targets, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(n_targets >= 1 && n_targets <= 65536, PCLB200_ERR_INVALID, "icp: a batch holds 1 to 65536 problems");
    std::vector<const Index*> idx(n_targets);
    for (int p = 0; p < n_targets; ++p) {
      PCLB_REQUIRE(targets[p] && targets[p]->idx, PCLB200_ERR_INVALID, "NULL argument");
      idx[p] = targets[p]->idx;
    }
    icp_set_target_batch(s, idx.data(), tgt_normals, stride_n, n_targets);
  });
}

int pclb200_icp_iterate_batch(pclb200_icp* icp, int max_steps, pclb200_icp_stats* stats)
{
  return on_ctx(icp, [&](Icp& s) { icp_iterate_batch(s, max_steps, stats); });
}

int pclb200_icp_get_correspondences_batch(pclb200_icp* icp, pclb200_corr* out, int64_t* counts)
{
  return on_ctx(icp, [&](Icp& s) {
    PCLB_REQUIRE(out && counts, PCLB200_ERR_INVALID, "NULL argument");
    icp_get_correspondences_batch(s, out, counts);
  });
}

int pclb200_icp_fitness_score_batch(pclb200_icp* icp, double max_range, double* scores)
{
  return on_ctx(icp, [&](Icp& s) {
    PCLB_REQUIRE(scores, PCLB200_ERR_INVALID, "NULL argument");
    icp_fitness_score_batch(s, max_range, scores);
  });
}

int pclb200_icp_get_cloud(pclb200_icp* icp, void* out_pts, size_t stride_out, void* out_normals, size_t stride_n)
{
  return on_ctx(icp, [&](Icp& s) {
    PCLB_REQUIRE(out_pts, PCLB200_ERR_INVALID, "NULL argument");
    icp_get_cloud(s, out_pts, stride_out, out_normals, stride_n);
  });
}

int pclb200_icp_get_correspondences(pclb200_icp* icp, pclb200_corr* out, size_t* n_out)
{
  return on_ctx(icp, [&](Icp& s) {
    PCLB_REQUIRE(out && n_out, PCLB200_ERR_INVALID, "NULL argument");
    *n_out = icp_get_correspondences(s, out);
  });
}

int pclb200_icp_align(pclb200_ctx* ctx, const pclb200_icp_params* params, const void* src, size_t n, size_t stride,
                      const void* src_normals, size_t stride_sn, const int32_t* src_indices, size_t n_idx,
                      const pclb200_index* idx_tgt, const void* tgt_normals, size_t stride_tn, const double guess[16],
                      void* out_cloud, size_t stride_out, pclb200_icp_stats* stats)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(params && idx_tgt && idx_tgt->idx, PCLB200_ERR_INVALID, "NULL argument");
    struct Guard {
      Icp* s;
      ~Guard() { icp_destroy(s); }
    } g{icp_create(c, *params)};
    icp_set_target(*g.s, idx_tgt->idx, tgt_normals, stride_tn);
    icp_set_source(*g.s, src, n, stride, src_normals, stride_sn, src_indices, n_idx, guess);
    icp_iterate(*g.s, std::numeric_limits<int>::max(), stats);
    if (out_cloud) {
      void* out_n = nullptr;
      if (src_normals)  // normals live inside the same records, at the same offset as in the input
        out_n = static_cast<unsigned char*>(out_cloud) +
                (static_cast<const unsigned char*>(src_normals) - static_cast<const unsigned char*>(src));
      icp_get_cloud(*g.s, out_cloud, stride_out, out_n, stride_sn);
    }
  });
}

int pclb200_fitness_score(pclb200_ctx* ctx, const pclb200_index* idx_tgt, const void* src, size_t n, size_t stride,
                          const int32_t* src_indices, size_t n_idx, int is_dense, const double T[16],
                          int scalar_is_double, double max_range, double* score)
{
  (void)is_dense;
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(idx_tgt && idx_tgt->idx && T && score, PCLB200_ERR_INVALID, "NULL argument");
    *score = fitness_score(c, *idx_tgt->idx, src, n, stride, src_indices, n_idx, T, scalar_is_double, max_range);
  });
}

int pclb200_fitness_score_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* src, size_t n,
                                  size_t stride, const int32_t* src_indices, size_t n_idx, int is_dense, const double T[16],
                                  int scalar_is_double, double max_range, double* score)
{
  (void)is_dense;
  return on_ctx(ctx, [&](Ctx& c) {
    const char* fault = idx_tile && idx_tile->idx && T && score && (src || !n) ? nullptr
                                                                              : "fitness_score_sharded: NULL argument";
    const double v = fitness_score_sharded(c, idx_tile ? idx_tile->idx : nullptr, src, n, stride, src_indices, n_idx, T,
                                           scalar_is_double, max_range, -1, fault);
    *score = v;
  });
}

// The collective calls below refuse on every rank when any rank refuses its arguments: a fault found here travels with the
// first exchange (require_same_count in icp.cu) instead of returning before it.
int pclb200_validate_transformation_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* src, size_t n,
                                            size_t stride, const double T[16], int scalar_is_double, double max_range,
                                            double* score)
{
  return on_ctx(ctx, [&](Ctx& c) {
    const char* fault = idx_tile && idx_tile->idx && T && score && (src || !n)
                            ? nullptr
                            : "validate_transformation_sharded: NULL argument";
    const double v = fitness_score_sharded(c, idx_tile ? idx_tile->idx : nullptr, src, n, stride, nullptr, 0, T, scalar_is_double, max_range,
                                           scalar_is_double ? kApplyValidationDouble : kApplyIcp, fault);
    *score = v;
  });
}

int pclb200_correspondences_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const pclb200_index* idx_src,
                                    const void* src, size_t n, size_t stride, const int32_t* src_indices, size_t n_idx,
                                    int is_dense, double max_dist, const void* tgt_normals, size_t stride_tn,
                                    pclb200_corr* out, float* out_xyz1, float* out_normals, size_t* n_out)
{
  (void)is_dense;  // non-finite source points never produce a correspondence on either setting
  return on_ctx(ctx, [&](Ctx& c) {
    const size_t nq = src_indices ? n_idx : n;
    const char* fault = nullptr;
    if (!idx_tile || !idx_tile->idx || !n_out || (nq && (!src || !out)) || (idx_src && !idx_src->idx))
      fault = "correspondences_sharded: NULL argument";
    const size_t m = correspondences_sharded(c, idx_tile ? idx_tile->idx : nullptr, idx_src ? idx_src->idx : nullptr, src, n, stride,
                                             src_indices, n_idx, max_dist, tgt_normals, stride_tn, out, out_xyz1,
                                             out_normals, fault);
    *n_out = m;
  });
}

int pclb200_correspondences_normals_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, int kind, const void* src,
                                            size_t n, size_t stride, const void* src_normals, size_t stride_sn,
                                            const void* tgt_normals, size_t stride_tn, const int32_t* src_indices,
                                            size_t n_idx, int k, double max_dist, pclb200_corr* out, float* out_xyz1,
                                            float* out_normals, size_t* n_out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    const size_t nq = src_indices ? n_idx : n;
    const char* fault = nullptr;
    if (!idx_tile || !idx_tile->idx || !n_out || (nq && k && (!src || !out)))
      fault = "correspondences_normals_sharded: NULL argument";
    else if (kind != PCLB200_CORR_NORMAL_SHOOTING && kind != PCLB200_CORR_BACK_PROJECTION)
      fault = "correspondences_normals_sharded: kind must be PCLB200_CORR_NORMAL_SHOOTING or PCLB200_CORR_BACK_PROJECTION";
    else if (k < 0)
      fault = "correspondences_normals_sharded: k < 0";
    else if (nq && k && !src_normals)
      fault = "correspondences_normals_sharded: source normals are required";
    else if (nq && k && kind == PCLB200_CORR_BACK_PROJECTION && !tgt_normals)
      fault = "correspondences_normals_sharded: back projection needs target normals";
    else if (out_normals && !tgt_normals)
      fault = "correspondences_normals_sharded: out_normals needs tgt_normals";
    const size_t m = correspondences_normals_sharded(c, idx_tile ? idx_tile->idx : nullptr, kind, src, n, stride,
                                                     src_normals, stride_sn, tgt_normals, stride_tn, src_indices, n_idx,
                                                     k, max_dist, out, out_xyz1, out_normals, fault);
    *n_out = m;
  });
}

int pclb200_inliers_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* src, size_t n, size_t stride,
                            const double T[16], float inlier_threshold, pclb200_corr* out, float* out_xyz1,
                            size_t* n_out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    const char* fault =
        idx_tile && idx_tile->idx && T && out && n_out && (src || !n) ? nullptr : "inliers_sharded: NULL argument";
    // pclb200_inliers: transformPointCloud (float), then d2 < inlier_threshold^2 (strict); no point passes a threshold of 0
    // on any rank, but every rank still takes part in the exchange
    const float max_range = inlier_threshold * inlier_threshold;
    const float gate = max_range > 0.f ? std::nextafter(max_range, -std::numeric_limits<float>::infinity()) : -1.f;
    const size_t m = correspondences_sharded(c, idx_tile ? idx_tile->idx : nullptr, nullptr, src, n, stride, nullptr, 0,
                                             0.0, nullptr, 0, out,
                                             out_xyz1, nullptr, fault, T, kApplyTransformsFloat, &gate);
    *n_out = m;
  });
}

int pclb200_gicp_covariances(pclb200_ctx* ctx, const pclb200_index* idx, const void* pts, size_t n, size_t stride, int k,
                             double gicp_epsilon, double* out_cov)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(idx && idx->idx && pts && out_cov, PCLB200_ERR_INVALID, "NULL argument");
    ProfScope ps(c, "gicp_covariances");
    gicp_covariances(c, *idx->idx, pts, n, stride, k, gicp_epsilon, out_cov);
  });
}

int pclb200_validate_transformation(pclb200_ctx* ctx, const pclb200_index* idx_tgt, const void* src, size_t n,
                                    size_t stride, const double T[16], int scalar_is_double, double max_range,
                                    double* score)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(idx_tgt && idx_tgt->idx && T && score, PCLB200_ERR_INVALID, "NULL argument");
    // transformation_validation_euclidean.hpp:62-75: T(0,0)*x + T(0,1)*y + T(0,2)*z + T(0,3) in Scalar, cast to float
    *score = fitness_score(c, *idx_tgt->idx, src, n, stride, nullptr, 0, T, scalar_is_double, max_range,
                           scalar_is_double ? kApplyValidationDouble : kApplyIcp);
  });
}

// Shared body of pclb200_fitness_score_batch / pclb200_validate_transformation_batch: the refusals of
// include/pclb200_batch.h, all checked before anything runs, then the batch in the single call's operation order `mode`
static void fitness_batch_call(Ctx& c, const char* name, const pclb200_index* const* targets, int32_t n_problems,
                               const void* src, size_t n, size_t stride, const int64_t* offsets, const double* transforms,
                               int mode, double max_range, double* scores)
{
  const std::string who(name);
  PCLB_REQUIRE(n_problems >= 1 && n_problems <= 65536, PCLB200_ERR_INVALID, who + ": a batch holds 1 to 65536 problems");
  PCLB_REQUIRE(targets && src && offsets && transforms && scores, PCLB200_ERR_INVALID, "NULL argument");
  const int B = n_problems;
  std::vector<const Index*> idx(B);
  for (int p = 0; p < B; ++p) {
    PCLB_REQUIRE(targets[p] && targets[p]->idx, PCLB200_ERR_INVALID, who + ": a NULL handle");
    PCLB_REQUIRE(targets[p]->idx->device == c.device, PCLB200_ERR_INVALID,
                 who + ": an index lives on another device than the context");
    idx[p] = targets[p]->idx;
  }
  PCLB_REQUIRE(offsets[0] == 0 && offsets[B] == (int64_t)n, PCLB200_ERR_INVALID, who + ": offsets must run from 0 to n");
  for (int p = 0; p < B; ++p)
    PCLB_REQUIRE(offsets[p + 1] > offsets[p], PCLB200_ERR_INVALID,
                 who + ": offsets must increase strictly (every problem holds a record)");
  PCLB_REQUIRE(n < (size_t)0x7fffffff, PCLB200_ERR_INVALID, who + ": a batch holds fewer than 2^31 - 1 records");
  PCLB_REQUIRE(stride >= 12 && stride % 4 == 0, PCLB200_ERR_INVALID, "stride must be a multiple of 4 and >= 12");
  ProfScope ps(c, "fitness_score_batch");
  fitness_score_batch(c, idx.data(), B, src, n, stride, offsets, transforms, mode, max_range, scores);
}

int pclb200_fitness_score_batch(pclb200_ctx* ctx, const pclb200_index* const* targets, int32_t n_problems, const void* src,
                                size_t n, size_t stride, const int64_t* offsets, const double* transforms,
                                int scalar_is_double, double max_range, double* scores)
{
  return on_ctx(ctx, [&](Ctx& c) {
    fitness_batch_call(c, "fitness_score_batch", targets, n_problems, src, n, stride, offsets, transforms,
                       scalar_is_double ? kApplyTransformsDouble : kApplyTransformsFloat, max_range, scores);
  });
}

int pclb200_validate_transformation_batch(pclb200_ctx* ctx, const pclb200_index* const* targets, int32_t n_problems,
                                          const void* src, size_t n, size_t stride, const int64_t* offsets,
                                          const double* transforms, int scalar_is_double, double max_range,
                                          double* scores)
{
  return on_ctx(ctx, [&](Ctx& c) {
    fitness_batch_call(c, "validate_transformation_batch", targets, n_problems, src, n, stride, offsets, transforms,
                       scalar_is_double ? kApplyValidationDouble : kApplyIcp, max_range, scores);
  });
}

int pclb200_inliers(pclb200_ctx* ctx, const pclb200_index* idx_tgt, const void* src, size_t n, size_t stride,
                    const double T[16], float inlier_threshold, pclb200_corr* out, size_t* n_out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(idx_tgt && idx_tgt->idx && T && out && n_out, PCLB200_ERR_INVALID, "NULL argument");
    // sample_consensus_prerejective.hpp:318-338: transformPointCloud (float), then nn_dists[0] < max_range (STRICT, float)
    const float max_range = inlier_threshold * inlier_threshold;
    const float gate = std::nextafter(max_range, -std::numeric_limits<float>::infinity());  // d2 <= gate  <=>  d2 < max_range
    *n_out = max_range > 0.f ? correspondences(c, *idx_tgt->idx, nullptr, src, n, stride, nullptr, 0, 1, 0.0, out, T,
                                               kApplyTransformsFloat, &gate)
                             : 0;
  });
}

// ---- normals ----------------------------------------------------------------------------------------------------------------
int pclb200_normals_knn(pclb200_ctx* ctx, const pclb200_index* h, const void* pts, size_t n, size_t stride,
                        const int32_t* indices, size_t n_idx, int is_dense, int k, const float viewpoint[3], float* out,
                        int* is_dense_out)
{
  (void)is_dense;
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(h && h->idx && out && viewpoint, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(k > 0, PCLB200_ERR_INVALID, "k must be positive (feature.hpp:135-176)");
    normals(c, *h->idx, pts, n, stride, indices, n_idx, out, is_dense_out,
            [&](const float4* d_q, size_t nq, float4* d_out, int* d_flag) {
              launch_normals(c, *h->idx, d_q, nq, k, viewpoint, d_out, d_flag);
            });
  });
}

int pclb200_normals_knn_batch(pclb200_ctx* ctx, const pclb200_index* const* indices, int32_t n_clouds, const void* pts,
                              size_t n, size_t stride, const int64_t* offsets, int k, const float* viewpoints, float* out,
                              int32_t* is_dense_out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(n_clouds >= 1 && n_clouds <= 65536, PCLB200_ERR_INVALID, "normals_knn_batch: a batch holds 1 to 65536 query sets");
    PCLB_REQUIRE(indices && pts && offsets && out, PCLB200_ERR_INVALID, "NULL argument");
    const int B = n_clouds;
    std::vector<Index*> idx(B);
    for (int b = 0; b < B; ++b) {
      PCLB_REQUIRE(indices[b] && indices[b]->idx, PCLB200_ERR_INVALID, "normals_knn_batch: a NULL handle");
      PCLB_REQUIRE(indices[b]->idx->device == c.device, PCLB200_ERR_INVALID,
                   "normals_knn_batch: an index lives on another device than the context");
      idx[b] = indices[b]->idx;
    }
    PCLB_REQUIRE(offsets[0] == 0 && offsets[B] == (int64_t)n, PCLB200_ERR_INVALID,
                 "normals_knn_batch: offsets must run from 0 to n");
    for (int b = 0; b < B; ++b)
      PCLB_REQUIRE(offsets[b + 1] > offsets[b], PCLB200_ERR_INVALID,
                   "normals_knn_batch: offsets must increase strictly (every query set holds a record)");
    PCLB_REQUIRE(n < (size_t)0x7fffffff, PCLB200_ERR_INVALID, "normals_knn_batch: a batch holds fewer than 2^31 - 1 records");
    PCLB_REQUIRE(stride >= 12 && stride % 4 == 0, PCLB200_ERR_INVALID, "stride must be a multiple of 4 and >= 12");
    PCLB_REQUIRE(k > 0, PCLB200_ERR_INVALID, "k must be positive (feature.hpp:135-176)");
    cudaStream_t st = c.stream;
    std::vector<float> vps(3 * (size_t)B, 0.f);
    if (viewpoints)
      std::copy(viewpoints, viewpoints + 3 * (size_t)B, vps.begin());
    // every record once, keyed in its own index's frame, then stably by set: each set's queries in its single call's order
    std::vector<float4> frames(B);
    for (int b = 0; b < B; ++b)
      frames[b] = make_float4(idx[b]->lo[0], idx[b]->lo[1], idx[b]->lo[2], idx[b]->morton_scale);
    DevBuf<float4> d_frames, dense;
    DevBuf<long long> d_offsets;
    d_frames.alloc(B, st);
    d_offsets.alloc(B + 1, st);
    PCLB_CUDA(cudaMemcpyAsync(d_frames.p, frames.data(), B * sizeof(float4), cudaMemcpyHostToDevice, st));
    PCLB_CUDA(cudaMemcpyAsync(d_offsets.p, offsets, (B + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
    dense.alloc(n, st);
    load_xyz_as_float4(c, pts, n, stride, nullptr, 0, dense.p, st);
    QueryBatch qb;
    {
      ProfScope ps(c, "query_sort");
      make_query_batch_framed(c, d_frames.p, d_offsets.p, B, dense.p, n, qb);
      sort_by_problem(c, d_offsets.p, B, qb);
    }
    DevBuf<float4> tmp;
    DevBuf<int> d_flags;
    d_flags.alloc(B, st);
    PCLB_CUDA(cudaMemsetAsync(d_flags.p, 0, B * sizeof(int), st));
    float4* const caller_out = reinterpret_cast<float4*>(out);
    {
      ProfScope ps(c, "normals_batch");
      launch_normals_batch(c, idx.data(), B, d_offsets.p, qb.q.p, n, k, vps.data(), out_on_device(c, caller_out, n, tmp),
                           d_flags.p);
    }
    std::vector<int> flags(B);
    PCLB_CUDA(cudaMemcpyAsync(flags.data(), d_flags.p, B * sizeof(int), cudaMemcpyDeviceToHost, st));
    copy_out(c, caller_out, tmp, n);
    check_device_error(c);
    if (is_dense_out)
      for (int b = 0; b < B; ++b)
        is_dense_out[b] = flags[b] ? 0 : 1;
  });
}

int pclb200_normals_radius(pclb200_ctx* ctx, const pclb200_index* h, const void* pts, size_t n, size_t stride,
                           const int32_t* indices, size_t n_idx, int is_dense, double radius, const float viewpoint[3],
                           float* out, int* is_dense_out)
{
  (void)is_dense;
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(h && h->idx && out && viewpoint, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(radius > 0.0, PCLB200_ERR_INVALID, "radius must be positive (feature.hpp:135-176)");
    normals(c, *h->idx, pts, n, stride, indices, n_idx, out, is_dense_out,
            [&](const float4* d_q, size_t nq, float4* d_out, int* d_flag) {
              launch_normals_radius(c, *h->idx, d_q, nq, (float)(radius * radius), viewpoint, d_out, d_flag);
            });
  });
}

int pclb200_normals_knn_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* pts, size_t n, size_t stride,
                                const int32_t* indices, size_t n_idx, int is_dense, int k, const float viewpoint[3],
                                float* out, int* is_dense_out)
{
  (void)is_dense;
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(idx_tile && idx_tile->idx && out && viewpoint, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(k > 0, PCLB200_ERR_INVALID, "k must be positive (feature.hpp:135-176)");
    normals_sharded(c, *idx_tile->idx, pts, n, stride, indices, n_idx, k, 0.f, out, is_dense_out,
                    [&](Index& local, const float4* d_q, size_t nq, float4* d_out, int* d_flag) {
                      launch_normals(c, local, d_q, nq, k, viewpoint, d_out, d_flag);
                    });
  });
}

int pclb200_normals_radius_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* pts, size_t n,
                                   size_t stride, const int32_t* indices, size_t n_idx, int is_dense, double radius,
                                   const float viewpoint[3], float* out, int* is_dense_out)
{
  (void)is_dense;
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(idx_tile && idx_tile->idx && out && viewpoint, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(radius > 0.0, PCLB200_ERR_INVALID, "radius must be positive (feature.hpp:135-176)");
    const float r2 = (float)(radius * radius);
    normals_sharded(c, *idx_tile->idx, pts, n, stride, indices, n_idx, 0, r2, out, is_dense_out,
                    [&](Index& local, const float4* d_q, size_t nq, float4* d_out, int* d_flag) {
                      launch_normals_radius(c, local, d_q, nq, r2, viewpoint, d_out, d_flag);
                    });
  });
}

// ---- k-NN and the outlier filters on a sharded map ---------------------------------------------------------------------------
int pclb200_knn_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* queries, size_t nq, size_t stride,
                        int k, int32_t* out_idx, float* out_d2, int* k_eff)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(idx_tile && idx_tile->idx && (!nq || (queries && out_idx && out_d2)), PCLB200_ERR_INVALID,
                 "NULL argument");
    const size_t n_out = nq * (size_t)std::max(k, 0);
    DevBuf<int32_t> ti;
    DevBuf<float> td;
    const int keff = knn_sharded(c, *idx_tile->idx, queries, nq, stride, k, out_on_device(c, out_idx, n_out, ti),
                                 out_on_device(c, out_d2, n_out, td));
    copy_out(c, out_idx, ti, n_out);
    copy_out(c, out_d2, td, n_out);
    check_device_error(c);
    if (k_eff)
      *k_eff = keff;
  });
}

int pclb200_knn_stats_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* pts, size_t n, size_t stride,
                              const int32_t* indices, size_t n_idx, int k, float* out_mean, float* out_kth)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(idx_tile && idx_tile->idx && (out_mean || out_kth), PCLB200_ERR_INVALID, "NULL argument");
    const size_t nq = indices ? n_idx : n;
    DevBuf<float> tm, tk;
    knn_stats_sharded(c, *idx_tile->idx, pts, n, stride, indices, n_idx, k, out_on_device(c, out_mean, nq, tm),
                      out_on_device(c, out_kth, nq, tk));
    copy_out(c, out_mean, tm, nq);
    copy_out(c, out_kth, tk, nq);
    check_device_error(c);
  });
}

int pclb200_statistical_outlier_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* pts, size_t n,
                                        size_t stride, const int32_t* indices, size_t n_idx, int mean_k, double std_mul,
                                        int negative, uint8_t* keep, double stats[3])
{
  return on_ctx(ctx, [&](Ctx& c) {
    const size_t nq = indices ? n_idx : n;
    PCLB_REQUIRE(idx_tile && idx_tile->idx && (keep || !nq), PCLB200_ERR_INVALID, "NULL argument");
    DevBuf<unsigned char> tk;
    DevBuf<double> d_stats;
    d_stats.alloc(3, c.stream);
    statistical_outlier_sharded(c, *idx_tile->idx, pts, n, stride, indices, n_idx, mean_k, std_mul, negative,
                                out_on_device(c, keep, nq, tk), d_stats.p);
    copy_out(c, keep, tk, nq);
    double h[3];
    PCLB_CUDA(cudaMemcpyAsync(h, d_stats.p, sizeof(h), cudaMemcpyDeviceToHost, c.stream));
    check_device_error(c);
    if (stats)
      std::copy(h, h + 3, stats);
  });
}

int pclb200_radius_outlier_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* pts, size_t n,
                                   size_t stride, const int32_t* indices, size_t n_idx, int is_dense, double radius,
                                   int min_pts, int negative, uint8_t* keep)
{
  return on_ctx(ctx, [&](Ctx& c) {
    const size_t nq = indices ? n_idx : n;
    PCLB_REQUIRE(idx_tile && idx_tile->idx && (keep || !nq), PCLB200_ERR_INVALID, "NULL argument");
    DevBuf<unsigned char> tk;
    radius_outlier_sharded(c, *idx_tile->idx, pts, n, stride, indices, n_idx, is_dense, radius, min_pts, negative,
                           out_on_device(c, keep, nq, tk));
    copy_out(c, keep, tk, nq);
    check_device_error(c);
  });
}

// ---- radius search and GICP covariances on a sharded map ----------------------------------------------------------------------
// A fault found here travels with the verdict exchange (shard_filter.cu) instead of returning before it.
int pclb200_radius_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* queries, size_t nq, size_t stride,
                           double radius, unsigned max_nn, int sorted, int64_t* out_offsets, int32_t** out_idx,
                           float** out_d2)
{
  (void)sorted;
  return on_ctx(ctx, [&](Ctx& c) {
    const char* fault = nullptr;
    if (!idx_tile || !idx_tile->idx || !out_offsets || !out_idx || !out_d2 || (nq && !queries))
      fault = "radius_sharded: NULL argument";
    else if (is_device_ptr(out_offsets))
      fault = "radius_sharded returns host arrays: out_offsets must be host memory";
    if (!fault) {
      *out_idx = nullptr;
      *out_d2 = nullptr;
    }
    radius_sharded(c, idx_tile ? idx_tile->idx : nullptr, queries, nq, stride, radius, max_nn, out_offsets,
                   [&](unsigned long long total) {
                     if (!nq)
                       return RadiusSinkBuffers{nullptr, nullptr};  // as pclb200_radius: no arrays for no query
                     int32_t* hi = static_cast<int32_t*>(malloc(std::max<size_t>(total, 1) * sizeof(int32_t)));
                     float* hd = static_cast<float*>(malloc(std::max<size_t>(total, 1) * sizeof(float)));
                     *out_idx = hi;  // owned by the caller from here on (pclb200_free), also on the error paths
                     *out_d2 = hd;
                     PCLB_REQUIRE(hi && hd, PCLB200_ERR_INTERNAL, "host allocation failed");
                     return RadiusSinkBuffers{hi, hd};
                   },
                   fault);
  });
}

int pclb200_radius_into_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* queries, size_t nq,
                                size_t stride, double radius, unsigned max_nn, int64_t* out_offsets, int32_t* out_idx,
                                float* out_d2, size_t capacity, size_t* total, int* all_fit)
{
  return on_ctx(ctx, [&](Ctx& c) {
    const char* fault = nullptr;
    if (!idx_tile || !idx_tile->idx || !out_offsets || !total || (nq && !queries))
      fault = "radius_into_sharded: NULL argument";
    else if (capacity > 0 && !(out_idx && out_d2))
      fault = "radius_into_sharded: NULL output buffers with a non-zero capacity";
    if (!fault)
      *total = 0;
    radius_sharded(c, idx_tile ? idx_tile->idx : nullptr, queries, nq, stride, radius, max_nn, out_offsets,
                   [&](unsigned long long n) {
                     *total = (size_t)n;
                     // every rank has its count here: one u64 minimum tells all of them whether every rank's lists fit
                     const bool fits = (size_t)n <= capacity;
                     const int every = ranks_min(c, fits ? 1 : 0) ? 1 : 0;
                     if (all_fit)
                       *all_fit = every;
                     if (!fits)
                       return RadiusSinkBuffers{nullptr, nullptr};  // offsets and *total are valid; call again with room
                     return RadiusSinkBuffers{out_idx, out_d2};
                   },
                   fault);
  });
}

int pclb200_gicp_covariances_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, const void* pts, size_t n,
                                     size_t stride, int k, double gicp_epsilon, double* out_cov)
{
  return on_ctx(ctx, [&](Ctx& c) {
    const char* fault =
        idx_tile && idx_tile->idx && (!n || (pts && out_cov)) ? nullptr : "gicp_covariances_sharded: NULL argument";
    gicp_covariances_sharded(c, idx_tile ? idx_tile->idx : nullptr, pts, n, stride, k, gicp_epsilon, out_cov, fault);
    check_device_error(c);
  });
}

// ---- Euclidean clustering --------------------------------------------------------------------------------------------------
int pclb200_cluster_labels(pclb200_ctx* ctx, const pclb200_index* h, double tolerance, int32_t* out_labels, size_t n_labels)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(h && h->idx && out_labels, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(tolerance >= 0.0, PCLB200_ERR_INVALID, "negative cluster tolerance");
    const Index& idx = *h->idx;
    PCLB_REQUIRE(!idx.labelled, PCLB200_ERR_INVALID,
                 "cluster_labels: an index built with caller ids (pclb200_index_build_ids) has no cloud to size the labels by");
    PCLB_REQUIRE(n_labels == idx.n_cloud, PCLB200_ERR_INVALID,
                 "out_labels must hold one entry per point of the cloud the index was built from");
    DevBuf<int32_t> tmp;
    cluster_labels(c, idx, tolerance, out_on_device(c, out_labels, n_labels, tmp));
    copy_out(c, out_labels, tmp, n_labels);
    check_device_error(c);
  });
}

int pclb200_cluster_labels_sharded(pclb200_ctx* ctx, const pclb200_index* idx_tile, double tolerance, int32_t* out_labels,
                                   int64_t* out_sizes, size_t n_labels)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(idx_tile && idx_tile->idx && out_labels, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID,
                 "sharded clusters need an active communicator (pclb200_comm_init or pclb200_comm_export / _import)");
    const Index& tile = *idx_tile->idx;
    PCLB_REQUIRE(tile.labelled, PCLB200_ERR_INVALID,
                 "sharded clusters: every rank's tile must be built with pclb200_index_build_ids");
    PCLB_REQUIRE(tolerance >= 0.0, PCLB200_ERR_INVALID, "negative cluster tolerance");
    PCLB_REQUIRE(n_labels == tile.n_cloud, PCLB200_ERR_INVALID,
                 "out_labels must hold one entry per record the tile was built from");
    DevBuf<int32_t> tmp;
    DevBuf<int64_t> tmp_sizes;
    cluster_labels_sharded(c, tile, tolerance, out_on_device(c, out_labels, n_labels, tmp),
                           out_on_device(c, out_sizes, n_labels, tmp_sizes));
    copy_out(c, out_labels, tmp, n_labels);
    copy_out(c, out_sizes, tmp_sizes, n_labels);
    check_device_error(c);
  });
}

int pclb200_comm_allgather_u64(pclb200_ctx* ctx, const uint64_t* send, size_t n, uint64_t* recv, size_t capacity,
                               size_t* n_total)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(n_total && (send || !n), PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID,
                 "allgather needs an active communicator (pclb200_comm_init or pclb200_comm_export / _import)");
    DevBuf<unsigned long long> staging, all;
    const unsigned long long* d = on_device(c, reinterpret_cast<const unsigned long long*>(send), n, staging);
    const size_t total = allgather_u64(c, d, n, all);
    if (recv && total && capacity >= total)
      PCLB_CUDA(cudaMemcpyAsync(recv, all.p, total * sizeof(uint64_t), cudaMemcpyDefault, c.stream));
    check_device_error(c);
    *n_total = total;
  });
}

// ---- voxel grid ---------------------------------------------------------------------------------------------------------------
int pclb200_voxelgrid(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx,
                      int is_dense, const float leaf[3], unsigned min_points_per_voxel, float* out_xyz1, size_t* n_out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(leaf && out_xyz1 && n_out, PCLB200_ERR_INVALID, "NULL argument");
    ProfScope ps(c, "voxelgrid");
    *n_out = voxelgrid(c, pts, n, stride, indices, n_idx, is_dense, leaf, min_points_per_voxel, out_xyz1, nullptr, 0,
                       nullptr);
  });
}

int pclb200_voxelgrid_tile(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const float grid_bounds[6],
                           const float leaf[3], unsigned min_points_per_voxel, float* out_xyz1, size_t* n_out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(leaf && out_xyz1 && n_out && grid_bounds, PCLB200_ERR_INVALID, "NULL argument");
    ProfScope ps(c, "voxelgrid");
    *n_out = voxelgrid(c, pts, n, stride, nullptr, 0, 0, leaf, min_points_per_voxel, out_xyz1, nullptr, 0, nullptr,
                       grid_bounds);
  });
}

int pclb200_voxelgrid_normals(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const void* normals,
                              size_t stride_n, const int32_t* indices, size_t n_idx, int is_dense, const float leaf[3],
                              unsigned min_points_per_voxel, float* out_xyz1, float* out_normal_curv, size_t* n_out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(leaf && out_xyz1 && n_out && normals && out_normal_curv, PCLB200_ERR_INVALID, "NULL argument");
    ProfScope ps(c, "voxelgrid");
    *n_out = voxelgrid(c, pts, n, stride, indices, n_idx, is_dense, leaf, min_points_per_voxel, out_xyz1, normals,
                       stride_n, out_normal_curv);
  });
}

int pclb200_voxelgrid_batch(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const int64_t* offsets,
                            int32_t n_clouds, const float leaf[3], unsigned min_points_per_voxel, const void* normals,
                            size_t stride_n, float* out_xyz1, float* out_normal_curv, int64_t* out_offsets)
{
  return on_ctx(ctx, [&](Ctx& c) {
    ProfScope ps(c, "voxelgrid_batch");
    voxelgrid_batch(c, pts, n, stride, offsets, n_clouds, leaf, min_points_per_voxel, normals, stride_n, out_xyz1,
                    out_normal_curv, out_offsets);
  });
}

int pclb200_voxelgrid_sharded(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const int32_t* ids,
                              const void* normals, size_t stride_n, const float leaf[3], unsigned min_points_per_voxel,
                              float* out_xyz1, float* out_normal_curv, uint32_t* out_voxel, size_t* n_out)
{
  return on_ctx(ctx, [&](Ctx& c) {
    voxelgrid_sharded(c, pts, n, stride, ids, normals, stride_n, leaf, min_points_per_voxel, out_xyz1, out_normal_curv,
                      out_voxel, n_out);
  });
}

// ---- multi-GPU ------------------------------------------------------------------------------------------------------------------
int pclb200_comm_unique_id(void* out_128_bytes)
{
  return guarded([&] {
    PCLB_REQUIRE(out_128_bytes, PCLB200_ERR_INVALID, "NULL argument");
    comm_unique_id(out_128_bytes);
  });
}

int pclb200_comm_init(pclb200_ctx* ctx, int rank, int nranks, const void* unique_id)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(nranks == 1 || unique_id, PCLB200_ERR_INVALID, "NULL argument");
    comm_init(c, rank, nranks, unique_id);
  });
}

int pclb200_comm_set_mode(pclb200_ctx* ctx, int mode)
{
  return on_ctx(ctx, [&](Ctx& c) { comm_set_mode(c, mode); });
}

int pclb200_comm_export(pclb200_ctx* ctx, void* out_handle_64_bytes)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(out_handle_64_bytes, PCLB200_ERR_INVALID, "NULL argument");
    comm_export(c, out_handle_64_bytes);
  });
}

int pclb200_comm_import(pclb200_ctx* ctx, int rank, int nranks, const void* handles)
{
  return on_ctx(ctx, [&](Ctx& c) {
    PCLB_REQUIRE(handles, PCLB200_ERR_INVALID, "NULL argument");
    comm_import(c, rank, nranks, handles);
  });
}

}  // extern "C"
