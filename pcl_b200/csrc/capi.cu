// capi.cu — the C boundary of libpclb200.so (include/pclb200.h).  No exception crosses it; there is no CPU
// fallback: every entry point either runs the CUDA path or returns an error status.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <limits>
#include <memory>

#include "internal.cuh"

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
void icp_set_source(Icp& s, const void* src, size_t n, size_t stride, const void* src_normals, size_t stride_n,
                    const int32_t* indices, size_t n_idx, const double* guess);
void icp_iterate(Icp& s, int max_steps, pclb200_icp_stats* stats);
void icp_get_cloud(Icp& s, void* out_pts, size_t stride_out, void* out_normals, size_t stride_n);
size_t icp_get_correspondences(Icp& s, pclb200_corr* out);
void estimate_pairs(Ctx& c, int est, const void* src, size_t stride_s, const void* tgt, const void* tgt_normals,
                    size_t stride_t, const pclb200_corr* corr, size_t n, int scalar_is_double, double* T_out,
                    const void* src_normals = nullptr, int enforce_same_dir = 1, int svd_correlation = 0);
size_t correspondences(Ctx& c, const Index& tgt, const Index* src_index, const void* src, size_t n, size_t stride,
                       const int32_t* indices, size_t n_idx, int is_dense, double max_dist, pclb200_corr* out,
                       const double* pre_T = nullptr, int pre_mode = 0, const float* gate_override = nullptr);
double fitness_score(Ctx& c, const Index& tgt, const void* src, size_t n, size_t stride, const int32_t* indices,
                     size_t n_idx, const double* T, int scalar_is_double, double max_range, int mode_override = -1);
void gicp_covariances(Ctx& c, Index& idx, const void* pts, size_t n, size_t stride, int k, double gicp_epsilon,
                      double* out);
// search.cu
void launch_normals(Ctx& c, Index& idx, const float4* d_q, size_t nq, int k, const float vp[3], float4* d_out,
                    int* d_not_dense);
void launch_knn_stats(Ctx& c, const Index& idx, const float4* d_q, size_t nq, int k, float* d_mean, float* d_kth);
// voxel.cu
size_t voxelgrid(Ctx& c, const void* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int is_dense,
                 const float leaf[3], unsigned min_pts, float* out_xyz1, const void* normals, size_t stride_n,
                 float* out_normal_curv, const float* grid_bounds = nullptr);
// comm.cu
void comm_unique_id(void* out128);
void comm_export(Ctx& c, void* out64);
void comm_import(Ctx& c, int rank, int nranks, const void* handles);
void comm_set_mode(Ctx& c, int mode);
void comm_init(Ctx& c, int rank, int nranks, const void* unique_id);
void comm_destroy(Ctx& c);

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

static inline unsigned grid_for(size_t n, int block) { return (unsigned)((n + block - 1) / block); }

__global__ void k_iota_slots(float4* q, size_t n)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n)
    q[i].w = __int_as_float((int)i);
}

__global__ void k_unpack_keys(const unsigned long long* __restrict__ keys, size_t n, int32_t* __restrict__ idx,
                              float* __restrict__ d2)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) {
    unsigned long long k = keys[i];
    idx[i] = (int32_t)(unsigned)(k & 0xffffffffULL);
    d2[i] = __uint_as_float((unsigned)(k >> 32));
  }
}

// keep only the first max_nn entries of every (sorted) segment
__global__ void k_truncate_segments(const unsigned long long* __restrict__ keys,
                                    const unsigned long long* __restrict__ off_in,
                                    const unsigned long long* __restrict__ off_out, size_t nq,
                                    unsigned long long* __restrict__ out)
{
  size_t q = blockIdx.x;
  if (q >= nq)
    return;
  const unsigned long long b = off_in[q], bo = off_out[q], len = off_out[q + 1] - off_out[q];
  for (unsigned long long j = threadIdx.x; j < len; j += blockDim.x)
    out[bo + j] = keys[b + j];
}

// max_nn <= 32 radius search = "the max_nn nearest inside the ball": k-NN rows (-1 padded) -> CSR
__global__ void k_count_row_entries(const int32_t* __restrict__ rows, size_t nq, int k, unsigned long long* __restrict__ counts)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  unsigned long long c = 0;
  for (int j = 0; j < k; ++j)
    if (rows[i * (size_t)k + j] >= 0)
      ++c;
  counts[i] = c;
}

__global__ void k_pack_rows(const int32_t* __restrict__ rows, const float* __restrict__ rows_d2, size_t nq, int k,
                            const unsigned long long* __restrict__ offsets, int32_t* __restrict__ idx,
                            float* __restrict__ d2)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  unsigned long long o = offsets[i];
  for (int j = 0; j < k; ++j) {
    const int32_t v = rows[i * (size_t)k + j];
    if (v < 0)
      break;  // rows are filled from the front
    idx[o] = v;
    d2[o] = rows_d2[i * (size_t)k + j];
    ++o;
  }
}

__global__ void k_clamp_counts(const unsigned long long* __restrict__ in, size_t n, unsigned long long cap,
                               unsigned long long* __restrict__ out)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n)
    out[i] = in[i] < cap ? in[i] : cap;
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

// Shared body of pclb200_radius / pclb200_radius_into.  `sink(total)` returns where the packed lists go (host or device
// pointers; {nullptr, nullptr} = do not deliver, e.g. the caller's buffers are too small); offsets are written to
// out_offsets (host or device, nq + 1 entries).
struct RadiusSinkBuffers {
  int32_t* idx;
  float* d2;
};

__global__ void k_offsets_to_i64(const unsigned long long* __restrict__ in, size_t n, int64_t* __restrict__ out)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n)
    out[i] = (int64_t)in[i];
}

template <typename Sink>
static void radius_impl(Ctx& c, const Index& idx, const void* queries, size_t nq, size_t stride, double radius,
                        unsigned max_nn, int64_t* out_offsets, Sink&& sink)
{
    cudaStream_t st = c.stream;
    auto write_offsets = [&](const unsigned long long* d_off) {
      if (is_device_ptr(out_offsets)) {
        k_offsets_to_i64<<<grid_for(nq + 1, 256), 256, 0, st>>>(d_off, nq + 1, out_offsets);
        ++c.launches;
      }
      else {
        static_assert(sizeof(unsigned long long) == sizeof(int64_t), "offset width");
        PCLB_CUDA(cudaMemcpyAsync(out_offsets, d_off, (nq + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
      }
    };
    auto deliver = [&](const RadiusSinkBuffers& o, const int32_t* di, const float* dd, unsigned long long n) {
      if (!o.idx || !o.d2 || n == 0)
        return;
      PCLB_CUDA(cudaMemcpyAsync(o.idx, di, n * sizeof(int32_t),
                                is_device_ptr(o.idx) ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
      PCLB_CUDA(cudaMemcpyAsync(o.d2, dd, n * sizeof(float),
                                is_device_ptr(o.d2) ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
    };
    const float r2 = (float)(radius * radius);  // kdtree_flann.hpp:398
    if (max_nn == 0 || (size_t)max_nn > idx.n_valid)
      max_nn = (unsigned)idx.n_valid;            // :382-383
    DevBuf<float4> dense;
    dense.alloc(nq, st);
    load_xyz_as_float4(c, queries, nq, stride, nullptr, 0, dense.p, st);
    QueryBatch qb;
    make_query_batch(c, idx, dense.p, nq, qb);
    DevBuf<unsigned long long> counts, offsets, keys_sorted;
    unsigned long long total = 0;
    {
      ProfScope ps(c, "radius_count");
      radius_count(c, idx, qb.q.p, nq, r2, counts, offsets, total);
    }
    // KNNRadiusResultSet semantics (kdtree_flann.hpp:382-391): the max_nn nearest among those with d2 < r2.  Normally
    // the whole ball is materialised, sorted and cut (the passes below: ~3 ms per million queries at ~30 neighbours).
    // When the balls hold far more than max_nn points that would move (or overflow on) data that is thrown away, so
    // for max_nn <= 32 the register k-NN kernel runs instead, started with the pruning bound just below r2 (every
    // d2 < r2 is <= that bound; a candidate AT the bound still enters through the index tie rule).
    if ((size_t)max_nn < idx.n_valid && max_nn <= 32 && total > 16ULL * (unsigned long long)nq * max_nn) {
      const int k = (int)max_nn;
      DevBuf<int32_t> rows;
      DevBuf<float> rows_d2;
      rows.alloc(nq * (size_t)k, st);
      rows_d2.alloc(nq * (size_t)k, st);
      {
        ProfScope ps(c, "radius_knn");
        launch_knn(c, idx, qb.q.p, nq, k, std::nextafter(r2, -std::numeric_limits<float>::infinity()), rows.p, rows_d2.p);
      }
      DevBuf<unsigned long long> cnt, off;
      cnt.alloc(nq + 1, st);
      off.alloc(nq + 1, st);
      PCLB_CUDA(cudaMemsetAsync(cnt.p, 0, (nq + 1) * sizeof(unsigned long long), st));
      k_count_row_entries<<<grid_for(nq, 256), 256, 0, st>>>(rows.p, nq, k, cnt.p);
      size_t tb = 0;
      PCLB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt.p, off.p, (int)(nq + 1), st));
      DevBuf<unsigned char> tmp;
      tmp.alloc(tb, st);
      PCLB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, cnt.p, off.p, (int)(nq + 1), st));
      c.launches += 2;
      unsigned long long kept = 0;
      PCLB_CUDA(cudaMemcpyAsync(&kept, off.p + nq, sizeof(kept), cudaMemcpyDeviceToHost, st));
      write_offsets(off.p);
      PCLB_CUDA(cudaStreamSynchronize(st));
      const RadiusSinkBuffers o = sink(kept);
      if (kept > 0 && o.idx && o.d2) {
        DevBuf<int32_t> di;
        DevBuf<float> dd;
        di.alloc(kept, st);
        dd.alloc(kept, st);
        k_pack_rows<<<grid_for(nq, 256), 256, 0, st>>>(rows.p, rows_d2.p, nq, k, off.p, di.p, dd.p);
        ++c.launches;
        deliver(o, di.p, dd.p, kept);
        PCLB_CUDA(cudaStreamSynchronize(st));
      }
      check_device_error(c);
      return;
    }
    {
      ProfScope ps(c, "radius");
      radius_fill_sorted(c, idx, qb.q.p, nq, r2, offsets, total, keys_sorted);
    }
    const unsigned long long* d_final_keys = nullptr;
    const unsigned long long* d_final_off = offsets.p;
    unsigned long long final_total = total;
    DevBuf<unsigned long long> counts2, offsets2, keys_trunc;
    if (total > 0) {
      d_final_keys = keys_sorted.p;
      if ((size_t)max_nn < idx.n_valid) {  // KNNRadius semantics: the max_nn nearest inside the ball
        counts2.alloc(nq + 1, st);
        offsets2.alloc(nq + 1, st);
        PCLB_CUDA(cudaMemsetAsync(counts2.p, 0, (nq + 1) * sizeof(unsigned long long), st));
        k_clamp_counts<<<grid_for(nq, 256), 256, 0, st>>>(counts.p, nq, (unsigned long long)max_nn, counts2.p);
        size_t tb = 0;
        PCLB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, counts2.p, offsets2.p, (int)(nq + 1), st));
        DevBuf<unsigned char> tmp;
        tmp.alloc(tb, st);
        PCLB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, counts2.p, offsets2.p, (int)(nq + 1), st));
        PCLB_CUDA(cudaMemcpyAsync(&final_total, offsets2.p + nq, sizeof(final_total), cudaMemcpyDeviceToHost, st));
        PCLB_CUDA(cudaStreamSynchronize(st));
        keys_trunc.alloc(std::max<unsigned long long>(final_total, 1), st);
        k_truncate_segments<<<(unsigned)nq, 64, 0, st>>>(keys_sorted.p, offsets.p, offsets2.p, nq, keys_trunc.p);
        c.launches += 3;
        d_final_keys = keys_trunc.p;
        d_final_off = offsets2.p;
      }
    }
    write_offsets(d_final_off);
    PCLB_CUDA(cudaStreamSynchronize(st));
    const RadiusSinkBuffers o = sink(final_total);
    if (final_total > 0 && o.idx && o.d2) {
      if (is_device_ptr(o.idx) && is_device_ptr(o.d2)) {  // device-resident result: the unpack kernel writes it in place
        k_unpack_keys<<<grid_for(final_total, 256), 256, 0, st>>>(d_final_keys, final_total, o.idx, o.d2);
        ++c.launches;
      }
      else {
        DevBuf<int32_t> di;
        DevBuf<float> dd;
        di.alloc(final_total, st);
        dd.alloc(final_total, st);
        k_unpack_keys<<<grid_for(final_total, 256), 256, 0, st>>>(d_final_keys, final_total, di.p, dd.p);
        ++c.launches;
        deliver(o, di.p, dd.p, final_total);
      }
      PCLB_CUDA(cudaStreamSynchronize(st));
    }
    check_device_error(c);
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
  return guarded([&] {
    PCLB_REQUIRE(ctx, PCLB200_ERR_INVALID, "ctx == NULL");
    PCLB_CUDA(cudaStreamSynchronize(ctx->c.stream));
  });
}

int pclb200_launch_count(pclb200_ctx* ctx, uint64_t* out)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && out, PCLB200_ERR_INVALID, "NULL argument");
    *out = ctx->c.launches;
  });
}

int pclb200_stream(pclb200_ctx* ctx, void** out_stream)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && out_stream, PCLB200_ERR_INVALID, "NULL argument");
    *out_stream = (void*)ctx->c.stream;
  });
}

void pclb200_free(void* p) { free(p); }

int pclb200_host_register(pclb200_ctx* ctx, void* host_ptr, size_t bytes)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && host_ptr && bytes, PCLB200_ERR_INVALID, "NULL argument or empty buffer");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    PCLB_REQUIRE(!is_device_ptr(host_ptr), PCLB200_ERR_INVALID, "pclb200_host_register: not a host pointer");
    const cudaError_t e = cudaHostRegister(host_ptr, bytes, cudaHostRegisterPortable);
    if (e == cudaErrorHostMemoryAlreadyRegistered) {
      cudaGetLastError();
      throw Error(PCLB200_ERR_INVALID, "pclb200_host_register: the buffer (or a part of it) is already registered");
    }
    PCLB_CUDA(e);
  });
}

int pclb200_host_unregister(pclb200_ctx* ctx, void* host_ptr)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && host_ptr, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    // nothing may still be copying out of it: wait for this context's stream
    PCLB_CUDA(cudaStreamSynchronize(ctx->c.stream));
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
  return guarded([&] {
    PCLB_REQUIRE(ctx, PCLB200_ERR_INVALID, "ctx == NULL");
    ctx->c.profiling = enable != 0;
  });
}

int pclb200_profile_reset(pclb200_ctx* ctx)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx, PCLB200_ERR_INVALID, "ctx == NULL");
    PCLB_CUDA(cudaStreamSynchronize(ctx->c.stream));
    for (auto& e : ctx->c.prof) {
      cudaEventDestroy(e.a);
      cudaEventDestroy(e.b);
    }
    ctx->c.prof.clear();
  });
}

int pclb200_profile_get(pclb200_ctx* ctx, const char* name, double* total_ms, uint64_t* count)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && name && total_ms && count, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_CUDA(cudaStreamSynchronize(ctx->c.stream));
    double t = 0.0;
    uint64_t n = 0;
    for (auto& e : ctx->c.prof)
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
  return guarded([&] {
    PCLB_REQUIRE(ctx && out, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    Index* idx = nullptr;
    {
      ProfScope ps(ctx->c, "index_build");
      idx = build_index(ctx->c, pts, n, stride, subset, n_subset);
    }
    *out = new pclb200_index{idx};
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
  return guarded([&] {
    PCLB_REQUIRE(ctx && h && h->idx, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(k >= 0, PCLB200_ERR_INVALID, "k < 0");
    Ctx& c = ctx->c;
    std::lock_guard<std::recursive_mutex> lk(c.mu);
    PCLB_CUDA(cudaSetDevice(c.device));
    const Index& idx = *h->idx;
    const int keff = (int)std::min<size_t>((size_t)k, idx.n_valid);  // kdtree_flann.hpp:241-242
    if (k_eff)
      *k_eff = keff;
    if (k == 0 || nq == 0)
      return;
    PCLB_REQUIRE(queries && out_idx && out_d2, PCLB200_ERR_INVALID, "NULL argument");
    cudaStream_t st = c.stream;
    DevBuf<float4> dense;
    dense.alloc(nq, st);
    load_xyz_as_float4(c, queries, nq, stride, nullptr, 0, dense.p, st);
    QueryBatch qb;
    make_query_batch(c, idx, dense.p, nq, qb);
    DevBuf<int32_t> d_idx;
    DevBuf<float> d_d2;
    const bool dev_out = is_device_ptr(out_idx) && is_device_ptr(out_d2);
    int32_t* pi = out_idx;
    float* pd = out_d2;
    if (!dev_out) {
      d_idx.alloc(nq * (size_t)k, st);
      d_d2.alloc(nq * (size_t)k, st);
      pi = d_idx.p;
      pd = d_d2.p;
    }
    {
      ProfScope ps(c, "knn");
      launch_knn(c, idx, qb.q.p, nq, k, std::numeric_limits<float>::infinity(), pi, pd);
    }
    if (!dev_out) {
      PCLB_CUDA(cudaMemcpyAsync(out_idx, pi, nq * (size_t)k * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
      PCLB_CUDA(cudaMemcpyAsync(out_d2, pd, nq * (size_t)k * sizeof(float), cudaMemcpyDeviceToHost, st));
    }
    check_device_error(c);
  });
}

int pclb200_knn_stats(pclb200_ctx* ctx, const pclb200_index* h, const void* pts, size_t n, size_t stride,
                      const int32_t* indices, size_t n_idx, int k, float* out_mean, float* out_kth)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && h && h->idx && (out_mean || out_kth), PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(k > 0, PCLB200_ERR_INVALID, "k must be positive");
    Ctx& c = ctx->c;
    std::lock_guard<std::recursive_mutex> lk(c.mu);
    PCLB_CUDA(cudaSetDevice(c.device));
    cudaStream_t st = c.stream;
    const size_t nq = indices ? n_idx : n;
    if (!nq)
      return;
    DevBuf<float4> dense;
    dense.alloc(nq, st);
    load_xyz_as_float4(c, pts, n, stride, indices, n_idx, dense.p, st);
    QueryBatch qb;
    make_query_batch(c, *h->idx, dense.p, nq, qb);
    DevBuf<float> dm, dk;
    float* pm = out_mean;
    float* pk = out_kth;
    const bool m_dev = out_mean && is_device_ptr(out_mean), k_dev = out_kth && is_device_ptr(out_kth);
    if (out_mean && !m_dev) {
      dm.alloc(nq, st);
      pm = dm.p;
    }
    if (out_kth && !k_dev) {
      dk.alloc(nq, st);
      pk = dk.p;
    }
    {
      ProfScope ps(c, "knn_stats");
      launch_knn_stats(c, *h->idx, qb.q.p, nq, k, pm, pk);
    }
    if (out_mean && !m_dev)
      PCLB_CUDA(cudaMemcpyAsync(out_mean, pm, nq * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (out_kth && !k_dev)
      PCLB_CUDA(cudaMemcpyAsync(out_kth, pk, nq * sizeof(float), cudaMemcpyDeviceToHost, st));
    check_device_error(c);
  });
}

// ---- radius -------------------------------------------------------------------------------------------------------
int pclb200_radius(pclb200_ctx* ctx, const pclb200_index* h, const void* queries, size_t nq, size_t stride,
                   double radius, unsigned max_nn, int sorted, int64_t* out_offsets, int32_t** out_idx, float** out_d2)
{
  (void)sorted;
  return guarded([&] {
    PCLB_REQUIRE(ctx && h && h->idx && out_offsets && out_idx && out_d2, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(!is_device_ptr(out_offsets), PCLB200_ERR_INVALID, "pclb200_radius returns host arrays: out_offsets must be host memory");
    Ctx& c = ctx->c;
    std::lock_guard<std::recursive_mutex> lk(c.mu);
    PCLB_CUDA(cudaSetDevice(c.device));
    *out_idx = nullptr;
    *out_d2 = nullptr;
    out_offsets[0] = 0;
    if (nq == 0)
      return;
    radius_impl(c, *h->idx, queries, nq, stride, radius, max_nn, out_offsets, [&](unsigned long long total) {
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
  return guarded([&] {
    PCLB_REQUIRE(ctx && h && h->idx && out_offsets && total, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(capacity == 0 || (out_idx && out_d2), PCLB200_ERR_INVALID, "NULL output buffers with a non-zero capacity");
    Ctx& c = ctx->c;
    std::lock_guard<std::recursive_mutex> lk(c.mu);
    PCLB_CUDA(cudaSetDevice(c.device));
    *total = 0;
    if (nq == 0) {
      const int64_t zero = 0;
      PCLB_CUDA(cudaMemcpy(out_offsets, &zero, sizeof(zero), cudaMemcpyDefault));
      return;
    }
    radius_impl(c, *h->idx, queries, nq, stride, radius, max_nn, out_offsets, [&](unsigned long long n) {
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
  return guarded([&] {
    PCLB_REQUIRE(ctx && idx_tgt && idx_tgt->idx && n_out, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    *n_out = correspondences(ctx->c, *idx_tgt->idx, idx_src ? idx_src->idx : nullptr, src, n, stride, src_indices, n_idx,
                             is_dense, max_dist, out);
  });
}

int pclb200_correspondences_normals(pclb200_ctx* ctx, const pclb200_index* idx_tgt, int kind, const void* src, size_t n,
                                    size_t stride, const void* src_normals, size_t stride_sn, const void* tgt_normals,
                                    size_t stride_tn, const int32_t* src_indices, size_t n_idx, int k, double max_dist,
                                    pclb200_corr* out, size_t* n_out)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && idx_tgt && idx_tgt->idx && n_out, PCLB200_ERR_INVALID, "NULL argument");
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
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    *n_out = correspondences_by_normals(ctx->c, *idx_tgt->idx, kind, src, n, stride, src_normals, stride_sn, tgt_normals,
                                        stride_tn, src_indices, n_idx, k, max_dist, out);
    check_device_error(ctx->c);
  });
}

int pclb200_reject_surface_normal(pclb200_ctx* ctx, const pclb200_corr* in, size_t n, const void* src_normals, size_t n_src,
                                  size_t stride_sn, const void* tgt_normals, size_t n_tgt, size_t stride_tn,
                                  double threshold, pclb200_corr* out, size_t* n_out)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && n_out, PCLB200_ERR_INVALID, "NULL argument");
    *n_out = 0;
    if (n == 0)
      return;
    PCLB_REQUIRE(in && out && src_normals && tgt_normals && n_src && n_tgt, PCLB200_ERR_INVALID,
                 "NULL argument (correspondence_rejection_surface_normal.cpp:49-54: the normals must be set)");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    *n_out = reject_surface_normal(ctx->c, in, n, src_normals, n_src, stride_sn, tgt_normals, n_tgt, stride_tn, threshold,
                                   out);
  });
}

// ---- estimators ---------------------------------------------------------------------------------------------------------
int pclb200_estimate_svd(pclb200_ctx* ctx, const void* src, size_t stride_s, const void* tgt, size_t stride_t,
                         const pclb200_corr* corr, size_t n, int scalar_is_double, double T_out[16])
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && T_out, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    estimate_pairs(ctx->c, PCLB200_EST_SVD, src, stride_s, tgt, nullptr, stride_t, corr, n, scalar_is_double, T_out);
  });
}

int pclb200_estimate_svd_correlation(pclb200_ctx* ctx, const void* src, size_t stride_s, const void* tgt, size_t stride_t,
                                     const pclb200_corr* corr, size_t n, int scalar_is_double, double T_out[16])
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && T_out, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    estimate_pairs(ctx->c, PCLB200_EST_SVD, src, stride_s, tgt, nullptr, stride_t, corr, n, scalar_is_double, T_out, nullptr,
                   1, 1);
  });
}

int pclb200_estimate_point_to_plane_lls(pclb200_ctx* ctx, const void* src, size_t stride_s, const void* tgt,
                                        const void* tgt_normals, size_t stride_t, const pclb200_corr* corr, size_t n,
                                        int scalar_is_double, double T_out[16])
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && T_out, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    estimate_pairs(ctx->c, PCLB200_EST_POINT_TO_PLANE_LLS, src, stride_s, tgt, tgt_normals, stride_t, corr, n,
                   scalar_is_double, T_out);
  });
}

int pclb200_estimate_symmetric_point_to_plane_lls(pclb200_ctx* ctx, const void* src, const void* src_normals,
                                                  size_t stride_s, const void* tgt, const void* tgt_normals,
                                                  size_t stride_t, const pclb200_corr* corr, size_t n,
                                                  int enforce_same_direction_normals, int scalar_is_double,
                                                  double T_out[16])
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && T_out, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    estimate_pairs(ctx->c, PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS, src, stride_s, tgt, tgt_normals, stride_t, corr, n,
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
  return guarded([&] {
    PCLB_REQUIRE(ctx && out, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    pclb200_icp_params P;
    if (params)
      P = *params;
    else
      pclb200_icp_default_params(&P);
    *out = new pclb200_icp{icp_create(ctx->c, P), ctx, ctx->c.device};
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
  return guarded([&] {
    PCLB_REQUIRE(icp && params, PCLB200_ERR_INVALID, "NULL argument");
    icp_set_params(*icp->s, *params);
  });
}

int pclb200_icp_set_rejectors(pclb200_icp* icp, const pclb200_rejector* list, int n)
{
  return guarded([&] {
    PCLB_REQUIRE(icp && (n <= 0 || list), PCLB200_ERR_INVALID, "NULL argument");
    icp_set_rejectors(*icp->s, list, n);
  });
}

int pclb200_reject(pclb200_ctx* ctx, const pclb200_rejector* rejector, const pclb200_corr* in, size_t n,
                   pclb200_corr* out, size_t* n_out, double* median_out)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && rejector && n_out && (n == 0 || (in && out)), PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(rejector->kind >= PCLB200_REJ_DISTANCE && rejector->kind <= PCLB200_REJ_TRIMMED, PCLB200_ERR_INVALID,
                 "unknown rejector kind");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    *n_out = reject_standalone(ctx->c, *rejector, in, n, out, median_out);
  });
}

int pclb200_icp_set_target(pclb200_icp* icp, const pclb200_index* idx_tgt, const void* tgt_normals, size_t stride_n)
{
  return guarded([&] {
    PCLB_REQUIRE(icp && idx_tgt && idx_tgt->idx, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(icp->ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(icp->ctx->c.device));
    icp_set_target(*icp->s, idx_tgt->idx, tgt_normals, stride_n);
  });
}

int pclb200_icp_set_source(pclb200_icp* icp, const void* src, size_t n, size_t stride, const void* src_normals,
                           size_t stride_n, const int32_t* src_indices, size_t n_idx, const double guess[16])
{
  return guarded([&] {
    PCLB_REQUIRE(icp, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(icp->ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(icp->ctx->c.device));
    icp_set_source(*icp->s, src, n, stride, src_normals, stride_n, src_indices, n_idx, guess);
  });
}

int pclb200_icp_iterate(pclb200_icp* icp, int max_steps, pclb200_icp_stats* stats)
{
  return guarded([&] {
    PCLB_REQUIRE(icp, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(icp->ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(icp->ctx->c.device));
    icp_iterate(*icp->s, max_steps, stats);
  });
}

int pclb200_icp_get_cloud(pclb200_icp* icp, void* out_pts, size_t stride_out, void* out_normals, size_t stride_n)
{
  return guarded([&] {
    PCLB_REQUIRE(icp && out_pts, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(icp->ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(icp->ctx->c.device));
    icp_get_cloud(*icp->s, out_pts, stride_out, out_normals, stride_n);
  });
}

int pclb200_icp_get_correspondences(pclb200_icp* icp, pclb200_corr* out, size_t* n_out)
{
  return guarded([&] {
    PCLB_REQUIRE(icp && out && n_out, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(icp->ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(icp->device));
    *n_out = icp_get_correspondences(*icp->s, out);
  });
}

int pclb200_icp_align(pclb200_ctx* ctx, const pclb200_icp_params* params, const void* src, size_t n, size_t stride,
                      const void* src_normals, size_t stride_sn, const int32_t* src_indices, size_t n_idx,
                      const pclb200_index* idx_tgt, const void* tgt_normals, size_t stride_tn, const double guess[16],
                      void* out_cloud, size_t stride_out, pclb200_icp_stats* stats)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && params && idx_tgt && idx_tgt->idx, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    struct Guard {
      Icp* s;
      ~Guard() { icp_destroy(s); }
    } g{icp_create(ctx->c, *params)};
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
  return guarded([&] {
    PCLB_REQUIRE(ctx && idx_tgt && idx_tgt->idx && T && score, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    *score = fitness_score(ctx->c, *idx_tgt->idx, src, n, stride, src_indices, n_idx, T, scalar_is_double, max_range);
  });
}

int pclb200_gicp_covariances(pclb200_ctx* ctx, const pclb200_index* idx, const void* pts, size_t n, size_t stride, int k,
                             double gicp_epsilon, double* out_cov)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && idx && idx->idx && pts && out_cov, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    ProfScope ps(ctx->c, "gicp_covariances");
    gicp_covariances(ctx->c, *idx->idx, pts, n, stride, k, gicp_epsilon, out_cov);
  });
}

int pclb200_validate_transformation(pclb200_ctx* ctx, const pclb200_index* idx_tgt, const void* src, size_t n,
                                    size_t stride, const double T[16], int scalar_is_double, double max_range,
                                    double* score)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && idx_tgt && idx_tgt->idx && T && score, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    // transformation_validation_euclidean.hpp:62-75: T(0,0)*x + T(0,1)*y + T(0,2)*z + T(0,3) in Scalar, cast to float
    *score = fitness_score(ctx->c, *idx_tgt->idx, src, n, stride, nullptr, 0, T, scalar_is_double, max_range,
                           scalar_is_double ? 3 : 0);
  });
}

int pclb200_inliers(pclb200_ctx* ctx, const pclb200_index* idx_tgt, const void* src, size_t n, size_t stride,
                    const double T[16], float inlier_threshold, pclb200_corr* out, size_t* n_out)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && idx_tgt && idx_tgt->idx && T && out && n_out, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    // sample_consensus_prerejective.hpp:318-338: transformPointCloud (float), then nn_dists[0] < max_range (STRICT, float)
    const float max_range = inlier_threshold * inlier_threshold;
    const float gate = std::nextafter(max_range, -std::numeric_limits<float>::infinity());  // d2 <= gate  <=>  d2 < max_range
    double Tf[16];
    for (int i = 0; i < 16; ++i)
      Tf[i] = (double)(float)T[i];
    *n_out = max_range > 0.f ? correspondences(ctx->c, *idx_tgt->idx, nullptr, src, n, stride, nullptr, 0, 1, 0.0, out, Tf, 1, &gate)
                             : 0;
  });
}

// ---- normals ----------------------------------------------------------------------------------------------------------------
int pclb200_normals_knn(pclb200_ctx* ctx, const pclb200_index* h, const void* pts, size_t n, size_t stride,
                        const int32_t* indices, size_t n_idx, int is_dense, int k, const float viewpoint[3], float* out,
                        int* is_dense_out)
{
  (void)is_dense;
  return guarded([&] {
    PCLB_REQUIRE(ctx && h && h->idx && out && viewpoint, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(k > 0, PCLB200_ERR_INVALID, "k must be positive (feature.hpp:135-176)");
    Ctx& c = ctx->c;
    std::lock_guard<std::recursive_mutex> lk(c.mu);
    PCLB_CUDA(cudaSetDevice(c.device));
    cudaStream_t st = c.stream;
    const size_t nq = indices ? n_idx : n;
    if (is_dense_out)
      *is_dense_out = 1;
    if (!nq)
      return;
    DevBuf<float4> dense;
    dense.alloc(nq, st);
    load_xyz_as_float4(c, pts, n, stride, indices, n_idx, dense.p, st);
    QueryBatch qb;
    make_query_batch(c, *h->idx, dense.p, nq, qb);
    DevBuf<float4> d_out;
    DevBuf<int> d_flag;
    d_flag.alloc(1, st);
    PCLB_CUDA(cudaMemsetAsync(d_flag.p, 0, sizeof(int), st));
    const bool dev_out = is_device_ptr(out);
    float4* po = reinterpret_cast<float4*>(out);
    if (!dev_out) {
      d_out.alloc(nq, st);
      po = d_out.p;
    }
    {
      ProfScope ps(c, "normals");
      launch_normals(c, *h->idx, qb.q.p, nq, k, viewpoint, po, d_flag.p);
    }
    int flag = 0;
    PCLB_CUDA(cudaMemcpyAsync(&flag, d_flag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    if (!dev_out)
      PCLB_CUDA(cudaMemcpyAsync(out, po, nq * sizeof(float4), cudaMemcpyDeviceToHost, st));
    check_device_error(c);
    if (is_dense_out)
      *is_dense_out = flag ? 0 : 1;
  });
}

int pclb200_normals_radius(pclb200_ctx* ctx, const pclb200_index* h, const void* pts, size_t n, size_t stride,
                           const int32_t* indices, size_t n_idx, int is_dense, double radius, const float viewpoint[3],
                           float* out, int* is_dense_out)
{
  (void)is_dense;
  return guarded([&] {
    PCLB_REQUIRE(ctx && h && h->idx && out && viewpoint, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(radius > 0.0, PCLB200_ERR_INVALID, "radius must be positive (feature.hpp:135-176)");
    Ctx& c = ctx->c;
    std::lock_guard<std::recursive_mutex> lk(c.mu);
    PCLB_CUDA(cudaSetDevice(c.device));
    cudaStream_t st = c.stream;
    const size_t nq = indices ? n_idx : n;
    if (is_dense_out)
      *is_dense_out = 1;
    if (!nq)
      return;
    DevBuf<float4> dense;
    dense.alloc(nq, st);
    load_xyz_as_float4(c, pts, n, stride, indices, n_idx, dense.p, st);
    QueryBatch qb;
    make_query_batch(c, *h->idx, dense.p, nq, qb);
    DevBuf<float4> d_out;
    DevBuf<int> d_flag;
    d_flag.alloc(1, st);
    PCLB_CUDA(cudaMemsetAsync(d_flag.p, 0, sizeof(int), st));
    const bool dev_out = is_device_ptr(out);
    float4* po = reinterpret_cast<float4*>(out);
    if (!dev_out) {
      d_out.alloc(nq, st);
      po = d_out.p;
    }
    {
      ProfScope ps(c, "normals");
      launch_normals_radius(c, *h->idx, qb.q.p, nq, (float)(radius * radius), viewpoint, po, d_flag.p);
    }
    int flag = 0;
    PCLB_CUDA(cudaMemcpyAsync(&flag, d_flag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    if (!dev_out)
      PCLB_CUDA(cudaMemcpyAsync(out, po, nq * sizeof(float4), cudaMemcpyDeviceToHost, st));
    check_device_error(c);
    if (is_dense_out)
      *is_dense_out = flag ? 0 : 1;
  });
}

// ---- Euclidean clustering --------------------------------------------------------------------------------------------------
int pclb200_cluster_labels(pclb200_ctx* ctx, const pclb200_index* h, double tolerance, int32_t* out_labels, size_t n_labels)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && h && h->idx && out_labels, PCLB200_ERR_INVALID, "NULL argument");
    PCLB_REQUIRE(tolerance >= 0.0, PCLB200_ERR_INVALID, "negative cluster tolerance");
    Ctx& c = ctx->c;
    std::lock_guard<std::recursive_mutex> lk(c.mu);
    PCLB_CUDA(cudaSetDevice(c.device));
    const Index& idx = *h->idx;
    PCLB_REQUIRE(n_labels == idx.n_cloud, PCLB200_ERR_INVALID,
                 "out_labels must hold one entry per point of the cloud the index was built from");
    cudaStream_t st = c.stream;
    DevBuf<int32_t> d;
    int32_t* pl = out_labels;
    const bool dev_out = is_device_ptr(out_labels);
    if (!dev_out) {
      d.alloc(n_labels, st);
      pl = d.p;
    }
    cluster_labels(c, idx, tolerance, pl);
    if (!dev_out)
      PCLB_CUDA(cudaMemcpyAsync(out_labels, pl, n_labels * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    check_device_error(c);
  });
}

// ---- voxel grid ---------------------------------------------------------------------------------------------------------------
int pclb200_voxelgrid(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx,
                      int is_dense, const float leaf[3], unsigned min_points_per_voxel, float* out_xyz1, size_t* n_out)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && leaf && out_xyz1 && n_out, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    ProfScope ps(ctx->c, "voxelgrid");
    *n_out = voxelgrid(ctx->c, pts, n, stride, indices, n_idx, is_dense, leaf, min_points_per_voxel, out_xyz1, nullptr, 0,
                       nullptr);
  });
}

int pclb200_voxelgrid_tile(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const float grid_bounds[6],
                           const float leaf[3], unsigned min_points_per_voxel, float* out_xyz1, size_t* n_out)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && leaf && out_xyz1 && n_out && grid_bounds, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    ProfScope ps(ctx->c, "voxelgrid");
    *n_out = voxelgrid(ctx->c, pts, n, stride, nullptr, 0, 0, leaf, min_points_per_voxel, out_xyz1, nullptr, 0, nullptr,
                       grid_bounds);
  });
}

int pclb200_voxelgrid_normals(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const void* normals,
                              size_t stride_n, const int32_t* indices, size_t n_idx, int is_dense, const float leaf[3],
                              unsigned min_points_per_voxel, float* out_xyz1, float* out_normal_curv, size_t* n_out)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && leaf && out_xyz1 && n_out && normals && out_normal_curv, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    ProfScope ps(ctx->c, "voxelgrid");
    *n_out = voxelgrid(ctx->c, pts, n, stride, indices, n_idx, is_dense, leaf, min_points_per_voxel, out_xyz1, normals,
                       stride_n, out_normal_curv);
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
  return guarded([&] {
    PCLB_REQUIRE(ctx && (nranks == 1 || unique_id), PCLB200_ERR_INVALID, "NULL argument");
    comm_init(ctx->c, rank, nranks, unique_id);
  });
}

int pclb200_comm_set_mode(pclb200_ctx* ctx, int mode)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    comm_set_mode(ctx->c, mode);
  });
}

int pclb200_comm_export(pclb200_ctx* ctx, void* out_handle_64_bytes)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && out_handle_64_bytes, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    comm_export(ctx->c, out_handle_64_bytes);
  });
}

int pclb200_comm_import(pclb200_ctx* ctx, int rank, int nranks, const void* handles)
{
  return guarded([&] {
    PCLB_REQUIRE(ctx && handles, PCLB200_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(ctx->c.mu);
    PCLB_CUDA(cudaSetDevice(ctx->c.device));
    comm_import(ctx->c, rank, nranks, handles);
  });
}

}  // extern "C"
