// pclb200_on_oracle.cpp — TEST DOUBLE.  The entry points of include/pclb200.h that the header-only facade
// (pcl_b200/pcl_compat/pcl/**) calls, answered by the CPU oracle (oracle/libpcl_oracle.so), so that the facade's HOST logic —
// argument marshalling, state bookkeeping, the reference's class behaviour around each call — can be exercised by
// `pytest -m "not gpu"` on a machine without a GPU.  It is built by tests/test_facade_on_oracle.py into a temporary
// directory under another file name, is never installed next to pcl_b200/libpclb200.so, and is not a fallback of the
// product: libpclb200.so has no CPU path and fails loudly without a device (tests/test_capi_symbols.py).
//
// What it mirrors of the real library: argument meaning, output layout, status codes for the cases the facade relies on.
// What it does not: device pointers, streams, profiling, the multi-GPU communicator (those entry points return
// PCLB200_ERR_INVALID with a message that names this file).
#include <pclb200.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <set>
#include <string>
#include <vector>

// ---- the oracle's C interface (oracle/pcl_oracle.cpp) -----------------------------------------------------------------
extern "C" {
struct orc_corr { int32_t index_query, index_match; float distance; };
struct orc_rejector { int32_t kind, min_correspondences; double p; };
struct orc_icp_params {
  int32_t max_iterations, use_reciprocal, estimator, scalar_is_double, with_normals_transform, source_has_normals, is_dense, nthreads;
  double max_correspondence_distance, transformation_epsilon, transformation_rotation_epsilon, euclidean_fitness_epsilon;
  int32_t correspondence_kind, correspondence_k;
};
struct orc_icp_ext {
  int32_t failure_after_max_iter, max_iterations_similar_transforms, svd_no_umeyama, enforce_same_direction_normals;
  double mse_threshold_absolute;
};
struct orc_icp_result {
  double final_transformation[16], last_transformation[16];
  int32_t converged, state, iterations, n_correspondences;
  double mse;
  long long total_correspondences;
};
void* orc_index_build(const float* pts, size_t n, size_t stride, const int32_t* subset, size_t n_subset);
void orc_index_free(void* h);
size_t orc_index_size(void* h);
int orc_knn(void* h, const float* q, size_t nq, size_t qstride, int k, int32_t* out_idx, float* out_d2, int nthreads);
int orc_radius(void* h, const float* q, size_t nq, size_t qstride, double radius, unsigned max_nn, int64_t* offsets, int32_t* out_idx,
               float* out_d2, int nthreads);
size_t orc_correspondences(void* h_tgt, const float* src, size_t n_src, size_t sstride, const int32_t* indices, size_t n_idx, int is_dense,
                           double max_distance, orc_corr* out, int nthreads);
size_t orc_correspondences_reciprocal(void* h_tgt, void* h_src, const float* src, size_t n_src, size_t sstride, const float* tgt,
                                      size_t tstride, const int32_t* indices, size_t n_idx, int is_dense, double max_distance, orc_corr* out,
                                      int nthreads);
size_t orc_correspondences_normals(void* h_tgt, int kind, const float* src, size_t n_src, size_t sstride, const float* sn, size_t snstride,
                                   const float* tgt, size_t tstride, const float* tn, size_t tnstride, const int32_t* indices, size_t n_idx,
                                   int k, double max_distance, orc_corr* out, int nthreads);
void orc_estimate_svd(const float* src, size_t sstride, const float* tgt, size_t tstride, const orc_corr* corr, size_t n, int scalar_is_double,
                      double* T_out);
void orc_estimate_svd_correlation(const float* src, size_t sstride, const float* tgt, size_t tstride, const orc_corr* corr, size_t n,
                                  int scalar_is_double, double* T_out);
int orc_estimate_point_to_plane_lls(const float* src, size_t sstride, const float* tgt, const float* tgt_normals, size_t tstride,
                                    const orc_corr* corr, size_t n, int scalar_is_double, double* T_out);
int orc_estimate_symmetric_lls(const float* src, const float* src_normals, size_t sstride, const float* tgt, const float* tgt_normals,
                               size_t tstride, const orc_corr* corr, size_t n, int enforce_same_direction, int scalar_is_double, double* T_out);
void orc_transform(float* pts, size_t n, size_t stride, int normal_off, const double* T, int scalar_is_double, int mode);
size_t orc_reject(const orc_rejector* r, const orc_corr* in, size_t n, orc_corr* out, double* median_out);
size_t orc_reject_surface_normal(const orc_corr* in, size_t n, const float* sn, size_t snstride, const float* tn, size_t tnstride,
                                 double threshold, orc_corr* out);
void orc_icp_align_full(const orc_icp_params* P, const orc_icp_ext* X, const orc_rejector* rej, int n_rej, void* h_tgt, const float* src,
                        size_t n_s, size_t sstride, const int32_t* indices, size_t n_idx, const float* tgt, size_t n_t, size_t tstride,
                        const double* guess, orc_icp_result* R, float* out_cloud, orc_corr* last_corr, size_t* n_last_corr);
void orc_icp_align_carry(const orc_icp_params* P, const orc_icp_ext* X, const orc_rejector* rej, int n_rej, void* h_tgt, const float* src,
                         size_t n_s, size_t sstride, const int32_t* indices, size_t n_idx, const float* tgt, size_t n_t, size_t tstride,
                         const double* guess, orc_icp_result* R, float* out_cloud, orc_corr* last_corr, size_t* n_last_corr,
                         double* prev_mse);
double orc_fitness_score(void* h_tgt, const float* src, size_t n_s, size_t sstride, const int32_t* indices, size_t n_idx, int is_dense,
                         const double* final_T, int scalar_is_double, double max_range, int nthreads);
long long orc_voxelgrid(const float* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int is_dense, const float leaf[3],
                        unsigned min_pts, float* out);
long long orc_voxelgrid_normals(const float* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int is_dense,
                                const float leaf[3], unsigned min_pts, float* out, long normal_off, float* out_nc);
int orc_normals_knn(void* h, const float* cloud, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int is_dense, int k,
                    const float vp[3], float* out, int nthreads);
int orc_normals_radius(void* h, const float* cloud, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int is_dense, double radius,
                       const float vp[3], float* out, int nthreads);
void orc_cluster_labels(void* h, size_t n_cloud, double tolerance, int32_t* out_labels);
void orc_knn_stats(void* h, const float* cloud, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int k, float* out_mean,
                   float* out_kth, int nthreads);
void orc_gicp_covariances(void* h, const float* cloud, size_t n, size_t stride, int k, double gicp_epsilon, double* out, int nthreads);
}

static_assert(sizeof(orc_corr) == sizeof(pclb200_corr) && sizeof(orc_rejector) == sizeof(pclb200_rejector), "record layouts");

namespace {
thread_local std::string g_err;
int fail(int code, const char* what)
{
  g_err = what;
  return code;
}
constexpr int kThreads = 4;
const orc_corr* oc(const pclb200_corr* c) { return reinterpret_cast<const orc_corr*>(c); }
orc_corr* oc(pclb200_corr* c) { return reinterpret_cast<orc_corr*>(c); }

// records of any stride -> n x `w` floats: xyz1 (w = 4) or xyz1 + normal + 0 (w = 8)
std::vector<float> pack(const void* pts, size_t n, size_t stride, const void* normals, size_t stride_n, int w)
{
  std::vector<float> v(n * (size_t)w, 0.f);
  for (size_t i = 0; i < n; ++i) {
    const float* p = reinterpret_cast<const float*>(static_cast<const unsigned char*>(pts) + i * stride);
    float* r = &v[i * (size_t)w];
    r[0] = p[0]; r[1] = p[1]; r[2] = p[2]; r[3] = 1.f;
    if (w == 8 && normals) {
      const float* q = reinterpret_cast<const float*>(static_cast<const unsigned char*>(normals) + i * stride_n);
      r[4] = q[0]; r[5] = q[1]; r[6] = q[2];
    }
  }
  return v;
}
// transformation_validation_euclidean.hpp:62-75: T(r,0)*x + T(r,1)*y + T(r,2)*z + T(r,3), left to right in Scalar, cast to float
template <typename S> void moved_by(const std::vector<float>& in, size_t n, const double T[16], std::vector<float>& out)
{
  out = in;
  for (size_t i = 0; i < n; ++i)
    for (int r = 0; r < 3; ++r) {
      volatile S a = static_cast<S>(T[4 * r]) * static_cast<S>(in[4 * i]);
      volatile S b = static_cast<S>(T[4 * r + 1]) * static_cast<S>(in[4 * i + 1]);
      volatile S c = static_cast<S>(T[4 * r + 2]) * static_cast<S>(in[4 * i + 2]);
      volatile S s1 = a + b;
      volatile S s2 = s1 + c;
      volatile S s3 = s2 + static_cast<S>(T[4 * r + 3]);
      out[4 * i + r] = static_cast<float>(s3);
    }
}
}  // namespace

struct pclb200_ctx {
  std::set<const void*> registered;
};
struct pclb200_index {
  void* tree = nullptr;
  std::vector<float> cloud;  // the WHOLE cloud the index was built from, n x 4
  size_t n = 0;
};
struct pclb200_icp {
  pclb200_icp_params P;
  std::vector<orc_rejector> chain;
  const pclb200_index* tgt = nullptr;
  std::vector<float> tgt_rec;  // n_t x 8
  bool tgt_normals = false;
  std::vector<float> src_rec;  // n x 8
  size_t n_src = 0;
  bool src_normals = false;
  std::vector<int32_t> indices;
  bool has_indices = false;
  double guess[16];
  bool has_guess = false;
  // the untruncated run (made at the first iterate after set_source) and the state after `done` iterations
  bool have_full = false;
  orc_icp_result full{}, cur{};
  std::vector<float> full_cloud, cur_cloud;
  std::vector<orc_corr> full_corr, cur_corr;
  int done = 0;
  bool finished = false;
  // the criteria's previous MSE, which outlives an align (icp.h:155): where the last iterate left it, and its value
  // when set_source started the current align (every replay of that align starts from it)
  double prev_mse = std::numeric_limits<double>::max(), prev_mse_at_source = std::numeric_limits<double>::max();
  double full_prev_mse = 0;
};

extern "C" {

int pclb200_version(void) { return PCLB200_VERSION; }
const char* pclb200_last_error(void) { return g_err.c_str(); }

int pclb200_create(int, pclb200_ctx** out)
{
  if (!out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  *out = new pclb200_ctx();
  return PCLB200_OK;
}
int pclb200_destroy(pclb200_ctx* ctx) { delete ctx; return PCLB200_OK; }
int pclb200_synchronize(pclb200_ctx*) { return PCLB200_OK; }
int pclb200_launch_count(pclb200_ctx*, uint64_t* out) { if (out) *out = 0; return PCLB200_OK; }
int pclb200_stream(pclb200_ctx*, void**) { return fail(PCLB200_ERR_INVALID, "tests/host/pclb200_on_oracle.cpp: no stream"); }
void pclb200_free(void* p) { std::free(p); }
int pclb200_host_register(pclb200_ctx* ctx, void* p, size_t bytes)
{
  if (!ctx || !p || bytes == 0) return fail(PCLB200_ERR_INVALID, "NULL argument");
  if (!ctx->registered.insert(p).second) return fail(PCLB200_ERR_INVALID, "host_register: already registered");
  return PCLB200_OK;
}
int pclb200_host_unregister(pclb200_ctx* ctx, void* p)
{
  if (!ctx || !p) return fail(PCLB200_ERR_INVALID, "NULL argument");
  if (ctx->registered.erase(p) == 0) return fail(PCLB200_ERR_INVALID, "host_unregister: not registered");
  return PCLB200_OK;
}
int pclb200_profile_enable(pclb200_ctx*, int) { return PCLB200_OK; }
int pclb200_profile_get(pclb200_ctx*, const char*, double* ms, uint64_t* cnt) { if (ms) *ms = 0; if (cnt) *cnt = 0; return PCLB200_OK; }
int pclb200_profile_reset(pclb200_ctx*) { return PCLB200_OK; }

int pclb200_index_build(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const int32_t* subset, size_t n_subset, pclb200_index** out)
{
  if (!ctx || !out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  *out = nullptr;
  if (stride < 12 || stride % 4) return fail(PCLB200_ERR_INVALID, "stride");
  if (n == 0 || !pts || (subset && n_subset == 0)) return fail(PCLB200_ERR_EMPTY, "empty cloud");
  auto* h = new pclb200_index();
  h->cloud = pack(pts, n, stride, nullptr, 0, 4);
  h->n = n;
  h->tree = orc_index_build(h->cloud.data(), n, 4, subset, subset ? n_subset : 0);
  if (orc_index_size(h->tree) == 0) {
    orc_index_free(h->tree);
    delete h;
    return fail(PCLB200_ERR_EMPTY, "no finite point");
  }
  *out = h;
  return PCLB200_OK;
}
int pclb200_index_destroy(pclb200_index* h)
{
  if (h) { orc_index_free(h->tree); delete h; }
  return PCLB200_OK;
}
int pclb200_index_size(const pclb200_index* h, size_t* n_valid)
{
  if (!h || !n_valid) return fail(PCLB200_ERR_INVALID, "NULL argument");
  *n_valid = orc_index_size(h->tree);
  return PCLB200_OK;
}
int pclb200_index_stats(const pclb200_index*, uint64_t out[4]) { for (int i = 0; i < 4; ++i) out[i] = 0; return PCLB200_OK; }

int pclb200_knn(pclb200_ctx* ctx, const pclb200_index* h, const void* q, size_t nq, size_t stride, int k, int32_t* out_idx, float* out_d2, int* k_eff)
{
  if (!ctx || !h) return fail(PCLB200_ERR_INVALID, "NULL argument");
  if (k < 0) return fail(PCLB200_ERR_INVALID, "k < 0");
  if (k_eff) *k_eff = (int)std::min<size_t>((size_t)k, orc_index_size(h->tree));
  if (k == 0 || nq == 0) return PCLB200_OK;
  if (!q || !out_idx || !out_d2) return fail(PCLB200_ERR_INVALID, "NULL argument");
  const std::vector<float> Q = pack(q, nq, stride, nullptr, 0, 4);
  orc_knn(h->tree, Q.data(), nq, 4, k, out_idx, out_d2, kThreads);
  return PCLB200_OK;
}

int pclb200_knn_stats(pclb200_ctx* ctx, const pclb200_index* h, const void* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int k,
                      float* out_mean, float* out_kth)
{
  if (!ctx || !h || !pts) return fail(PCLB200_ERR_INVALID, "NULL argument");
  const std::vector<float> C = pack(pts, n, stride, nullptr, 0, 4);
  const size_t cnt = indices ? n_idx : n;
  std::vector<float> mean(cnt ? cnt : 1), kth(cnt ? cnt : 1);
  orc_knn_stats(h->tree, C.data(), n, 4, indices, indices ? n_idx : 0, k, mean.data(), kth.data(), kThreads);
  if (out_mean) std::copy(mean.begin(), mean.begin() + cnt, out_mean);
  if (out_kth) std::copy(kth.begin(), kth.begin() + cnt, out_kth);
  return PCLB200_OK;
}

int pclb200_radius_into(pclb200_ctx* ctx, const pclb200_index* h, const void* q, size_t nq, size_t stride, double radius, unsigned max_nn,
                        int64_t* out_offsets, int32_t* out_idx, float* out_d2, size_t capacity, size_t* total)
{
  if (!ctx || !h || !out_offsets) return fail(PCLB200_ERR_INVALID, "NULL argument");
  if (!(radius >= 0)) return fail(PCLB200_ERR_INVALID, "radius < 0");
  out_offsets[0] = 0;
  if (total) *total = 0;
  if (nq == 0) return PCLB200_OK;
  const std::vector<float> Q = pack(q, nq, stride, nullptr, 0, 4);
  orc_radius(h->tree, Q.data(), nq, 4, radius, max_nn, out_offsets, nullptr, nullptr, kThreads);
  const size_t tot = (size_t)out_offsets[nq];
  if (total) *total = tot;
  if (tot > capacity || tot == 0) return PCLB200_OK;
  orc_radius(h->tree, Q.data(), nq, 4, radius, max_nn, out_offsets, out_idx, out_d2, kThreads);
  return PCLB200_OK;
}
int pclb200_radius(pclb200_ctx* ctx, const pclb200_index* h, const void* q, size_t nq, size_t stride, double radius, unsigned max_nn, int,
                   int64_t* out_offsets, int32_t** out_idx, float** out_d2)
{
  if (!out_idx || !out_d2) return fail(PCLB200_ERR_INVALID, "NULL argument");
  *out_idx = nullptr;
  *out_d2 = nullptr;
  size_t tot = 0;
  int rc = pclb200_radius_into(ctx, h, q, nq, stride, radius, max_nn, out_offsets, nullptr, nullptr, 0, &tot);
  if (rc != PCLB200_OK) return rc;
  *out_idx = static_cast<int32_t*>(std::malloc(std::max<size_t>(tot, 1) * sizeof(int32_t)));
  *out_d2 = static_cast<float*>(std::malloc(std::max<size_t>(tot, 1) * sizeof(float)));
  return pclb200_radius_into(ctx, h, q, nq, stride, radius, max_nn, out_offsets, *out_idx, *out_d2, tot, &tot);
}

int pclb200_correspondences(pclb200_ctx* ctx, const pclb200_index* idx_tgt, const pclb200_index* idx_src, const void* src, size_t n, size_t stride,
                            const int32_t* src_indices, size_t n_idx, int is_dense, double max_dist, pclb200_corr* out, size_t* n_out)
{
  if (!ctx || !idx_tgt || !out || !n_out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  *n_out = 0;
  if (n == 0) return PCLB200_OK;
  const std::vector<float> S = pack(src, n, stride, nullptr, 0, 4);
  *n_out = idx_src ? orc_correspondences_reciprocal(idx_tgt->tree, idx_src->tree, S.data(), n, 4, idx_tgt->cloud.data(), 4, src_indices,
                                                    src_indices ? n_idx : 0, is_dense, max_dist, oc(out), kThreads)
                   : orc_correspondences(idx_tgt->tree, S.data(), n, 4, src_indices, src_indices ? n_idx : 0, is_dense, max_dist, oc(out), kThreads);
  return PCLB200_OK;
}

int pclb200_correspondences_normals(pclb200_ctx* ctx, const pclb200_index* idx_tgt, int kind, const void* src, size_t n, size_t stride,
                                    const void* src_normals, size_t stride_sn, const void* tgt_normals, size_t stride_tn, const int32_t* src_indices,
                                    size_t n_idx, int k, double max_dist, pclb200_corr* out, size_t* n_out)
{
  if (!ctx || !idx_tgt || !src || !src_normals || !out || !n_out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  if (kind != PCLB200_CORR_NORMAL_SHOOTING && kind != PCLB200_CORR_BACK_PROJECTION) return fail(PCLB200_ERR_INVALID, "kind");
  if (kind == PCLB200_CORR_BACK_PROJECTION && !tgt_normals) return fail(PCLB200_ERR_INVALID, "back projection needs target normals");
  const std::vector<float> S = pack(src, n, stride, src_normals, stride_sn, 8);
  std::vector<float> T(idx_tgt->n * 8, 0.f);
  for (size_t i = 0; i < idx_tgt->n; ++i) {
    std::memcpy(&T[8 * i], &idx_tgt->cloud[4 * i], 16);
    if (tgt_normals) std::memcpy(&T[8 * i + 4], static_cast<const unsigned char*>(tgt_normals) + i * stride_tn, 12);
  }
  *n_out = orc_correspondences_normals(idx_tgt->tree, kind, S.data(), n, 8, S.data() + 4, 8, T.data(), 8, T.data() + 4, 8, src_indices,
                                       src_indices ? n_idx : 0, k, max_dist, oc(out), kThreads);
  return PCLB200_OK;
}

int pclb200_reject(pclb200_ctx* ctx, const pclb200_rejector* r, const pclb200_corr* in, size_t n, pclb200_corr* out, size_t* n_out, double* median_out)
{
  if (!ctx || !r || !out || !n_out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  if (r->kind < PCLB200_REJ_DISTANCE || r->kind > PCLB200_REJ_TRIMMED) return fail(PCLB200_ERR_INVALID, "rejector kind");
  *n_out = 0;
  if (median_out) *median_out = 0;
  if (n == 0) return PCLB200_OK;
  std::vector<orc_corr> tmp(n);
  double med = 0;
  const size_t m = orc_reject(reinterpret_cast<const orc_rejector*>(r), oc(in), n, tmp.data(), &med);
  std::copy(tmp.begin(), tmp.begin() + m, oc(out));
  *n_out = m;
  if (median_out) *median_out = med;
  return PCLB200_OK;
}
int pclb200_reject_surface_normal(pclb200_ctx* ctx, const pclb200_corr* in, size_t n, const void* src_normals, size_t, size_t stride_sn,
                                  const void* tgt_normals, size_t, size_t stride_tn, double threshold, pclb200_corr* out, size_t* n_out)
{
  if (!ctx || !src_normals || !tgt_normals || !out || !n_out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  std::vector<orc_corr> tmp(n ? n : 1);
  const size_t m = orc_reject_surface_normal(oc(in), n, static_cast<const float*>(src_normals), stride_sn / 4, static_cast<const float*>(tgt_normals),
                                             stride_tn / 4, threshold, tmp.data());
  std::copy(tmp.begin(), tmp.begin() + m, oc(out));
  *n_out = m;
  return PCLB200_OK;
}

int pclb200_estimate_svd(pclb200_ctx* ctx, const void* src, size_t ss, const void* tgt, size_t st, const pclb200_corr* corr, size_t n, int dbl, double T[16])
{
  if (!ctx || !src || !tgt || !T) return fail(PCLB200_ERR_INVALID, "NULL argument");
  orc_estimate_svd(static_cast<const float*>(src), ss / 4, static_cast<const float*>(tgt), st / 4, oc(corr), n, dbl, T);
  return PCLB200_OK;
}
int pclb200_estimate_svd_correlation(pclb200_ctx* ctx, const void* src, size_t ss, const void* tgt, size_t st, const pclb200_corr* corr, size_t n, int dbl,
                                     double T[16])
{
  if (!ctx || !src || !tgt || !T) return fail(PCLB200_ERR_INVALID, "NULL argument");
  orc_estimate_svd_correlation(static_cast<const float*>(src), ss / 4, static_cast<const float*>(tgt), st / 4, oc(corr), n, dbl, T);
  return PCLB200_OK;
}
int pclb200_estimate_point_to_plane_lls(pclb200_ctx* ctx, const void* src, size_t ss, const void* tgt, const void* tn, size_t st, const pclb200_corr* corr,
                                        size_t n, int dbl, double T[16])
{
  if (!ctx || !src || !tgt || !tn || !T) return fail(PCLB200_ERR_INVALID, "NULL argument");
  orc_estimate_point_to_plane_lls(static_cast<const float*>(src), ss / 4, static_cast<const float*>(tgt), static_cast<const float*>(tn), st / 4, oc(corr), n,
                                  dbl, T);
  return PCLB200_OK;
}
int pclb200_estimate_symmetric_point_to_plane_lls(pclb200_ctx* ctx, const void* src, const void* sn, size_t ss, const void* tgt, const void* tn, size_t st,
                                                  const pclb200_corr* corr, size_t n, int enforce, int dbl, double T[16])
{
  if (!ctx || !src || !sn || !tgt || !tn || !T) return fail(PCLB200_ERR_INVALID, "NULL argument");
  orc_estimate_symmetric_lls(static_cast<const float*>(src), static_cast<const float*>(sn), ss / 4, static_cast<const float*>(tgt),
                             static_cast<const float*>(tn), st / 4, oc(corr), n, enforce, dbl, T);
  return PCLB200_OK;
}

// ---- ICP session --------------------------------------------------------------------------------------------------------
void pclb200_icp_default_params(pclb200_icp_params* p)
{
  if (!p) return;
  std::memset(p, 0, sizeof(*p));
  p->max_iterations = 10;
  p->estimator = PCLB200_EST_SVD;
  p->is_dense = 1;
  p->enforce_same_direction_normals = 1;
  p->correspondence_kind = PCLB200_CORR_NEAREST;
  p->correspondence_k = 10;
  p->max_correspondence_distance = std::sqrt(std::numeric_limits<double>::max());
  p->euclidean_fitness_epsilon = -std::numeric_limits<double>::max();
  p->mse_threshold_absolute = 1e-12;
}
int pclb200_icp_create(pclb200_ctx* ctx, const pclb200_icp_params* params, pclb200_icp** out)
{
  if (!ctx || !out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  auto* s = new pclb200_icp();
  if (params) s->P = *params; else pclb200_icp_default_params(&s->P);
  *out = s;
  return PCLB200_OK;
}
int pclb200_icp_destroy(pclb200_icp* s) { delete s; return PCLB200_OK; }
int pclb200_icp_set_params(pclb200_icp* s, const pclb200_icp_params* p)
{
  if (!s || !p) return fail(PCLB200_ERR_INVALID, "NULL argument");
  s->P = *p;
  return PCLB200_OK;
}
int pclb200_icp_set_rejectors(pclb200_icp* s, const pclb200_rejector* list, int n)
{
  if (!s || n < 0 || (n > 0 && !list)) return fail(PCLB200_ERR_INVALID, "NULL argument");
  s->chain.clear();
  for (int i = 0; i < n; ++i) s->chain.push_back({list[i].kind, list[i].min_correspondences, list[i].p});
  return PCLB200_OK;
}
int pclb200_icp_set_target(pclb200_icp* s, const pclb200_index* idx, const void* tn, size_t stride_n)
{
  if (!s || !idx) return fail(PCLB200_ERR_INVALID, "NULL argument");
  s->tgt = idx;
  s->tgt_normals = tn != nullptr;
  s->tgt_rec = pack(idx->cloud.data(), idx->n, 16, tn, stride_n, 8);
  return PCLB200_OK;
}
int pclb200_icp_set_source(pclb200_icp* s, const void* src, size_t n, size_t stride, const void* sn, size_t stride_n, const int32_t* indices, size_t n_idx,
                           const double guess[16])
{
  if (!s || !src || n == 0) return fail(PCLB200_ERR_INVALID, "icp: empty source");
  s->src_rec = pack(src, n, stride, sn, stride_n, 8);
  s->n_src = n;
  s->src_normals = sn != nullptr;
  s->has_indices = indices != nullptr;
  s->indices.assign(indices, indices + (indices ? n_idx : 0));
  s->has_guess = guess != nullptr;
  if (guess) std::memcpy(s->guess, guess, sizeof(s->guess));
  s->prev_mse_at_source = s->prev_mse;
  s->have_full = false;
  s->done = 0;
  s->finished = false;
  return PCLB200_OK;
}

static int icp_run(pclb200_icp* s, int max_iterations, orc_icp_result& R, std::vector<float>& cloud, std::vector<orc_corr>& corr,
                   double* prev_mse)
{
  const pclb200_icp_params& P = s->P;
  const bool need_tn = P.estimator != PCLB200_EST_SVD || P.correspondence_kind == PCLB200_CORR_BACK_PROJECTION;
  const bool need_sn = P.estimator == PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS || P.correspondence_kind != PCLB200_CORR_NEAREST;
  if (need_tn && !s->tgt_normals) return fail(PCLB200_ERR_INVALID, "icp: this configuration needs target normals");
  if (need_sn && !s->src_normals) return fail(PCLB200_ERR_INVALID, "icp: this configuration needs source normals");
  orc_icp_params O{};
  O.max_iterations = max_iterations;
  O.use_reciprocal = P.use_reciprocal;
  O.estimator = P.estimator;
  O.scalar_is_double = P.scalar_is_double;
  O.with_normals_transform = P.with_normals_transform;
  O.source_has_normals = s->src_normals ? 1 : 0;
  O.is_dense = P.is_dense;
  O.nthreads = kThreads;
  O.max_correspondence_distance = P.max_correspondence_distance;
  O.transformation_epsilon = P.transformation_epsilon;
  O.transformation_rotation_epsilon = P.transformation_rotation_epsilon;
  O.euclidean_fitness_epsilon = P.euclidean_fitness_epsilon;
  O.correspondence_kind = P.correspondence_kind;
  O.correspondence_k = P.correspondence_k;
  orc_icp_ext X{P.failure_after_max_iter, P.max_iterations_similar_transforms, P.svd_no_umeyama, P.enforce_same_direction_normals, P.mse_threshold_absolute};
  *prev_mse = s->prev_mse_at_source;
  cloud.assign(s->src_rec.size(), 0.f);
  corr.assign(std::max<size_t>(s->has_indices ? s->indices.size() : s->n_src, 1), orc_corr{});
  size_t nc = 0;
  orc_icp_align_carry(&O, &X, s->chain.empty() ? nullptr : s->chain.data(), (int)s->chain.size(), s->tgt->tree, s->src_rec.data(), s->n_src, 8,
                      s->has_indices ? s->indices.data() : nullptr, s->has_indices ? s->indices.size() : 0, s->tgt_rec.data(), s->tgt->n, 8,
                      s->has_guess ? s->guess : nullptr, &R, cloud.data(), corr.data(), &nc, prev_mse);
  corr.resize(nc);
  return PCLB200_OK;
}

int pclb200_icp_iterate(pclb200_icp* s, int max_steps, pclb200_icp_stats* st)
{
  if (!s || !st) return fail(PCLB200_ERR_INVALID, "NULL argument");
  if (!s->tgt || s->src_rec.empty()) return fail(PCLB200_ERR_INVALID, "icp: target and source must be set");
  if (max_steps < 0) return fail(PCLB200_ERR_INVALID, "max_steps < 0");
  if (!s->have_full) {
    int rc = icp_run(s, s->P.max_iterations, s->full, s->full_cloud, s->full_corr, &s->full_prev_mse);
    if (rc != PCLB200_OK) return rc;
    s->have_full = true;
  }
  if (!s->finished && max_steps > 0) {
    // the loop ends after full.iterations iterations; a NO_CORRESPONDENCES exit is found one evaluation later
    const long long last = (long long)s->full.iterations + (s->full.state == PCLB200_CONV_NO_CORRESPONDENCES ? 1 : 0);
    const long long want = (long long)s->done + max_steps;
    if (want >= last) {
      s->cur = s->full; s->cur_cloud = s->full_cloud; s->cur_corr = s->full_corr;
      s->done = s->full.iterations;
      s->finished = true;
      s->prev_mse = s->full_prev_mse;
    }
    else {
      double replay_prev_mse;
      int rc = icp_run(s, (int)want, s->cur, s->cur_cloud, s->cur_corr, &replay_prev_mse);
      if (rc != PCLB200_OK) return rc;
      s->cur.state = PCLB200_CONV_NOT_CONVERGED;
      s->cur.converged = 0;
      s->done = (int)want;
      // the replay stopped on its iteration cap before its criteria recorded iteration `want`; the session's did
      s->prev_mse = s->cur.mse;
    }
  }
  std::memset(st, 0, sizeof(*st));
  if (s->done == 0 && !s->finished) {  // nothing evaluated yet
    for (int i = 0; i < 16; ++i) st->final_transformation[i] = s->has_guess ? s->guess[i] : (i % 5 == 0), st->last_transformation[i] = (i % 5 == 0);
    return PCLB200_OK;
  }
  st->converged = s->cur.converged;
  st->state = s->cur.state;
  st->iterations = s->cur.iterations;
  st->n_correspondences = s->cur.n_correspondences;
  st->mse = s->cur.mse;
  std::memcpy(st->final_transformation, s->cur.final_transformation, sizeof(st->final_transformation));
  std::memcpy(st->last_transformation, s->cur.last_transformation, sizeof(st->last_transformation));
  st->total_correspondences = s->cur.total_correspondences;
  return PCLB200_OK;
}

int pclb200_icp_get_cloud(pclb200_icp* s, void* out_pts, size_t stride_out, void* out_normals, size_t stride_n)
{
  if (!s || !out_pts || s->src_rec.empty()) return fail(PCLB200_ERR_INVALID, "icp: no source");
  std::vector<float> start;
  const std::vector<float>* c = &s->cur_cloud;
  if (s->done == 0 && !s->finished) {  // the guess applied to the input
    start = s->src_rec;
    double I[16];
    for (int i = 0; i < 16; ++i) I[i] = s->has_guess ? s->guess[i] : (i % 5 == 0);
    orc_transform(start.data(), s->n_src, 8, s->src_normals ? 4 : -1, I, s->P.scalar_is_double, s->P.with_normals_transform);
    c = &start;
  }
  for (size_t i = 0; i < s->n_src; ++i) {
    std::memcpy(static_cast<unsigned char*>(out_pts) + i * stride_out, &(*c)[8 * i], 12);
    if (out_normals && s->src_normals) std::memcpy(static_cast<unsigned char*>(out_normals) + i * stride_n, &(*c)[8 * i + 4], 12);
  }
  return PCLB200_OK;
}
int pclb200_icp_get_correspondences(pclb200_icp* s, pclb200_corr* out, size_t* n_out)
{
  if (!s || !out || !n_out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  std::copy(s->cur_corr.begin(), s->cur_corr.end(), oc(out));
  *n_out = (s->done == 0 && !s->finished) ? 0 : s->cur_corr.size();
  return PCLB200_OK;
}
int pclb200_icp_align(pclb200_ctx* ctx, const pclb200_icp_params* params, const void* src, size_t n, size_t stride, const void* sn, size_t stride_sn,
                      const int32_t* src_indices, size_t n_idx, const pclb200_index* idx_tgt, const void* tn, size_t stride_tn, const double guess[16],
                      void* out_cloud, size_t stride_out, pclb200_icp_stats* stats)
{
  pclb200_icp* s = nullptr;
  int rc = pclb200_icp_create(ctx, params, &s);
  if (rc == PCLB200_OK) rc = pclb200_icp_set_target(s, idx_tgt, tn, stride_tn);
  if (rc == PCLB200_OK) rc = pclb200_icp_set_source(s, src, n, stride, sn, stride_sn, src_indices, n_idx, guess);
  pclb200_icp_stats st;
  if (rc == PCLB200_OK) rc = pclb200_icp_iterate(s, std::numeric_limits<int>::max(), &st);
  if (rc == PCLB200_OK && stats) *stats = st;
  if (rc == PCLB200_OK && out_cloud) rc = pclb200_icp_get_cloud(s, out_cloud, stride_out, nullptr, 0);
  pclb200_icp_destroy(s);
  return rc;
}

int pclb200_fitness_score(pclb200_ctx* ctx, const pclb200_index* idx_tgt, const void* src, size_t n, size_t stride, const int32_t* src_indices, size_t n_idx,
                          int is_dense, const double T[16], int dbl, double max_range, double* score)
{
  if (!ctx || !idx_tgt || !src || !T || !score) return fail(PCLB200_ERR_INVALID, "NULL argument");
  const std::vector<float> S = pack(src, n, stride, nullptr, 0, 4);
  *score = orc_fitness_score(idx_tgt->tree, S.data(), n, 4, src_indices, src_indices ? n_idx : n, is_dense, T, dbl, max_range, kThreads);
  return PCLB200_OK;
}

int pclb200_gicp_covariances(pclb200_ctx* ctx, const pclb200_index* h, const void* pts, size_t n, size_t stride, int k, double eps, double* out)
{
  if (!ctx || !h || !pts || !out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  const std::vector<float> C = pack(pts, n, stride, nullptr, 0, 4);
  orc_gicp_covariances(h->tree, C.data(), n, 4, k, eps, out, kThreads);
  return PCLB200_OK;
}

int pclb200_validate_transformation(pclb200_ctx* ctx, const pclb200_index* idx_tgt, const void* src, size_t n, size_t stride, const double T[16], int dbl,
                                    double max_range, double* score)
{
  if (!ctx || !idx_tgt || !src || !T || !score) return fail(PCLB200_ERR_INVALID, "NULL argument");
  const std::vector<float> S = pack(src, n, stride, nullptr, 0, 4);
  std::vector<float> M;
  if (dbl) moved_by<double>(S, n, T, M); else moved_by<float>(S, n, T, M);
  std::vector<int32_t> ki(n ? n : 1);
  std::vector<float> kd(n ? n : 1);
  orc_knn(idx_tgt->tree, M.data(), n, 4, 1, ki.data(), kd.data(), kThreads);
  double sum = 0;
  size_t cnt = 0;
  for (size_t i = 0; i < n; ++i)
    if (ki[i] >= 0 && (double)kd[i] <= max_range) { sum += kd[i]; ++cnt; }
  *score = cnt ? sum / (double)cnt : std::numeric_limits<double>::max();
  return PCLB200_OK;
}
int pclb200_inliers(pclb200_ctx* ctx, const pclb200_index* idx_tgt, const void* src, size_t n, size_t stride, const double T[16], float thr, pclb200_corr* out,
                    size_t* n_out)
{
  if (!ctx || !idx_tgt || !src || !T || !out || !n_out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  std::vector<float> S = pack(src, n, stride, nullptr, 0, 4);
  double Tf[16];
  for (int i = 0; i < 16; ++i) Tf[i] = (double)(float)T[i];
  orc_transform(S.data(), n, 4, -1, Tf, 0, 1);  // pcl::transformPointCloud, float
  std::vector<int32_t> ki(n ? n : 1);
  std::vector<float> kd(n ? n : 1);
  orc_knn(idx_tgt->tree, S.data(), n, 4, 1, ki.data(), kd.data(), kThreads);
  const float max_range = thr * thr;
  size_t m = 0;
  for (size_t i = 0; i < n; ++i)
    if (std::isfinite(S[4 * i]) && std::isfinite(S[4 * i + 1]) && std::isfinite(S[4 * i + 2]) && ki[i] >= 0 && kd[i] < max_range)
      out[m++] = pclb200_corr{(int32_t)i, ki[i], kd[i]};
  *n_out = m;
  return PCLB200_OK;
}

int pclb200_normals_knn(pclb200_ctx* ctx, const pclb200_index* h, const void* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int is_dense,
                        int k, const float vp[3], float* out, int* dense_out)
{
  if (!ctx || !h || !pts || !vp || !out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  if (k <= 0) return fail(PCLB200_ERR_INVALID, "k <= 0");
  const std::vector<float> C = pack(pts, n, stride, nullptr, 0, 4);
  const int dense = orc_normals_knn(h->tree, C.data(), n, 4, indices, indices ? n_idx : 0, is_dense, k, vp, out, kThreads);
  if (dense_out) *dense_out = dense;
  return PCLB200_OK;
}
int pclb200_normals_radius(pclb200_ctx* ctx, const pclb200_index* h, const void* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx,
                           int is_dense, double radius, const float vp[3], float* out, int* dense_out)
{
  if (!ctx || !h || !pts || !vp || !out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  const std::vector<float> C = pack(pts, n, stride, nullptr, 0, 4);
  const int dense = orc_normals_radius(h->tree, C.data(), n, 4, indices, indices ? n_idx : 0, is_dense, radius, vp, out, kThreads);
  if (dense_out) *dense_out = dense;
  return PCLB200_OK;
}

int pclb200_cluster_labels(pclb200_ctx* ctx, const pclb200_index* h, double tolerance, int32_t* out_labels, size_t n_labels)
{
  if (!ctx || !h || !out_labels) return fail(PCLB200_ERR_INVALID, "NULL argument");
  if (n_labels != h->n) return fail(PCLB200_ERR_INVALID, "n_labels != points of the indexed cloud");
  orc_cluster_labels(h->tree, h->n, tolerance, out_labels);
  return PCLB200_OK;
}

static int voxel_rc(long long m, size_t* n_out)
{
  if (m < 0) return fail(PCLB200_ERR_LEAF_TOO_SMALL, "Leaf size is too small for the input dataset. Integer indices would overflow.");
  *n_out = (size_t)m;
  return PCLB200_OK;
}
int pclb200_voxelgrid(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int is_dense, const float leaf[3],
                      unsigned min_pts, float* out, size_t* n_out)
{
  if (!ctx || !leaf || !out || !n_out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  *n_out = 0;
  if (n == 0) return PCLB200_OK;
  const std::vector<float> C = pack(pts, n, stride, nullptr, 0, 4);
  return voxel_rc(orc_voxelgrid(C.data(), n, 4, indices, indices ? n_idx : 0, is_dense, leaf, min_pts, out), n_out);
}
int pclb200_voxelgrid_normals(pclb200_ctx* ctx, const void* pts, size_t n, size_t stride, const void* normals, size_t stride_n, const int32_t* indices,
                              size_t n_idx, int is_dense, const float leaf[3], unsigned min_pts, float* out, float* out_nc, size_t* n_out)
{
  if (!ctx || !leaf || !normals || !out || !out_nc || !n_out) return fail(PCLB200_ERR_INVALID, "NULL argument");
  *n_out = 0;
  if (n == 0) return PCLB200_OK;
  std::vector<float> C(n * 12, 0.f);  // xyz1 | normal n4 | curvature
  for (size_t i = 0; i < n; ++i) {
    std::memcpy(&C[12 * i], static_cast<const unsigned char*>(pts) + i * stride, 12);
    C[12 * i + 3] = 1.f;
    std::memcpy(&C[12 * i + 4], static_cast<const unsigned char*>(normals) + i * stride_n, 20);
  }
  return voxel_rc(orc_voxelgrid_normals(C.data(), n, 12, indices, indices ? n_idx : 0, is_dense, leaf, min_pts, out, 4, out_nc), n_out);
}
int pclb200_voxelgrid_tile(pclb200_ctx*, const void*, size_t, size_t, const float*, const float*, unsigned, float*, size_t*)
{
  return fail(PCLB200_ERR_INVALID, "tests/host/pclb200_on_oracle.cpp: voxelgrid_tile is not part of the test double");
}

int pclb200_comm_unique_id(void*) { return fail(PCLB200_ERR_INVALID, "tests/host/pclb200_on_oracle.cpp: no communicator"); }
int pclb200_comm_init(pclb200_ctx*, int, int, const void*) { return fail(PCLB200_ERR_INVALID, "tests/host/pclb200_on_oracle.cpp: no communicator"); }
int pclb200_comm_set_mode(pclb200_ctx*, int) { return fail(PCLB200_ERR_INVALID, "tests/host/pclb200_on_oracle.cpp: no communicator"); }
int pclb200_comm_export(pclb200_ctx*, void*) { return fail(PCLB200_ERR_INVALID, "tests/host/pclb200_on_oracle.cpp: no communicator"); }
int pclb200_comm_import(pclb200_ctx*, int, int, const void*) { return fail(PCLB200_ERR_INVALID, "tests/host/pclb200_on_oracle.cpp: no communicator"); }

}  // extern "C"
