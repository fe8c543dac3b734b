// consumers_host_test.cpp — the kernels behind the stand-alone consumers of the searcher (pcl_b200/csrc/icp_kernels.cuh:
// k_corr plain and reciprocal = pclb200_correspondences, k_fitness = pclb200_fitness_score, k_gicp_cov =
// pclb200_gicp_covariances) compiled for the HOST, run on the emulated thread block, against the CPU oracle
// (oracle/libpcl_oracle.so, linked: test infrastructure): correspondence lists bit for bit (gate, index subsets, non-finite
// source points, duplicates), the fitness score to 1e-12, the regularised covariances to 1e-9.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"


#include <cfloat>

static inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }

#include "../../pcl_b200/csrc/icp_kernels.cuh"
#include "../../pcl_b200/csrc/normals_corr_kernels.cuh"
#include "../../pcl_b200/csrc/cluster_kernels.cuh"
#include "../../pcl_b200/csrc/search_kernels.cuh"

extern "C" {
void* orc_index_build(const float* pts, size_t n, size_t stride, const int32_t* subset, size_t n_subset);
void orc_index_free(void* h);
int orc_knn(void* h, const float* q, size_t nq, size_t qstride, int k, int32_t* out_idx, float* out_d2, int nthreads);
size_t orc_correspondences(void* h_tgt, const float* src, size_t n_src, size_t sstride, const int32_t* indices, size_t n_idx, int is_dense,
                           double max_distance, pclb200_corr* out, int nthreads);
size_t orc_correspondences_reciprocal(void* h_tgt, void* h_src, const float* src, size_t n_src, size_t sstride, const float* tgt, size_t tstride,
                                      const int32_t* indices, size_t n_idx, int is_dense, double max_distance, pclb200_corr* out, int nthreads);
double orc_fitness_score(void* h_tgt, const float* src, size_t n_s, size_t sstride, const int32_t* indices, size_t n_idx, int is_dense,
                         const double* final_T, int scalar_is_double, double max_range, int nthreads);
void orc_gicp_covariances(void* h, const float* cloud, size_t n, size_t stride, int k, double gicp_epsilon, double* out, int nthreads);
size_t orc_correspondences_normals(void* h_tgt, int kind, const float* src, size_t n_src, size_t sstride, const float* sn, size_t snstride,
                                   const float* tgt, size_t tstride, const float* tn, size_t tnstride, const int32_t* indices, size_t n_idx,
                                   int k, double max_distance, pclb200_corr* out, int nthreads);
void orc_cluster_labels(void* h, size_t n_cloud, double tolerance, int32_t* out_labels);
size_t orc_reject_surface_normal(const pclb200_corr* in, size_t n, const float* sn, size_t snstride, const float* tn, size_t tnstride,
                                 double threshold, pclb200_corr* out);
}

// the fixed seed of the committed test, or PCLB_TEST_SEED for a fuzz run (tools/dev/fuzz_host_tests.sh)
static float gate_from_max_dist(double max_dist)   // icp.cu: the largest float not above max_dist^2
{
  const double m2 = max_dist * max_dist;
  if (!(m2 < (double)FLT_MAX)) return FLT_MAX;
  float g = (float)m2;
  if ((double)g > m2) g = std::nextafter(g, -INFINITY);
  return g;
}

template <typename F> static void launch(unsigned grid, int block, F kernel)
{
  blockDim.x = block;
  gridDim.x = grid ? grid : 1;
  for (unsigned b = 0; b < gridDim.x; ++b) { blockIdx_storage.x = b; warp_emu::run_block(block, kernel); }
  blockIdx_storage.x = 0;
  gridDim.x = 1;
}

static std::vector<float> xyz_of(const std::vector<float>& c4)
{
  std::vector<float> v(c4.size() / 4 * 3);
  for (std::size_t i = 0; i < c4.size() / 4; ++i) for (int d = 0; d < 3; ++d) v[3 * i + d] = c4[4 * i + d];
  return v;
}

// icp.cu: correspondences() — queries in slot order (the Morton sort of the real driver only permutes the launch order)
static std::vector<pclb200_corr> device_correspondences(const HostIndex& IT, const HostIndex* IS, const std::vector<float>& src, const std::vector<int32_t>* indices,
                                                        double max_dist)
{
  const std::size_t nq = indices ? indices->size() : src.size() / 4;
  std::vector<float4> q(nq);
  for (std::size_t i = 0; i < nq; ++i) {
    const float* p = &src[4 * (indices ? (std::size_t)(*indices)[i] : i)];
    q[i] = make_float4(p[0], p[1], p[2], __int_as_float((int)i));
  }
  std::vector<pclb200_corr> by_slot(nq), out;
  int d_error = 0;
  const TreeView T = IT.view(true);
  const float gate = gate_from_max_dist(max_dist);
  const unsigned grid = (unsigned)((nq + 127) / 128);
  if (IS)
    launch(grid, 128, [&] { k_corr<true>(T, q.data(), nq, gate, IS->nodes.data(), IS->pts.data(), IS->root, indices ? indices->data() : nullptr, by_slot.data(), &d_error); });
  else
    launch(grid, 128, [&] { k_corr<false>(T, q.data(), nq, gate, nullptr, nullptr, 0, indices ? indices->data() : nullptr, by_slot.data(), &d_error); });
  CHECK(d_error == 0, "traversal stack overflow flag");
  for (const pclb200_corr& c : by_slot) if (c.index_match >= 0) out.push_back(c);   // cub::DeviceSelect::If(CorrValid)
  return out;
}

static void compare_lists(const char* what, const std::vector<pclb200_corr>& got, const std::vector<pclb200_corr>& want)
{
  CHECK(got.size() == want.size(), "%s: %zu pairs, the oracle has %zu", what, got.size(), want.size());
  std::size_t bad = 0;
  for (std::size_t i = 0; i < got.size() && i < want.size(); ++i) bad += std::memcmp(&got[i], &want[i], sizeof(pclb200_corr)) != 0;
  CHECK(bad == 0, "%s: %zu records differ", what, bad);
  std::printf("%-58s %6zu pairs (oracle %zu)\n", what, got.size(), want.size());
}

int main()
{
  std::mt19937 rng(test_seed(99));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::normal_distribution<float> N(0.f, 1.f);
  const int nt = 6000, ns = 4000;
  std::vector<float> tgt(4 * nt, 1.f), src(4 * ns, 1.f);
  for (int i = 0; i < nt; ++i) { tgt[4 * i] = 2.f * U(rng); tgt[4 * i + 1] = 2.f * U(rng); tgt[4 * i + 2] = 0.2f * std::sin(4.f * tgt[4 * i]) + 0.01f * N(rng); }
  for (int i = 0; i < 40; ++i) std::memcpy(&tgt[4 * (nt - 1 - i)], &tgt[4 * i], 12);   // duplicated target points: the smaller index wins
  const float ca = std::cos(0.03f), sa = std::sin(0.03f);
  for (int i = 0; i < ns; ++i) {
    const float* t = &tgt[4 * (int)(U(rng) * nt)];
    src[4 * i] = ca * t[0] - sa * t[1] + 0.01f + 0.002f * N(rng);
    src[4 * i + 1] = sa * t[0] + ca * t[1] - 0.008f + 0.002f * N(rng);
    src[4 * i + 2] = t[2] + 0.004f + 0.002f * N(rng);
  }
  HostIndex IT, IS;
  build_index(IT, xyz_of(tgt), 4);
  build_index(IS, xyz_of(src), 4);
  void* ot = orc_index_build(tgt.data(), nt, 4, nullptr, 0);
  void* os = orc_index_build(src.data(), ns, 4, nullptr, 0);
  std::vector<int32_t> subset;
  for (int i = ns - 1; i >= 0; i -= 3) subset.push_back(i);   // a descending subset: output order is the subset's

  std::vector<pclb200_corr> want(ns);
  for (double md : {std::sqrt(std::numeric_limits<double>::max()), 0.05, 0.01, 0.0}) {
    char name[128];
    std::snprintf(name, sizeof name, "nearest, max distance %.3g", md > 1e10 ? INFINITY : md);
    want.resize(ns);
    want.resize(orc_correspondences(ot, src.data(), ns, 4, nullptr, 0, 1, md, want.data(), 2));
    compare_lists(name, device_correspondences(IT, nullptr, src, nullptr, md), want);
    std::snprintf(name, sizeof name, "reciprocal, max distance %.3g", md > 1e10 ? INFINITY : md);
    want.resize(ns);
    want.resize(orc_correspondences_reciprocal(ot, os, src.data(), ns, 4, tgt.data(), 4, nullptr, 0, 1, md, want.data(), 2));
    compare_lists(name, device_correspondences(IT, &IS, src, nullptr, md), want);
  }
  want.resize(ns);
  want.resize(orc_correspondences(ot, src.data(), ns, 4, subset.data(), subset.size(), 1, 0.03, want.data(), 2));
  compare_lists("nearest, index subset (descending)", device_correspondences(IT, nullptr, src, &subset, 0.03), want);
  want.resize(ns);
  want.resize(orc_correspondences_reciprocal(ot, os, src.data(), ns, 4, tgt.data(), 4, subset.data(), subset.size(), 1, 0.03, want.data(), 2));
  compare_lists("reciprocal, index subset (descending)", device_correspondences(IT, &IS, src, &subset, 0.03), want);
  {
    std::vector<float> holes = src;
    for (int i = 5; i < ns; i += 41) holes[4 * i + (i % 3)] = i % 2 ? std::numeric_limits<float>::quiet_NaN() : std::numeric_limits<float>::infinity();
    want.resize(ns);
    want.resize(orc_correspondences(ot, holes.data(), ns, 4, nullptr, 0, 0, 0.05, want.data(), 2));
    compare_lists("nearest, non-finite source points skipped", device_correspondences(IT, nullptr, holes, nullptr, 0.05), want);
  }

  {  // the reference's CorrespondenceEstimationSetSearchMethod clouds: 50 points with coordinates static_cast<float>(rand()), up to 2^31
    std::srand(7);
    const int m = 50;
    std::vector<float> a(4 * m, 1.f), b(4 * m, 1.f);
    for (int i = 0; i < m; ++i)
      for (int d = 0; d < 3; ++d) { a[4 * i + d] = static_cast<float>(std::rand()); b[4 * i + d] = static_cast<float>(std::rand()); }
    HostIndex IB2, IA2;
    build_index(IB2, xyz_of(b), 4);
    build_index(IA2, xyz_of(a), 4);
    void* ob2 = orc_index_build(b.data(), m, 4, nullptr, 0);
    void* oa2 = orc_index_build(a.data(), m, 4, nullptr, 0);
    want.resize(m);
    want.resize(orc_correspondences(ob2, a.data(), m, 4, nullptr, 0, 1, std::sqrt(std::numeric_limits<double>::max()), want.data(), 1));
    compare_lists("50 points with coordinates up to 2^31, nearest", device_correspondences(IB2, nullptr, a, nullptr, std::sqrt(std::numeric_limits<double>::max())), want);
    want.resize(m);
    want.resize(orc_correspondences_reciprocal(ob2, oa2, a.data(), m, 4, b.data(), 4, nullptr, 0, 1, std::sqrt(std::numeric_limits<double>::max()), want.data(), 1));
    compare_lists("50 points with coordinates up to 2^31, reciprocal", device_correspondences(IB2, &IA2, a, nullptr, std::sqrt(std::numeric_limits<double>::max())), want);
    orc_index_free(ob2);
    orc_index_free(oa2);
  }

  // ---- Registration::getFitnessScore: transform (float or double), 1-NN, mean of the squared distances <= max_range ----
  {
    const double a = 0.02, T[16] = {std::cos(a), -std::sin(a), 0, 0.004, std::sin(a), std::cos(a), 0, -0.003, 0, 0, 1, 0.001, 0, 0, 0, 1};
    const TreeView TV = IT.view(true);
    for (int dbl = 0; dbl < 2; ++dbl)
      for (double max_range : {std::numeric_limits<double>::max(), 1e-4, 1e-7, 0.0}) {
        Pending h;
        std::memset(&h, 0, sizeof h);
        for (int i = 0; i < 12; ++i) { h.f[i] = (float)T[i]; h.d[i] = dbl ? T[i] : (double)(float)T[i]; }
        h.apply = 1;
        h.mode = dbl ? 2 : 1;
        std::vector<float4> q(ns);
        for (int i = 0; i < ns; ++i) { q[i] = make_float4(src[4 * i], src[4 * i + 1], src[4 * i + 2], __int_as_float(i)); apply_pending(h, q[i].x, q[i].y, q[i].z); }
        const unsigned grid = 3;
        std::vector<double> partials(grid * kAccum, 0.0), accum(kAccum, -1.0);
        unsigned counter = 0;
        int d_error = 0;
        const GridSum sum{partials.data(), &counter, accum.data()};
        launch(grid, 256, [&] { k_fitness(TV, q.data(), (size_t)ns, max_range, sum, &d_error); });
        const double got = accum[0] > 0 ? accum[1] / accum[0] : std::numeric_limits<double>::max();
        const double wantf = orc_fitness_score(ot, src.data(), ns, 4, nullptr, ns, 1, T, dbl, max_range, 2);
        CHECK(d_error == 0 && std::fabs(got - wantf) <= 1e-12 * std::fabs(wantf), "fitness %s max_range %g: %.17g, the oracle's %.17g", dbl ? "double" : "float", max_range,
              got, wantf);
        std::printf("fitness score, %-6s max range %-12.3g %.12g over %.0f points (oracle %.12g)\n", dbl ? "double" : "float", max_range, got, accum[0], wantf);
      }
  }

  // ---- GICP covariances over exact k-NN rows -------------------------------------------------------------------------
  {
    const int k = 20;
    std::vector<int32_t> rows((size_t)nt * k);
    std::vector<float> rd((size_t)nt * k);
    orc_knn(ot, tgt.data(), nt, 4, k, rows.data(), rd.data(), 2);
    std::vector<int32_t> pos_of_orig(nt, -1);
    for (std::size_t p = 0; p < IT.pts.size(); ++p) { const int o = __float_as_int(IT.pts[p].w); if (o != kSentinelIndex) pos_of_orig[o] = (int32_t)p; }
    std::vector<float4> q(nt);
    for (int i = 0; i < nt; ++i) q[i] = make_float4(tgt[4 * i], tgt[4 * i + 1], tgt[4 * i + 2], 1.f);
    std::vector<double> got((size_t)nt * 9, -1.0), wantc((size_t)nt * 9, 0.0);
    launch((unsigned)((nt + 127) / 128), 128, [&] { k_gicp_cov(q.data(), (size_t)nt, rows.data(), k, k, IT.pts.data(), pos_of_orig.data(), 0.001, got.data()); });
    orc_gicp_covariances(ot, tgt.data(), nt, 4, k, 0.001, wantc.data(), 2);
    double worst = 0;
    for (std::size_t e = 0; e < got.size(); ++e) worst = std::max(worst, std::fabs(got[e] - wantc[e]));
    CHECK(worst < 1e-9, "GICP covariances: largest difference %.3g", worst);
    std::printf("GICP covariances k = 20: largest |difference| over %d matrices %.3g\n", nt, worst);
  }
  // ---- normal shooting / back projection over exact k-NN rows; the surface-normal rejector --------------------------------
  {
    auto unit_normals = [&](const std::vector<float>& c4, float tilt) {
      std::vector<float> n(c4.size(), 0.f);
      for (std::size_t i = 0; i < c4.size() / 4; ++i) {
        float nx = -0.8f * std::cos(4.f * c4[4 * i]) + tilt * N(rng), ny = tilt * N(rng), nz = 1.f;
        const float inv = 1.f / std::sqrt(nx * nx + ny * ny + nz * nz);
        n[4 * i] = nx * inv; n[4 * i + 1] = ny * inv; n[4 * i + 2] = nz * inv;
      }
      return n;
    };
    const std::vector<float> sn = unit_normals(src, 0.05f), tn = unit_normals(tgt, 0.05f);
    std::vector<int32_t> pos_of_orig(nt, -1);
    for (std::size_t p = 0; p < IT.pts.size(); ++p) { const int o = __float_as_int(IT.pts[p].w); if (o != kSentinelIndex) pos_of_orig[o] = (int32_t)p; }
    const float4* sn4 = reinterpret_cast<const float4*>(sn.data());
    const float4* tn4 = reinterpret_cast<const float4*>(tn.data());
    for (int kind : {PCLB200_CORR_NORMAL_SHOOTING, PCLB200_CORR_BACK_PROJECTION})
      for (int k : {10, 3})
        for (double md : {0.02, 0.0008})
          for (int use_subset = 0; use_subset < 2; ++use_subset) {
            const std::vector<int32_t>* ind = use_subset ? &subset : nullptr;
            const std::size_t nq = ind ? ind->size() : (std::size_t)ns;
            std::vector<float4> dense(nq);
            std::vector<float> q4(4 * nq);
            for (std::size_t i = 0; i < nq; ++i) {
              const float* p = &src[4 * (ind ? (std::size_t)(*ind)[i] : i)];
              dense[i] = make_float4(p[0], p[1], p[2], 1.f);
              std::memcpy(&q4[4 * i], p, 16);
            }
            std::vector<int32_t> rows(nq * k);
            std::vector<float> rd(nq * k);
            orc_knn(ot, q4.data(), nq, 4, k, rows.data(), rd.data(), 2);
            std::vector<pclb200_corr> by_slot(nq), got;
            launch((unsigned)((nq + 127) / 128), 128, [&] {
              k_corr_by_normals(dense.data(), nq, ind ? ind->data() : nullptr, sn4, kind, k, rows.data(), rd.data(), IT.pts.data(), pos_of_orig.data(), tn4, md, by_slot.data());
            });
            for (const pclb200_corr& c : by_slot) if (c.index_match >= 0) got.push_back(c);
            want.resize(ns);
            want.resize(orc_correspondences_normals(ot, kind, src.data(), ns, 4, sn.data(), 4, tgt.data(), 4, tn.data(), 4, ind ? ind->data() : nullptr, ind ? ind->size() : 0, k,
                                                    md, want.data(), 2));
            char name[128];
            std::snprintf(name, sizeof name, "%s, k = %d, max distance %.3g%s", kind == PCLB200_CORR_NORMAL_SHOOTING ? "normal shooting" : "back projection", k, md,
                          use_subset ? ", subset" : "");
            compare_lists(name, got, want);
          }
    // CorrespondenceRejectorSurfaceNormal on the nearest-neighbour pairs, incl. out-of-range records
    std::vector<pclb200_corr> pairs(ns);
    pairs.resize(orc_correspondences(ot, src.data(), ns, 4, nullptr, 0, 1, 0.05, pairs.data(), 2));
    for (double thr : {0.0, 0.9, 0.995, 1.0, -1.0}) {
      std::vector<pclb200_corr> marked(pairs.size()), got;
      launch((unsigned)((pairs.size() + 255) / 256), 256, [&] { k_mark_surface_normal(pairs.data(), pairs.size(), sn4, (size_t)ns, tn4, (size_t)nt, thr, marked.data()); });
      for (const pclb200_corr& c : marked) if (c.index_match >= 0) got.push_back(c);
      want.resize(pairs.size());
      want.resize(orc_reject_surface_normal(pairs.data(), pairs.size(), sn.data(), 4, tn.data(), 4, thr, want.data()));
      char name[96];
      std::snprintf(name, sizeof name, "surface-normal rejector, threshold %g", thr);
      compare_lists(name, got, want);
    }
  }
  // ---- Euclidean clustering: union-find over the tolerance graph, label = smallest original index of the component -------
  {
    const int nb = 5000;
    std::vector<float> blobs(4 * nb, 1.f);
    for (int i = 0; i < nb; ++i) {
      const int b = i % 23;
      blobs[4 * i] = 0.31f * (b % 5) + 0.02f * N(rng);
      blobs[4 * i + 1] = 0.29f * (b / 5) + 0.02f * N(rng);
      blobs[4 * i + 2] = 0.01f * N(rng);
    }
    for (int i = 0; i < 60; ++i) std::memcpy(&blobs[4 * (nb - 1 - i)], &blobs[4 * (7 * i)], 12);   // exact duplicates (distance 0)
    HostIndex IB;
    build_index(IB, xyz_of(blobs), 4);
    void* ob = orc_index_build(blobs.data(), nb, 4, nullptr, 0);
    const std::size_t np = IB.pts.size();
    for (double tol : {0.02, 0.008, 0.05, 0.2, 1e-9}) {
      const double t = (double)(float)tol;
      const float r2 = (float)(t * t), r2_below = std::nextafter(r2, -INFINITY);
      std::vector<int> parent(np), min_orig(np);
      std::vector<int32_t> labels(nb, -1), wantl(nb, -2);
      int d_error = 0;
      launch((unsigned)((np + 255) / 256), 256, [&] { k_cc_init(parent.data(), min_orig.data(), np); });
      launch((unsigned)((np + 127) / 128), 128, [&] { k_cc_union(IB.nodes.data(), IB.pts.data(), IB.root, np, r2, r2_below, parent.data(), &d_error); });
      launch((unsigned)((np + 255) / 256), 256, [&] { k_cc_min_orig(IB.pts.data(), np, parent.data(), min_orig.data()); });
      launch((unsigned)((np + 255) / 256), 256, [&] { k_cc_labels(IB.pts.data(), np, parent.data(), min_orig.data(), labels.data()); });
      orc_cluster_labels(ob, nb, tol, wantl.data());
      int bad = 0, comps = 0;
      for (int i = 0; i < nb; ++i) { bad += labels[i] != wantl[i]; comps += labels[i] == i; }
      CHECK(bad == 0 && d_error == 0, "clustering, tolerance %g: %d labels differ from the oracle's", tol, bad);
      std::printf("Euclidean clustering, tolerance %-8g %5d components over %d points, %d labels differ\n", tol, comps, nb, bad);
    }
    orc_index_free(ob);
  }
  // ---- the reference's TranslatedNormalEstimation surface (test_normal_estimation.cpp:266-275): 397 real points and 306 803
  //      default-constructed ones at the origin — one Morton code shared by 306 803 points: build, then k = 397 for every real point
  {
    const int real = 397, total = 640 * 480;
    std::vector<float> xyz(3 * (std::size_t)total, 0.f);
    for (int i = 0; i < real; ++i) { xyz[3 * i] = 100.f + 0.15f * U(rng); xyz[3 * i + 1] = 100.f + 0.15f * U(rng); xyz[3 * i + 2] = 100.f + 0.1f * U(rng); }
    HostIndex IM;
    build_index(IM, xyz, 0);
    const int k = 397;
    std::vector<float4> q(real);
    for (int i = 0; i < real; ++i) q[i] = make_float4(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], __int_as_float(i));
    std::vector<int32_t> oi((std::size_t)real * k, -7);
    std::vector<float> od((std::size_t)real * k, -7.f);
    int d_error = 0;
    launch((unsigned)((real + 127) / 128), 128, [&] { k_knn_any(IM.nodes.data(), IM.pts.data(), IM.root, q.data(), (size_t)real, k, INFINITY, oi.data(), od.data(), &d_error); });
    int bad = 0;
    std::vector<std::pair<float, int>> all(real);
    for (int i = 0; i < real; ++i) {
      for (int j = 0; j < real; ++j) all[j] = {dist2_rn(q[i].x, q[i].y, q[i].z, xyz[3 * j], xyz[3 * j + 1], xyz[3 * j + 2]), j};
      std::sort(all.begin(), all.end());
      for (int j = 0; j < k; ++j) if (oi[(std::size_t)i * k + j] != all[j].second || od[(std::size_t)i * k + j] != all[j].first) { ++bad; break; }
    }
    float4 qo = make_float4(0.f, 0.f, 0.f, __int_as_float(0));
    std::vector<int32_t> o2(20, -7);
    std::vector<float> d2(20, -7.f);
    launch(1, 128, [&] { k_knn_any(IM.nodes.data(), IM.pts.data(), IM.root, &qo, (size_t)1, 20, INFINITY, o2.data(), d2.data(), &d_error); });
    bool first_twenty = true;
    for (int j = 0; j < 20; ++j) first_twenty = first_twenty && o2[j] == real + j && d2[j] == 0.f;
    CHECK(bad == 0 && first_twenty && d_error == 0, "306 803 coincident points: %d of 397 k-NN rows differ, origin query ok %d, error flag %d", bad, (int)first_twenty, d_error);
    std::printf("306 803 coincident points + 397 real ones: %zu leaf slots, %zu nodes; k = 397 rows differing from brute force: %d\n", IM.pts.size(), IM.nodes.size(), bad);
  }
  orc_index_free(ot);
  orc_index_free(os);
  std::printf("%ld checks, %ld failures\n%s\n", g_checks, g_fail, g_fail ? "FAILED" : "PASSED");
  return g_fail ? 1 : 0;
}
