// search_host_test.cpp — the per-thread search kernels (pcl_b200/csrc/search_kernels.cuh: k_knn<K> for every compiled
// list size, k_knn_any, k_knn_stats, k_radius_count / k_radius_fill, k_normals<K>) compiled for the HOST and run, one
// emulated 128-thread block after the other, against brute force under the library's own distance expression and
// (d2, original index) order; normals against the facade's host computePointNormal on the brute-force list, bit for bit.
// CPU only, test infrastructure.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"


static inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }

#include "../../pcl_b200/csrc/search_kernels.cuh"

#include <pcl/features/normal_3d.h>
#include <pcl/point_types.h>

// the fixed seed of the committed test, or PCLB_TEST_SEED for a fuzz run (tools/dev/fuzz_host_tests.sh)
static void brute_all(const std::vector<float>& xyz, const float q[3], std::vector<std::pair<float, int>>& all)
{
  const int n = static_cast<int>(xyz.size() / 3);
  all.resize(n);
  for (int i = 0; i < n; ++i) all[i] = {dist2_rn(q[0], q[1], q[2], xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]), i};
  std::sort(all.begin(), all.end());
}

// runs `kernel(block)` for every block of 128 threads that covers nq queries
template <typename F> static void for_blocks(std::size_t nq, F kernel)
{
  blockDim.x = 128;
  const unsigned nblocks = static_cast<unsigned>((nq + 127) / 128);
  gridDim.x = nblocks;
  for (unsigned b = 0; b < nblocks; ++b) {
    blockIdx_storage.x = b;
    warp_emu::run_block(128, kernel);
  }
  blockIdx_storage.x = 0;
  gridDim.x = 1;
}

template <int K> static void knn_fixed(const char* name, const HostIndex& I, const std::vector<float4>& q, int k_out, float init_bound)
{
  const std::size_t nq = q.size();
  std::vector<int32_t> oi(nq * k_out, -7);
  std::vector<float> od(nq * k_out, -7.f);
  int d_error = 0;
  for_blocks(nq, [&] { k_knn<K>(I.nodes.data(), I.pts.data(), I.root, q.data(), nq, k_out, init_bound, oi.data(), od.data(), &d_error); });
  std::vector<std::pair<float, int>> all;
  int bad = 0;
  for (std::size_t i = 0; i < nq; ++i) {
    const float qq[3] = {q[i].x, q[i].y, q[i].z};
    if (!(std::isfinite(qq[0]) && std::isfinite(qq[1]) && std::isfinite(qq[2]))) { bad += !(oi[i * k_out] == -1 && std::isinf(od[i * k_out])); continue; }
    brute_all(I.xyz, qq, all);
    for (int j = 0; j < k_out; ++j) {
      // a finite init_bound acts as a closed radius: d2 <= bound enters the fresh list (the tie rule against the empty
      // entry), which is why the radius search with max_nn passes the largest float below r^2
      const bool have = j < (int)all.size() && all[j].first <= init_bound;
      if (have ? !(oi[i * k_out + j] == all[j].second && od[i * k_out + j] == all[j].first) : !(oi[i * k_out + j] == -1 && std::isinf(od[i * k_out + j]))) { ++bad; break; }
    }
  }
  CHECK(bad == 0 && d_error == 0, "%s k_knn<%d> (k_out %d): %d rows differ from brute force", name, K, k_out, bad);
}

static void run_scene(const char* name, const std::vector<float>& xyz, const std::vector<float>& queries)
{
  HostIndex I;
  build_index(I, xyz, 0);
  const std::size_t nq = queries.size() / 3;
  std::vector<float4> q(nq);
  for (std::size_t i = 0; i < nq; ++i) q[i] = make_float4(queries[3 * i], queries[3 * i + 1], queries[3 * i + 2], __int_as_float((int)i));
  const float inf = INFINITY;
  knn_fixed<1>(name, I, q, 1, inf);
  knn_fixed<2>(name, I, q, 2, inf);
  knn_fixed<4>(name, I, q, 3, inf);
  knn_fixed<8>(name, I, q, 7, inf);
  knn_fixed<10>(name, I, q, 10, inf);
  knn_fixed<16>(name, I, q, 13, inf);
  knn_fixed<20>(name, I, q, 20, inf);
  knn_fixed<32>(name, I, q, 32, inf);
  knn_fixed<8>(name, I, q, 8, 0.02f);   // bounded: radius search with max_nn
  std::vector<std::pair<float, int>> all;
  {  // any k: the list lives in the output rows
    const int k = 45;
    std::vector<int32_t> oi(nq * k, -7);
    std::vector<float> od(nq * k, -7.f);
    int d_error = 0;
    for_blocks(nq, [&] { k_knn_any(I.nodes.data(), I.pts.data(), I.root, q.data(), nq, k, inf, oi.data(), od.data(), &d_error); });
    int bad = 0;
    for (std::size_t i = 0; i < nq; ++i) {
      const float qq[3] = {q[i].x, q[i].y, q[i].z};
      if (!std::isfinite(qq[2])) continue;
      brute_all(I.xyz, qq, all);
      for (int j = 0; j < k; ++j) {
        const bool have = j < (int)all.size();
        if (have ? !(oi[i * k + j] == all[j].second && od[i * k + j] == all[j].first) : !(oi[i * k + j] == -1 && std::isinf(od[i * k + j]))) { ++bad; break; }
      }
    }
    CHECK(bad == 0 && d_error == 0, "%s k_knn_any k = 45: %d rows differ", name, bad);
  }
  {  // radius search: count, exclusive scan, fill; the keys sort to the brute-force list (strict d2 < r2)
    const float r2 = 0.0125f, r2_below = std::nextafter(r2, -INFINITY);
    std::vector<unsigned long long> counts(nq, 0), offsets(nq + 1, 0);
    int d_error = 0;
    for_blocks(nq, [&] { k_radius_count(I.nodes.data(), I.pts.data(), I.root, q.data(), nq, r2, r2_below, counts.data(), &d_error); });
    for (std::size_t i = 0; i < nq; ++i) offsets[i + 1] = offsets[i] + counts[i];
    std::vector<unsigned long long> keys(offsets[nq] + 1, 0);
    for_blocks(nq, [&] { k_radius_fill(I.nodes.data(), I.pts.data(), I.root, q.data(), nq, r2, r2_below, offsets.data(), keys.data(), &d_error); });
    int bad = 0;
    for (std::size_t i = 0; i < nq; ++i) {
      const float qq[3] = {q[i].x, q[i].y, q[i].z};
      if (!std::isfinite(qq[2])) { bad += counts[i] != 0; continue; }
      brute_all(I.xyz, qq, all);
      std::size_t want = 0;
      while (want < all.size() && all[want].first < r2) ++want;
      if (counts[i] != want) { ++bad; continue; }
      std::vector<unsigned long long> got(keys.begin() + offsets[i], keys.begin() + offsets[i + 1]);
      std::sort(got.begin(), got.end());
      for (std::size_t j = 0; j < want; ++j)
        if (got[j] != (((unsigned long long)__float_as_uint(all[j].first) << 32) | (unsigned)all[j].second)) { ++bad; break; }
    }
    CHECK(bad == 0 && d_error == 0, "%s radius count / fill: %d lists differ", name, bad);
  }
  {  // k-NN statistics of the outlier filters
    const int k = 9;
    std::vector<float> mean(nq, -1.f), kth(nq, -1.f);
    int d_error = 0;
    for_blocks(nq, [&] { k_knn_stats<10>(I.nodes.data(), I.pts.data(), I.root, q.data(), nq, k, mean.data(), kth.data(), &d_error); });
    int bad = 0;
    for (std::size_t i = 0; i < nq; ++i) {
      const float qq[3] = {q[i].x, q[i].y, q[i].z};
      if (!std::isfinite(qq[2])) { bad += !(mean[i] == 0.f && std::isinf(kth[i])); continue; }
      brute_all(I.xyz, qq, all);
      const int have = std::min<int>(k, (int)all.size());
      double sum = 0.0;
      for (int j = 1; j < have; ++j) sum += std::sqrt((double)all[j].first);
      const float m = have > 1 ? (float)(sum / (double)(have - 1)) : 0.f;
      const float kk = have == k ? all[k - 1].first : INFINITY;
      if (!(mean[i] == m && kth[i] == kk)) ++bad;
    }
    CHECK(bad == 0 && d_error == 0, "%s k_knn_stats: %d queries differ", name, bad);
  }
  {  // per-thread normals kernel against the host computePointNormal + flip on the brute-force list
    const int k = 10;
    std::vector<float4> out(nq, make_float4(-9.f, -9.f, -9.f, -9.f));
    int d_error = 0, not_dense = 0;
    const float vp[3] = {0.3f, 0.7f, 4.f};
    for_blocks(nq, [&] { k_normals<10>(I.nodes.data(), I.pts.data(), I.root, q.data(), nq, k, vp[0], vp[1], vp[2], out.data(), &not_dense, &d_error); });
    pcl::PointCloud<pcl::PointXYZ> cloud;
    for (std::size_t i = 0; i < I.xyz.size() / 3; ++i) cloud.emplace_back(I.xyz[3 * i], I.xyz[3 * i + 1], I.xyz[3 * i + 2]);
    int bad = 0;
    for (std::size_t i = 0; i < nq; ++i) {
      const float qq[3] = {q[i].x, q[i].y, q[i].z};
      if (!std::isfinite(qq[2])) { bad += !std::isnan(out[i].x); continue; }
      brute_all(I.xyz, qq, all);
      const int have = std::min<int>(k, (int)all.size());
      if (have < 3) { bad += !std::isnan(out[i].x); continue; }
      pcl::Indices idx;
      for (int j = 0; j < have; ++j) idx.push_back(all[j].second);
      Eigen::Vector4f plane;
      float curv = 0.f;
      pcl::computePointNormal(cloud, idx, plane, curv);
      float nx = plane[0], ny = plane[1], nz = plane[2];
      pcl::flipNormalTowardsViewpoint(pcl::PointXYZ(qq[0], qq[1], qq[2]), vp[0], vp[1], vp[2], nx, ny, nz);
      const float4 g = out[i];
      auto same = [](float a, float b) { return std::memcmp(&a, &b, 4) == 0 || (std::isnan(a) && std::isnan(b)); };
      if (!(same(g.x, nx) && same(g.y, ny) && same(g.z, nz) && same(g.w, curv))) ++bad;
    }
    CHECK(bad == 0 && d_error == 0, "%s k_normals<10>: %d normals differ from the host computePointNormal", name, bad);
  }
  {  // the list-based forms: statistics and normals from materialised k-NN rows (k > 32), normals from the radius search's
     // sorted (d2, index) keys (NormalEstimation::setRadiusSearch)
    const int k = 45;
    const float vp[3] = {0.3f, 0.7f, 4.f};
    std::vector<int32_t> pos_of_orig(I.xyz.size() / 3, -1);
    for (std::size_t p = 0; p < I.pts.size(); ++p) { const int o = __float_as_int(I.pts[p].w); if (o != kSentinelIndex) pos_of_orig[o] = (int32_t)p; }
    std::vector<int32_t> li(nq * k, -7);
    std::vector<float> ld(nq * k, -7.f);
    int d_error = 0, nd_lists = 0, nd_csr = 0;
    for_blocks(nq, [&] { k_knn_any(I.nodes.data(), I.pts.data(), I.root, q.data(), nq, k, inf, li.data(), ld.data(), &d_error); });
    std::vector<float> mean(nq, -1.f), kth(nq, -1.f);
    for_blocks(nq, [&] { k_stats_from_lists(q.data(), nq, k, li.data(), ld.data(), mean.data(), kth.data()); });
    std::vector<float4> out_l(nq, make_float4(-9.f, -9.f, -9.f, -9.f)), out_c(nq, make_float4(-9.f, -9.f, -9.f, -9.f));
    for_blocks(nq, [&] { k_normals_from_lists(I.pts.data(), pos_of_orig.data(), q.data(), nq, k, li.data(), 0, vp[0], vp[1], vp[2], out_l.data(), &nd_lists); });
    const float r2 = 0.0125f, r2_below = std::nextafter(r2, -INFINITY);
    std::vector<unsigned long long> counts(nq, 0), offsets(nq + 1, 0);
    for_blocks(nq, [&] { k_radius_count(I.nodes.data(), I.pts.data(), I.root, q.data(), nq, r2, r2_below, counts.data(), &d_error); });
    for (std::size_t i = 0; i < nq; ++i) offsets[i + 1] = offsets[i] + counts[i];
    std::vector<unsigned long long> keys(offsets[nq] + 1, 0);
    for_blocks(nq, [&] { k_radius_fill(I.nodes.data(), I.pts.data(), I.root, q.data(), nq, r2, r2_below, offsets.data(), keys.data(), &d_error); });
    for (std::size_t i = 0; i < nq; ++i) std::sort(keys.begin() + offsets[i], keys.begin() + offsets[i + 1]);   // cub::DeviceSegmentedSort in the driver
    for_blocks(nq, [&] { k_normals_from_csr(I.pts.data(), pos_of_orig.data(), q.data(), nq, offsets.data(), keys.data(), vp[0], vp[1], vp[2], out_c.data(), &nd_csr); });
    pcl::PointCloud<pcl::PointXYZ> cloud;
    for (std::size_t i = 0; i < I.xyz.size() / 3; ++i) cloud.emplace_back(I.xyz[3 * i], I.xyz[3 * i + 1], I.xyz[3 * i + 2]);
    auto same = [](float a, float b) { return std::memcmp(&a, &b, 4) == 0 || (std::isnan(a) && std::isnan(b)); };
    auto host_normal = [&](const float* qq, int have, float4& r) {
      if (have < 3) { r = make_float4(NAN, NAN, NAN, NAN); return; }
      pcl::Indices idx;
      for (int j = 0; j < have; ++j) idx.push_back(all[j].second);
      Eigen::Vector4f plane;
      float curv = 0.f;
      pcl::computePointNormal(cloud, idx, plane, curv);
      float nx = plane[0], ny = plane[1], nz = plane[2];
      pcl::flipNormalTowardsViewpoint(pcl::PointXYZ(qq[0], qq[1], qq[2]), vp[0], vp[1], vp[2], nx, ny, nz);
      r = make_float4(nx, ny, nz, curv);
    };
    int bad_stats = 0, bad_lists = 0, bad_csr = 0;
    for (std::size_t i = 0; i < nq; ++i) {
      const float qq[3] = {q[i].x, q[i].y, q[i].z};
      if (!std::isfinite(qq[2])) { bad_stats += !(mean[i] == 0.f && std::isinf(kth[i])); bad_lists += !std::isnan(out_l[i].x); bad_csr += !std::isnan(out_c[i].x); continue; }
      brute_all(I.xyz, qq, all);
      const int have = std::min<int>(k, (int)all.size());
      double sum = 0.0;
      for (int j = 1; j < have; ++j) sum += std::sqrt((double)all[j].first);
      const float m = have > 1 ? (float)(sum / (double)(have - 1)) : 0.f;
      if (!(mean[i] == m && kth[i] == (have == k ? all[k - 1].first : INFINITY))) ++bad_stats;
      float4 w;
      host_normal(qq, have, w);
      if (!(same(out_l[i].x, w.x) && same(out_l[i].y, w.y) && same(out_l[i].z, w.z) && same(out_l[i].w, w.w))) ++bad_lists;
      int in_ball = 0;
      while (in_ball < (int)all.size() && all[in_ball].first < r2) ++in_ball;
      host_normal(qq, in_ball, w);
      if (!(same(out_c[i].x, w.x) && same(out_c[i].y, w.y) && same(out_c[i].z, w.z) && same(out_c[i].w, w.w))) ++bad_csr;
    }
    CHECK(bad_stats == 0 && bad_lists == 0 && bad_csr == 0 && d_error == 0, "%s list-based forms: %d statistics, %d k-NN-list normals, %d radius normals differ", name, bad_stats,
          bad_lists, bad_csr);
  }
  std::printf("%-26s %6zu points %5zu queries: k_knn<1..32>, k_knn_any, radius, stats, normals, list-based stats / normals (k-NN rows, radius keys); ok so far: %ld checks, %ld failures\n", name, xyz.size() / 3, nq,
              g_checks, g_fail);
}

int main(int argc, char** argv)
{
  const int scale = argc > 1 ? std::atoi(argv[1]) : 1;
  std::mt19937 rng(test_seed(31337));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::normal_distribution<float> N(0.f, 1.f);
  auto cloud = [&](int n, auto gen) { std::vector<float> v; v.reserve(3 * n); for (int i = 0; i < n; ++i) { float p[3]; gen(i, p); v.insert(v.end(), p, p + 3); } return v; };
  auto queries_of = [&](const std::vector<float>& pts, int n_self, int n_off, int n_far) {
    std::vector<float> q;
    const int n = static_cast<int>(pts.size() / 3);
    for (int i = 0; i < n_self; ++i) { const int j = static_cast<int>(rng() % n); q.insert(q.end(), pts.begin() + 3 * j, pts.begin() + 3 * j + 3); }
    for (int i = 0; i < n_off; ++i) { const int j = static_cast<int>(rng() % n); for (int d = 0; d < 3; ++d) q.push_back(pts[3 * j + d] + 0.02f * N(rng)); }
    for (int i = 0; i < n_far; ++i) for (int d = 0; d < 3; ++d) q.push_back(3.f * U(rng) - 1.f);
    if (q.size() >= 12) q[3 * 3 + 2] = std::numeric_limits<float>::quiet_NaN();   // one non-finite query
    return q;
  };
  const auto vol = cloud(3000 * scale, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); });
  run_scene("uniform volume", vol, queries_of(vol, 60 * scale, 50 * scale, 18));
  const auto surf = cloud(4000 * scale, [&](int, float* p) { p[0] = 2.f * U(rng); p[1] = 2.f * U(rng); p[2] = 0.2f * std::sin(3.f * p[0]) + 0.001f * N(rng); });
  run_scene("surface", surf, queries_of(surf, 60 * scale, 50 * scale, 18));
  std::vector<float> lat;
  for (int x = 0; x < 11; ++x) for (int y = 0; y < 11; ++y) for (int z = 0; z < 11; ++z) { lat.push_back(0.1f * x); lat.push_back(0.1f * y); lat.push_back(0.1f * z); }
  run_scene("lattice, exact ties", lat, queries_of(lat, 60 * scale, 40 * scale, 28));
  std::vector<float> base = cloud(150, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); }), dup;
  for (int rep = 0; rep < 12; ++rep) dup.insert(dup.end(), base.begin(), base.end());
  run_scene("duplicates x12", dup, queries_of(base, 60 * scale, 40 * scale, 28));
  const auto few = cloud(7, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); });
  run_scene("seven points", few, queries_of(few, 7, 40, 17));
  std::printf("%ld checks, %ld failures\n%s\n", g_checks, g_fail, g_fail ? "FAILED" : "PASSED");
  return g_fail ? 1 : 0;
}
