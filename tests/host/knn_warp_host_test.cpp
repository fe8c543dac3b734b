// knn_warp_host_test.cpp — the warp-per-query k-NN kernel (pcl_b200/csrc/knn_warp.cuh: k_knn_warp, warp_sort32,
// warp_merge32, the ranked insertion, the certification rule, the shared-leaf handling) compiled for the HOST and run on
// an emulated warp (tests/host/warp_emu.h: 32 fibers in lock step, every *_sync primitive a rendezvous) against brute
// force.  CPU only, test infrastructure.  Every row the kernel certifies must equal the k smallest (d2, original index)
// pairs exactly; rows it hands to the per-thread fix-up (redo flag) are counted and must stay a minority on sensible
// start levels.  Start levels are varied on purpose — also far too fine ones, where leaves span several of the gathered
// cells (the case that hid a pruning bug on the device until every one of 10 M rows was compared).
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#include "host_index.h"
#include "check.h"


#include "../../pcl_b200/csrc/knn_warp.cuh"

#include <pcl/features/normal_3d.h>
#include <pcl/point_types.h>

// the fixed seed of the committed test, or PCLB_TEST_SEED for a fuzz run (tools/dev/fuzz_host_tests.sh)
static void brute_knn(const std::vector<float>& xyz, const float q[3], int k, std::vector<int>& idx, std::vector<float>& d2)
{
  const int n = static_cast<int>(xyz.size() / 3);
  std::vector<std::pair<float, int>> all(n);
  for (int i = 0; i < n; ++i) all[i] = {dist2_rn(q[0], q[1], q[2], xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]), i};
  std::partial_sort(all.begin(), all.begin() + std::min(k, n), all.end());
  idx.clear(); d2.clear();
  for (int j = 0; j < std::min(k, n); ++j) { idx.push_back(all[j].second); d2.push_back(all[j].first); }
}

static void run_scene(const char* name, const std::vector<float>& xyz, const std::vector<float>& queries, int k, int bmax, int b_start,
                      float r_first, double max_redo_fraction)
{
  HostIndex I;
  build_index(I, xyz, bmax);
  if (I.node_leaves.size() < I.nodes.size()) I.node_leaves.resize(I.nodes.size());
  const TreeView T = I.view(true);
  b_start = std::min(b_start, I.bmax);   // (an index built by the device kernels chooses its own finest level)
  if (b_start < 1) { std::printf("%-34s skipped: this index has no cell table\n", name); return; }
  const std::size_t nq = queries.size() / 3;
  std::vector<float4> q(nq);
  for (std::size_t i = 0; i < nq; ++i) q[i] = make_float4(queries[3 * i], queries[3 * i + 1], queries[3 * i + 2], __int_as_float(static_cast<int>(i)));
  std::vector<int32_t> out_idx(nq * k, -7);
  std::vector<float> out_d2(nq * k, -7.f);
  std::vector<unsigned char> redo(nq, 0);
  blockDim.x = 32;
  const long prims = warp_emu::run_warp([&] {
    k_knn_warp<false>(T, I.node_leaves.data(), b_start, r_first, q.data(), nq, k, out_idx.data(), out_d2.data(), 0.f, 0.f, 0.f, nullptr,
                      nullptr, redo.data());
  });
  std::size_t n_redo = 0;
  std::vector<int> bi;
  std::vector<float> bd;
  for (std::size_t i = 0; i < nq; ++i) {
    if (redo[i]) { ++n_redo; continue; }
    if (!(std::isfinite(q[i].x) && std::isfinite(q[i].y) && std::isfinite(q[i].z))) {
      CHECK(out_idx[i * k] == -1 && std::isinf(out_d2[i * k]), "%s q%zu: a non-finite query must give an empty row", name, i);
      continue;
    }
    brute_knn(xyz, &queries[3 * i], k, bi, bd);
    bool same = static_cast<int>(bi.size()) == k;
    for (int j = 0; same && j < k; ++j) same = out_idx[i * k + j] == bi[j] && out_d2[i * k + j] == bd[j];
    if (!same) {
      int j = 0;
      while (j < k && j < static_cast<int>(bi.size()) && out_idx[i * k + j] == bi[j] && out_d2[i * k + j] == bd[j]) ++j;
      CHECK(same, "%s q%zu (k %d, start level %d): row differs at rank %d: got (%g, %d) want (%g, %d)", name, i, k, b_start, j,
            (double)out_d2[i * k + j], out_idx[i * k + j], j < (int)bd.size() ? (double)bd[j] : -1.0, j < (int)bi.size() ? bi[j] : -1);
    }
    else
      ++g_checks;
  }
  CHECK(static_cast<double>(n_redo) <= max_redo_fraction * static_cast<double>(nq), "%s: %zu of %zu rows handed to the fix-up", name, n_redo, nq);
  std::printf("%-34s %6zu points %5zu queries k %2d  level %d r_first %-8g  certified %5zu  redo %4zu  %7ld warp primitives; ok so far: %ld checks, %ld failures\n",
              name, xyz.size() / 3, nq, k, b_start, (double)r_first, nq - n_redo, n_redo, prims, g_checks, g_fail);
}

// The NORMALS instantiation: the neighbour list stays in the warp, lane t folds query t's k neighbours in list order into
// the single-pass moments and solves the plane.  Compared bit for bit with the facade's host-side computePointNormal +
// flipNormalTowardsViewpoint on the brute-force list (those host functions are themselves pinned to the oracle and the
// reference's golden values by tests/test_facade_host.py); both sides use this machine's libm here.
static void run_normals(const char* name, const std::vector<float>& xyz, const std::vector<float>& queries, int k, int bmax, int b_start)
{
  HostIndex I;
  build_index(I, xyz, bmax);
  if (I.node_leaves.size() < I.nodes.size()) I.node_leaves.resize(I.nodes.size());
  const TreeView T = I.view(true);
  b_start = std::min(b_start, I.bmax);
  if (b_start < 1) { std::printf("%-34s skipped: this index has no cell table\n", name); return; }
  const std::size_t nq = queries.size() / 3;
  std::vector<float4> q(nq), out_n(nq, make_float4(-9.f, -9.f, -9.f, -9.f));
  for (std::size_t i = 0; i < nq; ++i) q[i] = make_float4(queries[3 * i], queries[3 * i + 1], queries[3 * i + 2], __int_as_float(static_cast<int>(i)));
  std::vector<unsigned char> redo(nq, 0);
  int not_dense = 0;
  const float vp[3] = {0.4f, 0.6f, 5.f};
  blockDim.x = 32;
  warp_emu::run_warp([&] {
    k_knn_warp<true>(T, I.node_leaves.data(), b_start, 0.f, q.data(), nq, k, nullptr, nullptr, vp[0], vp[1], vp[2], out_n.data(), &not_dense,
                     redo.data());
  });
  pcl::PointCloud<pcl::PointXYZ> cloud;
  for (std::size_t i = 0; i < xyz.size() / 3; ++i) cloud.emplace_back(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
  std::vector<int> bi;
  std::vector<float> bd;
  std::size_t n_redo = 0;
  for (std::size_t i = 0; i < nq; ++i) {
    if (redo[i]) { ++n_redo; continue; }
    brute_knn(xyz, &queries[3 * i], k, bi, bd);
    pcl::Indices idx(bi.begin(), bi.end());
    Eigen::Vector4f plane;
    float curv = 0.f;
    pcl::computePointNormal(cloud, idx, plane, curv);
    float nx = plane[0], ny = plane[1], nz = plane[2];
    pcl::flipNormalTowardsViewpoint(pcl::PointXYZ(queries[3 * i], queries[3 * i + 1], queries[3 * i + 2]), vp[0], vp[1], vp[2], nx, ny, nz);
    const float4 g = out_n[i];
    CHECK(std::memcmp(&g.x, &nx, 4) == 0 && std::memcmp(&g.y, &ny, 4) == 0 && std::memcmp(&g.z, &nz, 4) == 0 && std::memcmp(&g.w, &curv, 4) == 0,
          "%s q%zu: normal (%g %g %g | %g) want (%g %g %g | %g)", name, i, (double)g.x, (double)g.y, (double)g.z, (double)g.w, (double)nx, (double)ny,
          (double)nz, (double)curv);
  }
  std::printf("%-34s %6zu points %5zu queries k %2d  level %d: %zu normals compared bit for bit, %zu redo; ok so far: %ld checks, %ld failures\n", name,
              xyz.size() / 3, nq, k, b_start, nq - n_redo, n_redo, g_checks, g_fail);
}

int main(int argc, char** argv)
{
  const int scale = argc > 1 ? std::atoi(argv[1]) : 1;
  std::mt19937 rng(test_seed(424242));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::normal_distribution<float> N(0.f, 1.f);
  auto cloud = [&](int n, auto gen) { std::vector<float> v; v.reserve(3 * n); for (int i = 0; i < n; ++i) { float p[3]; gen(i, p); v.insert(v.end(), p, p + 3); } return v; };
  auto self_and_off = [&](const std::vector<float>& pts, int n_self, int n_off) {
    std::vector<float> q;
    const int n = static_cast<int>(pts.size() / 3);
    for (int i = 0; i < n_self; ++i) { const int j = static_cast<int>(rng() % n); q.insert(q.end(), pts.begin() + 3 * j, pts.begin() + 3 * j + 3); }
    for (int i = 0; i < n_off; ++i) { const int j = static_cast<int>(rng() % n); for (int d = 0; d < 3; ++d) q.push_back(pts[3 * j + d] + 0.01f * N(rng)); }
    return q;
  };
  {
    // a 2 x 2 sheet, ~6000 points: level 5 cells (1/32 of the frame) hold ~6 points, level 4 ~23, level 3 ~94
    const auto sheet = cloud(6000 * scale, [&](int, float* p) { p[0] = 2.f * U(rng); p[1] = 2.f * U(rng); p[2] = 0.2f * std::sin(3.f * p[0]) * std::cos(2.f * p[1]) + 0.001f * N(rng); });
    const auto q = self_and_off(sheet, 192 * scale, 64 * scale);
    run_scene("sheet, sensible level", sheet, q, 16, 6, 4, 0.f, 0.5);
    run_scene("sheet, sized first ball", sheet, q, 16, 6, 3, 0.05f, 0.5);
    run_scene("sheet, k 32", sheet, q, 32, 6, 3, 0.f, 0.5);
    run_scene("sheet, k 12, too fine a level", sheet, q, 12, 6, 6, 0.f, 1.0);      // leaves span several gathered cells; several attempts per row
    run_scene("sheet, k 20, finest level", sheet, q, 20, 6, 5, 0.004f, 1.0);
  }
  {
    const auto sheet = cloud(5000 * scale, [&](int, float* p) { p[0] = 2.f * U(rng); p[1] = 2.f * U(rng); p[2] = 0.2f * std::sin(3.f * p[0]) * std::cos(2.f * p[1]) + 0.001f * N(rng); });
    run_normals("normals k 16, sheet", sheet, self_and_off(sheet, 160 * scale, 32 * scale), 16, 6, 4);
    run_normals("normals k 12, sheet, fine level", sheet, self_and_off(sheet, 96 * scale, 0), 12, 6, 5);
    const auto vol = cloud(4000 * scale, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); });
    run_normals("normals k 20, volume", vol, self_and_off(vol, 96 * scale, 32 * scale), 20, 4, 2);
  }
  {
    // dense sheet inside a sparse volume: density changes by orders of magnitude, home cells of off-cloud queries are empty
    std::vector<float> mix = cloud(5000 * scale, [&](int, float* p) { p[0] = 2.f * U(rng); p[1] = 2.f * U(rng); p[2] = 1.f + 0.001f * N(rng); });
    const auto vol = cloud(900 * scale, [&](int, float* p) { p[0] = 2.f * U(rng); p[1] = 2.f * U(rng); p[2] = 2.f * U(rng); });
    mix.insert(mix.end(), vol.begin(), vol.end());
    auto q = self_and_off(mix, 160 * scale, 64 * scale);
    for (int i = 0; i < 32; ++i) { q.push_back(2.4f * U(rng) - 0.2f); q.push_back(2.4f * U(rng) - 0.2f); q.push_back(2.4f * U(rng) - 0.2f); }
    q[3 * 5 + 1] = std::numeric_limits<float>::quiet_NaN();   // a non-finite query: empty row
    run_scene("mixed density", mix, q, 16, 6, 4, 0.f, 0.8);
    run_scene("mixed density, fine level", mix, q, 16, 6, 6, 0.f, 1.0);
    run_scene("mixed density, k 24", mix, q, 24, 6, 5, 0.02f, 1.0);
  }
  {
    // map-scale frames: a 200 m map at 1e5 on the 1/128 m grid of its ulp (exact ties), a frame straddling zero (x - lo
    // rounds), a 1 m cube stretched by one point 1e6 away (every table level holds the cube in one cell)
    const auto map = cloud(4000 * scale, [&](int, float* p) { p[0] = 1e5f + 200.f * U(rng); p[1] = 1e5f + 200.f * U(rng); p[2] = std::round(256.f * std::sin((p[0] - 1e5f) / 15.f)) / 128.f; });
    run_scene("map at 1e5", map, self_and_off(map, 96 * scale, 32 * scale), 16, 6, 4, 0.f, 1.0);
    const auto straddle = cloud(4000 * scale, [&](int, float* p) { p[0] = -3e4f + 6e4f * U(rng); p[1] = 20.f * U(rng); p[2] = 3.f * std::sin(p[0] / 40.f); });
    run_scene("straddling zero", straddle, self_and_off(straddle, 96 * scale, 32 * scale), 24, 6, 5, 0.f, 1.0);
    auto outlier = cloud(3000, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); });
    const auto cube = outlier;
    outlier.insert(outlier.end(), {1e6f, 0.5f, 0.5f});
    run_scene("one outlier 1e6 away", outlier, self_and_off(cube, 32, 16), 16, 6, 4, 0.f, 1.0);
  }
  {
    // exact ties (a lattice) and duplicates: the (d2, index) order decides
    std::vector<float> lat;
    for (int x = 0; x < 14; ++x) for (int y = 0; y < 14; ++y) for (int z = 0; z < 14; ++z) { lat.push_back(0.1f * x); lat.push_back(0.1f * y); lat.push_back(0.1f * z); }
    std::vector<float> q;
    for (int i = 0; i < 96 * scale; ++i) { q.push_back(0.05f * (rng() % 27)); q.push_back(0.05f * (rng() % 27)); q.push_back(0.05f * (rng() % 27)); }
    run_scene("lattice, exact ties", lat, q, 16, 3, 2, 0.f, 0.9);
    run_scene("lattice, exact ties, k 27", lat, q, 27, 3, 1, 0.f, 0.9);
    std::vector<float> base = cloud(300, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); }), dup;
    for (int rep = 0; rep < 5; ++rep) dup.insert(dup.end(), base.begin(), base.end());
    run_scene("duplicates x5", dup, self_and_off(base, 64 * scale, 32 * scale), 16, 3, 2, 0.f, 0.9);
  }
  {
    // The shared-leaf case, constructed: level-3 cells of a unit frame (w = 1/8).  The query sits in cell (3, 2, 2), just
    // below the x = 0.5 boundary — a level-2 boundary, so the four x-neighbour cells belong to ANOTHER level-2 cell, which
    // is sparse enough (<= 8 points) to be a single leaf.  That leaf is returned for cells 3, 5 (and 7) of the 2 x 2 x 2
    // block while cell 1 is empty, and it is kept under lane 3, whose cell is the FARTHER one (the y boundary is 0.4 w
    // away, the z boundary 0.05 w).  The dense home cell fills the buffer and tightens the k-th distance below cell 3's
    // bound before the neighbours are looked at; the leaf's point in cell 5 belongs to the true 16 nearest.  A kernel that
    // prunes the shared leaf by cell 3's bound loses it.
    const float w = 0.125f;
    for (int rep = 0; rep < 6 * scale; ++rep) {
      std::vector<float> pts = {0.f, 0.f, 0.f, 1.f, 1.f, 1.f};
      const float q[3] = {0.5f - 0.05f * w, 0.375f - 0.4f * w, 0.375f - 0.05f * w};
      auto home = [&](float r) {   // a point of the home cell at distance ~r from q (towards the cell's interior)
        const float a = 0.2f + 1.1f * U(rng), b = 0.2f + 1.1f * U(rng);
        pts.push_back(q[0] - r * std::cos(a) * std::cos(b)); pts.push_back(q[1] - r * std::sin(a) * std::cos(b)); pts.push_back(q[2] - r * std::sin(b));
      };
      for (int i = 0; i < 12; ++i) home((0.01f + 0.04f * U(rng)) * w);
      for (int i = 0; i < 34; ++i) home((0.16f + 0.2f * U(rng)) * w);
      // the sparse level-2 cell on the other side of x = 0.5: one point in cell 5 (close), one in cell 3 (far), one in cell 7
      pts.push_back(0.5f + 0.02f * w); pts.push_back(q[1]); pts.push_back(0.375f + (0.02f + 0.02f * U(rng)) * w);
      pts.push_back(0.5f + 0.3f * w); pts.push_back(0.375f + 0.3f * w); pts.push_back(q[2]);
      pts.push_back(0.5f + 0.6f * w); pts.push_back(0.375f + 0.6f * w); pts.push_back(0.375f + 0.6f * w);
      std::vector<float> qs(q, q + 3);
      char name[64];
      std::snprintf(name, sizeof name, "shared leaf, constructed #%d", rep);
      run_scene(name, pts, qs, 16, 3, 3, 0.f, 0.0);
    }
  }
  std::printf("%ld checks, %ld failures\n%s\n", g_checks, g_fail, g_fail ? "FAILED" : "PASSED");
  return g_fail ? 1 : 0;
}
