// traverse_host_test.cpp — the DEVICE traversal header (pcl_b200/csrc/traverse.cuh: walk, nearest1, the cell-table
// look-ups and their conservative bounds) compiled for the host and run against brute force.
//
// Test infrastructure, CPU only: g++ sees the same source the kernels are built from; the CUDA intrinsics it uses are
// supplied below with the same rounding (round-to-nearest without contraction, directed rounding through <cfenv>).  The
// index (Morton-ordered padded leaves, 64-byte nodes holding both children's boxes, the (level, cell) -> subtree hash
// table) is built here on the host to the invariants lbvh.cu documents:
//   * leaves are whole radix-tree cells of <= 8 points; a node's two boxes bound its children's points exactly;
//   * the table maps every occupied cell of levels 1..bmax to the deepest node / leaf that holds all its points
//     (prefix_len(parent) < 3b <= prefix_len(child); a leaf that spans several level-b cells is entered for each).
// What is checked: for every query, with and without a seed, with and without the TRACK visitor and an inflated ball,
// nearest1 returns exactly the brute-force minimum of (d2, original index) under the library's distance expression and
// gate; TRACK's lower bound never exceeds the true second-nearest distance.  Scenes: uniform volume, a thin surface,
// duplicates beyond a leaf, a lattice full of exact ties, a degenerate line, far-away queries, tiny clouds.
#include "host_index.h"
#include "check.h"


// the fixed seed of the committed test, or PCLB_TEST_SEED for a fuzz run (tools/dev/fuzz_host_tests.sh)
static void run_scene(const char* name, const std::vector<float>& xyz, const std::vector<float>& queries, float gate, int bmax)
{
  const bool quiet = std::strncmp(name, "small cloud", 11) == 0;
  HostIndex I;
  build_index(I, xyz, bmax);
  const int nq = static_cast<int>(queries.size() / 3);
  const int n = static_cast<int>(xyz.size() / 3);
  std::vector<int> pos_of(n, -1);
  for (std::size_t p = 0; p < I.pts.size(); ++p) {
    const int o = __float_as_int(I.pts[p].w);
    if (o != kSentinelIndex) pos_of[o] = static_cast<int>(p);
  }
  std::mt19937 rng(test_seed(99));
  const float inf = INFINITY;
  for (int with_table = 0; with_table < 2; ++with_table) {
    const TreeView T = I.view(with_table != 0);
    for (int i = 0; i < nq; ++i) {
      const float* q = &queries[3 * i];
      const Truth t = brute(xyz, q, gate);
      for (int variant = 0; variant < 4; ++variant) {
        // 0: no seed   1: seed = the true answer   2: seed = a random point (a "previous match" after a large motion)
        // 3: TRACK visitor, inflated ball, random seed
        int seed = -1;
        if (variant == 1 && t.idx != kSentinelIndex) seed = pos_of[t.idx];
        if (variant >= 2) seed = pos_of[static_cast<int>(rng() % n)];
        WalkStats ws;
        bool ok;
        float best;
        int best_idx, best_pos;
        float lb2 = 0.f;
        if (variant < 3) {
          Nearest1T<false> v{q[0], q[1], q[2], gate, kSentinelIndex, -1, inf, inf, inf};
          ok = nearest1<false>(T, q[0], q[1], q[2], v, seed, 1.00001f, ws);
          best = v.best; best_idx = v.best_idx; best_pos = v.best_pos;
        }
        else {
          Nearest1T<true> v{q[0], q[1], q[2], gate, kSentinelIndex, -1, inf, inf, inf};
          ok = nearest1<true>(T, q[0], q[1], q[2], v, seed, 2.5f, ws);
          best = v.best; best_idx = v.best_idx; best_pos = v.best_pos;
          lb2 = v.lower_bound2();
        }
        CHECK(ok, "%s q%d v%d stack overflow", name, i, variant);
        if (t.idx == kSentinelIndex) {
          CHECK(best_pos < 0, "%s q%d v%d table%d: found %d beyond the gate", name, i, variant, with_table, best_idx);
          continue;
        }
        CHECK(best_idx == t.idx && best == t.d1, "%s q%d v%d table%d: got (%g, %d) want (%g, %d)", name, i, variant, with_table,
              (double)best, best_idx, (double)t.d1, t.idx);
        CHECK(best_pos >= 0 && __float_as_int(I.pts[best_pos].w) == best_idx, "%s q%d v%d position", name, i, variant);
        if (variant == 3)   // the bound the next iteration's skip test relies on: nothing but the match is closer than it
          CHECK(lb2 <= t.d2nd, "%s q%d table%d: lower bound %g above the true second distance %g", name, i, with_table, (double)lb2, (double)t.d2nd);
      }
    }
  }
  if (!quiet)
    std::printf("%-28s %6d points %6d queries  nodes %6zu leaves %6zu  bmax %d  table entries/slots %zu  ok so far: %ld checks, %ld failures\n",
                name, n, nq, I.nodes.size(), I.pts.size() / kLeafSize, I.bmax, I.slots.size(), g_checks, g_fail);
}

// The temporal-coherence skip of icp.cu: k_search<.., TRACK>, replayed: a query drifts for a number of iterations; every
// iteration either proves by still_nearest that the previous match is still the nearest neighbour (the walk is skipped,
// the bound decays) or searches with the TRACK visitor and stores sqrt(lower_bound2).  Whatever the path, the result must
// be the brute-force nearest neighbour — in particular a skip may never keep a match that stopped being the nearest.
static void run_coherence(const char* name, const std::vector<float>& xyz, int n_queries, float step, float gate, int bmax, std::mt19937& rng)
{
  HostIndex I;
  build_index(I, xyz, bmax);
  const TreeView T = I.view(true);
  const int n = static_cast<int>(xyz.size() / 3);
  std::normal_distribution<float> N(0.f, 1.f);
  const float inf = INFINITY;
  long skips = 0, searches = 0;
  for (int qi = 0; qi < n_queries; ++qi) {
    const int j = static_cast<int>(rng() % n);
    float p[3] = {xyz[3 * j] + 0.02f * N(rng), xyz[3 * j + 1] + 0.02f * N(rng), xyz[3 * j + 2] + 0.02f * N(rng)};
    int seed = -1;          // Match::pos of the previous iteration (-1: none)
    float prev_d2 = 0.f, lb = 0.f;
    float s = step;
    for (int it = 0; it < 14; ++it) {
      const float old[3] = {p[0], p[1], p[2]};
      for (int d = 0; d < 3; ++d) p[d] += s * N(rng);   // the increment of this iteration, shrinking like a converging ICP
      s *= 0.6f;
      const float delta = std::sqrt(dist2_rn(p[0], p[1], p[2], old[0], old[1], old[2]));
      int pos = -1;
      float d2 = 0.f, nlb = 0.f, lb_out = 0.f;
      if (seed >= 0 && still_nearest(prev_d2, lb, delta, &nlb)) {
        const float4 m = I.pts[seed];
        d2 = dist2_rn(p[0], p[1], p[2], m.x, m.y, m.z);
        pos = seed;   // (beyond the gate the kernel keeps the seed but marks the pair as not accepted)
        lb_out = nlb;
        ++skips;
      }
      else {
        Nearest1T<true> v{p[0], p[1], p[2], gate, kSentinelIndex, -1, inf, inf, inf};
        WalkStats ws;
        CHECK(nearest1<true>(T, p[0], p[1], p[2], v, seed, kTrackInflate, ws), "%s stack", name);
        if (v.best_pos >= 0) { pos = v.best_pos; d2 = v.best; lb_out = std::sqrt(v.lower_bound2()); }
        ++searches;
      }
      const Truth t = brute(xyz, p, inf);
      if (pos >= 0) {
        const bool accepted = d2 <= gate;
        if (accepted || seed >= 0)
          CHECK(__float_as_int(I.pts[pos].w) == t.idx && d2 == t.d1, "%s q%d it%d: kept (%g, %d), nearest is (%g, %d)%s", name, qi, it, (double)d2,
                __float_as_int(I.pts[pos].w), (double)t.d1, t.idx, seed >= 0 && lb_out == nlb ? " [skipped walk]" : "");
        CHECK(lb_out * lb_out * 0.9999f <= t.d2nd || lb_out == 0.f, "%s q%d it%d: bound %g above the second distance %g", name, qi, it,
              (double)lb_out, (double)std::sqrt(t.d2nd));
      }
      else
        CHECK(!(t.d1 <= gate), "%s q%d it%d: nothing found but %d is inside the gate", name, qi, it, t.idx);
      seed = pos;
      prev_d2 = d2;
      lb = lb_out;
    }
  }
  std::printf("%-28s %6d points %6d drifting queries x 14 iterations: %ld walks skipped, %ld searched; ok so far: %ld checks, %ld failures\n", name, n,
              n_queries, skips, searches, g_checks, g_fail);
}

int main(int argc, char** argv)
{
  const int scale = argc > 1 ? std::atoi(argv[1]) : 1;   // 1: seconds; larger: more points and queries
  std::mt19937 rng(test_seed(20250923));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::normal_distribution<float> N(0.f, 1.f);
  auto cloud = [&](int n, auto gen) { std::vector<float> v; v.reserve(3 * n); for (int i = 0; i < n; ++i) { float p[3]; gen(i, p); v.insert(v.end(), p, p + 3); } return v; };
  auto near_queries = [&](const std::vector<float>& pts, int nq, float jitter, float far_frac) {
    std::vector<float> q;
    const int n = static_cast<int>(pts.size() / 3);
    for (int i = 0; i < nq; ++i) {
      if (U(rng) < far_frac) { for (int d = 0; d < 3; ++d) q.push_back(4.f * U(rng) - 1.5f); continue; }
      const int j = static_cast<int>(rng() % n);
      for (int d = 0; d < 3; ++d) q.push_back(pts[3 * j + d] + jitter * N(rng));
    }
    return q;
  };
  const float no_gate = INFINITY;
  {
    const auto pts = cloud(6000 * scale, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); });
    run_scene("uniform volume", pts, near_queries(pts, 1500 * scale, 0.01f, 0.1f), no_gate, 4);
    run_scene("uniform volume, gate", pts, near_queries(pts, 800 * scale, 0.02f, 0.2f), 0.02f * 0.02f, 4);
    run_scene("uniform volume, bmax 1", pts, near_queries(pts, 400 * scale, 0.05f, 0.1f), no_gate, 1);
  }
  {
    const auto pts = cloud(8000 * scale, [&](int, float* p) { p[0] = 10.f * U(rng); p[1] = 10.f * U(rng); p[2] = 0.5f * std::sin(p[0]) * std::cos(0.7f * p[1]) + 0.002f * N(rng); });
    run_scene("surface", pts, near_queries(pts, 1500 * scale, 0.01f, 0.05f), no_gate, 6);
    run_scene("surface, offset frame", cloud(4000 * scale, [&](int, float* p) { p[0] = 1000.f + 3.f * U(rng); p[1] = -500.f + 3.f * U(rng); p[2] = 20.f + 0.01f * N(rng); }),
              cloud(600 * scale, [&](int, float* p) { p[0] = 1000.f + 3.f * U(rng); p[1] = -500.f + 3.f * U(rng); p[2] = 20.f + 0.05f * N(rng); }), no_gate, 5);
  }
  {  // map-scale frames: a 200 m map at 1e5 on the 1/128 m grid of its ulp (exact ties), a frame straddling zero (x - lo
     // rounds), a 1 m cube stretched by one point 1e6 away (runs of equal Morton codes far beyond a leaf)
    const auto map = cloud(4000 * scale, [&](int, float* p) { p[0] = 1e5f + 200.f * U(rng); p[1] = 1e5f + 200.f * U(rng); p[2] = std::round(256.f * std::sin((p[0] - 1e5f) / 15.f)) / 128.f; });
    run_scene("map at 1e5", map, near_queries(map, 800 * scale, 1.f, 0.05f), no_gate, 6);
    run_scene("map at 1e5, gate", map, near_queries(map, 400 * scale, 2.f, 0.05f), 9.f, 6);
    const auto straddle = cloud(4000 * scale, [&](int, float* p) { p[0] = -3e4f + 6e4f * U(rng); p[1] = 20.f * U(rng); p[2] = 3.f * std::sin(p[0] / 40.f); });
    run_scene("straddling zero", straddle, near_queries(straddle, 800 * scale, 5.f, 0.05f), no_gate, 6);
    auto outlier = cloud(4000 * scale, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); });
    const auto cube = outlier;
    outlier.insert(outlier.end(), {1e6f, 0.5f, 0.5f});
    run_scene("one outlier 1e6 away", outlier, near_queries(cube, 800 * scale, 0.01f, 0.05f), no_gate, 6);
  }
  {
    std::vector<float> base = cloud(400, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); });
    std::vector<float> pts;
    for (int rep = 0; rep < 12; ++rep) pts.insert(pts.end(), base.begin(), base.end());   // every point 12 times: runs of equal codes beyond a leaf
    run_scene("duplicates x12", pts, near_queries(base, 500 * scale, 1e-4f, 0.1f), no_gate, 3);
    std::vector<float> qd(base.begin(), base.begin() + 3 * 200);
    run_scene("duplicates x12, exact hits", pts, qd, no_gate, 3);
  }
  {
    std::vector<float> pts;
    for (int x = 0; x < 13; ++x) for (int y = 0; y < 13; ++y) for (int z = 0; z < 13; ++z) { pts.push_back((float)x); pts.push_back((float)y); pts.push_back((float)z); }
    std::vector<float> q;
    for (int i = 0; i < 600 * scale; ++i) { q.push_back((rng() % 25) * 0.5f); q.push_back((rng() % 25) * 0.5f); q.push_back((rng() % 25) * 0.5f); }   // cell centres and faces: 2-, 4-, 8-way ties
    run_scene("lattice, exact ties", pts, q, no_gate, 3);
  }
  {
    const auto pts = cloud(1777, [&](int i, float* p) { p[0] = p[1] = p[2] = i / 1776.f; });
    run_scene("collinear", pts, near_queries(pts, 500 * scale, 0.01f, 0.2f), no_gate, 5);
    const auto flat = cloud(3000, [&](int, float* p) { p[0] = U(rng); p[1] = 0.25f; p[2] = U(rng); });   // zero extent along y
    run_scene("planar, zero extent axis", flat, near_queries(flat, 500 * scale, 0.01f, 0.2f), no_gate, 5);
  }
  {
    const auto tiny = cloud(5, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); });
    run_scene("five points", tiny, near_queries(tiny, 100, 0.3f, 0.3f), no_gate, 1);
    const auto one = cloud(1, [&](int, float* p) { p[0] = 0.3f; p[1] = 0.2f; p[2] = 0.1f; });
    run_scene("single point", one, near_queries(one, 50, 0.3f, 0.3f), no_gate, 0);
    const auto nine = cloud(9, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); });
    run_scene("nine points", nine, near_queries(nine, 100, 0.3f, 0.3f), no_gate, 1);
  }
  {  // temporal coherence: skipped walks must never change a result
    const auto vol = cloud(5000 * scale, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); });
    run_coherence("coherence, volume", vol, 400 * scale, 0.01f, no_gate, 4, rng);
    run_coherence("coherence, volume, gate", vol, 300 * scale, 0.02f, 0.03f * 0.03f, 4, rng);
    const auto surf = cloud(6000 * scale, [&](int, float* p) { p[0] = 4.f * U(rng); p[1] = 4.f * U(rng); p[2] = 0.3f * std::sin(2.f * p[0]) + 0.001f * N(rng); });
    run_coherence("coherence, surface", surf, 400 * scale, 0.005f, no_gate, 6, rng);
    std::vector<float> lat;
    for (int x = 0; x < 12; ++x) for (int y = 0; y < 12; ++y) for (int z = 0; z < 12; ++z) { lat.push_back(0.1f * x); lat.push_back(0.1f * y); lat.push_back(0.1f * z); }
    run_coherence("coherence, lattice (ties)", lat, 300 * scale, 0.02f, no_gate, 3, rng);
  }
  {  // points and queries ON cell boundaries of a [0, 1]^3 frame (multiples of 1/64, one ulp either side): the places where
     // the fp32 cell bound of cell_gap2 has to be conservative
    std::vector<float> pts = {0.f, 0.f, 0.f, 1.f, 1.f, 1.f};
    auto snap = [&](float v) {
      const float g = std::round(v * 64.f) / 64.f;
      const int k = static_cast<int>(rng() % 3);
      return k == 0 ? g : k == 1 ? std::nextafter(g, 2.f) : std::max(0.f, std::nextafter(g, -1.f));
    };
    for (int i = 0; i < 3000 * scale; ++i) { pts.push_back(std::min(1.f, snap(U(rng)))); pts.push_back(std::min(1.f, snap(U(rng)))); pts.push_back(std::min(1.f, snap(U(rng)))); }
    std::vector<float> q;
    for (int i = 0; i < 1200 * scale; ++i) { q.push_back(snap(U(rng))); q.push_back(snap(U(rng))); q.push_back(snap(U(rng))); }
    run_scene("on cell boundaries", pts, q, no_gate, 6);
  }
  for (int rep = 0; rep < 150 * scale; ++rep) {   // many small random clouds: every tree shape around the leaf size, every bmax
    const int n = 1 + static_cast<int>(rng() % 120);
    const int shape = static_cast<int>(rng() % 3);
    const auto pts = cloud(n, [&](int, float* p) {
      p[0] = U(rng); p[1] = shape == 1 ? 0.5f : U(rng); p[2] = shape == 2 ? std::floor(4.f * U(rng)) / 4.f : U(rng);
    });
    char name[64];
    std::snprintf(name, sizeof name, "small cloud #%d", rep);
    const long before = g_fail;
    const int bmax = n >= 4 ? 1 + static_cast<int>(rng() % 4) : 0;
    run_scene(name, pts, near_queries(pts, 40, 0.2f, 0.3f), rep % 3 == 0 ? 0.05f : no_gate, bmax);
    if (g_fail != before) std::printf("  ^ failure in %s (n = %d, shape %d, bmax %d)\n", name, n, shape, bmax);
  }
  std::printf("%ld checks, %ld failures\n%s\n", g_checks, g_fail, g_fail ? "FAILED" : "PASSED");
  return g_fail ? 1 : 0;
}
