// lbvh_host_test.cpp — the index BUILD kernels (pcl_b200/csrc/lbvh_kernels.cuh: bounding box, Morton keys, Karras radix
// tree over the points, the cut into cell-aligned leaves, the cell table, refit, packing) compiled for the HOST and run in
// lbvh.cu's sequence (tests/host/device_build.h: std::stable_sort / partial_sum where the driver calls CUB).  CPU only, test
// infrastructure.  Checked on every scene: the invariants the walks rely on —
//   * every finite point sits in exactly one leaf slot with its original index; leaves hold 1..8 points, in Morton order;
//   * each node's two boxes are the exact bounds of its children's points; node_leaves gives each subtree's leaf range;
//   * the cell table: for every level b <= bmax and every indexed point, the look-up of the point's level-b cell returns a
//     subtree that holds ALL points of that cell, and — when it is an internal node — ONLY points of that cell;
// and, on top, the reference host builder of host_index.h must agree on the leaves point for point.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#define PCLB_TEST_DEVICE_BUILD 1
#include "host_index.h"
#include "check.h"


#include <map>
#include <set>

// the fixed seed of the committed test, or PCLB_TEST_SEED for a fuzz run (tools/dev/fuzz_host_tests.sh)
struct Sub { std::vector<int> points; float lo[3], hi[3]; int first_leaf, n_leaves; };

static Sub collect(const HostIndex& I, int ref, int& bad_boxes, int& bad_ranges)
{
  Sub s;
  for (int d = 0; d < 3; ++d) { s.lo[d] = INFINITY; s.hi[d] = -INFINITY; }
  if (ref < 0) {
    const int leaf = ~ref;
    s.first_leaf = leaf; s.n_leaves = 1;
    for (int j = 0; j < kLeafSize; ++j) {
      const float4 p = I.pts[(std::size_t)leaf * kLeafSize + j];
      if (__float_as_int(p.w) == kSentinelIndex) continue;
      s.points.push_back(__float_as_int(p.w));
      const float v[3] = {p.x, p.y, p.z};
      for (int d = 0; d < 3; ++d) { s.lo[d] = std::min(s.lo[d], v[d]); s.hi[d] = std::max(s.hi[d], v[d]); }
    }
    return s;
  }
  const BvhNode& nd = I.nodes[ref];
  Sub a = collect(I, nd.d.x, bad_boxes, bad_ranges), b = collect(I, nd.d.y, bad_boxes, bad_ranges);
  const float alo[3] = {nd.a.x, nd.a.y, nd.a.z}, ahi[3] = {nd.a.w, nd.b.x, nd.b.y}, blo[3] = {nd.b.z, nd.b.w, nd.c.x}, bhi[3] = {nd.c.y, nd.c.z, nd.c.w};
  for (int d = 0; d < 3; ++d)
    if (alo[d] != a.lo[d] || ahi[d] != a.hi[d] || blo[d] != b.lo[d] || bhi[d] != b.hi[d]) ++bad_boxes;
  s.points = a.points;
  s.points.insert(s.points.end(), b.points.begin(), b.points.end());
  for (int d = 0; d < 3; ++d) { s.lo[d] = std::min(a.lo[d], b.lo[d]); s.hi[d] = std::max(a.hi[d], b.hi[d]); }
  s.first_leaf = a.first_leaf;
  s.n_leaves = a.n_leaves + b.n_leaves;
  if (b.first_leaf != a.first_leaf + a.n_leaves) ++bad_ranges;                          // a subtree's leaves are consecutive
  if (I.node_leaves[ref].x != s.first_leaf || I.node_leaves[ref].y != s.n_leaves) ++bad_ranges;
  return s;
}

static void run_scene(const char* name, const std::vector<float>& xyz, bool unique_codes = true)
{
  HostIndex I;
  device_build::build(I, xyz, true);
  const int n = static_cast<int>(xyz.size() / 3);
  // ---- leaves ----
  std::vector<int> seen(n, 0);
  int bad_slots = 0, bad_leaf_sizes = 0, bad_order = 0;
  const std::size_t n_leaves = I.pts.size() / kLeafSize;
  unsigned long long prev_key = 0;
  for (std::size_t l = 0; l < n_leaves; ++l) {
    int cnt = 0;
    bool tail = false;
    for (int j = 0; j < kLeafSize; ++j) {
      const float4 p = I.pts[l * kLeafSize + j];
      const int o = __float_as_int(p.w);
      if (o == kSentinelIndex) { tail = true; if (!std::isinf(p.x)) ++bad_slots; continue; }
      if (tail) ++bad_slots;                                        // points first, padding after
      if (o < 0 || o >= n || p.x != xyz[3 * o] || p.y != xyz[3 * o + 1] || p.z != xyz[3 * o + 2]) { ++bad_slots; continue; }
      ++seen[o];
      ++cnt;
      const unsigned long long key = (expand21(morton_cell(p.z, I.lo[2], I.scale)) << 2) | (expand21(morton_cell(p.y, I.lo[1], I.scale)) << 1) |
                                     expand21(morton_cell(p.x, I.lo[0], I.scale));
      if (key < prev_key) ++bad_order;
      prev_key = key;
    }
    if (cnt < 1 || cnt > kLeafSize) ++bad_leaf_sizes;
  }
  int missing = 0;
  for (int i = 0; i < n; ++i) missing += seen[i] != 1;
  CHECK(bad_slots == 0 && bad_leaf_sizes == 0 && bad_order == 0 && missing == 0, "%s: %d bad slots, %d bad leaf sizes, %d out of Morton order, %d points not exactly once",
        name, bad_slots, bad_leaf_sizes, bad_order, missing);
  // ---- nodes ----
  int bad_boxes = 0, bad_ranges = 0;
  const Sub all = collect(I, I.root, bad_boxes, bad_ranges);
  CHECK(bad_boxes == 0 && bad_ranges == 0 && (int)all.points.size() == n && all.n_leaves == (int)n_leaves, "%s: %d child boxes not exact, %d leaf ranges wrong, %zu points under the root",
        name, bad_boxes, bad_ranges, all.points.size());
  // ---- the reference host builder cuts the same leaves ----
  HostIndex R;
  build_index_reference(R, xyz, 0);
  bool same_leaves = R.pts.size() == I.pts.size();
  for (std::size_t i = 0; same_leaves && i < I.pts.size(); ++i)
    same_leaves = std::memcmp(&R.pts[i], &I.pts[i], sizeof(float4)) == 0 || (std::isinf(R.pts[i].x) && std::isinf(I.pts[i].x));
  // (inside a run of EQUAL codes longer than a leaf the Karras tree cuts by index bits, the reference builder in the middle:
  //  both are valid, so the comparison is made where codes are unique)
  if (unique_codes) CHECK(same_leaves, "%s: the host reference builder and the device kernels cut different leaves", name);
  // ---- cell table ----
  int bad_cells = 0, levels = 0;
  if (I.log2_slots) {
    const TreeView T = I.view(true);
    levels = I.bmax;
    for (int b = 1; b <= I.bmax; ++b) {
      std::map<unsigned, std::vector<int>> cells;   // key -> points of the cell
      for (int i = 0; i < n; ++i) {
        const unsigned cx = morton_cell(xyz[3 * i], I.lo[0], I.scale) >> (21 - b), cy = morton_cell(xyz[3 * i + 1], I.lo[1], I.scale) >> (21 - b),
                       cz = morton_cell(xyz[3 * i + 2], I.lo[2], I.scale) >> (21 - b);
        cells[cell_key(b, cx, cy, cz)].push_back(i);
      }
      for (const auto& kv : cells) {
        const int ref = cell_lookup(T.cells, kv.first);
        if (ref == kDone) { ++bad_cells; continue; }
        int bb = 0, br = 0;
        const Sub s = collect(I, ref, bb, br);
        std::set<int> in(s.points.begin(), s.points.end());
        bool holds_all = true;
        for (int i : kv.second) holds_all = holds_all && in.count(i);
        if (!holds_all) { ++bad_cells; continue; }
        if (ref >= 0 && s.points.size() != kv.second.size()) ++bad_cells;   // an internal node is exactly the cell
      }
      // and no stale entry: a key of an empty cell is absent
      const unsigned probe = cell_key(b, (1u << b) - 1u, 0u, (1u << b) - 1u);
      if (!cells.count(probe) && cell_lookup(T.cells, probe) != kDone) ++bad_cells;
    }
  }
  CHECK(bad_cells == 0, "%s: %d cells of the table are wrong", name, bad_cells);
  std::printf("%-30s %6d points: %5zu leaves, %5zu nodes, cell table levels 1..%d (%zu slots); ok so far: %ld checks, %ld failures\n", name, n, n_leaves,
              I.nodes.size(), levels, I.slots.size(), g_checks, g_fail);
}

int main(int argc, char** argv)
{
  const int scale = argc > 1 ? std::atoi(argv[1]) : 1;
  std::mt19937 rng(test_seed(2718));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::normal_distribution<float> N(0.f, 1.f);
  auto cloud = [&](int n, auto gen) { std::vector<float> v; v.reserve(3 * n); for (int i = 0; i < n; ++i) { float p[3]; gen(i, p); v.insert(v.end(), p, p + 3); } return v; };
  run_scene("uniform volume", cloud(5000 * scale, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); }));
  run_scene("surface", cloud(6000 * scale, [&](int, float* p) { p[0] = 10.f * U(rng); p[1] = 10.f * U(rng); p[2] = 0.5f * std::sin(p[0]) * std::cos(0.7f * p[1]) + 0.002f * N(rng); }));
  run_scene("offset frame", cloud(3000 * scale, [&](int, float* p) { p[0] = 1000.f + 3.f * U(rng); p[1] = -500.f + 3.f * U(rng); p[2] = 20.f + 0.01f * N(rng); }));
  {
    std::vector<float> base = cloud(400, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); }), dup;
    for (int rep = 0; rep < 12; ++rep) dup.insert(dup.end(), base.begin(), base.end());
    run_scene("duplicates x12", dup, false);
  }
  {
    std::vector<float> lat;
    for (int x = 0; x < 13; ++x) for (int y = 0; y < 13; ++y) for (int z = 0; z < 13; ++z) { lat.push_back((float)x); lat.push_back((float)y); lat.push_back((float)z); }
    run_scene("lattice", lat);
  }
  // map-scale frames: a 200 m map at 1e5 on the 1/128 m grid of its ulp, a frame straddling zero, a 1 m cube stretched by
  // one point 1e6 away (runs of equal Morton codes far beyond a leaf)
  run_scene("map at 1e5", cloud(4000 * scale, [&](int, float* p) { p[0] = 1e5f + 200.f * U(rng); p[1] = 1e5f + 200.f * U(rng); p[2] = std::round(256.f * std::sin((p[0] - 1e5f) / 15.f)) / 128.f; }));
  run_scene("straddling zero", cloud(4000 * scale, [&](int, float* p) { p[0] = -3e4f + 6e4f * U(rng); p[1] = 20.f * U(rng); p[2] = 3.f * std::sin(p[0] / 40.f); }));
  {
    auto outlier = cloud(4000 * scale, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); });
    outlier.insert(outlier.end(), {1e6f, 0.5f, 0.5f});
    run_scene("one outlier 1e6 away", outlier, false);
  }
  run_scene("collinear", cloud(1777, [&](int i, float* p) { p[0] = p[1] = p[2] = i / 1776.f; }));
  run_scene("planar, zero extent axis", cloud(3000, [&](int, float* p) { p[0] = U(rng); p[1] = 0.25f; p[2] = U(rng); }));
  run_scene("mixed density", cloud(4000 * scale, [&](int i, float* p) { p[0] = 2.f * U(rng); p[1] = 2.f * U(rng); p[2] = (i % 7) ? 1.f + 0.001f * N(rng) : 2.f * U(rng); }));
  run_scene("just above one leaf", cloud(9, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); }));
  run_scene("one leaf", cloud(8, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); }));
  run_scene("below the table threshold", cloud(255, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); }));
  run_scene("all the same point", cloud(300, [&](int, float* p) { p[0] = 0.25f; p[1] = 0.25f; p[2] = 0.25f; }), false);
  std::printf("%ld checks, %ld failures\n%s\n", g_checks, g_fail, g_fail ? "FAILED" : "PASSED");
  return g_fail ? 1 : 0;
}
