// lbvh_batch_host_test.cpp — the batch index build (pcl_b200/csrc/lbvh_kernels.cuh: the *_batch kernels) compiled for the
// HOST and run on emulated thread blocks (tests/host/warp_emu.h) in the sequence of lbvh.cu: build_index_batch, with
// std::stable_sort where the driver sorts with CUB and plain loops where it scans by key.  Each cloud's handle is compared
// with the single build of that cloud alone (tests/host/device_build.h):
//   * byte-equal: n_cloud, n_valid, n_leaves, root, lo, hi, morton scale, the padded points (sentinels included), the
//     nodes, the per-node leaf ranges, and the cell table's bmax, log2_slots, entries, occupied cells per level and margin;
//   * equal as a set: the cell table's (key, reference) slots.  Where keys collide, a key's slot depends on the order in
//     which the inserts arrive, so the slot bytes are not compared.
// Batches of 1, 3 and 37 clouds: 1, 8 and 9 points (one leaf, two leaves), 255 and 256 finite points (either side of the
// cell-table threshold), NaN and Inf records, runs of identical points, a zero-extent and a planar frame, frames 1e-3 and 1e4
// wide far from the origin.  PCLB_TEST_SEED perturbs the scenes.  CPU only.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <map>
#include <numeric>

#include "../../pcl_b200/csrc/lbvh_kernels.cuh"
#include "device_build.h"

template <typename F> static void launch_grid(unsigned grid, int block, F kernel)
{
  gridDim.x = grid ? grid : 1;
  blockDim.x = block;
  for (unsigned b = 0; b < gridDim.x; ++b) {
    blockIdx_storage.x = b;
    warp_emu::run_block(block, kernel);
  }
  gridDim.x = 1;
  blockIdx_storage.x = 0;
}
template <typename F> static void launch_n(std::size_t n, F kernel) { launch_grid((unsigned)((n + 255) / 256), 256, kernel); }

// one handle of the batch, in host memory
struct Handle {
  std::size_t n_cloud = 0, n_valid = 0;
  int n_leaves = 0, root = 0;
  float lo[3], hi[3], scale = 1.f;
  std::vector<float4> pts;
  std::vector<BvhNode> nodes;
  std::vector<int2> node_leaves;
  std::vector<unsigned long long> slots;
  CellTableHost cells;
};

// lbvh.cu: build_index_batch, step by step
static void batch_build(const std::vector<std::vector<float>>& clouds, std::vector<Handle>& out)
{
  const int B = (int)clouds.size();
  std::vector<long long> off(B + 1, 0), tiles(B + 1, 0);
  for (int k = 0; k < B; ++k) off[k + 1] = off[k] + (long long)(clouds[k].size() / 3);
  const std::size_t n = (std::size_t)off[B];
  std::vector<float4> dense(n);
  for (int k = 0; k < B; ++k)
    for (std::size_t i = 0; i < clouds[k].size() / 3; ++i)
      dense[off[k] + i] = make_float4(clouds[k][3 * i], clouds[k][3 * i + 1], clouds[k][3 * i + 2], 1.f);
  std::vector<BuildCloud> cl(B);
  for (int k = 0; k < B; ++k) {
    cl[k].first = off[k];
    cl[k].n = off[k + 1] - off[k];
    tiles[k + 1] = tiles[k] + (cl[k].n + kBatchTile - 1) / kBatchTile;
  }
  // 1. boxes
  std::vector<BBoxAcc> acc(B);
  for (auto& a : acc) {
    for (int d = 0; d < 3; ++d) { a.lo[d] = 0x7fffffff; a.hi[d] = (int)0x80000000; }
    a.count = 0;
  }
  launch_grid((unsigned)tiles[B], 256, [&] { k_bbox_batch(dense.data(), cl.data(), tiles.data(), B, acc.data()); });
  for (int k = 0; k < B; ++k) {
    if (acc[k].count == 0) { std::printf("cloud %d has no finite point\n", k); std::exit(3); }
    cl[k].nv = (int)acc[k].count;
    float hi[3];
    morton_frame(acc[k], cl[k].lo, hi, cl[k].scale);
  }
  // 2. keys, sort by key, stable sort by cloud
  std::vector<unsigned long long> keys_in(n), keys1(n), keys(n);
  std::vector<int32_t> vals_in(n), vals1(n), vals(n), pos(n), perm(n);
  std::vector<unsigned> cloud_in(n), cloud_of(n);
  launch_n(n, [&] { k_morton_batch(dense.data(), n, off.data(), B, cl.data(), keys_in.data(), vals_in.data()); });
  {
    std::vector<std::size_t> o(n);
    std::iota(o.begin(), o.end(), 0);
    std::stable_sort(o.begin(), o.end(), [&](std::size_t a, std::size_t b) { return keys_in[a] < keys_in[b]; });
    for (std::size_t i = 0; i < n; ++i) { keys1[i] = keys_in[o[i]]; vals1[i] = vals_in[o[i]]; }
  }
  launch_n(n, [&] { k_cloud_of_sorted(vals1.data(), n, off.data(), B, cloud_in.data(), pos.data()); });
  {
    std::vector<std::size_t> o(n);
    std::iota(o.begin(), o.end(), 0);
    std::stable_sort(o.begin(), o.end(), [&](std::size_t a, std::size_t b) { return cloud_in[a] < cloud_in[b]; });
    for (std::size_t i = 0; i < n; ++i) { cloud_of[i] = cloud_in[o[i]]; perm[i] = pos[o[i]]; }
  }
  launch_n(n, [&] { k_permute_sorted(keys1.data(), vals1.data(), perm.data(), n, off.data(), B, keys.data(), vals.data()); });
  // 3. trees, cuts, scans by cloud, histograms
  const std::size_t n_tree = n - (std::size_t)B;
  std::vector<int2> kchildren(n_tree), krange(n_tree);
  std::vector<int> knode_parent(n_tree), keep(n_tree, 0), new_id(n_tree), kpoint_parent(n), leaf_flag(n, 0), leaf_incl(n);
  std::vector<unsigned> node_cloud(n_tree, ~0u);
  launch_n(n, [&] {
    k_karras_points_batch(keys.data(), n, off.data(), B, cl.data(), kchildren.data(), knode_parent.data(),
                          kpoint_parent.data(), krange.data(), node_cloud.data());
  });
  launch_n(n, [&] {
    k_mark_cells_batch(n, off.data(), B, cl.data(), krange.data(), knode_parent.data(), kpoint_parent.data(), keep.data(),
                       leaf_flag.data());
  });
  for (std::size_t i = 0; i < n_tree; ++i) CHECK(node_cloud[i] != ~0u, "node position %zu has no cloud", i);
  for (std::size_t i = 0; i < n; ++i)  // cub::DeviceScan::InclusiveSumByKey
    leaf_incl[i] = leaf_flag[i] + (i > 0 && cloud_of[i] == cloud_of[i - 1] ? leaf_incl[i - 1] : 0);
  for (std::size_t i = 0; i < n_tree; ++i)  // cub::DeviceScan::ExclusiveSumByKey
    new_id[i] = i > 0 && node_cloud[i] == node_cloud[i - 1] ? new_id[i - 1] + keep[i - 1] : 0;
  std::vector<CloudSummary> sum(B);
  std::memset(sum.data(), 0, B * sizeof(CloudSummary));
  launch_grid((unsigned)tiles[B], 256, [&] { k_prefix_hist_batch(keys.data(), cl.data(), tiles.data(), B, sum.data()); });
  launch_n(B, [&] { k_cut_summary(cl.data(), B, leaf_incl.data(), new_id.data(), keep.data(), sum.data()); });
  // 4. handles
  out.assign(B, Handle());
  std::vector<long long> leaves(B + 1, 0), nodes(B + 1, 0), slots(B + 1, 0);
  for (int k = 0; k < B; ++k) {
    BuildCloud& C = cl[k];
    Handle& h = out[k];
    h.n_cloud = (std::size_t)C.n;
    h.n_valid = (std::size_t)C.nv;
    morton_frame(acc[k], h.lo, h.hi, h.scale);
    int n_int = 0;
    if (C.nv <= kLeafSize) { h.n_leaves = 1; h.root = ~0; }
    else {
      CHECK(sum[k].n_leaves >= 2 && sum[k].n_int == sum[k].n_leaves - 1, "cloud %d: inconsistent cut", k);
      h.n_leaves = sum[k].n_leaves;
      n_int = sum[k].n_int;
      h.root = 0;
      if (C.nv >= 256) h.cells = cell_table_plan(sum[k].hist, C.nv, h.lo, h.hi, h.scale);
    }
    h.pts.assign((std::size_t)h.n_leaves * kLeafSize, make_float4(1, 2, 3, 4));  // garbage: the clear must overwrite it
    h.nodes.assign(n_int, BvhNode());
    h.node_leaves.assign(n_int, make_int2(-5, -5));
    h.slots.assign(h.cells.log2_slots ? (std::size_t)1 << h.cells.log2_slots : 0, 0xdeadbeefull);
    C.n_leaves = h.n_leaves;
    C.n_int = n_int;
    C.pts = h.pts.data();
    C.nodes = h.nodes.data();
    C.node_leaves = h.node_leaves.data();
    if (h.cells.log2_slots) C.cells = cell_table_view(reinterpret_cast<uint2*>(h.slots.data()), h.cells);
    C.leaf_first = leaves[k];
    C.node_first = nodes[k];
    leaves[k + 1] = leaves[k] + C.n_leaves;
    nodes[k + 1] = nodes[k] + n_int;
    slots[k + 1] = slots[k] + (long long)h.slots.size();
  }
  const std::size_t n_leaves = (std::size_t)leaves[B], n_int = (std::size_t)nodes[B];
  std::vector<int> leaf_start(n_leaves), node_parent(n_int), leaf_parent(n_leaves);
  std::vector<int2> children(n_int);
  std::vector<float4> leaf_lo(n_leaves), leaf_hi(n_leaves), node_lo(n_int), node_hi(n_int);
  std::vector<unsigned> flags(n_int, 0u);
  launch_n(std::max<std::size_t>(n_leaves * kLeafSize, (std::size_t)slots[B]),
           [&] { k_clear_outputs_batch(cl.data(), B, leaves.data(), slots.data()); });
  launch_n((std::size_t)B * kLeafSize, [&] { k_gather_small_batch(dense.data(), vals.data(), cl.data(), B); });
  launch_n(n, [&] {
    k_leaf_starts_batch(n, off.data(), B, cl.data(), leaf_flag.data(), leaf_incl.data(), leaf_start.data());
  });
  launch_n(n, [&] {
    k_scatter_cells_batch(dense.data(), vals.data(), n, off.data(), B, cl.data(), leaf_incl.data(), leaf_start.data());
  });
  launch_n(n, [&] {
    k_link_cells_batch(n, off.data(), B, cl.data(), kchildren.data(), krange.data(), keep.data(), new_id.data(),
                       leaf_incl.data(), keys.data(), children.data(), node_parent.data(), leaf_parent.data());
  });
  launch_n(n_leaves, [&] {
    k_refit_batch(cl.data(), B, leaves.data(), children.data(), node_parent.data(), leaf_parent.data(), leaf_lo.data(),
                  leaf_hi.data(), node_lo.data(), node_hi.data(), flags.data());
  });
  if (n_int)
    launch_n(n_int, [&] {
      k_pack_nodes_batch(cl.data(), B, nodes.data(), children.data(), leaf_lo.data(), leaf_hi.data(), node_lo.data(),
                         node_hi.data());
    });
}

static int level_of(unsigned key) { return (31 - __builtin_clz(key)) / 3; }

static void compare(const Handle& h, const std::vector<float>& xyz, int k, const char* scene)
{
  HostIndex I;
  device_build::build(I, xyz, true);
  std::size_t nv = 0;
  for (std::size_t i = 0; i < xyz.size() / 3; ++i)
    nv += std::isfinite(xyz[3 * i]) && std::isfinite(xyz[3 * i + 1]) && std::isfinite(xyz[3 * i + 2]);
  CHECK(h.n_cloud == xyz.size() / 3, "%s cloud %d: n_cloud %zu != %zu", scene, k, h.n_cloud, xyz.size() / 3);
  CHECK(h.n_valid == nv, "%s cloud %d: n_valid %zu != %zu", scene, k, h.n_valid, nv);
  CHECK((std::size_t)h.n_leaves * kLeafSize == I.pts.size(), "%s cloud %d: %d leaves, single %zu", scene, k, h.n_leaves,
        I.pts.size() / kLeafSize);
  CHECK(h.root == I.root, "%s cloud %d: root", scene, k);
  CHECK(std::memcmp(h.lo, I.lo, sizeof h.lo) == 0 && std::memcmp(h.hi, I.hi, sizeof h.hi) == 0, "%s cloud %d: box", scene, k);
  CHECK(std::memcmp(&h.scale, &I.scale, 4) == 0, "%s cloud %d: scale", scene, k);
  CHECK(h.pts.size() == I.pts.size() && std::memcmp(h.pts.data(), I.pts.data(), h.pts.size() * sizeof(float4)) == 0,
        "%s cloud %d: points", scene, k);
  CHECK(h.nodes.size() == I.nodes.size() &&
            (h.nodes.empty() || std::memcmp(h.nodes.data(), I.nodes.data(), h.nodes.size() * sizeof(BvhNode)) == 0),
        "%s cloud %d: nodes", scene, k);
  CHECK(h.node_leaves.size() == I.node_leaves.size() &&
            (h.node_leaves.empty() ||
             std::memcmp(h.node_leaves.data(), I.node_leaves.data(), h.node_leaves.size() * sizeof(int2)) == 0),
        "%s cloud %d: node leaves", scene, k);
  CHECK(h.cells.log2_slots == I.log2_slots && h.cells.bmax == I.bmax, "%s cloud %d: table shape", scene, k);
  CHECK(std::memcmp(&h.cells.margin, &I.margin, 4) == 0 || h.cells.log2_slots == 0, "%s cloud %d: margin", scene, k);
  // the single table's entries, per level, and as a set of (key, reference)
  std::vector<std::pair<unsigned, unsigned>> a, b;
  uint64_t occ[16] = {0};
  for (const uint2& s : I.slots)
    if (s.x) { a.emplace_back(s.x, s.y); ++occ[level_of(s.x)]; }
  for (unsigned long long s : h.slots)
    if (s) b.emplace_back((unsigned)(s & 0xffffffffu), (unsigned)(s >> 32));
  CHECK(h.cells.entries == a.size(), "%s cloud %d: %llu entries, single table holds %zu", scene, k,
        (unsigned long long)h.cells.entries, a.size());
  CHECK(std::memcmp(occ, h.cells.occupied, sizeof occ) == 0, "%s cloud %d: occupied cells per level", scene, k);
  std::sort(a.begin(), a.end());
  std::sort(b.begin(), b.end());
  CHECK(a == b, "%s cloud %d: cell-table entries differ as a set (%zu vs %zu)", scene, k, a.size(), b.size());
}

static std::vector<float> random_cloud(std::mt19937& rng, std::size_t n, float width, const float shift[3], bool planar)
{
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::vector<float> xyz(3 * n);
  for (std::size_t i = 0; i < n; ++i)
    for (int d = 0; d < 3; ++d) xyz[3 * i + d] = (planar && d == 2) ? shift[2] : shift[d] + width * U(rng);
  return xyz;
}

int main()
{
  std::mt19937 rng(test_seed(20261018u));
  const float qnan = std::numeric_limits<float>::quiet_NaN(), inf = INFINITY;
  const float o0[3] = {0.f, 0.f, 0.f}, far_[3] = {1e5f, -2e5f, 3e4f}, mid[3] = {-7.f, 3.f, 11.f};
  // the kinds of clouds the batches are made of
  std::vector<std::pair<const char*, std::vector<float>>> kinds;
  kinds.emplace_back("1 point", random_cloud(rng, 1, 1.f, mid, false));
  kinds.emplace_back("8 points", random_cloud(rng, 8, 1.f, mid, false));
  kinds.emplace_back("9 points", random_cloud(rng, 9, 1.f, mid, false));
  {
    auto c = random_cloud(rng, 256, 2.f, o0, false);
    c[3 * 77 + 1] = qnan;  // 255 finite points: no cell table
    kinds.emplace_back("255 finite of 256", c);
  }
  kinds.emplace_back("256 points", random_cloud(rng, 256, 2.f, o0, false));
  {
    auto c = random_cloud(rng, 3000, 5.f, mid, false);
    for (int i = 0; i < 3000; i += 97) c[3 * i + (i % 3)] = (i % 2) ? qnan : -inf;
    c[3 * 5] = inf;
    kinds.emplace_back("NaN and Inf records", c);
  }
  {
    auto c = random_cloud(rng, 600, 1.f, o0, false);
    for (int i = 100; i < 140; ++i) for (int d = 0; d < 3; ++d) c[3 * i + d] = c[3 * 99 + d];  // 41 identical points
    kinds.emplace_back("identical points", c);
  }
  {
    std::vector<float> c(3 * 300);
    for (int i = 0; i < 300; ++i) { c[3 * i] = 1.5f; c[3 * i + 1] = -2.f; c[3 * i + 2] = 0.25f; }
    kinds.emplace_back("zero extent", c);
  }
  kinds.emplace_back("planar", random_cloud(rng, 2000, 3.f, mid, true));
  kinds.emplace_back("1e-3 wide far out", random_cloud(rng, 1500, 1e-3f, far_, false));
  kinds.emplace_back("1e4 wide far out", random_cloud(rng, 1500, 1e4f, far_, false));
  kinds.emplace_back("5000 points", random_cloud(rng, 5000, 10.f, mid, false));

  struct Batch { const char* name; std::vector<int> kinds; };
  std::vector<Batch> batches;
  batches.push_back({"B = 1", {11}});
  batches.push_back({"B = 3", {2, 9, 10}});
  {
    Batch b{"B = 37", {}};
    for (int k = 0; k < 37; ++k) b.kinds.push_back(k < (int)kinds.size() ? k : (int)(rng() % kinds.size()));
    std::shuffle(b.kinds.begin(), b.kinds.end(), rng);
    batches.push_back(b);
  }
  for (const Batch& bt : batches) {
    std::vector<std::vector<float>> clouds;
    for (int k : bt.kinds) clouds.push_back(kinds[k].second);
    std::vector<Handle> out;
    batch_build(clouds, out);
    for (std::size_t k = 0; k < clouds.size(); ++k) compare(out[k], clouds[k], (int)k, kinds[bt.kinds[k]].first);
    std::printf("%s: %zu clouds compared (%ld checks, %ld failures so far)\n", bt.name, clouds.size(), g_checks, g_fail);
  }
  std::printf("%ld checks, %ld failures\n", g_checks, g_fail);
  if (g_fail) return 1;
  std::printf("PASSED\n");
  return 0;
}
