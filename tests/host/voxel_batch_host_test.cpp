// voxel_batch_host_test.cpp — the batch VoxelGrid (pcl_b200/csrc/voxel_kernels.cuh: k_vg_keys_batch, k_vg_heads_batch,
// k_vg_offsets_batch, with the batch build's k_bbox_batch from lbvh_kernels.cuh and the single call's run, filter and
// reduce kernels) compiled for the HOST and run on emulated thread blocks in the sequence of voxel.cu: voxelgrid_batch,
// with std::stable_sort and a flagged copy where the driver calls CUB.  Each cloud's rows, normal / curvature rows and
// count are compared bit for bit with the CPU oracle's VoxelGrid of that cloud alone (oracle/libpcl_oracle.so, linked:
// test infrastructure), which voxel_host_test.cpp holds to the single kernels.
// Batches of 1, 3 and 37 clouds: two clouds with identical coordinates (their voxel keys coincide), NaN and Inf records,
// an all-NaN cloud, a one-point cloud, a cloud the minimum empties, a zero-extent axis, points exactly on voxel faces, a
// cloud 1e4 away; fine, coarse and anisotropic leaves; min_points_per_voxel 0, 1 and 3; xyz1 and PointNormal records; and
// the overflow guard on one cloud of a batch.  PCLB_TEST_SEED perturbs the scenes.  CPU only.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <numeric>

#include "../../pcl_b200/csrc/lbvh_kernels.cuh"
#include "../../pcl_b200/csrc/voxel_kernels.cuh"

extern "C" long long orc_voxelgrid(const float* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int is_dense, const float leaf[3],
                                   unsigned min_pts, float* out);
extern "C" long long orc_voxelgrid_normals(const float* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int is_dense,
                                           const float leaf[3], unsigned min_pts, float* out, long normal_off, float* out_nc);

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
template <typename F> static void launch(std::size_t n, int block, F kernel) { launch_grid((unsigned)((n + block - 1) / block), block, kernel); }

// voxel.cu: voxelgrid_batch, on host memory.  recs: the batch's records of S floats (xyz at 0; normal at 4 and curvature
// at 8 when with_normals); off: B + 1 record offsets.  Returns the number of rows, or -1 - k when cloud k trips the guard.
static long long batch_voxelgrid(const std::vector<float>& recs, std::size_t S, const std::vector<long long>& off, const float leaf[3], unsigned min_pts,
                                 bool with_normals, std::vector<float4>& out, std::vector<float4>& out_nc, std::vector<long long>& out_off)
{
  using namespace pclb200;
  const int B = (int)off.size() - 1;
  const std::size_t n = (std::size_t)off[B];
  out.clear(); out_nc.clear();
  out_off.assign(B + 1, 0);
  std::vector<float4> dense(n);
  for (std::size_t i = 0; i < n; ++i) dense[i] = make_float4(recs[S * i], recs[S * i + 1], recs[S * i + 2], 1.f);
  // pass 1: boxes (lbvh.cu: cloud_boxes) -> grids
  std::vector<long long> tiles(B + 1, 0);
  std::vector<BuildCloud> cl(B);
  std::vector<BBoxAcc> acc(B);
  for (int k = 0; k < B; ++k) {
    cl[k].first = off[k];
    cl[k].n = off[k + 1] - off[k];
    tiles[k + 1] = tiles[k] + (cl[k].n + kBatchTile - 1) / kBatchTile;
    for (int d = 0; d < 3; ++d) { acc[k].lo[d] = 0x7fffffff; acc[k].hi[d] = (int)0x80000000; }
    acc[k].count = 0;
  }
  launch_grid((unsigned)tiles[B], 256, [&] { k_bbox_batch(dense.data(), cl.data(), tiles.data(), B, acc.data()); });
  std::vector<VgParams> grid(B);
  std::size_t n_valid = 0;
  for (int k = 0; k < B; ++k) {
    n_valid += (std::size_t)acc[k].count;
    if (!acc[k].count) continue;
    float mn[3], mx[3];
    for (int d = 0; d < 3; ++d) { mn[d] = vord2f(acc[k].lo[d]); mx[d] = vord2f(acc[k].hi[d]); }
    if (!vg_grid(mn, mx, leaf, grid[k])) return -1 - k;
  }
  if (n_valid == 0) return 0;
  // pass 2: keys ; pass 3: stable sort over 32 + bits(B) key bits
  std::vector<unsigned long long> keys_in(n), keys(n);
  std::vector<int32_t> vals_in(n), vals(n);
  launch(n, 256, [&] { k_vg_keys_batch(dense.data(), n, off.data(), B, grid.data(), keys_in.data(), vals_in.data()); });
  {
    int cloud_bits = 0;
    while ((1 << cloud_bits) <= B) ++cloud_bits;
    for (std::size_t i = 0; i < n; ++i) CHECK(keys_in[i] >> (32 + cloud_bits) == 0, "key %zu beyond the sorted bits", i);
    std::vector<std::size_t> order(n);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](std::size_t a, std::size_t b) { return keys_in[a] < keys_in[b]; });
    for (std::size_t i = 0; i < n; ++i) { keys[i] = keys_in[order[i]]; vals[i] = vals_in[order[i]]; }
  }
  // pass 4: run heads over the finite records, runs, minimum-points filter, per-cloud row offsets
  std::vector<unsigned char> head(n_valid);
  launch(n_valid, 256, [&] { k_vg_heads_batch(keys.data(), n_valid, head.data()); });
  std::vector<unsigned> starts;   // cub::DeviceSelect::Flagged over a counting iterator
  for (std::size_t j = 0; j < n_valid; ++j) if (head[j]) starts.push_back(static_cast<unsigned>(j));
  std::size_t n_runs = starts.size();
  std::vector<long long> d_off(B + 1);
  if (min_pts <= 1) launch(B + 1, 256, [&] { k_vg_offsets_batch(keys.data(), starts.data(), 1, &n_runs, B, d_off.data()); });
  std::vector<RunRef> runs_all(n_runs), runs;
  launch(n_runs, 256, [&] { k_vg_runs(starts.data(), n_runs, n_valid, runs_all.data()); });
  const RunRef* d_runs = runs_all.data();
  std::size_t n_out = n_runs;
  if (min_pts > 1) {
    std::vector<unsigned char> keep(n_runs);
    launch(n_runs, 256, [&] { k_vg_keep(starts.data(), n_runs, n_valid, min_pts, keep.data()); });
    for (std::size_t m = 0; m < n_runs; ++m) if (keep[m]) runs.push_back(runs_all[m]);
    n_out = runs.size();
    d_runs = runs.data();
    launch(B + 1, 256, [&] { k_vg_offsets_batch(keys.data(), reinterpret_cast<const unsigned*>(d_runs), 2, &n_out, B, d_off.data()); });
  }
  out_off = d_off;
  if (n_out == 0) return 0;
  // pass 5: centroids and normal / curvature planes over the whole batch
  out.assign(n_out, make_float4(0, 0, 0, 0));
  launch(n_out, 128, [&] { k_vg_centroids(dense.data(), vals.data(), d_runs, n_out, out.data()); });
  if (with_normals) {
    std::vector<float4> nc(2 * n);
    const unsigned char* src = reinterpret_cast<const unsigned char*>(recs.data()) + 16;
    launch(n, 256, [&] { k_vg_load_nc(src, S * 4, nullptr, n, nc.data()); });
    out_nc.assign(2 * n_out, make_float4(0, 0, 0, 0));
    launch(n_out, 128, [&] { k_vg_normals(nc.data(), vals.data(), d_runs, n_out, out_nc.data()); });
  }
  return static_cast<long long>(n_out);
}

static bool any_finite(const std::vector<float>& c, std::size_t S)
{
  for (std::size_t i = 0; i < c.size() / S; ++i)
    if (std::isfinite(c[S * i]) && std::isfinite(c[S * i + 1]) && std::isfinite(c[S * i + 2])) return true;
  return false;
}

// one batch against the oracle cloud by cloud; expect_guard = the cloud that must trip the guard first, or -1
static void run_batch(const char* name, const std::vector<std::vector<float>>& clouds, std::size_t S, const float leaf[3], unsigned min_pts,
                      int expect_guard = -1)
{
  const int B = (int)clouds.size();
  const bool with_normals = S >= 12;
  std::vector<long long> off(B + 1, 0);
  std::vector<float> recs;
  for (int k = 0; k < B; ++k) {
    off[k + 1] = off[k] + (long long)(clouds[k].size() / S);
    recs.insert(recs.end(), clouds[k].begin(), clouds[k].end());
  }
  std::vector<float4> g, gnc;
  std::vector<long long> goff;
  const long long m = batch_voxelgrid(recs, S, off, leaf, min_pts, with_normals, g, gnc, goff);
  if (expect_guard >= 0) {
    CHECK(m == -1 - expect_guard, "%s: guard result %lld, expected cloud %d", name, m, expect_guard);
    const auto& c = clouds[expect_guard];
    std::vector<float> o(4 * (c.size() / S + 1));
    CHECK(orc_voxelgrid(c.data(), c.size() / S, S, nullptr, 0, 0, leaf, min_pts, o.data()) == -1, "%s: the oracle does not trip on cloud %d", name, expect_guard);
    std::printf("%-44s B = %d: cloud %d trips the guard; ok so far: %ld checks, %ld failures\n", name, B, expect_guard, g_checks, g_fail);
    return;
  }
  CHECK(m >= 0 && goff[0] == 0 && goff[B] == m, "%s: %lld rows, offsets end at %lld", name, m, goff[B]);
  if (m < 0) return;
  int bad_count = 0, bad = 0, bad_nc = 0, empty = 0;
  for (int k = 0; k < B; ++k) {
    const auto& c = clouds[k];
    const std::size_t nk = c.size() / S;
    std::vector<float> o(4 * nk), onc(8 * nk);
    long long mo = 0;
    if (any_finite(c, S))
      mo = with_normals ? orc_voxelgrid_normals(c.data(), nk, S, nullptr, 0, 0, leaf, min_pts, o.data(), 4, onc.data())
                        : orc_voxelgrid(c.data(), nk, S, nullptr, 0, 0, leaf, min_pts, o.data());
    const long long mk = goff[k + 1] - goff[k];
    if (mk != mo) { ++bad_count; if (bad_count <= 5) std::printf("  %s: cloud %d has %lld rows, the oracle %lld\n", name, k, mk, mo); continue; }
    empty += mk == 0;
    for (long long i = 0; i < mk; ++i) {
      if (std::memcmp(&g[goff[k] + i], &o[4 * i], 16) != 0) ++bad;
      if (with_normals && std::memcmp(&gnc[2 * (goff[k] + i)], &onc[8 * i], 20) != 0) ++bad_nc;
    }
  }
  CHECK(bad_count == 0 && bad == 0 && bad_nc == 0, "%s: %d counts, %d rows and %d normal rows differ from the oracle", name, bad_count, bad, bad_nc);
  std::printf("%-44s B = %d: %d clouds compared, %lld rows, %d empty; ok so far: %ld checks, %ld failures\n", name, B, B, m, empty, g_checks, g_fail);
}

int main()
{
  std::mt19937 rng(test_seed(2718));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::normal_distribution<float> N(0.f, 1.f);
  const float nan = std::numeric_limits<float>::quiet_NaN(), inf = std::numeric_limits<float>::infinity();
  for (std::size_t S : {4, 12}) {
    // one record of S floats: xyz1, and for PointNormal a unit normal and a curvature
    auto rec = [&](std::vector<float>& v, float x, float y, float z) {
      const std::size_t b = v.size();
      v.resize(b + S, 0.f);
      v[b] = x; v[b + 1] = y; v[b + 2] = z; v[b + 3] = 1.f;
      if (S >= 12) {
        float nx = 0.3f * N(rng), ny = 0.3f * N(rng), nz = 1.f;
        const float inv = 1.f / std::sqrt(nx * nx + ny * ny + nz * nz);
        v[b + 4] = nx * inv; v[b + 5] = ny * inv; v[b + 6] = nz * inv; v[b + 8] = 0.01f * U(rng);
      }
    };
    // the scene kinds; kind 0 and 1 are the same coordinates
    auto scene = [&](int kind, int n) {
      std::vector<float> v;
      switch (kind % 9) {
        case 0: case 1: {  // identical coordinates (the generator restarts), so the two clouds' voxel keys coincide
          std::mt19937 twin(test_seed(99 + kind / 9));
          std::uniform_real_distribution<float> T(0.f, 1.f);
          for (int i = 0; i < n; ++i) rec(v, T(twin), T(twin), 0.5f * T(twin));
          break;
        }
        case 2:  // NaN and Inf records among finite ones
          for (int i = 0; i < n; ++i) {
            const int r = i % 7;
            rec(v, r == 3 ? nan : 2.f * U(rng), r == 5 ? inf : 2.f * U(rng), r == 6 ? -inf : U(rng));
          }
          break;
        case 3:  // no finite record: an empty range
          for (int i = 0; i < 1 + n / 50; ++i) rec(v, nan, i % 2 ? 1.f : nan, inf);
          break;
        case 4:  // one point
          rec(v, 3.f * U(rng), -2.f, 7.f * U(rng));
          break;
        case 5:  // sparse: every voxel holds one or two points, so a minimum of 3 empties the cloud
          for (int i = 0; i < 1 + n / 20; ++i) rec(v, 10.f * i + 0.01f * U(rng), 3.f * (i % 2), 0.f);
          break;
        case 6:  // zero extent along y
          for (int i = 0; i < n; ++i) rec(v, U(rng), 1.25f, 0.3f * U(rng));
          break;
        case 7:  // a lattice exactly on voxel faces of the 0.125 leaf
          for (int i = 0; i < n; ++i) rec(v, 0.125f * (i % 9), 0.125f * ((i / 9) % 5), 0.0625f * (i % 3));
          break;
        default:  // 1e4 away from the origin
          for (int i = 0; i < n; ++i) rec(v, 1e4f + 5.f * U(rng), -1e4f + 5.f * U(rng), 1e4f + N(rng));
          break;
      }
      return v;
    };
    const char* rt = S == 4 ? "xyz1" : "PointNormal";
    const float fine[3] = {0.125f, 0.125f, 0.125f}, coarse[3] = {0.5f, 0.5f, 0.5f}, aniso[3] = {0.25f, 0.05f, 0.125f};
    const float* leaves[3] = {fine, coarse, aniso};
    const char* leaf_name[3] = {"fine leaf", "coarse leaf", "anisotropic leaf"};
    for (int l = 0; l < 3; ++l)
      for (unsigned min_pts : {0u, 1u, 3u}) {
        char name[96];
        std::vector<std::vector<float>> b1 = {scene(2, 900)};
        std::snprintf(name, sizeof(name), "%s, %s, min %u", rt, leaf_name[l], min_pts);
        run_batch(name, b1, S, leaves[l], min_pts);
        std::vector<std::vector<float>> b3 = {scene(0, 700), scene(1, 700), scene(3, 40)};
        run_batch(name, b3, S, leaves[l], min_pts);
        std::vector<std::vector<float>> b37;
        for (int k = 0; k < 37; ++k) b37.push_back(scene(k, 50 + (int)(400 * U(rng))));
        run_batch(name, b37, S, leaves[l], min_pts);
      }
    // a cloud of a few tiles of k_bbox_batch among small ones
    {
      std::vector<std::vector<float>> big = {scene(4, 1), scene(8, 9000), scene(2, 300), scene(6, 5000)};
      char name[96];
      std::snprintf(name, sizeof(name), "%s, clouds over several box tiles", rt);
      run_batch(name, big, S, fine, 0);
    }
    // the guard: cloud 2 spans 1e3 units at a 0.001 leaf; the first cloud that trips is named
    {
      std::vector<std::vector<float>> g = {scene(6, 100), scene(3, 10), scene(6, 100), scene(8, 100)};
      std::vector<float> wide;
      for (int i = 0; i < 200; ++i) rec(wide, 1000.f * U(rng), 1000.f * U(rng), 1000.f * U(rng));
      g[2] = wide;
      g[3] = wide;
      const float tiny[3] = {0.001f, 0.001f, 0.001f};
      char name[96];
      std::snprintf(name, sizeof(name), "%s, overflow guard", rt);
      run_batch(name, g, S, tiny, 0, 2);
    }
  }
  std::printf("%ld checks, %ld failures\n%s\n", g_checks, g_fail, g_fail ? "FAILED" : "PASSED");
  return g_fail ? 1 : 0;
}
