// voxel_host_test.cpp — the VoxelGrid kernels (pcl_b200/csrc/voxel_kernels.cuh) compiled for the HOST and run in voxel.cu's
// sequence (std::stable_sort and a flagged copy where the driver calls CUB), against the CPU oracle's VoxelGrid
// (oracle/libpcl_oracle.so, linked: test infrastructure): centroids bit for bit and in the same order, the normal /
// curvature planes of PointNormal records bit for bit, the minimum-points filter, non-finite points, index subsets.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"


#include <numeric>


#include "../../pcl_b200/csrc/voxel_kernels.cuh"

extern "C" long long orc_voxelgrid(const float* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int is_dense, const float leaf[3],
                                   unsigned min_pts, float* out);
extern "C" long long orc_voxelgrid_normals(const float* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx, int is_dense,
                                           const float leaf[3], unsigned min_pts, float* out, long normal_off, float* out_nc);

// the fixed seed of the committed test, or PCLB_TEST_SEED for a fuzz run (tools/dev/fuzz_host_tests.sh)
template <typename F> static void launch(std::size_t n, int block, F kernel)
{
  const unsigned grid = static_cast<unsigned>((n + block - 1) / block);
  blockDim.x = block;
  gridDim.x = grid ? grid : 1;
  for (unsigned b = 0; b < gridDim.x; ++b) { blockIdx_storage.x = b; warp_emu::run_block(block, kernel); }
  blockIdx_storage.x = 0;
  gridDim.x = 1;
}

// voxel.cu: voxelgrid(), on host memory.  cloud: n records of `stride` floats (xyz at 0, normal at 4, curvature at 8 when
// with_normals).  Returns the number of voxels; -1 = the overflow guard fired.
static long long device_voxelgrid(const std::vector<float>& cloud, std::size_t stride, const std::vector<int32_t>* indices, const float leaf[3], unsigned min_pts,
                                  bool with_normals, std::vector<float4>& out, std::vector<float4>& out_nc)
{
  using namespace pclb200;
  const std::size_t n = cloud.size() / stride, cnt = indices ? indices->size() : n;
  out.clear(); out_nc.clear();
  if (cnt == 0) return 0;
  std::vector<float4> dense(cnt);
  for (std::size_t i = 0; i < cnt; ++i) { const float* r = &cloud[(indices ? (std::size_t)(*indices)[i] : i) * stride]; dense[i] = make_float4(r[0], r[1], r[2], 1.f); }
  MinMaxAcc acc;
  for (int d = 0; d < 3; ++d) { acc.lo[d] = 0x7fffffff; acc.hi[d] = (int)0x80000000; }
  acc.count = 0;
  {
    blockDim.x = 256;
    gridDim.x = static_cast<unsigned>(std::min<std::size_t>((cnt + 255) / 256, 8));
    for (unsigned b = 0; b < gridDim.x; ++b) { blockIdx_storage.x = b; warp_emu::run_block(256, [&] { k_vg_minmax(dense.data(), cnt, &acc); }); }
    blockIdx_storage.x = 0; gridDim.x = 1;
  }
  const std::size_t n_valid = static_cast<std::size_t>(acc.count);
  if (n_valid == 0) return 0;
  float mn[3], mx[3], inv[3];
  for (int d = 0; d < 3; ++d) { mn[d] = vord2f(acc.lo[d]); mx[d] = vord2f(acc.hi[d]); inv[d] = 1.0f / leaf[d]; }
  volatile float e0 = (mx[0] - mn[0]) * inv[0], e1 = (mx[1] - mn[1]) * inv[1], e2 = (mx[2] - mn[2]) * inv[2];
  const std::int64_t dx = (std::int64_t)e0 + 1, dy = (std::int64_t)e1 + 1, dz = (std::int64_t)e2 + 1;
  if (dx * dy * dz > (std::int64_t)std::numeric_limits<std::int32_t>::max()) return -1;
  VgParams gp;
  int div_b[3];
  for (int d = 0; d < 3; ++d) {
    volatile float lo_s = mn[d] * inv[d], hi_s = mx[d] * inv[d];
    gp.inv[d] = inv[d];
    gp.min_b[d] = (int)std::floor(lo_s);
    div_b[d] = (int)std::floor(hi_s) - gp.min_b[d] + 1;
  }
  gp.mul[0] = 1; gp.mul[1] = div_b[0]; gp.mul[2] = div_b[0] * div_b[1];
  std::vector<unsigned> keys_in(cnt), keys(cnt);
  std::vector<int32_t> vals_in(cnt), vals(cnt);
  launch(cnt, 256, [&] { k_vg_keys(dense.data(), cnt, gp, keys_in.data(), vals_in.data()); });
  {  // cub::DeviceRadixSort::SortPairs, 32 key bits, stable
    std::vector<std::size_t> order(cnt);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](std::size_t a, std::size_t b) { return keys_in[a] < keys_in[b]; });
    for (std::size_t i = 0; i < cnt; ++i) { keys[i] = keys_in[order[i]]; vals[i] = vals_in[order[i]]; }
  }
  std::vector<unsigned char> head(n_valid);
  launch(n_valid, 256, [&] { k_vg_heads(keys.data(), n_valid, head.data()); });
  std::vector<unsigned> starts;   // cub::DeviceSelect::Flagged over a counting iterator
  for (std::size_t j = 0; j < n_valid; ++j) if (head[j]) starts.push_back(static_cast<unsigned>(j));
  const std::size_t n_runs = starts.size();
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
  }
  if (n_out == 0) return 0;
  out.assign(n_out, make_float4(0, 0, 0, 0));
  launch(n_out, 128, [&] { k_vg_centroids(dense.data(), vals.data(), d_runs, n_out, out.data()); });
  if (with_normals) {
    std::vector<float4> nc(2 * cnt);
    const unsigned char* src = reinterpret_cast<const unsigned char*>(cloud.data()) + 16;
    launch(cnt, 256, [&] { k_vg_load_nc(src, stride * 4, indices ? indices->data() : nullptr, cnt, nc.data()); });
    out_nc.assign(2 * n_out, make_float4(0, 0, 0, 0));
    launch(n_out, 128, [&] { k_vg_normals(nc.data(), vals.data(), d_runs, n_out, out_nc.data()); });
  }
  return static_cast<long long>(n_out);
}

static void run_scene(const char* name, const std::vector<float>& cloud, std::size_t stride, const std::vector<int32_t>* indices, float lx, float ly, float lz,
                      unsigned min_pts, bool dense)
{
  const float leaf[3] = {lx, ly, lz};
  const std::size_t n = cloud.size() / stride;
  std::vector<float4> g, gnc;
  const bool with_normals = stride >= 12;
  const long long m = device_voxelgrid(cloud, stride, indices, leaf, min_pts, with_normals, g, gnc);
  std::vector<float> o(4 * std::max<std::size_t>(n, 1)), onc(8 * std::max<std::size_t>(n, 1));
  const long long mo = with_normals ? orc_voxelgrid_normals(cloud.data(), n, stride, indices ? indices->data() : nullptr, indices ? indices->size() : 0, dense ? 1 : 0, leaf,
                                                            min_pts, o.data(), 4, onc.data())
                                    : orc_voxelgrid(cloud.data(), n, stride, indices ? indices->data() : nullptr, indices ? indices->size() : 0, dense ? 1 : 0, leaf, min_pts,
                                                    o.data());
  CHECK(m == mo, "%s: %lld voxels, the oracle has %lld", name, m, mo);
  int bad = 0, bad_nc = 0;
  for (long long i = 0; i < m && i < mo; ++i) {
    if (std::memcmp(&g[i], &o[4 * i], 16) != 0) ++bad;
    if (with_normals && std::memcmp(&gnc[2 * i], &onc[8 * i], 20) != 0) ++bad_nc;   // normal x y z, its fourth float, curvature
  }
  if (with_normals && m > 0) {   // the planes compared are real: unit normals, the averaged curvature
    const float4 a = gnc[0], c = gnc[1];
    CHECK(std::fabs(a.x * a.x + a.y * a.y + a.z * a.z - 1.f) < 1e-5f && c.x > 0.f && c.x < 0.011f, "%s: first voxel normal (%g %g %g) curvature %g", name, a.x, a.y, a.z, c.x);
  }
  CHECK(bad == 0 && bad_nc == 0, "%s: %d centroids and %d normal / curvature records differ from the oracle", name, bad, bad_nc);
  std::printf("%-36s %6zu records -> %6lld voxels (oracle %lld); ok so far: %ld checks, %ld failures\n", name, indices ? indices->size() : n, m, mo, g_checks, g_fail);
}

int main(int argc, char** argv)
{
  const int scale = argc > 1 ? std::atoi(argv[1]) : 1;
  std::mt19937 rng(test_seed(1618));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::normal_distribution<float> N(0.f, 1.f);
  auto xyz1 = [&](int n, auto gen) { std::vector<float> v(4 * (std::size_t)n, 1.f); for (int i = 0; i < n; ++i) gen(i, &v[4 * (std::size_t)i]); return v; };
  const auto vol = xyz1(20000 * scale, [&](int, float* p) { p[0] = U(rng); p[1] = U(rng); p[2] = U(rng); });
  run_scene("uniform cube, leaf 0.05", vol, 4, nullptr, 0.05f, 0.05f, 0.05f, 0, true);
  run_scene("uniform cube, anisotropic leaf", vol, 4, nullptr, 0.1f, 0.03f, 0.07f, 0, true);
  run_scene("uniform cube, min 3 points", vol, 4, nullptr, 0.04f, 0.04f, 0.04f, 3, true);
  run_scene("uniform cube, leaf larger than cloud", vol, 4, nullptr, 5.f, 5.f, 5.f, 0, true);
  auto moved = xyz1(15000 * scale, [&](int, float* p) { p[0] = -120.f + 30.f * U(rng); p[1] = 40.f + 30.f * U(rng); p[2] = -3.f + 2.f * N(rng); });
  run_scene("offset sweep, leaf 0.5", moved, 4, nullptr, 0.5f, 0.5f, 0.5f, 0, true);
  {
    auto holes = vol;
    for (std::size_t i = 0; i < holes.size() / 4; i += 37) holes[4 * i + (i % 3)] = std::numeric_limits<float>::quiet_NaN();
    run_scene("non-finite points, not dense", holes, 4, nullptr, 0.05f, 0.05f, 0.05f, 0, false);
    std::vector<int32_t> idx;
    for (int i = 0; i < (int)(vol.size() / 4); i += 3) idx.push_back(i);
    run_scene("index subset", vol, 4, &idx, 0.05f, 0.05f, 0.05f, 0, true);
  }
  {
    // pcl::PointNormal records: xyz1 | normal 0 | curvature pad3
    const int n = 12000 * scale;
    std::vector<float> pn(12 * (std::size_t)n, 0.f);
    for (int i = 0; i < n; ++i) {
      float* r = &pn[12 * (std::size_t)i];
      r[0] = 2.f * U(rng); r[1] = 2.f * U(rng); r[2] = 0.3f * std::sin(3.f * r[0]); r[3] = 1.f;
      float nx = -0.9f * std::cos(3.f * r[0]), ny = 0.05f * N(rng), nz = 1.f;
      const float inv = 1.f / std::sqrt(nx * nx + ny * ny + nz * nz);
      r[4] = nx * inv; r[5] = ny * inv; r[6] = nz * inv; r[7] = 0.f;
      r[8] = 0.01f * U(rng);
    }
    run_scene("PointNormal, all fields", pn, 12, nullptr, 0.06f, 0.06f, 0.06f, 0, true);
    run_scene("PointNormal, min 2 points", pn, 12, nullptr, 0.03f, 0.03f, 0.03f, 2, true);
  }
  {
    auto tiny = xyz1(2000, [&](int, float* p) { p[0] = 100.f * U(rng); p[1] = 100.f * U(rng); p[2] = 100.f * U(rng); });
    run_scene("overflow guard (leaf too small)", tiny, 4, nullptr, 0.01f, 0.01f, 0.01f, 0, true);
  }
  std::printf("%ld checks, %ld failures\n%s\n", g_checks, g_fail, g_fail ? "FAILED" : "PASSED");
  return g_fail ? 1 : 0;
}
