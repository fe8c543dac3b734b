// normals_batch_host_test.cpp — the batch k-NN normals kernels (pcl_b200/csrc/knn_warp.cuh: k_knn_warp_batch;
// search_kernels.cuh: k_normals_batch<K>, k_knn_any_batch, k_normals_from_lists_batch) compiled for the HOST and run on
// emulated thread blocks (tests/host/warp_emu.h) in the sequence of search.cu: launch_normals_batch, against the single
// kernels run set by set as launch_normals runs them.  Every output row and every set's not-dense flag must be byte-equal.
// The indices are built by the real build kernels (tests/host/device_build.h).  Each set gets its own viewpoint and its own
// warp start level (0 on some sets with a cell table, so a batch mixes both paths); set 1 searches a shifted copy of cloud
// 0 in cloud 0's index, and the last set searches its cloud in cloud 0's index.  Batches of 1, 3 and 37 sets of: 1, 2, 8
// and 9 points, NaN and Inf records, identical points, zero extent, a planar cloud, frames 1e-3 and 1e4 wide far from the
// origin, clouds on both sides of the cell-table threshold.  The queries are each cloud's points (every third of the larger
// clouds); k = 3, 8, 10, 16, 20, 32 and 40.  PCLB_TEST_SEED perturbs the
// scenes.  CPU only.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

static inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }

#include "../../pcl_b200/csrc/search_kernels.cuh"
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
static unsigned grid128(std::size_t n) { return (unsigned)((n + 127) / 128); }
// the warp kernel's grid-stride loop: at most 2 blocks of 8 warps, so most warps take several batches of 32 queries
static unsigned grid_warp(std::size_t n) { return (unsigned)std::min<std::size_t>((n + 255) / 256, 2); }

// one set's index and what the driver decides for it
struct Set {
  HostIndex I;
  std::size_t n_valid = 0;
  std::vector<int32_t> pos_of_orig;
  int level = 0;
  float r_first = 0.f;
  // launch_normals's choice: the warp kernel for k = 12..32 on an index with a cell table that holds k points
  bool warp(int k) const { return level >= 1 && k >= 12 && k <= 32 && (std::size_t)k <= n_valid; }
};

template <int K> static void normals_single(const Set& S, const float4* q, std::size_t nq, int k, const float vp[3],
                                           float4* out, int* flag, int* d_error, const unsigned char* only)
{
  launch_grid(grid128(nq), 128, [&] {
    k_normals<K>(S.I.nodes.data(), S.I.pts.data(), S.I.root, q, nq, k, vp[0], vp[1], vp[2], out, flag, d_error, only);
  });
}
template <int K> static void normals_batch(const NormalsCloud* tab, const long long* off, int B, const float4* q,
                                          std::size_t nq, int k, float4* out, int* d_error, const unsigned char* only)
{
  launch_grid(grid128(nq), 128, [&] { k_normals_batch<K>(tab, off, B, q, nq, k, out, d_error, only); });
}
#define PCLB_BY_K(F, ...)                 \
  do {                                    \
    if (k <= 4) F<4>(__VA_ARGS__);        \
    else if (k <= 8) F<8>(__VA_ARGS__);   \
    else if (k <= 10) F<10>(__VA_ARGS__); \
    else if (k <= 16) F<16>(__VA_ARGS__); \
    else if (k <= 20) F<20>(__VA_ARGS__); \
    else F<32>(__VA_ARGS__);              \
  } while (0)

// search.cu: launch_normals of one set (queries q, w = the row in out)
static void single(const Set& S, const std::vector<float4>& q, int k, const float vp[3], std::vector<float4>& out, int& flag)
{
  const std::size_t nq = q.size();
  int d_error = 0;
  if (k > 32) {
    std::vector<int32_t> li(nq * k, -9);
    std::vector<float> ld(nq * k, -9.f);
    launch_grid(grid128(nq), 128, [&] {
      k_knn_any(S.I.nodes.data(), S.I.pts.data(), S.I.root, q.data(), nq, k, INFINITY, li.data(), ld.data(), &d_error);
    });
    launch_grid(grid128(nq), 128, [&] {
      k_normals_from_lists(S.I.pts.data(), S.pos_of_orig.data(), q.data(), nq, k, li.data(), 0, vp[0], vp[1], vp[2],
                           out.data(), &flag);
    });
  }
  else {
    std::vector<unsigned char> redo(nq, 0);
    const unsigned char* only = nullptr;
    if (S.warp(k)) {
      launch_grid(grid_warp(nq), 256, [&] {
        k_knn_warp<true>(S.I.view(true), S.I.node_leaves.data(), S.level, S.r_first, q.data(), nq, k, nullptr, nullptr,
                         vp[0], vp[1], vp[2], out.data(), &flag, redo.data());
      });
      only = redo.data();
    }
    PCLB_BY_K(normals_single, S, q.data(), nq, k, vp, out.data(), &flag, &d_error, only);
  }
  CHECK(d_error == 0, "single: traversal error");
}

// search.cu: launch_normals_batch
static void batch(const std::vector<const Set*>& sets, const std::vector<long long>& off, const std::vector<float4>& q,
                  int k, const std::vector<float>& vps, std::vector<float4>& out, std::vector<int>& flags)
{
  const int B = (int)sets.size();
  const std::size_t nq = q.size();
  std::vector<NormalsCloud> tab(B);
  bool any_warp = false;
  for (int b = 0; b < B; ++b) {
    const Set& S = *sets[b];
    NormalsCloud& e = tab[b];
    e.tree = S.I.view(true);
    e.node_leaves = S.I.node_leaves.data();
    e.pos_of_orig = k > 32 ? S.pos_of_orig.data() : nullptr;
    const bool warp = S.warp(k);
    e.level = warp ? S.level : 0;
    e.r_first = warp ? S.r_first : 0.f;
    for (int d = 0; d < 3; ++d) e.vp[d] = vps[3 * b + d];
    e.not_dense = &flags[b];
    any_warp = any_warp || warp;
  }
  int d_error = 0;
  if (k > 32) {
    std::vector<int32_t> li(nq * k, -9);
    std::vector<float> ld(nq * k, -9.f);
    launch_grid(grid128(nq), 128, [&] {
      k_knn_any_batch(tab.data(), off.data(), B, q.data(), nq, k, INFINITY, li.data(), ld.data(), &d_error);
    });
    launch_grid(grid128(nq), 128, [&] {
      k_normals_from_lists_batch(tab.data(), off.data(), B, q.data(), nq, k, li.data(), out.data());
    });
  }
  else {
    std::vector<unsigned char> redo(nq, 0);
    const unsigned char* only = nullptr;
    if (any_warp) {
      launch_grid(grid_warp(nq), 256, [&] { k_knn_warp_batch(tab.data(), off.data(), B, q.data(), nq, k, out.data(), redo.data()); });
      only = redo.data();
    }
    PCLB_BY_K(normals_batch, tab.data(), off.data(), B, q.data(), nq, k, out.data(), &d_error, only);
  }
  CHECK(d_error == 0, "batch: traversal error");
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
  std::mt19937 rng(test_seed(20261019u));
  std::normal_distribution<float> N(0.f, 1.f);
  const float qnan = std::numeric_limits<float>::quiet_NaN(), inf = INFINITY;
  const float o0[3] = {0.f, 0.f, 0.f}, far_[3] = {1e5f, -2e5f, 3e4f}, mid[3] = {-7.f, 3.f, 11.f};
  std::vector<std::pair<const char*, std::vector<float>>> kinds;
  kinds.emplace_back("1 point", random_cloud(rng, 1, 1.f, mid, false));
  kinds.emplace_back("2 points", random_cloud(rng, 2, 1.f, mid, false));
  kinds.emplace_back("8 points", random_cloud(rng, 8, 1.f, mid, false));
  kinds.emplace_back("9 points", random_cloud(rng, 9, 1.f, mid, false));
  {
    auto c = random_cloud(rng, 256, 2.f, o0, false);
    c[3 * 77 + 1] = qnan;  // 255 finite points: no cell table
    kinds.emplace_back("255 finite of 256", c);
  }
  {
    auto c = random_cloud(rng, 900, 5.f, mid, false);
    for (int i = 0; i < 900; i += 97) c[3 * i + (i % 3)] = (i % 2) ? qnan : -inf;
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
  kinds.emplace_back("planar", random_cloud(rng, 600, 3.f, mid, true));
  kinds.emplace_back("1e-3 wide far out", random_cloud(rng, 500, 1e-3f, far_, false));
  kinds.emplace_back("1e4 wide far out", random_cloud(rng, 500, 1e4f, far_, false));
  kinds.emplace_back("1200 points", random_cloud(rng, 1200, 10.f, mid, false));

  struct Batch { const char* name; std::vector<int> kinds; };
  std::vector<Batch> batches;
  batches.push_back({"B = 1", {11}});
  batches.push_back({"B = 3", {8, 3, 10}});
  {
    Batch b{"B = 37", {}};
    for (int j = 0; j < 37; ++j) b.kinds.push_back(j < (int)kinds.size() ? j : (int)(rng() % kinds.size()));
    std::shuffle(b.kinds.begin(), b.kinds.end(), rng);
    batches.push_back(b);
  }
  const int ks[] = {3, 8, 10, 16, 20, 32, 40};
  for (const Batch& bt : batches) {
    const int B = (int)bt.kinds.size();
    std::vector<Set> built(B);
    std::vector<std::vector<float>> qsets(B);
    for (int b = 0; b < B; ++b) {
      const std::vector<float>& xyz = kinds[bt.kinds[b]].second;
      Set& S = built[b];
      device_build::build(S.I, xyz, true);
      for (std::size_t i = 0; i < xyz.size() / 3; ++i)
        S.n_valid += std::isfinite(xyz[3 * i]) && std::isfinite(xyz[3 * i + 1]) && std::isfinite(xyz[3 * i + 2]);
      S.pos_of_orig.assign(xyz.size() / 3, -1);
      for (std::size_t j = 0; j < S.I.pts.size(); ++j)
        if (__float_as_int(S.I.pts[j].w) != kSentinelIndex) S.pos_of_orig[__float_as_int(S.I.pts[j].w)] = (int32_t)j;
      // the start level: a fine and a coarse one, and none on every third set with a table
      if (S.I.log2_slots && b % 3 != 2) {
        S.level = std::max(1, std::min(S.I.bmax, 2 + b % 2));
        S.r_first = (b % 4 == 1) ? 0.1f * (float)(1u << (21 - S.level)) / S.I.scale : 0.f;  // a sized first ball
      }
      // the queries: the cloud's own points, every third of a large cloud (the warp emulation is slow)
      for (std::size_t i = 0; i < xyz.size() / 3; i += xyz.size() > 900 ? 3 : 1)
        qsets[b].insert(qsets[b].end(), xyz.begin() + 3 * i, xyz.begin() + 3 * i + 3);
    }
    // set 1 searches a shifted copy of cloud 0 in cloud 0's index, the last set its own cloud in cloud 0's index
    std::vector<const Set*> sets(B);
    for (int b = 0; b < B; ++b) sets[b] = &built[b];
    if (B > 2) {
      qsets[1] = qsets[0];
      for (float& v : qsets[1]) v += 0.01f * N(rng);
      sets[1] = sets[B - 1] = &built[0];
    }
    std::vector<long long> off(B + 1, 0);
    for (int b = 0; b < B; ++b) off[b + 1] = off[b] + (long long)(qsets[b].size() / 3);
    const std::size_t n = (std::size_t)off[B];
    std::vector<float4> q(n);
    std::vector<float> vps(3 * B);
    for (int b = 0; b < B; ++b) {
      for (long long i = off[b]; i < off[b + 1]; ++i) {
        const float* p = &qsets[b][3 * (i - off[b])];
        q[i] = make_float4(p[0], p[1], p[2], __int_as_float((int)i));
      }
      // the origin, far above or far below: the flip differs between sets
      const float side = b % 3 == 0 ? 0.f : (b % 3 == 1 ? 1e3f : -1e3f);
      for (int d = 0; d < 3; ++d) vps[3 * b + d] = side * (d == 2 ? 1.f : 0.3f) + 0.1f * N(rng);
    }
    for (int k : ks) {
      std::vector<float4> got(n, make_float4(-7.f, -7.f, -7.f, -7.f));
      std::vector<int> flags(B, 0);
      batch(sets, off, q, k, vps, got, flags);
      for (int b = 0; b < B; ++b) {
        const std::size_t nq = (std::size_t)(off[b + 1] - off[b]);
        std::vector<float4> qb(nq), want(nq, make_float4(-7.f, -7.f, -7.f, -7.f));
        for (std::size_t i = 0; i < nq; ++i) { qb[i] = q[off[b] + i]; qb[i].w = __int_as_float((int)i); }
        int flag = 0;
        single(*sets[b], qb, k, &vps[3 * b], want, flag);
        CHECK(std::memcmp(want.data(), got.data() + off[b], nq * sizeof(float4)) == 0, "%s k %d set %d (%s): rows differ",
              bt.name, k, b, kinds[bt.kinds[b]].first);
        CHECK(flag == flags[b], "%s k %d set %d (%s): not-dense flag %d, single %d", bt.name, k, b,
              kinds[bt.kinds[b]].first, flags[b], flag);
      }
    }
    std::printf("%s: %d sets compared (%ld checks, %ld failures so far)\n", bt.name, B, g_checks, g_fail);
  }
  std::printf("%ld checks, %ld failures\n", g_checks, g_fail);
  if (g_fail) return 1;
  std::printf("PASSED\n");
  return 0;
}
