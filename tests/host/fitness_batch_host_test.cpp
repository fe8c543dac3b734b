// fitness_batch_host_test.cpp — the batch fitness score kernels (pcl_b200/csrc/icp_kernels.cuh: k_transform_batch,
// k_fitness_batch over batch_blocks's table) compiled for the HOST and run on emulated thread blocks (tests/host/warp_emu.h)
// in the sequence of icp.cu: fitness_batch, against k_fitness run problem by problem as fitness_score runs it (the points
// moved by k_transform's transform_one, one grid of persistent_blocks per problem).  Each problem's accumulator row (all
// kAccum doubles), its counter and the device error flag must be byte-equal to the single run's.  The grids are capped at
// three blocks so that the larger problems are grid-stride loops, as persistent_blocks makes them on the device.  The
// indices are built by the real build kernels (tests/host/device_build.h).  Batches of 1, 3 and 37 problems of: 1 point,
// 255 / 256 / 257 points, a problem whose grid is capped, NaN and Inf records, an all-NaN problem, a problem moved beyond
// max_range; several problems share one target.  Every batch runs in the four operation orders of the two entry points
// (fitness: float / double; validation: float / double) and with max_range = DBL_MAX, a value that drops some pairs,
// and 0.  PCLB_TEST_SEED perturbs the scenes.  CPU only.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <cfloat>
#include <random>

static inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }

#include "../../pcl_b200/csrc/icp_kernels.cuh"
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
// internal.cuh: persistent_blocks, with a cap of 3 blocks in place of 8 per SM
static unsigned grid_of(std::size_t n) { return (unsigned)std::max<std::size_t>(1, std::min<std::size_t>((n + 255) / 256, 3)); }

// icp.cu: make_pending
static Pending make_pending(const double* T, int mode)
{
  Pending h;
  std::memset(&h, 0, sizeof h);
  for (int i = 0; i < 12; ++i) {
    h.f[i] = (float)T[i];
    h.d[i] = T[i];
  }
  h.apply = 1;
  h.mode = mode;
  return h;
}

struct Sums {
  std::vector<double> accum;  // kAccum per problem
  std::vector<unsigned> counter;
  int d_error = 0;
};

// icp.cu: fitness_score of one problem (k_transform, then k_fitness over one grid)
static void single(const HostIndex& I, const float4* src, std::size_t n, const double* T, int mode, double max_range,
                   double* accum, unsigned& counter, int& d_error)
{
  std::vector<float4> q(src, src + n);
  const Pending P = make_pending(T, mode);
  for (std::size_t i = 0; i < n; ++i) transform_one(P, q.data(), i, nullptr);
  const unsigned grid = grid_of(n);
  std::vector<double> partials((std::size_t)grid * kAccum, -3.0);
  const GridSum sum{partials.data(), &counter, accum};
  const TreeView TV = I.view(true);
  launch_grid(grid, 256, [&] { k_fitness(TV, q.data(), n, max_range, sum, &d_error); });
}

// icp.cu: fitness_batch (one k_transform_batch, one k_fitness_batch over the table of every problem's own grid)
static void batch(const std::vector<const HostIndex*>& tgt, const std::vector<long long>& off, const std::vector<float4>& src,
                  const std::vector<double>& T, int mode, double max_range, Sums& out)
{
  const int B = (int)tgt.size();
  const std::size_t n = src.size();
  std::vector<float4> q = src;
  std::vector<Pending> P(B);
  std::vector<TreeView> trees(B);
  for (int p = 0; p < B; ++p) {
    P[p] = make_pending(&T[16 * (std::size_t)p], mode);
    trees[p] = tgt[p]->view(true);
  }
  launch_grid(2, 256, [&] { k_transform_batch(q.data(), n, off.data(), B, P.data(), nullptr); });
  const std::vector<BatchBlock> tab = batch_blocks(off, [](std::size_t m) { return grid_of(m); });
  std::vector<double> partials(tab.size() * kAccum, -3.0);
  out.accum.assign((std::size_t)B * kAccum, -1.0);
  out.counter.assign(B, 0u);
  out.d_error = 0;
  const GridSum sum{partials.data(), out.counter.data(), out.accum.data()};
  launch_grid((unsigned)tab.size(), 256, [&] { k_fitness_batch(tab.data(), trees.data(), q.data(), max_range, sum, &out.d_error); });
}

static std::vector<float> random_cloud(std::mt19937& rng, std::size_t n, float width, float shift)
{
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::vector<float> xyz(3 * n);
  for (float& v : xyz) v = shift + width * U(rng);
  return xyz;
}

int main()
{
  std::mt19937 rng(test_seed(20261020u));
  std::normal_distribution<float> N(0.f, 1.f);
  std::uniform_real_distribution<double> U(-1.0, 1.0);
  const float qnan = std::numeric_limits<float>::quiet_NaN(), inf = INFINITY;

  // three targets; every problem's source is noisy points of its target's region
  const int n_targets = 3;
  std::vector<HostIndex> targets(n_targets);
  const float t_width[n_targets] = {2.f, 5.f, 1.f}, t_shift[n_targets] = {0.f, -3.f, 10.f};
  for (int t = 0; t < n_targets; ++t) device_build::build(targets[t], random_cloud(rng, 700 + 150 * t, t_width[t], t_shift[t]), true);

  struct Kind { const char* name; std::size_t n; int nonfinite; bool far; };  // nonfinite: 0 none, 1 some, 2 all
  const std::vector<Kind> kinds = {{"1 point", 1, 0, false},         {"255 points", 255, 0, false},
                                   {"256 points", 256, 0, false},    {"257 points", 257, 0, false},
                                   {"capped grid", 1000, 0, false},  {"NaN and Inf records", 300, 1, false},
                                   {"all NaN", 40, 2, false},        {"beyond max_range", 200, 0, true}};

  struct Batch { const char* name; std::vector<int> kinds; };
  std::vector<Batch> batches;
  batches.push_back({"B = 1", {4}});
  batches.push_back({"B = 3", {0, 5, 3}});
  {
    Batch b{"B = 37", {}};
    for (int j = 0; j < 37; ++j) b.kinds.push_back(j < (int)kinds.size() ? j : (int)(rng() % kinds.size()));
    std::shuffle(b.kinds.begin(), b.kinds.end(), rng);
    batches.push_back(b);
  }
  const struct { const char* name; int mode; } modes[] = {{"fitness float", kApplyTransformsFloat},
                                                          {"fitness double", kApplyTransformsDouble},
                                                          {"validation float", kApplyIcp},
                                                          {"validation double", kApplyValidationDouble}};
  const double ranges[] = {std::numeric_limits<double>::max(), 2e-3, 0.0};
  long dbl_max_scores = 0, dropped_scores = 0;
  for (const Batch& bt : batches) {
    const int B = (int)bt.kinds.size();
    std::vector<const HostIndex*> tgt(B);
    std::vector<long long> off(B + 1, 0);
    std::vector<float4> src;
    std::vector<double> T(16 * (std::size_t)B);
    for (int p = 0; p < B; ++p) {
      const Kind& k = kinds[bt.kinds[p]];
      const int t = p % n_targets;  // every target serves several problems of a batch of 3 or more
      tgt[p] = &targets[t];
      const std::vector<float>& txyz = targets[t].xyz;
      const std::size_t nt = txyz.size() / 3;
      for (std::size_t i = 0; i < k.n; ++i) {
        const std::size_t j = rng() % nt;
        float4 v = make_float4(txyz[3 * j] + 0.02f * N(rng), txyz[3 * j + 1] + 0.02f * N(rng), txyz[3 * j + 2] + 0.02f * N(rng),
                               1.f);
        if (k.nonfinite == 2 || (k.nonfinite == 1 && i % 29 == 3)) {
          const float bad = (i % 2) ? qnan : ((i % 3) ? inf : -inf);
          (i % 3 == 0 ? v.x : (i % 3 == 1 ? v.y : v.z)) = bad;
        }
        src.push_back(v);
      }
      off[p + 1] = off[p] + (long long)k.n;
      // a small rotation about z and a translation; the far problem is moved 100 away
      const double a = 0.03 * U(rng), c = std::cos(a), s = std::sin(a);
      const double tx = k.far ? 100.0 : 0.01 * U(rng), ty = 0.01 * U(rng), tz = 0.01 * U(rng);
      const double M[16] = {c, -s, 0, tx, s, c, 0, ty, 0, 0, 1, tz, 0, 0, 0, 1};
      std::copy(M, M + 16, T.begin() + 16 * (std::size_t)p);
    }
    for (const auto& m : modes)
      for (double max_range : ranges) {
        Sums got;
        batch(tgt, off, src, T, m.mode, max_range, got);
        CHECK(got.d_error == 0, "%s %s: batch traversal error", bt.name, m.name);
        for (int p = 0; p < B; ++p) {
          const std::size_t n = (std::size_t)(off[p + 1] - off[p]);
          std::vector<double> want(kAccum, -1.0);
          unsigned counter = 0;
          int d_error = 0;
          single(*tgt[p], &src[(std::size_t)off[p]], n, &T[16 * (std::size_t)p], m.mode, max_range, want.data(), counter,
                 d_error);
          CHECK(std::memcmp(want.data(), &got.accum[(std::size_t)p * kAccum], kAccum * sizeof(double)) == 0,
                "%s %s max_range %g problem %d (%s): sums %.17g / %.17g, single %.17g / %.17g", bt.name, m.name, max_range, p,
                kinds[bt.kinds[p]].name, got.accum[(std::size_t)p * kAccum], got.accum[(std::size_t)p * kAccum + 1], want[0],
                want[1]);
          CHECK(got.counter[p] == 0 && counter == 0, "%s %s problem %d: counters not reset", bt.name, m.name, p);
          dbl_max_scores += want[0] == 0.0;
          dropped_scores += want[0] > 0.0 && want[0] < (double)n && kinds[bt.kinds[p]].nonfinite == 0;
        }
      }
    std::printf("%s: %d problems compared (%ld checks, %ld failures so far)\n", bt.name, B, g_checks, g_fail);
  }
  // the scenes reach both edges of the score: problems with no pair (DBL_MAX) and problems whose pairs max_range thins
  CHECK(dbl_max_scores > 0 && dropped_scores > 0, "scenes: %ld empty scores, %ld thinned", dbl_max_scores, dropped_scores);
  std::printf("%ld checks, %ld failures\n", g_checks, g_fail);
  if (g_fail) return 1;
  std::printf("PASSED\n");
  return 0;
}
