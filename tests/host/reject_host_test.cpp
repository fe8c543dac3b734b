// reject_host_test.cpp — the correspondence-rejector kernels (pcl_b200/csrc/reject_kernels.cuh) compiled for the HOST and run
// in reject.cu's sequence (std::stable_sort where the driver calls cub::DeviceRadixSort, a flagged copy for DeviceSelect),
// against the CPU oracle's rejectors (oracle/libpcl_oracle.so, linked: test infrastructure): the surviving records, their
// order and the reported median, bit for bit — distance ties, duplicated matches, negative matches, empty / single-record
// lists, and chains where each rejector filters the previous one's output (icp.hpp:187-201).
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <cfloat>

struct orc_rejector { int32_t kind, min_correspondences; double p; };
extern "C" size_t orc_reject(const orc_rejector* r, const pclb200_corr* in, size_t n, pclb200_corr* out, double* median_out);

// the fixed seed of the committed test, or PCLB_TEST_SEED for a fuzz run (tools/dev/fuzz_host_tests.sh)
#include "reject_twin.h"

// reject.cu: reject_standalone()
static std::vector<pclb200_corr> reject_standalone(const pclb200_rejector& r, const std::vector<pclb200_corr>& in, double& median)
{
  using namespace pclb200;
  const size_t n = in.size();
  median = 0.0;
  if (n == 0) return {};
  Arrays a;
  a.d2.resize(n); a.match.resize(n); a.acc.resize(n); a.tie.resize(n);
  std::vector<int> perm(n), keep_sorted(n);
  int trimmed = 0;
  double info[2] = {0, 0};
  launch(grid_for(n, 256), 256, [&] { k_rej_unpack(in.data(), n, a.d2.data(), a.match.data(), a.tie.data(), a.acc.data(), r.kind == PCLB200_REJ_ONE_TO_ONE ? 1 : 0); });
  apply_rejector(r, a, perm, keep_sorted, info, trimmed);
  median = info[0];
  const int use_perm = (r.kind == PCLB200_REJ_ONE_TO_ONE) || (r.kind == PCLB200_REJ_TRIMMED && trimmed);
  std::vector<pclb200_corr> staged(n), out;
  std::vector<unsigned char> flag(n);
  launch(grid_for(n, 256), 256, [&] { k_rej_flag_in_order(a.acc.data(), perm.data(), keep_sorted.data(), n, use_perm, in.data(), staged.data(), flag.data()); });
  for (size_t j = 0; j < n; ++j) if (flag[j]) out.push_back(staged[j]);
  return out;
}

static const char* kind_name(int k) { static const char* s[] = {"distance", "median", "one-to-one", "trimmed"}; return s[k]; }

static void compare(const char* scene, const pclb200_rejector& r, const std::vector<pclb200_corr>& in)
{
  double med = -7, omed = -7;
  const std::vector<pclb200_corr> got = reject_standalone(r, in, med);
  std::vector<pclb200_corr> want(in.size() ? in.size() : 1);
  const orc_rejector o{r.kind, r.min_correspondences, r.p};
  want.resize(orc_reject(&o, in.data(), in.size(), want.data(), &omed));
  if (in.empty()) omed = 0.0;
  CHECK(got.size() == want.size(), "%s / %s p=%g: %zu survivors, the oracle keeps %zu", scene, kind_name(r.kind), r.p, got.size(), want.size());
  size_t bad = 0;
  for (size_t i = 0; i < got.size() && i < want.size(); ++i) bad += std::memcmp(&got[i], &want[i], sizeof(pclb200_corr)) != 0;
  CHECK(bad == 0, "%s / %s p=%g: %zu records differ", scene, kind_name(r.kind), r.p, bad);
  if (r.kind == PCLB200_REJ_MEDIAN) CHECK(std::memcmp(&med, &omed, 8) == 0, "%s: median %.17g, the oracle's %.17g", scene, med, omed);
}

int main(int argc, char** argv)
{
  const int scale = argc > 1 ? std::atoi(argv[1]) : 1;
  std::mt19937 rng(test_seed(2718));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  struct Scene { const char* name; std::vector<pclb200_corr> c; };
  std::vector<Scene> scenes;
  auto make = [&](const char* name, int n, int n_targets, int levels, bool negatives) {
    Scene s{name, {}};
    for (int i = 0; i < n; ++i) {
      float d = U(rng) * U(rng) * 0.01f;
      if (levels > 0) d = std::floor(d * 100.f * levels) / (100.f * levels);   // few distinct distances: ties everywhere
      int m = (int)(U(rng) * n_targets);
      if (negatives && i % 11 == 3) m = -1;
      s.c.push_back(pclb200_corr{i, m, d});
    }
    scenes.push_back(std::move(s));
  };
  make("random, targets shared ~3x", 3000 * scale, 1000 * scale, 0, false);
  make("distance ties (12 levels)", 2500 * scale, 600 * scale, 12, false);
  make("all to one target", 700, 1, 4, false);
  make("one-to-one already", 900, 1 << 30, 0, false);
  make("negative matches", 1500, 400, 6, true);
  make("single record", 1, 5, 0, false);
  make("two records", 2, 1, 1, false);
  make("exactly one block", 256, 64, 3, false);
  make("one past a block", 257, 64, 3, false);
  scenes.push_back(Scene{"empty", {}});
  {
    Scene s{"every distance equal", {}};
    for (int i = 0; i < 1200; ++i) s.c.push_back(pclb200_corr{i, i % 300, 0.0025f});
    scenes.push_back(std::move(s));
  }
  {  // any non-NaN distance a caller may pass: -0.0 equal to +0.0, negatives before zero, +inf after FLT_MAX
    Scene s{"signed distances, -0.0, inf", {}};
    const float v[] = {0.f, -0.f, -1e-3f, 2e-3f, -2e-3f, 1e-40f, -1e-40f, FLT_MAX, INFINITY, -INFINITY, 5e-4f, -0.f};
    for (int i = 0; i < 600; ++i) s.c.push_back(pclb200_corr{i, (int)(U(rng) * 150), v[i % 12]});
    scenes.push_back(std::move(s));
  }
  for (const Scene& s : scenes) {
    const long f0 = g_fail;
    for (double p : {0.03, 0.05, 0.0, 1.0}) compare(s.name, pclb200_rejector{PCLB200_REJ_DISTANCE, 0, p}, s.c);
    for (double p : {1.0, 1.5, 0.5, 0.0}) compare(s.name, pclb200_rejector{PCLB200_REJ_MEDIAN, 0, p}, s.c);
    compare(s.name, pclb200_rejector{PCLB200_REJ_ONE_TO_ONE, 0, 0.0}, s.c);
    for (double p : {0.5, 0.9, 1.0, 0.0, 0.3333}) for (int mn : {0, 7, 100000}) compare(s.name, pclb200_rejector{PCLB200_REJ_TRIMMED, mn, p}, s.c);
    // chains: each rejector sees the previous one's output
    const pclb200_rejector chains[3][3] = {{{PCLB200_REJ_MEDIAN, 0, 1.2}, {PCLB200_REJ_ONE_TO_ONE, 0, 0}, {PCLB200_REJ_TRIMMED, 3, 0.8}},
                                           {{PCLB200_REJ_ONE_TO_ONE, 0, 0}, {PCLB200_REJ_DISTANCE, 0, 0.06}, {PCLB200_REJ_MEDIAN, 0, 2.0}},
                                           {{PCLB200_REJ_TRIMMED, 0, 0.7}, {PCLB200_REJ_MEDIAN, 0, 1.0}, {PCLB200_REJ_ONE_TO_ONE, 0, 0}}};
    for (const auto& ch : chains) {
      std::vector<pclb200_corr> g = s.c, o = s.c;
      for (const pclb200_rejector& r : ch) {
        double m1, m2 = 0;
        g = reject_standalone(r, g, m1);
        std::vector<pclb200_corr> t(o.size() ? o.size() : 1);
        const orc_rejector orr{r.kind, r.min_correspondences, r.p};
        t.resize(o.empty() ? 0 : orc_reject(&orr, o.data(), o.size(), t.data(), &m2));
        o.swap(t);
      }
      CHECK(g.size() == o.size() && (g.empty() || std::memcmp(g.data(), o.data(), g.size() * sizeof(pclb200_corr)) == 0), "%s: chain starting with %s differs (%zu vs %zu)", s.name,
            kind_name(ch[0].kind), g.size(), o.size());
    }
    std::printf("%-30s %6zu records  %s\n", s.name, s.c.size(), g_fail == f0 ? "ok" : "DIFFERS");
  }
  std::printf("%ld checks, %ld failures\n%s\n", g_checks, g_fail, g_fail ? "FAILED" : "PASSED");
  return g_fail ? 1 : 0;
}
