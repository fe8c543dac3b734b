// reject_sharded_host_test.cpp — the sharded rejector kernels (pcl_b200/csrc/reject_sharded_kernels.cuh) compiled for the HOST
// and run in reject.cu's apply_rejector_sharded sequence for R = 1, 2, 3, 5, 8 simulated ranks in one process: this program
// does the cross-rank sum (histograms) and min (one-to-one tables) where comm.cu would exchange them, for both one-to-one
// protocols (peer tables read directly; the NCCL minimum).  The union of every rank's survivors must equal the CPU oracle's
// rejector (oracle/libpcl_oracle.so, linked: test infrastructure) on the concatenation of the shards in rank order, record
// for record, and the median must be the oracle's — for every rejector, trimmed with keep = 0, 1, c - 1, c, and chains.
// Inputs: runs of exact distance ties, several queries per target, entries that are not accepted, ranks with no accepted
// entry, array order different from slot order (the ICP's Morton order), target positions different from target indices.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <array>
#include <numeric>

static inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) { const unsigned long long o = *p; if (v < o) *p = v; return o; }
template <typename T> static inline T __ldcv(const T* p) { return *p; }

struct orc_rejector { int32_t kind, min_correspondences; double p; };
extern "C" size_t orc_reject_chain(const orc_rejector* r, int n_r, const pclb200_corr* in, size_t n, pclb200_corr* out,
                                   double* median_out);

#include "reject_twin.h"
#include "../../pcl_b200/csrc/reject_sharded_kernels.cuh"

// one rank's arrays, as run_rejectors builds them from the Match array (index i = Morton order of the queries)
struct Rank {
  size_t n = 0;
  unsigned long long offset = 0;
  std::vector<float> d2;
  std::vector<int> mt, acc;      // mt = position of the target in the (Morton-ordered) target array
  std::vector<unsigned> tie;     // slot
};
struct World {
  std::vector<Rank> ranks;
  std::vector<float4> tgt_pts;   // w = original index bits
  size_t n_cloud = 0;
};

enum { kPeer = 0, kNccl = 1 };

// reject.cu: apply_rejector_sharded, every rank in turn, the exchanges done here
static void apply_sharded(World& w, const pclb200_rejector& r, int o2o_mode, double* median)
{
  using namespace pclb200;
  const int R = (int)w.ranks.size();
  if (r.kind == PCLB200_REJ_DISTANCE) {  // local
    const float md = (float)r.p * (float)r.p;
    for (Rank& k : w.ranks) launch(grid_for(k.n, 256), 256, [&] { k_rej_distance(k.d2.data(), k.acc.data(), k.n, md); });
    return;
  }
  if (r.kind == PCLB200_REJ_MEDIAN || r.kind == PCLB200_REJ_TRIMMED) {
    const bool wide = r.kind == PCLB200_REJ_TRIMMED;
    const int passes = (wide ? 64 : 32) / kSelDigitBits;
    std::vector<std::vector<unsigned long long>> hist(R, std::vector<unsigned long long>(kSelBins, 0));
    std::vector<SelState> sel(R);
    std::vector<std::array<double, 2>> info(R);
    std::memset(sel.data(), 0, sel.size() * sizeof(SelState));
    for (int p = 0; p < passes; ++p) {
      const int shift = (passes - 1 - p) * kSelDigitBits;
      for (int q = 0; q < R; ++q) {
        Rank& k = w.ranks[q];
        const unsigned g = std::min<unsigned>(std::max(1u, grid_for(k.n, 256)), 3u);  // a few blocks: several flushes
        if (wide) launch(g, 256, [&] { k_sel_hist<true>(k.d2.data(), k.tie.data(), k.acc.data(), k.n, k.offset, shift, p == 0, &sel[q], hist[q].data()); });
        else launch(g, 256, [&] { k_sel_hist<false>(k.d2.data(), k.tie.data(), k.acc.data(), k.n, k.offset, shift, p == 0, &sel[q], hist[q].data()); });
      }
      std::vector<unsigned long long> sum(kSelBins, 0);   // comm_allreduce_u64(sum)
      for (int q = 0; q < R; ++q) for (int b = 0; b < kSelBins; ++b) sum[b] += hist[q][b];
      for (int q = 0; q < R; ++q) {
        hist[q] = sum;
        k_sel_decide(hist[q].data(), shift, p == 0, p == passes - 1, r.kind, std::min(1.0f, std::max(0.0f, (float)r.p)), (unsigned)r.min_correspondences, r.p, &sel[q], info[q].data());
        for (int b = 0; b < kSelBins; ++b) CHECK(hist[q][b] == 0, "histogram not cleared");
      }
    }
    for (int q = 1; q < R; ++q) CHECK(std::memcmp(&sel[q], &sel[0], sizeof(SelState)) == 0, "ranks disagree on the selection");
    for (int q = 0; q < R; ++q) {
      Rank& k = w.ranks[q];
      if (wide) launch(grid_for(k.n, 256), 256, [&] { k_sel_trim_apply(k.d2.data(), k.tie.data(), k.acc.data(), k.n, k.offset, &sel[q]); });
      else launch(grid_for(k.n, 256), 256, [&] { k_rej_threshold(k.d2.data(), k.acc.data(), k.n, info[q].data()); });
    }
    if (median && !wide) *median = info[0][0];
    return;
  }
  // ONE_TO_ONE
  std::vector<std::vector<unsigned long long>> table(R, std::vector<unsigned long long>(w.n_cloud, ~0ull));
  std::vector<unsigned long long> recv(w.n_cloud);
  for (int q = 0; q < R; ++q) {
    Rank& k = w.ranks[q];
    launch(grid_for(k.n, 256), 256, [&] { k_o2o_min(k.d2.data(), k.tie.data(), k.mt.data(), k.acc.data(), k.n, k.offset, w.tgt_pts.data(), table[q].data()); });
  }
  PeerTables tabs;
  if (o2o_mode == kPeer) {  // barrier, then every rank reads every table
    tabs.n_read = R;
    for (int q = 0; q < R; ++q) tabs.read[q] = table[q].data();
  }
  else {                    // ncclAllReduce(min) of the tables into recv
    for (size_t t = 0; t < w.n_cloud; ++t) { unsigned long long m = ~0ull; for (int q = 0; q < R; ++q) m = std::min(m, table[q][t]); recv[t] = m; }
    tabs.n_read = 1;
    tabs.read[0] = recv.data();
  }
  for (int q = 0; q < R; ++q) {
    Rank& k = w.ranks[q];
    launch(grid_for(k.n, 256), 256, [&] { k_o2o_keep(k.d2.data(), k.tie.data(), k.mt.data(), k.acc.data(), k.n, k.offset, w.tgt_pts.data(), peer_table_set(tabs)); });
  }
  for (int q = 0; q < R; ++q) {  // second barrier, sparse reset: the table must be all ~0 again
    Rank& k = w.ranks[q];
    launch(grid_for(k.n, 256), 256, [&] { k_o2o_reset(k.mt.data(), k.n, w.tgt_pts.data(), table[q].data()); });
    size_t dirty = 0;
    for (unsigned long long v : table[q]) dirty += v != ~0ull;
    CHECK(dirty == 0, "rank %d: %zu table entries left after the reset", q, dirty);
  }
}

// the accepted entries of all ranks as the single process sees them: ordered by global position offset + slot
static std::vector<pclb200_corr> survivors(const World& w)
{
  std::vector<pclb200_corr> out;
  for (const Rank& k : w.ranks)
    for (size_t i = 0; i < k.n; ++i)
      if (k.acc[i]) out.push_back(pclb200_corr{(int)(k.offset + k.tie[i]), __float_as_int(w.tgt_pts[k.mt[i]].w), k.d2[i]});
  std::sort(out.begin(), out.end(), [](const pclb200_corr& a, const pclb200_corr& b) { return a.index_query < b.index_query; });
  return out;
}

// the oracle's chain of the ICP loop: every stage sees the survivors in position order, and so does the result
static std::vector<pclb200_corr> oracle(const std::vector<pclb200_rejector>& chain, const std::vector<pclb200_corr>& in,
                                        double* median)
{
  std::vector<pclb200_corr> out(in.size() ? in.size() : 1);
  std::vector<orc_rejector> o;
  for (const pclb200_rejector& r : chain) o.push_back(orc_rejector{r.kind, r.min_correspondences, r.p});
  double m = 0.0;
  out.resize(in.empty() ? 0 : orc_reject_chain(o.data(), (int)o.size(), in.data(), in.size(), out.data(), &m));
  if (median) *median = m;
  return out;
}

static bool same(const std::vector<pclb200_corr>& a, const std::vector<pclb200_corr>& b)
{
  return a.size() == b.size() && (a.empty() || std::memcmp(a.data(), b.data(), a.size() * sizeof(pclb200_corr)) == 0);
}

static const char* kind_name(int k) { static const char* s[] = {"distance", "median", "one-to-one", "trimmed"}; return s[k]; }

// every chain on the world, for both one-to-one protocols; each chain starts from the world's acceptance flags
static void check_chain(const char* scene, const World& w0, const std::vector<pclb200_rejector>& chain)
{
  for (int mode : {kPeer, kNccl}) {
    World w = w0;
    double med = -7, omed = -8;
    const std::vector<pclb200_corr> in = survivors(w);
    for (const pclb200_rejector& r : chain)
      apply_sharded(w, r, mode, &med);
    const std::vector<pclb200_corr> o = oracle(chain, in, &omed);
    if (chain.size() == 1 && chain[0].kind == PCLB200_REJ_MEDIAN && !in.empty())
      CHECK(std::memcmp(&med, &omed, 8) == 0, "%s, R=%zu: median %.9g, the oracle's %.9g", scene, w.ranks.size(), med, omed);
    const std::vector<pclb200_corr> g = survivors(w);
    CHECK(same(g, o), "%s, R=%zu, %s, chain of %zu starting with %s p=%g min=%d: %zu survivors, the oracle keeps %zu", scene,
          w.ranks.size(), mode == kPeer ? "peer tables" : "NCCL min", chain.size(), kind_name(chain[0].kind), chain[0].p,
          chain[0].min_correspondences, g.size(), o.size());
  }
}

int main()
{
  std::mt19937 rng(test_seed(31337));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  struct Spec { const char* name; int n; int n_targets; int levels; double p_acc; };
  const Spec specs[] = {{"random distances", 2400, 800, 0, 0.8},
                        {"distance ties (6 levels)", 2000, 300, 6, 0.9},
                        {"every distance equal", 900, 200, -1, 1.0},
                        {"all to one target", 500, 1, 3, 0.7},
                        {"sparse acceptance", 1500, 2000, 4, 0.05},
                        {"tiny", 7, 3, 2, 0.6}};
  for (const Spec& sp : specs) {
    for (int R : {1, 2, 3, 5, 8}) {
      World w;
      // target: positions permuted against original indices
      w.n_cloud = (size_t)sp.n_targets + 3;
      std::vector<int> orig(w.n_cloud);
      std::iota(orig.begin(), orig.end(), 0);
      std::shuffle(orig.begin(), orig.end(), rng);
      for (size_t p = 0; p < w.n_cloud; ++p) w.tgt_pts.push_back(make_float4(0.f, 0.f, 0.f, __int_as_float(orig[p])));
      // uneven shards, every rank >= 1 query; rank 1 (if any) accepts nothing
      std::vector<size_t> cuts{0};
      for (int q = 1; q < R; ++q) cuts.push_back((size_t)(sp.n * (double)q * q / ((double)R * R)) + (size_t)q);
      cuts.push_back((size_t)sp.n + (size_t)R);
      unsigned long long off = 0;
      for (int q = 0; q < R; ++q) {
        Rank k;
        k.n = cuts[q + 1] - cuts[q];
        k.offset = off;
        off += k.n;
        std::vector<unsigned> slots(k.n);
        std::iota(slots.begin(), slots.end(), 0u);
        std::shuffle(slots.begin(), slots.end(), rng);   // array order = Morton order of the queries, not slot order
        for (size_t i = 0; i < k.n; ++i) {
          float d = U(rng) * U(rng) * 0.01f;
          if (sp.levels > 0) d = std::floor(d * 100.f * sp.levels) / (100.f * sp.levels);
          if (sp.levels < 0) d = 0.0025f;
          const bool matched = U(rng) < 0.97f;
          k.d2.push_back(d);
          k.mt.push_back(matched ? (int)(U(rng) * sp.n_targets) % (int)w.n_cloud : -1);
          k.tie.push_back(slots[i]);
          k.acc.push_back(matched && U(rng) < sp.p_acc && !(R > 2 && q == 1) ? 1 : 0);
        }
        w.ranks.push_back(std::move(k));
      }
      const long f0 = g_fail;
      const size_t c = survivors(w).size();
      for (double p : {0.03, 0.05, 0.0}) check_chain(sp.name, w, {{PCLB200_REJ_DISTANCE, 0, p}});
      for (double p : {1.0, 1.5, 0.5, 0.0, 3.0}) check_chain(sp.name, w, {{PCLB200_REJ_MEDIAN, 0, p}});
      check_chain(sp.name, w, {{PCLB200_REJ_ONE_TO_ONE, 0, 0.0}});
      // trimmed: keep = 0, 1, c - 1, c, and the usual ratios
      check_chain(sp.name, w, {{PCLB200_REJ_TRIMMED, 0, 0.0}});
      check_chain(sp.name, w, {{PCLB200_REJ_TRIMMED, 1, 0.0}});
      check_chain(sp.name, w, {{PCLB200_REJ_TRIMMED, (int)(c > 0 ? c - 1 : 0), 0.0}});
      check_chain(sp.name, w, {{PCLB200_REJ_TRIMMED, 0, 1.0}});
      for (double p : {0.5, 0.9, 0.3333}) for (int mn : {0, 7, 100000}) check_chain(sp.name, w, {{PCLB200_REJ_TRIMMED, mn, p}});
      check_chain(sp.name, w, {{PCLB200_REJ_MEDIAN, 0, 3.0}, {PCLB200_REJ_ONE_TO_ONE, 0, 0}, {PCLB200_REJ_TRIMMED, 100, 0.9}, {PCLB200_REJ_DISTANCE, 0, 0.2}});
      check_chain(sp.name, w, {{PCLB200_REJ_MEDIAN, 0, 1.2}, {PCLB200_REJ_ONE_TO_ONE, 0, 0}, {PCLB200_REJ_TRIMMED, 3, 0.8}});
      check_chain(sp.name, w, {{PCLB200_REJ_ONE_TO_ONE, 0, 0}, {PCLB200_REJ_DISTANCE, 0, 0.06}, {PCLB200_REJ_MEDIAN, 0, 2.0}});
      check_chain(sp.name, w, {{PCLB200_REJ_TRIMMED, 0, 0.7}, {PCLB200_REJ_MEDIAN, 0, 1.0}, {PCLB200_REJ_ONE_TO_ONE, 0, 0}});
      std::printf("%-26s R=%d %6zu accepted  %s\n", sp.name, R, c, g_fail == f0 ? "ok" : "DIFFERS");
    }
  }
  std::printf("%ld checks, %ld failures\n%s\n", g_checks, g_fail, g_fail ? "FAILED" : "PASSED");
  return g_fail ? 1 : 0;
}
