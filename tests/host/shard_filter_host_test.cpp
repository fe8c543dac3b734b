// shard_filter_host_test.cpp — the kernels of k-NN queries and outlier filters over a sharded map (pcl_b200/csrc/
// shard_filter_kernels.cuh) compiled for the HOST and run in shard_filter.cu's sequence for R = 1, 2, 3, 5, 8 simulated
// ranks in one process, under both exchange protocols (shard_sim.h: every rank's table read directly, or the tables
// end to end in one zeroed table summed over the ranks).  It checks
//   - the id mapping: every record number of a k-NN row becomes the local map's id of that record, padding -1 stays;
//     a tile's ids come out of its Morton array with the padding's sentinel;
//   - the SOR sums: every rank's partials (a fixed-order grid sum over its queries), the exchange and the rank-order fold
//     give every rank the same (valid, mean, thr), bit for bit, within 1e-12 relative of the reference's sequential
//     arithmetic over the concatenation of the ranks' queries (statistical_outlier_removal.hpp:100-112);
//   - both masks against the facade's rules (pcl_compat/pcl/filters/outlier_removal.h), negative both ways, ROR dense and
//     not, with k-th distances exactly at r^2, +inf and non-finite queries.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include "shard_sim.h"
#include "../../pcl_b200/csrc/shard_filter_kernels.cuh"

// the facade's StatisticalOutlierRemoval::classify arithmetic over one process's distances (outlier_removal.h)
static void facade_sor(const std::vector<float>& d, long long valid, double std_mul, double out[3])
{
  double sum = 0, sq_sum = 0;
  for (const float& x : d) {
    sum += x;
    sq_sum += x * x;
  }
  const double mean = sum / static_cast<double>(valid);
  const double variance = (sq_sum - sum * sum / static_cast<double>(valid)) / (static_cast<double>(valid) - 1);
  out[0] = (double)valid;
  out[1] = mean;
  out[2] = mean + std_mul * std::sqrt(variance);
}
static unsigned char facade_sor_keep(float d, double thr, bool negative)
{
  return ((!negative && d > thr) || (negative && d <= thr)) ? 0 : 1;
}
// the facade's RadiusOutlierRemoval::classify rule for one query
static unsigned char facade_ror_keep(const float4& p, float kth, bool is_dense, double radius, bool negative)
{
  const double nn_dists_max = radius * radius;
  const float r2f = static_cast<float>(radius * radius);
  if (is_dense) {
    if (std::isfinite(kth)) {
      if ((!negative && nn_dists_max < kth) || (negative && nn_dists_max >= kth)) return 0;
    }
    else if (!negative) return 0;
    return 1;
  }
  if (!finite3(p)) return 0;
  const bool enough = kth < r2f;
  return ((!negative && !enough) || (negative && enough)) ? 0 : 1;
}

static void run_ids(std::mt19937& rng)
{
  using namespace pclb200;
  // a local map of 700 records whose ids ascend with gaps; rows of k = 9 with padding
  std::vector<unsigned> local_ids;
  unsigned id = 3;
  for (int i = 0; i < 700; ++i) local_ids.push_back(id += 1 + rng() % 50);
  local_ids.back() = 2147483646u;
  std::vector<int32_t> rows(300 * 9), want(rows.size());
  for (size_t i = 0; i < rows.size(); ++i) {
    rows[i] = (i % 9 >= 7 && i % 4 == 0) ? -1 : (int32_t)(rng() % local_ids.size());
    want[i] = rows[i] < 0 ? -1 : (int32_t)local_ids[rows[i]];
  }
  launch(3, 256, [&] { k_sf_row_ids(rows.data(), rows.size(), local_ids.data()); });
  CHECK(rows == want, "row ids differ");
  std::vector<float4> pts;
  std::vector<unsigned long long> want_ids;
  for (int i = 0; i < 90; ++i) {
    const int v = (i % 7 == 3) ? kSentinelIndex : (int)(rng() % 2147483647u);
    pts.push_back(make_float4(0.f, 0.f, 0.f, __int_as_float(v)));
    want_ids.push_back((unsigned)v);
  }
  std::vector<unsigned long long> got(pts.size());
  launch(1, 64, [&] { k_sf_tile_ids(pts.data(), pts.size(), got.data()); });
  CHECK(got == want_ids, "tile ids differ");
}

static void run_sor(const char* name, int R, int mode, const std::vector<std::vector<float4>>& q,
                    const std::vector<std::vector<float>>& d, double std_mul, double* worst)
{
  using namespace pclb200;
  std::vector<unsigned long long> words(R, kSorWords);
  SimTables t(mode, R, words.data(), sizeof(unsigned long long));
  for (int r = 0; r < R; ++r) {
    const size_t nq = q[r].size();
    const unsigned grid = 1 + (unsigned)(nq / 700);  // the driver's persistent grid, at host scale
    std::vector<double> partials((size_t)grid * kAccum), accum(kAccum);
    unsigned counter = 0;
    launch(grid, 256, [&] {
      k_sf_sor_partials(q[r].data(), d[r].data(), nq, GridSum{partials.data(), &counter, accum.data()}, t.local(r));
    });
    CHECK(counter == 0, "%s R=%d rank %d: the ticket counter was not reset", name, R, r);
  }
  const PeerTables view = t.publish();
  std::vector<float> all_d;
  long long valid = 0;
  for (int r = 0; r < R; ++r) {
    all_d.insert(all_d.end(), d[r].begin(), d[r].end());
    for (const float4& p : q[r]) valid += finite3(p);
  }
  double want[3];
  facade_sor(all_d, valid, std_mul, want);
  std::vector<std::array<double, 3>> got(R);
  bool same = true;
  for (int r = 0; r < R; ++r) {
    launch(1, 32, [&] { k_sf_sor_fold(peer_table_set(view), std_mul, got[r].data()); });
    same = same && std::memcmp(got[r].data(), got[0].data(), sizeof(got[0])) == 0;
  }
  CHECK(same, "%s R=%d: the ranks' statistics differ", name, R);
  CHECK(got[0][0] == want[0], "%s R=%d: valid %.17g, the facade counts %.17g", name, R, got[0][0], want[0]);
  const double rel_mean = std::fabs(got[0][1] - want[1]) / std::fabs(want[1]);
  const double rel_thr = std::fabs(got[0][2] - want[2]) / std::fabs(want[2]);
  CHECK(rel_mean <= 1e-12 && rel_thr <= 1e-12, "%s R=%d: mean %.17g vs %.17g, thr %.17g vs %.17g", name, R, got[0][1],
        want[1], got[0][2], want[2]);
  *worst = std::max(*worst, rel_thr);
  // the masks: byte for byte the facade's rule on this rank's threshold, and on the facade's own threshold away from it
  long differ = 0;
  for (int r = 0; r < R; ++r)
    for (bool negative : {false, true}) {
      std::vector<unsigned char> keep(q[r].size());
      launch(2, 256, [&] { k_sf_sor_mask(d[r].data(), d[r].size(), got[r].data(), negative, keep.data()); });
      for (size_t i = 0; i < keep.size(); ++i) {
        differ += keep[i] != facade_sor_keep(d[r][i], got[r][2], negative);
        if (std::fabs((double)d[r][i] - want[2]) > 1e-12 * std::fabs(want[2]))
          differ += keep[i] != facade_sor_keep(d[r][i], want[2], negative);
      }
    }
  CHECK(differ == 0, "%s R=%d: %ld SOR mask entries differ from the facade's", name, R, differ);
  std::printf("%-22s R=%d %-5s thr rel diff %.2e %s\n", name, R, mode == kPeer ? "peer" : "nccl", rel_thr,
              (same && differ == 0 && rel_thr <= 1e-12) ? "ok" : "DIFFERS");
}

static void run_ror(const std::vector<float4>& q, const std::vector<float>& kth, double radius)
{
  using namespace pclb200;
  for (unsigned long long dense : {0ull, 1ull})
    for (int negative : {0, 1}) {
      std::vector<unsigned char> keep(q.size());
      launch(2, 256, [&] {
        k_sf_ror_mask(q.data(), kth.data(), q.size(), &dense, radius * radius, (float)(radius * radius), negative,
                      keep.data());
      });
      long differ = 0;
      for (size_t i = 0; i < q.size(); ++i) differ += keep[i] != facade_ror_keep(q[i], kth[i], dense != 0, radius, negative != 0);
      CHECK(differ == 0, "ROR dense=%llu negative=%d: %ld entries differ from the facade's", dense, negative, differ);
    }
}

int main()
{
  std::mt19937 rng(test_seed(20261017u));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  run_ids(rng);

  // per-rank queries (some non-finite, whose mean the statistics report as 0) and mean distances: a spread of scales, a
  // cluster of equal values (exact-tie lattices give equal means) and a tail of outliers
  const int n_all = 20000;
  std::vector<float4> Q;
  std::vector<float> D;
  for (int i = 0; i < n_all; ++i) {
    float4 p = make_float4(U(rng), U(rng), U(rng), 1.f);
    float m = 0.01f + 0.004f * U(rng);
    if (i % 11 == 0) m = 0.0125f;
    if (i % 97 == 0) m = 0.05f + 0.1f * U(rng);
    if (i % 313 == 5) { p.y = NAN; m = 0.f; }
    if (i % 409 == 7) { p.z = -INFINITY; m = 0.f; }
    Q.push_back(p);
    D.push_back(m);
  }
  double worst = 0.0;
  for (int R : {1, 2, 3, 5, 8}) {
    std::vector<std::pair<const char*, std::vector<int>>> cuts;  // each: rank of every query, in rank order when concatenated
    {
      std::vector<int> a(n_all);
      for (int i = 0; i < n_all; ++i) a[i] = (int)((long long)i * R / n_all);
      cuts.push_back({"contiguous", a});
    }
    {
      std::vector<int> a(n_all);
      for (int i = 0; i < n_all; ++i) a[i] = (int)(rng() % R);
      if (R > 2) for (int i = 0; i < n_all; ++i) if (a[i] == 1) a[i] = 0;  // a rank with no query
      cuts.push_back({"random, one rank empty", a});
    }
    for (const auto& cut : cuts)
      for (int mode : {kPeer, kNccl}) {
        std::vector<std::vector<float4>> q(R);
        std::vector<std::vector<float>> d(R);
        for (int i = 0; i < n_all; ++i) { q[cut.second[i]].push_back(Q[i]); d[cut.second[i]].push_back(D[i]); }
        run_sor(cut.first, R, mode, q, d, 1.0, &worst);
        run_sor(cut.first, R, mode, q, d, 0.25, &worst);
      }
  }

  // ROR: k-th distances exactly at r^2 (float and double), just around it, +inf; finite and non-finite queries
  const double radius = 0.1;
  const float r2f = (float)(radius * radius);
  std::vector<float4> q;
  std::vector<float> kth;
  for (int i = 0; i < 4000; ++i) {
    float4 p = make_float4(U(rng), U(rng), U(rng), 1.f);
    if (i % 37 == 0) p.x = NAN;
    float k = r2f * 2.f * U(rng);
    switch (i % 9) {
      case 0: k = r2f; break;
      case 1: k = std::nextafter(r2f, 0.f); break;
      case 2: k = std::nextafter(r2f, 1.f); break;
      case 3: k = INFINITY; break;
      case 4: k = (float)(radius * radius); break;
      default: break;
    }
    q.push_back(p);
    kth.push_back(k);
  }
  run_ror(q, kth, radius);
  run_ror(q, kth, 0.125);  // r^2 exact in float

  std::printf("worst thr rel diff %.3e\n%ld checks, %ld failures\n", worst, g_checks, g_fail);
  if (g_fail == 0) std::printf("PASSED\n");
  return g_fail ? 1 : 0;
}
