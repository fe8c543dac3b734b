// shard_radius_host_test.cpp — radius search over a sharded map (pcl_b200/csrc/shard_filter.cu: radius_sharded) with its
// id mapping kernel (shard_filter_kernels.cuh: k_sf_row_ids) compiled for the HOST, for R = 1, 2, 3, 5, 8 simulated ranks
// in one process, under both exchange protocols of the halo (shard_sim.h: every rank's table read directly, or the tables
// end to end in one zeroed table summed over the ranks).  For every rank it checks
//   - the id mapping of both paths of radius_search on the local map: the sorted keys ((d2 bits << 32) | record, unpacked
//     as k_unpack_keys does) and the register k-NN rows of max_nn <= 32 (-1 padded, packed as k_pack_rows does), each
//     mapped by k_sf_row_ids, equal the brute-force lists of the whole map: ids, d2, (d2, id) order, max_nn cut;
//   - the verdict and all_fit exchanges: one u64 minimum over the ranks' words gives every rank the same verdict, a
//     refusal on one rank refuses on all, and a rank whose capacity alone is short makes all_fit 0 everywhere until it
//     grows; the lists of the ranks whose lists fitted are the same bytes on the second call.
// Scenes: random points and a lattice of spacing 1/8 (exact ties, points exactly on the sphere); partitions: slabs,
// random, overlapping tiles that share ids; queries: tile points, lattice points, far and non-finite points; a rank
// with no query.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <map>
#include <set>

#include "shard_sim.h"
#include "../../pcl_b200/csrc/shard_normals_kernels.cuh"
#include "../../pcl_b200/csrc/shard_filter_kernels.cuh"

using Entry = std::pair<float, int>;  // (d2, id or record): the library's order

// the radius list of q over pts (labels: the number each point answers with), strict d2 < r2, sorted, cut at max_nn
static std::vector<Entry> ball(const std::vector<float4>& pts, const std::vector<int>& labels, const float4& q, float r2,
                               size_t max_nn)
{
  std::vector<Entry> out;
  if (!finite3(q)) return out;
  for (size_t i = 0; i < pts.size(); ++i) {
    const float d = d2_of(q, pts[i]);
    if (d < r2) out.push_back({d, labels[i]});
  }
  std::sort(out.begin(), out.end());
  if (max_nn && out.size() > max_nn) out.resize(max_nn);
  return out;
}

// one rank's local map: its tile and every point of the other tiles in the box of its queries widened by the reach of
// r2 (the selection of shard_normals_host_test.cpp, checked there against the kernels under both protocols), sorted by
// id, each id once
static std::vector<float4> local_map(const std::vector<std::vector<float4>>& tiles, int r, const std::vector<float4>& q,
                                     float r2, int mode)
{
  using namespace pclb200;
  const int R = (int)tiles.size();
  std::vector<unsigned long long> box(kHaloBoxWords, kNoHaloBox);
  if (r2 > 0.f) launch(2, 64, [&] { k_halo_box(q.data(), nullptr, r2, q.size(), box.data()); });
  std::vector<unsigned long long> boxes((size_t)kHaloBoxWords * R, kNoHaloBox);
  std::copy(box.begin(), box.end(), boxes.begin() + (size_t)kHaloBoxWords * r);
  // every sender's points for rank r through the tables of the protocol
  std::vector<unsigned long long> cnt((size_t)R * R, 0);
  for (int s = 0; s < R; ++s) {
    HaloOut o;
    std::memset(&o, 0, sizeof o);
    o.count = cnt.data() + (size_t)R * s;
    launch(2, 64, [&] { k_halo_select(tiles[s].data(), tiles[s].size(), boxes.data(), R, s, o); });
  }
  const std::vector<unsigned long long> n_table = segment_table_sizes(cnt.data(), R);
  SimTables t(mode, R, n_table.data(), sizeof(float4));
  std::vector<float4> self(tiles[r].size());
  for (int s = 0; s < R; ++s) {
    std::vector<unsigned long long> cursor(R, 0);
    std::vector<float4> own(tiles[s].size());
    HaloOut o;
    std::memset(&o, 0, sizeof o);
    o.count = cursor.data();
    o.dst[s] = own.data();
    segment_writes(reinterpret_cast<float4*>(t.local(s)), cnt.data(), R, s, o.dst);
    launch(2, 64, [&] { k_halo_select(tiles[s].data(), tiles[s].size(), boxes.data(), R, s, o); });
    if (s == r) self = own;
  }
  const PeerTables view = t.publish();
  const PeerSegments<float4> rs = segment_reads<float4>(view, cnt.data(), R, r);
  std::vector<float4> all = self;
  all.resize(self.size() + rs.begin[rs.n]);
  launch(2, 64, [&] { k_gather_segments(rs, all.data() + self.size()); });
  std::map<int, float4> by_id;
  for (const float4& p : all) by_id.emplace(id_of(p), p);
  std::vector<float4> out;
  for (const auto& kv : by_id) out.push_back(kv.second);
  return out;
}

// one rank's call: offsets and mapped ids / d2 as radius_sharded delivers them; rows: the register k-NN path
static void rank_lists(const std::vector<float4>& local, const std::vector<float4>& q, float r2, size_t max_nn, bool rows,
                       std::vector<long long>& off, std::vector<int32_t>& idx, std::vector<float>& d2)
{
  std::vector<int> rec(local.size());
  std::vector<unsigned> local_ids(local.size());
  for (size_t i = 0; i < local.size(); ++i) { rec[i] = (int)i; local_ids[i] = (unsigned)id_of(local[i]); }
  off.assign(1, 0);
  idx.clear();
  d2.clear();
  for (const float4& p : q) {
    const std::vector<Entry> b = ball(local, rec, p, r2, max_nn);
    if (rows) {  // a k-NN row of k = max_nn, -1 padded, packed from the front (k_pack_rows)
      std::vector<int32_t> row(max_nn, -1);
      for (size_t j = 0; j < b.size(); ++j) row[j] = b[j].second;
      for (size_t j = 0; j < max_nn && row[j] >= 0; ++j) { idx.push_back(row[j]); d2.push_back(b[j].first); }
    }
    else  // the sorted keys of the ball, unpacked (k_unpack_keys: the low 32 bits, the high 32 bits as a float)
      for (const Entry& e : b) {
        const unsigned long long key = (unsigned long long)__float_as_int(e.first) << 32 | (unsigned)e.second;
        idx.push_back((int32_t)(unsigned)(key & 0xffffffffULL));
        d2.push_back(__int_as_float((int)(unsigned)(key >> 32)));
      }
    off.push_back((long long)idx.size());
  }
  launch(3, 256, [&] { pclb200::k_sf_row_ids(idx.data(), idx.size(), local_ids.data()); });
}

static unsigned long long ranks_min(const std::vector<unsigned long long>& words)
{
  return *std::min_element(words.begin(), words.end());
}

static void run_case(const char* name, const std::vector<std::vector<float4>>& tiles,
                     const std::vector<std::vector<float4>>& queries, float r2, size_t max_nn, int mode)
{
  const int R = (int)tiles.size();
  std::vector<float4> whole;
  {
    std::map<int, float4> by_id;
    for (const auto& t : tiles) for (const float4& p : t) by_id[id_of(p)] = p;
    for (const auto& kv : by_id) whole.push_back(kv.second);
  }
  std::vector<int> whole_ids(whole.size());
  for (size_t i = 0; i < whole.size(); ++i) whole_ids[i] = id_of(whole[i]);
  long bad = 0;
  std::vector<unsigned long long> totals(R);
  std::vector<std::vector<int32_t>> first_idx(R);
  for (int r = 0; r < R; ++r) {
    const std::vector<float4> local = local_map(tiles, r, queries[r], r2, mode);
    // the whole map's lists
    std::vector<long long> want_off(1, 0);
    std::vector<int32_t> want_idx;
    std::vector<float> want_d2;
    for (const float4& p : queries[r]) {
      for (const Entry& e : ball(whole, whole_ids, p, r2, max_nn)) { want_idx.push_back(e.second); want_d2.push_back(e.first); }
      want_off.push_back((long long)want_idx.size());
    }
    for (bool rows : {false, true}) {
      if (rows && (max_nn == 0 || max_nn > 32)) continue;
      std::vector<long long> off;
      std::vector<int32_t> idx;
      std::vector<float> d2;
      rank_lists(local, queries[r], r2, max_nn, rows, off, idx, d2);
      const bool same = off == want_off && idx == want_idx && d2.size() == want_d2.size() &&
                        (d2.empty() || std::memcmp(d2.data(), want_d2.data(), d2.size() * sizeof(float)) == 0);
      CHECK(same, "%s R=%d rank %d r2 %g max_nn %zu %s: the lists differ from the whole map's", name, R, r, r2, max_nn,
            rows ? "rows" : "keys");
      bad += !same;
      if (!rows) { totals[r] = idx.size(); first_idx[r] = idx; }
    }
  }
  // the verdict: one rank refuses, every rank refuses; none refuses, every rank goes on
  for (int bad_rank = -1; bad_rank < R; ++bad_rank) {
    std::vector<unsigned long long> words(R);
    for (int r = 0; r < R; ++r) words[r] = r == bad_rank ? 0 : 1;
    CHECK(ranks_min(words) == (bad_rank < 0 ? 1ull : 0ull), "%s R=%d: verdict with rank %d refusing", name, R, bad_rank);
  }
  // all_fit: rank R - 1 alone is one entry short, then grows to its total; the others' lists fit both times
  if (totals[R - 1] > 0) {
    std::vector<unsigned long long> cap(R), words(R);
    for (int r = 0; r < R; ++r) cap[r] = r == R - 1 ? totals[r] - 1 : totals[r] + 3;
    for (int r = 0; r < R; ++r) words[r] = totals[r] <= cap[r] ? 1 : 0;
    CHECK(ranks_min(words) == 0, "%s R=%d: all_fit with a short rank", name, R);
    cap[R - 1] = totals[R - 1];
    for (int r = 0; r < R; ++r) words[r] = totals[r] <= cap[r] ? 1 : 0;
    CHECK(ranks_min(words) == 1, "%s R=%d: all_fit after growing", name, R);
    for (int r = 0; r < R - 1; ++r) {
      const std::vector<float4> local = local_map(tiles, r, queries[r], r2, mode);
      std::vector<long long> off;
      std::vector<int32_t> idx;
      std::vector<float> d2;
      rank_lists(local, queries[r], r2, max_nn, false, off, idx, d2);
      CHECK(idx == first_idx[r], "%s R=%d rank %d: the second call's lists differ", name, R, r);
    }
  }
  std::printf("%-22s R=%d %-5s r2=%-10.4g max_nn=%-4zu %s\n", name, R, mode == kPeer ? "peer" : "nccl", r2, max_nn,
              bad ? "DIFFERS" : "ok");
}

int main()
{
  std::mt19937 rng(test_seed(20261017u));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::vector<float4> map;
  for (int i = 0; i < 400; ++i) map.push_back(make_float4(U(rng), U(rng), U(rng), 0.f));
  for (int i = 0; i < 8; ++i)
    for (int j = 0; j < 8; ++j)
      for (int l = 0; l < 3; ++l) map.push_back(make_float4(0.125f * i, 0.125f * j, 0.25f + 0.125f * l, 0.f));
  for (int i = 0; i < 20; ++i) map.push_back(map[i * 7]);  // the same point under another id: exact ties
  std::vector<int> ids(map.size());
  for (size_t i = 0; i < ids.size(); ++i) ids[i] = (int)(i * 7919 + 5);
  ids[1] = 2147483646;
  std::shuffle(ids.begin(), ids.end(), rng);
  for (size_t i = 0; i < map.size(); ++i) map[i].w = __int_as_float(ids[i]);
  std::vector<float4> extra;
  for (int i = 0; i < 6; ++i) extra.push_back(make_float4(0.125f * i, 0.375f, 0.375f, 0.f));
  extra.push_back(make_float4(5.f, 5.f, 5.f, 0.f));
  extra.push_back(make_float4(NAN, 0.f, 0.f, 0.f));
  for (int R : {1, 2, 3, 5, 8}) {
    std::vector<std::pair<const char*, std::vector<std::vector<float4>>>> parts;
    {
      std::vector<std::vector<float4>> t(R);
      for (const float4& p : map) t[std::min(R - 1, (int)(p.x * R))].push_back(p);
      parts.push_back({"slabs", t});
    }
    {
      std::vector<std::vector<float4>> t(R);
      for (const float4& p : map) t[rng() % R].push_back(p);
      parts.push_back({"random", t});
    }
    if (R > 1) {
      std::vector<std::vector<float4>> t(R);
      for (const float4& p : map) {
        const int r = std::min(R - 1, (int)(p.x * R));
        t[r].push_back(p);
        if (r + 1 < R && p.x * R > r + 0.8f) t[r + 1].push_back(p);
      }
      parts.push_back({"overlapping", t});
    }
    for (const auto& pt : parts) {
      std::vector<std::vector<float4>> queries(R);
      for (int r = 0; r < R; ++r) {
        for (size_t i = 0; i < pt.second[r].size(); i += 3) queries[r].push_back(pt.second[r][i]);
        if (r % 2 == 0) queries[r].insert(queries[r].end(), extra.begin(), extra.end());
      }
      if (R > 2) queries[1].clear();  // a rank with no query
      for (int mode : {kPeer, kNccl})
        for (const auto& c : std::vector<std::pair<float, size_t>>{{0.125f * 0.125f, 0}, {0.125f * 0.125f, 5},
                                                                    {0.2f * 0.2f, 32}, {0.2f * 0.2f, 40}, {0.f, 0},
                                                                    {0.05f * 0.05f, 1}})
          run_case(pt.first, pt.second, queries, c.first, c.second, mode);
    }
  }
  std::printf("%ld checks, %ld failures\n", g_checks, g_fail);
  if (g_fail == 0) std::printf("PASSED\n");
  return g_fail ? 1 : 0;
}
