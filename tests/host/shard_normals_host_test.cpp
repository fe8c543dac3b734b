// shard_normals_host_test.cpp — the halo kernels of normal estimation over a sharded map (pcl_b200/csrc/
// shard_normals_kernels.cuh) compiled for the HOST and run in shard_normals.cu's sequence for R = 1, 2, 3, 5, 8 simulated
// ranks in one process: this program does the cross-rank steps comm.cu would do (the u64 minimum of the boxes, the sum of
// the counts, the tables of shard_sim.h), and places the segments with the layout functions of peer_tables.cuh that
// the driver calls.  For every rank it checks
//   - the box: the u64 fold of k_halo_box equals a reference fold of the outward-rounded boxes of its finite queries;
//   - the halo: exactly the points of the other tiles inside that box (a brute-force selection), each once per sender,
//     under both exchange protocols, and the tile itself is counted whole;
//   - exactness: for every query the brute-force whole-map neighbour list, every point tied at the k-th distance
//     included (radius: every point with d2 <= r2), lies in the tile plus the halo.
// Scenes: random points and a lattice whose spacing is a power of two (exact distance ties, points exactly at the k-th
// distance and exactly on box faces); partitions: slabs, random, overlapping tiles that share ids, a far tile with fewer
// than k points; k = 3, 16, 40 and a radius; queries: the tile's points, lattice points, far and non-finite points.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <map>
#include <set>

#include "shard_sim.h"
#include "../../pcl_b200/csrc/shard_normals_kernels.cuh"

// k-th smallest d2 from q over pts (+inf when fewer than k): what launch_knn_stats returns on an index of pts
static float kth_d2(const std::vector<float4>& pts, const float4& q, int k)
{
  std::vector<float> d;
  for (const float4& p : pts) d.push_back(d2_of(q, p));
  if ((int)d.size() < k) return INFINITY;
  std::nth_element(d.begin(), d.begin() + (k - 1), d.end());
  return d[k - 1];
}

// reference box of a query set: outward-rounded faces, folded as floats (not as keys)
struct RefBox { bool any = false; float lo[3], hi[3]; };
static RefBox ref_box(const std::vector<float4>& q, const std::vector<float>& rho2)
{
  RefBox b;
  for (size_t i = 0; i < q.size(); ++i) {
    if (!finite3(q[i])) continue;
    // the reach covers rho (1 + 2^-21) + 2^-61 in exact arithmetic (the bound the kernel header derives, with room)
    const float h = pclb200::halo_reach(rho2[i]);
    const double rho = std::sqrt((double)rho2[i]);
    CHECK((double)h >= rho * (1.0 + std::ldexp(1.0, -21)) + std::ldexp(1.0, -61), "reach %.9g for rho2 %.9g", h, rho2[i]);
    const float v[3] = {q[i].x, q[i].y, q[i].z};
    for (int a = 0; a < 3; ++a) {
      const float lo = __fsub_rd(v[a], h), hi = __fadd_ru(v[a], h);
      b.lo[a] = b.any ? std::min(b.lo[a], lo) : lo;
      b.hi[a] = b.any ? std::max(b.hi[a], hi) : hi;
    }
    b.any = true;
  }
  return b;
}
static bool in_ref(const RefBox& b, const float4& p)
{
  return b.any && p.x >= b.lo[0] && p.x <= b.hi[0] && p.y >= b.lo[1] && p.y <= b.hi[1] && p.z >= b.lo[2] && p.z <= b.hi[2];
}

// One scene, one partition, one neighbourhood (k > 0, or r2): every rank's halo by both protocols, checked.
static void run_case(const char* name, const std::vector<std::vector<float4>>& tiles,
                     const std::vector<std::vector<float4>>& queries, int k, float r2, int mode, std::mt19937& rng)
{
  using namespace pclb200;
  const int R = (int)tiles.size();
  std::vector<float4> whole;  // every id once
  {
    std::map<int, float4> by_id;
    for (const auto& t : tiles) for (const float4& p : t) by_id[id_of(p)] = p;
    for (const auto& kv : by_id) whole.push_back(kv.second);
  }
  // each tile as a labelled index's point array: some padding slots (+inf, w = kSentinelIndex) in between
  std::vector<std::vector<float4>> idx_pts(R);
  for (int r = 0; r < R; ++r) {
    std::vector<float4> t = tiles[r];
    std::shuffle(t.begin(), t.end(), rng);
    for (size_t i = 0; i < t.size(); ++i) {
      idx_pts[r].push_back(t[i]);
      if (i % 5 == 2) idx_pts[r].push_back(kPad);
    }
    for (int j = 0; j < 3; ++j) idx_pts[r].push_back(kPad);
  }
  // bound + boxes
  std::vector<unsigned long long> boxes((size_t)kHaloBoxWords * R, kNoHaloBox);
  std::vector<RefBox> ref(R);
  for (int r = 0; r < R; ++r) {
    const auto& q = queries[r];
    std::vector<float> rho2(q.size(), r2);
    if (k > 0)
      for (size_t i = 0; i < q.size(); ++i) rho2[i] = finite3(q[i]) ? kth_d2(tiles[r], q[i], k) : INFINITY;
    std::vector<unsigned long long> mine(kHaloBoxWords, kNoHaloBox);
    launch(2, 64, [&] { k_halo_box(q.data(), k > 0 ? rho2.data() : nullptr, r2, q.size(), mine.data()); });
    for (int a = 0; a < kHaloBoxWords; ++a) boxes[(size_t)kHaloBoxWords * r + a] = mine[a];  // the u64 minimum: one writer
    ref[r] = ref_box(q, rho2);
    bool same = ref[r].any ? mine[0] != kNoHaloBox : mine[0] == kNoHaloBox;
    for (int a = 0; a < 3 && ref[r].any && same; ++a)
      same = halo_key_value((unsigned)mine[a]) == ref[r].lo[a] &&
             halo_key_value((unsigned)(0xffffffffull - mine[3 + a])) == ref[r].hi[a];
    CHECK(same, "%s R=%d rank %d: the box differs from the reference fold", name, R, r);
  }
  // counts
  std::vector<unsigned long long> cnt((size_t)R * R, 0);
  for (int s = 0; s < R; ++s) {
    HaloOut o;
    std::memset(&o, 0, sizeof o);
    o.count = cnt.data() + (size_t)R * s;
    launch(3, 64, [&] { k_halo_select(idx_pts[s].data(), idx_pts[s].size(), boxes.data(), R, s, o); });
  }
  auto sent = [&](int s, int r) { return s == r ? 0ull : cnt[(size_t)s * R + r]; };
  unsigned long long all = 0;
  for (int s = 0; s < R; ++s) {
    for (int r = 0; r < R; ++r) all += sent(s, r);
    CHECK(cnt[(size_t)s * R + s] == tiles[s].size(), "%s R=%d rank %d: tile counted %llu of %zu", name, R, s,
          cnt[(size_t)s * R + s], tiles[s].size());
  }
  // publish: every rank writes its segments, by destination, into its table of comm_segment_tables
  const std::vector<unsigned long long> n_table = segment_table_sizes(cnt.data(), R);
  SimTables t(mode, R, n_table.data(), sizeof(float4));
  std::vector<std::vector<float4>> local(R);
  for (int s = 0; s < R; ++s) {
    local[s].assign(tiles[s].size(), make_float4(0.f, 0.f, 0.f, 0.f));
    std::vector<unsigned long long> cursor(R, 0);
    HaloOut o;
    std::memset(&o, 0, sizeof o);
    o.count = cursor.data();
    o.dst[s] = local[s].data();
    segment_writes(reinterpret_cast<float4*>(t.local(s)), cnt.data(), R, s, o.dst);
    launch(3, 64, [&] { k_halo_select(idx_pts[s].data(), idx_pts[s].size(), boxes.data(), R, s, o); });
    for (int r = 0; r < R; ++r)
      CHECK(cursor[r] == (r == s ? tiles[s].size() : sent(s, r)), "%s R=%d rank %d: wrote %llu to rank %d", name, R, s,
            cursor[r], r);
  }
  const PeerTables view = t.publish();
  long bad = 0;
  for (int r = 0; r < R; ++r) {
    const PeerSegments<float4> rs = segment_reads<float4>(view, cnt.data(), R, r);
    local[r].resize(tiles[r].size() + rs.begin[rs.n]);
    launch(2, 64, [&] { k_gather_segments(rs, local[r].data() + tiles[r].size()); });
    // the tile part: the tile, every point once
    std::multiset<int> got_tile, want_tile;
    for (size_t i = 0; i < tiles[r].size(); ++i) { got_tile.insert(id_of(local[r][i])); want_tile.insert(id_of(tiles[r][i])); }
    CHECK(got_tile == want_tile, "%s R=%d rank %d: the tile part differs", name, R, r);
    // the halo: per sender, exactly the sender's points in the reference box
    std::multiset<std::pair<int, int>> got, want;  // (id, bits of x) so a copy of the wrong point shows
    for (size_t i = tiles[r].size(); i < local[r].size(); ++i) got.insert({id_of(local[r][i]), __float_as_int(local[r][i].x)});
    for (int s = 0; s < R; ++s)
      if (s != r)
        for (const float4& p : tiles[s]) if (in_ref(ref[r], p)) want.insert({id_of(p), __float_as_int(p.x)});
    CHECK(got == want, "%s R=%d rank %d: halo of %zu points, the reference selection has %zu", name, R, r, got.size(),
          want.size());
    bad += got != want;
    // exactness: every whole-map neighbour of every query is in the local map
    std::set<int> have;
    for (const float4& p : local[r]) have.insert(id_of(p));
    for (const float4& q : queries[r]) {
      if (!finite3(q)) continue;
      const float bound = k > 0 ? kth_d2(whole, q, k) : r2;
      for (const float4& p : whole)
        if (d2_of(q, p) <= bound && !have.count(id_of(p))) {
          ++bad;
          CHECK(false, "%s R=%d rank %d: neighbour id %d (d2 %.9g <= %.9g) of query (%g %g %g) is missing", name, R, r,
                id_of(p), d2_of(q, p), bound, q.x, q.y, q.z);
        }
    }
  }
  std::printf("%-24s R=%d %-5s k=%-2d halo %-6llu %s\n", name, R, mode == kPeer ? "peer" : "nccl", k, all,
              bad ? "DIFFERS" : "ok");
}

int main()
{
  std::mt19937 rng(test_seed(20261017u));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  // the map: random points in the unit cube, and an 8 x 8 x 3 lattice of spacing 1/8 (exact squared distances: ties at
  // the k-th distance, neighbours exactly on the faces of a box whose reach is a lattice distance)
  std::vector<float4> map;
  for (int i = 0; i < 500; ++i) map.push_back(make_float4(U(rng), U(rng), U(rng), 0.f));
  for (int i = 0; i < 8; ++i)
    for (int j = 0; j < 8; ++j)
      for (int l = 0; l < 3; ++l) map.push_back(make_float4(0.125f * i, 0.125f * j, 0.25f + 0.125f * l, 0.f));
  std::vector<int> ids(map.size());
  for (size_t i = 0; i < ids.size(); ++i) ids[i] = (int)(i * 7919 + 5);
  ids[1] = 2147483646;
  std::shuffle(ids.begin(), ids.end(), rng);
  for (size_t i = 0; i < map.size(); ++i) map[i].w = __int_as_float(ids[i]);
  std::vector<float4> extra;  // queries besides the tile's own points
  for (int i = 0; i < 6; ++i) extra.push_back(make_float4(0.125f * i, 0.375f, 0.375f, 0.f));
  extra.push_back(make_float4(0.5f + 0.0625f, 0.5f, 0.375f, 0.f));
  extra.push_back(make_float4(5.f, 5.f, 5.f, 0.f));
  extra.push_back(make_float4(NAN, 0.f, 0.f, 0.f));
  extra.push_back(make_float4(0.f, -INFINITY, 0.f, 0.f));
  for (int R : {1, 2, 3, 5, 8}) {
    std::vector<std::pair<const char*, std::vector<std::vector<float4>>>> parts;
    {
      std::vector<std::vector<float4>> t(R);  // slabs along x, cut through lattice columns
      for (const float4& p : map) t[std::min(R - 1, (int)(p.x * R))].push_back(p);
      parts.push_back({"slabs", t});
    }
    {
      std::vector<std::vector<float4>> t(R);
      for (const float4& p : map) t[rng() % R].push_back(p);
      parts.push_back({"random", t});
    }
    if (R > 1) {
      std::vector<std::vector<float4>> t(R);  // overlapping slabs: points near a cut are held by both ranks, same id
      for (const float4& p : map) {
        const int r = std::min(R - 1, (int)(p.x * R));
        t[r].push_back(p);
        if (r + 1 < R && p.x * R > r + 0.8f) t[r + 1].push_back(p);
      }
      parts.push_back({"overlapping", t});
      std::vector<std::vector<float4>> f = parts[0].second;  // the last tile: 2 far points, fewer than k
      f[R - 2].insert(f[R - 2].end(), f[R - 1].begin(), f[R - 1].end());
      f[R - 1] = {make_float4(9.f, 9.f, 9.f, __int_as_float(7)), make_float4(9.f, 9.25f, 9.f, __int_as_float(11))};
      parts.push_back({"a far tile of 2 points", f});
    }
    for (const auto& pt : parts) {
      std::vector<std::vector<float4>> queries(R);
      for (int r = 0; r < R; ++r) {
        for (size_t i = 0; i < pt.second[r].size(); i += 2) queries[r].push_back(pt.second[r][i]);
        if (r % 2 == 0) queries[r].insert(queries[r].end(), extra.begin(), extra.end());
      }
      if (R > 2) queries[1].clear();  // a rank with no query still takes part
      for (int mode : {kPeer, kNccl}) {
        for (int k : {3, 16, 40}) run_case(pt.first, pt.second, queries, k, 0.f, mode, rng);
        run_case(pt.first, pt.second, queries, 0, 0.125f * 0.125f, mode, rng);  // radius 1/8: lattice points on the sphere
      }
    }
  }
  std::printf("%ld checks, %ld failures\n", g_checks, g_fail);
  if (g_fail == 0) std::printf("PASSED\n");
  return g_fail ? 1 : 0;
}
