// shard_target_host_test.cpp — the sharded-target exchange kernels (pcl_b200/csrc/shard_target_kernels.cuh) compiled for the
// HOST and run in icp.cu's exchange_shard_matches sequence for R = 1, 2, 3, 5, 8 simulated ranks in one process: this
// program does the cross-rank steps comm.cu would do, for both protocols (peer: every rank's arrays read directly; NCCL:
// min of the keys, non-winners' records zeroed, max of the records' bit patterns).  Every rank's tile match is the exact
// (d2, id) minimum of its tile within the gate (what k_search returns).  The gathered match and record of every query, on
// every rank, must be the brute-force argmin over the whole map under the (d2, id) rule, bit for bit; k_fitness_reduce must
// count exactly and sum to 1e-12.  Inputs: exact distance ties across ranks, points held by two ranks under one id,
// duplicated points under different ids, ids near 2^31 - 1, a rank with no match within the gate, spatial and random
// partitions, tile matches beyond the gate carried as kNotAccepted seeds, non-finite queries.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

static inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }

#include "shard_sim.h"
#include "../../pcl_b200/csrc/shard_target_kernels.cuh"

static unsigned blocks(size_t n) { return (unsigned)((n + 255) / 256); }

static bool same_bits(const float4& a, const float4& b) { return std::memcmp(&a, &b, sizeof(float4)) == 0; }

struct MapPoint { float4 p, n; };  // p.w = id bits
struct Best { int at = -1; float d2 = 0.f; int id = 0; };
// (d2, id) minimum over pts with d2 <= gate (gate < 0: no gate)
static Best argmin(const std::vector<MapPoint>& pts, const float4& q, float gate)
{
  Best b;
  if (!finite3(q)) return b;
  for (size_t j = 0; j < pts.size(); ++j) {
    const float d = d2_of(q, pts[j].p);
    const int id = __float_as_int(pts[j].p.w);
    if (gate >= 0.f && !(d <= gate)) continue;
    if (b.at < 0 || d < b.d2 || (d == b.d2 && id < b.id)) { b.at = (int)j; b.d2 = d; b.id = id; }
  }
  return b;
}

static void run_case(const char* name, const std::vector<std::vector<MapPoint>>& tiles, const std::vector<float4>& q,
                     float gate, bool with_normals, int mode)
{
  using namespace pclb200;
  const int R = (int)tiles.size();
  const size_t n = q.size();
  std::vector<MapPoint> whole;
  for (const auto& t : tiles) whole.insert(whole.end(), t.begin(), t.end());
  LoopCtrl ctrl;
  std::memset(&ctrl, 0, sizeof ctrl);
  // per rank: the tile match (k_search's result), the published arrays
  std::vector<std::vector<Match>> match(R, std::vector<Match>(n));
  std::vector<std::vector<float4>> tp(R), tn(R);
  std::vector<std::vector<unsigned long long>> key(R, std::vector<unsigned long long>(n, 7));
  std::vector<std::vector<float4>> rp(R, std::vector<float4>(n)), rn(R, std::vector<float4>(n));
  for (int r = 0; r < R; ++r) {
    for (const MapPoint& m : tiles[r]) { tp[r].push_back(m.p); tn[r].push_back(m.n); }
    for (size_t i = 0; i < n; ++i) {
      const Best b = argmin(tiles[r], q[i], gate);
      Match m{-1, 0.f};
      if (b.at >= 0) m = Match{b.at, b.d2};
      else {  // a carried-over seed beyond the gate (the TRACK skip test) is a match that is not accepted
        const Best any = argmin(tiles[r], q[i], -1.f);
        if (any.at >= 0 && (i % 3) == 0) m = Match{any.at | kNotAccepted, any.d2};
      }
      match[r][i] = m;
    }
  }
  auto recs = [&](int r) { return ShardRecords{key[r].data(), rp[r].data(), with_normals ? rn[r].data() : nullptr}; };
  for (int r = 0; r < R; ++r) {
    const ShardRecords mine = recs(r);
    launch(blocks(n), 256, [&] { k_shard_publish(match[r].data(), n, tp[r].data(), with_normals ? tn[r].data() : nullptr, &ctrl, mine); });
  }
  ShardReadSet rs;
  std::memset(&rs, 0, sizeof rs);
  std::vector<unsigned long long> gkey(n);
  std::vector<float4> gp(n), gn(n);
  if (mode == kPeer) {
    rs.n = R;
    for (int r = 0; r < R; ++r) { rs.key[r] = key[r].data(); rs.pts[r] = rp[r].data(); rs.nrm[r] = rn[r].data(); }
  }
  else {
    for (size_t i = 0; i < n; ++i) { unsigned long long m = ~0ull; for (int r = 0; r < R; ++r) m = std::min(m, key[r][i]); gkey[i] = m; }
    for (int r = 0; r < R; ++r) {
      const ShardRecords mine = recs(r);
      launch(blocks(n), 256, [&] { k_shard_keep_winners(gkey.data(), n, &ctrl, mine); });
    }
    auto umax = [&](std::vector<std::vector<float4>>& a, std::vector<float4>& out) {
      for (size_t i = 0; i < n; ++i) {
        unsigned w[4] = {0, 0, 0, 0};
        for (int r = 0; r < R; ++r) { unsigned x[4]; std::memcpy(x, &a[r][i], 16); for (int k = 0; k < 4; ++k) w[k] = std::max(w[k], x[k]); }
        std::memcpy(&out[i], w, 16);
      }
    };
    umax(rp, gp);
    if (with_normals) umax(rn, gn);
    rs.n = 1;
    rs.key[0] = gkey.data(); rs.pts[0] = gp.data(); rs.nrm[0] = gn.data();
  }
  long bad = 0;
  for (int r = 0; r < R; ++r) {  // every rank gathers; all must hold the same, correct answer
    std::vector<Match> gm(n, Match{12345, 1.f});
    std::vector<float4> gpts(n), gnrm(n);
    launch(blocks(n), 256, [&] { k_shard_gather(rs, n, &ctrl, gm.data(), gpts.data(), with_normals ? gnrm.data() : nullptr); });
    for (size_t i = 0; i < n; ++i) {
      const Best t = argmin(whole, q[i], gate);
      if (t.at < 0) {
        const bool ok = gm[i].pos == ((int)i | kNotAccepted) && !match_accepted(gm[i]);
        bad += !ok;
        CHECK(ok, "%s R=%d rank %d query %zu: a match where the whole map has none", name, R, r, i);
        continue;
      }
      // the lowest rank holding the winning id supplies the record; an id on two ranks names the same record anyway
      const MapPoint& w = whole[t.at];
      const bool ok = gm[i].pos == (int)i && match_accepted(gm[i]) && __float_as_int(gm[i].d2) == __float_as_int(t.d2) &&
                      same_bits(gpts[i], w.p) && (!with_normals || same_bits(gnrm[i], w.n));
      bad += !ok;
      CHECK(ok, "%s R=%d rank %d query %zu: id %d d2 %.9g, want id %d d2 %.9g", name, R, r, i, __float_as_int(gpts[i].w),
            gm[i].d2, t.id, t.d2);
    }
  }
  // fitness: the tiles' ungated nearest keys by slot, the minimum over the ranks, k_fitness_reduce's count and sum
  for (double max_range : {std::numeric_limits<double>::max(), (double)gate}) {
    std::vector<std::vector<unsigned long long>> fk(R, std::vector<unsigned long long>(n));
    for (int r = 0; r < R; ++r)
      for (size_t i = 0; i < n; ++i) {
        const Best b = argmin(tiles[r], q[i], -1.f);
        fk[r][i] = b.at < 0 ? kNoShardMatch : (((unsigned long long)__float_as_uint(b.d2) << 32) | (unsigned)b.id);
      }
    PeerTables fs;
    std::vector<unsigned long long> fmin(n);
    if (mode == kPeer) { fs.n_read = R; for (int r = 0; r < R; ++r) fs.read[r] = fk[r].data(); }
    else {
      for (size_t i = 0; i < n; ++i) { unsigned long long m = ~0ull; for (int r = 0; r < R; ++r) m = std::min(m, fk[r][i]); fmin[i] = m; }
      fs.n_read = 1;
      fs.read[0] = fmin.data();
    }
    const unsigned grid = 3;
    std::vector<double> partials(grid * kAccum, 0.0), accum(kAccum, -1.0);
    unsigned counter = 0;
    const GridSum sum{partials.data(), &counter, accum.data()};
    launch(grid, 256, [&] { k_fitness_reduce(peer_table_set(fs), n, max_range, sum); });
    double cnt = 0, s = 0;
    for (size_t i = 0; i < n; ++i) {
      const Best t = argmin(whole, q[i], -1.f);
      if (t.at >= 0 && (double)t.d2 <= max_range) { cnt += 1; s += t.d2; }
    }
    CHECK(accum[0] == cnt && std::fabs(accum[1] - s) <= 1e-12 * std::fabs(s), "%s R=%d fitness: count %g sum %.17g, want %g %.17g",
          name, R, accum[0], accum[1], cnt, s);
  }
  std::printf("%-26s R=%d %-5s %zu queries %s\n", name, R, mode == kPeer ? "peer" : "nccl", n, bad ? "DIFFERS" : "ok");
}

int main()
{
  std::mt19937 rng(test_seed(20261016u));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  // the map: random points, a lattice (equidistant neighbours: exact ties), duplicates under other ids
  std::vector<MapPoint> map;
  auto add = [&](float x, float y, float z) {
    MapPoint m;
    m.p = make_float4(x, y, z, 0.f);
    m.n = make_float4(U(rng) - 0.5f, U(rng) - 0.5f, U(rng) - 0.5f, 0.f);
    map.push_back(m);
  };
  for (int i = 0; i < 1500; ++i) add(U(rng), U(rng), U(rng));
  for (int i = 0; i < 8; ++i) for (int j = 0; j < 8; ++j) add(0.125f * i, 0.125f * j, 0.5f);
  for (int i = 0; i < 40; ++i) { MapPoint m = map[i * 7]; m.n = make_float4(U(rng), U(rng), U(rng), 0.f); map.push_back(m); }
  // ids: distinct, a few near 2^31 - 1 (unsigned key packing), in no particular order
  std::vector<int> ids(map.size());
  for (size_t i = 0; i < ids.size(); ++i) ids[i] = (int)(i * 977 + 13);
  ids[3] = 2147483646; ids[5] = 2147483645; ids[700] = 2147483600; ids[1501] = 2147483640; ids[1502] = 0;
  std::shuffle(ids.begin(), ids.end(), rng);
  for (size_t i = 0; i < map.size(); ++i) map[i].p.w = __int_as_float(ids[i]);
  // queries: near the map, lattice midpoints (ties), far away (no match), non-finite
  std::vector<float4> q;
  for (int i = 0; i < 600; ++i) { const MapPoint& m = map[(i * 13) % map.size()]; q.push_back(make_float4(m.p.x + 0.01f * (U(rng) - 0.5f), m.p.y + 0.01f * (U(rng) - 0.5f), m.p.z, 0.f)); }
  for (int i = 0; i < 7; ++i) for (int j = 0; j < 7; ++j) q.push_back(make_float4(0.125f * i + 0.0625f, 0.125f * j + 0.0625f, 0.5f, 0.f));
  for (int i = 0; i < 7; ++i) q.push_back(make_float4(0.125f * i + 0.0625f, 0.25f, 0.5f, 0.f));
  for (int i = 0; i < 30; ++i) q.push_back(make_float4(3.f + U(rng), U(rng), U(rng), 0.f));
  q.push_back(make_float4(NAN, 0.f, 0.f, 0.f));
  q.push_back(make_float4(0.5f, INFINITY, 0.5f, 0.f));
  const float gate = 0.01f;
  for (int R : {1, 2, 3, 5, 8}) {
    for (int mode : {kPeer, kNccl}) {
      // spatial slabs along x; the lattice's equidistant neighbours straddle the cuts
      std::vector<std::vector<MapPoint>> slabs(R);
      for (const MapPoint& m : map) slabs[std::min(R - 1, (int)(m.p.x * R))].push_back(m);
      run_case("slabs", slabs, q, gate, true, mode);
      // random partition, some points held by two ranks under one id
      std::vector<std::vector<MapPoint>> rnd(R);
      for (size_t i = 0; i < map.size(); ++i) {
        rnd[rng() % R].push_back(map[i]);
        if (R > 1 && i % 50 == 0) rnd[rng() % R].push_back(map[i]);
      }
      run_case("random", rnd, q, gate, true, mode);
      run_case("random, no normals", rnd, q, gate, false, mode);
      // the last rank's tile lies beyond every query's gate
      if (R > 1) {
        std::vector<std::vector<MapPoint>> far = slabs;
        far[R - 1].clear();
        for (int i = 0; i < 5; ++i) { MapPoint m = map[i]; m.p.z += 10.f; m.p.w = __int_as_float(2000000000 + i); far[R - 1].push_back(m); }
        run_case("a tile out of reach", far, q, gate, true, mode);
      }
    }
  }
  std::printf("%ld checks, %ld failures\n", g_checks, g_fail);
  if (g_fail == 0) std::printf("PASSED\n");
  return g_fail ? 1 : 0;
}
