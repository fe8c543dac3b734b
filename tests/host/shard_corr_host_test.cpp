// shard_corr_host_test.cpp — the kernels of the correspondence lists over a sharded map (pcl_b200/csrc/shard_target_kernels.cuh:
// k_tile_keys, k_keys_to_corr; driver icp.cu: correspondences_sharded) compiled for the HOST and run for R = 1, 2, 3, 5, 8
// simulated ranks in one process, under both exchange protocols (peer: every rank's key table read directly; NCCL: the
// element-wise minimum of the tables).  Each rank searches a host-built index of its tile, labelled with the map's ids,
// and the whole source.  The list every rank builds must be, byte for byte, the brute-force list over the whole map under
// the (d2, id) rule within the gate, nearest and reciprocal (the reverse search: the source point nearest to the winning
// map point, smaller index on ties, must be the query).  Inputs: exact ties across ranks (a lattice and repeated points
// under other ids), ids held by two ranks, ids near 2^31 - 1, a tile out of reach, non-finite queries, source points
// repeated so that the reverse search's verdict differs between the tied map points' neighbours.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <cfloat>

static inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }

#include "shard_sim.h"
#include "../../pcl_b200/csrc/shard_target_kernels.cuh"

struct MapPoint { float x, y, z; int id; };

// (d2, index) minimum over pts within d2 <= gate; -1 when none
static int argmin(const std::vector<float4>& pts, const float4& q, float gate, const std::vector<int>& label, float* d2)
{
  int best = -1;
  float bd = 0.f;
  if (!finite3(q)) return -1;
  for (size_t j = 0; j < pts.size(); ++j) {
    const float d = d2_of(q, pts[j]);
    if (!(d <= gate)) continue;
    if (best < 0 || d < bd || (d == bd && label[j] < label[best])) { best = (int)j; bd = d; }
  }
  if (d2) *d2 = bd;
  return best;
}

static void run_case(const char* name, const std::vector<std::vector<MapPoint>>& tiles, const std::vector<float4>& src,
                     const HostIndex& IS, const std::vector<int32_t>* sub, float gate, bool recip, int mode)
{
  const int R = (int)tiles.size();
  const size_t nq = sub ? sub->size() : src.size();
  // the whole map: every id once (an id held by two ranks names the same point)
  std::vector<float4> whole;
  std::vector<int> wid;
  for (const auto& t : tiles)
    for (const MapPoint& m : t)
      if (std::find(wid.begin(), wid.end(), m.id) == wid.end()) { whole.push_back(make_float4(m.x, m.y, m.z, 0.f)); wid.push_back(m.id); }
  std::vector<int> src_label(src.size());
  for (size_t i = 0; i < src.size(); ++i) src_label[i] = (int)i;
  std::vector<float4> q(nq);
  for (size_t i = 0; i < nq; ++i) { q[i] = src[sub ? (size_t)(*sub)[i] : i]; q[i].w = __int_as_float((int)i); }
  // per rank: its tile's index labelled with ids, its key table (2 nq words when reciprocal)
  const size_t words = recip ? 2 * nq : nq;
  std::vector<std::vector<unsigned long long>> tab(R, std::vector<unsigned long long>(words, 7ull));
  for (int r = 0; r < R; ++r) {
    std::vector<float> xyz;
    for (const MapPoint& m : tiles[r]) { xyz.push_back(m.x); xyz.push_back(m.y); xyz.push_back(m.z); }
    HostIndex IT;
    build_index(IT, xyz, 4);
    for (float4& p : IT.pts)
      if (__float_as_int(p.w) != kSentinelIndex) p.w = __int_as_float(tiles[r][__float_as_int(p.w)].id);
    std::vector<Match> match(nq);
    int d_error = 0;
    const TreeView T = IT.view(true);
    if (recip)
      launch(3, 256, [&] { k_tile_keys<true>(T, q.data(), nq, gate, IS.nodes.data(), IS.pts.data(), IS.root, sub ? sub->data() : nullptr, tab[r].data(), match.data(), &d_error); });
    else
      launch(3, 256, [&] { k_tile_keys<false>(T, q.data(), nq, gate, nullptr, nullptr, 0, nullptr, tab[r].data(), match.data(), &d_error); });
    CHECK(d_error == 0, "%s: traversal stack overflow flag", name);
  }
  PeerTables t;
  std::vector<unsigned long long> red(words, ~0ull);
  if (mode == kPeer) { t.n_read = R; for (int r = 0; r < R; ++r) t.read[r] = tab[r].data(); }
  else {
    for (int r = 0; r < R; ++r) for (size_t i = 0; i < words; ++i) red[i] = std::min(red[i], tab[r][i]);
    t.n_read = 1;
    t.read[0] = red.data();
  }
  // the brute-force list over the whole map
  std::vector<pclb200_corr> want;
  for (size_t i = 0; i < nq; ++i) {
    float d2 = 0.f;
    const int j = argmin(whole, q[i], gate, wid, &d2);
    if (j < 0) continue;
    const int qi = sub ? (*sub)[i] : (int)i;
    if (recip) {
      std::vector<float4> s4(src.begin(), src.end());
      const int b = argmin(s4, whole[j], gate, src_label, nullptr);
      if (b != qi) continue;
    }
    want.push_back(pclb200_corr{qi, wid[j], d2});
  }
  long bad = 0;
  for (int r = 0; r < R; ++r) {  // every rank reduces the same tables
    std::vector<pclb200_corr> by_slot(nq), got;
    launch((unsigned)((nq + 255) / 256), 256, [&] { k_keys_to_corr(peer_table_set(t), nq, recip ? 1 : 0, sub ? sub->data() : nullptr, by_slot.data()); });
    for (const pclb200_corr& c : by_slot) if (c.index_match >= 0) got.push_back(c);   // compact_corr_to
    const bool ok = got.size() == want.size() && std::memcmp(got.data(), want.data(), got.size() * sizeof(pclb200_corr)) == 0;
    bad += !ok;
    CHECK(ok, "%s R=%d rank %d: %zu pairs, brute force %zu", name, R, r, got.size(), want.size());
  }
  std::printf("%-34s R=%d %-5s %-10s %5zu pairs %s\n", name, R, mode == kPeer ? "peer" : "nccl", recip ? "reciprocal" : "nearest",
              want.size(), bad ? "DIFFERS" : "ok");
}

// normal shooting / back projection: every rank's k nearest of its tile (brute force under the (d2, id) rule: what
// launch_knn returns, padded with (-1, +inf) when the tile holds fewer), k_knn_keys, k_merge_rows over the segment
// tables, k_candidate_scores and, after the minimum of the score tables, k_select_sharded; against select_by_normals
// (the single-process choice) over the brute-force k nearest of the whole map, keff = min(k, distinct finite ids)
static void run_normals_case(const char* name, const std::vector<std::vector<MapPoint>>& tiles,
                             const std::vector<std::vector<float4>>& tile_nrm, const std::vector<float4>& src,
                             const std::vector<float4>& src_nrm, int kind, int k, double max_dist, int mode)
{
  const int R = (int)tiles.size();
  const size_t nq = src.size();
  std::vector<float4> whole, wnrm;
  std::vector<int> wid;
  for (int r = 0; r < R; ++r)
    for (size_t j = 0; j < tiles[r].size(); ++j) {
      const MapPoint& m = tiles[r][j];
      if (std::find(wid.begin(), wid.end(), m.id) == wid.end()) {
        whole.push_back(make_float4(m.x, m.y, m.z, 0.f)); wnrm.push_back(tile_nrm[r][j]); wid.push_back(m.id);
      }
    }
  int n_fin = 0;
  for (const float4& p : whole) n_fin += finite3(p);
  const int keff = std::min(k, n_fin);
  // k nearest of pts (indices into pts, ascending (d2, label)), padded with -1
  auto knn = [&](const std::vector<float4>& pts, const std::vector<int>& label, const float4& q, std::vector<int>& row) {
    std::vector<std::pair<std::pair<float, int>, int>> c;
    if (finite3(q))
      for (size_t j = 0; j < pts.size(); ++j)
        if (finite3(pts[j])) c.push_back({{d2_of(q, pts[j]), label[j]}, (int)j});
    std::sort(c.begin(), c.end());
    row.assign(keff, -1);
    for (int j = 0; j < keff && j < (int)c.size(); ++j) row[j] = c[j].second;
  };
  const size_t nk = nq * (size_t)keff;
  std::vector<std::vector<unsigned long long>> rows(R, std::vector<unsigned long long>(nk));
  std::vector<std::vector<float4>> tp(R);
  std::vector<std::vector<unsigned>> sid(R);
  std::vector<std::vector<int>> spos(R);
  for (int r = 0; r < R; ++r) {
    std::vector<int> lab;
    for (const MapPoint& m : tiles[r]) { tp[r].push_back(make_float4(m.x, m.y, m.z, __int_as_float(m.id))); lab.push_back(m.id); }
    std::vector<int32_t> idx(nk);
    std::vector<float> d2(nk);
    std::vector<int> row;
    for (size_t i = 0; i < nq; ++i) {
      knn(tp[r], lab, src[i], row);
      for (int j = 0; j < keff; ++j) {
        idx[i * keff + j] = row[j] < 0 ? -1 : lab[row[j]];
        d2[i * keff + j] = row[j] < 0 ? INFINITY : d2_of(src[i], tp[r][row[j]]);
      }
    }
    launch(2, 256, [&] { k_knn_keys(idx.data(), d2.data(), nk, rows[r].data()); });
    std::vector<std::pair<unsigned, int>> v;
    for (size_t j = 0; j < tp[r].size(); ++j) v.push_back({(unsigned)tiles[r][j].id, (int)j});
    std::sort(v.begin(), v.end());
    for (const auto& e : v) { sid[r].push_back(e.first); spos[r].push_back(e.second); }
  }
  PeerTables seg;   // the segment tables: every rank's rows, in place (peer) or gathered (NCCL): R tables either way
  seg.n_read = R;
  for (int r = 0; r < R; ++r) seg.read[r] = rows[r].data();
  std::vector<std::vector<unsigned long long>> merged(R, std::vector<unsigned long long>(nk)), score(R, std::vector<unsigned long long>(nk));
  for (int r = 0; r < R; ++r) {
    launch((unsigned)((nq + 255) / 256), 256, [&] { k_merge_rows(peer_table_set(seg), nq, keff, merged[r].data()); });
    launch((unsigned)((nq + 255) / 256), 256, [&] {
      k_candidate_scores(merged[r].data(), nq, keff, kind, src.data(), nullptr, src_nrm.data(), sid[r].data(), spos[r].data(),
                         sid[r].size(), tp[r].data(), tile_nrm[r].data(), score[r].data());
    });
  }
  PeerTables st;
  std::vector<unsigned long long> red(nk, ~0ull);
  if (mode == kPeer) { st.n_read = R; for (int r = 0; r < R; ++r) st.read[r] = score[r].data(); }
  else {
    for (int r = 0; r < R; ++r) for (size_t i = 0; i < nk; ++i) red[i] = std::min(red[i], score[r][i]);
    st.n_read = 1;
    st.read[0] = red.data();
  }
  // the single-process answer over the whole map
  std::vector<pclb200_corr> want;
  std::vector<int32_t> pos_of(whole.size());
  for (size_t j = 0; j < whole.size(); ++j) pos_of[j] = (int)j;
  for (size_t i = 0; i < nq; ++i) {
    if (!finite3(src[i]) || keff == 0) continue;
    std::vector<int> row;
    knn(whole, wid, src[i], row);
    std::vector<float> rd2(keff);
    for (int j = 0; j < keff; ++j) rd2[j] = d2_of(src[i], whole[row[j]]);
    const float4 n = src_nrm[i];
    const int j = select_by_normals<false>(kind, keff, row.data(), rd2.data(), src[i].x, src[i].y, src[i].z, n.x, n.y, n.z,
                                           whole.data(), pos_of.data(), wnrm.data(), max_dist);
    if (j >= 0) want.push_back(pclb200_corr{(int)i, wid[row[j]], rd2[j]});
  }
  long bad = 0;
  for (int r = 0; r < R; ++r) {
    std::vector<pclb200_corr> by_slot(nq), got;
    std::vector<Match> match(nq);
    launch((unsigned)((nq + 255) / 256), 256, [&] {
      k_select_sharded(merged[r].data(), peer_table_set(st), nq, keff, kind, src.data(), nullptr, max_dist, sid[r].data(),
                       spos[r].data(), sid[r].size(), by_slot.data(), match.data());
    });
    for (const pclb200_corr& c : by_slot) if (c.index_match >= 0) got.push_back(c);
    const bool ok = got.size() == want.size() && std::memcmp(got.data(), want.data(), got.size() * sizeof(pclb200_corr)) == 0;
    bad += !ok;
    CHECK(ok, "%s R=%d rank %d kind %d k %d: %zu pairs, single process %zu", name, R, r, kind, k, got.size(), want.size());
  }
  std::printf("%-34s R=%d %-5s kind %d k=%-2d keff=%-2d %5zu pairs %s\n", name, R, mode == kPeer ? "peer" : "nccl", kind, k,
              keff, want.size(), bad ? "DIFFERS" : "ok");
}

int main()
{
  std::mt19937 rng(test_seed(20261017u));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  // the map: random points, a lattice (equidistant neighbours: exact ties), points repeated under other ids
  std::vector<MapPoint> map;
  for (int i = 0; i < 900; ++i) map.push_back(MapPoint{U(rng), U(rng), 0.3f * U(rng), 0});
  for (int i = 0; i < 8; ++i) for (int j = 0; j < 8; ++j) map.push_back(MapPoint{0.125f * i, 0.125f * j, 0.5f, 0});
  for (int i = 0; i < 30; ++i) map.push_back(map[i * 11]);
  std::vector<int> ids(map.size());
  for (size_t i = 0; i < ids.size(); ++i) ids[i] = (int)(i * 977 + 13);
  ids[3] = 2147483646; ids[5] = 2147483645; ids[700] = 2147483600; ids[901] = 2147483640; ids[902] = 0;
  std::shuffle(ids.begin(), ids.end(), rng);
  for (size_t i = 0; i < map.size(); ++i) map[i].id = ids[i];
  // the source: near the map, lattice midpoints (ties), repeated source points (the reverse search's tie rule), far
  // points and non-finite ones
  std::vector<float4> src;
  for (int i = 0; i < 500; ++i) { const MapPoint& m = map[(i * 13) % map.size()]; src.push_back(make_float4(m.x + 0.01f * (U(rng) - 0.5f), m.y + 0.01f * (U(rng) - 0.5f), m.z, 1.f)); }
  for (int i = 0; i < 7; ++i) for (int j = 0; j < 7; ++j) src.push_back(make_float4(0.125f * i + 0.0625f, 0.125f * j + 0.0625f, 0.5f, 1.f));
  for (int i = 0; i < 20; ++i) src.push_back(src[i * 5]);
  for (int i = 0; i < 10; ++i) src.push_back(make_float4(3.f + U(rng), U(rng), U(rng), 1.f));
  src.push_back(make_float4(NAN, 0.f, 0.f, 1.f));
  src.push_back(make_float4(0.5f, INFINITY, 0.5f, 1.f));
  HostIndex IS;
  std::vector<float> fin;   // the source index holds the finite points, labelled by their source index
  std::vector<int> fin_idx;
  for (size_t i = 0; i < src.size(); ++i) if (finite3(src[i])) { fin.insert(fin.end(), {src[i].x, src[i].y, src[i].z}); fin_idx.push_back((int)i); }
  build_index(IS, fin, 4);
  for (float4& p : IS.pts)
    if (__float_as_int(p.w) != kSentinelIndex) p.w = __int_as_float(fin_idx[__float_as_int(p.w)]);
  std::vector<int32_t> sub;
  for (int i = (int)src.size() - 1; i >= 0; i -= 3) sub.push_back(i);
  const float inlier_gate = std::nextafter(0.0001f, -INFINITY);
  for (int R : {1, 2, 3, 5, 8}) {
    for (int mode : {kPeer, kNccl}) {
      std::vector<std::vector<MapPoint>> slabs(R), rnd(R);
      for (const MapPoint& m : map) slabs[std::min(R - 1, (int)(m.x * R))].push_back(m);
      for (size_t i = 0; i < map.size(); ++i) {
        rnd[i < (size_t)R ? i : rng() % R].push_back(map[i]);
        if (R > 1 && i % 40 == 0) rnd[(i + 1) % R].push_back(map[i]);   // held by two ranks under one id
      }
      for (bool recip : {false, true}) {
        for (float gate : {FLT_MAX, 0.0004f, inlier_gate}) {
          run_case("slabs", slabs, src, IS, nullptr, gate, recip, mode);
          run_case("random, shared ids", rnd, src, IS, nullptr, gate, recip, mode);
        }
        run_case("random, descending subset", rnd, src, IS, &sub, 0.0004f, recip, mode);
        if (R > 1) {
          std::vector<std::vector<MapPoint>> far = slabs;
          far[R - 2].insert(far[R - 2].end(), far[R - 1].begin(), far[R - 1].end());
          far[R - 1] = {MapPoint{40.f, 40.f, 40.f, 2000000001}, MapPoint{40.f, 40.f, 40.f, 2000000000}};
          run_case("a tile out of reach", far, src, IS, nullptr, FLT_MAX, recip, mode);
        }
      }
    }
  }
  // normal shooting / back projection: random unit normals with a few NaN, a small map (a whole map with fewer than k
  // points: k = 40 > 35 ids) and tiles with fewer than k points
  auto unit = [&](void) {
    float x = U(rng) - 0.5f, y = U(rng) - 0.5f, z = U(rng) - 0.5f;
    const float l = std::sqrt(x * x + y * y + z * z);
    return make_float4(x / l, y / l, z / l, 0.f);
  };
  std::vector<float4> snrm(src.size());
  for (size_t i = 0; i < src.size(); ++i) snrm[i] = i % 97 == 5 ? make_float4(NAN, 0.f, 0.f, 0.f) : unit();
  std::vector<float4> qsrc(src.begin(), src.begin() + 200);
  qsrc.push_back(make_float4(NAN, 0.f, 0.f, 1.f));
  for (int R : {1, 2, 3, 5, 8}) {
    for (int mode : {kPeer, kNccl}) {
      for (int small : {0, 1}) {
        const size_t n_map = small ? 35 : map.size();
        std::vector<std::vector<MapPoint>> rnd(R);
        std::vector<std::vector<float4>> rn(R);
        for (size_t i = 0; i < n_map; ++i) {
          const float4 nv = i % 53 == 7 ? make_float4(NAN, NAN, NAN, 0.f) : unit();
          const int r = (int)(i < (size_t)R ? i : rng() % R);
          rnd[r].push_back(map[i]); rn[r].push_back(nv);
          if (R > 1 && i % 40 == 0) { rnd[(r + 1) % R].push_back(map[i]); rn[(r + 1) % R].push_back(nv); }  // shared id
        }
        for (int kind : {PCLB200_CORR_NORMAL_SHOOTING, PCLB200_CORR_BACK_PROJECTION})
          for (int k : {1, 10, 40})
            for (double md : {DBL_MAX, 0.0004})
              run_normals_case(small ? "normals, small map" : "normals, random, shared ids", rnd, rn, qsrc, snrm, kind, k,
                               md, mode);
      }
    }
  }
  std::printf("%ld checks, %ld failures\n", g_checks, g_fail);
  if (g_fail == 0) std::printf("PASSED\n");
  return g_fail ? 1 : 0;
}
