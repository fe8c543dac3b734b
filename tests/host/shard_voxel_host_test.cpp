// shard_voxel_host_test.cpp — the kernels of VoxelGrid over a sharded map (pcl_b200/csrc/shard_voxel_kernels.cuh) compiled
// for the HOST and run in shard_voxel.cu's sequence for R = 1, 2, 3, 5, 8 simulated ranks in one process, under both
// exchange protocols (shard_sim.h), with std::stable_sort / a flagged copy / a unique-by-key where the driver calls CUB.
// The reference is the single-process VoxelGrid of the whole map (the kernels of voxel_kernels.cuh in voxel.cu's sequence,
// indices = the union of the ids in ascending order).  For every scene it checks
//   - every rank's rows, concatenated and sorted by voxel index, equal the reference's rows byte for byte (centroids and,
//     with normals, the normal / curvature planes), and the voxel indices equal the reference's keys;
//   - no voxel is returned by two ranks, each rank's voxels ascend, and no rank returns more rows than it has records;
//   - the guard: the sharded grid trips it exactly when the whole map's does.
// Scenes: random points with dense clusters and a lattice whose coordinates are multiples of a leaf, non-finite records;
// partitions: slabs, random, slabs sharing the records near a cut under one id, a far tile, slabs cut on voxel faces, one
// rank empty; leaves giving about 1 to 50 records per voxel; min_points_per_voxel 0, 1 and 3; a grid whose voxel indices
// reach 2^31 and beyond while the guard passes (the sort compares the bits of the key the driver's does, kSvKeyBits).
// At least one kept voxel must pass min_points_per_voxel only on its whole-map count (no rank's share does).
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <map>
#include <numeric>
#include <set>

#include "shard_sim.h"
#include "../../pcl_b200/csrc/voxel_kernels.cuh"
#include "../../pcl_b200/csrc/shard_voxel_kernels.cuh"

using namespace pclb200;

struct Rec {
  float4 p;  // w = id
  float4 n0, n1;
};
struct Rows {
  std::vector<float4> xyz, nc;
  std::vector<unsigned> vox;
};

// starts of the flagged positions (cub::DeviceSelect::Flagged over a counting iterator)
static std::vector<unsigned> flagged(const std::vector<unsigned char>& head)
{
  std::vector<unsigned> s;
  for (size_t j = 0; j < head.size(); ++j)
    if (head[j]) s.push_back((unsigned)j);
  return s;
}

// k_vg_minmax over n dense points
static MinMaxAcc minmax(const std::vector<float4>& p)
{
  MinMaxAcc acc;
  for (int d = 0; d < 3; ++d) { acc.lo[d] = 0x7fffffff; acc.hi[d] = (int)0x80000000; }
  acc.count = 0;
  if (!p.empty()) launch((unsigned)std::min<size_t>((p.size() + 255) / 256, 4), 256, [&] { k_vg_minmax(p.data(), p.size(), &acc); });
  return acc;
}

// voxel.cu: voxelgrid() over dense points (and their normal planes); false when the guard trips
static bool single(const std::vector<float4>& pts, const std::vector<float4>& nc, const float leaf[3], unsigned min_pts, Rows& out)
{
  const size_t cnt = pts.size();
  out = Rows();
  const MinMaxAcc h = minmax(pts);
  if (h.count == 0) return true;
  float mn[3], mx[3];
  for (int d = 0; d < 3; ++d) { mn[d] = vord2f(h.lo[d]); mx[d] = vord2f(h.hi[d]); }
  VgParams gp;
  if (!vg_grid(mn, mx, leaf, gp)) return false;
  const size_t n_valid = h.count;
  std::vector<unsigned> keys_in(cnt), keys(cnt);
  std::vector<int32_t> vals_in(cnt), vals(cnt);
  launch((unsigned)((cnt + 255) / 256), 256, [&] { k_vg_keys(pts.data(), cnt, gp, keys_in.data(), vals_in.data()); });
  std::vector<size_t> order(cnt);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return keys_in[a] < keys_in[b]; });
  for (size_t i = 0; i < cnt; ++i) { keys[i] = keys_in[order[i]]; vals[i] = vals_in[order[i]]; }
  std::vector<unsigned char> head(n_valid);
  launch((unsigned)((n_valid + 255) / 256), 256, [&] { k_vg_heads(keys.data(), n_valid, head.data()); });
  const std::vector<unsigned> starts = flagged(head);
  const size_t n_runs = starts.size();
  std::vector<RunRef> runs_all(n_runs), runs;
  std::vector<unsigned char> keep(n_runs, 1);
  launch((unsigned)((n_runs + 255) / 256), 256, [&] { k_vg_runs(starts.data(), n_runs, n_valid, runs_all.data()); });
  if (min_pts > 1) launch((unsigned)((n_runs + 255) / 256), 256, [&] { k_vg_keep(starts.data(), n_runs, n_valid, min_pts, keep.data()); });
  for (size_t m = 0; m < n_runs; ++m)
    if (keep[m]) { runs.push_back(runs_all[m]); out.vox.push_back(keys[starts[m]]); }
  const size_t n_out = runs.size();
  out.xyz.assign(n_out, make_float4(0, 0, 0, 0));
  if (n_out) launch((unsigned)((n_out + 127) / 128), 128, [&] { k_vg_centroids(pts.data(), vals.data(), runs.data(), n_out, out.xyz.data()); });
  if (!nc.empty() && n_out) {
    out.nc.assign(2 * n_out, make_float4(0, 0, 0, 0));
    launch((unsigned)((n_out + 127) / 128), 128, [&] { k_vg_normals(nc.data(), vals.data(), runs.data(), n_out, out.nc.data()); });
  }
  return true;
}

static long g_split_kept = 0;  // kept voxels that no rank's share alone would keep

// shard_voxel.cu over R simulated ranks; false when the union grid trips the guard
static bool sharded(const std::vector<std::vector<Rec>>& tiles, bool normals, const float leaf[3], unsigned min_pts, int mode,
                    std::vector<Rows>& out, unsigned long long& shared)
{
  const int R = (int)tiles.size(), per = sv_units(normals);
  // boxes: every rank's keys, one u64 minimum
  std::vector<std::vector<float4>> dense(R), nc(R);
  std::vector<std::vector<int32_t>> ids(R);
  std::vector<unsigned long long> w((size_t)kSvBoxWords * R, ~0ull);
  for (int r = 0; r < R; ++r) {
    for (const Rec& x : tiles[r]) {
      dense[r].push_back(make_float4(x.p.x, x.p.y, x.p.z, 1.f));
      ids[r].push_back(__float_as_int(x.p.w));
      nc[r].push_back(x.n0);
      nc[r].push_back(x.n1);
    }
    sv_fold_box(minmax(dense[r]), w.data() + (size_t)kSvBoxWords * r);
  }
  SvBoxes boxes = {};
  boxes.n = R;
  unsigned long long u[kSvBoxWords];
  for (int a = 0; a < kSvBoxWords; ++a) u[a] = kSvNoBox;
  for (int s = 0; s < R; ++s) {
    boxes.any[s] = sv_box(w.data() + (size_t)kSvBoxWords * s, boxes.lo[s], boxes.hi[s]);
    for (int a = 0; a < kSvBoxWords; ++a) u[a] = std::min(u[a], w[(size_t)kSvBoxWords * s + a]);
  }
  out.assign(R, Rows());
  float mn[3], mx[3];
  if (!sv_box(u, mn, mx)) return true;
  VgParams gp;
  if (!vg_grid(mn, mx, leaf, gp)) return false;
  SvRanges rg;
  launch(1, 32, [&] { k_sv_ranges(boxes, gp, &rg); });
  // exchange: counts, then the segments through the simulated tables
  std::vector<unsigned long long> cnt((size_t)R * R, 0);
  for (int s = 0; s < R; ++s) {
    SvOut o;
    std::memset(&o, 0, sizeof o);
    o.count = cnt.data() + (size_t)R * s;
    launch(3, 64, [&] { k_sv_select(dense[s].data(), ids[s].data(), normals ? nc[s].data() : nullptr, dense[s].size(), gp, &rg, R, s, o); });
  }
  std::vector<unsigned long long> units(cnt);
  for (auto& x : units) x *= per;
  const std::vector<unsigned long long> n_table = segment_table_sizes(units.data(), R);
  SimTables t(mode, R, n_table.data(), sizeof(float4));
  std::vector<std::vector<float4>> local(R);
  std::vector<size_t> n_own(R), n_local(R, 0);
  shared = 0;
  for (int s = 0; s < R; ++s) {
    n_own[s] = cnt[(size_t)s * R + s];
    for (int x = 0; x < R; ++x) n_local[s] += cnt[(size_t)x * R + s];
    for (int x = 0; x < R; ++x) shared += x == s ? 0 : cnt[(size_t)s * R + x];
    local[s].assign(n_local[s] * per, make_float4(0, 0, 0, 0));
    std::vector<unsigned long long> cursor(R, 0);
    SvOut o;
    std::memset(&o, 0, sizeof o);
    o.count = cursor.data();
    o.dst[s] = local[s].data();
    segment_writes(reinterpret_cast<float4*>(t.local(s)), units.data(), R, s, o.dst);
    launch(3, 64, [&] { k_sv_select(dense[s].data(), ids[s].data(), normals ? nc[s].data() : nullptr, dense[s].size(), gp, &rg, R, s, o); });
    for (int x = 0; x < R; ++x) CHECK(cursor[x] == cnt[(size_t)s * R + x], "rank %d wrote %llu records to rank %d, counted %llu", s, cursor[x], x, cnt[(size_t)s * R + x]);
  }
  const PeerTables view = t.publish();
  // centroids, on every rank
  std::vector<std::map<unsigned, unsigned>> share(R);  // voxel -> this rank's own finite records in it
  for (int r = 0; r < R; ++r) {
    const PeerSegments<float4> rs = segment_reads<float4>(view, units.data(), R, r);
    launch(2, 64, [&] { k_gather_segments(rs, local[r].data() + n_own[r] * per); });
    SvSenders snd = {};
    for (int s = -1; s < R; ++s) {
      const int from = s < 0 ? r : s;
      if (s == r) continue;
      snd.rank[snd.n] = from;
      snd.begin[snd.n + 1] = snd.begin[snd.n] + cnt[(size_t)from * R + r];
      ++snd.n;
    }
    const size_t n = n_local[r];
    if (!n) continue;
    std::vector<unsigned long long> keys_in(n), keys(n), ukeys;
    std::vector<int32_t> vals_in(n), vals(n), uvals;
    std::vector<unsigned char> holder(n);
    std::vector<float4> pts(normals ? n : 0), ncl(normals ? 2 * n : 0);
    launch((unsigned)((n + 255) / 256), 256, [&] { k_sv_keys(local[r].data(), n, gp, snd, keys_in.data(), vals_in.data(), holder.data(), normals ? pts.data() : nullptr, normals ? ncl.data() : nullptr); });
    for (size_t i = 0; i < n_own[r]; ++i) ++share[r][(unsigned)(keys_in[i] >> 32)];
    std::vector<size_t> order(n);
    std::iota(order.begin(), order.end(), 0);
    const unsigned long long sorted_bits = ~0ull >> (64 - kSvKeyBits);  // cub::DeviceRadixSort over [0, kSvKeyBits)
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return (keys_in[a] & sorted_bits) < (keys_in[b] & sorted_bits); });
    for (size_t i = 0; i < n; ++i) { keys[i] = keys_in[order[i]]; vals[i] = vals_in[order[i]]; }
    for (size_t i = 0; i < n; ++i)  // cub::DeviceSelect::UniqueByKey: the first of every run of equal keys
      if (i == 0 || keys[i] != keys[i - 1]) { ukeys.push_back(keys[i]); uvals.push_back(vals[i]); }
    const size_t n_u = ukeys.size();
    std::vector<unsigned char> head(n), uhead(n_u);
    launch((unsigned)((n + 255) / 256), 256, [&] { k_sv_heads(keys.data(), n, head.data()); });
    launch((unsigned)((n_u + 255) / 256), 256, [&] { k_sv_heads(ukeys.data(), n_u, uhead.data()); });
    const std::vector<unsigned> starts_all = flagged(head), starts_u = flagged(uhead);
    CHECK(starts_all.size() == starts_u.size(), "rank %d: %zu voxel runs of the keys, %zu of the unique keys", r, starts_all.size(), starts_u.size());
    const size_t n_runs = starts_u.size();
    std::vector<unsigned char> mask(n_runs), keep(n_runs);
    std::vector<RunRef> runs_all(n_runs), runs;
    std::vector<unsigned> voxel(n_runs);
    launch((unsigned)((n_runs + 255) / 256), 256, [&] { k_sv_holders(starts_all.data(), n_runs, n, vals.data(), holder.data(), mask.data()); });
    launch((unsigned)((n_runs + 255) / 256), 256, [&] { k_vg_runs(starts_u.data(), n_runs, n_u, runs_all.data()); });
    launch((unsigned)((n_runs + 255) / 256), 256, [&] { k_sv_own(runs_all.data(), ukeys.data(), mask.data(), n_runs, r, min_pts, keep.data(), voxel.data()); });
    for (size_t m = 0; m < n_runs; ++m)
      if (keep[m]) { runs.push_back(runs_all[m]); out[r].vox.push_back(voxel[m]); }
    const size_t m = runs.size();
    out[r].xyz.assign(m, make_float4(0, 0, 0, 0));
    if (m) launch((unsigned)((m + 127) / 128), 128, [&] { k_vg_centroids(normals ? pts.data() : local[r].data(), uvals.data(), runs.data(), m, out[r].xyz.data()); });
    if (normals && m) {
      out[r].nc.assign(2 * m, make_float4(0, 0, 0, 0));
      launch((unsigned)((m + 127) / 128), 128, [&] { k_vg_normals(ncl.data(), uvals.data(), runs.data(), m, out[r].nc.data()); });
    }
  }
  // kept voxels that pass min_pts only on the whole map's count
  for (int r = 0; r < R; ++r)
    for (unsigned v : out[r].vox) {
      unsigned most = 0;
      for (int s = 0; s < R; ++s) {
        auto it = share[s].find(v);
        if (it != share[s].end()) most = std::max(most, it->second);
      }
      g_split_kept += min_pts > 1 && most < min_pts;
    }
  return true;
}

static void run_case(const char* name, const std::vector<std::vector<Rec>>& tiles, float leaf1, unsigned min_pts, bool normals, int mode)
{
  const int R = (int)tiles.size();
  const float leaf[3] = {leaf1, leaf1, leaf1};
  std::map<int, Rec> by_id;  // the whole map: every id once, ascending
  for (const auto& t : tiles) for (const Rec& x : t) by_id[__float_as_int(x.p.w)] = x;
  std::vector<float4> pts, nc;
  for (const auto& kv : by_id) { pts.push_back(make_float4(kv.second.p.x, kv.second.p.y, kv.second.p.z, 1.f)); nc.push_back(kv.second.n0); nc.push_back(kv.second.n1); }
  Rows want;
  const bool ok_single = single(pts, normals ? nc : std::vector<float4>(), leaf, min_pts, want);
  std::vector<Rows> got;
  unsigned long long shared = 0;
  const bool ok_sharded = sharded(tiles, normals, leaf, min_pts, mode, got, shared);
  CHECK(ok_single == ok_sharded, "%s R=%d leaf %g: the guard trips on %s only", name, R, leaf1, ok_single ? "the sharded grid" : "the whole map");
  bool same = ok_single == ok_sharded;
  size_t rows = 0;
  if (ok_single && ok_sharded) {
    std::vector<std::pair<unsigned, std::pair<int, size_t>>> all;  // (voxel, (rank, row))
    for (int r = 0; r < R; ++r) {
      CHECK(got[r].vox.size() <= tiles[r].size(), "%s R=%d rank %d: %zu rows from %zu records", name, R, r, got[r].vox.size(), tiles[r].size());
      for (size_t i = 0; i < got[r].vox.size(); ++i) {
        if (i) CHECK(got[r].vox[i] > got[r].vox[i - 1], "%s R=%d rank %d: voxels not ascending", name, R, r);
        all.push_back({got[r].vox[i], {r, i}});
      }
    }
    std::stable_sort(all.begin(), all.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
    rows = all.size();
    same = all.size() == want.vox.size();
    CHECK(same, "%s R=%d leaf %g min %u: %zu rows, the whole map has %zu", name, R, leaf1, min_pts, all.size(), want.vox.size());
    for (size_t i = 0; same && i < all.size(); ++i) {
      const Rows& g = got[all[i].second.first];
      const size_t j = all[i].second.second;
      same = all[i].first == want.vox[i] && std::memcmp(&g.xyz[j], &want.xyz[i], 16) == 0 &&
             (!normals || std::memcmp(&g.nc[2 * j], &want.nc[2 * i], 32) == 0);
      CHECK(same, "%s R=%d leaf %g min %u normals %d: row %zu (voxel %u on rank %d) differs from the whole map's (voxel %u)", name, R, leaf1, min_pts, normals, i, all[i].first,
            all[i].second.first, want.vox[i]);
    }
  }
  std::printf("%-22s R=%d %-4s leaf %-6g min %u %-7s %6zu rows, %6llu shared records %s\n", name, R, mode == kPeer ? "peer" : "nccl", leaf1, min_pts,
              normals ? "normals" : "xyz", rows, shared, !ok_single ? "guard" : same ? "ok" : "DIFFERS");
}

int main()
{
  std::mt19937 rng(test_seed(20261018u));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::normal_distribution<float> N(0.f, 1.f);
  std::vector<Rec> map;
  auto add = [&](float x, float y, float z) {
    Rec r;
    r.p = make_float4(x, y, z, 0.f);
    const float nx = N(rng), ny = N(rng), nz = 1.f, inv = 1.f / std::sqrt(nx * nx + ny * ny + nz * nz);
    r.n0 = make_float4(nx * inv, ny * inv, nz * inv, 0.f);
    r.n1 = make_float4(0.01f * U(rng), 0.f, 0.f, 0.f);
    map.push_back(r);
  };
  for (int i = 0; i < 1200; ++i) add(U(rng), U(rng), 0.5f * U(rng));
  for (int c = 0; c < 4; ++c) {  // dense clusters: up to ~50 records per voxel at the smaller leaves
    const float cx = U(rng), cy = U(rng), cz = 0.5f * U(rng);
    for (int i = 0; i < 60; ++i) add(cx + 0.02f * N(rng), cy + 0.02f * N(rng), cz + 0.02f * N(rng));
  }
  for (int i = 0; i < 8; ++i)  // a lattice on the faces of leaf 0.125
    for (int j = 0; j < 8; ++j) add(0.125f * i, 0.125f * j, 0.25f);
  for (int i = 0; i < 12; ++i) map[(size_t)i * 97].p.y = i % 2 ? NAN : INFINITY;
  std::vector<int> idv(map.size());
  for (size_t i = 0; i < idv.size(); ++i) idv[i] = (int)(i * 104729u % 2000000000u) + 3;
  idv[5] = 2147483646;
  std::shuffle(idv.begin(), idv.end(), rng);
  for (size_t i = 0; i < map.size(); ++i) map[i].p.w = __int_as_float(idv[i]);
  auto xf = [](const Rec& r) { return std::isfinite(r.p.x) ? r.p.x : 0.f; };
  for (int R : {1, 2, 3, 5, 8}) {
    std::vector<std::pair<const char*, std::vector<std::vector<Rec>>>> parts;
    {
      std::vector<std::vector<Rec>> t(R);
      for (const Rec& p : map) t[std::min(R - 1, std::max(0, (int)(xf(p) * R)))].push_back(p);
      parts.push_back({"slabs", t});
    }
    {
      std::vector<std::vector<Rec>> t(R);
      for (const Rec& p : map) t[rng() % R].push_back(p);
      parts.push_back({"random", t});
    }
    {
      std::vector<std::vector<Rec>> t(R);  // slabs cut on voxel faces of leaf 0.125 (whole voxel columns per rank)
      for (const Rec& p : map) t[std::min(R - 1, std::max(0, (int)std::floor(xf(p) * 8.f) * R / 9))].push_back(p);
      parts.push_back({"voxel faces", t});
    }
    if (R > 1) {
      std::vector<std::vector<Rec>> t(R);  // the records near a cut held by both neighbours, one id
      for (const Rec& p : map) {
        const int r = std::min(R - 1, std::max(0, (int)(xf(p) * R)));
        t[r].push_back(p);
        if (r + 1 < R && xf(p) * R > r + 0.8f) t[r + 1].push_back(p);
      }
      parts.push_back({"shared ids", t});
      std::vector<std::vector<Rec>> f = parts[0].second;  // the last tile: 2 far records
      f[R - 2].insert(f[R - 2].end(), f[R - 1].begin(), f[R - 1].end());
      f[R - 1].clear();
      Rec a = map[1], b = map[2];
      a.p = make_float4(9.f, 9.f, 9.f, __int_as_float(1));
      b.p = make_float4(9.f, 9.25f, 9.f, __int_as_float(2));
      f[R - 1] = {a, b};
      parts.push_back({"far tile", f});
      std::vector<std::vector<Rec>> e(R);  // the last rank empty
      for (size_t i = 0; i < map.size(); ++i) e[i % (R - 1)].push_back(map[i]);
      parts.push_back({"one rank empty", e});
    }
    int mode = kPeer;
    for (const auto& pt : parts) {
      for (float leaf : {0.04f, 0.125f, 0.3f})
        for (unsigned mp : {0u, 1u, 3u}) {
          run_case(pt.first, pt.second, leaf, mp, mp != 1, mode);
          mode = mode == kPeer ? kNccl : kPeer;
        }
      if (R > 1 && std::string(pt.first) == "far tile")  // only the union grid is too large for this leaf
        for (int md : {kPeer, kNccl}) run_case(pt.first, pt.second, 0.003f, 0, false, md);
    }
  }
  {
    // voxel indices at and above 2^31 while the guard passes (leaf 1: int(extent) + 1 = 1290 per axis, div_b = 1291): the
    // far corner is voxel 2 151 685 170, whose low 31 bits are voxel 4 201 522; rank 0 holds records of both, with the ids
    // of the lower voxel on either side of the corner's
    const float4 pn = make_float4(0.f, 0.f, 1.f, 0.f), cv = make_float4(0.005f, 0.f, 0.f, 0.f);
    auto rec = [&](float x, float y, float z, int id) { return Rec{make_float4(x, y, z, __int_as_float(id)), pn, cv}; };
    std::vector<std::vector<Rec>> t(2);
    t[0] = {rec(608.5f, 672.5f, 2.5f, 1), rec(1290.4f, 1290.4f, 1290.4f, 2), rec(608.25f, 672.75f, 2.25f, 3), rec(0.5f, 0.5f, 0.5f, 4)};
    t[1] = {rec(0.7f, 0.7f, 0.7f, 5), rec(1290.3f, 1290.3f, 1290.3f, 6), rec(608.75f, 672.25f, 2.75f, 7)};
    for (int md : {kPeer, kNccl})
      for (bool nrm : {false, true}) run_case("voxels above 2^31", t, 1.f, 0, nrm, md);
  }
  CHECK(g_split_kept > 0, "no kept voxel passed min_points_per_voxel on its whole-map count alone");
  std::printf("%ld kept voxels pass min_points_per_voxel only on the whole map's count\n", g_split_kept);
  std::printf("%ld checks, %ld failures\n", g_checks, g_fail);
  if (g_fail == 0) std::printf("PASSED\n");
  return g_fail ? 1 : 0;
}
