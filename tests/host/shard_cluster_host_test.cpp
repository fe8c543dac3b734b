// shard_cluster_host_test.cpp — Euclidean clustering over a sharded map (pcl_b200/csrc/shard_cluster_kernels.cuh, with the
// halo kernels of shard_normals_kernels.cuh and the union-find of cluster_kernels.cuh) compiled for the HOST and run in
// shard_cluster.cu's sequence for R = 1, 2, 3, 5, 8 simulated ranks in one process: this program does the cross-rank steps
// comm.cu would do (the u64 minimum of the boxes, the tables of shard_sim.h), and places the segments with the
// layout functions of peer_tables.cuh that the driver calls.  Every rank's labels and sizes are compared with a brute-force connected-components of the whole map (union of
// the tiles' ids, d2 < r2 under the library's distance).
// Scenes: a zig-zag chain crossing every slab boundary many times (a component's pieces on one rank joined only through
// other ranks), blobs straddling the boundaries, a power-of-two lattice at exactly the tolerance (no edge) and just above
// it (one component), duplicated coordinates under other ids, non-finite records, ids near 2^31 - 2 and tolerance 0;
// partitions: slabs, random, overlapping slabs sharing ids, and slabs plus a 1-point tile.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <map>
#include <set>

#include "shard_sim.h"
#include "../../pcl_b200/csrc/shard_normals_kernels.cuh"
#include "../../pcl_b200/csrc/cluster_kernels.cuh"
#include "../../pcl_b200/csrc/shard_cluster_kernels.cuh"

static unsigned blocks(size_t n) { return (unsigned)std::min<size_t>(3, (n + 63) / 64); }  // a grid-stride loop over n

// per simulated rank: what shard_cluster.cu keeps between the exchanges
struct Rank {
  std::vector<float4> pts;         // the tile index's point array (finite records, padding between)
  std::vector<int> slot_of_pos;    // position -> record of the tile
  size_t n_records = 0;
  std::vector<float4> local;       // tile, then halo
  std::vector<unsigned> sent_ids, recv_ids, local_ids, lab_id;
  std::vector<int32_t> lab;
  std::vector<unsigned long long> edges;
};

// the all-gather of allgather_u64 over the ranks' arrays
static std::vector<unsigned long long> allgather(int mode, const std::vector<std::vector<unsigned long long>>& in)
{
  const int R = (int)in.size();
  std::vector<unsigned long long> n(R);
  size_t total = 0;
  for (int s = 0; s < R; ++s) { n[s] = in[s].size(); total += n[s]; }
  if (!total) return {};
  SimTables t(mode, R, n.data(), sizeof(unsigned long long));
  for (int s = 0; s < R; ++s)
    if (n[s]) launch(blocks(n[s]), 64, [&] { k_gather_segments(one_segment(in[s].data(), n[s]), t.local(s)); });
  const PeerTables view = t.publish();
  std::vector<std::vector<unsigned long long>> out(R, std::vector<unsigned long long>(total));
  for (int r = 0; r < R; ++r) {
    launch(blocks(total), 64, [&] { k_gather_segments(table_runs<unsigned long long>(view, n.data()), out[r].data()); });
    if (r) CHECK(out[r] == out[0], "allgather: rank %d differs", r);
  }
  return out[0];
}

// tiles: every rank's records (w = id, possibly non-finite); checks every rank's labels and sizes against brute force
static void run_case(const char* scene, const char* part, const std::vector<std::vector<float4>>& tiles, double tolerance,
                     int mode, std::mt19937& rng)
{
  const int R = (int)tiles.size();
  const double tol = (double)(float)tolerance;
  const float r2 = (float)(tol * tol), r2_below = std::nextafter(r2, -INFINITY);
  // brute force over the whole map (each id once, finite points)
  std::map<int, float4> by_id;
  for (const auto& t : tiles) for (const float4& p : t) if (finite3(p)) by_id[id_of(p)] = p;
  std::vector<float4> whole;
  for (const auto& kv : by_id) whole.push_back(kv.second);
  const int n = (int)whole.size();
  std::vector<int> par(n);
  for (int i = 0; i < n; ++i) par[i] = i;
  std::function<int(int)> find = [&](int x) { while (par[x] != x) x = par[x] = par[par[x]]; return x; };
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < i; ++j)
      if (d2_of(whole[i], whole[j]) < r2) { const int a = find(i), b = find(j); par[std::max(a, b)] = std::min(a, b); }
  std::map<int, int> want_label;  // id -> smallest id of its component
  std::map<int, long long> comp_size;
  for (int i = 0; i < n; ++i) { want_label[id_of(whole[i])] = id_of(whole[find(i)]); ++comp_size[id_of(whole[find(i)])]; }

  std::vector<Rank> rk(R);
  for (int r = 0; r < R; ++r) {
    Rank& k = rk[r];
    k.n_records = tiles[r].size();
    std::vector<int> rec(tiles[r].size());
    for (size_t i = 0; i < rec.size(); ++i) rec[i] = (int)i;
    std::shuffle(rec.begin(), rec.end(), rng);
    for (size_t i = 0; i < rec.size(); ++i) {
      if (!finite3(tiles[r][rec[i]])) continue;
      k.pts.push_back(tiles[r][rec[i]]);
      k.slot_of_pos.push_back(rec[i]);
      if (i % 5 == 2) { k.pts.push_back(kPad); k.slot_of_pos.push_back(-1); }
    }
    for (int j = 0; j < 3; ++j) { k.pts.push_back(kPad); k.slot_of_pos.push_back(-1); }
  }
  // ---- halo (shard_normals.cu: sharded_local_map with the tile's points as queries, k = 0, r2) ----
  std::vector<unsigned long long> boxes((size_t)kHaloBoxWords * R, kNoHaloBox);
  for (int r = 0; r < R; ++r)
    launch(2, 64, [&] { k_halo_box(rk[r].pts.data(), nullptr, r2, rk[r].pts.size(), boxes.data() + (size_t)kHaloBoxWords * r); });
  std::vector<unsigned long long> cnt((size_t)R * R, 0);
  for (int s = 0; s < R; ++s) {
    HaloOut o;
    std::memset(&o, 0, sizeof o);
    o.count = cnt.data() + (size_t)R * s;
    launch(3, 64, [&] { k_halo_select(rk[s].pts.data(), rk[s].pts.size(), boxes.data(), R, s, o); });
  }
  unsigned long long all = 0;
  for (int s = 0; s < R; ++s)
    for (int r = 0; r < R; ++r) all += s == r ? 0ull : cnt[(size_t)s * R + r];
  const std::vector<unsigned long long> n_table = segment_table_sizes(cnt.data(), R);
  SimTables halo(mode, R, n_table.data(), sizeof(float4));
  for (int s = 0; s < R; ++s) {
    Rank& k = rk[s];
    const size_t n_tile = cnt[(size_t)s * R + s];
    k.local.assign(n_tile, make_float4(0.f, 0.f, 0.f, 0.f));
    std::vector<unsigned long long> cursor(R, 0);
    HaloOut o;
    std::memset(&o, 0, sizeof o);
    o.count = cursor.data();
    o.dst[s] = k.local.data();
    segment_writes(reinterpret_cast<float4*>(halo.local(s)), cnt.data(), R, s, o.dst);
    launch(3, 64, [&] { k_halo_select(k.pts.data(), k.pts.size(), boxes.data(), R, s, o); });
    // this rank's own segments, one run at the start of its table (the HaloTrace's sent ids)
    k.sent_ids.assign(n_table[s], 0);
    if (n_table[s]) launch((unsigned)((n_table[s] + 255) / 256), 256, [&] { k_halo_ids(reinterpret_cast<const float4*>(halo.local(s)), n_table[s], k.sent_ids.data()); });
  }
  const PeerTables halo_view = halo.publish();
  for (int r = 0; r < R; ++r) {
    Rank& k = rk[r];
    const PeerSegments<float4> rs = segment_reads<float4>(halo_view, cnt.data(), R, r);
    const size_t n_tile = k.local.size();
    k.local.resize(n_tile + rs.begin[rs.n]);
    if (rs.begin[rs.n]) launch(2, 64, [&] { k_gather_segments(rs, k.local.data() + n_tile); });
    for (size_t i = n_tile; i < k.local.size(); ++i) k.recv_ids.push_back((unsigned)id_of(k.local[i]));
    // the local map: sorted by id, each id once, indexed; then the unchanged clustering kernels
    std::map<unsigned, float4> lm;
    for (const float4& p : k.local) lm[(unsigned)id_of(p)] = p;
    std::vector<float> xyz;
    for (const auto& kv : lm) { k.local_ids.push_back(kv.first); xyz.insert(xyz.end(), {kv.second.x, kv.second.y, kv.second.z}); }
    const size_t m = k.local_ids.size();
    HostIndex I;
    build_index(I, xyz, 0);
    const size_t np = I.pts.size();
    std::vector<int> parent(np), min_orig(np);
    k.lab.assign(m, -1);
    int d_error = 0;
    launch((unsigned)((np + 255) / 256), 256, [&] { k_cc_init(parent.data(), min_orig.data(), np); });
    launch((unsigned)((np + 127) / 128), 128, [&] { k_cc_union(I.nodes.data(), I.pts.data(), I.root, np, r2, r2_below, parent.data(), &d_error); });
    launch((unsigned)((np + 255) / 256), 256, [&] { k_cc_min_orig(I.pts.data(), np, parent.data(), min_orig.data()); });
    launch((unsigned)((np + 255) / 256), 256, [&] { k_cc_labels(I.pts.data(), np, parent.data(), min_orig.data(), k.lab.data()); });
    CHECK(d_error == 0, "%s %s: traversal error", scene, part);
    k.lab_id.assign(m, 0);
    launch(blocks(m), 64, [&] { k_sc_label_ids(k.lab.data(), k.local_ids.data(), m, k.lab_id.data()); });
  }
  // ---- stitch: the answers, then the edges ----
  const std::vector<unsigned long long> ans = segment_answers(cnt, R);
  const std::vector<unsigned long long> n_ans = segment_table_sizes(ans.data(), R);
  if (all) {
    SimTables t(mode, R, n_ans.data(), sizeof(unsigned));
    for (int r = 0; r < R; ++r) {
      unsigned* mine = reinterpret_cast<unsigned*>(t.local(r));
      if (!rk[r].recv_ids.empty())
        launch(blocks(rk[r].recv_ids.size()), 64, [&] { k_sc_answer(rk[r].recv_ids.data(), rk[r].recv_ids.size(), rk[r].local_ids.data(), rk[r].local_ids.size(), rk[r].lab_id.data(), mine); });
    }
    const PeerTables view = t.publish();
    for (int me = 0; me < R; ++me) {
      Rank& k = rk[me];
      const PeerSegments<unsigned> rs = segment_reads<unsigned>(view, ans.data(), R, me);
      k.edges.assign(k.sent_ids.size(), 0);
      if (!k.sent_ids.empty())
        launch(blocks(k.sent_ids.size()), 64, [&] { k_sc_edges(k.sent_ids.data(), k.sent_ids.size(), k.local_ids.data(), k.local_ids.size(), k.lab_id.data(), rs, k.edges.data()); });
      std::sort(k.edges.begin(), k.edges.end());
      k.edges.erase(std::unique(k.edges.begin(), k.edges.end()), k.edges.end());
    }
  }
  std::vector<std::vector<unsigned long long>> per_rank(R);
  for (int r = 0; r < R; ++r) per_rank[r] = rk[r].edges;
  const std::vector<unsigned long long> edges = allgather(mode, per_rank);
  std::vector<unsigned> ends(2 * edges.size());
  if (!edges.empty()) launch(blocks(edges.size()), 64, [&] { k_sc_split(edges.data(), edges.size(), ends.data()); });
  std::sort(ends.begin(), ends.end());
  ends.erase(std::unique(ends.begin(), ends.end()), ends.end());
  const std::vector<unsigned>& nodes = ends;
  const size_t n_nodes = nodes.size();
  std::vector<int> gparent(n_nodes), root(n_nodes);
  if (n_nodes) {
    launch(blocks(n_nodes), 64, [&] { k_sc_init(gparent.data(), n_nodes); });
    launch(blocks(edges.size()), 64, [&] { k_sc_unite(edges.data(), edges.size(), nodes.data(), n_nodes, gparent.data()); });
    launch(blocks(n_nodes), 64, [&] { k_sc_roots(n_nodes, gparent.data(), root.data()); });
  }
  // ---- labels and sizes ----
  std::vector<std::vector<unsigned long long>> node_cnt(R, std::vector<unsigned long long>(n_nodes, 0)), local_cnt(R);
  for (int r = 0; r < R; ++r) {
    Rank& k = rk[r];
    const size_t m = k.local_ids.size();
    std::vector<unsigned char> dup(m, 0);
    local_cnt[r].assign(m, 0);
    const unsigned long long lower = segment_start(ans.data(), R, r, r);
    if (lower) launch(blocks(lower), 64, [&] { k_sc_mark_lower(k.recv_ids.data(), lower, k.local_ids.data(), m, dup.data()); });
    launch(blocks(k.pts.size()), 64, [&] { k_sc_count(k.pts.data(), k.pts.size(), k.local_ids.data(), m, k.lab.data(), k.lab_id.data(), dup.data(), nodes.data(), n_nodes, node_cnt[r].data(), local_cnt[r].data()); });
  }
  std::vector<unsigned long long> comp(n_nodes, 0), node_sum(n_nodes, 0);
  if (n_nodes) {
    SimTables t(mode, R, n_nodes);
    for (int r = 0; r < R; ++r) std::copy(node_cnt[r].begin(), node_cnt[r].end(), t.local(r));
    const PeerTables view = t.publish();
    launch(blocks(n_nodes), 64, [&] { k_sc_sum(peer_table_set(view), n_nodes, node_sum.data()); });
    launch(blocks(n_nodes), 64, [&] { k_sc_fold(node_sum.data(), n_nodes, root.data(), comp.data()); });
  }
  long bad = 0;
  std::map<int, int> label_seen;  // id -> the label some rank gave it
  for (int r = 0; r < R; ++r) {
    Rank& k = rk[r];
    std::vector<int32_t> labels(k.n_records, -1);
    std::vector<int64_t> sizes(k.n_records, 0);
    launch(blocks(k.pts.size()), 64, [&] { k_sc_output(k.pts.data(), k.slot_of_pos.data(), k.pts.size(), k.local_ids.data(), k.local_ids.size(), k.lab.data(), k.lab_id.data(), nodes.data(), n_nodes, root.data(), comp.data(), local_cnt[r].data(), labels.data(), sizes.data()); });
    for (size_t i = 0; i < k.n_records; ++i) {
      const float4& p = tiles[r][i];
      const int wl = finite3(p) ? want_label[id_of(p)] : -1;
      const long long ws = finite3(p) ? comp_size[wl] : 0;
      if (labels[i] != wl || sizes[i] != ws) {
        if (++bad <= 3) CHECK(false, "%s %s R=%d rank %d record %zu (id %d): label %d size %lld, want %d size %lld", scene, part, R, r, i, id_of(p), labels[i], (long long)sizes[i], wl, ws);
      }
      if (finite3(p)) {
        auto it = label_seen.find(id_of(p));
        if (it != label_seen.end()) CHECK(it->second == labels[i], "%s %s: id %d labelled differently on two ranks", scene, part, id_of(p));
        label_seen[id_of(p)] = labels[i];
      }
    }
  }
  CHECK(bad == 0, "%s %s R=%d %s: %ld records differ", scene, part, R, mode == kPeer ? "peer" : "nccl", bad);
  std::printf("%-22s %-12s R=%d %-5s tol=%-10.6g halo %-5llu edges %-4zu nodes %-4zu comps %-4zu %s\n", scene, part, R,
              mode == kPeer ? "peer" : "nccl", tolerance, all, edges.size(), n_nodes, comp_size.size(), bad ? "DIFFERS" : "ok");
}

int main()
{
  std::mt19937 rng(test_seed(20261018u));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::normal_distribution<float> N(0.f, 1.f);
  struct Scene { const char* name; std::vector<float4> pts; double tol; };
  std::vector<Scene> scenes;
  {  // zig-zag: 6 passes along x over [0, 1], 0.1 apart in y, joined alternately at x = 0 and x = 1
    std::vector<float4> z;
    const float step = 0.02f;
    for (int pass = 0; pass < 6; ++pass) {
      for (int i = 0; i <= 50; ++i) z.push_back(make_float4(pass % 2 ? 1.f - step * i : step * i, 0.1f * pass, 0.f, 0.f));
      if (pass < 5)
        for (int j = 1; j < 5; ++j) z.push_back(make_float4(pass % 2 ? 0.f : 1.f, 0.1f * pass + step * j, 0.f, 0.f));
    }
    z.push_back(make_float4(0.5f, 0.05f, 0.f, 0.f));  // a lone point between two passes
    scenes.push_back({"zig-zag chain", z, 0.025});
  }
  {  // blobs centred on the slab boundaries of every R, plus a few stray points
    std::vector<float4> b;
    const float centres[] = {0.5f, 1.f / 3, 2.f / 3, 0.2f, 0.4f, 0.6f, 0.8f, 0.125f, 0.875f};
    for (int c = 0; c < 9; ++c)
      for (int i = 0; i < 40; ++i) b.push_back(make_float4(centres[c] + 0.02f * N(rng), 0.3f * (c % 3) + 0.02f * N(rng), 0.02f * N(rng), 0.f));
    for (int i = 0; i < 20; ++i) b.push_back(make_float4(U(rng), U(rng), U(rng), 0.f));
    for (int i = 0; i < 15; ++i) b.push_back(b[7 * i]);  // duplicated coordinates under other ids
    b.push_back(make_float4(NAN, 0.f, 0.f, 0.f));
    b.push_back(make_float4(0.5f, INFINITY, 0.f, 0.f));
    scenes.push_back({"blobs", b, 0.02});
    scenes.push_back({"blobs, tolerance 0", b, 0.0});
  }
  {  // 8 x 8 x 2 lattice of spacing 1/8: neighbours exactly at the tolerance (no edge), and just above it (one component)
    std::vector<float4> l;
    for (int i = 0; i < 8; ++i) for (int j = 0; j < 8; ++j) for (int k = 0; k < 2; ++k) l.push_back(make_float4(0.125f * i + 0.0625f, 0.125f * j, 0.125f * k, 0.f));
    scenes.push_back({"lattice at tolerance", l, 0.125});
    scenes.push_back({"lattice above", l, 0.125 * (1.0 + 1e-6)});
  }
  for (Scene& sc : scenes) {  // ids: scattered, shuffled, one near 2^31 - 2
    std::vector<int> ids(sc.pts.size());
    for (size_t i = 0; i < ids.size(); ++i) ids[i] = (int)(i * 7919 + 3);
    ids[0] = 2147483646;
    ids[1] = 2147483645;
    std::shuffle(ids.begin(), ids.end(), rng);
    for (size_t i = 0; i < ids.size(); ++i) sc.pts[i].w = __int_as_float(ids[i]);
  }
  for (int R : {1, 2, 3, 5, 8}) {
    for (const Scene& sc : scenes) {
      std::vector<std::pair<const char*, std::vector<std::vector<float4>>>> parts;
      auto slab = [&](const float4& p) { return std::min(R - 1, std::max(0, std::isfinite(p.x) ? (int)(p.x * R) : 0)); };
      {
        std::vector<std::vector<float4>> t(R);
        for (const float4& p : sc.pts) t[slab(p)].push_back(p);
        parts.push_back({"slabs", t});
      }
      {
        std::vector<std::vector<float4>> t(R);
        for (const float4& p : sc.pts) t[rng() % R].push_back(p);
        parts.push_back({"random", t});
      }
      if (R > 1) {
        std::vector<std::vector<float4>> t(R);  // points near a cut held by both neighbours, same id
        for (const float4& p : sc.pts) {
          const int r = slab(p);
          t[r].push_back(p);
          if (r + 1 < R && std::isfinite(p.x) && p.x * R > r + 0.8f) t[r + 1].push_back(p);
        }
        parts.push_back({"overlapping", t});
        std::vector<std::vector<float4>> f = parts[0].second;  // the last tile: 1 point of its own
        f[R - 2].insert(f[R - 2].end(), f[R - 1].begin(), f[R - 1].end());
        f[R - 1] = {make_float4(0.5f, 0.5f, 0.5f, __int_as_float(2147483644))};
        parts.push_back({"1-point tile", f});
      }
      for (auto& pt : parts) {
        bool empty = false;
        for (const auto& t : pt.second) {
          bool any = false;
          for (const float4& p : t) any |= finite3(p);
          empty |= !any;  // build_index_ids refuses a tile without a finite point
        }
        if (empty) continue;
        for (int mode : {kPeer, kNccl}) run_case(sc.name, pt.first, pt.second, sc.tol, mode, rng);
      }
    }
  }
  std::printf("%ld checks, %ld failures\n", g_checks, g_fail);
  if (g_fail == 0) std::printf("PASSED\n");
  return g_fail ? 1 : 0;
}
