// icp_batch_targets_host_test.cpp — the batch kernels of pcl_b200/csrc/icp_kernels.cuh with one target per problem
// (k_search_batch, k_accum_dmma_batch and k_accum_batch with TARGETS, k_solve_batch with the targets' rmax, over a
// BatchTarget table) and the per-problem query key (lbvh_kernels.cuh: k_problem_frame_keys), compiled for the HOST and run
// on a lock-step emulation of their thread blocks (tests/host/warp_emu.h), against the single-problem kernels run on each
// problem against its own target, driven the way icp.cu drives both.  Three targets in boxes that differ by orders of
// magnitude in place and size; problems take them in turn, so a target serves several problems.  Checked: each problem's
// keys and query order equal k_stage_records's in its own target's frame; after every iteration, per problem, the
// matches, the moved queries, the accumulators, the loop state, the pending transform and the solve output are
// byte-equal to the single run, and so is the final transform.  1, 3 and 7 problems; SVD, point-to-plane and symmetric;
// float and double; tracking off, on and automatic.  CPU only.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <cfloat>

#include "../../pcl_b200/csrc/icp_kernels.cuh"
#include "../../pcl_b200/csrc/lbvh_kernels.cuh"

static float gate_from_max_dist(double max_dist)   // icp.cu: the largest float not above max_dist^2
{
  const double m2 = max_dist * max_dist;
  if (!(m2 < (double)FLT_MAX)) return FLT_MAX;
  float g = (float)m2;
  if ((double)g > m2) g = std::nextafter(g, -INFINITY);
  return g;
}

// the grids of this test (icp.cu: persistent_blocks with a handful of SMs): several blocks per problem from 257 points on
static unsigned wgrid(size_t n) { return (unsigned)std::max<size_t>(1, std::min<size_t>((n + 255) / 256, 3)); }
static unsigned agrid(size_t n) { return (unsigned)std::max<size_t>(1, std::min<size_t>((n + 255) / 256, 2)); }
static unsigned ggrid(size_t n) { return (unsigned)std::max<size_t>(1, std::min<size_t>((n + 255) / 256, 4)); }

template <typename F> static void launch_grid(unsigned grid, int block, F kernel)
{
  gridDim.x = grid;
  blockDim.x = block;
  for (unsigned b = 0; b < grid; ++b) {
    blockIdx_storage.x = b;
    warp_emu::run_block(block, kernel);
  }
  gridDim.x = 1;
  blockIdx_storage.x = 0;
}

// a target: the surface z = f(x, y) scaled by `scale` and moved by `shift`
struct Target {
  float scale, shift[3];
  std::vector<float> xyz;
  std::vector<float4> normals;  // by position of the index, {n, plane_offset} (icp.cu: normals_by_pos)
  HostIndex I;
  double rmax;
};

static void surface_point(const Target& T, float x, float y, float* p, float* n)
{
  const float z = 0.2f * std::sin(2.f * x) * std::cos(2.f * y);
  p[0] = T.scale * x + T.shift[0]; p[1] = T.scale * y + T.shift[1]; p[2] = T.scale * z + T.shift[2];
  float m[3] = {-0.4f * std::cos(2.f * x) * std::cos(2.f * y), 0.4f * std::sin(2.f * x) * std::sin(2.f * y), 1.f};
  const float inv = 1.f / std::sqrt(m[0] * m[0] + m[1] * m[1] + m[2] * m[2]);
  for (int d = 0; d < 3; ++d) n[d] = m[d] * inv;
}

static void make_target(Target& T, unsigned seed)
{
  std::mt19937 rng(test_seed(seed));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  const size_t nt = 5000;
  std::vector<float> tn(3 * nt);
  T.xyz.resize(3 * nt);
  for (size_t i = 0; i < nt; ++i) surface_point(T, 2.5f * U(rng), 2.5f * U(rng), &T.xyz[3 * i], &tn[3 * i]);
  build_index(T.I, T.xyz, 4);
  const float qn = std::numeric_limits<float>::quiet_NaN();
  T.normals.resize(T.I.pts.size());
  for (size_t p = 0; p < T.I.pts.size(); ++p) {
    const int o = __float_as_int(T.I.pts[p].w);
    if (o == kSentinelIndex) { T.normals[p] = make_float4(qn, qn, qn, 0.f); continue; }
    T.normals[p] = make_float4(tn[3 * o], tn[3 * o + 1], tn[3 * o + 2], 0.f);
    T.normals[p].w = plane_offset(T.normals[p], T.I.pts[p]);
  }
  double rmax = 0.0;   // icp.cu: frame_rmax
  for (int r = 0; r < 3; ++r) { const double m = std::max(std::fabs((double)T.I.lo[r]), std::fabs((double)T.I.hi[r])); rmax += m * m; }
  T.rmax = std::sqrt(rmax);
}

// the per-problem loop state icp_set_source / icp_iterate leave before the first iteration
static LoopCtrl fresh_ctrl(const HostIndex& I, int track_mode)
{
  LoopCtrl L;
  std::memset(&L, 0, sizeof L);
  L.state = PCLB200_CONV_NOT_CONVERGED;
  L.prev_mse = std::numeric_limits<double>::max();
  for (int i = 0; i < 16; ++i) L.final_T[i] = L.last_T[i] = (i % 5 == 0) ? 1.0 : 0.0;
  L.track_next = track_mode == PCLB200_TRACK_ON ? 1 : 0;
  for (int r = 0; r < 3; ++r) L.origin[r] = 0.5f * (I.lo[r] + I.hi[r]);
  return L;
}

// slots of pts[0..n) in the order of stable-sorted keys (lbvh.cu: sort_queries), each query {xyz, slot + base}
static std::vector<float4> sorted_queries(const std::vector<float4>& pts, const std::vector<unsigned>& keys, size_t base)
{
  std::vector<int32_t> order(pts.size());
  for (size_t i = 0; i < order.size(); ++i) order[i] = (int32_t)i;
  std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return keys[a] < keys[b]; });
  std::vector<float4> q(pts.size());
  for (size_t j = 0; j < q.size(); ++j) {
    const float4 v = pts[order[j]];
    q[j] = make_float4(v.x, v.y, v.z, __int_as_float((int)(order[j] + base)));
  }
  return q;
}

static void run(const char* name, const std::vector<Target>& tg, const std::vector<size_t>& sizes, int est, bool dbl,
                int track_mode)
{
  const int B = (int)sizes.size(), K = (int)tg.size();
  const bool sym = est == PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS;
  auto target_of = [&](int p) -> const Target& { return tg[(p + B) % K]; };
  std::vector<long long> off(1, 0);
  for (size_t n : sizes) off.push_back(off.back() + (long long)n);
  const size_t total = (size_t)off.back();
  // the sources: patches of each problem's target surface, each moved by its own small rigid motion, and their normals
  std::mt19937 rng(test_seed(29 + (unsigned)B));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::vector<float4> raw(total), raw_nrm(total);
  for (int p = 0; p < B; ++p) {
    const Target& T = target_of(p);
    const float a = 0.02f * (float)(p + 1), c = std::cos(a), s = std::sin(a);
    const float tx = 0.01f * (float)(p % 3), ty = -0.005f * (float)p;
    const float x0 = 0.2f + 0.1f * (float)p, y0 = 0.3f;
    for (long long i = off[p]; i < off[p + 1]; ++i) {
      float q[3], m[3];
      surface_point(T, x0 + 1.2f * U(rng), y0 + 1.2f * U(rng), q, m);
      // rotate about the target's own origin so that the motion is small whatever the target's place
      const float lx = q[0] - T.shift[0], ly = q[1] - T.shift[1];
      raw[i] = make_float4(c * lx - s * ly + T.shift[0] + tx, s * lx + c * ly + T.shift[1] + ty, q[2] + 0.003f, 1.f);
      raw_nrm[i] = make_float4(c * m[0] - s * m[1], s * m[0] + c * m[1], m[2], 0.f);
    }
  }
  // ---- the query order: k_problem_frame_keys over the batch against k_stage_records over each problem alone
  std::vector<float4> frames(B);
  std::vector<BatchTarget> table(B);
  for (int p = 0; p < B; ++p) {
    const Target& T = target_of(p);
    frames[p] = make_float4(T.I.lo[0], T.I.lo[1], T.I.lo[2], T.I.scale);
    const TreeView v = T.I.view(true);
    table[p] = BatchTarget{v.nodes, v.pts, T.normals.data(), v.root, v.cells, T.rmax};
  }
  std::vector<unsigned> bkeys(total);
  std::vector<int32_t> bvals(total);
  launch_grid((unsigned)((total + 255) / 256), 256, [&] {
    k_problem_frame_keys(raw.data(), total, off.data(), B, frames.data(), bkeys.data(), bvals.data());
  });
  std::vector<float4> cur = sorted_queries(raw, bkeys, 0);   // by key, then stably by problem
  std::stable_sort(cur.begin(), cur.end(), [&](const float4& a, const float4& b) {
    return problem_of(off.data(), B, __float_as_int(a.w)) < problem_of(off.data(), B, __float_as_int(b.w));
  });
  std::vector<std::vector<float4>> single_cur(B);
  for (int p = 0; p < B; ++p) {
    const Target& T = target_of(p);
    const size_t n = sizes[p];
    std::vector<float4> mine(raw.begin() + off[p], raw.begin() + off[p + 1]);
    std::vector<unsigned> keys(n);
    std::vector<int32_t> vals(n);
    launch_grid((unsigned)((n + 255) / 256), 256, [&] {
      k_stage_records<float4>(mine.data(), n, 1u, nullptr, nullptr, T.I.lo[0], T.I.lo[1], T.I.lo[2], T.I.scale,
                              keys.data(), vals.data());
    });
    CHECK(std::memcmp(keys.data(), &bkeys[off[p]], n * sizeof(unsigned)) == 0, "%s problem %d: query keys differ", name, p);
    single_cur[p] = sorted_queries(mine, keys, (size_t)off[p]);
    CHECK(std::memcmp(single_cur[p].data(), &cur[off[p]], n * sizeof(float4)) == 0, "%s problem %d: query orders differ", name, p);
  }
  std::vector<float4> nrm(total);
  for (size_t j = 0; j < total; ++j) nrm[j] = raw_nrm[__float_as_int(cur[j].w)];

  const int tmode = sym ? (dbl ? kApplyTransformsDouble : kApplyTransformsFloat) : kApplyIcp;  // with_normals_transform for sym
  CritParams crit;
  crit.max_iterations = 12;
  crit.failure_after_max_iter = 0;
  crit.max_iterations_similar = 0;
  crit.scalar_is_double = dbl ? 1 : 0;
  crit.track_mode = track_mode;
  crit.rot_eps = 0.0;
  crit.trans_eps = 1e-10;
  crit.rel_mse = 1e-6;
  crit.abs_mse = 1e-12;
  crit.rmax = 0.0;   // the batch reads each problem's from the table
  int d_error = 0;
  IterArgs base;
  std::memset(&base, 0, sizeof base);
  base.plane_offsets = 1;
  base.gate = gate_from_max_dist(0.08);
  base.d_error = &d_error;
  base.enforce_same_dir = 1;
  base.track_sel = track_mode == PCLB200_TRACK_AUTO;
  base.peer.nranks = 0;

  // ---- the single runs: one problem each, its own target and grids
  struct Single {
    std::vector<float4> cur, nrm;
    std::vector<Match> match;
    std::vector<float> lbs;
    std::vector<double> partials, accum;
    Pending pending;
    LoopCtrl ctrl;
    SolveOut so;
    unsigned counter = 0;
    unsigned long long skip = 0;
  };
  std::vector<Single> single(B);
  for (int p = 0; p < B; ++p) {
    Single& r = single[p];
    r.cur.assign(cur.begin() + off[p], cur.begin() + off[p + 1]);
    r.nrm.assign(nrm.begin() + off[p], nrm.begin() + off[p + 1]);
    r.match.assign(sizes[p], Match{-1, 0.f});
    r.lbs.assign(sizes[p], 0.f);
    r.partials.assign(4 * 128, 0.0);
    r.accum.assign(kAccum, 0.0);
    std::memset(&r.pending, 0, sizeof r.pending);
    r.pending.mode = tmode;
    std::memset(&r.so, 0, sizeof r.so);
    r.ctrl = fresh_ctrl(target_of(p).I, track_mode);
    if (est == PCLB200_EST_SVD) k_seed_origin(r.cur.data(), nullptr, sizes[p], r.ctrl.origin);
  }
  // ---- the batch: the same problems end to end, each against its own target
  std::vector<Match> match(total, Match{-1, 0.f});
  std::vector<float> lbs(total, 0.f);
  std::vector<Pending> pending(B);
  std::vector<LoopCtrl> ctrl(B);
  for (int p = 0; p < B; ++p) ctrl[p] = fresh_ctrl(target_of(p).I, track_mode);
  std::vector<SolveOut> so(B);
  std::memset(pending.data(), 0, B * sizeof(Pending));
  std::memset(so.data(), 0, B * sizeof(SolveOut));
  for (auto& q : pending) q.mode = tmode;
  std::vector<unsigned> counter(B, 0);
  std::vector<unsigned long long> skip(B, 0);
  std::vector<double> accum((size_t)B * kAccum, 0.0);
  const std::vector<BatchBlock> wt = batch_blocks(off, wgrid), at = batch_blocks(off, sym ? ggrid : agrid);
  std::vector<double> partials(at.size() * 128, 0.0);
  std::vector<long long> offsets = off;
  if (est == PCLB200_EST_SVD)   // icp.cu seeds the SVD origin only
    launch_grid((unsigned)((B + 255) / 256), 256, [&] { k_seed_origin_batch(cur.data(), offsets.data(), B, ctrl.data()); });

  IterArgs ab = base;   // the target fields stay empty: the batch reads them from the table
  ab.cur = cur.data();
  ab.n = total;
  ab.pending = pending.data();
  ab.partials = ab.partials2 = partials.data();
  ab.counter = counter.data();
  ab.accum = accum.data();
  ab.skip_count = skip.data();
  ab.cur_normals = sym ? nrm.data() : nullptr;
  ab.ctrl = ctrl.data();
  int iterations = 0;
  for (int it = 0; it < crit.max_iterations + 1; ++it) {
    for (int p = 0; p < B; ++p) {   // icp_iterate of each problem against its own target
      Single& r = single[p];
      const Target& T = target_of(p);
      const TreeView v = T.I.view(true);
      IterArgs a = base;
      a.nodes = v.nodes; a.pts = v.pts; a.root = v.root; a.cells = v.cells;
      a.tgt_normals = T.normals.data();
      a.cur = r.cur.data();
      a.n = sizes[p];
      a.pending = &r.pending;
      a.origin = r.ctrl.origin;
      a.partials = a.partials2 = r.partials.data();
      a.counter = &r.counter;
      a.accum = r.accum.data();
      a.skip_count = &r.skip;
      a.cur_normals = sym ? r.nrm.data() : nullptr;
      a.ctrl = &r.ctrl;
      CritParams cp = crit;
      cp.rmax = T.rmax;
      const unsigned g = wgrid(sizes[p]);
      if (track_mode != PCLB200_TRACK_ON) launch_grid(g, 256, [&] { k_search<false, false>(a, r.match.data(), r.lbs.data()); });
      if (track_mode != PCLB200_TRACK_OFF) launch_grid(g, 256, [&] { k_search<false, true>(a, r.match.data(), r.lbs.data()); });
      if (est == PCLB200_EST_SVD)
        launch_grid(agrid(sizes[p]), 256, [&] { k_accum_dmma<PCLB200_EST_SVD>(a, r.match.data()); });
      else if (est == PCLB200_EST_POINT_TO_PLANE_LLS)
        launch_grid(agrid(sizes[p]), 256, [&] { k_accum_dmma<PCLB200_EST_POINT_TO_PLANE_LLS>(a, r.match.data()); });
      else
        launch_grid(ggrid(sizes[p]), 256, [&] { k_accum<PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS>(a, r.match.data()); });
      launch_grid(1, 32, [&] {
        k_solve(r.accum.data(), est, dbl ? 1 : 0, tmode, r.ctrl.origin, 3, &r.pending, &r.so, 0, &r.ctrl, cp);
      });
    }
    // icp_iterate_batch with a batch of targets: one launch per stage
    const unsigned wn = (unsigned)wt.size(), an = (unsigned)at.size();
    const BatchTarget* tt = table.data();
    if (track_mode != PCLB200_TRACK_ON)
      launch_grid(wn, 256, [&] { k_search_batch<false, true>(ab, wt.data(), match.data(), lbs.data(), tt); });
    if (track_mode != PCLB200_TRACK_OFF)
      launch_grid(wn, 256, [&] { k_search_batch<true, true>(ab, wt.data(), match.data(), lbs.data(), tt); });
    if (est == PCLB200_EST_SVD)
      launch_grid(an, 256, [&] { k_accum_dmma_batch<PCLB200_EST_SVD, true>(ab, at.data(), match.data(), tt); });
    else if (est == PCLB200_EST_POINT_TO_PLANE_LLS)
      launch_grid(an, 256, [&] { k_accum_dmma_batch<PCLB200_EST_POINT_TO_PLANE_LLS, true>(ab, at.data(), match.data(), tt); });
    else
      launch_grid(an, 256, [&] { k_accum_batch<PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS, true>(ab, at.data(), match.data(), tt); });
    launch_grid((unsigned)((B * 32 + 255) / 256), 256, [&] {
      k_solve_batch(accum.data(), B, est, dbl ? 1 : 0, tmode, pending.data(), so.data(), 0, ctrl.data(), crit, tt);
    });
    bool all_done = true;
    for (int p = 0; p < B; ++p) {
      const Single& r = single[p];
      const size_t n = sizes[p];
      CHECK(std::memcmp(&match[off[p]], r.match.data(), n * sizeof(Match)) == 0, "%s it %d problem %d: matches differ", name, it, p);
      CHECK(std::memcmp(&cur[off[p]], r.cur.data(), n * sizeof(float4)) == 0, "%s it %d problem %d: queries differ", name, it, p);
      if (sym)
        CHECK(std::memcmp(&nrm[off[p]], r.nrm.data(), n * sizeof(float4)) == 0, "%s it %d problem %d: normals differ", name, it, p);
      CHECK(std::memcmp(&accum[(size_t)p * kAccum], r.accum.data(), kAccum * sizeof(double)) == 0,
            "%s it %d problem %d: accumulators differ", name, it, p);
      CHECK(std::memcmp(&ctrl[p], &r.ctrl, sizeof(LoopCtrl)) == 0, "%s it %d problem %d: loop states differ", name, it, p);
      CHECK(std::memcmp(&pending[p], &r.pending, sizeof(Pending)) == 0, "%s it %d problem %d: pending transforms differ", name, it, p);
      CHECK(std::memcmp(&so[p], &r.so, sizeof(SolveOut)) == 0, "%s it %d problem %d: solve outputs differ", name, it, p);
      CHECK(skip[p] == r.skip, "%s it %d problem %d: skip counts differ", name, it, p);
      all_done = all_done && ctrl[p].done;
    }
    iterations = it + 1;
    if (all_done) break;
  }
  int converged = 0, none = 0;
  for (int p = 0; p < B; ++p) {
    CHECK(std::memcmp(ctrl[p].final_T, single[p].ctrl.final_T, sizeof(ctrl[p].final_T)) == 0, "%s problem %d: final transforms differ",
          name, p);
    converged += ctrl[p].converged;
    none += ctrl[p].state == PCLB200_CONV_NO_CORRESPONDENCES;
  }
  CHECK(d_error == 0, "%s: device error flag %d", name, d_error);
  std::printf("%-40s B = %d, %d iterations, %d converged, %d without correspondences\n", name, B, iterations, converged, none);
}

int main()
{
  // three targets: the unit surface, the same far from the origin, and a larger one in a box of another size
  std::vector<Target> tg(3);
  tg[0].scale = 1.f;  tg[0].shift[0] = 0.f;     tg[0].shift[1] = 0.f;    tg[0].shift[2] = 0.f;
  tg[1].scale = 1.f;  tg[1].shift[0] = 1000.f;  tg[1].shift[1] = -600.f; tg[1].shift[2] = 40.f;
  tg[2].scale = 1.5f;  tg[2].shift[0] = -30.f;   tg[2].shift[1] = 12.f;   tg[2].shift[2] = -5.f;
  for (int k = 0; k < 3; ++k) make_target(tg[k], 5 + 7 * (unsigned)k);
  const std::vector<std::vector<size_t>> sets = {{300}, {1, 2, 700}, {1000, 2, 37, 257, 1, 555, 129}};
  const int ests[3] = {PCLB200_EST_SVD, PCLB200_EST_POINT_TO_PLANE_LLS, PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS};
  const char* est_name[3] = {"svd", "point-to-plane", "symmetric"};
  const int tracks[3] = {PCLB200_TRACK_OFF, PCLB200_TRACK_ON, PCLB200_TRACK_AUTO};
  const char* track_name[3] = {"off", "on", "auto"};
  for (const auto& sizes : sets)
    for (int e = 0; e < 3; ++e)
      for (int dbl = 0; dbl < 2; ++dbl)
        for (int t = 0; t < 3; ++t) {
          char name[96];
          std::snprintf(name, sizeof name, "%s %s tracking %s", est_name[e], dbl ? "double" : "float", track_name[t]);
          run(name, tg, sizes, ests[e], dbl != 0, tracks[t]);
        }
  std::printf("%ld checks, %ld failures\n%s\n", g_checks, g_fail, g_fail ? "FAILED" : "PASSED");
  return g_fail ? 1 : 0;
}
