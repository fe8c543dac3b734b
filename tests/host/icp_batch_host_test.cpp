// icp_batch_host_test.cpp — the batch kernels of pcl_b200/csrc/icp_kernels.cuh (k_search_batch, k_accum_dmma_batch,
// k_accum_batch, k_solve_batch, k_seed_origin_batch over batch_blocks's table) compiled for the HOST and run on a lock-step
// emulation of their thread blocks (tests/host/warp_emu.h), against the single-problem kernels run on each problem alone,
// driven the way icp.cu drives both (icp_iterate, icp_iterate_batch).  The grids are capped small so that problems span
// several virtual blocks.  Checked: every block table covers each problem's grid exactly once, in block order; after every
// iteration, per problem, the matches, the moved queries, the accumulators, the loop state, the pending transform and the
// solve output are byte-equal to the single run, and so is the final transform.  1, 3 and 7 problems with sizes that are
// not multiples of 32 or 256, 1- and 2-point problems; SVD, point-to-plane and symmetric; float and double; tracking off,
// on and automatic.  CPU only.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <cfloat>

#include "../../pcl_b200/csrc/icp_kernels.cuh"

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

struct Surface {
  std::vector<float> xyz;      // target
  std::vector<float4> normals; // by position of the index, {n, plane_offset} (icp.cu: normals_by_pos)
  HostIndex I;
};

static void surface_point(float x, float y, float* p, float* n)
{
  p[0] = x; p[1] = y; p[2] = 0.2f * std::sin(2.f * x) * std::cos(2.f * y);
  float m[3] = {-0.4f * std::cos(2.f * x) * std::cos(2.f * y), 0.4f * std::sin(2.f * x) * std::sin(2.f * y), 1.f};
  const float inv = 1.f / std::sqrt(m[0] * m[0] + m[1] * m[1] + m[2] * m[2]);
  for (int d = 0; d < 3; ++d) n[d] = m[d] * inv;
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

static void check_table(const std::vector<BatchBlock>& t, const std::vector<long long>& off, unsigned (*grid)(size_t),
                        const char* name)
{
  size_t k = 0;
  for (size_t p = 0; p + 1 < off.size(); ++p) {
    const size_t n = (size_t)(off[p + 1] - off[p]);
    const unsigned g = grid(n);
    for (unsigned v = 0; v < g; ++v, ++k) {
      CHECK(k < t.size(), "%s: table too short", name);
      if (k >= t.size()) return;
      const BatchBlock& b = t[k];
      CHECK(b.problem == (int)p && b.vblock == v && b.vgrid == g && b.part == k - v && b.begin == (unsigned long long)off[p] &&
                b.n == n, "%s: block %zu is not block %u of problem %zu's grid", name, k, v, p);
    }
  }
  CHECK(k == t.size(), "%s: %zu blocks for %zu in the grids", name, t.size(), k);
}

static void run(const char* name, const Surface& S, const std::vector<size_t>& sizes, int est, bool dbl, int track_mode)
{
  const HostIndex& I = S.I;
  const TreeView T = I.view(true);
  const int B = (int)sizes.size();
  const bool sym = est == PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS;
  std::vector<long long> off(1, 0);
  for (size_t n : sizes) off.push_back(off.back() + (long long)n);
  const size_t total = (size_t)off.back();
  // the sources: patches of the surface, each moved by its own small rigid motion, and their normals
  std::mt19937 rng(test_seed(17 + (unsigned)B));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::vector<float4> cur(total), nrm(total);
  for (int p = 0; p < B; ++p) {
    const float a = 0.02f * (float)(p + 1), c = std::cos(a), s = std::sin(a), tx = 0.01f * (float)(p % 3), ty = -0.005f * (float)p;
    const float x0 = 0.2f + 0.1f * (float)p, y0 = 0.3f;
    for (long long i = off[p]; i < off[p + 1]; ++i) {
      float q[3], m[3];
      surface_point(x0 + 1.2f * U(rng), y0 + 1.2f * U(rng), q, m);
      cur[i] = make_float4(c * q[0] - s * q[1] + tx, s * q[0] + c * q[1] + ty, q[2] + 0.003f, __int_as_float((int)i));
      nrm[i] = make_float4(c * m[0] - s * m[1], s * m[0] + c * m[1], m[2], 0.f);
    }
  }
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
  {
    double rmax = 0.0;
    for (int r = 0; r < 3; ++r) { const double m = std::max(std::fabs((double)I.lo[r]), std::fabs((double)I.hi[r])); rmax += m * m; }
    crit.rmax = std::sqrt(rmax);
  }
  int d_error = 0;
  IterArgs base;
  std::memset(&base, 0, sizeof base);
  base.nodes = T.nodes; base.pts = T.pts; base.root = T.root;
  base.tgt_normals = S.normals.data();
  base.plane_offsets = 1;
  base.gate = gate_from_max_dist(0.08);
  base.d_error = &d_error;
  base.enforce_same_dir = 1;
  base.cells = T.cells;
  base.track_sel = track_mode == PCLB200_TRACK_AUTO;
  base.peer.nranks = 0;

  // ---- the single runs: one problem each, its own grids
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
    r.ctrl = fresh_ctrl(I, track_mode);
    if (est == PCLB200_EST_SVD) k_seed_origin(r.cur.data(), nullptr, sizes[p], r.ctrl.origin);
  }
  // ---- the batch: the same problems end to end
  std::vector<Match> match(total, Match{-1, 0.f});
  std::vector<float> lbs(total, 0.f);
  std::vector<Pending> pending(B);
  std::vector<LoopCtrl> ctrl(B, fresh_ctrl(I, track_mode));
  std::vector<SolveOut> so(B);
  std::memset(pending.data(), 0, B * sizeof(Pending));
  std::memset(so.data(), 0, B * sizeof(SolveOut));
  for (auto& q : pending) q.mode = tmode;
  std::vector<unsigned> counter(B, 0);
  std::vector<unsigned long long> skip(B, 0);
  std::vector<double> accum((size_t)B * kAccum, 0.0);
  const std::vector<BatchBlock> wt = batch_blocks(off, wgrid), at = batch_blocks(off, sym ? ggrid : agrid);
  check_table(wt, off, wgrid, "search table");
  check_table(at, off, sym ? ggrid : agrid, "accumulation table");
  std::vector<double> partials(at.size() * 128, 0.0);
  std::vector<long long> offsets = off;
  if (est == PCLB200_EST_SVD)   // icp.cu seeds the SVD origin only
    launch_grid((unsigned)((B + 255) / 256), 256, [&] { k_seed_origin_batch(cur.data(), offsets.data(), B, ctrl.data()); });

  IterArgs ab = base;
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
    for (int p = 0; p < B; ++p) {   // icp_iterate of each problem
      Single& r = single[p];
      IterArgs a = base;
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
        k_solve(r.accum.data(), est, dbl ? 1 : 0, tmode, r.ctrl.origin, 3, &r.pending, &r.so, 0, &r.ctrl, crit);
      });
    }
    // icp_iterate_batch: one launch per stage
    const unsigned wn = (unsigned)wt.size(), an = (unsigned)at.size();
    if (track_mode != PCLB200_TRACK_ON) launch_grid(wn, 256, [&] { k_search_batch<false>(ab, wt.data(), match.data(), lbs.data()); });
    if (track_mode != PCLB200_TRACK_OFF) launch_grid(wn, 256, [&] { k_search_batch<true>(ab, wt.data(), match.data(), lbs.data()); });
    if (est == PCLB200_EST_SVD)
      launch_grid(an, 256, [&] { k_accum_dmma_batch<PCLB200_EST_SVD>(ab, at.data(), match.data()); });
    else if (est == PCLB200_EST_POINT_TO_PLANE_LLS)
      launch_grid(an, 256, [&] { k_accum_dmma_batch<PCLB200_EST_POINT_TO_PLANE_LLS>(ab, at.data(), match.data()); });
    else
      launch_grid(an, 256, [&] { k_accum_batch<PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS>(ab, at.data(), match.data()); });
    launch_grid((unsigned)((B * 32 + 255) / 256), 256, [&] {
      k_solve_batch(accum.data(), B, est, dbl ? 1 : 0, tmode, pending.data(), so.data(), 0, ctrl.data(), crit);
    });
    bool all_done = true;
    for (int p = 0; p < B; ++p) {
      const Single& r = single[p];
      const size_t n = sizes[p];
      CHECK(std::memcmp(&match[off[p]], r.match.data(), n * sizeof(Match)) == 0, "%s it %d problem %d: matches differ", name, it, p);
      CHECK(std::memcmp(&cur[off[p]], r.cur.data(), n * sizeof(float4)) == 0 || n == 0, "%s it %d problem %d: queries differ", name, it, p);
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
  Surface S;
  std::mt19937 rng(test_seed(5));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  const size_t nt = 6000;
  std::vector<float> tn(3 * nt);
  S.xyz.resize(3 * nt);
  for (size_t i = 0; i < nt; ++i) surface_point(2.5f * U(rng), 2.5f * U(rng), &S.xyz[3 * i], &tn[3 * i]);
  build_index(S.I, S.xyz, 4);
  const float qn = std::numeric_limits<float>::quiet_NaN();
  S.normals.resize(S.I.pts.size());
  for (size_t p = 0; p < S.I.pts.size(); ++p) {
    const int o = __float_as_int(S.I.pts[p].w);
    if (o == kSentinelIndex) { S.normals[p] = make_float4(qn, qn, qn, 0.f); continue; }
    S.normals[p] = make_float4(tn[3 * o], tn[3 * o + 1], tn[3 * o + 2], 0.f);
    S.normals[p].w = plane_offset(S.normals[p], S.I.pts[p]);
  }
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
          run(name, S, sizes, ests[e], dbl != 0, tracks[t]);
        }
  std::printf("%ld checks, %ld failures\n%s\n", g_checks, g_fail, g_fail ? "FAILED" : "PASSED");
  return g_fail ? 1 : 0;
}
