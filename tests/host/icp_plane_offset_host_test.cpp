// icp_plane_offset_host_test.cpp — the point-to-plane rows of k_accum_dmma (pcl_b200/csrc/icp_kernels.cuh) compiled for
// the HOST and run on a lock-step emulation of a 256-thread block (tests/host/warp_emu.h).  An ICP session stages its
// target normals with plane_offset in w (icp.cu: normals_by_pos, IterArgs::plane_offsets = 1) and the accumulation gathers
// that one record per pair; normals without it make the accumulation gather the matched point as well.  On a target whose
// normals include NaN and infinite components, over an index with padding slots (NaN normals, as normals_by_pos stages
// them): every row of the one-record form equals the row of the two gathers bit for bit, the two accumulations are
// bit-identical, and both equal plain fp64 sums with the pairs on non-finite normals skipped.  The one-record run is
// given no target points: it must not read them.  CPU only.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <cfloat>

#include "../../pcl_b200/csrc/icp_kernels.cuh"

int main()
{
  std::mt19937 rng(test_seed(91));
  std::uniform_real_distribution<float> U(0.f, 1.f);
  std::normal_distribution<float> N(0.f, 1.f);
  const std::size_t nt = 2500, ns = 3000;
  // a bumpy sheet 40 m above the frame's origin: plane_offset is large against the residual it is part of
  std::vector<float> txyz(3 * nt), tn(3 * nt);
  for (std::size_t i = 0; i < nt; ++i) {
    const float x = 3.f * U(rng) - 1.f, y = 3.f * U(rng) + 2.f, z = 0.3f * std::sin(2.f * x) + 40.f;
    txyz[3 * i] = x; txyz[3 * i + 1] = y; txyz[3 * i + 2] = z;
    float n[3] = {N(rng), N(rng), 1.f};
    const float inv = 1.f / std::sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
    for (int d = 0; d < 3; ++d) tn[3 * i + d] = n[d] * inv;
    if (i % 7 == 3) tn[3 * i + i % 3] = std::numeric_limits<float>::quiet_NaN();   // one NaN component, on each axis in turn
    if (i % 11 == 5) tn[3 * i + 1] = -std::numeric_limits<float>::infinity();
  }
  HostIndex I;
  build_index(I, txyz, 4);
  const float qn = std::numeric_limits<float>::quiet_NaN();
  std::vector<float4> staged(I.pts.size()), plain(I.pts.size());   // {n, plane_offset} / {n, 0}
  std::vector<int> real;   // positions holding a target point
  int padding = 0;
  for (std::size_t p = 0; p < I.pts.size(); ++p) {
    const int o = __float_as_int(I.pts[p].w);
    if (o == kSentinelIndex) {
      staged[p] = plain[p] = make_float4(qn, qn, qn, 0.f);
      ++padding;
      continue;
    }
    plain[p] = staged[p] = make_float4(tn[3 * o], tn[3 * o + 1], tn[3 * o + 2], 0.f);
    staged[p].w = plane_offset(staged[p], I.pts[p]);
    real.push_back((int)p);
  }
  CHECK(padding > 0, "the index has no padding slot to stage");
  std::vector<float4> cur(ns);
  std::vector<Match> match(ns);
  for (std::size_t i = 0; i < ns; ++i) {
    const int pos = real[(std::size_t)(U(rng) * (float)real.size()) % real.size()];
    const float4 q = I.pts[pos];
    cur[i] = make_float4(q.x + 0.02f * N(rng), q.y + 0.02f * N(rng), q.z + 0.02f * N(rng), __int_as_float((int)i));
    match[i].pos = i % 13 == 0 ? -1 : (i % 17 == 0 ? pos | kNotAccepted : pos);
    match[i].d2 = dist2_rn(cur[i].x, cur[i].y, cur[i].z, q.x, q.y, q.z);
  }
  std::vector<double> partials2(128, 0.0), accum1(kAccum, 0.0), accum2(kAccum, 0.0);
  unsigned counter = 0;
  int d_error = 0;
  IterArgs one, two;   // one record per pair (the session's layout) / the point and its normal
  std::memset(&one, 0, sizeof one);
  one.tgt_normals = staged.data();
  one.plane_offsets = 1;
  one.cur = cur.data();
  one.n = ns;
  one.partials2 = partials2.data();
  one.counter = &counter;
  one.d_error = &d_error;
  one.peer.nranks = 0;
  two = one;
  one.pts = nullptr;
  one.accum = accum1.data();
  two.pts = I.pts.data();
  two.tgt_normals = plain.data();
  two.plane_offsets = 0;
  two.accum = accum2.data();
  int rows_differ = 0, skipped = 0;
  double ref[kAccum] = {0};
  for (std::size_t i = 0; i < ns; ++i) {
    const Match m = match[i];
    const float4 p = match_accepted(m) ? cur[i] : make_float4(0.f, 0.f, 0.f, 0.f);   // k_accum_dmma
    float ra[8], rb[8], oa[8], ob[8];
    pair_rows<PCLB200_EST_POINT_TO_PLANE_LLS>(one, m, p, ra, rb);
    pair_rows<PCLB200_EST_POINT_TO_PLANE_LLS>(two, m, p, oa, ob);
    if (std::memcmp(ra, oa, sizeof ra) != 0 || std::memcmp(rb, ob, sizeof rb) != 0) ++rows_differ;
    if (!match_accepted(m)) continue;
    // plain fp64 sums of point_to_plane_lls.hpp:182-245 on the matched point
    const float4 q = I.pts[match_pos(m)], nn = plain[match_pos(m)];
    ref[0] += 1.0;
    ref[1] += (double)m.d2;
    if (!(std::isfinite(nn.x) && std::isfinite(nn.y) && std::isfinite(nn.z))) {
      ++skipped;
      continue;
    }
    const float sx = p.x, sy = p.y, sz = p.z, dx = q.x, dy = q.y, dz = q.z, nx = nn.x, ny = nn.y, nz = nn.z;
    const float A = nz * sy - ny * sz, B = nx * sz - nz * sx, C = ny * sx - nx * sy;
    const float D = nx * dx + ny * dy + nz * dz - nx * sx - ny * sy - nz * sz;
    const double v[6] = {A, B, C, nx, ny, nz};
    int k = 2;
    for (int r = 0; r < 6; ++r)
      for (int c = r; c < 6; ++c, ++k)
        ref[k] += (r >= 3) ? (double)((float)v[r] * (float)v[c]) : v[r] * v[c];   // the normal-normal block adds FLOAT products
    for (int r = 0; r < 6; ++r) ref[23 + r] += v[r] * (double)D;
  }
  CHECK(rows_differ == 0, "%d of %zu rows of one record differ from the rows of the two gathers", rows_differ, ns);
  CHECK(skipped > 0, "no accepted pair has a non-finite normal");
  blockDim.x = 256;
  warp_emu::run_block(256, [&] { k_accum_dmma<PCLB200_EST_POINT_TO_PLANE_LLS>(one, match.data()); });
  warp_emu::run_block(256, [&] { k_accum_dmma<PCLB200_EST_POINT_TO_PLANE_LLS>(two, match.data()); });
  CHECK(std::memcmp(accum1.data(), accum2.data(), kAccLls * sizeof(double)) == 0,
        "the accumulations of one record and of the two gathers differ");
  double worst = 0.0;
  for (int k = 0; k < kAccLls; ++k) {
    const double e = std::fabs(accum1[k] - ref[k]) / (1.0 + std::fabs(ref[k]));
    worst = std::isnan(e) ? INFINITY : std::max(worst, e);
  }
  CHECK(worst < 1e-11, "accumulated sums differ from plain fp64 sums by %g (relative)", worst);
  CHECK(d_error == 0, "device error flag %d", d_error);
  std::printf("point-to-plane rows from one record: %zu -> %zu points, %d padding slots, %d pairs on non-finite normals\n", ns, nt,
              padding, skipped);
  std::printf("%ld checks, %ld failures\n%s\n", g_checks, g_fail, g_fail ? "FAILED" : "PASSED");
  return g_fail ? 1 : 0;
}
