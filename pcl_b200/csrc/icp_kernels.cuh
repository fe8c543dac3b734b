// icp_kernels.cuh — the device side of one ICP iteration: the loop state, the search kernel (k_search), the normal
// equations on the fp64 tensor cores (k_accum_dmma) and per-thread (k_accum, k_accum_pairs: add_pair_terms),
// one fixed-order grid sum for all of them (grid_fold), the single-thread solve with
// the convergence criteria in its tail (k_solve).  A header so that icp.cu stays the host-side driver and so that
// tests/host/icp_host_test.cpp can compile the SAME source for the host (a lock-step emulation of a thread block) and run
// whole iterations against the oracle's arithmetic.
#pragma once
#include "internal.cuh"
#include "corr_select.cuh"
#include "grid_sum.cuh"
#include "peer_exchange.cuh"
#include "traverse.cuh"

namespace pclb200 {

// accumulator slots (fp64)
//   common : [0] accepted pairs, [1] sum of squared distances
//   SVD    : [2..4] sum(p-o)  [5..7] sum(q-o)  [8..16] sum (q-o)(p-o)^T row-major, about an origin o near the pairs:
//            k_solve forms sum(q-o)(p-o)^T / n - m_q m_p^T (m = centroid - o), whose relative error grows like
//            (|m| / spread of the pairs)^2, so o must lie near the pairs.  o is a float point (p - o is exact in fp64):
//            in the loop LoopCtrl::origin, stand-alone the first pair's target point that is finite.
//   LLS    : [2..22] upper triangle of A^T A (row-major order 0,1,..5,7,..), [23..28] A^T b
constexpr int kAccSvd = 17;
constexpr int kAccLls = 29;

// transform left in device memory between iterations
struct Pending {
  float f[12];   // rows 0..2 of T_k, already rounded like the reference (cast<float>)
  double d[12];  // same rows in double (Transformer<double> path)
  int apply;     // 0 = identity / nothing to apply
  int mode;      // kApply* (internal.cuh): the reference's operation order
};

struct SolveOut {
  double T[16];  // row-major, rounded to Scalar
  double n;
  double sum_d;
  int ok;
  int pad;
};

// Loop state that lives on the device so that a whole align() can be enqueued without a host round trip per iteration:
// k_solve composes final = T_k * final, counts the iteration and evaluates DefaultConvergenceCriteria itself; once a
// criterion fires (or there are too few correspondences) `done` turns the remaining enqueued kernels into no-ops.
struct LoopCtrl {
  int done;                // remaining enqueued iterations must not run
  int iterations;          // nr_iterations_
  int state;               // PCLB200_CONV_*
  int converged;
  int iterations_similar;  // DefaultConvergenceCriteria::iterations_similar_transforms_
  int track_next;          // the next search keeps / uses the temporal-coherence bounds
  int lb_valid;            // the previous search wrote them
  int n_run;               // iterations executed since the host last reset it
  double prev_mse, mse, n_corr;
  long long total_corr;
  double final_T[16], last_T[16];
  // origin of the SVD sums (x, y, z; [3] unused), on the device because the iterations are enqueued ahead: k_solve sets
  // it to the float-rounded centroid of each iteration's target points, taken from the (cross-rank) totals so that every
  // rank holds the same one.  The first iteration uses the first finite point of the staged source (k_seed_origin) on a
  // single rank, and the target's bounding-box centre with a communicator.
  float origin[4];
};

struct CritParams {  // what DefaultConvergenceCriteria and the tracking heuristic need (pclb200_icp_params subset)
  int max_iterations, failure_after_max_iter, max_iterations_similar, scalar_is_double, track_mode;
  double rot_eps, trans_eps, rel_mse, abs_mse;
  double rmax;  // sqrt(sum_axis max(|lo|, |hi|)^2) of the target frame: bounds the displacement a rotation causes
};

__device__ __forceinline__ void apply_pending(const Pending& P, float& x, float& y, float& z)
{
  const float px = x, py = y, pz = z;
  if (P.mode == kApplyIcp) {
    x = ((P.f[0] * px + P.f[1] * py) + P.f[2] * pz) + P.f[3];
    y = ((P.f[4] * px + P.f[5] * py) + P.f[6] * pz) + P.f[7];
    z = ((P.f[8] * px + P.f[9] * py) + P.f[10] * pz) + P.f[11];
  }
  else if (P.mode == kApplyTransformsFloat) {
    x = P.f[0] * px + (P.f[1] * py + (P.f[2] * pz + P.f[3]));
    y = P.f[4] * px + (P.f[5] * py + (P.f[6] * pz + P.f[7]));
    z = P.f[8] * px + (P.f[9] * py + (P.f[10] * pz + P.f[11]));
  }
  else if (P.mode == kApplyValidationDouble) {
    const double dx = px, dy = py, dz = pz;
    x = (float)(((P.d[0] * dx + P.d[1] * dy) + P.d[2] * dz) + P.d[3]);
    y = (float)(((P.d[4] * dx + P.d[5] * dy) + P.d[6] * dz) + P.d[7]);
    z = (float)(((P.d[8] * dx + P.d[9] * dy) + P.d[10] * dz) + P.d[11]);
  }
  else {  // kApplyTransformsDouble
    const double dx = px, dy = py, dz = pz;
    x = (float)(((P.d[3] + dx * P.d[0]) + dy * P.d[1]) + dz * P.d[2]);
    y = (float)(((P.d[7] + dx * P.d[4]) + dy * P.d[5]) + dz * P.d[6]);
    z = (float)(((P.d[11] + dx * P.d[8]) + dy * P.d[9]) + dz * P.d[10]);
  }
}

__device__ __forceinline__ void apply_pending_normal(const Pending& P, float& x, float& y, float& z)
{
  const float px = x, py = y, pz = z;
  if (P.mode == kApplyIcp) {
    x = (P.f[0] * px + P.f[1] * py) + P.f[2] * pz;
    y = (P.f[4] * px + P.f[5] * py) + P.f[6] * pz;
    z = (P.f[8] * px + P.f[9] * py) + P.f[10] * pz;
  }
  else if (P.mode == kApplyTransformsFloat) {
    x = P.f[0] * px + (P.f[1] * py + P.f[2] * pz);
    y = P.f[4] * px + (P.f[5] * py + P.f[6] * pz);
    z = P.f[8] * px + (P.f[9] * py + P.f[10] * pz);
  }
  else {  // the double orders
    const double dx = px, dy = py, dz = pz;
    x = (float)((dx * P.d[0] + dy * P.d[1]) + dz * P.d[2]);
    y = (float)((dx * P.d[4] + dy * P.d[5]) + dz * P.d[6]);
    z = (float)((dx * P.d[8] + dy * P.d[9]) + dz * P.d[10]);
  }
}

__device__ __forceinline__ void transform_one(const Pending& P, float4* __restrict__ pts, size_t i,
                                              float4* __restrict__ normals /* nullable */)
{
  float4 p = pts[i];
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z)))
    return;
  apply_pending(P, p.x, p.y, p.z);
  pts[i] = p;
  if (normals) {
    float4 m = normals[i];
    if (P.mode == kApplyIcp && !(isfinite(m.x) && isfinite(m.y) && isfinite(m.z)))
      return;  // icp.hpp:97-98
    apply_pending_normal(P, m.x, m.y, m.z);
    normals[i] = m;
  }
}

// a batch (BatchBlock below): point i moved by the Pending of its problem, where that one applies
__global__ void k_transform_batch(float4* __restrict__ pts, size_t n, const long long* __restrict__ offsets,
                                  int n_problems, const Pending* __restrict__ P, float4* __restrict__ normals)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const Pending& Q = P[problem_of(offsets, n_problems, (long long)i)];
    if (Q.apply)
      transform_one(Q, pts, i, normals);
  }
}

struct IterArgs {
  const BvhNode* nodes;
  const float4* pts;
  int root;
  const float4* tgt_normals;  // Morton order of the target (LLS only)
  int plane_offsets;          // 1: w of tgt_normals = plane_offset of the point there (normals_by_pos), 0: w unused
  float4* cur;                // source, Morton order, w = slot
  size_t n;
  const Pending* pending;
  float gate;
  const float* origin;        // origin of the SVD sums: LoopCtrl::origin (3 floats)
  double* partials;           // gridDim.x * kAccum
  double* partials2;          // gridDim.x * 128 (two 8x8 fp64 tiles per block: k_accum_dmma)
  unsigned* counter;
  double* accum;              // kAccum
  int* d_error;
  // reciprocal (optional)
  const BvhNode* s_nodes;
  const float4* s_pts;
  int s_root;
  const int32_t* src_orig;    // slot -> original source index (nullable = identity)
  unsigned long long* skip_count;  // queries answered by the temporal-coherence test (statistics)
  float4* cur_normals;             // source normals, same order as cur (symmetric objective), rotated with T_k
  int enforce_same_dir;
  CellTable cells;                 // cell table of the target index (walks start at the candidate ball)
  LoopCtrl* ctrl;                  // device-side loop state: a finished loop (`done`) turns the kernel into a no-op
  int track_sel;                   // 1: the search kernel runs only if ctrl->track_next matches its TRACK flavour
  // fused cross-GPU reduce (optional): peer-mapped exchange buffers + this iteration's sequence number
  PeerView peer;
  unsigned long long seq;
};

// Fused all-reduce over NVLink peer memory (replaces a separate ncclAllReduce launch); called by every thread of the
// LAST block of an accumulating kernel once a.accum[0..kAccum) holds this rank's totals.
__device__ __forceinline__ void peer_exchange(const IterArgs& a)
{
  peer_exchange(a.peer, a.seq, a.accum, a.accum, kAccum, 0.0, [](double s, double x) { return s + x; }, a.d_error);
}

// match of one query, in the (Hilbert) slot order of `cur`: this iteration's result and the next iteration's seed
struct __align__(8) Match {
  int pos;   // position of the nearest target point in the Morton array; -1 = none inside the gate;
             // kNotAccepted set = found, but not a correspondence of this iteration (gate on a carried-over match,
             // reciprocal test failed, dropped by a rejector) — still the seed of the next search
  float d2;  // squared distance to it
};
constexpr int kNotAccepted = 1 << 30;
constexpr int kPosMask = kNotAccepted - 1;
__host__ __device__ __forceinline__ bool match_accepted(const Match& m) { return m.pos >= 0 && !(m.pos & kNotAccepted); }
__host__ __device__ __forceinline__ int match_pos(const Match& m) { return m.pos & kPosMask; }  // only if m.pos >= 0

#ifdef PCLB_STATS
__device__ unsigned long long g_walk_stats[8];
__device__ unsigned long long g_walk_imbalance[2];
__device__ unsigned long long g_walk_hist[64];
#endif

// kRelMargin, kTrackInflate, still_nearest: traverse.cuh (host-testable: tests/host/traverse_host_test.cpp)

// ---- normal equations on the fp64 tensor cores ------------------------------------------------------------------------
// The 3x3 / 6x6 normal equations of one ICP iteration are sums of outer products over the correspondences, i.e. V^T V
// with one row of <= 8 components per pair — a dense fp64 contraction.  A warp stages the rows of its 32 pairs in shared
// memory (two 32 x 8 float tiles: every component is a float, or a float minus the fp64 accumulation origin) and issues
// mma.sync.m8n8k4.f64: lane (g = lane / 4, t = lane % 4) feeds component g of pair 4 * step + t as both the A (row g,
// column t) and the B (row t, column g) fragment, and holds C[g][2t], C[g][2t + 1].  The whole accumulator tile lives
// in TWO fp64 registers per lane instead of 29 per thread, so the accumulation can ride in the search kernel.
//   SVD  : tile 0 = sum w u^T, w = (q - o, 1, d2), u = (p - o, 1)   -> sum q p^T, sum q, sum p, n, sum d2
//   LLS  : tile 0 = sum v v^T, v = (A, B, C, nx, ny, nz, D)         -> A^T A without its normal-normal block, A^T b
//          tile 1 column 0 = sum w, w = (nx nx, nx ny, nx nz, ny ny, ny nz, nz nz as FLOAT products — the reference
//          adds float products there, point_to_plane_lls.hpp:228-233 —, d2, 1)
// Products are exact fp64 products of the widened floats (the reference multiplies the same widened values), sums are
// fp64 in a fixed order: bitwise reproducible, and within fp64 round-off of the oracle's sequential sums.
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b)
{
#ifdef PCLB_HOST_EMULATION  // tests/host: the fragment layout of the instruction, emulated across the lanes of the warp
  emu_dmma884(c0, c1, a, b);
#else
  asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
#endif
}

#ifndef PCLB_ACCUM_BLOCKS
#define PCLB_ACCUM_BLOCKS 5
#endif
constexpr int kAccumBlocksPerSM = PCLB_ACCUM_BLOCKS;

// The target point's own part of the point-to-plane residual nx dx + ny dy + nz dz - nx sx - ny sy - nz sz
// (point_to_plane_lls.hpp:235): that float expression is evaluated left to right (no fma: -fmad=false), so its first
// three terms depend on the target point alone and give the same bits whenever they are computed.  The Morton-ordered
// target normals of an ICP session carry it in their w lane ({nx, ny, nz, plane_offset}, IterArgs::plane_offsets), so
// that the accumulation gathers one 16-B record per pair instead of the point and its normal.
__host__ __device__ __forceinline__ float plane_offset(const float4& n, const float4& q)
{
  return n.x * q.x + n.y * q.y + n.z * q.z;
}

// One pair's row of the contraction: ra = the MMA operand (w for SVD, v for LLS), rb = u (SVD) / the eight plain sums'
// terms (LLS).  The gathers of the pair's target records (SVD: the matched point; LLS: its normal, and the point only
// when the normals carry no plane_offset) are issued here; rows of pairs that are not accepted stay zero.
template <int EST>
__device__ __forceinline__ void pair_rows(const IterArgs& a, const Match& m, const float4& p, float (&ra)[8], float (&rb)[8])
{
#pragma unroll
  for (int k = 0; k < 8; ++k)
    ra[k] = rb[k] = 0.f;
  if (match_accepted(m)) {
    if (EST == PCLB200_EST_SVD) {
      const float4 q = ldg4(a.pts + m.pos);
      ra[0] = q.x; ra[1] = q.y; ra[2] = q.z; ra[3] = 1.f; ra[4] = m.d2;
      rb[0] = p.x; rb[1] = p.y; rb[2] = p.z; rb[3] = 1.f;
    }
    else {
      rb[6] = m.d2;
      rb[7] = 1.f;
      const float4 nn = ldg4(a.tgt_normals + m.pos);
      if (isfinite(nn.x) && isfinite(nn.y) && isfinite(nn.z)) {  // point_to_plane_lls.hpp:182-190
        const float sx = p.x, sy = p.y, sz = p.z, nx = nn.x, ny = nn.y, nz = nn.z;
        // float expressions, widened to double when they enter the products, exactly as :202-204 and :235
        // (no fma: -fmad=false)
        ra[0] = nz * sy - ny * sz;
        ra[1] = nx * sz - nz * sx;
        ra[2] = ny * sx - nx * sy;
        ra[3] = nx; ra[4] = ny; ra[5] = nz;
        if (a.plane_offsets) {
          ra[6] = nn.w - nx * sx - ny * sy - nz * sz;  // nn.w = plane_offset(nn, q): the same bits
        }
        else {
          const float4 q = ldg4(a.pts + m.pos);
          ra[6] = nx * q.x + ny * q.y + nz * q.z - nx * sx - ny * sy - nz * sz;
        }
        rb[0] = nx * nx; rb[1] = nx * ny; rb[2] = nx * nz;
        rb[3] = ny * ny; rb[4] = ny * nz; rb[5] = nz * nz;
      }
    }
  }
}

// tiles: 2 x 32 x 8 floats of this warp's shared memory.  Must be called by all 32 lanes (converged).  Even steps
// accumulate into (ca, cb), odd steps into (da, db): two independent MMA chains.  LLS: w collects component g of the
// plain sums (float products of the normal, d2, count) over this lane's pairs — an MMA would spend a whole 8x8x4 tile on
// them, and one fp64 register per lane is cheaper than eight per thread.
template <int EST>
__device__ __forceinline__ void mma_rows(const IterArgs& a, float* __restrict__ tiles, int lane, const float (&ra)[8],
                                         const float (&rb)[8], double& ca, double& cb, double& da, double& db, double& w)
{
  float* tA = tiles;
  float* tB = tiles + 32 * 8;
  *reinterpret_cast<float4*>(tA + lane * 8) = make_float4(ra[0], ra[1], ra[2], ra[3]);
  *reinterpret_cast<float4*>(tA + lane * 8 + 4) = make_float4(ra[4], ra[5], ra[6], ra[7]);
  *reinterpret_cast<float4*>(tB + lane * 8) = make_float4(rb[0], rb[1], rb[2], rb[3]);
  *reinterpret_cast<float4*>(tB + lane * 8 + 4) = make_float4(rb[4], rb[5], rb[6], rb[7]);
  __syncwarp();
  const int g = lane >> 2, t = lane & 3;
  const double og = EST == PCLB200_EST_SVD && g < 3 ? (double)a.origin[g] : 0.0;
#pragma unroll
  for (int st = 0; st < 8; ++st) {
    const int row = (4 * st + t) * 8;
    double va = (double)tA[row + g];
    if (EST == PCLB200_EST_SVD) {
      double vb = (double)tB[row + g];
      if (g < 3) {  // coordinates enter shifted by the accumulation origin, in fp64; pairs that are not accepted stay zero
        const bool on = tA[row + 3] != 0.f;
        va = on ? va - og : 0.0;
        vb = on ? vb - og : 0.0;
      }
      if (st & 1)
        dmma884(da, db, va, vb);     // C1[i][j] += w_i u_j
      else
        dmma884(ca, cb, va, vb);
    }
    else {
      if (st & 1)
        dmma884(da, db, va, va);     // C1[i][j] += v_i v_j
      else
        dmma884(ca, cb, va, va);
      w += (double)tB[row + g];
    }
  }
  __syncwarp();
}

// where accumulator slot k of the kAccum layout (top of this file) sits in the two 8x8 tiles: tile * 64 + row * 8 + col
__device__ __forceinline__ int dmma_accum_source(int est, int k)
{
  if (est == PCLB200_EST_SVD) {
    if (k == 0) return 3 * 8 + 3;
    if (k == 1) return 4 * 8 + 3;
    if (k < 5) return 3 * 8 + (k - 2);
    if (k < 8) return (k - 5) * 8 + 3;
    if (k < 17) return ((k - 8) / 3) * 8 + (k - 8) % 3;
    return -1;
  }
  if (k == 0) return 64 + 7 * 8;
  if (k == 1) return 64 + 6 * 8;
  if (k < 23) {
    int t = k - 2, r = 0;
    while (t >= 6 - r) {
      t -= 6 - r;
      ++r;
    }
    const int c = r + t;
    if (r >= 3)
      return 64 + ((r == 3 ? c - 3 : (r == 4 ? 3 + (c - 4) : 5))) * 8;
    return r * 8 + c;
  }
  if (k < 29) return (k - 23) * 8 + 6;
  return -1;
}

// warp tiles -> block (fixed order) -> grid (fixed order, last block) -> the kAccum layout k_solve reads -> peers.
// Must be called by every thread of every block; blockDim.x = NWARPS * 32 >= 128.
template <int EST, int NWARPS, class G>
__device__ __forceinline__ void fold_tiles_and_publish(const IterArgs& a, double c1a, double c1b, double w, const G& grid)
{
  __shared__ double s_tiles[NWARPS][128];
  __shared__ double s_fin[128];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  s_tiles[warp][g * 8 + 2 * t] = c1a;
  s_tiles[warp][g * 8 + 2 * t + 1] = c1b;
  s_tiles[warp][64 + lane] = 0.0;       // tile 1: only column 0 is used (the eight plain sums)
  s_tiles[warp][96 + lane] = 0.0;
  __syncwarp();
  {
    double v = w;  // lane (g, t) holds plain sum g over its pairs: fold the four t lanes
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    if (t == 0)
      s_tiles[warp][64 + g * 8] = v;
  }
  __syncthreads();
  if (!grid_fold<128, 128>(&s_tiles[0][0], NWARPS, a.partials2, a.counter, is_last, s_fin, grid))
    return;
  __syncthreads();
  if (threadIdx.x < kAccum) {
    const int src = dmma_accum_source(EST, threadIdx.x);
    a.accum[threadIdx.x] = src >= 0 ? s_fin[src] : 0.0;
  }
  if (threadIdx.x == 0)
    *a.counter = 0;
  peer_exchange(a);
}

// Search kernel, one query per thread: apply the pending T_k in place (reference fp32 operation order, icp.hpp:49-111)
// -> [TRACK: skip test] -> exact 1-NN started at the candidate ball (traverse.cuh: nearest1 — seed = previous match,
// cell-table start, ordinary exact walk below) -> gate -> optional reciprocal back-search.
// lbs (TRACK only): per query, a lower bound on the DISTANCE to every target point other than the match; 0 = unknown.
// 5 blocks of 256 threads per SM (<= 48 registers).  The walk is a chain of dependent loads that occupancy hides, but at
// 6 blocks (40 registers) the visitor and walk state spill inside the node loop; on H100 the 5-block build is 6 % faster.
// search_queries: the body, over the queries of this block's place in `grid` (grid_sum.cuh: k_search runs on the
// launch's grid, k_search_batch on one problem's grid inside the batch launch)
template <bool RECIP, bool TRACK, class G>
__device__ __forceinline__ void search_queries(const IterArgs& a, Match* __restrict__ match, float* __restrict__ lbs,
                                               const G& grid)
{
  if (a.ctrl) {  // enqueued ahead of the host: a finished loop, or the other TRACK flavour, leaves nothing to do
    if (a.ctrl->done || (a.track_sel && (a.ctrl->track_next != 0) != TRACK))
      return;
  }
  const bool lb_ok = a.ctrl ? a.ctrl->lb_valid != 0 : true;  // bounds of an earlier TRACK phase say nothing now
  __shared__ Pending sP;
  if (threadIdx.x == 0)
    sP = *a.pending;
  __syncthreads();
  const TreeView T{a.nodes, a.pts, a.root, a.cells};
  const int lane = threadIdx.x & 31;
  bool overflow = false;
  unsigned skipped = 0;
  WalkStats ws{};
#ifdef PCLB_STATS
  unsigned my_nodes = 0;
#endif
  const size_t stride = (size_t)grid.blocks() * blockDim.x;
  for (size_t base = grid.block() * (size_t)blockDim.x + (threadIdx.x & ~31); base < a.n; base += stride) {
    const size_t i = base + lane;
    const bool in_range = i < a.n;
    float4 p = in_range ? a.cur[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    Match prev;
    prev.pos = -1;
    prev.d2 = 0.f;
    if (in_range)
      prev = match[i];
    Match m;
    m.pos = -1;
    m.d2 = 0.f;
    float lb_out = 0.f;
    if (in_range && isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
      // non-finite points: transformCloud leaves them untouched (icp.hpp:90-91), no correspondence (:173-174)
      float delta = 0.f;
      if (sP.apply) {
        const float ox = p.x, oy = p.y, oz = p.z;
        apply_pending(sP, p.x, p.y, p.z);
        a.cur[i] = p;
        delta = sqrtf(dist2_rn(p.x, p.y, p.z, ox, oy, oz));
        if (a.cur_normals) {
          float4 nn = a.cur_normals[i];
          apply_pending_normal(sP, nn.x, nn.y, nn.z);
          a.cur_normals[i] = nn;
        }
      }
      const int seed = prev.pos >= 0 ? match_pos(prev) : -1;
      float nlb = 0.f;
      if (TRACK && !RECIP && seed >= 0 && lb_ok && still_nearest(prev.d2, lbs[i], delta, &nlb)) {
        const float4 q = ldg4(a.pts + seed);
        m.d2 = dist2_rn(p.x, p.y, p.z, q.x, q.y, q.z);
        // distance[0] > max_dist_sqr drops the pair (correspondence_estimation.hpp:176); the match stays the seed
        m.pos = m.d2 <= a.gate ? seed : (seed | kNotAccepted);
        lb_out = nlb;
        ++skipped;
      }
      else {
        const float inf = __int_as_float(0x7f800000);
        Nearest1T<TRACK> v{p.x, p.y, p.z, a.gate, kSentinelIndex, -1, inf, inf, inf};
#ifdef PCLB_STATS
        const unsigned nodes_before = ws.n[1];
#endif
        if (!nearest1<TRACK>(T, p.x, p.y, p.z, v, seed, TRACK ? kTrackInflate : 1.00001f, ws))
          overflow = true;
#ifdef PCLB_STATS
        my_nodes = ws.n[1] - nodes_before;
#endif
        if (v.best_pos >= 0) {
          m.pos = v.best_pos;
          m.d2 = v.best;
          lb_out = TRACK ? sqrtf(v.lower_bound2()) : 0.f;
          if (RECIP) {
            // correspondence_estimation.hpp:259-269: 1-NN of the matched target point back into the source
            const float4 q = ldg4(a.pts + v.best_pos);
            Nearest1 b{q.x, q.y, q.z, a.gate, kSentinelIndex, -1};
            if (!traverse(a.s_nodes, a.s_pts, a.s_root, q.x, q.y, q.z, b))
              overflow = true;
            const int slot = __float_as_int(p.w);
            const int my_orig = a.src_orig ? a.src_orig[slot] : slot;
            if (!(b.best_pos >= 0 && b.best_idx == my_orig))
              m.pos |= kNotAccepted;
          }
        }
      }
    }
    if (in_range) {
      match[i] = m;
      if (TRACK)
        lbs[i] = lb_out;
    }
#ifdef PCLB_STATS
    {
      // per-warp imbalance of the node visits: sum over lanes and 32 x max over lanes (their ratio = lane utilisation bound)
      unsigned sm = my_nodes, mx = my_nodes;
      for (int o = 16; o > 0; o >>= 1) {
        sm += __shfl_xor_sync(0xffffffffu, sm, o);
        mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      }
      if (lane == 0) {
        atomicAdd(&g_walk_imbalance[0], (unsigned long long)sm);
        atomicAdd(&g_walk_imbalance[1], (unsigned long long)mx * 32ull);
      }
      atomicAdd(&g_walk_hist[min(my_nodes, 63u)], 1ull);
      my_nodes = 0;
    }
#endif
  }
#ifdef PCLB_STATS
  for (int k = 0; k < 8; ++k)
    atomicAdd(&g_walk_stats[k], (unsigned long long)ws.n[k]);
#endif
  if (TRACK) {
    for (int o = 16; o > 0; o >>= 1)
      skipped += __shfl_xor_sync(0xffffffffu, skipped, o);
    if (lane == 0 && skipped)
      atomicAdd(a.skip_count, (unsigned long long)skipped);
  }
  if (overflow)
    atomicExch(a.d_error, kErrStackOverflow);
}

template <bool RECIP, bool TRACK>
__global__ void __launch_bounds__(256, 5)
k_search(const IterArgs a, Match* __restrict__ match, float* __restrict__ lbs)
{
  search_queries<RECIP, TRACK>(a, match, lbs, HwGrid());
}

// Streaming accumulation on the fp64 tensor cores: one pass over (source point, match) pairs, the normal equations
// built by pair_rows + mma_rows.  The kernel is bound by the latency of match -> gather: resident warps are what hides
// it (two pairs in flight per thread at half the occupancy was slower), so the state is kept to ten fp64 registers of
// accumulators per lane instead of 29 per thread.
template <int EST, class G>
__device__ __forceinline__ void accum_dmma_pairs(const IterArgs& a, const Match* __restrict__ match, const G& grid)
{
  if (a.ctrl && a.ctrl->done)
    return;
  __shared__ __align__(16) float s_stage[8][2 * 32 * 8];
  const int lane = threadIdx.x & 31;
  double ca = 0.0, cb = 0.0, da = 0.0, db = 0.0, w = 0.0;
  const size_t stride = (size_t)grid.blocks() * blockDim.x;
  float* tiles = s_stage[threadIdx.x >> 5];
  for (size_t base = grid.block() * (size_t)blockDim.x + (threadIdx.x & ~31); base < a.n; base += stride) {
    const size_t i = base + lane;
    Match m;
    m.pos = -1;
    m.d2 = 0.f;
    if (i < a.n)
      m = match[i];
    float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
    if (match_accepted(m))
      p = a.cur[i];
    float ra[8], rb[8];
    pair_rows<EST>(a, m, p, ra, rb);
    mma_rows<EST>(a, tiles, lane, ra, rb, ca, cb, da, db, w);
  }
  fold_tiles_and_publish<EST, 8>(a, ca + da, cb + db, w, grid);
}

template <int EST>
__global__ void __launch_bounds__(256, kAccumBlocksPerSM)
k_accum_dmma(const IterArgs a, const Match* __restrict__ match)
{
  accum_dmma_pairs<EST>(a, match, HwGrid());
}

// One pair's terms of the normal equations (slot layout at the top of this file), added to acc[2..): p source point, q
// target point, o the accumulation origin (SVD), nq the target normal (LLS), np the source normal and enforce_same_dir
// (symmetric objective).  A pair whose normal is not finite adds nothing here: the estimator skips it, but it is still a
// correspondence, so the callers count it in acc[0..1] first.
template <int EST>
__device__ __forceinline__ void add_pair_terms(double* acc, const float4& p, const float4& q, const float3& o,
                                               const float4& nq, const float4& np, int enforce_same_dir)
{
  if (EST == PCLB200_EST_SVD) {
    const double px = (double)p.x - (double)o.x, py = (double)p.y - (double)o.y, pz = (double)p.z - (double)o.z;
    const double qx = (double)q.x - (double)o.x, qy = (double)q.y - (double)o.y, qz = (double)q.z - (double)o.z;
    acc[2] += px; acc[3] += py; acc[4] += pz;
    acc[5] += qx; acc[6] += qy; acc[7] += qz;
    acc[8] += qx * px; acc[9] += qx * py; acc[10] += qx * pz;
    acc[11] += qy * px; acc[12] += qy * py; acc[13] += qy * pz;
    acc[14] += qz * px; acc[15] += qz * py; acc[16] += qz * pz;
  }
  else if (EST == PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS) {
    // symmetric_point_to_plane_lls.hpp:166-193: n = n1 +/- n2, v = [(p+q) x n, n], A^T A += v v^T, A^T b += v ((q-p).n)
    const float4 &n1 = np, &n2 = nq;
    const double d12 = (double)n1.x * n2.x + (double)n1.y * n2.y + (double)n1.z * n2.z;
    const double sg = (!enforce_same_dir || d12 >= 0.0) ? 1.0 : -1.0;
    const double nx = (double)n1.x + sg * n2.x, ny = (double)n1.y + sg * n2.y, nz = (double)n1.z + sg * n2.z;
    if (!(isfinite(nx) && isfinite(ny) && isfinite(nz)))
      return;
    const double sx = (double)p.x + q.x, sy = (double)p.y + q.y, sz = (double)p.z + q.z;
    const double v[6] = {sy * nz - sz * ny, sz * nx - sx * nz, sx * ny - sy * nx, nx, ny, nz};
    const double b = ((double)q.x - p.x) * nx + ((double)q.y - p.y) * ny + ((double)q.z - p.z) * nz;
    int t = 2;
#pragma unroll
    for (int r = 0; r < 6; ++r)
#pragma unroll
      for (int cc = r; cc < 6; ++cc)
        acc[t++] += v[r] * v[cc];
#pragma unroll
    for (int r = 0; r < 6; ++r)
      acc[23 + r] += v[r] * b;
  }
  else {
    if (!(isfinite(nq.x) && isfinite(nq.y) && isfinite(nq.z)))
      return;  // point_to_plane_lls.hpp:182-190
    const float sx = p.x, sy = p.y, sz = p.z, dx = q.x, dy = q.y, dz = q.z, nx = nq.x, ny = nq.y, nz = nq.z;
    // float expressions widened to double, exactly as :202-204 and :235 (no fma: -fmad=false)
    const double A = (double)(nz * sy - ny * sz);
    const double B = (double)(nx * sz - nz * sx);
    const double C = (double)(ny * sx - nx * sy);
    const double D = (double)(nx * dx + ny * dy + nz * dz - nx * sx - ny * sy - nz * sz);
    acc[2] += A * A; acc[3] += A * B; acc[4] += A * C;
    acc[5] += A * (double)nx; acc[6] += A * (double)ny; acc[7] += A * (double)nz;
    acc[8] += B * B; acc[9] += B * C;
    acc[10] += B * (double)nx; acc[11] += B * (double)ny; acc[12] += B * (double)nz;
    acc[13] += C * C;
    acc[14] += C * (double)nx; acc[15] += C * (double)ny; acc[16] += C * (double)nz;
    acc[17] += (double)(nx * nx); acc[18] += (double)(nx * ny); acc[19] += (double)(nx * nz);
    acc[20] += (double)(ny * ny); acc[21] += (double)(ny * nz);
    acc[22] += (double)(nz * nz);
    acc[23] += A * D; acc[24] += B * D; acc[25] += C * D;
    acc[26] += (double)nx * D; acc[27] += (double)ny * D; acc[28] += (double)nz * D;
  }
}

// The symmetric objective inside the loop (the other estimators run on k_accum_dmma): one streaming pass over (source
// point, match) pairs, per-thread fp64 sums, fixed reduction order.
template <int EST, class G>
__device__ __forceinline__ void accum_pairs(const IterArgs& a, const Match* __restrict__ match, const G& grid)
{
  static_assert(EST == PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS, "the other estimators accumulate in k_accum_dmma");
  if (a.ctrl && a.ctrl->done)
    return;
  double acc[kAccLls];
#pragma unroll
  for (int t = 0; t < kAccLls; ++t)
    acc[t] = 0.0;
  for (size_t i = grid.block() * (size_t)blockDim.x + threadIdx.x; i < a.n; i += (size_t)grid.blocks() * blockDim.x) {
    const Match m = match[i];
    if (!match_accepted(m))
      continue;
    const float4 p = a.cur[i];
    const float4 q = ldg4(a.pts + m.pos);
    acc[0] += 1.0;
    acc[1] += (double)m.d2;
    const float4 n2 = ldg4(a.tgt_normals + m.pos);
    const float4 n1 = a.cur_normals[i];
    add_pair_terms<EST>(acc, p, q, float3{}, n2, n1, a.enforce_same_dir);
  }
  if (block_reduce_and_publish<kAccLls>(acc, GridSum{a.partials, a.counter, a.accum}, grid))
    peer_exchange(a);
}

template <int EST>
__global__ void __launch_bounds__(256)
k_accum(const IterArgs a, const Match* __restrict__ match)
{
  accum_pairs<EST>(a, match, HwGrid());
}

// ---- accumulation over an explicit correspondence list (stand-alone estimators) ------------------------
struct PairArgs {
  const float4* src;          // dense, original order
  const float4* tgt;          // dense, original order
  const float4* tgt_normals;  // dense, original order (LLS)
  const float4* src_normals;  // dense, original order (symmetric LLS)
  int enforce_same_dir;
  const pclb200_corr* corr;   // nullable: pair i <-> i
  size_t n;
  float ox, oy, oz;
  GridSum pub;                // the grid sum's partials / counter / totals
};

template <int EST>
__global__ void __launch_bounds__(256)
k_accum_pairs(const PairArgs a)
{
  constexpr int NACC = EST == PCLB200_EST_SVD ? kAccSvd : kAccLls;
  double acc[NACC];
#pragma unroll
  for (int t = 0; t < NACC; ++t)
    acc[t] = 0.0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < a.n; i += (size_t)gridDim.x * blockDim.x) {
    const int qi = a.corr ? a.corr[i].index_query : (int)i;
    const int mi = a.corr ? a.corr[i].index_match : (int)i;
    const float4 p = ldg4(a.src + qi), q = ldg4(a.tgt + mi);
    acc[0] += 1.0;
    if (a.corr)
      acc[1] += (double)a.corr[i].distance;
    if (EST == PCLB200_EST_SVD)
      add_pair_terms<EST>(acc, p, q, make_float3(a.ox, a.oy, a.oz), float4{}, float4{}, 0);
    // a caller's list may pair a non-finite point (the search never does): the LLS estimators skip the pair
    else if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && isfinite(q.x) && isfinite(q.y) && isfinite(q.z))
      add_pair_terms<EST>(acc, p, q, float3{}, ldg4(a.tgt_normals + mi),
                          EST == PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS ? ldg4(a.src_normals + qi) : float4{},
                          a.enforce_same_dir);
  }
  block_reduce_and_publish<NACC>(acc, a.pub);
}

// ---- solve (one thread): accumulators -> T_k ------------------------------------------------------------
__device__ double det3_dev(const double* m)
{
  return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}

// one-sided Jacobi SVD of a row-major 3x3 (stands in for Eigen::JacobiSVD inside Eigen::umeyama)
__device__ void svd3_dev(const double* Ain, double* U, double* s, double* V)
{
  double A[9];
  for (int i = 0; i < 9; ++i) {
    A[i] = Ain[i];
    V[i] = (i % 4 == 0) ? 1.0 : 0.0;
  }
  const double eps = 2.220446049250313e-16;
  for (int sweep = 0; sweep < 60; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double alpha = 0, beta = 0, gamma = 0;
        for (int i = 0; i < 3; ++i) {
          alpha += A[3 * i + p] * A[3 * i + p];
          beta += A[3 * i + q] * A[3 * i + q];
          gamma += A[3 * i + p] * A[3 * i + q];
        }
        if (gamma == 0.0 || fabs(gamma) <= eps * sqrt(alpha * beta))
          continue;
        rotated = true;
        double zeta = (beta - alpha) / (2.0 * gamma);
        double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
        for (int i = 0; i < 3; ++i) {
          double ap = A[3 * i + p], aq = A[3 * i + q];
          A[3 * i + p] = c * ap - sn * aq;
          A[3 * i + q] = sn * ap + c * aq;
          double vp = V[3 * i + p], vq = V[3 * i + q];
          V[3 * i + p] = c * vp - sn * vq;
          V[3 * i + q] = sn * vp + c * vq;
        }
      }
    if (!rotated)
      break;
  }
  double nrm[3];
  for (int j = 0; j < 3; ++j)
    nrm[j] = sqrt(A[j] * A[j] + A[3 + j] * A[3 + j] + A[6 + j] * A[6 + j]);
  int ord[3] = {0, 1, 2};
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2 - a; ++b)
      if (nrm[ord[b]] < nrm[ord[b + 1]]) {
        int t = ord[b]; ord[b] = ord[b + 1]; ord[b + 1] = t;
      }
  double Vs[9];
  for (int j = 0; j < 3; ++j) {
    s[j] = nrm[ord[j]];
    for (int i = 0; i < 3; ++i) {
      Vs[3 * i + j] = V[3 * i + ord[j]];
      U[3 * i + j] = s[j] > 0.0 ? A[3 * i + ord[j]] / s[j] : 0.0;
    }
  }
  for (int i = 0; i < 9; ++i)
    V[i] = Vs[i];
  const double tiny = s[0] * eps * 8.0;
  if (s[0] <= 0.0) {
    for (int i = 0; i < 9; ++i)
      U[i] = (i % 4 == 0) ? 1.0 : 0.0;
    return;
  }
  if (s[1] <= tiny) {
    double u0[3] = {U[0], U[3], U[6]};
    int m = 0;
    if (fabs(u0[1]) < fabs(u0[m])) m = 1;
    if (fabs(u0[2]) < fabs(u0[m])) m = 2;
    double e[3] = {0, 0, 0};
    e[m] = 1.0;
    double w[3] = {u0[1] * e[2] - u0[2] * e[1], u0[2] * e[0] - u0[0] * e[2], u0[0] * e[1] - u0[1] * e[0]};
    double wn = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    for (int i = 0; i < 3; ++i)
      U[3 * i + 1] = w[i] / wn;
  }
  if (s[2] <= tiny) {
    double a[3] = {U[0], U[3], U[6]}, b[3] = {U[1], U[4], U[7]};
    U[2] = a[1] * b[2] - a[2] * b[1];
    U[5] = a[2] * b[0] - a[0] * b[2];
    U[8] = a[0] * b[1] - a[1] * b[0];
  }
}

__device__ bool solve6_dev(double (*A)[7], double* x)
{
  for (int c = 0; c < 6; ++c) {
    int piv = c;
    for (int r = c + 1; r < 6; ++r)
      if (fabs(A[r][c]) > fabs(A[piv][c]))
        piv = r;
    if (A[piv][c] == 0.0)
      return false;
    if (piv != c)
      for (int j = 0; j < 7; ++j) {
        double t = A[piv][j]; A[piv][j] = A[c][j]; A[c][j] = t;
      }
    for (int r = c + 1; r < 6; ++r) {
      double f = A[r][c] / A[c][c];
      for (int j = c; j < 7; ++j)
        A[r][j] -= f * A[c][j];
    }
  }
  for (int r = 5; r >= 0; --r) {
    double acc = A[r][6];
    for (int j = r + 1; j < 6; ++j)
      acc -= A[r][j] * x[j];
    x[r] = acc / A[r][r];
  }
  return true;
}

// svd_correlation != 0: TransformationEstimationSVD with use_umeyama_ = false — getTransformationFromCorrelation
// (transformation_estimation_svd.hpp:183-225): H = sum (p - cp)(q - cq)^T = U S V^T, R = V U^T with the last column of V
// negated when det(U) det(V) < 0, t = cq - R cp.  The same least-squares rotation as Umeyama's, by the reference's other
// formula (the sums are the same accumulators: H is n times the transpose of Umeyama's covariance).
// C = A * B, row-major, Eigen's coefficient order, in Scalar S (final = T_k * final, icp.hpp:223)
template <typename S>
__device__ void mat4_mul_dev(const double* A, const double* B, double* C)
{
  S R[16];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c)
      R[4 * r + c] = (((S)A[4 * r] * (S)B[c] + (S)A[4 * r + 1] * (S)B[4 + c]) + (S)A[4 * r + 2] * (S)B[8 + c]) +
                     (S)A[4 * r + 3] * (S)B[12 + c];
  for (int i = 0; i < 16; ++i)
    C[i] = (double)R[i];
}

// DefaultConvergenceCriteria::hasConverged (impl/default_convergence_criteria.hpp:49-140) on the loop state L; T = T_k
template <typename S>
__device__ bool has_converged_dev(LoopCtrl& L, const CritParams& P, const double* Td)
{
  if (L.state != PCLB200_CONV_NOT_CONVERGED) {
    L.iterations_similar = 0;
    L.state = PCLB200_CONV_NOT_CONVERGED;
  }
  bool is_similar = false;
  if (L.iterations >= P.max_iterations) {
    if (!P.failure_after_max_iter) {
      L.state = PCLB200_CONV_ITERATIONS;
      return true;
    }
    L.state = PCLB200_CONV_FAILURE_AFTER_MAX_ITERATIONS;
  }
  S T[16];
  for (int i = 0; i < 16; ++i)
    T[i] = (S)Td[i];
  const double rotation_threshold = P.rot_eps > 0 ? P.rot_eps : 0.99999;
  const double cos_angle = 0.5 * (T[0] + T[5] + T[10] - 1);
  const double translation_sqr = T[3] * T[3] + T[7] * T[7] + T[11] * T[11];
  if (cos_angle >= rotation_threshold && translation_sqr <= P.trans_eps) {
    if (L.iterations_similar >= P.max_iterations_similar) {
      L.state = PCLB200_CONV_TRANSFORM;
      return true;
    }
    is_similar = true;
  }
  const double cur_mse = L.mse;
  if (fabs(cur_mse - L.prev_mse) < P.abs_mse) {
    if (L.iterations_similar >= P.max_iterations_similar) {
      L.state = PCLB200_CONV_ABS_MSE;
      return true;
    }
    is_similar = true;
  }
  if (fabs(cur_mse - L.prev_mse) / L.prev_mse < P.rel_mse) {
    if (L.iterations_similar >= P.max_iterations_similar) {
      L.state = PCLB200_CONV_REL_MSE;
      return true;
    }
    is_similar = true;
  }
  if (is_similar)
    ++L.iterations_similar;
  else
    L.iterations_similar = 0;
  L.prev_mse = cur_mse;
  return false;
}

// origin: the SVD sums' origin (3 floats in device memory; nullptr = 0)
__global__ void k_solve(const double* __restrict__ accum, int est, int scalar_is_double, int mode, const float* origin,
                        int min_corr, Pending* pending, SolveOut* out, int svd_correlation, LoopCtrl* ctrl,
                        CritParams crit)
{
  if (threadIdx.x != 0 || blockIdx.x != 0)
    return;
#include "solve_body.inc"
}

// k_solve of one problem of a batch (k_solve_batch): the same body on the problem's own accumulators and loop state
__device__ __forceinline__ void solve_one(const double* __restrict__ accum, int est, int scalar_is_double, int mode,
                                          const float* origin, int min_corr, Pending* pending, SolveOut* out,
                                          int svd_correlation, LoopCtrl* ctrl, const CritParams& crit)
{
#include "solve_body.inc"
}

// An origin of the SVD sums (slot layout at the top of this file): the first finite point of pts, or of
// pts[corr[i].index_match] over a pair list; `out` is left as it was when there is none.  One thread: the scan normally stops at the first point.
__global__ void k_seed_origin(const float4* __restrict__ pts, const pclb200_corr* __restrict__ corr, size_t n, float* out)
{
  for (size_t i = 0; i < n; ++i) {
    const float4 p = pts[corr ? (size_t)corr[i].index_match : i];
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
      out[0] = p.x;
      out[1] = p.y;
      out[2] = p.z;
      return;
    }
  }
}

// ---- a batch of problems in one loop (icp.cu: icp_iterate_batch) ------------------------------------------------------
// B problems share the target and the parameters; problem p owns the queries [begin, begin + n) of `cur` (each problem's
// queries in the order its own session stages them), and slot p of the per-problem arrays that IterArgs points to in a
// batch: pending, ctrl (its origin is the problem's SVD origin), skip_count, counter, accum (kAccum each).  Every stage is
// one launch: the grid each problem's single align would launch is laid end to end with the others', and a table tells
// each block its problem and its place in that problem's grid.  A block works for one problem only, so the per-block
// tests (done, the tracking flavour) and the shared Pending stay what they are in a single align, and the fixed-order
// grid sum runs over the problem's own partials in its own block order: the same fp64 sums, bit for bit.
struct BatchBlock {
  int problem;
  unsigned vblock, vgrid;  // this block's place in the problem's grid
  unsigned part;           // the problem's first partials slot (blocks before it, over all problems)
  unsigned long long begin, n;  // the problem's queries
};

// the block table of a grid of grid(n_p) blocks per problem p, laid end to end (off: B + 1 record offsets); each problem's
// partials slots start at its first block's place in the table
template <typename Grid>
inline std::vector<BatchBlock> batch_blocks(const std::vector<long long>& off, Grid grid)
{
  std::vector<BatchBlock> h;
  for (size_t p = 0; p + 1 < off.size(); ++p) {
    const size_t n = (size_t)(off[p + 1] - off[p]);
    const unsigned g = grid(n), part = (unsigned)h.size();
    for (unsigned v = 0; v < g; ++v)
      h.push_back(BatchBlock{(int)p, v, g, part, (unsigned long long)off[p], (unsigned long long)n});
  }
  return h;
}

// A batch of scan pairs (icp.cu: icp_set_target_batch): problem p's own target, everything its single session derives
// from its index.  The one-target batch reads the target from IterArgs instead (TARGETS = false below).
struct BatchTarget {
  const BvhNode* nodes;
  const float4* pts;
  const float4* normals;  // normals_by_pos of the problem's index (nullable: SVD)
  int root;
  CellTable cells;
  double rmax;            // CritParams::rmax of the problem's target frame
};

// a's per-problem pointers narrowed to the problem of block b
__device__ __forceinline__ IterArgs problem_args(const IterArgs& a, const BatchBlock& b)
{
  IterArgs p = a;
  p.cur = a.cur + b.begin;
  p.n = b.n;
  if (a.cur_normals)
    p.cur_normals = a.cur_normals + b.begin;
  p.pending = a.pending + b.problem;
  p.ctrl = a.ctrl + b.problem;
  p.origin = p.ctrl->origin;
  p.skip_count = a.skip_count + b.problem;
  p.partials = a.partials + (size_t)b.part * kAccum;
  p.partials2 = a.partials2 + (size_t)b.part * 128;
  p.counter = a.counter + b.problem;
  p.accum = a.accum + (size_t)b.problem * kAccum;
  return p;
}

// ... and, with TARGETS, its target read from the problem's record of the table
template <bool TARGETS>
__device__ __forceinline__ IterArgs problem_args(const IterArgs& a, const BatchBlock& b, const BatchTarget* targets)
{
  IterArgs p = problem_args(a, b);
  if (TARGETS) {
    const BatchTarget& t = targets[b.problem];
    p.nodes = t.nodes;
    p.pts = t.pts;
    p.tgt_normals = t.normals;
    p.root = t.root;
    p.cells = t.cells;
  }
  return p;
}

template <bool TRACK, bool TARGETS = false>
__global__ void __launch_bounds__(256, 5)
k_search_batch(const IterArgs a, const BatchBlock* __restrict__ blocks, Match* __restrict__ match, float* __restrict__ lbs,
               const BatchTarget* __restrict__ targets = nullptr)
{
  const BatchBlock b = blocks[blockIdx.x];
  search_queries<false, TRACK>(problem_args<TARGETS>(a, b, targets), match + b.begin, lbs + b.begin,
                               VirtualGrid{b.vblock, b.vgrid});
}

template <int EST, bool TARGETS = false>
__global__ void __launch_bounds__(256, kAccumBlocksPerSM)
k_accum_dmma_batch(const IterArgs a, const BatchBlock* __restrict__ blocks, const Match* __restrict__ match,
                   const BatchTarget* __restrict__ targets = nullptr)
{
  const BatchBlock b = blocks[blockIdx.x];
  accum_dmma_pairs<EST>(problem_args<TARGETS>(a, b, targets), match + b.begin, VirtualGrid{b.vblock, b.vgrid});
}

template <int EST, bool TARGETS = false>
__global__ void __launch_bounds__(256)
k_accum_batch(const IterArgs a, const BatchBlock* __restrict__ blocks, const Match* __restrict__ match,
              const BatchTarget* __restrict__ targets = nullptr)
{
  const BatchBlock b = blocks[blockIdx.x];
  accum_pairs<EST>(problem_args<TARGETS>(a, b, targets), match + b.begin, VirtualGrid{b.vblock, b.vgrid});
}

// one warp per problem (lane 0 solves): k_solve of each problem on its own accumulators and loop state; targets
// (nullable): each problem's rmax replaces crit's
__global__ void k_solve_batch(const double* __restrict__ accum, int n_problems, int est, int scalar_is_double, int mode,
                              Pending* pending, SolveOut* out, int svd_correlation, LoopCtrl* ctrl, CritParams crit,
                              const BatchTarget* __restrict__ targets = nullptr)
{
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  const int p = (int)(t >> 5);
  if ((t & 31) || p >= n_problems)
    return;
  if (targets)
    crit.rmax = targets[p].rmax;
  solve_one(accum + (size_t)p * kAccum, est, scalar_is_double, mode, ctrl[p].origin, 3, pending + p, out + p,
            svd_correlation, ctrl + p, crit);
}

// k_seed_origin of every problem that has not run an iteration yet, one thread per problem, into its loop state
__global__ void k_seed_origin_batch(const float4* __restrict__ cur, const long long* __restrict__ offsets, int n_problems,
                                    LoopCtrl* ctrl)
{
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_problems || ctrl[p].iterations != 0 || ctrl[p].done)
    return;
  const float4* q = cur + offsets[p];
  const size_t n = (size_t)(offsets[p + 1] - offsets[p]);
  for (size_t i = 0; i < n; ++i) {
    const float4 v = q[i];
    if (isfinite(v.x) && isfinite(v.y) && isfinite(v.z)) {
      ctrl[p].origin[0] = v.x;
      ctrl[p].origin[1] = v.y;
      ctrl[p].origin[2] = v.z;
      return;
    }
  }
}

// ---- the stages between search and accumulate (drivers: run_rejectors and the normal-based estimators in icp.cu) --------
// Match array <-> flat rejector arrays (tie-break = slot = position in the source index list = the order of the
// reference's correspondences_ vector; target identity = position in the Morton array)
__global__ void k_match_to_arrays(const float4* __restrict__ cur, const Match* __restrict__ match, size_t n,
                                  float* __restrict__ d2, int* __restrict__ mt, unsigned* __restrict__ tie, int* __restrict__ acc)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const Match m = match[i];
  d2[i] = m.d2;
  mt[i] = m.pos >= 0 ? match_pos(m) : -1;
  tie[i] = (unsigned)__float_as_int(cur[i].w);
  acc[i] = match_accepted(m) ? 1 : 0;
}

__global__ void k_arrays_to_match(const int* __restrict__ acc, size_t n, Match* __restrict__ match)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) {
    const int pos = match[i].pos;
    if (pos >= 0)
      match[i].pos = acc[i] ? (pos & kPosMask) : (pos | kNotAccepted);
  }
}

// CorrespondenceEstimationNormalShooting / ...BackProjection inside the loop: the candidate rows come from the
// exact k-NN kernel (rows addressed by slot), the choice is corr_select.cuh's; the result is a Match like the 1-NN
// search kernels produce, so the rejectors / accumulation / solve downstream are unchanged.
__global__ void __launch_bounds__(128)
k_select_match(const float4* __restrict__ cur, const float4* __restrict__ cur_normals, size_t n, int kind, int k,
               const int32_t* __restrict__ nn_idx, const float* __restrict__ nn_d2, const float4* __restrict__ tgt_pts,
               const int32_t* __restrict__ pos_of_orig, const float4* __restrict__ tgt_nrm_by_pos, double max_dist,
               Match* __restrict__ match)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const float4 p = cur[i];
  Match m;
  m.pos = -1;
  m.d2 = 0.f;
  if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
    const size_t slot = (size_t)(unsigned)__float_as_int(p.w);
    const float4 nn = cur_normals[i];
    const int32_t* row_idx = nn_idx + slot * (size_t)k;
    const float* row_d2 = nn_d2 + slot * (size_t)k;
    const int j = select_by_normals<true>(kind, k, row_idx, row_d2, p.x, p.y, p.z, nn.x, nn.y, nn.z, tgt_pts,
                                          pos_of_orig, tgt_nrm_by_pos, max_dist);
    if (j >= 0 && row_idx[j] >= 0) {
      m.pos = pos_of_orig[row_idx[j]];
      m.d2 = row_d2[j];
    }
  }
  match[i] = m;
}

// CorrespondenceRejectorSurfaceNormal inside the loop: rotated source normal vs the matched target's normal
__global__ void k_reject_surface_normal(const float4* __restrict__ cur_normals, const float4* __restrict__ tgt_nrm_by_pos,
                                        const int* __restrict__ mt, size_t n, double threshold, int* __restrict__ acc)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n || !acc[i])
    return;
  if (!surface_normal_keeps(cur_normals[i], tgt_nrm_by_pos[mt[i]], threshold))
    acc[i] = 0;
}

// ---- consumers of the same searcher outside the loop (drivers in icp.cu) ------------------------------------------------
// correspondences by slot: match = original target index or -1
template <bool RECIP>
__global__ void __launch_bounds__(128)
k_corr(const TreeView T, const float4* __restrict__ q,
       size_t nq, float gate, const BvhNode* __restrict__ s_nodes, const float4* __restrict__ s_pts, int s_root,
       const int32_t* __restrict__ src_orig, pclb200_corr* __restrict__ out, int* __restrict__ d_error)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nq)
    return;
  const float4 p = __ldg(q + i);
  const int slot = __float_as_int(p.w);
  const int my_orig = src_orig ? src_orig[slot] : slot;
  pclb200_corr r;
  r.index_query = my_orig;
  r.index_match = -1;
  r.distance = 0.f;
  if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
    Nearest1 v{p.x, p.y, p.z, gate, kSentinelIndex, -1};
    WalkStats ws{};
    if (!nearest1<false>(T, p.x, p.y, p.z, v, -1, 1.00001f, ws))
      atomicExch(d_error, kErrStackOverflow);
    if (v.best_pos >= 0) {
      bool keep = true;
      if (RECIP) {
        const float4 t = ldg4(T.pts + v.best_pos);
        Nearest1 b{t.x, t.y, t.z, gate, kSentinelIndex, -1};
        if (!traverse(s_nodes, s_pts, s_root, t.x, t.y, t.z, b))
          atomicExch(d_error, kErrStackOverflow);
        keep = b.best_pos >= 0 && b.best_idx == my_orig;
      }
      if (keep) {
        r.index_match = v.best_idx;
        r.distance = v.best;
      }
    }
  }
  out[slot] = r;
}


// fitness: sum of d2 <= max_range and count (registration.hpp:146-163)
__global__ void __launch_bounds__(256)
k_fitness(const TreeView T, const float4* __restrict__ q, size_t nq, double max_range, GridSum sum, int* d_error)
{
  double acc[2] = {0.0, 0.0};
  bool overflow = false;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nq; i += (size_t)gridDim.x * blockDim.x) {
#include "fitness_body.inc"
  }
  if (overflow)
    atomicExch(d_error, kErrStackOverflow);
  block_reduce_and_publish<2>(acc, sum);
}

// k_fitness of a batch of problems in one launch (icp.cu: fitness_batch): block b of the table (batch_blocks) runs as block
// b.vblock of the grid of b.vgrid blocks that k_fitness would be launched with over problem b.problem's queries
// q[b.begin, b.begin + b.n) alone, searching that problem's tree trees[b.problem].  Its sums go through the problem's own
// partials (from slot b.part), counter and accumulator (kAccum doubles per problem) in the problem's own block order: the
// single call's sums, bit for bit.
__global__ void __launch_bounds__(256)
k_fitness_batch(const BatchBlock* __restrict__ blocks, const TreeView* __restrict__ trees, const float4* __restrict__ q_all,
                double max_range, GridSum sum, int* d_error)
{
  const BatchBlock b = blocks[blockIdx.x];
  const TreeView T = trees[b.problem];
  const float4* __restrict__ q = q_all + b.begin;
  const size_t nq = b.n;
  double acc[2] = {0.0, 0.0};
  bool overflow = false;
  for (size_t i = b.vblock * (size_t)blockDim.x + threadIdx.x; i < nq; i += (size_t)b.vgrid * blockDim.x) {
#include "fitness_body.inc"
  }
  if (overflow)
    atomicExch(d_error, kErrStackOverflow);
  const GridSum mine{sum.partials + (size_t)b.part * kAccum, sum.counter + b.problem, sum.accum + (size_t)b.problem * kAccum};
  block_reduce_and_publish<2>(acc, mine, VirtualGrid{b.vblock, b.vgrid});
}

// GeneralizedIterativeClosestPoint::computeCovariances, one thread per point over exact k-NN rows (driver: gicp_covariances)
__global__ void __launch_bounds__(128)
k_gicp_cov(const float4* __restrict__ q, size_t n, const int32_t* __restrict__ rows, int k_rows, int k_div,
           const float4* __restrict__ pts, const int32_t* __restrict__ pos_of_orig, double gicp_epsilon,
           double* __restrict__ out)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const float4 qq = q[i];
  double o[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (isfinite(qq.x) && isfinite(qq.y) && isfinite(qq.z)) {
    double mean[3] = {0.0, 0.0, 0.0}, cov[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    const int32_t* row = rows + i * (size_t)k_rows;
    for (int j = 0; j < k_rows; ++j) {
      const int32_t oi = row[j];
      if (oi < 0)
        break;
      const float4 p = ldg4(pts + pos_of_orig[oi]);
      const double ptx = (double)__fsub_rn(p.x, qq.x), pty = (double)__fsub_rn(p.y, qq.y), ptz = (double)__fsub_rn(p.z, qq.z);
      mean[0] += ptx; mean[1] += pty; mean[2] += ptz;
      cov[0] += ptx * ptx;
      cov[3] += pty * ptx; cov[4] += pty * pty;
      cov[6] += ptz * ptx; cov[7] += ptz * pty; cov[8] += ptz * ptz;
    }
    const double kk = (double)k_div;
    for (int d = 0; d < 3; ++d)
      mean[d] /= kk;
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c <= r; ++c) {
        cov[3 * r + c] /= kk;
        cov[3 * r + c] -= mean[r] * mean[c];
        cov[3 * c + r] = cov[3 * r + c];
      }
    double U[9], sv[3], V[9];
    svd3_dev(cov, U, sv, V);
    for (int kc = 0; kc < 3; ++kc) {
      const double v = kc == 2 ? gicp_epsilon : 1.0;
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c)
          o[3 * r + c] += v * U[3 * r + kc] * U[3 * c + kc];
    }
  }
  for (int e = 0; e < 9; ++e)
    out[9 * i + e] = o[e];
}

}  // namespace pclb200
