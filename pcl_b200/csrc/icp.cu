// icp.cu — the per-iteration hot loop of pcl::IterativeClosestPoint, device resident.
//
// Reference loop: registration/include/pcl/registration/impl/icp.hpp:164-241
//   determineCorrespondences (impl/correspondence_estimation.hpp:145-218)  N_src x 1-NN + distance gate
//   estimateRigidTransformation (impl/transformation_estimation_svd.hpp:137-155 -> Umeyama,
//       common/impl/eigen.hpp:675-734; or impl/transformation_estimation_point_to_plane_lls.hpp:166-268)
//   transformCloud (impl/icp.hpp:49-111) ; final = T_k * final (:223) ; convergence (:238)
//
// One iteration here = a search kernel over the Morton-ordered source:
//   [apply the previous iteration's T_k to the point, in the reference's fp32 operation order, and
//    write it back]  ->  exact 1-NN in the LBVH with the gate as the initial bound
// then an accumulation kernel: fp64 sums of the 17 (Umeyama) or 29 (point-to-plane) terms, warp/block/grid
// reduction with a FIXED order (deterministic), last block folds the per-block partials; then (after the
// cross-GPU all-reduce, if any) a one-warp solve kernel that leaves T_k in device memory for the next
// iteration and does the loop's bookkeeping in its tail: final = T_k * final, the iteration count and
// DefaultConvergenceCriteria (default_convergence_criteria.hpp:49-140) in the caller's Scalar, on a LoopCtrl in
// device memory.  icp_iterate enqueues the iterations and synchronises once per call, or once per iteration
// when a stage between search and solve needs the host.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <limits>
#include <memory>

#include "internal.cuh"
#include "corr_select.cuh"
#include "traverse.cuh"
#include "icp_kernels.cuh"
#include "shard_target_kernels.cuh"

namespace pclb200 {

void comm_allreduce_sum(Ctx& c, double* d_buf, int count);  // comm.cu (no-op without a communicator)
bool comm_active(const Ctx& c);
bool comm_peer_view(Ctx& c, PeerView* view, unsigned long long* seq);
bool comm_peer_fused(const Ctx& c);  // the per-iteration exchange happens inside the accumulate kernel
int comm_nranks(const Ctx& c);

// ---- misc streaming kernels (transform_one and k_transform_batch: icp_kernels.cuh) ---------------------------------
__device__ __forceinline__ void transform_range(const Pending& P, float4* __restrict__ pts, size_t n,
                                                float4* __restrict__ normals /* nullable */)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    transform_one(P, pts, i, normals);
}

// the transform k_solve left for the next iteration
__global__ void k_apply_pending(float4* __restrict__ pts, size_t n, const Pending* __restrict__ pending,
                                float4* __restrict__ normals /* nullable */)
{
  const Pending P = *pending;
  if (P.apply)
    transform_range(P, pts, n, normals);
}

// a transform known to the host, passed by value so that no host buffer has to outlive the launch
__global__ void k_transform(float4* __restrict__ pts, size_t n, const Pending P, float4* __restrict__ normals)
{
  transform_range(P, pts, n, normals);
}

__global__ void k_set_pending(Pending* p, const Pending P) { *p = P; }
__global__ void k_clear_apply(Pending* p) { p->apply = 0; }

// output record i = source record i with xyz (and the normal at float nrm_word, when >= 0) transformed by P as
// k_transform does: a non-finite point keeps its whole record, a non-finite normal under kApplyIcp stays as it was.  Every
// record is read once and written once.  vec: stride is a multiple of 16 and both arrays are 16-byte aligned.
__global__ void k_assemble_records(const unsigned char* __restrict__ raw, size_t n, size_t stride, int nrm_word,
                                   const Pending P, int vec, unsigned char* __restrict__ out)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
#include "assemble_body.inc"
}

// a batch: record i moved by the final transform of its problem (the offsets of icp_set_source_batch)
__global__ void k_assemble_records_batch(const unsigned char* __restrict__ raw, size_t n, size_t stride, int nrm_word,
                                         const long long* __restrict__ offsets, int n_problems,
                                         const Pending* __restrict__ finals, int vec, unsigned char* __restrict__ out)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const Pending P = finals[problem_of(offsets, n_problems, (long long)i)];
#include "assemble_body.inc"
}

// strided write-back of a dense float4 array: xyz into out + i*stride (+ optional w = 1 when stride >= 16)
__global__ void k_scatter_xyz(const float4* __restrict__ src, size_t n, unsigned char* __restrict__ out, size_t stride,
                              int write_w, float w)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  float4 v = src[i];
  float* o = reinterpret_cast<float*>(out + i * stride);
  o[0] = v.x; o[1] = v.y; o[2] = v.z;
  if (write_w)
    o[3] = w;
}

// =============================================================================================================
// host side
// =============================================================================================================

// ---- GICP covariances -----------------------------------------------------------------------------------------------
// GeneralizedIterativeClosestPoint::computeCovariances (registration/impl/gicp.hpp:69-147): per point, the covariance
// of its k nearest neighbours relative to the point (float differences widened to double), mean removed, SVD, singular
// values replaced by (1, 1, gicp_epsilon), reassembled from the columns of U.  One thread per point over the exact k-NN
// rows of launch_knn; the 3x3 Jacobi SVD is k_solve's.
void gicp_covariances(Ctx& c, Index& idx, const void* pts, size_t n, size_t stride, int k, double gicp_epsilon,
                      double* out)
{
  cudaStream_t st = c.stream;
  if (n == 0)
    return;
  PCLB_REQUIRE(k >= 1, PCLB200_ERR_INVALID, "k must be positive");
  const int keff = (int)std::min<size_t>((size_t)k, idx.n_valid);
  DevBuf<float4> dense;
  QueryBatch qb = load_queries(c, idx, pts, n, stride, nullptr, 0, dense);
  DevBuf<int32_t> rows;
  DevBuf<float> rows_d2;
  rows.alloc(n * (size_t)keff, st);
  rows_d2.alloc(n * (size_t)keff, st);
  launch_knn(c, idx, qb.q.p, n, keff, std::numeric_limits<float>::infinity(), rows.p, rows_d2.p);
  ensure_pos_of_orig(c, idx);
  DevBuf<double> tmp;
  double* d_o = out_on_device(c, out, n * 9, tmp);
  k_gicp_cov<<<grid_for(n, 128), 128, 0, st>>>(dense.p, n, rows.p, keff, k, idx.pts.p, idx.pos_of_orig.p, gicp_epsilon, d_o);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  copy_out(c, out, tmp, n * 9);
  check_device_error(c);
}

#ifdef PCLB_STATS
extern "C" __attribute__((visibility("default"))) int pclb200_debug_walk_stats(unsigned long long out[8], int reset)
{
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(out, g_walk_stats, 8 * sizeof(unsigned long long));
  if (reset) {
    unsigned long long z[8] = {0};
    cudaMemcpyToSymbol(g_walk_stats, z, sizeof(z));
  }
  return 0;
}
extern "C" __attribute__((visibility("default"))) int pclb200_debug_walk_hist(unsigned long long out[66], int reset)
{
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(out, g_walk_imbalance, 2 * sizeof(unsigned long long));
  cudaMemcpyFromSymbol(out + 2, g_walk_hist, 64 * sizeof(unsigned long long));
  if (reset) {
    unsigned long long z[64] = {0};
    cudaMemcpyToSymbol(g_walk_imbalance, z, 2 * sizeof(unsigned long long));
    cudaMemcpyToSymbol(g_walk_hist, z, sizeof(z));
  }
  return 0;
}
#endif

float gate_from_max_dist(double max_dist)
{
  // d2 (float) is kept iff (double)d2 <= max_dist^2  <=>  d2 <= largest float <= max_dist^2
  const double m2 = max_dist * max_dist;
  if (!(m2 < (double)FLT_MAX))
    return FLT_MAX;
  float g = (float)m2;
  if ((double)g > m2)
    g = std::nextafter(g, -INFINITY);
  return g;
}

struct Reducer {  // scratch of the grid sums (grid_fold)
  DevBuf<double> partials;
  DevBuf<double> partials2;  // max_blocks * 128 (k_accum_dmma)
  DevBuf<unsigned> counter;
  DevBuf<double> accum;
  unsigned max_blocks = 0;
  void init(Ctx& c, unsigned blocks)
  {
    max_blocks = blocks;
    partials.alloc((size_t)blocks * kAccum, c.stream);
    partials2.alloc((size_t)blocks * 128, c.stream);
    counter.alloc(1, c.stream);
    accum.alloc(kAccum, c.stream);
    PCLB_CUDA(cudaMemsetAsync(counter.p, 0, sizeof(unsigned), c.stream));
    PCLB_CUDA(cudaMemsetAsync(accum.p, 0, kAccum * sizeof(double), c.stream));
  }
  GridSum sum() const { return GridSum{partials.p, counter.p, accum.p}; }
};

// pinned host memory of one session (the batch read-back), freed with it
struct PinnedBuf {
  void* p = nullptr;
  size_t bytes = 0;
  PinnedBuf() = default;
  PinnedBuf(const PinnedBuf&) = delete;
  PinnedBuf& operator=(const PinnedBuf&) = delete;
  PinnedBuf(PinnedBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
  PinnedBuf& operator=(PinnedBuf&& o) noexcept
  {
    if (this != &o) {
      release();
      p = o.p; bytes = o.bytes;
      o.p = nullptr; o.bytes = 0;
    }
    return *this;
  }
  ~PinnedBuf() { release(); }
  void reserve(size_t b)
  {
    if (b <= bytes)
      return;
    release();
    PCLB_CUDA(cudaMallocHost(&p, b));
    bytes = b;
  }
  void release()
  {
    if (p)
      cudaFreeHost(p);
    p = nullptr;
    bytes = 0;
  }
};

// the state of a batch session (icp_set_source_batch): B > 0 problems over consecutive record ranges of the source, the
// per-problem slots the batch kernels index (icp_kernels.cuh: BatchBlock) and the block tables of the three grids
struct IcpBatch {
  int B = 0;                         // 0: a single-problem session
  std::vector<long long> offsets;    // B + 1
  DevBuf<long long> d_offsets;
  DevBuf<int32_t> rel;               // record -> its index within its problem (index_query of the lists)
  DevBuf<BatchBlock> wtab, atab, gtab;  // the search's grids, k_accum_dmma's, k_accum's
  unsigned a_blocks = 0, g_blocks = 0;  // partials slots of atab / gtab
  DevBuf<Pending> pending;
  DevBuf<LoopCtrl> ctrl;
  DevBuf<SolveOut> solve_out;
  DevBuf<unsigned long long> skip_count;
  DevBuf<unsigned> counter;
  DevBuf<double> partials, accum;
  std::vector<LoopCtrl> loop;
  std::vector<int64_t> total_skipped;
  PinnedBuf host;                    // B loop states, B skip counts, the device error flag
};

// a batch of scan pairs (icp_set_target_batch): problem p of the next batch source is registered against idx[p]
struct IcpTargets {
  int B = 0;                            // 0: the session's one target (Icp::tgt)
  std::vector<const Index*> idx;        // problem -> its index (kept alive by the caller)
  bool all_normals = false;             // every problem's target normals were given
  std::vector<DevBuf<float4>> normals;  // normals_by_pos of each distinct (index, normals) pair
  DevBuf<BatchTarget> table;            // problem -> its target (icp_kernels.cuh)
  DevBuf<float4> frames;                // problem -> {lo, morton_scale} of its index: the frame of its query order
};

struct Icp {
  Ctx* ctx = nullptr;
  pclb200_icp_params P;
  const Index* tgt = nullptr;
  DevBuf<float4> tgt_normals;   // Morton order of tgt
  // source
  size_t n_all = 0;             // records in the caller's source cloud
  size_t n_q = 0;               // indexed source points (queries)
  DevBuf<float4> src_all;       // original order, all records (for the output cloud)
  DevBuf<float4> src_normals;   // original order (optional)
  DevBuf<int32_t> src_orig;     // slot -> original source index (when indices were given)
  DevBuf<float4> cur;           // Morton order, w = slot
  DevBuf<float4> cur_normals;   // source normals in the order of `cur` (symmetric objective only)
  DevBuf<Match> match;          // Morton order: this iteration's matches = next iteration's seeds
  DevBuf<LoopCtrl> ctrl;        // device copy of `loop` for one icp_iterate call: k_solve advances it every iteration
  DevBuf<float> lb;             // per query: lower bound on the distance to every OTHER target point (TRACK searches)
  DevBuf<int32_t> cur_label;    // Morton order: original source index of cur[i] (labels of the reciprocal tree)
  bool have_src_normals = false;
  DevBuf<unsigned char> src_raw; // the caller's records verbatim (kept when stride != 16) for output = *input_
  size_t src_stride = 0;
  ptrdiff_t src_normal_off = -1; // byte offset of nx inside a record, when the normals live in the same records
  // device state
  DevBuf<Pending> pending;
  DevBuf<SolveOut> solve_out;
  DevBuf<unsigned long long> skip_count;
  int64_t total_skipped = 0;
  std::vector<pclb200_rejector> rejectors;  // applied in order after every search (icp.hpp:187-201)
  // sharded source: global position of this rank's slot 0 (offset_r, DESIGN.md §5), valid for communicator shard_comm
  unsigned long long shard_offset = 0, shard_comm = 0;
  std::shared_ptr<PeerTableEntry> o2o;  // one-to-one rejector table of a sharded session
  // sharded target (icp_set_target_sharded): `tgt` is this rank's tile, `frame` the union of all tiles' boxes (lo, hi,
  // morton_scale: the frame of one index over the whole map).  Per iteration the tile's matches are published in
  // `shard_tab` (keys, then point records, then normal records; mapped into every rank) and the winners gathered into
  // gmatch / gpts / gnrm, which the accumulate kernels read instead of the tile.
  bool sharded_target = false;
  Index frame;
  bool shard_checked = false;  // the first iterate after set_source checked that every rank staged n_q queries
  std::shared_ptr<PeerTableEntry> shard_tab;
  DevBuf<Match> gmatch;
  DevBuf<float4> gpts, gnrm;
  Reducer red;
  // the loop state between icp_iterate calls (Scalar-typed values are kept in double; float mode rounds after every
  // operation): counters, DefaultConvergenceCriteria state, final / last transform, tracking decision
  LoopCtrl loop;
  IcpBatch batch;
  IcpTargets targets;
};

static void set_identity(double* T)
{
  for (int i = 0; i < 16; ++i)
    T[i] = (i % 5 == 0) ? 1.0 : 0.0;
}

static int transform_mode(const pclb200_icp_params& P)
{
  if (!P.with_normals_transform)
    return kApplyIcp;
  return P.scalar_is_double ? kApplyTransformsDouble : kApplyTransformsFloat;
}

// rows 0..2 of the row-major 4x4 T, applied in the operation order `mode` (kApply*)
static Pending make_pending(const double* T, int mode, int apply)
{
  Pending h;
  for (int i = 0; i < 12; ++i) {
    h.f[i] = (float)T[i];
    h.d[i] = T[i];
  }
  h.apply = apply;
  h.mode = mode;
  return h;
}

// the session's Pending slot set to h, in stream order (h travels as a kernel argument: nothing waits for the copy)
static void set_pending(Ctx& c, Pending* d, const Pending& h)
{
  k_set_pending<<<1, 1, 0, c.stream>>>(d, h);
  ++c.launches;
}

// pts[0..n) (and their normals, when given) transformed in place by T in the operation order `mode`
static void transform_on_device(Ctx& c, const double* T, int mode, float4* pts, size_t n, float4* normals)
{
  if (n == 0)
    return;
  k_transform<<<persistent_blocks(c, n), 256, 0, c.stream>>>(pts, n, make_pending(T, mode, 1), normals);
  ++c.launches;
}

// Everything an align() starts afresh (icp.hpp:120-136).  The previous MSE is DefaultConvergenceCriteria's member, and
// that object lives as long as the IterativeClosestPoint (icp.h:155): it starts at DBL_MAX when the session is created
// (default_convergence_criteria.h:283) and is written only by the criteria (…criteria.hpp:137), so the first iteration
// of the next align is compared with the last MSE the previous one recorded.
void icp_reset_state(Icp& s, const double* guess)
{
  LoopCtrl& L = s.loop;
  const double prev_mse = L.prev_mse;
  memset(&L, 0, sizeof(L));
  L.state = PCLB200_CONV_NOT_CONVERGED;
  L.prev_mse = prev_mse;
  set_identity(L.last_T);
  if (guess) {
    for (int i = 0; i < 16; ++i)
      L.final_T[i] = s.P.scalar_is_double ? guess[i] : (double)(float)guess[i];
  }
  else
    set_identity(L.final_T);
  s.total_skipped = 0;
  PCLB_CUDA(cudaMemsetAsync(s.skip_count.p, 0, sizeof(unsigned long long), s.ctx->stream));
}

Icp* icp_create(Ctx& c, const pclb200_icp_params& P)
{
  std::unique_ptr<Icp> s(new Icp());
  s->ctx = &c;
  s->P = P;
  s->pending.alloc(1, c.stream);
  s->solve_out.alloc(1, c.stream);
  s->ctrl.alloc(1, c.stream);
  s->skip_count.alloc(1, c.stream);
  s->red.init(c, (unsigned)c.sm_count * 16);
  s->loop.prev_mse = std::numeric_limits<double>::max();
  icp_reset_state(*s, nullptr);
  set_pending(c, s->pending.p, make_pending(s->loop.final_T, transform_mode(P), 0));
  return s.release();
}

void icp_destroy(Icp* s) { delete s; }

void icp_set_params(Icp& s, const pclb200_icp_params& P) { s.P = P; }

void icp_set_rejectors(Icp& s, const pclb200_rejector* list, int n)
{
  s.rejectors.assign(list, list + (n > 0 ? n : 0));
  for (const auto& r : s.rejectors)
    PCLB_REQUIRE(r.kind >= PCLB200_REJ_DISTANCE && r.kind <= PCLB200_REJ_SURFACE_NORMAL, PCLB200_ERR_INVALID,
                 "unknown rejector kind");
}

static bool has_surface_normal_rejector(const Icp& s)
{
  for (const auto& r : s.rejectors)
    if (r.kind == PCLB200_REJ_SURFACE_NORMAL)
      return true;
  return false;
}

// the session keeps a rotated copy of the source normals only for the components that read them every iteration
static bool needs_cur_normals(const Icp& s)
{
  return s.P.estimator == PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS || s.P.correspondence_kind != PCLB200_CORR_NEAREST ||
         has_surface_normal_rejector(s);
}

static bool rejector_is_global(const pclb200_rejector& r)
{
  return r.kind == PCLB200_REJ_MEDIAN || r.kind == PCLB200_REJ_TRIMMED || r.kind == PCLB200_REJ_ONE_TO_ONE;
}

// Sharded source: once per session and communicator, before the first iteration that needs it (set_source is not a
// collective call, so it cannot be done there): offset_r by one exchange of n_q, and the one-to-one tables.
static void prepare_sharded_rejectors(Icp& s)
{
  Ctx& c = *s.ctx;
  bool global = false, o2o = false;
  for (const auto& r : s.rejectors) {
    global = global || rejector_is_global(r);
    o2o = o2o || r.kind == PCLB200_REJ_ONE_TO_ONE;
  }
  if (!global)
    return;
  if (s.shard_comm != comm_id(c)) {
    unsigned long long total = 0;
    s.shard_offset = comm_shard_offset(c, s.n_q, &total);
    s.shard_comm = comm_id(c);
    PCLB_REQUIRE(total <= 0xffffffffull, PCLB200_ERR_INVALID,
                 "icp: the rejector chain on a sharded source needs fewer than 2^32 queries over all ranks");
  }
  if (o2o) {
    PCLB_REQUIRE(!s.tgt->labelled, PCLB200_ERR_INVALID,
                 "icp: the one-to-one rejector on a sharded source keeps a table per target record, which an index built "
                 "with caller ids does not define");
    comm_peer_tables(c, s.o2o, s.tgt->n_cloud);
  }
}

static void run_rejectors(Icp& s)
{
  Ctx& c = *s.ctx;
  cudaStream_t st = c.stream;
  const size_t n = s.n_q;
  const bool sharded = comm_active(c);
  ShardedRejectArgs sa;
  sa.tgt_pts = s.tgt->pts.p;
  sa.n_cloud = s.tgt->n_cloud;
  sa.offset = s.shard_offset;
  sa.o2o = &s.o2o;
  DevBuf<float> d2;
  DevBuf<int> mt, acc;
  DevBuf<unsigned> tie;
  d2.alloc(n, st);
  mt.alloc(n, st);
  acc.alloc(n, st);
  tie.alloc(n, st);
  if (n) {
    k_match_to_arrays<<<grid_for(n, 256), 256, 0, st>>>(s.cur.p, s.match.p, n, d2.p, mt.p, tie.p, acc.p);
    ++c.launches;
  }
  RejectArrays a;
  a.n = n;
  a.d2 = d2.p;
  a.match = mt.p;
  a.tie = tie.p;
  a.acc = acc.p;
  for (const auto& r : s.rejectors) {
    if (r.kind == PCLB200_REJ_SURFACE_NORMAL) {
      PCLB_REQUIRE(s.cur_normals.p && s.tgt_normals.p, PCLB200_ERR_INVALID,
                   "icp: the surface-normal rejector needs source and target normals (set the rejectors before the source)");
      if (n) {
        k_reject_surface_normal<<<grid_for(n, 256), 256, 0, st>>>(s.cur_normals.p, s.tgt_normals.p, mt.p, n, r.p, acc.p);
        ++c.launches;
      }
      continue;
    }
    // a rank takes part in every exchange of the chain even with no correspondence at all
    if (sharded && rejector_is_global(r))
      apply_rejector_sharded(c, r, a, sa);
    else
      apply_rejector(c, r, a, nullptr, nullptr, nullptr, nullptr);
  }
  if (n) {
    k_arrays_to_match<<<grid_for(n, 256), 256, 0, st>>>(acc.p, n, s.match.p);
    ++c.launches;
  }
  PCLB_CUDA(cudaGetLastError());
}

// the normal of position j with the plane_offset of the point there in w (icp_kernels.cuh); padding keeps a NaN normal
__device__ __forceinline__ float4 normal_record(const float4* __restrict__ nrm, int rec, const float4& q)
{
  const float qn = __int_as_float(0x7fc00000);
  if (rec < 0)
    return make_float4(qn, qn, qn, 0.f);
  float4 n = nrm[rec];
  n.w = plane_offset(n, q);
  return n;
}

__global__ void k_permute_normals(const float4* __restrict__ nrm_orig, const float4* __restrict__ pts, size_t n_padded,
                                  float4* __restrict__ out)
{
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n_padded)
    return;
  const float4 q = pts[j];
  const int oi = __float_as_int(q.w);
  out[j] = normal_record(nrm_orig, oi == kSentinelIndex ? -1 : oi, q);
}

// a labelled index (build_index_ids): its w lanes are ids, so the record of position j is slot_of_pos[j]
__global__ void k_permute_normals_by_slot(const float4* __restrict__ nrm_rec, const int32_t* __restrict__ slot_of_pos,
                                          const float4* __restrict__ pts, size_t n_padded, float4* __restrict__ out)
{
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n_padded)
    return;
  out[j] = normal_record(nrm_rec, slot_of_pos[j], pts[j]);
}

// the normals (one per record of the cloud idx was built from) in the Morton order of idx, as the LLS accumulation reads
// them: {nx, ny, nz, plane_offset}.  The other readers (normal-based correspondences, the surface-normal rejector, the
// symmetric objective, the record rows of correspondences_sharded) read xyz only.
static void normals_by_pos(Ctx& c, const Index* idx, const void* normals, size_t stride_n, DevBuf<float4>& out)
{
  DevBuf<float4> dense;
  dense.alloc(idx->n_cloud, c.stream);
  load_vec3_as_float4(c, normals, idx->n_cloud, stride_n, dense.p, c.stream);
  out.alloc(idx->pts.n, c.stream);
  if (idx->labelled)
    k_permute_normals_by_slot<<<grid_for(idx->pts.n, 256), 256, 0, c.stream>>>(dense.p, idx->slot_of_pos.p, idx->pts.p,
                                                                              idx->pts.n, out.p);
  else
    k_permute_normals<<<grid_for(idx->pts.n, 256), 256, 0, c.stream>>>(dense.p, idx->pts.p, idx->pts.n, out.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

static void stage_target_normals(Icp& s, const Index* idx, const void* tgt_normals, size_t stride_n)
{
  s.tgt_normals.release();
  if (tgt_normals)
    normals_by_pos(*s.ctx, idx, tgt_normals, stride_n, s.tgt_normals);
}

static void drop_source(Icp& s);

void icp_set_target(Icp& s, const Index* idx, const void* tgt_normals, size_t stride_n)
{
  if (s.targets.B) {  // a source staged for a batch of targets is ordered in their frames, not in this one's
    drop_source(s);
    s.targets = IcpTargets();
  }
  s.tgt = idx;
  s.sharded_target = false;
  stage_target_normals(s, idx, tgt_normals, stride_n);
}

// float <-> u64 whose unsigned order is the float order (-0 < +0), so that a u64 minimum is a float minimum
static unsigned long long ordered_bits(float f)
{
  uint32_t u;
  memcpy(&u, &f, 4);
  return (u & 0x80000000u) ? (~u & 0xffffffffu) : (u | 0x80000000u);
}
static float from_ordered_bits(unsigned long long k)
{
  uint32_t u = (uint32_t)k;
  u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

// Collective: one u64 minimum over the six box floats of every rank's tile (the maxima as 2^32 - 1 - key) -> the union
// box, exact, and the frame one index over the whole map would have (lbvh.cu: morton_sort, the same arithmetic).
static void union_frame(Ctx& c, const Index& tile, Index& frame)
{
  cudaStream_t st = c.stream;
  unsigned long long h[6];
  for (int r = 0; r < 3; ++r) {
    h[r] = ordered_bits(tile.lo[r]);
    h[3 + r] = 0xffffffffull - ordered_bits(tile.hi[r]);
  }
  DevBuf<unsigned long long> d;
  d.alloc(6, st);
  PCLB_CUDA(cudaMemcpyAsync(d.p, h, sizeof(h), cudaMemcpyHostToDevice, st));
  comm_allreduce_u64(c, d.p, d.p, 6, kU64Min);
  PCLB_CUDA(cudaMemcpyAsync(h, d.p, sizeof(h), cudaMemcpyDeviceToHost, st));
  check_device_error(c);
  float ext = 0.f;
  for (int r = 0; r < 3; ++r) {
    frame.lo[r] = from_ordered_bits(h[r]);
    frame.hi[r] = from_ordered_bits(0xffffffffull - h[3 + r]);
    ext = std::max(ext, frame.hi[r] - frame.lo[r]);
  }
  frame.morton_scale = ext > 0.f ? 2097152.f / ext : 1.f;
  if (!std::isfinite(frame.morton_scale))
    frame.morton_scale = 1.f;
}

// Collective: one u64 minimum over (n, ~n, verdict) gives the smallest and the largest n of all ranks and whether every
// rank accepted its own arguments (fault: this rank's reason to refuse, or null), so that a refusal happens on every rank
// and no rank is left waiting in an exchange the others never enter
static void require_same_count(Ctx& c, unsigned long long n, const char* msg, const char* fault = nullptr)
{
  cudaStream_t st = c.stream;
  unsigned long long h[3] = {n, ~n, fault ? 0ull : 1ull};
  DevBuf<unsigned long long> d;
  d.alloc(3, st);
  PCLB_CUDA(cudaMemcpyAsync(d.p, h, sizeof(h), cudaMemcpyHostToDevice, st));
  comm_allreduce_u64(c, d.p, d.p, 3, kU64Min);
  PCLB_CUDA(cudaMemcpyAsync(h, d.p, sizeof(h), cudaMemcpyDeviceToHost, st));
  check_device_error(c);
  PCLB_REQUIRE(!fault, PCLB200_ERR_INVALID, fault);
  PCLB_REQUIRE(h[2], PCLB200_ERR_INVALID, "another rank refused its arguments");
  PCLB_REQUIRE(h[0] == ~h[1], PCLB200_ERR_INVALID, msg);
}

void icp_set_target_sharded(Icp& s, const Index* tile, const void* tgt_normals, size_t stride_n)
{
  Ctx& c = *s.ctx;
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID,
               "icp: a sharded target needs an active communicator (pclb200_comm_init or pclb200_comm_export / _import)");
  PCLB_REQUIRE(tile->labelled, PCLB200_ERR_INVALID,
               "icp: every rank's tile of a sharded target must be built with pclb200_index_build_ids");
  union_frame(c, *tile, s.frame);
  s.tgt = tile;
  s.sharded_target = true;
  s.shard_comm = 0;
  stage_target_normals(s, tile, tgt_normals, stride_n);
}

// frame of the query order and of the loop's box-derived values: the whole map's
static const Index& target_frame(const Icp& s) { return s.sharded_target ? s.frame : *s.tgt; }

// The refusals of a sharded-target session (the same on every rank, before any exchange) and, once per source, the check
// that every rank staged the same number of queries.
static void check_sharded_target(Icp& s)
{
  Ctx& c = *s.ctx;
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID, "icp: a sharded target needs an active communicator");
  PCLB_REQUIRE(!s.P.use_reciprocal, PCLB200_ERR_INVALID,
               "icp: reciprocal correspondences are not available with a sharded target (the reverse search needs the "
               "whole map's answer for every target point)");
  PCLB_REQUIRE(s.P.correspondence_kind == PCLB200_CORR_NEAREST, PCLB200_ERR_INVALID,
               "icp: the normal-shooting and back-projection estimators are not available with a sharded target");
  PCLB_REQUIRE(s.rejectors.empty(), PCLB200_ERR_INVALID,
               "icp: rejector chains are not available with a sharded target");
  if (!s.shard_checked) {
    require_same_count(c, s.n_q, "icp: with a sharded target every rank must pass the same whole source to set_source");
    PCLB_REQUIRE(s.n_q <= (size_t)kPosMask, PCLB200_ERR_INVALID, "icp: a sharded target takes fewer than 2^30 queries");
    s.shard_checked = true;
  }
}

// words of the tables of exchange_shard_records: the keys, rounded up so that the records are 16-byte aligned, then the
// point records and the normal records
static size_t shard_record_words(size_t n, bool with_normals)
{
  return ((n + 1) & ~(size_t)1) + 2 * n * (with_normals ? 2 : 1);
}

// The tile's matches match[0..n) (by query) -> the whole map's, on every rank (shard_target_kernels.cuh): gmatch, and the
// winners' records in gpts / gnrm.  t has shard_record_words(n, tile_nrm != null) words.  Peer path: publish, barrier,
// gather from every rank's arrays, barrier (no rank overwrites its arrays while a peer may still read them).  NCCL path:
// publish, min of the keys, non-winners' records zeroed, max of the records' bit patterns, gather.  ctrl (nullable): a
// finished loop turns the kernels into no-ops.  The ICP session's loop and correspondences_sharded share it.
static void exchange_shard_records(Ctx& c, const PeerTables& t, const Match* match, size_t n, const float4* tile_pts,
                                   const float4* tile_nrm, const LoopCtrl* ctrl, Match* gmatch, float4* gpts,
                                   float4* gnrm)
{
  cudaStream_t st = c.stream;
  const bool with_normals = tile_nrm != nullptr;
  const size_t kw = (n + 1) & ~(size_t)1;
  const size_t words = shard_record_words(n, with_normals);
  auto records = [&](unsigned long long* base) {
    ShardRecords r;
    r.key = base;
    r.pts = reinterpret_cast<float4*>(r.key + kw);
    r.nrm = with_normals ? r.pts + n : nullptr;
    return r;
  };
  const ShardRecords mine = records(t.local);
  ShardReadSet rs;
  memset(&rs, 0, sizeof(rs));
  rs.n = t.n_read;
  for (int r = 0; r < t.n_read; ++r) {
    rs.key[r] = t.read[r];
    rs.pts[r] = reinterpret_cast<const float4*>(t.read[r] + kw);
    rs.nrm[r] = with_normals ? rs.pts[r] + n : nullptr;
  }
  if (n) {
    k_shard_publish<<<grid_for(n, 256), 256, 0, st>>>(match, n, tile_pts, tile_nrm, ctrl, mine);
    ++c.launches;
  }
  if (t.peer)
    comm_barrier(c);
  else {
    const ShardRecords all = records(t.recv);
    comm_allreduce_u64(c, mine.key, all.key, n, kU64Min);
    if (n) {
      k_shard_keep_winners<<<grid_for(n, 256), 256, 0, st>>>(all.key, n, ctrl, mine);
      ++c.launches;
    }
    comm_allreduce_u32_max(c, reinterpret_cast<const unsigned*>(mine.pts), reinterpret_cast<unsigned*>(all.pts),
                           (words - kw) * 2);
  }
  if (n) {
    k_shard_gather<<<grid_for(n, 256), 256, 0, st>>>(rs, n, ctrl, gmatch, gpts, with_normals ? gnrm : nullptr);
    ++c.launches;
  }
  comm_tables_release(c, t);
  PCLB_CUDA(cudaGetLastError());
}

// The session's matches of this iteration -> the whole map's, through its own table (shard_tab)
static void exchange_shard_matches(Icp& s, bool with_normals)
{
  Ctx& c = *s.ctx;
  const PeerTables t = comm_peer_tables(c, s.shard_tab, shard_record_words(s.n_q, with_normals));
  exchange_shard_records(c, t, s.match.p, s.n_q, s.tgt->pts.p, with_normals ? s.tgt_normals.p : nullptr, s.ctrl.p,
                         s.gmatch.p, s.gpts.p, s.gnrm.p);
}

__global__ void k_cur_labels(const float4* __restrict__ cur, const int32_t* __restrict__ src_orig, size_t n,
                             int32_t* __restrict__ label)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const int slot = __float_as_int(cur[i].w);
  label[i] = src_orig ? src_orig[slot] : slot;
}

__global__ void k_gather_cur_normals(const float4* __restrict__ cur, const float4* __restrict__ nrm_all,
                                     const int32_t* __restrict__ src_orig, size_t n, float4* __restrict__ out)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const int slot = __float_as_int(cur[i].w);
  out[i] = nrm_all[src_orig ? src_orig[slot] : slot];
}

__global__ void k_gather_subset(const float4* __restrict__ all, const int32_t* __restrict__ sub, size_t n,
                                float4* __restrict__ out)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n)
    out[i] = all[sub[i]];
}

// The caller's records into the session (src_all, src_raw) and their queries into qb, in the order of the target frame.
static void stage_source(Icp& s, const void* src, size_t n, size_t stride, const void* src_normals, size_t stride_n,
                         const int32_t* indices, size_t n_idx, QueryBatch* qb)
{
  Ctx& c = *s.ctx;
  cudaStream_t st = c.stream;
  s.n_all = n;
  s.shard_comm = 0;
  s.shard_checked = false;
  s.src_all.alloc(n, st);
  s.src_stride = stride;
  s.src_raw.release();
  s.src_normal_off = -1;
  if (src_normals) {
    const ptrdiff_t off = static_cast<const unsigned char*>(src_normals) - static_cast<const unsigned char*>(src);
    if (stride_n == stride && off > 0 && off % 4 == 0 && (size_t)off + 12 <= stride)
      s.src_normal_off = off;
  }
  // The records are read once, from device memory: host records take one contiguous H2D into the session's own copy
  // (src_raw, or src_all when they already are PointXYZ float4s), device records are copied by the staging pass itself.
  // Every field other than xyz / normals is carried through to the output.
  const unsigned char* recs = static_cast<const unsigned char*>(src);
  unsigned char* copy = nullptr;
  float4* dense = s.src_all.p;
  const bool host_src = !is_device_ptr(src);
  if (stride != 16) {
    s.src_raw.alloc(n * stride, st);
    if (host_src) {
      PCLB_CUDA(cudaMemcpyAsync(s.src_raw.p, src, n * stride, cudaMemcpyHostToDevice, st));
      recs = s.src_raw.p;
    }
    else
      copy = s.src_raw.p;
  }
  else if (host_src) {
    PCLB_CUDA(cudaMemcpyAsync(s.src_all.p, src, n * 16, cudaMemcpyHostToDevice, st));
    recs = reinterpret_cast<const unsigned char*>(s.src_all.p);
    dense = nullptr;
  }
  s.n_q = indices ? n_idx : n;
  s.src_orig.release();
  {
    ProfScope ps(c, "query_sort");
    stage_records(c, target_frame(s), recs, n, stride, copy, dense, indices ? nullptr : qb);
    if (indices) {
      // index subset: the queries are gathered from the staged points and sorted on their own
      s.src_orig.alloc(n_idx, st);
      PCLB_CUDA(cudaMemcpyAsync(s.src_orig.p, indices, n_idx * sizeof(int32_t), cudaMemcpyDefault, st));
      DevBuf<float4> sub;
      sub.alloc(n_idx, st);
      if (n_idx) {
        k_gather_subset<<<grid_for(n_idx, 256), 256, 0, st>>>(s.src_all.p, s.src_orig.p, n_idx, sub.p);
        ++c.launches;
      }
      make_query_batch(c, target_frame(s), sub.p, s.n_q, *qb);
    }
  }
}

// The staged queries qb become the session's `cur`, with their normals and the per-query arrays of the loop
static void finish_source(Icp& s, QueryBatch& qb, const void* src_normals, size_t stride_n)
{
  Ctx& c = *s.ctx;
  cudaStream_t st = c.stream;
  const size_t n = s.n_all, stride = s.src_stride;
  s.cur = std::move(qb.q);
  // Nothing in the loop reads the source normals except through cur_normals; the output reads normals that live in the
  // records from src_raw.  So a dense copy is staged only for cur_normals or for normals kept outside the records.
  s.have_src_normals = src_normals != nullptr;
  s.src_normals.release();
  const bool normals_in_raw = s.src_normal_off >= 0 && s.src_raw.p;
  if (src_normals && (needs_cur_normals(s) || !normals_in_raw)) {
    s.src_normals.alloc(n, st);
    if (normals_in_raw)
      load_vec3_as_float4(c, s.src_raw.p + s.src_normal_off, n, stride, s.src_normals.p, st);
    else
      load_vec3_as_float4(c, src_normals, n, stride_n, s.src_normals.p, st);
  }
  s.cur_normals.release();
  if (needs_cur_normals(s)) {
    PCLB_REQUIRE(s.have_src_normals, PCLB200_ERR_INVALID,
                 "icp: the symmetric objective, the normal-based correspondence estimators and the surface-normal "
                 "rejector need source normals");
    s.cur_normals.alloc(s.n_q, st);
    if (s.n_q) {
      k_gather_cur_normals<<<grid_for(s.n_q, 256), 256, 0, st>>>(s.cur.p, s.src_normals.p, s.src_orig.p, s.n_q,
                                                                 s.cur_normals.p);
      ++c.launches;
    }
  }
  s.match.alloc(s.n_q, st);
  PCLB_CUDA(cudaMemsetAsync(s.match.p, 0xff, s.n_q * sizeof(Match), st));  // pos = -1: no seed yet
  s.lb.alloc(s.n_q, st);
  s.cur_label.alloc(s.n_q, st);
  if (s.n_q) {
    k_cur_labels<<<grid_for(s.n_q, 256), 256, 0, st>>>(s.cur.p, s.src_orig.p, s.n_q, s.cur_label.p);
    ++c.launches;
  }
}

static bool is_identity(const double* T)
{
  for (int i = 0; i < 16; ++i)
    if (T[i] != ((i % 5 == 0) ? 1.0 : 0.0))
      return false;
  return true;
}

void icp_set_source(Icp& s, const void* src, size_t n, size_t stride, const void* src_normals, size_t stride_n,
                    const int32_t* indices, size_t n_idx, const double* guess)
{
  Ctx& c = *s.ctx;
  PCLB_REQUIRE(s.tgt != nullptr, PCLB200_ERR_INVALID, "icp: no target set (registration.hpp:77-81)");
  PCLB_REQUIRE(src != nullptr && n > 0, PCLB200_ERR_INVALID, "icp: empty source");
  PCLB_REQUIRE(stride >= 12 && stride % 4 == 0, PCLB200_ERR_INVALID, "stride must be a multiple of 4 and >= 12");
  PCLB_REQUIRE(!s.targets.B, PCLB200_ERR_INVALID,
               "icp: a session holding a batch of targets takes a batch source (set_source_batch); set_target returns it "
               "to one target");
  s.batch = IcpBatch();
  QueryBatch qb;
  stage_source(s, src, n, stride, src_normals, stride_n, indices, n_idx, &qb);
  finish_source(s, qb, src_normals, stride_n);
  icp_reset_state(s, guess);
  // icp.hpp:125-134: a non-identity guess is applied once, before the first search
  if (!is_identity(s.loop.final_T))
    transform_on_device(c, s.loop.final_T, transform_mode(s.P), s.cur.p, s.n_q, s.cur_normals.p);
  set_pending(c, s.pending.p, make_pending(s.loop.last_T, transform_mode(s.P), 0));
  PCLB_CUDA(cudaGetLastError());
}

static void fill_stats(const LoopCtrl& L, int64_t total_skipped, pclb200_icp_stats* st)
{
  if (!st)
    return;
  st->converged = L.converged ? 1 : 0;
  st->state = L.state;
  st->iterations = L.iterations;
  st->reserved = 0;
  st->n_correspondences = (int64_t)L.n_corr;
  st->total_correspondences = L.total_corr;
  st->total_skipped_walks = total_skipped;
  st->mse = L.mse;
  for (int i = 0; i < 16; ++i) {
    st->final_transformation[i] = L.final_T[i];
    st->last_transformation[i] = L.last_T[i];
  }
}

// CritParams::rmax of the frame F
static double frame_rmax(const Index& F)
{
  double rmax = 0.0;
  for (int r = 0; r < 3; ++r) {
    const double m = std::max(std::fabs((double)F.lo[r]), std::fabs((double)F.hi[r]));
    rmax += m * m;
  }
  return std::sqrt(rmax);
}

// what DefaultConvergenceCriteria and the tracking decision of k_solve read
static CritParams crit_params(const Icp& s, int track_mode)
{
  CritParams crit;
  crit.max_iterations = s.P.max_iterations;
  crit.failure_after_max_iter = s.P.failure_after_max_iter;
  crit.max_iterations_similar = s.P.max_iterations_similar_transforms;
  crit.scalar_is_double = s.P.scalar_is_double;
  crit.track_mode = track_mode;
  crit.rot_eps = s.P.transformation_rotation_epsilon;
  crit.trans_eps = s.P.transformation_epsilon;
  crit.rel_mse = s.P.euclidean_fitness_epsilon;
  crit.abs_mse = s.P.mse_threshold_absolute;
  crit.rmax = frame_rmax(target_frame(s));
  return crit;
}

// the search and accumulation arguments that do not depend on where the loop state lives
static IterArgs loop_args(const Icp& s, int track_mode)
{
  const Index& T = *s.tgt;
  IterArgs a;
  memset(&a, 0, sizeof(a));
  a.nodes = T.nodes.p;
  a.pts = T.pts.p;
  a.root = T.root;
  a.tgt_normals = s.tgt_normals.p;
  a.plane_offsets = 1;  // normals_by_pos; the sharded target's record exchange (gnrm) moves whole records
  a.cur = s.cur.p;
  a.n = s.n_q;
  a.gate = gate_from_max_dist(s.P.max_correspondence_distance);
  a.d_error = s.ctx->d_error;
  a.src_orig = s.src_orig.p;
  a.cur_normals = s.cur_normals.p;
  a.enforce_same_dir = s.P.enforce_same_direction_normals;
  a.cells = tree_view(T).cells;
  a.track_sel = track_mode == PCLB200_TRACK_AUTO;  // the search runs only in the flavour of the device's decision
  return a;
}

// The do-while of icp.hpp:164-241.  Every iteration enqueues correspondence estimation -> rejector chain -> accumulation
// -> (NCCL all-reduce) -> k_solve, and k_solve's tail does the loop's bookkeeping on the device copy of the loop state:
// final = T_k * final, the iteration count, DefaultConvergenceCriteria, the tracking decision and the correspondence
// totals.  Once a criterion fires `done` turns the kernels still queued into no-ops.
void icp_iterate(Icp& s, int max_steps, pclb200_icp_stats* stats)
{
  Ctx& c = *s.ctx;
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(!s.batch.B, PCLB200_ERR_INVALID, "icp: a batch session advances with iterate_batch");
  PCLB_REQUIRE(s.tgt && s.cur.p, PCLB200_ERR_INVALID, "icp: set_target and set_source must precede iterate");
  PCLB_REQUIRE(s.P.estimator == PCLB200_EST_SVD || s.tgt_normals.p, PCLB200_ERR_INVALID,
               "icp: point-to-plane needs target normals");
  PCLB_REQUIRE(s.P.estimator != PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS || s.cur_normals.p, PCLB200_ERR_INVALID,
               "icp: the symmetric objective needs source normals (choose the estimator before set_source)");
  if (s.sharded_target)
    check_sharded_target(s);
  // a sharded source sees only its own shard in the reciprocal tree: a different answer, not a smaller one
  PCLB_REQUIRE(!(comm_active(c) && s.P.use_reciprocal), PCLB200_ERR_INVALID,
               "icp: reciprocal correspondences are not available with a sharded source (multi-GPU communicator)");
  // the reference's do-while runs at least once per align(); a caller stepping one iteration at a time resumes a
  // NOT_CONVERGED session, and a fresh session (iterations == 0) always enters
  if (s.loop.state == PCLB200_CONV_NOT_CONVERGED && max_steps > 0) {
    const Index& T = *s.tgt;
    const int kind = s.P.correspondence_kind;
    const bool normal_based = kind != PCLB200_CORR_NEAREST;  // setCorrespondenceEstimation(NormalShooting / BackProjection)
    int keff = 0;
    if (normal_based) {
      PCLB_REQUIRE(kind == PCLB200_CORR_NORMAL_SHOOTING || kind == PCLB200_CORR_BACK_PROJECTION, PCLB200_ERR_INVALID,
                   "icp: unknown correspondence_kind");
      PCLB_REQUIRE(!s.P.use_reciprocal, PCLB200_ERR_INVALID,
                   "icp: reciprocal correspondences are only built for the nearest-neighbour estimator");
      PCLB_REQUIRE(s.cur_normals.p, PCLB200_ERR_INVALID, "icp: the normal-based estimators need source normals");
      PCLB_REQUIRE(kind != PCLB200_CORR_BACK_PROJECTION || s.tgt_normals.p, PCLB200_ERR_INVALID,
                   "icp: back projection needs target normals");
      keff = (int)std::min<size_t>((size_t)std::max(s.P.correspondence_k, 0), T.n_valid);
      PCLB_REQUIRE(keff > 0, PCLB200_ERR_INVALID, "icp: correspondence_k must be positive");
    }
    if (comm_active(c))
      prepare_sharded_rejectors(s);
    const bool nccl_path = comm_active(c) && !comm_peer_fused(c);  // collectives launched by NCCL
    // a sharded target sums the gathered pairs, already the whole map's, on every rank: no accumulator exchange
    const bool host_reduce = nccl_path && !s.sharded_target;
    // The normal-based estimators' k-NN rows, rejector chains (their sorts synchronise), the reciprocal tree rebuilt
    // every iteration, the symmetric objective and an NCCL collective: the loop state is read back after every
    // iteration and the loop stops once k_solve sets `done`.  Otherwise every iteration this call may run is enqueued
    // at once and the stream is synchronised once.
    const bool needs_host_between = normal_based || !s.rejectors.empty() || s.P.use_reciprocal ||
                                    s.P.estimator == PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS || nccl_path;
    // Temporal coherence (still_nearest) pays once the cloud has almost stopped moving: tracking the lower bounds makes a
    // walk look at a wider ball, so AUTO switches it on when the last increment displaced no point by more than half the
    // RMS correspondence distance (k_solve), and the skip test fires from the following iteration on.  Only the plain
    // nearest-neighbour search keeps the bounds.
    const int track_mode = (normal_based || s.P.use_reciprocal) ? (int)PCLB200_TRACK_OFF : s.P.track_mode;
    const CritParams crit = crit_params(s, track_mode);
    const Index& F = target_frame(s);
    if (track_mode != PCLB200_TRACK_AUTO)  // AUTO carries the last decision over from the previous call
      s.loop.track_next = track_mode == PCLB200_TRACK_ON ? 1 : 0;
    LoopCtrl* h_ctrl = static_cast<LoopCtrl*>(c.pinned);
    unsigned long long* h_skipped = reinterpret_cast<unsigned long long*>(h_ctrl + 1);
    int* h_err = reinterpret_cast<int*>(h_skipped + 1);
    static_assert(sizeof(LoopCtrl) % 8 == 0, "the skip count follows the loop state in the pinned block");
    const bool first = s.loop.iterations == 0;
    // the first iteration's SVD origin (LoopCtrl::origin); k_seed_origin replaces it wherever the rank holds the whole
    // source (a single rank, a sharded target)
    if (first)
      for (int r = 0; r < 3; ++r)
        s.loop.origin[r] = 0.5f * (F.lo[r] + F.hi[r]);
    *h_ctrl = s.loop;
    PCLB_CUDA(cudaMemcpyAsync(s.ctrl.p, h_ctrl, sizeof(LoopCtrl), cudaMemcpyHostToDevice, st));
    if (first && s.P.estimator == PCLB200_EST_SVD && (!comm_active(c) || s.sharded_target)) {
      k_seed_origin<<<1, 1, 0, st>>>(s.cur.p, nullptr, s.n_q, s.ctrl.p->origin);
      ++c.launches;
    }
    // one synchronise reads the loop state, the skip count (statistics) and the device error flag
    auto read_back = [&]() {
      PCLB_CUDA(cudaMemcpyAsync(h_ctrl, s.ctrl.p, sizeof(LoopCtrl), cudaMemcpyDeviceToHost, st));
      PCLB_CUDA(cudaMemcpyAsync(h_skipped, s.skip_count.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
      PCLB_CUDA(cudaMemcpyAsync(h_err, c.d_error, sizeof(int), cudaMemcpyDeviceToHost, st));
      PCLB_CUDA(cudaStreamSynchronize(st));
      if (*h_err)
        raise_device_error(c, *h_err);
      s.loop = *h_ctrl;
      s.total_skipped = (int64_t)*h_skipped;
    };
    IterArgs a = loop_args(s, track_mode);
    a.pending = s.pending.p;
    a.origin = s.ctrl.p->origin;
    a.partials = s.red.partials.p;
    a.partials2 = s.red.partials2.p;
    a.counter = s.red.counter.p;
    a.accum = s.red.accum.p;
    a.skip_count = s.skip_count.p;
    a.ctrl = s.ctrl.p;
    const unsigned grid = persistent_blocks(c, s.n_q);
    // the search: 72 blocks per SM over the 5 that are resident, so a block walks only a few warp rounds and the SMs run
    // out of work together (18 left the last blocks walking alone; a block per warp round pays for every launch that a
    // finished loop or the unwanted tracking flavour returns from at once)
    const unsigned wgrid = persistent_blocks(c, s.n_q, 256, 72);
    const unsigned agrid = std::min(persistent_blocks(c, s.n_q, 256, kAccumBlocksPerSM), s.red.max_blocks);
    const int n_enq = std::min(max_steps, std::max(1, s.P.max_iterations - s.loop.iterations));
    // sharded target: the accumulate kernels read the gathered records and the global matches
    const bool shard_nrm = s.sharded_target && s.P.estimator != PCLB200_EST_SVD && s.tgt_normals.p;
    if (s.sharded_target) {
      if (s.gmatch.n != s.n_q) {
        s.gmatch.alloc(s.n_q, st);
        s.gpts.alloc(s.n_q, st);
      }
      if (shard_nrm && s.gnrm.n != s.n_q)
        s.gnrm.alloc(s.n_q, st);
    }
    IterArgs ga = a;
    ga.pts = s.gpts.p;
    ga.tgt_normals = shard_nrm ? s.gnrm.p : nullptr;
    Match* const acc_match = s.sharded_target ? s.gmatch.p : s.match.p;
    const IterArgs& aa = s.sharded_target ? ga : a;
    for (int k = 0; k < n_enq; ++k) {
      std::unique_ptr<Index> src_index;
      {
        ProfScope ps(c, "icp_search");
        if (normal_based || s.P.use_reciprocal) {
          k_apply_pending<<<grid, 256, 0, st>>>(s.cur.p, s.n_q, s.pending.p, s.cur_normals.p);
          k_clear_apply<<<1, 1, 0, st>>>(s.pending.p);
          c.launches += 2;
        }
        if (normal_based) {
          // k-NN candidates, then the normal-based choice
          DevBuf<int32_t> nn_idx;
          DevBuf<float> nn_d2;
          nn_idx.alloc(s.n_q * (size_t)keff, st);
          nn_d2.alloc(s.n_q * (size_t)keff, st);
          launch_knn(c, T, s.cur.p, s.n_q, keff, std::numeric_limits<float>::infinity(), nn_idx.p, nn_d2.p);
          ensure_pos_of_orig(c, const_cast<Index&>(T));
          k_select_match<<<grid_for(s.n_q, 128), 128, 0, st>>>(s.cur.p, s.cur_normals.p, s.n_q, kind, keff, nn_idx.p,
                                                              nn_d2.p, T.pts.p, T.pos_of_orig.p, s.tgt_normals.p,
                                                              s.P.max_correspondence_distance, s.match.p);
          ++c.launches;
        }
        else if (s.P.use_reciprocal) {
          // tree_reciprocal_ is rebuilt over the transformed source every iteration
          // (correspondence_estimation.hpp:117-135 via setInputSource at icp.hpp:175)
          src_index.reset(build_index_from_device(c, s.cur.p, s.n_q, s.cur_label.p));
          a.s_nodes = src_index->nodes.p;
          a.s_pts = src_index->pts.p;
          a.s_root = src_index->root;
          k_search<true, false><<<wgrid, 256, 0, st>>>(a, s.match.p, s.lb.p);
          ++c.launches;
        }
        else {
          bool plain = track_mode != PCLB200_TRACK_ON, track = track_mode != PCLB200_TRACK_OFF;
          if (track_mode == PCLB200_TRACK_AUTO && needs_host_between) {  // the host has read this iteration's decision
            track = s.loop.track_next != 0;
            plain = !track;
          }
          if (plain) {
            k_search<false, false><<<wgrid, 256, 0, st>>>(a, s.match.p, s.lb.p);
            ++c.launches;
          }
          if (track) {
            k_search<false, true><<<wgrid, 256, 0, st>>>(a, s.match.p, s.lb.p);
            ++c.launches;
          }
        }
      }
      if (!s.rejectors.empty()) {
        ProfScope ps(c, "icp_reject");
        run_rejectors(s);
      }
      if (s.sharded_target) {
        ProfScope ps(c, "icp_exchange");
        exchange_shard_matches(s, shard_nrm);
      }
      else  // drawn after the rejector chain's exchanges: every rank takes the sequence numbers in the same order
        comm_peer_view(c, &a.peer, &a.seq);
      {
        ProfScope ps(c, "icp_accum");
        if (s.P.estimator == PCLB200_EST_SVD)
          k_accum_dmma<PCLB200_EST_SVD><<<agrid, 256, 0, st>>>(aa, acc_match);
        else if (s.P.estimator == PCLB200_EST_POINT_TO_PLANE_LLS)
          k_accum_dmma<PCLB200_EST_POINT_TO_PLANE_LLS><<<agrid, 256, 0, st>>>(aa, acc_match);
        else
          k_accum<PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS><<<grid, 256, 0, st>>>(aa, acc_match);
        ++c.launches;
      }
      if (host_reduce) {
        ProfScope ps(c, "allreduce");
        comm_allreduce_sum(c, s.red.accum.p, kAccum);
      }
      {
        ProfScope ps(c, "solve");
        k_solve<<<1, 32, 0, st>>>(s.red.accum.p, s.P.estimator, s.P.scalar_is_double, transform_mode(s.P), a.origin, 3,
                                  s.pending.p, s.solve_out.p, s.P.svd_no_umeyama, s.ctrl.p, crit);
        ++c.launches;
      }
      PCLB_CUDA(cudaGetLastError());
      if (needs_host_between) {
        read_back();
        if (s.loop.done)
          break;
      }
    }
    if (!needs_host_between)
      read_back();
  }
  fill_stats(s.loop, s.total_skipped, stats);
}

// correspondences of the last evaluated iteration (Registration::correspondences_, what PCL hands to the
// visualisation callback at icp.hpp:228-236), ordered by position in the source index list
__global__ void k_matches_to_corr(const float4* __restrict__ cur, const Match* __restrict__ match, size_t n,
                                  const float4* __restrict__ tgt_pts, const int32_t* __restrict__ src_orig,
                                  pclb200_corr* __restrict__ by_slot)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const int slot = __float_as_int(cur[i].w);
  const Match m = match[i];
  pclb200_corr r;
  r.index_query = src_orig ? src_orig[slot] : slot;
  const bool acc = match_accepted(m);
  r.index_match = acc ? __float_as_int(tgt_pts[m.pos].w) : -1;
  r.distance = acc ? m.d2 : 0.f;
  by_slot[slot] = r;
}

// whether a loop has evaluated correspondences since its last reset: a loop that stopped with NO_CORRESPONDENCES in its
// first evaluation (iterations == 0) keeps the list that stopped it, as correspondences_ does (icp.hpp:204-213)
static bool has_evaluated(const LoopCtrl& L)
{
  return L.iterations > 0 || L.state != PCLB200_CONV_NOT_CONVERGED;
}

size_t icp_get_correspondences(Icp& s, pclb200_corr* out)
{
  Ctx& c = *s.ctx;
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(!s.batch.B, PCLB200_ERR_INVALID, "icp: a batch session hands its lists out through get_correspondences_batch");
  PCLB_REQUIRE(s.tgt && s.cur.p && s.match.p, PCLB200_ERR_INVALID, "icp: no iteration has run");
  if (!s.n_q || !has_evaluated(s.loop))
    return 0;
  DevBuf<pclb200_corr> by_slot;
  by_slot.alloc(s.n_q, st);
  // sharded target: the global matches point into the gathered records, whose w lanes are the map's ids
  k_matches_to_corr<<<grid_for(s.n_q, 256), 256, 0, st>>>(s.cur.p, s.sharded_target ? s.gmatch.p : s.match.p, s.n_q,
                                                          s.sharded_target ? s.gpts.p : s.tgt->pts.p, s.src_orig.p, by_slot.p);
  ++c.launches;
  const size_t m = compact_corr_to(c, by_slot.p, s.n_q, out);
  PCLB_CUDA(cudaStreamSynchronize(st));
  return m;
}

// ---- a batch of problems in one loop (include/pclb200_batch.h) ---------------------------------------------------------
// key of the second, stable pass of the batch's query sort: the problem of the record whose query sits at j
__global__ void k_problem_keys(const float4* __restrict__ q, size_t n, const long long* __restrict__ offsets,
                               int n_problems, unsigned* __restrict__ keys, int32_t* __restrict__ vals)
{
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n)
    return;
  keys[j] = (unsigned)problem_of(offsets, n_problems, __float_as_int(q[j].w));
  vals[j] = (int32_t)j;
}

__global__ void k_gather_by(const float4* __restrict__ q, const int32_t* __restrict__ vals, size_t n,
                            float4* __restrict__ out)
{
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j < n)
    out[j] = q[vals[j]];
}

void sort_by_problem(Ctx& c, const long long* d_offsets, int n_problems, QueryBatch& qb)
{
  cudaStream_t st = c.stream;
  const size_t n = qb.n;
  DevBuf<unsigned> keys_in, keys;
  DevBuf<int32_t> vals_in, vals;
  keys_in.alloc(n, st);
  keys.alloc(n, st);
  vals_in.alloc(n, st);
  vals.alloc(n, st);
  k_problem_keys<<<grid_for(n, 256), 256, 0, st>>>(qb.q.p, n, d_offsets, n_problems, keys_in.p, vals_in.p);
  ++c.launches;
  int bits = 1;
  while ((1 << bits) < n_problems)
    ++bits;
  size_t tmp_bytes = 0;
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys_in.p, keys.p, vals_in.p, vals.p, (int)n, 0, bits, st));
  DevBuf<unsigned char> tmp;
  tmp.alloc(tmp_bytes, st);
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, keys_in.p, keys.p, vals_in.p, vals.p, (int)n, 0, bits, st));
  c.launches += 2;
  DevBuf<float4> sorted;
  sorted.alloc(n, st);
  k_gather_by<<<grid_for(n, 256), 256, 0, st>>>(qb.q.p, vals.p, n, sorted.p);
  ++c.launches;
  qb.q = std::move(sorted);
}

__global__ void k_relative_index(const long long* __restrict__ offsets, int n_problems, size_t n, int32_t* __restrict__ rel)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n)
    rel[i] = (int32_t)((long long)i - offsets[problem_of(offsets, n_problems, (long long)i)]);
}

// the lists of problems that have run no iteration are empty (icp_get_correspondences); counts[p] = the list of p's length
__global__ void k_mask_and_count(pclb200_corr* __restrict__ by_slot, size_t n, const long long* __restrict__ offsets,
                                 int n_problems, const int* __restrict__ live, unsigned long long* __restrict__ counts)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n || by_slot[i].index_match < 0)
    return;
  const int p = problem_of(offsets, n_problems, (long long)i);
  if (live[p])
    atomicAdd(counts + p, 1ull);
  else
    by_slot[i].index_match = -1;
}

// k_matches_to_corr of a batch of scan pairs: each match is a position in its own problem's target
__global__ void k_matches_to_corr_targets(const float4* __restrict__ cur, const Match* __restrict__ match, size_t n,
                                          const long long* __restrict__ offsets, int n_problems,
                                          const BatchTarget* __restrict__ targets, const int32_t* __restrict__ rel,
                                          pclb200_corr* __restrict__ by_slot)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const int slot = __float_as_int(cur[i].w);
  const Match m = match[i];
  pclb200_corr r;
  r.index_query = rel[slot];
  const bool acc = match_accepted(m);
  r.index_match = acc ? __float_as_int(targets[problem_of(offsets, n_problems, slot)].pts[m.pos].w) : -1;
  r.distance = acc ? m.d2 : 0.f;
  by_slot[slot] = r;
}

// what a batch refuses (include/pclb200_batch.h), checked by set_target_batch, set_source_batch and every iterate_batch
static void check_batch_params(const Icp& s)
{
  Ctx& c = *s.ctx;
  PCLB_REQUIRE(!comm_active(c), PCLB200_ERR_INVALID, "icp: a batch runs on one GPU: no communicator, no sharded target");
  PCLB_REQUIRE(s.rejectors.empty(), PCLB200_ERR_INVALID, "icp: a batch takes no rejector chain");
  PCLB_REQUIRE(!s.P.use_reciprocal, PCLB200_ERR_INVALID, "icp: a batch takes no reciprocal correspondences");
  PCLB_REQUIRE(s.P.correspondence_kind == PCLB200_CORR_NEAREST, PCLB200_ERR_INVALID,
               "icp: a batch takes nearest-neighbour correspondences only");
}

static void check_batch_session(const Icp& s)
{
  PCLB_REQUIRE(s.tgt != nullptr, PCLB200_ERR_INVALID, "icp: no target set (registration.hpp:77-81)");
  PCLB_REQUIRE(!s.sharded_target, PCLB200_ERR_INVALID, "icp: a batch runs on one GPU: no communicator, no sharded target");
  check_batch_params(s);
}

// the session without a source (its batch read-back buffer kept: freeing pinned memory synchronises the device)
static void drop_source(Icp& s)
{
  PinnedBuf host = std::move(s.batch.host);
  s.batch = IcpBatch();
  s.batch.host = std::move(host);
  s.cur.release();
  s.src_all.release();
  s.src_raw.release();
  s.match.release();
  s.n_all = s.n_q = 0;
}

void icp_set_target_batch(Icp& s, const Index* const* targets, const void* const* tgt_normals, size_t stride_n,
                          int n_targets)
{
  Ctx& c = *s.ctx;
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(n_targets >= 1 && n_targets <= 65536, PCLB200_ERR_INVALID, "icp: a batch holds 1 to 65536 problems");
  check_batch_params(s);
  const int B = n_targets;
  for (int p = 0; p < B; ++p)
    PCLB_REQUIRE(targets[p]->device == c.device, PCLB200_ERR_INVALID, "icp: a target index lives on another device");
  bool all_normals = tgt_normals != nullptr;
  for (int p = 0; all_normals && p < B; ++p)
    all_normals = tgt_normals[p] != nullptr;
  PCLB_REQUIRE(s.P.estimator == PCLB200_EST_SVD || all_normals, PCLB200_ERR_INVALID,
               "icp: point-to-plane and the symmetric objective need every problem's target normals");
  IcpTargets T;
  T.B = B;
  T.idx.assign(targets, targets + B);
  T.all_normals = all_normals;
  std::vector<BatchTarget> h(B);
  std::vector<float4> frames(B);
  std::vector<std::pair<std::pair<const Index*, const void*>, const float4*>> staged;  // one normals_by_pos per pair
  for (int p = 0; p < B; ++p) {
    const Index& I = *targets[p];
    const void* nrm = tgt_normals ? tgt_normals[p] : nullptr;
    const float4* by_pos = nullptr;
    if (nrm) {
      for (const auto& e : staged)
        if (e.first.first == &I && e.first.second == nrm)
          by_pos = e.second;
      if (!by_pos) {
        T.normals.emplace_back();
        normals_by_pos(c, &I, nrm, stride_n, T.normals.back());
        by_pos = T.normals.back().p;
        staged.push_back({{&I, nrm}, by_pos});
      }
    }
    const TreeView v = tree_view(I);
    h[p] = BatchTarget{v.nodes, v.pts, by_pos, v.root, v.cells, frame_rmax(I)};
    frames[p] = make_float4(I.lo[0], I.lo[1], I.lo[2], I.morton_scale);
  }
  T.table.alloc(B, st);
  T.frames.alloc(B, st);
  PCLB_CUDA(cudaMemcpyAsync(T.table.p, h.data(), B * sizeof(BatchTarget), cudaMemcpyHostToDevice, st));
  PCLB_CUDA(cudaMemcpyAsync(T.frames.p, frames.data(), B * sizeof(float4), cudaMemcpyHostToDevice, st));
  drop_source(s);
  s.targets = std::move(T);
  s.tgt = targets[0];
  s.sharded_target = false;
  s.tgt_normals.release();
}

// batch_blocks's table (icp_kernels.cuh) on the device; *slots = its blocks (partials slots)
template <typename Grid>
static void batch_table(Ctx& c, const std::vector<long long>& off, Grid grid, DevBuf<BatchBlock>& out, unsigned* slots)
{
  const std::vector<BatchBlock> h = batch_blocks(off, grid);
  if (slots)
    *slots = (unsigned)h.size();
  out.alloc(h.size(), c.stream);
  PCLB_CUDA(cudaMemcpyAsync(out.p, h.data(), h.size() * sizeof(BatchBlock), cudaMemcpyHostToDevice, c.stream));
}

void icp_set_source_batch(Icp& s, const void* src, size_t n, size_t stride, const void* src_normals, size_t stride_n,
                          const int64_t* offsets, int n_problems, const double* guesses)
{
  Ctx& c = *s.ctx;
  cudaStream_t st = c.stream;
  check_batch_session(s);
  PCLB_REQUIRE(n_problems >= 1 && n_problems <= 65536, PCLB200_ERR_INVALID, "icp: a batch holds 1 to 65536 problems");
  PCLB_REQUIRE(src != nullptr && n > 0 && offsets != nullptr, PCLB200_ERR_INVALID, "icp: empty source");
  PCLB_REQUIRE(n < (size_t)0x7fffffff, PCLB200_ERR_INVALID, "icp: a batch holds fewer than 2^31 - 1 records");
  PCLB_REQUIRE(stride >= 12 && stride % 4 == 0, PCLB200_ERR_INVALID, "stride must be a multiple of 4 and >= 12");
  PCLB_REQUIRE(offsets[0] == 0 && offsets[n_problems] == (int64_t)n, PCLB200_ERR_INVALID,
               "icp: batch offsets must run from 0 to n");
  for (int p = 0; p < n_problems; ++p)
    PCLB_REQUIRE(offsets[p + 1] > offsets[p], PCLB200_ERR_INVALID,
                 "icp: batch offsets must increase strictly (every problem holds a record)");
  PCLB_REQUIRE(s.P.estimator != PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS || src_normals, PCLB200_ERR_INVALID,
               "icp: the symmetric objective needs source normals");
  const bool per_target = s.targets.B > 0;
  PCLB_REQUIRE(!per_target || n_problems == s.targets.B, PCLB200_ERR_INVALID,
               "icp: a batch source holds one problem per target of set_target_batch");
  const int B = n_problems;
  PinnedBuf host = std::move(s.batch.host);  // kept across batches: freeing pinned memory synchronises the device
  s.batch = IcpBatch();
  IcpBatch& b = s.batch;
  b.host = std::move(host);
  b.B = B;
  b.offsets.assign(offsets, offsets + B + 1);
  b.d_offsets.alloc(B + 1, st);
  PCLB_CUDA(cudaMemcpyAsync(b.d_offsets.p, b.offsets.data(), (B + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
  // the queries of all problems in the order of the target frame (a batch of targets: each in its own target's frame)
  // (stable), then by problem (stable): within each problem the order make_query_batch gives that problem alone; w = the
  // record's index in the batch
  QueryBatch qb;
  stage_source(s, src, n, stride, src_normals, stride_n, nullptr, 0, per_target ? nullptr : &qb);
  {
    ProfScope ps(c, "query_sort");
    if (per_target)  // src_all holds the staged xyz
      make_query_batch_framed(c, s.targets.frames.p, b.d_offsets.p, B, s.src_all.p, n, qb);
    sort_by_problem(c, b.d_offsets.p, B, qb);
  }
  finish_source(s, qb, src_normals, stride_n);
  b.rel.alloc(n, st);
  k_relative_index<<<grid_for(n, 256), 256, 0, st>>>(b.d_offsets.p, B, n, b.rel.p);
  ++c.launches;
  // each problem's grids are the ones its own align launches (icp_iterate)
  batch_table(c, b.offsets, [&](size_t m) { return persistent_blocks(c, m, 256, 72); }, b.wtab, nullptr);
  batch_table(c, b.offsets, [&](size_t m) { return std::min(persistent_blocks(c, m, 256, kAccumBlocksPerSM), s.red.max_blocks); },
              b.atab, &b.a_blocks);
  batch_table(c, b.offsets, [&](size_t m) { return persistent_blocks(c, m); }, b.gtab, &b.g_blocks);
  b.ctrl.alloc(B, st);
  b.solve_out.alloc(B, st);
  b.skip_count.alloc(B, st);
  b.counter.alloc(B, st);
  b.accum.alloc((size_t)B * kAccum, st);
  PCLB_CUDA(cudaMemsetAsync(b.skip_count.p, 0, B * sizeof(unsigned long long), st));
  PCLB_CUDA(cudaMemsetAsync(b.counter.p, 0, B * sizeof(unsigned), st));
  PCLB_CUDA(cudaMemsetAsync(b.accum.p, 0, (size_t)B * kAccum * sizeof(double), st));
  b.host.reserve(B * (sizeof(LoopCtrl) + sizeof(unsigned long long)) + sizeof(int));
  // every problem's loop state as icp_set_source of a new session leaves it (its own criteria, previous MSE DBL_MAX);
  // a guess that is not the identity moves its queries once
  icp_reset_state(s, nullptr);
  b.loop.assign(B, s.loop);
  for (LoopCtrl& L : b.loop)
    L.prev_mse = std::numeric_limits<double>::max();
  b.total_skipped.assign(B, 0);
  const int mode = transform_mode(s.P);
  std::vector<Pending> h(B);
  bool any_guess = false;
  for (int p = 0; p < B; ++p) {
    if (guesses)
      for (int i = 0; i < 16; ++i)
        b.loop[p].final_T[i] = s.P.scalar_is_double ? guesses[16 * p + i] : (double)(float)guesses[16 * p + i];
    const bool moved = !is_identity(b.loop[p].final_T);
    any_guess = any_guess || moved;
    h[p] = make_pending(b.loop[p].final_T, mode, moved ? 1 : 0);
  }
  b.pending.alloc(B, st);
  PCLB_CUDA(cudaMemcpyAsync(b.pending.p, h.data(), B * sizeof(Pending), cudaMemcpyHostToDevice, st));
  if (any_guess) {
    k_transform_batch<<<persistent_blocks(c, n), 256, 0, st>>>(s.cur.p, n, b.d_offsets.p, B, b.pending.p, s.cur_normals.p);
    ++c.launches;
  }
  for (int p = 0; p < B; ++p)
    h[p] = make_pending(b.loop[p].last_T, mode, 0);
  PCLB_CUDA(cudaMemcpyAsync(b.pending.p, h.data(), B * sizeof(Pending), cudaMemcpyHostToDevice, st));
  PCLB_CUDA(cudaGetLastError());
}

// icp_iterate of every problem of the batch at once: every stage one launch, the per-problem loop states read back once
// per call (the symmetric objective: once per iteration, as icp_iterate does)
void icp_iterate_batch(Icp& s, int max_steps, pclb200_icp_stats* stats)
{
  Ctx& c = *s.ctx;
  cudaStream_t st = c.stream;
  IcpBatch& b = s.batch;
  const int B = b.B;
  PCLB_REQUIRE(B > 0, PCLB200_ERR_INVALID, "icp: iterate_batch needs a batch source (set_source_batch)");
  check_batch_session(s);
  const IcpTargets& TB = s.targets;
  const BatchTarget* targets = TB.B ? TB.table.p : nullptr;  // null: every problem against the session's target
  PCLB_REQUIRE(s.P.estimator == PCLB200_EST_SVD || (targets ? TB.all_normals : s.tgt_normals.p != nullptr),
               PCLB200_ERR_INVALID, "icp: point-to-plane needs target normals");
  PCLB_REQUIRE(s.P.estimator != PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS || s.cur_normals.p, PCLB200_ERR_INVALID,
               "icp: the symmetric objective needs source normals (choose the estimator before set_source_batch)");
  int budget = 0;
  for (int p = 0; p < B; ++p)
    if (b.loop[p].state == PCLB200_CONV_NOT_CONVERGED && max_steps > 0)
      budget = std::max(budget, std::max(1, s.P.max_iterations - b.loop[p].iterations));
  if (budget > 0) {
    const int track_mode = s.P.track_mode;
    const CritParams crit = crit_params(s, track_mode);
    LoopCtrl* h_ctrl = static_cast<LoopCtrl*>(b.host.p);
    unsigned long long* h_skipped = reinterpret_cast<unsigned long long*>(h_ctrl + B);
    int* h_err = reinterpret_cast<int*>(h_skipped + B);
    for (int p = 0; p < B; ++p) {
      LoopCtrl& L = b.loop[p];
      if (L.state == PCLB200_CONV_NOT_CONVERGED) {
        if (track_mode != PCLB200_TRACK_AUTO)
          L.track_next = track_mode == PCLB200_TRACK_ON ? 1 : 0;
        const Index& F = targets ? *TB.idx[p] : target_frame(s);
        if (L.iterations == 0)
          for (int r = 0; r < 3; ++r)
            L.origin[r] = 0.5f * (F.lo[r] + F.hi[r]);
      }
      h_ctrl[p] = L;
      if (L.state != PCLB200_CONV_NOT_CONVERGED)
        h_ctrl[p].done = 1;  // its blocks return at once
    }
    PCLB_CUDA(cudaMemcpyAsync(b.ctrl.p, h_ctrl, B * sizeof(LoopCtrl), cudaMemcpyHostToDevice, st));
    if (s.P.estimator == PCLB200_EST_SVD) {
      k_seed_origin_batch<<<grid_for(B, 256), 256, 0, st>>>(s.cur.p, b.d_offsets.p, B, b.ctrl.p);
      ++c.launches;
    }
    const bool sym = s.P.estimator == PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS;
    const size_t part_words = sym ? (size_t)b.g_blocks * kAccum : (size_t)b.a_blocks * 128;
    if (b.partials.n < part_words)
      b.partials.alloc(part_words, st);
    auto read_back = [&]() {
      PCLB_CUDA(cudaMemcpyAsync(h_ctrl, b.ctrl.p, B * sizeof(LoopCtrl), cudaMemcpyDeviceToHost, st));
      PCLB_CUDA(cudaMemcpyAsync(h_skipped, b.skip_count.p, B * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
      PCLB_CUDA(cudaMemcpyAsync(h_err, c.d_error, sizeof(int), cudaMemcpyDeviceToHost, st));
      PCLB_CUDA(cudaStreamSynchronize(st));
      if (*h_err)
        raise_device_error(c, *h_err);
      bool all_done = true;
      for (int p = 0; p < B; ++p) {
        if (b.loop[p].state == PCLB200_CONV_NOT_CONVERGED) {  // the others' states stay as they were
          b.loop[p] = h_ctrl[p];
          b.total_skipped[p] = (int64_t)h_skipped[p];
        }
        all_done = all_done && h_ctrl[p].done;
      }
      return all_done;
    };
    IterArgs a = loop_args(s, track_mode);
    a.pending = b.pending.p;
    a.partials = b.partials.p;
    a.partials2 = b.partials.p;
    a.counter = b.counter.p;
    a.accum = b.accum.p;
    a.skip_count = b.skip_count.p;
    a.ctrl = b.ctrl.p;
    const int n_enq = std::min(max_steps, budget);
    for (int k = 0; k < n_enq; ++k) {
      {
        ProfScope ps(c, "icp_search");
        const unsigned g = (unsigned)b.wtab.n;
        if (track_mode != PCLB200_TRACK_ON) {
          if (targets)
            k_search_batch<false, true><<<g, 256, 0, st>>>(a, b.wtab.p, s.match.p, s.lb.p, targets);
          else
            k_search_batch<false><<<g, 256, 0, st>>>(a, b.wtab.p, s.match.p, s.lb.p);
          ++c.launches;
        }
        if (track_mode != PCLB200_TRACK_OFF) {
          if (targets)
            k_search_batch<true, true><<<g, 256, 0, st>>>(a, b.wtab.p, s.match.p, s.lb.p, targets);
          else
            k_search_batch<true><<<g, 256, 0, st>>>(a, b.wtab.p, s.match.p, s.lb.p);
          ++c.launches;
        }
      }
      {
        ProfScope ps(c, "icp_accum");
        const unsigned ag = (unsigned)b.atab.n, gg = (unsigned)b.gtab.n;
        constexpr int kSvd = PCLB200_EST_SVD, kPlane = PCLB200_EST_POINT_TO_PLANE_LLS,
                      kSym = PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS;
        if (s.P.estimator == kSvd && targets)
          k_accum_dmma_batch<kSvd, true><<<ag, 256, 0, st>>>(a, b.atab.p, s.match.p, targets);
        else if (s.P.estimator == kSvd)
          k_accum_dmma_batch<kSvd><<<ag, 256, 0, st>>>(a, b.atab.p, s.match.p);
        else if (s.P.estimator == kPlane && targets)
          k_accum_dmma_batch<kPlane, true><<<ag, 256, 0, st>>>(a, b.atab.p, s.match.p, targets);
        else if (s.P.estimator == kPlane)
          k_accum_dmma_batch<kPlane><<<ag, 256, 0, st>>>(a, b.atab.p, s.match.p);
        else if (targets)
          k_accum_batch<kSym, true><<<gg, 256, 0, st>>>(a, b.gtab.p, s.match.p, targets);
        else
          k_accum_batch<kSym><<<gg, 256, 0, st>>>(a, b.gtab.p, s.match.p);
        ++c.launches;
      }
      {
        ProfScope ps(c, "solve");
        k_solve_batch<<<grid_for((size_t)B * 32, 256), 256, 0, st>>>(b.accum.p, B, s.P.estimator, s.P.scalar_is_double,
                                                                     transform_mode(s.P), b.pending.p, b.solve_out.p,
                                                                     s.P.svd_no_umeyama, b.ctrl.p, crit, targets);
        ++c.launches;
      }
      PCLB_CUDA(cudaGetLastError());
      if (sym && read_back())
        break;
    }
    if (!sym)
      read_back();
  }
  if (stats)
    for (int p = 0; p < B; ++p)
      fill_stats(b.loop[p], b.total_skipped[p], stats + p);
}

void icp_get_correspondences_batch(Icp& s, pclb200_corr* out, int64_t* counts)
{
  Ctx& c = *s.ctx;
  cudaStream_t st = c.stream;
  const IcpBatch& b = s.batch;
  const int B = b.B;
  PCLB_REQUIRE(B > 0, PCLB200_ERR_INVALID, "icp: get_correspondences_batch needs a batch source (set_source_batch)");
  const size_t n = s.n_q;
  DevBuf<pclb200_corr> by_slot;
  by_slot.alloc(n, st);
  if (s.targets.B)
    k_matches_to_corr_targets<<<grid_for(n, 256), 256, 0, st>>>(s.cur.p, s.match.p, n, b.d_offsets.p, B,
                                                                s.targets.table.p, b.rel.p, by_slot.p);
  else
    k_matches_to_corr<<<grid_for(n, 256), 256, 0, st>>>(s.cur.p, s.match.p, n, s.tgt->pts.p, b.rel.p, by_slot.p);
  std::vector<int> live(B);
  for (int p = 0; p < B; ++p)
    live[p] = has_evaluated(b.loop[p]);
  DevBuf<int> d_live;
  DevBuf<unsigned long long> d_counts;
  d_live.alloc(B, st);
  d_counts.alloc(B, st);
  PCLB_CUDA(cudaMemcpyAsync(d_live.p, live.data(), B * sizeof(int), cudaMemcpyHostToDevice, st));
  PCLB_CUDA(cudaMemsetAsync(d_counts.p, 0, B * sizeof(unsigned long long), st));
  k_mask_and_count<<<grid_for(n, 256), 256, 0, st>>>(by_slot.p, n, b.d_offsets.p, B, d_live.p, d_counts.p);
  c.launches += 2;
  PCLB_CUDA(cudaGetLastError());
  std::vector<unsigned long long> h(B);
  compact_corr_to(c, by_slot.p, n, out);  // synchronises: live has reached the device
  PCLB_CUDA(cudaMemcpyAsync(h.data(), d_counts.p, B * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  for (int p = 0; p < B; ++p)
    counts[p] = (int64_t)h[p];
}

// output = *input_ ; transformCloud(*input_, output, final_transformation_) — icp.hpp:265-267
void icp_get_cloud(Icp& s, void* out_pts, size_t stride_out, void* out_normals, size_t stride_n)
{
  Ctx& c = *s.ctx;
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(s.src_all.p, PCLB200_ERR_INVALID, "icp: no source");
  const bool do_n = out_normals && s.have_src_normals;
  const int mode = transform_mode(s.P);
  // a batch: every record moves by its own problem's final transform
  const IcpBatch& b = s.batch;
  DevBuf<Pending> finals;
  if (b.B) {
    std::vector<Pending> h(b.B);
    for (int p = 0; p < b.B; ++p)
      h[p] = make_pending(b.loop[p].final_T, mode, 1);
    finals.alloc(b.B, st);
    PCLB_CUDA(cudaMemcpyAsync(finals.p, h.data(), b.B * sizeof(Pending), cudaMemcpyHostToDevice, st));
  }
  const bool normals_inside =
      do_n && s.src_normal_off >= 0 &&
      static_cast<unsigned char*>(out_normals) - static_cast<unsigned char*>(out_pts) == s.src_normal_off && stride_n == stride_out;
  if (s.src_raw.p && stride_out == s.src_stride && (!do_n || normals_inside)) {
    // output = *input_ (all fields) with xyz / normals transformed: one pass over the records, one contiguous copy out
    DevBuf<unsigned char> rec;
    unsigned char* d_rec = out_on_device(c, static_cast<unsigned char*>(out_pts), s.n_all * stride_out, rec);
    const int vec = stride_out % 16 == 0 && reinterpret_cast<uintptr_t>(d_rec) % 16 == 0;  // src_raw is 16-aligned
    {
      ProfScope ps(c, "transform_out");
      const int nrm_word = do_n ? (int)(s.src_normal_off / 4) : -1;
      if (b.B)
        k_assemble_records_batch<<<grid_for(s.n_all, 256), 256, 0, st>>>(s.src_raw.p, s.n_all, stride_out, nrm_word,
                                                                         b.d_offsets.p, b.B, finals.p, vec, d_rec);
      else
        k_assemble_records<<<grid_for(s.n_all, 256), 256, 0, st>>>(s.src_raw.p, s.n_all, stride_out, nrm_word,
                                                                   make_pending(s.loop.final_T, mode, 1), vec, d_rec);
      ++c.launches;
    }
    PCLB_CUDA(cudaGetLastError());
    copy_out(c, static_cast<unsigned char*>(out_pts), rec, s.n_all * stride_out);
    PCLB_CUDA(cudaStreamSynchronize(st));
    return;
  }
  // every other layout: dense xyz (and normals) transformed, then written to the caller's arrays
  DevBuf<float4> tmp, tmpn;
  tmp.alloc(s.n_all, st);
  PCLB_CUDA(cudaMemcpyAsync(tmp.p, s.src_all.p, s.n_all * sizeof(float4), cudaMemcpyDeviceToDevice, st));
  if (do_n) {
    tmpn.alloc(s.n_all, st);
    if (s.src_normals.p)
      PCLB_CUDA(cudaMemcpyAsync(tmpn.p, s.src_normals.p, s.n_all * sizeof(float4), cudaMemcpyDeviceToDevice, st));
    else  // normals that live in the records, not staged by set_source
      load_vec3_as_float4(c, s.src_raw.p + s.src_normal_off, s.n_all, s.src_stride, tmpn.p, st);
  }
  {
    ProfScope ps(c, "transform_out");
    if (b.B) {
      k_transform_batch<<<persistent_blocks(c, s.n_all), 256, 0, st>>>(tmp.p, s.n_all, b.d_offsets.p, b.B, finals.p,
                                                                       do_n ? tmpn.p : nullptr);
      ++c.launches;
    }
    else
      transform_on_device(c, s.loop.final_T, mode, tmp.p, s.n_all, do_n ? tmpn.p : nullptr);
  }
  auto write_back = [&](const DevBuf<float4>& d, void* out, size_t stride, int write_w, float w) {
    if (stride == 16 && write_w) {
      PCLB_CUDA(cudaMemcpyAsync(out, d.p, s.n_all * 16, is_device_ptr(out) ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
      return;
    }
    if (is_device_ptr(out)) {
      k_scatter_xyz<<<grid_for(s.n_all, 256), 256, 0, st>>>(d.p, s.n_all, (unsigned char*)out, stride, write_w, w);
      ++c.launches;
    }
    else {
      // host strided output: only x,y,z (and w) of each record may be touched
      std::vector<float4> hbuf(s.n_all);
      PCLB_CUDA(cudaMemcpyAsync(hbuf.data(), d.p, s.n_all * 16, cudaMemcpyDeviceToHost, st));
      PCLB_CUDA(cudaStreamSynchronize(st));
      unsigned char* o = static_cast<unsigned char*>(out);
      for (size_t i = 0; i < s.n_all; ++i) {
        float* f = reinterpret_cast<float*>(o + i * stride);
        f[0] = hbuf[i].x; f[1] = hbuf[i].y; f[2] = hbuf[i].z;
        if (write_w)
          f[3] = w;
      }
    }
  };
  // src_all keeps the caller's w (PointXYZ: 1.0 after align(), registration.hpp:213-216)
  write_back(tmp, out_pts, stride_out, stride_out >= 16 ? 1 : 0, 1.0f);
  if (do_n)
    write_back(tmpn, out_normals, stride_n, 0, 0.f);
  PCLB_CUDA(cudaStreamSynchronize(st));
}

// ---- stand-alone estimators ----------------------------------------------------------------------------------
void estimate_pairs(Ctx& c, int est, const void* src, size_t stride_s, const void* tgt, const void* tgt_normals,
                    size_t stride_t, const pclb200_corr* corr, size_t n, int scalar_is_double, double* T_out,
                    const void* src_normals, int enforce_same_dir, int svd_correlation)
{
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(src && tgt && n > 0, PCLB200_ERR_INVALID, "estimate: empty input");
  // the caller's arrays are indexed by corr[].index_*; without their sizes we need the max index
  size_t n_src = n, n_tgt = n;
  DevBuf<pclb200_corr> staged_corr;
  const pclb200_corr* d_corr = on_device(c, corr, n, staged_corr);
  if (corr) {
    std::vector<pclb200_corr> hc;
    const pclb200_corr* hcorr = corr;
    if (d_corr == corr) {  // the caller's list is in device memory: scan a host copy
      hc.resize(n);
      PCLB_CUDA(cudaMemcpy(hc.data(), corr, n * sizeof(pclb200_corr), cudaMemcpyDeviceToHost));
      hcorr = hc.data();
    }
    int mq = 0, mm = 0;
    for (size_t i = 0; i < n; ++i) {
      PCLB_REQUIRE(hcorr[i].index_query >= 0 && hcorr[i].index_match >= 0, PCLB200_ERR_INVALID, "negative index");
      mq = std::max(mq, hcorr[i].index_query);
      mm = std::max(mm, hcorr[i].index_match);
    }
    n_src = (size_t)mq + 1;
    n_tgt = (size_t)mm + 1;
    PCLB_CUDA(cudaStreamSynchronize(st));
  }
  DevBuf<float4> ds, dt, dn;
  ds.alloc(n_src, st);
  dt.alloc(n_tgt, st);
  load_xyz_as_float4(c, src, n_src, stride_s, nullptr, 0, ds.p, st);
  load_xyz_as_float4(c, tgt, n_tgt, stride_t, nullptr, 0, dt.p, st);
  DevBuf<float4> dsn;
  if (est != PCLB200_EST_SVD) {
    PCLB_REQUIRE(tgt_normals, PCLB200_ERR_INVALID, "point-to-plane needs target normals");
    dn.alloc(n_tgt, st);
    load_vec3_as_float4(c, tgt_normals, n_tgt, stride_t, dn.p, st);
  }
  if (est == PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS) {
    PCLB_REQUIRE(src_normals, PCLB200_ERR_INVALID, "the symmetric objective needs source normals");
    dsn.alloc(n_src, st);
    load_vec3_as_float4(c, src_normals, n_src, stride_s, dsn.p, st);
  }
  Reducer red;
  const unsigned grid = persistent_blocks(c, n, 256, 4);
  red.init(c, grid);
  DevBuf<SolveOut> so;
  so.alloc(1, st);
  PairArgs a;
  memset(&a, 0, sizeof(a));
  a.src = ds.p;
  a.tgt = dt.p;
  a.tgt_normals = dn.p;
  a.src_normals = dsn.p;
  a.enforce_same_dir = enforce_same_dir;
  a.corr = d_corr;
  a.n = n;
  a.ox = a.oy = a.oz = 0.f;
  a.pub = red.sum();
  DevBuf<float4> origin;  // the SVD sums' origin (icp_kernels.cuh): the first pair's target point that is finite, else 0
  if (est == PCLB200_EST_SVD) {
    origin.alloc(1, st);
    PCLB_CUDA(cudaMemsetAsync(origin.p, 0, sizeof(float4), st));
    k_seed_origin<<<1, 1, 0, st>>>(dt.p, d_corr, n, &origin.p->x);
    float4 o;
    PCLB_CUDA(cudaMemcpyAsync(&o, origin.p, sizeof(float4), cudaMemcpyDeviceToHost, st));
    PCLB_CUDA(cudaStreamSynchronize(st));
    a.ox = o.x; a.oy = o.y; a.oz = o.z;
    k_accum_pairs<PCLB200_EST_SVD><<<grid, 256, 0, st>>>(a);
    ++c.launches;
  }
  else if (est == PCLB200_EST_POINT_TO_PLANE_LLS)
    k_accum_pairs<PCLB200_EST_POINT_TO_PLANE_LLS><<<grid, 256, 0, st>>>(a);
  else
    k_accum_pairs<PCLB200_EST_SYMMETRIC_POINT_TO_PLANE_LLS><<<grid, 256, 0, st>>>(a);
  k_solve<<<1, 32, 0, st>>>(red.accum.p, est, scalar_is_double, kApplyIcp, origin.p ? &origin.p->x : nullptr, 1,
                            nullptr, so.p, svd_correlation, nullptr, CritParams{});
  c.launches += 2;
  SolveOut h;
  PCLB_CUDA(cudaMemcpyAsync(&h, so.p, sizeof(h), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < 16; ++i)
    T_out[i] = h.T[i];
}

// ---- correspondences (materialised) -----------------------------------------------------------------------------
size_t correspondences(Ctx& c, const Index& tgt, const Index* src_index, const void* src, size_t n, size_t stride,
                       const int32_t* indices, size_t n_idx, int is_dense, double max_dist, pclb200_corr* out,
                       const double* pre_T, int pre_mode, const float* gate_override)
{
  (void)is_dense;  // non-finite source points never produce a correspondence on either setting
  cudaStream_t st = c.stream;
  const size_t nq = indices ? n_idx : n;
  if (nq == 0)
    return 0;
  DevBuf<float4> dense;
  dense.alloc(nq, st);
  load_xyz_as_float4(c, src, n, stride, indices, n_idx, dense.p, st);
  if (pre_T)  // the caller's cloud is searched after a rigid transform (consumers that validate a pose)
    transform_on_device(c, pre_T, pre_mode, dense.p, nq, nullptr);
  DevBuf<int32_t> staged_ind;
  const int32_t* d_ind = on_device(c, indices, n_idx, staged_ind);
  QueryBatch qb;
  make_query_batch(c, tgt, dense.p, nq, qb);
  DevBuf<pclb200_corr> by_slot;
  by_slot.alloc(nq, st);
  const float gate = gate_override ? *gate_override : gate_from_max_dist(max_dist);
  if (src_index)
    k_corr<true><<<grid_for(nq, 128), 128, 0, st>>>(tree_view(tgt), qb.q.p, nq, gate,
                                                   src_index->nodes.p, src_index->pts.p, src_index->root, d_ind,
                                                   by_slot.p, c.d_error);
  else
    k_corr<false><<<grid_for(nq, 128), 128, 0, st>>>(tree_view(tgt), qb.q.p, nq, gate, nullptr,
                                                    nullptr, 0, d_ind, by_slot.p, c.d_error);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  const size_t m = compact_corr_to(c, by_slot.p, nq, out);
  check_device_error(c);
  return m;
}

// ---- fitness score ------------------------------------------------------------------------------------------------
double fitness_score(Ctx& c, const Index& tgt, const void* src, size_t n, size_t stride, const int32_t* indices,
                     size_t n_idx, const double* T, int scalar_is_double, double max_range, int mode_override)
{
  cudaStream_t st = c.stream;
  // registration.hpp:141-144: the index subset is used only when it is a strict subset
  const bool use_sub = indices && n_idx != n;
  const size_t nq = use_sub ? n_idx : n;
  if (!nq)
    return std::numeric_limits<double>::max();
  DevBuf<float4> dense;
  dense.alloc(nq, st);
  load_xyz_as_float4(c, src, n, stride, use_sub ? indices : nullptr, use_sub ? n_idx : 0, dense.p, st);
  // default: pcl::transformPointCloud
  const int mode = mode_override >= 0 ? mode_override : (scalar_is_double ? kApplyTransformsDouble : kApplyTransformsFloat);
  transform_on_device(c, T, mode, dense.p, nq, nullptr);
  QueryBatch qb;
  make_query_batch(c, tgt, dense.p, nq, qb);
  Reducer red;
  const unsigned grid = persistent_blocks(c, nq);
  red.init(c, grid);
  k_fitness<<<grid, 256, 0, st>>>(tree_view(tgt), qb.q.p, nq, max_range, red.sum(), c.d_error);
  ++c.launches;
  double acc[2];
  PCLB_CUDA(cudaMemcpyAsync(acc, red.accum.p, sizeof(acc), cudaMemcpyDeviceToHost, st));
  check_device_error(c);
  return acc[0] > 0 ? acc[1] / acc[0] : std::numeric_limits<double>::max();
}

// fitness_score of B problems at once (DESIGN.md §3): problem p = the dense points pts[off[p], off[p+1]) (device; moved
// in place) under transforms[16p..16p+16) in the operation order `mode`, scored against tgt[p].  gtab: batch_blocks's
// table of the grid fitness_score launches for each problem alone, `slots` its blocks.  The queries of each problem reach
// k_fitness_batch in make_query_batch's order for that problem alone and its sums run over its own grid, so scores[p] is
// fitness_score's value bit for bit.  Every stage is one launch for the whole batch; the sums come back in one copy, and
// the stream synchronises once.
static void fitness_batch(Ctx& c, const Index* const* tgt, int B, float4* pts, size_t n, const long long* d_offsets,
                          const DevBuf<BatchBlock>& gtab, unsigned slots, const double* transforms, int mode,
                          double max_range, double* scores)
{
  cudaStream_t st = c.stream;
  std::vector<Pending> h(B);
  std::vector<float4> frames(B);
  std::vector<TreeView> trees(B);
  for (int p = 0; p < B; ++p) {
    h[p] = make_pending(transforms + 16 * (size_t)p, mode, 1);
    frames[p] = make_float4(tgt[p]->lo[0], tgt[p]->lo[1], tgt[p]->lo[2], tgt[p]->morton_scale);
    trees[p] = tree_view(*tgt[p]);
  }
  DevBuf<Pending> pending;
  DevBuf<float4> d_frames;
  DevBuf<TreeView> d_trees;
  pending.alloc(B, st);
  d_frames.alloc(B, st);
  d_trees.alloc(B, st);
  PCLB_CUDA(cudaMemcpyAsync(pending.p, h.data(), B * sizeof(Pending), cudaMemcpyHostToDevice, st));
  PCLB_CUDA(cudaMemcpyAsync(d_frames.p, frames.data(), B * sizeof(float4), cudaMemcpyHostToDevice, st));
  PCLB_CUDA(cudaMemcpyAsync(d_trees.p, trees.data(), B * sizeof(TreeView), cudaMemcpyHostToDevice, st));
  k_transform_batch<<<persistent_blocks(c, n), 256, 0, st>>>(pts, n, d_offsets, B, pending.p, nullptr);
  ++c.launches;
  QueryBatch qb;
  {
    ProfScope ps(c, "query_sort");
    make_query_batch_framed(c, d_frames.p, d_offsets, B, pts, n, qb);
    sort_by_problem(c, d_offsets, B, qb);
  }
  DevBuf<double> partials, accum;
  DevBuf<unsigned> counter;
  partials.alloc((size_t)slots * kAccum, st);
  accum.alloc((size_t)B * kAccum, st);
  counter.alloc(B, st);
  PCLB_CUDA(cudaMemsetAsync(counter.p, 0, B * sizeof(unsigned), st));
  {
    ProfScope ps(c, "fitness_batch");
    k_fitness_batch<<<(unsigned)gtab.n, 256, 0, st>>>(gtab.p, d_trees.p, qb.q.p, max_range,
                                                      GridSum{partials.p, counter.p, accum.p}, c.d_error);
    ++c.launches;
  }
  PCLB_CUDA(cudaGetLastError());
  std::vector<double> acc(2 * (size_t)B);
  PCLB_CUDA(cudaMemcpy2DAsync(acc.data(), 2 * sizeof(double), accum.p, kAccum * sizeof(double), 2 * sizeof(double), B,
                              cudaMemcpyDeviceToHost, st));
  check_device_error(c);
  for (int p = 0; p < B; ++p)
    scores[p] = acc[2 * p] > 0 ? acc[2 * p + 1] / acc[2 * p] : std::numeric_limits<double>::max();
}

// pclb200_fitness_score_batch / pclb200_validate_transformation_batch (mode: the single call's operation order), after the
// C boundary has checked the arguments
void fitness_score_batch(Ctx& c, const Index* const* tgt, int B, const void* src, size_t n, size_t stride,
                         const int64_t* offsets, const double* transforms, int mode, double max_range, double* scores)
{
  cudaStream_t st = c.stream;
  const std::vector<long long> off(offsets, offsets + B + 1);
  DevBuf<long long> d_offsets;
  d_offsets.alloc(B + 1, st);
  PCLB_CUDA(cudaMemcpyAsync(d_offsets.p, off.data(), (B + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
  DevBuf<BatchBlock> gtab;
  unsigned slots = 0;
  batch_table(c, off, [&](size_t m) { return persistent_blocks(c, m); }, gtab, &slots);
  DevBuf<float4> dense;
  dense.alloc(n, st);
  load_xyz_as_float4(c, src, n, stride, nullptr, 0, dense.p, st);
  fitness_batch(c, tgt, B, dense.p, n, d_offsets.p, gtab, slots, transforms, mode, max_range, scores);
}

// getFitnessScore(max_range) of every problem of a batch session under its current final transform, on scratch of its
// own: the loop state, the matches and `cur` stay as they were
void icp_fitness_score_batch(Icp& s, double max_range, double* scores)
{
  Ctx& c = *s.ctx;
  cudaStream_t st = c.stream;
  const IcpBatch& b = s.batch;
  const int B = b.B;
  PCLB_REQUIRE(B > 0, PCLB200_ERR_INVALID, "icp: fitness_score_batch needs a batch source (set_source_batch)");
  std::vector<const Index*> tgt(B, s.tgt);
  if (s.targets.B)
    tgt = s.targets.idx;
  std::vector<double> T(16 * (size_t)B);
  for (int p = 0; p < B; ++p)
    std::copy(b.loop[p].final_T, b.loop[p].final_T + 16, T.begin() + 16 * (size_t)p);
  DevBuf<float4> pts;
  pts.alloc(s.n_all, st);
  PCLB_CUDA(cudaMemcpyAsync(pts.p, s.src_all.p, s.n_all * sizeof(float4), cudaMemcpyDeviceToDevice, st));
  fitness_batch(c, tgt.data(), B, pts.p, s.n_all, b.d_offsets.p, b.gtab, b.g_blocks, T.data(),
                s.P.scalar_is_double ? kApplyTransformsDouble : kApplyTransformsFloat, max_range, scores);
}

// Collective getFitnessScore over a map sharded across ranks (every rank passes its tile and the same source): the
// tile's nearest key of every query by slot, the minimum over the ranks (the peer-mapped tables after a barrier, or an
// NCCL min reduction), then fitness_score's count and sum over the winners in slot order — the same value on every rank.
// mode_override as in fitness_score (validateTransformation's order); fault: this rank's refusal (require_same_count).
double fitness_score_sharded(Ctx& c, const Index* tile, const void* src, size_t n, size_t stride, const int32_t* indices,
                             size_t n_idx, const double* T, int scalar_is_double, double max_range, int mode_override,
                             const char* fault)
{
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID,
               "fitness_score_sharded needs an active communicator (pclb200_comm_init or pclb200_comm_export / _import)");
  if (!fault && !tile->labelled)
    fault = "fitness_score_sharded: every rank's tile must be built with pclb200_index_build_ids";
  const bool use_sub = indices && n_idx != n;
  const size_t nq = use_sub ? n_idx : n;
  require_same_count(c, nq, "fitness_score_sharded: every rank must pass the same source", fault);
  if (!nq)
    return std::numeric_limits<double>::max();
  DevBuf<float4> dense;
  dense.alloc(nq, st);
  load_xyz_as_float4(c, src, n, stride, use_sub ? indices : nullptr, use_sub ? n_idx : 0, dense.p, st);
  const int mode = mode_override >= 0 ? mode_override : (scalar_is_double ? kApplyTransformsDouble : kApplyTransformsFloat);
  transform_on_device(c, T, mode, dense.p, nq, nullptr);
  QueryBatch qb;
  make_query_batch(c, *tile, dense.p, nq, qb);
  const PeerTables t = comm_scratch_tables(c, nq);
  const unsigned grid = persistent_blocks(c, nq);
  k_tile_keys<false><<<grid, 256, 0, st>>>(tree_view(*tile), qb.q.p, nq, std::numeric_limits<float>::infinity(), nullptr,
                                           nullptr, 0, nullptr, t.local, nullptr, c.d_error);
  ++c.launches;
  comm_tables_publish(c, t, kU64Min);
  Reducer red;
  red.init(c, grid);
  k_fitness_reduce<<<grid, 256, 0, st>>>(peer_table_set(t), nq, max_range, red.sum());
  ++c.launches;
  comm_tables_release(c, t);  // no rank rewrites its table (the next call) while a peer may still read it
  PCLB_CUDA(cudaGetLastError());
  double acc[2];
  PCLB_CUDA(cudaMemcpyAsync(acc, red.accum.p, sizeof(acc), cudaMemcpyDeviceToHost, st));
  check_device_error(c);
  return acc[0] > 0 ? acc[1] / acc[0] : std::numeric_limits<double>::max();
}

// the flagged rows of rows[0..n) in order (m of them) to the caller's host or device array of float4 rows
static void compact_rows_to(Ctx& c, const float4* rows, const unsigned char* flag, size_t n, size_t m, float* out)
{
  cudaStream_t st = c.stream;
  if (!m)
    return;
  DevBuf<float4> tmp;
  float4* d_out = out_on_device(c, reinterpret_cast<float4*>(out), m, tmp);
  DevBuf<int> count;
  count.alloc(1, st);
  size_t tmp_bytes = 0;
  PCLB_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp_bytes, rows, flag, d_out, count.p, (int)n, st));
  DevBuf<unsigned char> scratch;
  scratch.alloc(tmp_bytes, st);
  PCLB_CUDA(cub::DeviceSelect::Flagged(scratch.p, tmp_bytes, rows, flag, d_out, count.p, (int)n, st));
  c.launches += 2;
  copy_out(c, reinterpret_cast<float4*>(out), tmp, m);
}

// a labelled tile's ids by position (padding: kSentinelIndex) and the positions, for the sort of
// correspondences_normals_sharded
__global__ void k_tile_ids_pos(const float4* __restrict__ pts, size_t n, unsigned* __restrict__ ids, int* __restrict__ pos)
{
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n)
    return;
  ids[j] = (unsigned)__float_as_int(pts[j].w);
  pos[j] = (int)j;
}

// The record rows of a sharded list: the tile matches match[0..nq) (by slot) -> the winners' points (and normals, when
// with_normals: tile_nrm by position) through exchange_shard_records, as k_corr_rows's rows and flags by slot.  The scratch
// table is drawn at table_words (>= shard_record_words), the size of the call's other exchanges, so it stays mapped.
static void records_of_matches(Ctx& c, const Index* tile, const float4* tile_nrm, bool with_normals, const Match* match,
                               const pclb200_corr* by_slot, size_t nq, bool with_pts, size_t table_words,
                               DevBuf<float4>& row_pts, DevBuf<float4>& row_nrm, DevBuf<unsigned char>& flag)
{
  cudaStream_t st = c.stream;
  ProfScope ps(c, "shard_corr_records");
  DevBuf<float4> gpts, gnrm;
  DevBuf<Match> gmatch;
  if (with_normals) {
    gnrm.alloc(nq, st);
    row_nrm.alloc(nq, st);
  }
  gmatch.alloc(nq, st);
  gpts.alloc(nq, st);
  exchange_shard_records(c, comm_scratch_tables(c, table_words), match, nq, tile->pts.p,
                         with_normals ? tile_nrm : nullptr, nullptr, gmatch.p, gpts.p, gnrm.p);
  if (with_pts)
    row_pts.alloc(nq, st);
  flag.alloc(nq, st);
  k_corr_rows<<<grid_for(nq, 256), 256, 0, st>>>(by_slot, gpts.p, gnrm.p, nq, row_pts.p, row_nrm.p, flag.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

// Collective correspondences() over a map sharded across ranks// Collective correspondences() over a map sharded across ranks (every rank passes its tile and the same whole source):
// per slot this tile's key within the gate (and, reciprocal, the key again where the tile point's reverse search onto the
// source returns the query), the minimum over the ranks through the scratch tables, then correspondences()'s list, the
// same on every rank.  out_xyz1 / out_normals (nullable): the matched map point {x, y, z, 1} and its normal {nx, ny, nz, 0}
// per output correspondence, moved by the record exchange of the ICP session (exchange_shard_records); tgt_normals has
// one record per record of the tile.  pre_T / pre_mode / gate_override as in correspondences() (inliers).  fault: this
// rank's refusal of its arguments, agreed on by every rank before any exchange (require_same_count).
size_t correspondences_sharded(Ctx& c, const Index* tile, const Index* src_index, const void* src, size_t n, size_t stride,
                               const int32_t* indices, size_t n_idx, double max_dist, const void* tgt_normals,
                               size_t stride_tn, pclb200_corr* out, float* out_xyz1, float* out_normals, const char* fault,
                               const double* pre_T, int pre_mode, const float* gate_override)
{
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID,
               "correspondences_sharded needs an active communicator (pclb200_comm_init or pclb200_comm_export / _import)");
  if (!fault && !tile->labelled)
    fault = "correspondences_sharded: every rank's tile must be built with pclb200_index_build_ids";
  if (!fault && src_index && src_index->labelled)
    fault = "correspondences_sharded: the source index of reciprocal correspondences must be built without ids";
  if (!fault && out_normals && !tgt_normals)
    fault = "correspondences_sharded: out_normals needs tgt_normals";
  for (const float* o : {out_xyz1, out_normals})
    if (!fault && o && is_device_ptr(o) && reinterpret_cast<uintptr_t>(o) % 16)
      fault = "correspondences_sharded: device rows out_xyz1 / out_normals must be 16-byte aligned";
  const bool recip = src_index != nullptr, rows = out_xyz1 || out_normals;
  const size_t nq = indices ? n_idx : n;
  // the count and the variant (reciprocal, records, normals): every rank must lay its tables out alike
  require_same_count(c, (unsigned long long)nq << 3 | (recip ? 1 : 0) | (rows ? 2 : 0) | (out_normals ? 4 : 0),
                     "correspondences_sharded: every rank must pass the same whole source, reciprocal or not, and ask "
                     "for the same record rows",
                     fault);
  if (nq == 0)
    return 0;
  DevBuf<float4> dense;
  dense.alloc(nq, st);
  load_xyz_as_float4(c, src, n, stride, indices, n_idx, dense.p, st);
  if (pre_T)
    transform_on_device(c, pre_T, pre_mode, dense.p, nq, nullptr);
  DevBuf<int32_t> staged_ind;
  const int32_t* d_ind = on_device(c, indices, n_idx, staged_ind);
  QueryBatch qb;
  make_query_batch(c, *tile, dense.p, nq, qb);
  const float gate = gate_override ? *gate_override : gate_from_max_dist(max_dist);
  // one scratch size for the key and the record exchange keeps the table mapped across both (and across calls)
  const size_t words = std::max(recip ? 2 * nq : nq, rows ? shard_record_words(nq, out_normals != nullptr) : 0);
  DevBuf<Match> match;
  if (rows)
    match.alloc(nq, st);
  DevBuf<pclb200_corr> by_slot;
  by_slot.alloc(nq, st);
  {
    ProfScope ps(c, "shard_corr_keys");
    PeerTables t = comm_scratch_tables(c, words);
    t.words = recip ? 2 * nq : nq;  // the NCCL reduction moves the keys only
    const unsigned grid = persistent_blocks(c, nq);
    if (recip)
      k_tile_keys<true><<<grid, 256, 0, st>>>(tree_view(*tile), qb.q.p, nq, gate, src_index->nodes.p, src_index->pts.p,
                                              src_index->root, d_ind, t.local, match.p, c.d_error);
    else
      k_tile_keys<false><<<grid, 256, 0, st>>>(tree_view(*tile), qb.q.p, nq, gate, nullptr, nullptr, 0, nullptr, t.local,
                                               match.p, c.d_error);
    ++c.launches;
    comm_tables_publish(c, t, kU64Min);
    k_keys_to_corr<<<grid_for(nq, 256), 256, 0, st>>>(peer_table_set(t), nq, recip ? 1 : 0, d_ind, by_slot.p);
    ++c.launches;
    comm_tables_release(c, t);
    PCLB_CUDA(cudaGetLastError());
  }
  DevBuf<float4> row_pts, row_nrm;
  DevBuf<unsigned char> flag;
  if (rows) {
    DevBuf<float4> tile_nrm;
    if (out_normals)
      normals_by_pos(c, tile, tgt_normals, stride_tn, tile_nrm);
    records_of_matches(c, tile, tile_nrm.p, out_normals != nullptr, match.p, by_slot.p, nq, out_xyz1 != nullptr, words,
                       row_pts, row_nrm, flag);
  }
  const size_t m = compact_corr_to(c, by_slot.p, nq, out);
  if (out_xyz1)
    compact_rows_to(c, row_pts.p, flag.p, nq, m, out_xyz1);
  if (out_normals)
    compact_rows_to(c, row_nrm.p, flag.p, nq, m, out_normals);
  check_device_error(c);
  PCLB_CUDA(cudaStreamSynchronize(st));
  return m;
}

int comm_nranks(const Ctx& c);  // comm.cu

// Collective correspondences_by_normals over a map sharded across ranks (normal shooting / back projection; the layout
// of correspondences_sharded).  keff is the whole map's clamp.  Each rank's k-NN rows of its tile, as keys, travel through
// the segment tables (peer path: read in place; NCCL: all-gathered), every rank merges the R rows of each query into the
// whole map's row (shard_target_kernels.cuh), scores the merged candidates its tile holds and publishes the scores'
// bit patterns (~0 elsewhere) for one u64 minimum, and runs select_by_normals's choice on the result.  The tile's ids are
// sorted once per call to find a candidate's position.  Resident per rank at the peak: its rows (nq keff 8 B), the other
// ranks' rows under NCCL ((R - 1) nq keff 8 B), the merged row and the scores (2 nq keff 8 B).
size_t correspondences_normals_sharded(Ctx& c, const Index* tile, int kind, const void* src, size_t n, size_t stride,
                                       const void* src_normals, size_t stride_sn, const void* tgt_normals,
                                       size_t stride_tn, const int32_t* indices, size_t n_idx, int k, double max_dist,
                                       pclb200_corr* out, float* out_xyz1, float* out_normals, const char* fault)
{
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID,
               "correspondences_normals_sharded needs an active communicator (pclb200_comm_init or pclb200_comm_export / "
               "_import)");
  if (!fault && !tile->labelled)
    fault = "correspondences_normals_sharded: every rank's tile must be built with pclb200_index_build_ids";
  for (const float* o : {out_xyz1, out_normals})
    if (!fault && o && is_device_ptr(o) && reinterpret_cast<uintptr_t>(o) % 16)
      fault = "correspondences_normals_sharded: device rows out_xyz1 / out_normals must be 16-byte aligned";
  const bool rows = out_xyz1 || out_normals;
  const size_t nq = indices ? n_idx : n;
  const int R = comm_nranks(c);
  // the count, the kind, k and the rows asked for: every rank must lay its tables out alike
  require_same_count(c, ((((unsigned long long)nq << 2 | (unsigned)kind) << 1 | (rows ? 1 : 0)) << 1 |
                         (out_normals ? 1 : 0)) << 32 | (unsigned)k,
                     "correspondences_normals_sharded: every rank must pass the same whole source, kind and k, and ask "
                     "for the same record rows",
                     fault);
  if (nq == 0 || k == 0)
    return 0;
  const int keff = sharded_keff(c, *tile, k);
  if (keff <= 0)
    return 0;
  const size_t nk = nq * (size_t)keff;
  DevBuf<float4> dense, sn, tile_nrm;
  QueryBatch qb = load_queries(c, *tile, src, n, stride, indices, n_idx, dense);
  sn.alloc(n, st);
  load_vec3_as_float4(c, src_normals, n, stride_sn, sn.p, st);
  if (tgt_normals)
    normals_by_pos(c, tile, tgt_normals, stride_tn, tile_nrm);
  DevBuf<int32_t> staged_ind;
  const int32_t* d_ind = on_device(c, indices, n_idx, staged_ind);
  // the tile's ids sorted, with their positions (padding sorts last under kSentinelIndex)
  const size_t np = tile->pts.n;
  DevBuf<unsigned> ids_in, sid;
  DevBuf<int> pos_in, spos;
  ids_in.alloc(np, st);
  pos_in.alloc(np, st);
  sid.alloc(np, st);
  spos.alloc(np, st);
  k_tile_ids_pos<<<grid_for(np, 256), 256, 0, st>>>(tile->pts.p, np, ids_in.p, pos_in.p);
  ++c.launches;
  {
    size_t tb = 0;
    PCLB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, ids_in.p, sid.p, pos_in.p, spos.p, (int)np, 0, 32, st));
    DevBuf<unsigned char> tmp;
    tmp.alloc(tb, st);
    PCLB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, ids_in.p, sid.p, pos_in.p, spos.p, (int)np, 0, 32, st));
    c.launches += 2;
  }
  DevBuf<unsigned long long> merged;
  merged.alloc(nk, st);
  {
    ProfScope ps(c, "shard_corr_knn");
    DevBuf<int32_t> nn_idx;
    DevBuf<float> nn_d2;
    nn_idx.alloc(nk, st);
    nn_d2.alloc(nk, st);
    launch_knn(c, *tile, qb.q.p, nq, keff, std::numeric_limits<float>::infinity(), nn_idx.p, nn_d2.p);
    std::vector<unsigned long long> cnt(R, (unsigned long long)nk);
    const PeerTables t = comm_segment_tables(c, cnt.data(), sizeof(unsigned long long));
    k_knn_keys<<<persistent_blocks(c, nk), 256, 0, st>>>(nn_idx.p, nn_d2.p, nk, t.local);
    ++c.launches;
    comm_tables_publish(c, t, kU64Sum);  // NCCL: the tables lie end to end in one zeroed table, one writer per word
    k_merge_rows<<<grid_for(nq, 256), 256, 0, st>>>(peer_table_set(t), nq, keff, merged.p);
    ++c.launches;
    comm_tables_release(c, t);
    PCLB_CUDA(cudaGetLastError());
  }
  DevBuf<pclb200_corr> by_slot;
  by_slot.alloc(nq, st);
  DevBuf<Match> match;
  if (rows)
    match.alloc(nq, st);
  {
    ProfScope ps(c, "shard_corr_select");
    PeerTables t = comm_scratch_tables(c, rows ? std::max(nk, shard_record_words(nq, out_normals != nullptr)) : nk);
    t.words = nk;
    k_candidate_scores<<<grid_for(nq, 256), 256, 0, st>>>(merged.p, nq, keff, kind, dense.p, d_ind, sn.p, sid.p, spos.p,
                                                           np, tile->pts.p, tile_nrm.p, t.local);
    ++c.launches;
    comm_tables_publish(c, t, kU64Min);
    k_select_sharded<<<grid_for(nq, 256), 256, 0, st>>>(merged.p, peer_table_set(t), nq, keff, kind, dense.p, d_ind,
                                                         max_dist, sid.p, spos.p, np, by_slot.p, match.p);
    ++c.launches;
    comm_tables_release(c, t);
    PCLB_CUDA(cudaGetLastError());
  }
  DevBuf<float4> row_pts, row_nrm;
  DevBuf<unsigned char> flag;
  if (rows)
    records_of_matches(c, tile, tile_nrm.p, out_normals != nullptr, match.p, by_slot.p, nq, out_xyz1 != nullptr,
                       std::max(nk, shard_record_words(nq, out_normals != nullptr)), row_pts, row_nrm, flag);
  const size_t m = compact_corr_to(c, by_slot.p, nq, out);
  if (out_xyz1)
    compact_rows_to(c, row_pts.p, flag.p, nq, m, out_xyz1);
  if (out_normals)
    compact_rows_to(c, row_nrm.p, flag.p, nq, m, out_normals);
  check_device_error(c);
  PCLB_CUDA(cudaStreamSynchronize(st));
  return m;
}

}  // namespace pclb200
