// internal.cuh — shared declarations of libpclb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/pclb200.h"
#include "../../include/pclb200_sharded.h"

namespace pclb200 {

// ---------------------------------------------------------------------------------------------
// errors: C++ exceptions inside the library, converted to status codes at the C boundary
// ---------------------------------------------------------------------------------------------
struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define PCLB_CUDA(expr)                                                                         \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess)                                                                      \
      throw ::pclb200::Error(PCLB200_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e) + \
                                                   " (" + __FILE__ + ":" + std::to_string(__LINE__) + ")"); \
  } while (0)

#define PCLB_REQUIRE(cond, code, msg)                 \
  do {                                                \
    if (!(cond))                                      \
      throw ::pclb200::Error((code), (msg));          \
  } while (0)

// ---------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------
struct Comm;  // NCCL wrapper (comm.cu)

struct ProfEvent {
  const char* name;
  cudaEvent_t a, b;
};

struct Ctx {
  std::recursive_mutex mu;           // every C-ABI entry point holds it: calls on one ctx serialise (PCL's query
                                     // methods are const and may be called from several OpenMP threads)
  int device = 0;
  bool profiling = false;            // pclb200_profile_enable: CUDA-event pairs around the named kernels
  std::vector<ProfEvent> prof;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  uint64_t launches = 0;  // kernels launched by this library (incl. CUB passes, counted per call)
  void* pinned = nullptr; // small pinned staging block for per-iteration read-backs
  size_t pinned_bytes = 0;
  int* d_error = nullptr; // device-side error flag: 0 or one of kErr*
  Comm* comm = nullptr;
};

// values a kernel stores into *Ctx::d_error
enum { kErrStackOverflow = 1, kErrPeerTimeout = 2 };
// the Error a non-zero device error flag stands for; clears the flag (on the ctx stream) and throws it
[[noreturn]] void raise_device_error(Ctx& c, int code);
// synchronises the ctx stream, then raise_device_error if a kernel set the flag
void check_device_error(Ctx& c);

// records a CUDA-event pair around a region of the ctx stream when profiling is on
struct ProfScope {
  Ctx& c;
  cudaEvent_t b = nullptr;
  ProfScope(Ctx& ctx, const char* name) : c(ctx)
  {
    if (!c.profiling)
      return;
    ProfEvent e{name, nullptr, nullptr};
    if (cudaEventCreate(&e.a) != cudaSuccess || cudaEventCreate(&e.b) != cudaSuccess)
      return;
    cudaEventRecord(e.a, c.stream);
    b = e.b;
    c.prof.push_back(e);
  }
  ~ProfScope()
  {
    if (b)
      cudaEventRecord(b, c.stream);
  }
};

// Device memory comes from a small per-stream block cache (alloc.cu): after the first align() every request is
// served from blocks the previous call returned, so the steady-state loop never enters the driver's allocator
// (cudaMallocAsync pool growth showed up as multi-millisecond host stalls between launches on shared boxes).
// Re-use is safe without events because a ctx issues all its work on ONE stream: a block handed out again is
// only touched by work enqueued after the work that used it before.
void* cached_alloc(cudaStream_t s, size_t bytes);
void cached_free(cudaStream_t s, void* p);
void cached_release_all(cudaStream_t s);

// stream-ordered device buffer
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  cudaStream_t s = nullptr;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n), s(o.s) { o.p = nullptr; o.n = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept
  {
    if (this != &o) {
      release();
      p = o.p; n = o.n; s = o.s;
      o.p = nullptr; o.n = 0;
    }
    return *this;
  }
  void alloc(size_t count, cudaStream_t stream)
  {
    release();
    s = stream;
    n = count;
    if (count)
      p = static_cast<T*>(cached_alloc(stream, count * sizeof(T)));
  }
  void release()
  {
    if (p)
      cached_free(s, p);
    p = nullptr;
    n = 0;
  }
  ~DevBuf() { release(); }
  size_t bytes() const { return n * sizeof(T); }
};

bool is_device_ptr(const void* p);

#ifdef __CUDACC__
// blocks of a 1-D launch over n items.  Only the .cu drivers launch; the kernel headers compiled by g++ for the host
// tests (tests/host) bring their own launcher and grid size.
inline unsigned grid_for(size_t n, int block) { return (unsigned)((n + block - 1) / block); }
// the same for a grid-stride kernel, capped at per_sm blocks per SM (at least one block)
inline unsigned persistent_blocks(const Ctx& c, size_t n, int block = 256, int per_sm = 8)
{
  return (unsigned)std::max<size_t>(1, std::min<size_t>(grid_for(n, block), (size_t)c.sm_count * per_sm));
}
#endif

// Any caller array may live in host or device memory (DESIGN.md §1).  The kernels read an input through on_device: the
// caller's pointer when it is device memory (or null / empty), else `staging` after an upload of its first n elements
// enqueued on the ctx stream.  A strided array passes T = unsigned char and the byte count up to its last needed byte.
template <typename T>
const T* on_device(Ctx& c, const T* p, size_t n, DevBuf<T>& staging)
{
  if (!p || n == 0 || is_device_ptr(p))
    return p;
  staging.alloc(n, c.stream);
  PCLB_CUDA(cudaMemcpyAsync(staging.p, p, n * sizeof(T), cudaMemcpyHostToDevice, c.stream));
  return staging.p;
}
// The kernels write an output of n elements through out_on_device: the caller's pointer when it is device memory (or
// null), else the temporary `tmp`.  copy_out then moves the first n elements of the temporary to the caller; it does
// nothing when the kernel wrote in place.
template <typename T>
T* out_on_device(Ctx& c, T* p, size_t n, DevBuf<T>& tmp)
{
  if (!p || is_device_ptr(p))
    return p;
  tmp.alloc(n, c.stream);
  return tmp.p;
}
template <typename T>
void copy_out(Ctx& c, T* p, const DevBuf<T>& tmp, size_t n)
{
  if (tmp.p && n)
    PCLB_CUDA(cudaMemcpyAsync(p, tmp.p, n * sizeof(T), cudaMemcpyDeviceToHost, c.stream));
}
// Keeps the entries of a device correspondence list with index_match >= 0 (or those whose flag is set), in order, and
// writes them to the caller's host or device array.  Returns their number; the ctx stream has synchronised once to read
// it, and the copy to the caller is enqueued after that.
size_t compact_corr_to(Ctx& c, const pclb200_corr* d_in, size_t n, pclb200_corr* caller_out);
size_t compact_corr_to(Ctx& c, const pclb200_corr* d_in, const unsigned char* d_flags, size_t n, pclb200_corr* caller_out);

// Copies `count` records of `rec_bytes` (<= stride) from a strided host-or-device array into a
// dense device array of float4 {x,y,z,w_fill}: the layout every kernel reads with 128-bit loads.
// If `subset` != NULL, record i is src[subset[i]].
void load_xyz_as_float4(Ctx& c, const void* src, size_t n_records, size_t stride, const int32_t* subset,
                        size_t n_subset, float4* d_out, cudaStream_t s);
// same for normals (3 floats at `src`, any stride) -> float4 {nx,ny,nz,0}
void load_vec3_as_float4(Ctx& c, const void* src, size_t n_records, size_t stride, float4* d_out,
                         cudaStream_t s);

// ---------------------------------------------------------------------------------------------
// LBVH index
// ---------------------------------------------------------------------------------------------
// One internal node = 64 B = four 128-bit loads: both children's boxes + their references.
//   a = (l.min.x, l.min.y, l.min.z, l.max.x)  b = (l.max.y, l.max.z, r.min.x, r.min.y)
//   c = (r.min.z, r.max.x, r.max.y, r.max.z)  d = (left, right, 0, 0)
// child reference >= 0: internal node id; < 0: ~leaf_id.
struct __align__(16) BvhNode {
  float4 a, b, c;
  int4 d;
};

#ifndef PCLB_LEAF
#define PCLB_LEAF 8
#endif
constexpr int kLeafSize = PCLB_LEAF;  // points per leaf (multiple of 8): 8 points = one 128-byte line of float4
static_assert(kLeafSize % 8 == 0 && kLeafSize >= 8 && kLeafSize <= 64, "leaf size must be a multiple of 8");
// A walk pushes at most one entry per level.  The radix tree is at most 63 (key bits) + 31 (index tie-break bits)
// = 94 levels deep, so 96 entries can never overflow (the overflow check stays as a guard, not as an expected path).
constexpr int kStackSize = 96;      // traversal stack entries per query
constexpr int kSentinelIndex = 0x7fffffff;

// host-side description of the index's cell table (lbvh.cu builds it, traverse.cuh: CellTable reads it)
struct CellTableHost {
  unsigned log2_slots = 0;  // 0 = no table
  int bmax = 0;             // finest level present (cells of 2^-bmax of the frame per axis)
  uint64_t entries = 0;
  float margin = 0.f;
  uint64_t occupied[16] = {0};  // occupied cells per level (index = level), from the prefix-length histogram
};

struct Index {
  Ctx* ctx = nullptr;
  int device = 0;
  size_t n_cloud = 0;   // records in the caller's cloud (index space of results)
  size_t n_valid = 0;   // finite points indexed
  int n_leaves = 0;
  int root = 0;         // child-reference encoding
  float lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};  // bounding box of the valid points
  float morton_scale = 1.f;                     // 2^21 / max extent
  DevBuf<float4> pts;   // n_leaves*kLeafSize, Morton order, w = original index bits; padded with +inf
  DevBuf<BvhNode> nodes;  // n_leaves-1
  DevBuf<int32_t> pos_of_orig;  // n_cloud: position in `pts` of original index i, or -1 (lazy)
  DevBuf<int2> node_leaves;     // per internal node: {first leaf, number of leaves} — a subtree's leaves are consecutive
  DevBuf<uint2> cell_slots;     // hash table (level, cell) -> deepest node / leaf holding every point of the cell
  CellTableHost cells;          // its description (traverse.cuh: CellTable is the device-side view)
  // labelled index (build_index_ids): w = the caller's id of the point, which says nothing about its record; slot_of_pos
  // maps a position in `pts` to the caller's record (-1 for padding).  Nothing may size a table by the largest id.
  bool labelled = false;
  DevBuf<int32_t> slot_of_pos;
  size_t bytes() const
  {
    return pts.bytes() + nodes.bytes() + pos_of_orig.bytes() + cell_slots.bytes() + node_leaves.bytes() + slot_of_pos.bytes();
  }
};

Index* build_index(Ctx& c, const void* pts, size_t n, size_t stride, const int32_t* subset, size_t n_subset);
// cloud k = records [offsets[k], offsets[k + 1]) of pts (offsets: host, n_clouds + 1 entries): what build_index makes of
// each cloud alone, in one build whose every stage is one launch for the whole batch.  All or nothing: throws, with no
// handle left, on any error.
std::vector<std::unique_ptr<Index>> build_index_batch(Ctx& c, const void* pts, size_t n, size_t stride,
                                                      const int64_t* offsets, int n_clouds);
// point i labelled ids[i] (non-negative, distinct, < 2^31 - 1) instead of i: one tile of a map sharded across ranks
Index* build_index_ids(Ctx& c, const void* pts, size_t n, size_t stride, const int32_t* ids);
// the faults of the caller's ids d_ids[0..n) (device): kIdOutOfRange (outside [0, 2^31 - 2]) | kIdRepeated; synchronises
enum { kIdOutOfRange = 1, kIdRepeated = 2 };
int id_faults(Ctx& c, const int32_t* d_ids, size_t n);
// device-resident source already dense float4 (w ignored): used for the reciprocal source tree (rebuilt every iteration:
// no cell table) and for the local map of a sharded map (shard_normals.cu: with the cell table)
Index* build_index_from_device(Ctx& c, const float4* d_pts, size_t n, const int32_t* d_orig /*nullable*/,
                               bool cell_table = false);
// The local map of a map sharded across the communicator's ranks (collective, shard_normals.cu): this rank's tile
// (labelled) plus every point of the other tiles that can be a neighbour of one of the dense queries d_q[0..nq) on the
// whole map, sorted by id and indexed as an ordinary index (record i = the i-th smallest id).  k > 0: the k nearest; else
// every point within d2 <= r2 (normals: the radius neighbours; clusters: the tile's points as queries, every edge).
// stages names the ProfScopes; trace (nullable) receives what the halo exchange moved, for a caller that answers back
// along it (shard_cluster.cu).
struct ShardedMapStages {
  const char* bound;  // the k-th distance bound (k > 0)
  const char* halo;   // boxes and halo exchange
  const char* build;  // sort by id and index
};
struct HaloTrace {
  std::vector<unsigned long long> cnt;  // R x R: cnt[s R + r] = points rank s sent to rank r (s == r: its whole tile)
  DevBuf<unsigned> local_ids;           // the local map's ids by record (ascending, each once; the first n_cloud)
  DevBuf<unsigned> recv_ids;            // the received points' ids: by sender, each sender's segment in its order
  DevBuf<unsigned> sent_ids;            // the ids this rank sent: by destination, each segment in the order it wrote it
};
Index* sharded_local_map(Ctx& c, const Index& tile, const float4* d_q, size_t nq, int k, float r2,
                         const ShardedMapStages& stages, HaloTrace* trace = nullptr);
void ensure_pos_of_orig(Ctx& c, Index& idx);

// Morton-ordered batch of query points (dense float4 xyz + original slot), so neighbouring threads
// walk neighbouring subtrees.
struct QueryBatch {
  size_t n = 0;
  DevBuf<float4> q;       // n, xyz + w = original slot bits
};
void make_query_batch(Ctx& c, const Index& ref_frame, const float4* d_q /*n, w ignored*/, size_t n,
                      QueryBatch& out);
// One pass over n strided records in device memory (xyz at offset 0, stride a multiple of 4): the whole records into
// `copy` and xyz into `dense` (float4, w = the record's w when stride == 16, else 1), each nullable, and, when qb is given,
// the query batch make_query_batch would make of those points (read from `dense`, or from `recs` when dense is null and
// stride == 16) without another pass over them.
void stage_records(Ctx& c, const Index& ref_frame, const unsigned char* recs, size_t n, size_t stride, unsigned char* copy,
                   float4* dense, QueryBatch* qb);
// a batch of problems over consecutive ranges of points: the problem of point i, offsets[p] <= i < offsets[p + 1]
__host__ __device__ __forceinline__ int problem_of(const long long* offsets, int n_problems, long long i)
{
  int lo = 0, hi = n_problems - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (offsets[mid] <= i)
      lo = mid;
    else
      hi = mid - 1;
  }
  return lo;
}
// make_query_batch of the dense points d_q[0..n), each keyed in its own problem's frame (d_offsets: B + 1 entries, device;
// d_frames: B x {lo, morton_scale}, device).  The queries of one problem keep the order make_query_batch gives them in
// that problem's frame; the problems interleave until a stable sort by problem follows.
void make_query_batch_framed(Ctx& c, const float4* d_frames, const long long* d_offsets, int n_problems,
                             const float4* d_q, size_t n, QueryBatch& out);
// stably sorts the query batch qb by the problem of each query's record (w; d_offsets: B + 1 entries, device), so that the
// queries of problem p fill [offsets[p], offsets[p+1]) in the order they had
void sort_by_problem(Ctx& c, const long long* d_offsets, int n_problems, QueryBatch& qb);
// load_xyz_as_float4 of a caller's query points into `dense` (kept alive: some kernels read it in input order), then
// make_query_batch over it
QueryBatch load_queries(Ctx& c, const Index& ref_frame, const void* pts, size_t n, size_t stride, const int32_t* subset,
                        size_t n_subset, DevBuf<float4>& dense);

// ---------------------------------------------------------------------------------------------
// search / registration kernels (search.cu, icp.cu, voxel.cu)
// ---------------------------------------------------------------------------------------------
// exact k-NN for a Morton-ordered batch; results scattered to row `slot` (w of the query)
void launch_knn(Ctx& c, const Index& idx, const float4* d_q, size_t nq, int k, float init_bound,
                int32_t* d_out_idx, float* d_out_d2 /* nq*k, row = slot */);
// counts / fills for radius search: neighbours with d2 < r2
void launch_radius_count(Ctx& c, const Index& idx, const float4* d_q, size_t nq, float r2,
                         unsigned long long* d_counts /* by slot */);
void launch_radius_fill(Ctx& c, const Index& idx, const float4* d_q, size_t nq, float r2,
                        const unsigned long long* d_offsets /* by slot, exclusive */,
                        unsigned long long* d_keys /* (d2 bits << 32) | index */);

// sorted radius neighbourhoods as CSR rows of packed keys ((d2 bits << 32) | original index), addressed by query slot
void radius_count(Ctx& c, const Index& idx, const float4* d_q, size_t nq, float r2, DevBuf<unsigned long long>& counts,
                  DevBuf<unsigned long long>& offsets, unsigned long long& total);
void radius_fill_sorted(Ctx& c, const Index& idx, const float4* d_q, size_t nq, float r2,
                        const DevBuf<unsigned long long>& offsets, unsigned long long total,
                        DevBuf<unsigned long long>& keys_sorted);
void radius_csr(Ctx& c, const Index& idx, const float4* d_q, size_t nq, float r2, DevBuf<unsigned long long>& counts,
                DevBuf<unsigned long long>& offsets, DevBuf<unsigned long long>& keys_sorted, unsigned long long& total);
// radiusSearch of a caller's query batch (pclb200_radius / pclb200_radius_into).  `sink(total)` returns where the packed
// lists go (host or device pointers; {nullptr, nullptr} = do not deliver, e.g. the caller's buffers are too small);
// offsets are written to out_offsets (host or device, nq + 1 entries).
struct RadiusSinkBuffers {
  int32_t* idx;
  float* d2;
};
void radius_search(Ctx& c, const Index& idx, const void* queries, size_t nq, size_t stride, double radius, unsigned max_nn,
                   int64_t* out_offsets, const std::function<RadiusSinkBuffers(unsigned long long)>& sink);
void launch_normals(Ctx& c, Index& idx, const float4* d_q, size_t nq, int k, const float vp[3], float4* d_out,
                    int* d_not_dense);
void launch_normals_radius(Ctx& c, Index& idx, const float4* d_q, size_t nq, float r2, const float vp[3], float4* d_out,
                           int* d_not_dense);
// the k-NN normals of B query sets in one launch sequence: d_q = the queries of every set, sorted by set (set b fills
// [offsets[b], offsets[b+1]) of d_q, d_offsets on the device) and each in the order of idx[b]'s frame, w = the query's
// row in d_out; set b is searched in idx[b], flipped towards vps[3b..3b+2] (host) and flags d_flags[b] (zeroed)
void launch_normals_batch(Ctx& c, Index* const* idx, int B, const long long* d_offsets, const float4* d_q, size_t nq, int k,
                          const float* vps, float4* d_out, int* d_flags);
void launch_knn_stats(Ctx& c, const Index& idx, const float4* d_q, size_t nq, int k, float* d_mean, float* d_kth);
// launch_knn_stats's d_kth through materialised k-NN lists (nq * k entries of scratch), whatever k: the warp-cooperative
// search answers k = 12..32 on an index with a cell table, much faster than the per-thread statistics kernel
void launch_knn_kth(Ctx& c, const Index& idx, const float4* d_q, size_t nq, int k, float* d_kth);
// correspondences chosen among the k nearest with the help of normals; surface-normal rejector (normals_corr.cu)
size_t correspondences_by_normals(Ctx& c, Index& tgt, int kind, const void* src, size_t n, size_t stride,
                                  const void* src_normals, size_t stride_sn, const void* tgt_normals, size_t stride_tn,
                                  const int32_t* indices, size_t n_idx, int k, double max_dist, pclb200_corr* out);
size_t reject_surface_normal(Ctx& c, const pclb200_corr* in, size_t n, const void* src_normals, size_t n_src,
                             size_t stride_sn, const void* tgt_normals, size_t n_tgt, size_t stride_tn,
                             double threshold, pclb200_corr* out);

// The launches of the VoxelGrid kernels voxelgrid() and the VoxelGrid of a sharded map share (voxel.cu defines the kernels
// of voxel_kernels.cuh, shard_voxel.cu runs them through these).  vg_minmax: the min / max / count of k_vg_minmax over n
// dense points, synchronised.  vg_load_normals: the normal planes (k_vg_load_nc) of n records of a host-or-device array,
// or of its records indices[0..n_idx).  vg_runs: k_vg_runs.  vg_reduce: k_vg_centroids, and k_vg_normals when nc is given.
struct MinMaxAcc;
struct RunRef;
MinMaxAcc vg_minmax(Ctx& c, const float4* d_pts, size_t n);
void vg_load_normals(Ctx& c, const void* normals, size_t n, size_t stride_n, const int32_t* indices, size_t n_idx,
                     float4* d_nc);
void vg_runs(Ctx& c, const unsigned* starts, size_t n_runs, size_t n_valid, RunRef* runs);
void vg_reduce(Ctx& c, const float4* pts, const float4* nc, const int32_t* vals, const RunRef* runs, size_t n_runs,
               float4* out, float4* out_nc);
// The box and finite count of every cloud k = records [offsets[k], offsets[k + 1]) of the dense d_pts (offsets: host,
// n_clouds + 1 entries) into out[k] (host), in one launch of the batch build's k_bbox_batch (lbvh.cu) over tiles that never
// straddle a cloud; synchronised.  Its accumulator encodes the box as k_vg_minmax's does, so out[k] is what vg_minmax
// gives of cloud k alone, up to the sign of a zero, which no voxel key depends on.
void cloud_boxes(Ctx& c, const float4* d_pts, const int64_t* offsets, int n_clouds, MinMaxAcc* out);

// connected components of the d2 < tolerance^2 graph over the indexed points (cluster.cu)
void cluster_labels(Ctx& c, const Index& idx, double tolerance, int32_t* d_labels /* idx.n_cloud */);
// the same over a map sharded across the communicator's ranks (collective, shard_cluster.cu): labels and, when d_sizes is
// not null, component sizes of the tile's records (tile.n_cloud entries each, on the device)
void cluster_labels_sharded(Ctx& c, const Index& tile, double tolerance, int32_t* d_labels, int64_t* d_sizes);
// min(k, the number of distinct finite ids of a map sharded across the communicator's ranks), the same on every rank
// (collective, shard_filter.cu: the clamp of pclb200_knn_sharded)
int sharded_keff(Ctx& c, const Index& tile, int k);
// every rank's d_send[0..n) concatenated in rank order, identically on every rank (collective, comm.cu: the count
// exchange, then comm_segment_tables); returns the total
size_t allgather_u64(Ctx& c, const unsigned long long* d_send, size_t n, DevBuf<unsigned long long>& out);

// flat per-correspondence arrays the rejectors work on (reject.cu)
struct RejectArrays {
  size_t n = 0;
  const float* d2 = nullptr;      // squared distance
  const int* match = nullptr;     // index_match (any non-negative id that identifies the target point)
  const unsigned* tie = nullptr;  // position in the input list (tie-break)
  int* acc = nullptr;             // in/out: 1 = still a correspondence
};
void apply_rejector(Ctx& c, const pclb200_rejector& r, const RejectArrays& a, int* perm, int* keep_sorted, double* d_info,
                    int* trimmed_flag);

// accumulators of one ICP iteration (all fp64), see icp.cu
constexpr int kAccum = 40;

// the operation order of the reference that a rigid transform on the device reproduces (Pending::mode, icp_kernels.cuh)
enum {
  kApplyIcp = 0,               // icp.hpp:49-111, float
  kApplyTransformsFloat = 1,   // transforms.hpp, SSE float order
  kApplyTransformsDouble = 2,  // transforms.hpp, double order
  kApplyValidationDouble = 3,  // transformation_validation_euclidean.hpp:62-75 with a double matrix (left to right, cast at the end)
};

// Cross-GPU exchange block of the fused reduce (comm.cu): every rank owns one, mapped into every peer through CUDA IPC
//   flags[kMaxRanks]                  u64, the latest sequence number published by each peer
//   slots[2][kMaxRanks][kAccum]       fp64: the accumulators of one ICP iteration (accumulate kernels, icp_kernels.cuh)
//   words[2][kMaxRanks][kU64Words]    u64: sums, minima and barriers of the rejector chain on a sharded source (reject.cu)
// so a kernel on rank r stores its values straight into rank p's region[.][r][.] over NVLink.  Both regions follow one
// protocol (peer_exchange.cuh) with the same flags and one sequence counter.
constexpr int kMaxRanks = 8;
constexpr int kU64Words = 256;  // one histogram of 8-bit digits; also holds kMaxRanks IPC handles (8 words each)
constexpr size_t kPeerSlotsOffset = kMaxRanks * sizeof(unsigned long long);
constexpr size_t kPeerWordsOffset = kPeerSlotsOffset + 2ull * kMaxRanks * kAccum * sizeof(double);
constexpr size_t kPeerBlockBytes = kPeerWordsOffset + 2ull * kMaxRanks * kU64Words * sizeof(unsigned long long);
struct PeerView {
  int rank = 0;
  int nranks = 0;                       // 0 / 1 = no exchange
  unsigned long long* flags[kMaxRanks]; // flags[p] = base of rank p's block (its flag array; peer-mapped, [rank] = self)
  double* slots[kMaxRanks];             // slots[p] = base of rank p's slot array
};

// ---- cross-rank u64 collectives (comm.cu) for the rejector chain on a sharded source (reject.cu) ----------------------
enum { kU64Sum = 0, kU64Min = 1 };
// element-wise sum / min over the ranks, enqueued on the ctx stream; send == recv is allowed.  The peer-mapped path moves
// at most kU64Words words; NCCL any count.
void comm_allreduce_u64(Ctx& c, const unsigned long long* d_send, unsigned long long* d_recv, size_t count, int op);
// global position of this rank's first query (sum of n_q over the lower ranks) and the total; one exchange, synchronises
unsigned long long comm_shard_offset(Ctx& c, unsigned long long n_q, unsigned long long* total);
// Tables of u64 through which the ranks' kernels exchange whole arrays (DESIGN.md §5): the one-to-one rejector's, the
// sharded target's, and the scratch of the sharded normals, clusters and fitness.  Every exchange is: this rank's kernels
// write `local`; comm_tables_publish; kernels read the tables (peer_tables.cuh: peer_table_set, segment_reads);
// comm_tables_release.
//   peer path  every rank's own table, mapped into every rank: read[s] = rank s's.  Publish and release are barriers, the
//              second so that no rank rewrites its table while a peer may still read it.
//   NCCL path  publish is one all-reduce of send[0..words) into recv; release is nothing.  comm_peer_tables: send = local,
//              and read[0] = recv is the reduction.  comm_segment_tables: the per-rank tables end to end in one zeroed
//              table, so that a u64 sum with one writer per word copies them; read[s] = rank s's table in recv.
struct PeerTables {
  unsigned long long* local = nullptr;          // this rank's table
  int n_read = 0;                               // tables to read
  const unsigned long long* read[kMaxRanks] = {};
  bool peer = false;
  unsigned long long* send = nullptr;           // NCCL path: the all-reduce of comm_tables_publish
  unsigned long long* recv = nullptr;
  size_t words = 0;
};
// The owner (a session) holds its table, freed with it; the communicator keeps a weak reference and unmaps / frees the
// table when it is destroyed first.  A table of n_words u64 (initially all ~0) is allocated and, on the peer path, mapped
// into every rank on first use, and again when n_words or the communicator changes.
struct PeerTableEntry;
PeerTables comm_peer_tables(Ctx& c, std::shared_ptr<PeerTableEntry>& owner, size_t n_words);
PeerTables comm_scratch_tables(Ctx& c, size_t n_words);  // a table owned by the communicator (one call's scratch)
// a table per rank of n[s] elements of elem_bytes (every rank passes the same n), from the scratch table: peer path, every
// rank's sized to the largest; NCCL path, laid end to end in rank order, each from a word boundary, zeroed
PeerTables comm_segment_tables(Ctx& c, const unsigned long long* n, size_t elem_bytes);
void comm_tables_publish(Ctx& c, const PeerTables& t, int op);  // barrier, or the NCCL all-reduce (kU64Sum / kU64Min)
void comm_tables_release(Ctx& c, const PeerTables& t);          // barrier, or nothing
void comm_barrier(Ctx& c);  // peer path: every rank has reached this point of its stream; NCCL path: nothing
// NCCL path only: element-wise max of uint32 bit patterns (an exact copy of the one non-zero contribution)
void comm_allreduce_u32_max(Ctx& c, const unsigned* d_send, unsigned* d_recv, size_t count);
unsigned long long comm_id(const Ctx& c);  // identifies the communicator (0 = none): cached shard offsets check it

// sharded form of apply_rejector (reject.cu): MEDIAN / TRIMMED / ONE_TO_ONE over the union of all ranks' arrays
struct ShardedRejectArgs {
  const float4* tgt_pts = nullptr;  // Morton-ordered target, w = original index: the one-to-one table index
  size_t n_cloud = 0;               // target records
  unsigned long long offset = 0;    // global position of slot 0 of this rank
  std::shared_ptr<PeerTableEntry>* o2o = nullptr;  // the session's one-to-one table
};
void apply_rejector_sharded(Ctx& c, const pclb200_rejector& r, const RejectArrays& a, const ShardedRejectArgs& s);

}  // namespace pclb200
