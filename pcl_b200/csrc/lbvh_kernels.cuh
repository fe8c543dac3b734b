// lbvh_kernels.cuh — the device side of the index build: bounding box, Morton / Hilbert keys, the Karras radix tree over the
// sorted points, the cut into cell-aligned leaves, the cell table, bottom-up refit, node packing.  A header so that lbvh.cu
// stays the host-side driver (CUB sorts and scans between the kernels) and tests/host/lbvh_host_test.cpp can compile the
// SAME kernels for the host, run the same sequence with std:: algorithms in CUB's place, check the invariants the walks
// rely on and search the result against brute force.  The *_batch kernels build a batch of clouds in one pass, each
// cloud through the single build's own code (tests/host/lbvh_batch_host_test.cpp compares them with single builds).
#pragma once
#include <cmath>

#include "internal.cuh"
#include "traverse.cuh"

namespace pclb200 {

// ---- bbox ---------------------------------------------------------------------------------------
// floats mapped to order-preserving signed ints so atomicMin/Max work
__device__ __forceinline__ int f2ord(float f)
{
  int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__host__ __device__ __forceinline__ float ord2f(int i)
{
  int j = i >= 0 ? i : i ^ 0x7fffffff;
#ifdef __CUDA_ARCH__
  return __int_as_float(j);
#else
  float f;
  memcpy(&f, &j, 4);
  return f;
#endif
}

struct BBoxAcc {
  int lo[3];
  int hi[3];
  unsigned long long count;
};

// one thread's box and finite count, folded over its warp and into *acc (lanes that saw no finite point add nothing)
__device__ __forceinline__ void bbox_publish(float lo[3], float hi[3], unsigned cnt, BBoxAcc* acc)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if ((threadIdx.x & 31) == 0 && cnt) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      atomicMin(&acc->lo[d], f2ord(lo[d]));
      atomicMax(&acc->hi[d], f2ord(hi[d]));
    }
    atomicAdd(&acc->count, (unsigned long long)cnt);
  }
}

__global__ void k_bbox(const float4* __restrict__ p, size_t n, BBoxAcc* acc)
{
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  unsigned cnt = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float4 v = __ldg(p + i);
    if (isfinite(v.x) && isfinite(v.y) && isfinite(v.z)) {
      lo[0] = fminf(lo[0], v.x); hi[0] = fmaxf(hi[0], v.x);
      lo[1] = fminf(lo[1], v.y); hi[1] = fmaxf(hi[1], v.y);
      lo[2] = fminf(lo[2], v.z); hi[2] = fmaxf(hi[2], v.z);
      ++cnt;
    }
  }
  bbox_publish(lo, hi, cnt, acc);
}

// ---- Morton keys --------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long morton63(float x, float y, float z, float lx, float ly, float lz,
                                                       float scale)
{
  return (expand21(morton_cell(z, lz, scale)) << 2) | (expand21(morton_cell(y, ly, scale)) << 1) |
         expand21(morton_cell(x, lx, scale));
}

// 63-bit Hilbert index of the same 21-bit cell coordinates (Skilling's transpose algorithm).  Used to ORDER QUERIES
// only: a run of 32 consecutive points along the Hilbert curve is always a compact cluster (the Z-order curve jumps),
// so the packet walk of a warp touches fewer nodes.  The tree itself needs Morton prefixes and stays Morton-ordered.
__device__ __forceinline__ unsigned long long hilbert63(float x, float y, float z, float lx, float ly, float lz,
                                                        float scale)
{
  unsigned X[3];
  X[0] = morton_cell(x, lx, scale);
  X[1] = morton_cell(y, ly, scale);
  X[2] = morton_cell(z, lz, scale);
  const unsigned M = 1u << 20;
  for (unsigned Q = M; Q > 1; Q >>= 1) {
    const unsigned P = Q - 1;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      if (X[i] & Q)
        X[0] ^= P;
      else {
        const unsigned t = (X[0] ^ X[i]) & P;
        X[0] ^= t;
        X[i] ^= t;
      }
    }
  }
  X[1] ^= X[0];
  X[2] ^= X[1];
  unsigned t = 0;
  for (unsigned Q = M; Q > 1; Q >>= 1)
    if (X[2] & Q)
      t ^= Q - 1;
  X[0] ^= t; X[1] ^= t; X[2] ^= t;
  return (expand21(X[0]) << 2) | (expand21(X[1]) << 1) | expand21(X[2]);
}

// value = record slot i; for invalid (non-finite) points key = ~0 so they sort last
template <bool HILBERT>
__global__ void k_morton(const float4* __restrict__ p, size_t n, float lx, float ly, float lz, float scale,
                         unsigned long long* __restrict__ keys, int32_t* __restrict__ vals)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  float4 v = __ldg(p + i);
  bool ok = isfinite(v.x) && isfinite(v.y) && isfinite(v.z);
  keys[i] = !ok ? ~0ULL
                : (HILBERT ? hilbert63(v.x, v.y, v.z, lx, ly, lz, scale) : morton63(v.x, v.y, v.z, lx, ly, lz, scale));
  vals[i] = (int32_t)i;
}

// The key a query batch is sorted by: the top 32 bits (31..62) of hilbert63, ~0 for a non-finite point (it sorts last).
// 10.7 bits per axis give cells about a leaf wide, as coherent an order as the full index, in half the radix passes.
__device__ __forceinline__ unsigned hilbert_key32(float x, float y, float z, float lx, float ly, float lz, float scale)
{
  if (!(isfinite(x) && isfinite(y) && isfinite(z)))
    return ~0u;
  return (unsigned)(hilbert63(x, y, z, lx, ly, lz, scale) >> 31);
}

// a unit that starts at word `word` (< 4) of a record, into the record's head (its first four words); a float4 unit
// starts at word 0 and is the whole head
__device__ __forceinline__ void put_head(float* head, unsigned, const float4& v) { *reinterpret_cast<float4*>(head) = v; }
__device__ __forceinline__ void put_head(float* head, unsigned word, float v) { head[word] = v; }

// One pass over n strided records (xyz at offset 0): the whole record into `copy`, xyz into `dense` as float4 (w = the
// record's w when a record is 16 bytes, else 1) and, into keys / vals, the point's hilbert_key32 and its slot.  Each
// output is nullable.  U: the unit the records are moved in (float4 when the stride is a multiple of 16 and recs / copy
// are 16-byte aligned, else float); units = record stride / sizeof(U).  Each warp moves the contiguous bytes of its 32
// records as consecutive units across its lanes, so every load and every store of the copy covers whole sectors (one
// record per lane would touch 32 sectors per instruction, 16 B of each at a 48-B stride), and hands each record's first
// 16 bytes to the lane of that record through shared memory.  blockDim.x = 256.
template <typename U>
__global__ void __launch_bounds__(256)
k_stage_records(const U* __restrict__ recs, size_t n, unsigned units, U* __restrict__ copy, float4* __restrict__ dense,
                float lx, float ly, float lz, float scale, unsigned* __restrict__ keys, int32_t* __restrict__ vals)
{
  constexpr unsigned kWords = sizeof(U) / 4;
  __shared__ __align__(16) float s_head[8][32][4];  // per warp: the first four words of each of its records
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t first = blockIdx.x * (size_t)blockDim.x + (threadIdx.x & ~31u);
  if (first >= n)
    return;  // the whole warp
  const unsigned nrec = (unsigned)min((size_t)32, n - first);
  const U* src = recs + first * units;
  U* dst = copy ? copy + first * units : nullptr;
  for (unsigned f = lane; f < nrec * units; f += 32) {
    const unsigned rec = f / units, word = (f - rec * units) * kWords;
    if (!dst && word >= 4)
      continue;
    const U v = src[f];
    if (dst)
      dst[f] = v;
    if (word < 4)
      put_head(s_head[warp][rec], word, v);
  }
  __syncwarp();
  if (lane >= nrec)
    return;
  const size_t i = first + lane;
  const float4 h = *reinterpret_cast<const float4*>(s_head[warp][lane]);
  const float x = h.x, y = h.y, z = h.z;
  if (dense)
    dense[i] = make_float4(x, y, z, units * sizeof(U) == 16 ? h.w : 1.f);
  if (keys) {
    keys[i] = hilbert_key32(x, y, z, lx, ly, lz, scale);
    vals[i] = (int32_t)i;
  }
}

// The key k_stage_records gives point i, in the frame of its own problem instead of one frame for all: a batch of
// problems over consecutive ranges of pts (offsets: B + 1 entries), frames[p] = {lo[0..2], morton_scale} of problem p's
// target.  Sorted by these keys and then stably by problem, each problem's points fall in the order its own frame gives.
__global__ void k_problem_frame_keys(const float4* __restrict__ pts, size_t n, const long long* __restrict__ offsets,
                                     int n_problems, const float4* __restrict__ frames, unsigned* __restrict__ keys,
                                     int32_t* __restrict__ vals)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const float4 f = frames[problem_of(offsets, n_problems, (long long)i)];
  const float4 v = pts[i];
  keys[i] = hilbert_key32(v.x, v.y, v.z, f.x, f.y, f.z, f.w);
  vals[i] = (int32_t)i;
}

// sorted gather: out[j] = {xyz of slot vals[j], orig index bits}; pads the tail with +inf sentinels
__global__ void k_gather_sorted(const float4* __restrict__ p, const int32_t* __restrict__ vals,
                                const int32_t* __restrict__ orig_of_slot, size_t n_valid, size_t n_padded,
                                float4* __restrict__ out)
{
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n_padded)
    return;
  if (j < n_valid) {
    int32_t slot = vals[j];
    float4 v = __ldg(p + slot);
    int32_t oi = orig_of_slot ? orig_of_slot[slot] : slot;
    out[j] = make_float4(v.x, v.y, v.z, __int_as_float(oi));
  }
  else {
    const float inf = __int_as_float(0x7f800000);
    out[j] = make_float4(inf, inf, inf, __int_as_float(kSentinelIndex));
  }
}

// ---- refit --------------------------------------------------------------------------------------
__device__ __forceinline__ void refit_item(int leaf, const float4* __restrict__ pts, int n_leaves,
                                           const int2* __restrict__ children, const int* __restrict__ node_parent,
                                           const int* __restrict__ leaf_parent, float4* __restrict__ leaf_lo,
                                           float4* __restrict__ leaf_hi, float4* __restrict__ node_lo,
                                           float4* __restrict__ node_hi, unsigned* __restrict__ flags)
{
  if (leaf >= n_leaves)
    return;
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
#pragma unroll
  for (int j = 0; j < kLeafSize; ++j) {
    float4 p = __ldg(pts + (size_t)leaf * kLeafSize + j);
    if (__float_as_int(p.w) != kSentinelIndex) {
      lo[0] = fminf(lo[0], p.x); hi[0] = fmaxf(hi[0], p.x);
      lo[1] = fminf(lo[1], p.y); hi[1] = fmaxf(hi[1], p.y);
      lo[2] = fminf(lo[2], p.z); hi[2] = fmaxf(hi[2], p.z);
    }
  }
  leaf_lo[leaf] = make_float4(lo[0], lo[1], lo[2], 0.f);
  leaf_hi[leaf] = make_float4(hi[0], hi[1], hi[2], 0.f);
  if (n_leaves == 1)
    return;
  int cur = leaf_parent[leaf];
  while (cur >= 0) {
    __threadfence();
    if (atomicAdd(&flags[cur], 1u) == 0u)
      return;  // first child to arrive: the sibling's thread finishes this node
    __threadfence();
    int2 ch = children[cur];
    float4 alo = ch.x < 0 ? __ldcg(leaf_lo + ~ch.x) : __ldcg(node_lo + ch.x);
    float4 ahi = ch.x < 0 ? __ldcg(leaf_hi + ~ch.x) : __ldcg(node_hi + ch.x);
    float4 blo = ch.y < 0 ? __ldcg(leaf_lo + ~ch.y) : __ldcg(node_lo + ch.y);
    float4 bhi = ch.y < 0 ? __ldcg(leaf_hi + ~ch.y) : __ldcg(node_hi + ch.y);
    node_lo[cur] = make_float4(fminf(alo.x, blo.x), fminf(alo.y, blo.y), fminf(alo.z, blo.z), 0.f);
    node_hi[cur] = make_float4(fmaxf(ahi.x, bhi.x), fmaxf(ahi.y, bhi.y), fmaxf(ahi.z, bhi.z), 0.f);
    cur = node_parent[cur];
  }
}

__global__ void k_refit(const float4* __restrict__ pts, int n_leaves, const int2* __restrict__ children,
                        const int* __restrict__ node_parent, const int* __restrict__ leaf_parent,
                        float4* __restrict__ leaf_lo, float4* __restrict__ leaf_hi, float4* __restrict__ node_lo,
                        float4* __restrict__ node_hi, unsigned* __restrict__ flags)
{
  refit_item(blockIdx.x * blockDim.x + threadIdx.x, pts, n_leaves, children, node_parent, leaf_parent, leaf_lo, leaf_hi,
             node_lo, node_hi, flags);
}

__device__ __forceinline__ void pack_nodes_item(int i, int n_internal, const int2* __restrict__ children,
                                                const float4* __restrict__ leaf_lo, const float4* __restrict__ leaf_hi,
                                                const float4* __restrict__ node_lo, const float4* __restrict__ node_hi,
                                                BvhNode* __restrict__ nodes)
{
  if (i >= n_internal)
    return;
  int2 ch = children[i];
  float4 alo = ch.x < 0 ? leaf_lo[~ch.x] : node_lo[ch.x];
  float4 ahi = ch.x < 0 ? leaf_hi[~ch.x] : node_hi[ch.x];
  float4 blo = ch.y < 0 ? leaf_lo[~ch.y] : node_lo[ch.y];
  float4 bhi = ch.y < 0 ? leaf_hi[~ch.y] : node_hi[ch.y];
  BvhNode nd;
  nd.a = make_float4(alo.x, alo.y, alo.z, ahi.x);
  nd.b = make_float4(ahi.y, ahi.z, blo.x, blo.y);
  nd.c = make_float4(blo.z, bhi.x, bhi.y, bhi.z);
  nd.d = make_int4(ch.x, ch.y, 0, 0);
  nodes[i] = nd;
}

__global__ void k_pack_nodes(int n_internal, const int2* __restrict__ children, const float4* __restrict__ leaf_lo,
                             const float4* __restrict__ leaf_hi, const float4* __restrict__ node_lo,
                             const float4* __restrict__ node_hi, BvhNode* __restrict__ nodes)
{
  pack_nodes_item(blockIdx.x * blockDim.x + threadIdx.x, n_internal, children, leaf_lo, leaf_hi, node_lo, node_hi, nodes);
}

// ---- cell-aligned leaves --------------------------------------------------------------------------------------
// A leaf is a whole radix-tree cell holding <= kLeafSize points (the subtree of the Karras tree over POINTS whose
// parent holds more), stored padded to kLeafSize slots with +inf sentinels.  Compared with "kLeafSize consecutive
// Morton points" the leaf boxes never straddle a cell boundary: measured with tools/lbvh_emul.cpp on the bench
// surface the average leaf diagonal drops 2.5x, a seeded 1-NN walk needs 1.9 instead of 5.8 leaf scans and 25
// instead of 45 node visits, a 32-query packet 59 instead of 79 nodes.

// Karras 2012 over the sorted point keys (ties by index); also records each node's key range [lo, hi].
__device__ __forceinline__ int delta_pt(const unsigned long long* __restrict__ keys, int n, int i, int j)
{
  if (j < 0 || j >= n)
    return -1;
  const unsigned long long x = keys[i] ^ keys[j];
  if (x == 0)
    return 64 + __clz(i ^ j);
  return __clzll((long long)x);
}

__global__ void k_karras_points(const unsigned long long* __restrict__ keys, int n, int2* __restrict__ children,
                                int* __restrict__ node_parent, int* __restrict__ point_parent, int2* __restrict__ range)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
#include "karras_points_body.inc"
}

// keep[i] = node i stays an internal node of the final tree (holds more than kLeafSize points);
// leaf_flag[pos] = 1 at the first sorted position of every leaf cell
__global__ void k_mark_cells(int n, const int2* __restrict__ range, const int* __restrict__ node_parent,
                             const int* __restrict__ point_parent, int* __restrict__ keep, int* __restrict__ leaf_flag)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
#include "mark_cells_body.inc"
}

__device__ __forceinline__ void leaf_starts_item(int i, int n, const int* __restrict__ leaf_flag,
                                                 const int* __restrict__ leaf_incl, int* __restrict__ leaf_start)
{
  if (i < n && leaf_flag[i])
    leaf_start[leaf_incl[i] - 1] = i;
}

__global__ void k_leaf_starts(int n, const int* __restrict__ leaf_flag, const int* __restrict__ leaf_incl,
                              int* __restrict__ leaf_start)
{
  leaf_starts_item(blockIdx.x * blockDim.x + threadIdx.x, n, leaf_flag, leaf_incl, leaf_start);
}

__global__ void k_fill_sentinels(float4* __restrict__ out, size_t n)
{
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j < n) {
    const float inf = __int_as_float(0x7f800000);
    out[j] = make_float4(inf, inf, inf, __int_as_float(kSentinelIndex));
  }
}

// sorted position -> padded leaf slot
__device__ __forceinline__ void scatter_cells_item(int pos, const float4* __restrict__ p,
                                                   const int32_t* __restrict__ vals,
                                                   const int32_t* __restrict__ orig_of_slot, int n,
                                                   const int* __restrict__ leaf_incl, const int* __restrict__ leaf_start,
                                                   float4* __restrict__ out)
{
  if (pos >= n)
    return;
  const int leaf = leaf_incl[pos] - 1;
  const int32_t slot = vals[pos];
  const float4 v = __ldg(p + slot);
  const int32_t oi = orig_of_slot ? orig_of_slot[slot] : slot;
  out[(size_t)leaf * kLeafSize + (pos - leaf_start[leaf])] = make_float4(v.x, v.y, v.z, __int_as_float(oi));
}

__global__ void k_scatter_cells(const float4* __restrict__ p, const int32_t* __restrict__ vals,
                                const int32_t* __restrict__ orig_of_slot, int n, const int* __restrict__ leaf_incl,
                                const int* __restrict__ leaf_start, float4* __restrict__ out)
{
  scatter_cells_item(blockIdx.x * blockDim.x + threadIdx.x, p, vals, orig_of_slot, n, leaf_incl, leaf_start, out);
}

// ---- cell table -------------------------------------------------------------------------------------------------------
struct CellTableW {
  unsigned long long* slots;  // packed {key (low 32), reference (high 32)}; nullptr = not built
  unsigned shift, mask;
  int bmax;
};

// number of leading bits two 63-bit Morton codes share (63 when they are equal)
__device__ __forceinline__ int prefix_len63(unsigned long long a, unsigned long long b)
{
  const unsigned long long x = a ^ b;
  return x == 0 ? 63 : __clzll((long long)x) - 1;
}

// hist[l] = number of adjacent sorted pairs that share exactly l leading bits: the number of occupied cells of level b is
// 1 + sum_{l < 3b} hist[l], which sizes the table before it is filled
__global__ void k_prefix_hist(const unsigned long long* __restrict__ keys, int n, unsigned* __restrict__ hist)
{
  __shared__ unsigned sh[64];
  if (threadIdx.x < 64)
    sh[threadIdx.x] = 0;
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x + 1; i < n; i += gridDim.x * blockDim.x)
    atomicAdd(&sh[prefix_len63(keys[i - 1], keys[i])], 1u);
  __syncthreads();
  if (threadIdx.x < 64 && sh[threadIdx.x])
    atomicAdd(&hist[threadIdx.x], sh[threadIdx.x]);
}

// every third bit of v, packed (inverse of expand21)
__device__ __forceinline__ unsigned compact21(unsigned long long v)
{
  v &= 0x1249249249249249ULL;
  v = (v | v >> 2) & 0x10c30c30c30c30c3ULL;
  v = (v | v >> 4) & 0x100f00f00f00f00fULL;
  v = (v | v >> 8) & 0x1f0000ff0000ffULL;
  v = (v | v >> 16) & 0x1f00000000ffffULL;
  v = (v | v >> 32) & 0x1fffffULL;
  return (unsigned)v;
}

// (level b, cell of Morton code `code`) -> ref.  Several threads may insert the same pair (a leaf that spans several
// cells is inserted once per point): the first wins, the others see their own key and stop.
__device__ __forceinline__ void cell_insert(const CellTableW& T, int b, unsigned long long code, int ref)
{
  const unsigned long long P = code >> (63 - 3 * b);
  const unsigned key = cell_key(b, compact21(P), compact21(P >> 1), compact21(P >> 2));
  const unsigned long long packed = ((unsigned long long)(unsigned)ref << 32) | key;
  unsigned h = (key * 0x9E3779B1u) >> T.shift;
  for (;;) {
    const unsigned long long old = atomicCAS(T.slots + h, 0ULL, packed);
    if (old == 0ULL || (unsigned)old == key)
      return;
    h = (h + 1u) & T.mask;
  }
}

// children / parents of the final tree (kept nodes renumbered by new_id; everything below becomes a leaf)
__global__ void k_link_cells(int n, const int2* __restrict__ children, const int2* __restrict__ range,
                             const int* __restrict__ keep, const int* __restrict__ new_id,
                             const int* __restrict__ leaf_incl, const unsigned long long* __restrict__ keys,
                             int2* __restrict__ out_children, int* __restrict__ out_node_parent,
                             int* __restrict__ out_leaf_parent, int2* __restrict__ out_node_leaves, CellTableW cells)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
#include "link_cells_body.inc"
}

// ---- host decisions every build shares ------------------------------------------------------------------------------
// the index's frame from its bbox accumulator: box of the finite points, ONE isotropic scale so Morton cells are cubes
inline void morton_frame(const BBoxAcc& h, float lo[3], float hi[3], float& scale)
{
  float ext = 0.f;
  for (int d = 0; d < 3; ++d) {
    lo[d] = ord2f(h.lo[d]);
    hi[d] = ord2f(h.hi[d]);
    ext = std::max(ext, hi[d] - lo[d]);
  }
  scale = ext > 0.f ? 2097152.f / ext : 1.f;
  if (!std::isfinite(scale))
    scale = 1.f;
}

// The cell table of an index of nv >= 256 points (traverse.cuh: CellTable): levels 1..bmax, bmax = the finest level
// (<= kCellMaxBits) whose occupied cells still hold >= 4 indexed points on average — finer levels would mostly map single
// points.  The number of entries is known exactly from the prefix-length histogram (k_prefix_hist); the table gets >= 2
// slots per entry.  log2_slots = 0: no table.
inline CellTableHost cell_table_plan(const unsigned hist[64], int nv, const float lo[3], const float hi[3], float scale)
{
  CellTableHost t;
  uint64_t cum = 1, entries = 0;
  int l = 0, bmax = 0;
  for (int b = 1; b <= kCellMaxBits; ++b) {
    for (; l < 3 * b; ++l)
      cum += hist[l];
    if (cum > (uint64_t)nv / 4)
      break;
    bmax = b;
    entries += cum;
    t.occupied[b] = cum;
  }
  if (bmax >= 1) {
    unsigned lg = 6;
    while (((uint64_t)1 << lg) < 2 * entries)
      ++lg;
    t.log2_slots = lg;
    t.bmax = bmax;
    t.entries = entries;
    float m = 0.f;
    for (int d = 0; d < 3; ++d)
      m = std::max(m, std::max(std::fabs(lo[d]), std::fabs(hi[d])));
    m = std::max(m, 2097152.f / scale);
    t.margin = 2e-6f * m;
  }
  return t;
}

// the kernels' view of a planned table whose slots are allocated (and zeroed before the first insert)
inline CellTableW cell_table_view(uint2* slots, const CellTableHost& t)
{
  return CellTableW{reinterpret_cast<unsigned long long*>(slots), 32 - t.log2_slots, (1u << t.log2_slots) - 1u, t.bmax};
}

// ---- a batch of clouds in one build ---------------------------------------------------------------------------------
// Cloud c is the records [first, first + n) of one dense array.  Each stage runs the single build's body on the cloud's
// base pointers: sorted positions of cloud c start at `first`, its radix-tree node scratch at first - c (a cloud of n
// points has at most n - 1 nodes), its final leaves and nodes at leaf_first / node_first of the batch's scratch.
constexpr int kBatchTile = 4096;  // points per block of the per-cloud reductions (tiles never straddle two clouds)

struct BuildCloud {
  long long first = 0;       // first record (= first sorted position) of the cloud
  long long n = 0;           // records
  int nv = 0;                // finite points
  float lo[3] = {0, 0, 0}, scale = 1.f;  // the cloud's Morton frame
  // known after the cut (the second read-back)
  int n_leaves = 0, n_int = 0;
  long long leaf_first = 0, node_first = 0;  // in the batch's leaf / final-node scratch
  float4* pts = nullptr;     // the cloud's handle: n_leaves * kLeafSize
  BvhNode* nodes = nullptr;  // n_int
  int2* node_leaves = nullptr;
  CellTableW cells{nullptr, 0, 0, 0};
};

// what the host reads after the cut: the leaf and node counts, and the prefix-length histogram (nv >= 256 only)
struct CloudSummary {
  int n_leaves, n_int;
  unsigned hist[64];
};

// per cloud, the box and finite count of its records; block b works on tile b - tiles[c] of cloud c = problem_of(tiles, b)
__global__ void k_bbox_batch(const float4* __restrict__ p, const BuildCloud* __restrict__ clouds,
                             const long long* __restrict__ tiles, int n_clouds, BBoxAcc* acc)
{
  const int c = problem_of(tiles, n_clouds, (long long)blockIdx.x);
  const BuildCloud& C = clouds[c];
  const long long t0 = (blockIdx.x - tiles[c]) * (long long)kBatchTile;
  const long long end = t0 + kBatchTile < C.n ? t0 + kBatchTile : C.n;
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  unsigned cnt = 0;
  for (long long i = t0 + threadIdx.x; i < end; i += blockDim.x) {
    float4 v = __ldg(p + C.first + i);
    if (isfinite(v.x) && isfinite(v.y) && isfinite(v.z)) {
      lo[0] = fminf(lo[0], v.x); hi[0] = fmaxf(hi[0], v.x);
      lo[1] = fminf(lo[1], v.y); hi[1] = fmaxf(hi[1], v.y);
      lo[2] = fminf(lo[2], v.z); hi[2] = fmaxf(hi[2], v.z);
      ++cnt;
    }
  }
  bbox_publish(lo, hi, cnt, acc + c);
}

// k_morton<false> of every point in its own cloud's frame; vals = the record (global)
__global__ void k_morton_batch(const float4* __restrict__ p, size_t n, const long long* __restrict__ offsets,
                               int n_clouds, const BuildCloud* __restrict__ clouds, unsigned long long* __restrict__ keys,
                               int32_t* __restrict__ vals)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const BuildCloud& C = clouds[problem_of(offsets, n_clouds, (long long)i)];
  const float4 v = __ldg(p + i);
  const bool ok = isfinite(v.x) && isfinite(v.y) && isfinite(v.z);
  keys[i] = !ok ? ~0ULL : morton63(v.x, v.y, v.z, C.lo[0], C.lo[1], C.lo[2], C.scale);
  vals[i] = (int32_t)i;
}

// after the sort by key: the cloud of each sorted record (the key of the stable sort by cloud) and its position
__global__ void k_cloud_of_sorted(const int32_t* __restrict__ vals, size_t n, const long long* __restrict__ offsets,
                                  int n_clouds, unsigned* __restrict__ cloud, int32_t* __restrict__ pos)
{
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n)
    return;
  cloud[j] = (unsigned)problem_of(offsets, n_clouds, (long long)vals[j]);
  pos[j] = (int32_t)j;
}

// the permutation of the sort by cloud applied: each cloud's range is its single build's sorted keys and local slots
__global__ void k_permute_sorted(const unsigned long long* __restrict__ keys_in, const int32_t* __restrict__ vals_in,
                                 const int32_t* __restrict__ perm, size_t n, const long long* __restrict__ offsets,
                                 int n_clouds, unsigned long long* __restrict__ keys, int32_t* __restrict__ vals)
{
  const size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (k >= n)
    return;
  const int32_t j = perm[k];
  keys[k] = keys_in[j];
  vals[k] = vals_in[j] - (int32_t)offsets[problem_of(offsets, n_clouds, (long long)k)];
}

// work item g of a launch over all records: cloud c and the cloud's local item g - first
#define PCLB_BATCH_ITEM(offsets, n_clouds, n)                                      \
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;            \
  if (g >= (long long)(n))                                                         \
    return;                                                                        \
  const int c = problem_of(offsets, n_clouds, g);                                  \
  const BuildCloud& C = clouds[c];                                                 \
  const int i = (int)(g - C.first);

// karras_points_item of every cloud of more than kLeafSize points; node_cloud[node] = the cloud of every node position
__global__ void k_karras_points_batch(const unsigned long long* __restrict__ keys_all, size_t n_all,
                                      const long long* __restrict__ offsets, int n_clouds,
                                      const BuildCloud* __restrict__ clouds, int2* __restrict__ children_all,
                                      int* __restrict__ node_parent_all, int* __restrict__ point_parent_all,
                                      int2* __restrict__ range_all, unsigned* __restrict__ node_cloud)
{
  PCLB_BATCH_ITEM(offsets, n_clouds, n_all)
  const long long nb = C.first - c;
  if (i < C.n - 1)
    node_cloud[nb + i] = (unsigned)c;
  if (C.nv <= kLeafSize)
    return;
  const unsigned long long* __restrict__ keys = keys_all + C.first;
  const int n = C.nv;
  int2* __restrict__ children = children_all + nb;
  int* __restrict__ node_parent = node_parent_all + nb;
  int* __restrict__ point_parent = point_parent_all + C.first;
  int2* __restrict__ range = range_all + nb;
#include "karras_points_body.inc"
}

__global__ void k_mark_cells_batch(size_t n_all, const long long* __restrict__ offsets, int n_clouds,
                                   const BuildCloud* __restrict__ clouds, const int2* __restrict__ range_all,
                                   const int* __restrict__ node_parent_all, const int* __restrict__ point_parent_all,
                                   int* __restrict__ keep_all, int* __restrict__ leaf_flag_all)
{
  PCLB_BATCH_ITEM(offsets, n_clouds, n_all)
  if (C.nv <= kLeafSize)
    return;
  const long long nb = C.first - c;
  const int n = C.nv;
  const int2* __restrict__ range = range_all + nb;
  const int* __restrict__ node_parent = node_parent_all + nb;
  const int* __restrict__ point_parent = point_parent_all + C.first;
  int* __restrict__ keep = keep_all + nb;
  int* __restrict__ leaf_flag = leaf_flag_all + C.first;
#include "mark_cells_body.inc"
}

// k_prefix_hist of every cloud of >= 256 points into its summary (zeroed), over tiles as k_bbox_batch
__global__ void k_prefix_hist_batch(const unsigned long long* __restrict__ keys, const BuildCloud* __restrict__ clouds,
                                    const long long* __restrict__ tiles, int n_clouds, CloudSummary* __restrict__ out)
{
  __shared__ unsigned sh[64];
  const int c = problem_of(tiles, n_clouds, (long long)blockIdx.x);
  const BuildCloud& C = clouds[c];
  if (C.nv < 256)
    return;  // the whole block
  if (threadIdx.x < 64)
    sh[threadIdx.x] = 0;
  __syncthreads();
  const long long t0 = (blockIdx.x - tiles[c]) * (long long)kBatchTile;
  const long long end = t0 + kBatchTile < C.nv ? t0 + kBatchTile : C.nv;
  const unsigned long long* k = keys + C.first;
  for (long long i = (t0 > 0 ? t0 : 1) + threadIdx.x; i < end; i += blockDim.x)
    atomicAdd(&sh[prefix_len63(k[i - 1], k[i])], 1u);
  __syncthreads();
  if (threadIdx.x < 64 && sh[threadIdx.x])
    atomicAdd(&out[c].hist[threadIdx.x], sh[threadIdx.x]);
}

// the leaf and node counts of each cloud's cut (one thread per cloud; a cloud of <= kLeafSize points is one leaf)
__global__ void k_cut_summary(const BuildCloud* __restrict__ clouds, int n_clouds, const int* __restrict__ leaf_incl,
                              const int* __restrict__ new_id, const int* __restrict__ keep, CloudSummary* __restrict__ out)
{
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_clouds)
    return;
  const BuildCloud& C = clouds[c];
  if (C.nv <= kLeafSize) {
    out[c].n_leaves = 1;
    out[c].n_int = 0;
    return;
  }
  const long long nb = C.first - c, last = nb + C.nv - 2;
  out[c].n_leaves = leaf_incl[C.first + C.nv - 1];
  out[c].n_int = new_id[last] + keep[last];
}

// the handles' sentinel padding (leaf space: n_leaves * kLeafSize per cloud) and zeroed cell-table slots (slot space)
__global__ void k_clear_outputs_batch(const BuildCloud* __restrict__ clouds, int n_clouds,
                                      const long long* __restrict__ leaf_offsets, const long long* __restrict__ slot_offsets)
{
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (g < leaf_offsets[n_clouds] * kLeafSize) {
    const int c = problem_of(leaf_offsets, n_clouds, g / kLeafSize);
    const float inf = __int_as_float(0x7f800000);
    clouds[c].pts[g - leaf_offsets[c] * kLeafSize] = make_float4(inf, inf, inf, __int_as_float(kSentinelIndex));
  }
  if (g < slot_offsets[n_clouds]) {
    const int c = problem_of(slot_offsets, n_clouds, g);
    clouds[c].cells.slots[g - slot_offsets[c]] = 0ULL;
  }
}

// k_gather_sorted of every cloud of <= kLeafSize points: its one leaf (kLeafSize items per cloud)
__global__ void k_gather_small_batch(const float4* __restrict__ p, const int32_t* __restrict__ vals,
                                     const BuildCloud* __restrict__ clouds, int n_clouds)
{
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (g >= (long long)n_clouds * kLeafSize)
    return;
  const BuildCloud& C = clouds[g / kLeafSize];
  if (C.nv > kLeafSize)
    return;
  const size_t j = (size_t)(g % kLeafSize);
  if (j < (size_t)C.nv) {
    const int32_t slot = vals[C.first + j];
    const float4 v = __ldg(p + C.first + slot);
    C.pts[j] = make_float4(v.x, v.y, v.z, __int_as_float(slot));
  }
  else {
    const float inf = __int_as_float(0x7f800000);
    C.pts[j] = make_float4(inf, inf, inf, __int_as_float(kSentinelIndex));
  }
}

__global__ void k_leaf_starts_batch(size_t n, const long long* __restrict__ offsets, int n_clouds,
                                    const BuildCloud* __restrict__ clouds, const int* __restrict__ leaf_flag,
                                    const int* __restrict__ leaf_incl, int* __restrict__ leaf_start)
{
  PCLB_BATCH_ITEM(offsets, n_clouds, n)
  if (C.nv <= kLeafSize)
    return;
  leaf_starts_item(i, C.nv, leaf_flag + C.first, leaf_incl + C.first, leaf_start + C.leaf_first);
}

__global__ void k_scatter_cells_batch(const float4* __restrict__ p, const int32_t* __restrict__ vals, size_t n,
                                      const long long* __restrict__ offsets, int n_clouds,
                                      const BuildCloud* __restrict__ clouds, const int* __restrict__ leaf_incl,
                                      const int* __restrict__ leaf_start)
{
  PCLB_BATCH_ITEM(offsets, n_clouds, n)
  if (C.nv <= kLeafSize)
    return;
  scatter_cells_item(i, p + C.first, vals + C.first, nullptr, C.nv, leaf_incl + C.first, leaf_start + C.leaf_first,
                     C.pts);
}

__global__ void k_link_cells_batch(size_t n_all, const long long* __restrict__ offsets, int n_clouds,
                                   const BuildCloud* __restrict__ clouds, const int2* __restrict__ children_all,
                                   const int2* __restrict__ range_all, const int* __restrict__ keep_all,
                                   const int* __restrict__ new_id_all, const int* __restrict__ leaf_incl_all,
                                   const unsigned long long* __restrict__ keys_all, int2* __restrict__ out_children_all,
                                   int* __restrict__ out_node_parent_all, int* __restrict__ out_leaf_parent_all)
{
  PCLB_BATCH_ITEM(offsets, n_clouds, n_all)
  if (C.nv <= kLeafSize)
    return;
  const long long nb = C.first - c;
  const int n = C.nv;
  const int2* __restrict__ children = children_all + nb;
  const int2* __restrict__ range = range_all + nb;
  const int* __restrict__ keep = keep_all + nb;
  const int* __restrict__ new_id = new_id_all + nb;
  const int* __restrict__ leaf_incl = leaf_incl_all + C.first;
  const unsigned long long* __restrict__ keys = keys_all + C.first;
  int2* __restrict__ out_children = out_children_all + C.node_first;
  int* __restrict__ out_node_parent = out_node_parent_all + C.node_first;
  int* __restrict__ out_leaf_parent = out_leaf_parent_all + C.leaf_first;
  int2* __restrict__ out_node_leaves = C.node_leaves;
  const CellTableW cells = C.cells;
#include "link_cells_body.inc"
}

// leaf space: every cloud's n_leaves leaves end to end (leaf_offsets)
__global__ void k_refit_batch(const BuildCloud* __restrict__ clouds, int n_clouds,
                              const long long* __restrict__ leaf_offsets, const int2* __restrict__ children,
                              const int* __restrict__ node_parent, const int* __restrict__ leaf_parent,
                              float4* __restrict__ leaf_lo, float4* __restrict__ leaf_hi, float4* __restrict__ node_lo,
                              float4* __restrict__ node_hi, unsigned* __restrict__ flags)
{
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (g >= leaf_offsets[n_clouds])
    return;
  const BuildCloud& C = clouds[problem_of(leaf_offsets, n_clouds, g)];
  if (C.nv <= kLeafSize)
    return;
  const long long lb = C.leaf_first, nb = C.node_first;
  refit_item((int)(g - lb), C.pts, C.n_leaves, children + nb, node_parent + nb, leaf_parent + lb, leaf_lo + lb,
             leaf_hi + lb, node_lo + nb, node_hi + nb, flags + nb);
}

// node space: every cloud's n_int final nodes end to end (node_offsets)
__global__ void k_pack_nodes_batch(const BuildCloud* __restrict__ clouds, int n_clouds,
                                   const long long* __restrict__ node_offsets, const int2* __restrict__ children,
                                   const float4* __restrict__ leaf_lo, const float4* __restrict__ leaf_hi,
                                   const float4* __restrict__ node_lo, const float4* __restrict__ node_hi)
{
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (g >= node_offsets[n_clouds])
    return;
  const BuildCloud& C = clouds[problem_of(node_offsets, n_clouds, g)];
  const long long lb = C.leaf_first, nb = C.node_first;
  pack_nodes_item((int)(g - nb), C.n_int, children + nb, leaf_lo + lb, leaf_hi + lb, node_lo + nb, node_hi + nb, C.nodes);
}
#undef PCLB_BATCH_ITEM

// ---- host orchestration -------------------------------------------------------------------------

}  // namespace pclb200
