// lbvh_kernels.cuh — the device side of the index build: bounding box, Morton / Hilbert keys, the Karras radix tree over the
// sorted points, the cut into cell-aligned leaves, the cell table, bottom-up refit, node packing.  A header so that lbvh.cu
// stays the host-side driver (CUB sorts and scans between the kernels) and tests/host/lbvh_host_test.cpp can compile the
// SAME kernels for the host, run the same sequence with std:: algorithms in CUB's place, check the invariants the walks
// rely on and search the result against brute force.
#pragma once
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
__global__ void k_refit(const float4* __restrict__ pts, int n_leaves, const int2* __restrict__ children,
                        const int* __restrict__ node_parent, const int* __restrict__ leaf_parent,
                        float4* __restrict__ leaf_lo, float4* __restrict__ leaf_hi, float4* __restrict__ node_lo,
                        float4* __restrict__ node_hi, unsigned* __restrict__ flags)
{
  int leaf = blockIdx.x * blockDim.x + threadIdx.x;
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

__global__ void k_pack_nodes(int n_internal, const int2* __restrict__ children, const float4* __restrict__ leaf_lo,
                             const float4* __restrict__ leaf_hi, const float4* __restrict__ node_lo,
                             const float4* __restrict__ node_hi, BvhNode* __restrict__ nodes)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
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
  if (i >= n - 1)
    return;
  int d = (delta_pt(keys, n, i, i + 1) - delta_pt(keys, n, i, i - 1)) >= 0 ? 1 : -1;
  int dmin = delta_pt(keys, n, i, i - d);
  int lmax = 2;
  while (delta_pt(keys, n, i, i + lmax * d) > dmin)
    lmax <<= 1;
  int l = 0;
  for (int t = lmax >> 1; t >= 1; t >>= 1)
    if (delta_pt(keys, n, i, i + (l + t) * d) > dmin)
      l += t;
  int j = i + l * d;
  int dnode = delta_pt(keys, n, i, j);
  int s = 0;
  int t = l;
  do {
    t = (t + 1) >> 1;
    if (delta_pt(keys, n, i, i + (s + t) * d) > dnode)
      s += t;
  } while (t > 1);
  int gamma = i + s * d + min(d, 0);
  int left, right;
  if (min(i, j) == gamma) {
    left = ~gamma;
    point_parent[gamma] = i;
  }
  else {
    left = gamma;
    node_parent[gamma] = i;
  }
  if (max(i, j) == gamma + 1) {
    right = ~(gamma + 1);
    point_parent[gamma + 1] = i;
  }
  else {
    right = gamma + 1;
    node_parent[gamma + 1] = i;
  }
  children[i] = make_int2(left, right);
  range[i] = make_int2(min(i, j), max(i, j));
  if (i == 0)
    node_parent[0] = -1;
}

// keep[i] = node i stays an internal node of the final tree (holds more than kLeafSize points);
// leaf_flag[pos] = 1 at the first sorted position of every leaf cell
__global__ void k_mark_cells(int n, const int2* __restrict__ range, const int* __restrict__ node_parent,
                             const int* __restrict__ point_parent, int* __restrict__ keep, int* __restrict__ leaf_flag)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n - 1) {
    const int2 r = range[i];
    const int cnt = r.y - r.x + 1;
    const int par = node_parent[i];
    const int pcnt = par < 0 ? 0x7fffffff : (range[par].y - range[par].x + 1);
    keep[i] = cnt > kLeafSize ? 1 : 0;
    if (cnt <= kLeafSize && pcnt > kLeafSize)
      leaf_flag[r.x] = 1;
  }
  if (i < n) {
    const int par = point_parent[i];
    if (range[par].y - range[par].x + 1 > kLeafSize)
      leaf_flag[i] = 1;  // a single point whose sibling subtree is large
  }
}

__global__ void k_leaf_starts(int n, const int* __restrict__ leaf_flag, const int* __restrict__ leaf_incl,
                              int* __restrict__ leaf_start)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && leaf_flag[i])
    leaf_start[leaf_incl[i] - 1] = i;
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
__global__ void k_scatter_cells(const float4* __restrict__ p, const int32_t* __restrict__ vals,
                                const int32_t* __restrict__ orig_of_slot, int n, const int* __restrict__ leaf_incl,
                                const int* __restrict__ leaf_start, float4* __restrict__ out)
{
  int pos = blockIdx.x * blockDim.x + threadIdx.x;
  if (pos >= n)
    return;
  const int leaf = leaf_incl[pos] - 1;
  const int32_t slot = vals[pos];
  const float4 v = __ldg(p + slot);
  const int32_t oi = orig_of_slot ? orig_of_slot[slot] : slot;
  out[(size_t)leaf * kLeafSize + (pos - leaf_start[leaf])] = make_float4(v.x, v.y, v.z, __int_as_float(oi));
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
  if (i >= n - 1 || !keep[i])
    return;
  const int nid = new_id[i];
  const int2 ch = children[i];
  int ref[2];
  const int c2[2] = {ch.x, ch.y};
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int cc = c2[k];
    if (cc >= 0 && keep[cc]) {
      ref[k] = new_id[cc];
      out_node_parent[new_id[cc]] = nid;
    }
    else {
      const int first = cc >= 0 ? range[cc].x : ~cc;
      const int leaf = leaf_incl[first] - 1;
      ref[k] = ~leaf;
      out_leaf_parent[leaf] = nid;
    }
  }
  out_children[nid] = make_int2(ref[0], ref[1]);
  {
    // a subtree's leaves are consecutive in Morton order: the warp-cooperative k-NN gathers whole cells as one range
    const int fl = leaf_incl[range[i].x] - 1, ll = leaf_incl[range[i].y] - 1;
    out_node_leaves[nid] = make_int2(fl, ll - fl + 1);
  }
  if (i == 0)
    out_node_parent[nid] = -1;
  if (cells.slots == nullptr)
    return;
  // cell table: child C is the deepest node that holds every indexed point of a 3b-bit prefix cell exactly when
  //   prefix_len(this node) < 3b <= prefix_len(C).
  // (Nodes cut INSIDE a run of equal codes have prefix length 63 like their parent and never qualify: only purely
  // spatial cells enter the table.)
  const int l_self = prefix_len63(keys[range[i].x], keys[range[i].y]);
  if (i == 0)  // the root holds every point of the cells its own prefix spans (degenerate frames only)
    for (int b = 1; b <= cells.bmax && 3 * b <= l_self; ++b)
      cell_insert(cells, b, keys[0], nid);
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int cc = c2[k];
    const int first = cc >= 0 ? range[cc].x : ~cc;
    const int last = cc >= 0 ? range[cc].y : ~cc;
    const int l_child = cc >= 0 ? prefix_len63(keys[first], keys[last]) : 63;
    const bool is_leaf = !(cc >= 0 && keep[cc]);
    for (int b = l_self / 3 + 1; b <= cells.bmax; ++b) {  // 3b > l_self
      if (3 * b <= l_child)
        cell_insert(cells, b, keys[first], ref[k]);
      else if (is_leaf)
        // a leaf that spans several level-b cells still holds every indexed point of each of them
        for (int j = first; j <= last; ++j)
          cell_insert(cells, b, keys[j], ref[k]);
      else
        break;  // a kept child with a shorter prefix: its own thread inserts the finer levels
    }
  }
}

// ---- host orchestration -------------------------------------------------------------------------

}  // namespace pclb200
