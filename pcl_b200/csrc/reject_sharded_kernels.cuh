// reject_sharded_kernels.cuh — the rejectors that need the whole correspondence set (median, trimmed, one-to-one) on a
// source sharded across ranks (driver: reject.cu, apply_rejector_sharded).  Every rank reaches the decision a single
// process makes over the concatenation of the shards in rank order, without gathering the shards:
//   median / trimmed: one global order statistic by radix select, 8-bit digits from the most significant one; per digit
//     a histogram of this rank's candidates (k_sel_hist), the cross-rank sum (comm.cu), and a one-thread decision
//     (k_sel_decide) that fixes the digit and the rank left inside the chosen bin, in device memory;
//   one-to-one: per target record the smallest (distance, global position) key over all ranks, through one u64 table per
//     rank (k_o2o_min / k_o2o_keep / k_o2o_reset).
// Keys: median d2 bits (32-bit); trimmed and one-to-one (d2 bits << 32) | (offset + slot), unique, ordered like the
// single process's (distance, input position) sort: the loop's squared distances are never negative or -0.0, so their
// raw bits order like reject_kernels.cuh's rej_key.  A header of its own so that tests/host/reject_sharded_host_test.cpp
// can compile the kernels for the host and simulate several ranks in one process.
#pragma once
#include "internal.cuh"
#include "peer_tables.cuh"

namespace pclb200 {

constexpr int kSelDigitBits = 8;
constexpr int kSelBins = 1 << kSelDigitBits;
static_assert(kSelBins <= kU64Words, "a histogram must fit the peer block's u64 region");

struct SelState {
  unsigned long long prefix;  // key bits fixed so far (the selected key once every digit is decided)
  unsigned long long rank;    // rank of the wanted key among the keys that share the prefix
  unsigned long long count;   // global number of accepted entries (the first pass's histogram total)
  int active;                 // 1: a key is being selected; 0: median of nothing / trimmed keeps everything
  int reject_all;             // median of nothing, or trimmed to keep = 0
};

template <bool WIDE>
__device__ __forceinline__ unsigned long long sel_key(const float* d2, const unsigned* tie, size_t i, unsigned long long offset)
{
  const unsigned long long b = (unsigned long long)__float_as_uint(d2[i]);
  return WIDE ? ((b << 32) | (offset + tie[i])) : b;
}

// histogram of the digit at `shift` over the accepted entries whose higher digits equal the prefix (pass 0: all of them);
// shared-memory bins, one global flush per block
template <bool WIDE>
__global__ void __launch_bounds__(256)
k_sel_hist(const float* __restrict__ d2, const unsigned* __restrict__ tie, const int* __restrict__ acc, size_t n,
           unsigned long long offset, int shift, int first, const SelState* __restrict__ st, unsigned long long* __restrict__ hist)
{
  __shared__ unsigned bins[kSelBins];
  for (int b = threadIdx.x; b < kSelBins; b += blockDim.x)
    bins[b] = 0;
  __syncthreads();
  const bool run = first || st->active;
  const unsigned long long high = first ? 0ull : st->prefix >> (shift + kSelDigitBits);
  if (run) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
      if (!acc[i])
        continue;
      const unsigned long long k = sel_key<WIDE>(d2, tie, i, offset);
      if (first || (k >> (shift + kSelDigitBits)) == high)
        atomicAdd(&bins[(unsigned)(k >> shift) & (kSelBins - 1)], 1u);
    }
  }
  __syncthreads();
  for (int b = threadIdx.x; b < kSelBins; b += blockDim.x)
    if (bins[b])
      atomicAdd(&hist[b], (unsigned long long)bins[b]);
}

// <<<1, 1>>> after the cross-rank sum of `hist`: on the first pass derives the global count and the wanted rank
//   MEDIAN : rank c / 2 (k_rej_median); c == 0 rejects everything
//   TRIMMED: keep = max(floorf(overlap * (float)c), min) (k_rej_trim); keep >= c keeps everything, keep == 0 rejects all,
//            otherwise the key of rank keep - 1 is the largest survivor
// then fixes the digit at `shift` and clears `hist` for the next pass.  On the last MEDIAN pass writes info = {median,
// median * factor} (k_rej_threshold's input; {0, -1} when c == 0).
__global__ void k_sel_decide(unsigned long long* __restrict__ hist, int shift, int first, int last, int kind, float overlap,
                             unsigned min_corr, double factor, SelState* __restrict__ st, double* __restrict__ info)
{
  SelState s = *st;
  if (first) {
    unsigned long long c = 0;
    for (int b = 0; b < kSelBins; ++b)
      c += hist[b];
    s.prefix = 0;
    s.count = c;
    s.active = 0;
    s.reject_all = 0;
    s.rank = 0;
    if (kind == PCLB200_REJ_MEDIAN) {
      if (c == 0)
        s.reject_all = 1;
      else {
        s.active = 1;
        s.rank = c / 2;
      }
    }
    else {
      unsigned long long keep = (unsigned long long)floorf(overlap * (float)c);
      if (keep < min_corr)
        keep = min_corr;
      if (keep < c) {
        if (keep == 0)
          s.reject_all = 1;
        else {
          s.active = 1;
          s.rank = keep - 1;
        }
      }
    }
  }
  if (s.active) {
    unsigned long long below = 0;
    int d = 0;
    for (; d < kSelBins - 1; ++d) {
      if (below + hist[d] > s.rank)
        break;
      below += hist[d];
    }
    s.rank -= below;
    s.prefix |= (unsigned long long)d << shift;
  }
  for (int b = 0; b < kSelBins; ++b)
    hist[b] = 0;
  *st = s;
  if (last && kind == PCLB200_REJ_MEDIAN) {
    if (s.active) {
      const double med = (double)__uint_as_float((unsigned)s.prefix);
      info[0] = med;
      info[1] = med * factor;
    }
    else {
      info[0] = 0.0;
      info[1] = -1.0;
    }
  }
}

// trimmed: an accepted entry survives iff its key is <= the selected key
__global__ void k_sel_trim_apply(const float* __restrict__ d2, const unsigned* __restrict__ tie, int* __restrict__ acc,
                                 size_t n, unsigned long long offset, const SelState* __restrict__ st)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n || !acc[i])
    return;
  if (st->reject_all || (st->active && sel_key<true>(d2, tie, i, offset) > st->prefix))
    acc[i] = 0;
}

// one-to-one, step 1: the smallest key per target record (original index, so independent of the index build)
__global__ void k_o2o_min(const float* __restrict__ d2, const unsigned* __restrict__ tie, const int* __restrict__ mt,
                          const int* __restrict__ acc, size_t n, unsigned long long offset, const float4* __restrict__ tgt_pts,
                          unsigned long long* __restrict__ table)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n || !acc[i])
    return;
  const int t = __float_as_int(tgt_pts[mt[i]].w);
  atomicMin(&table[t], sel_key<true>(d2, tie, i, offset));
}

// step 2 (after the barrier / the min all-reduce): an entry survives iff no table holds a smaller key for its target
__global__ void k_o2o_keep(const float* __restrict__ d2, const unsigned* __restrict__ tie, const int* __restrict__ mt,
                           int* __restrict__ acc, size_t n, unsigned long long offset, const float4* __restrict__ tgt_pts,
                           const PeerTableSet<unsigned long long> tabs)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n || !acc[i])
    return;
  const int t = __float_as_int(tgt_pts[mt[i]].w);
  const unsigned long long k = sel_key<true>(d2, tie, i, offset);
  for (int p = 0; p < tabs.n; ++p)
    if (__ldcv(tabs.t[p] + t) < k) {  // peer tables: read through to memory, never a stale cached line
      acc[i] = 0;
      return;
    }
}

// step 3 (after the second barrier): back to ~0 every entry this rank may have written (every matched entry: a superset
// of those that were accepted at step 1; the others were ~0 already)
__global__ void k_o2o_reset(const int* __restrict__ mt, size_t n, const float4* __restrict__ tgt_pts,
                            unsigned long long* __restrict__ table)
{
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n || mt[i] < 0)
    return;
  table[__float_as_int(tgt_pts[mt[i]].w)] = ~0ull;
}

}  // namespace pclb200
