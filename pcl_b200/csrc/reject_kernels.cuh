// reject_kernels.cuh — the kernels of the correspondence rejectors (driver: reject.cu), in a header of their own so that
// tests/host/reject_host_test.cpp can compile them for the host and replay reject.cu's sequence against the oracle.
#pragma once
#include "internal.cuh"

namespace pclb200 {

__global__ void k_rej_count(const int* __restrict__ acc, size_t n, unsigned long long* __restrict__ count)
{
  unsigned c = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    c += acc[i] ? 1u : 0u;
  for (int o = 16; o > 0; o >>= 1)
    c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c)
    atomicAdd(count, (unsigned long long)c);
}

__global__ void k_rej_distance(const float* __restrict__ d2, int* __restrict__ acc, size_t n, float max_d2)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n && acc[i] && !(d2[i] < max_d2))
    acc[i] = 0;
}

// A caller's list may hold any non-NaN distance: -0.0 becomes +0.0 (the reference compares them equal), then the sign
// flip makes the unsigned order of the bits the order of the values, negatives and +inf included.
__device__ __forceinline__ unsigned rej_key(float d)
{
  const unsigned u = __float_as_uint(d) == 0x80000000u ? 0u : __float_as_uint(d);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float rej_key_value(unsigned k)
{
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__global__ void k_rej_keys32(const float* __restrict__ d2, const int* __restrict__ acc, size_t n,
                             unsigned* __restrict__ keys)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n)
    keys[i] = acc[i] ? rej_key(d2[i]) : 0xffffffffu;
}

// median = sorted[count / 2]; threshold = median * factor in double (correspondence_rejection_median_distance.cpp:57-65)
__global__ void k_rej_median(const unsigned* __restrict__ sorted, const unsigned long long* __restrict__ count,
                             double factor, double* __restrict__ out /* [0] median, [1] threshold */)
{
  const unsigned long long c = *count;
  if (c == 0) {
    out[0] = 0.0;
    out[1] = -1.0;
    return;
  }
  const double med = (double)rej_key_value(sorted[c / 2]);
  out[0] = med;
  out[1] = med * factor;
}

__global__ void k_rej_threshold(const float* __restrict__ d2, int* __restrict__ acc, size_t n,
                                const double* __restrict__ thr)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n && acc[i] && !((double)d2[i] <= thr[1]))
    acc[i] = 0;
}

// (distance, input position) key: ascending distance, ties by input order
__global__ void k_rej_keys64(const float* __restrict__ d2, const unsigned* __restrict__ tie, const int* __restrict__ acc,
                             size_t n, unsigned long long* __restrict__ keys, int* __restrict__ vals)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  keys[i] = acc[i] ? (((unsigned long long)rej_key(d2[i]) << 32) | tie[i]) : ~0ULL;
  vals[i] = (int)i;
}

__global__ void k_rej_gather_match(const int* __restrict__ match, const int* __restrict__ acc, const int* __restrict__ vals,
                                   size_t n, unsigned* __restrict__ keys)
{
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n)
    return;
  const int i = vals[j];
  keys[j] = acc[i] ? (unsigned)match[i] : 0xffffffffu;
}

// after the stable sort by match: keep the first entry of every run
__global__ void k_rej_heads(const unsigned* __restrict__ mkeys, const int* __restrict__ vals, size_t n,
                            const unsigned long long* __restrict__ count, int* __restrict__ acc,
                            int* __restrict__ keep_sorted)
{
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n)
    return;
  const bool live = j < *count;
  const bool head = live && (j == 0 || mkeys[j] != mkeys[j - 1]);
  if (live)
    acc[vals[j]] = head ? 1 : 0;
  if (keep_sorted)
    keep_sorted[j] = head ? 1 : 0;
}

// trimmed: entry j of the distance-sorted list survives iff j < keep, keep = max(floor(overlap * float(count)), min)
__global__ void k_rej_trim(const int* __restrict__ vals, size_t n, const unsigned long long* __restrict__ count,
                           float overlap, unsigned min_corr, int* __restrict__ acc, int* __restrict__ keep_sorted,
                           int* __restrict__ trimmed_flag)
{
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  const unsigned long long c = *count;
  unsigned long long keep = (unsigned long long)floorf(overlap * (float)c);
  if (keep < min_corr)
    keep = min_corr;
  const bool trim = keep < c;
  if (j == 0 && trimmed_flag)
    *trimmed_flag = trim ? 1 : 0;
  if (j >= n)
    return;
  const bool live = j < c;
  if (live && trim)
    acc[vals[j]] = j < keep ? 1 : 0;
  if (keep_sorted)
    keep_sorted[j] = live && (!trim || j < keep) ? 1 : 0;
}

// ---- stand-alone entry point: unpack the records, emit the survivors in the reference's order ---------------------------
__global__ void k_rej_unpack(const pclb200_corr* __restrict__ in, size_t n, float* __restrict__ d2, int* __restrict__ match,
                             unsigned* __restrict__ tie, int* __restrict__ acc, int drop_negative)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const pclb200_corr c = in[i];
  d2[i] = c.distance;
  match[i] = c.index_match;
  tie[i] = (unsigned)i;
  acc[i] = (drop_negative && c.index_match < 0) ? 0 : 1;
}

__global__ void k_rej_flag_in_order(const int* __restrict__ acc, const int* __restrict__ perm,
                                    const int* __restrict__ keep_sorted, size_t n, int use_perm,
                                    const pclb200_corr* __restrict__ in, pclb200_corr* __restrict__ staged,
                                    unsigned char* __restrict__ flag)
{
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n)
    return;
  if (use_perm) {
    staged[j] = in[perm[j]];
    flag[j] = keep_sorted[j] ? 1 : 0;
  }
  else {
    staged[j] = in[j];
    flag[j] = acc[j] ? 1 : 0;
  }
}

}  // namespace pclb200
