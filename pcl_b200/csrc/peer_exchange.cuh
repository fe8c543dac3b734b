// peer_exchange.cuh — the device side of the fused cross-rank exchange over the peer-mapped blocks (layout: internal.cuh,
// mappings: comm.cu).  One protocol for both regions of the block: the accumulate kernels' fp64 sums (icp_kernels.cuh)
// and the u64 sums, minima and barriers of the rejector chain on a sharded source (comm.cu: k_peer_u64).
#pragma once
#include "internal.cuh"

namespace pclb200 {

// ~10 s of clock64() on an H100: a peer that has not published by then is dead, and the exchange fails loudly
// (*d_error = kErrPeerTimeout) instead of hanging the GPU
constexpr long long kPeerTimeoutCycles = 20000000000LL;

// the region of rank p's block that carries elements of type T, and its per-rank stride in elements
template <typename T>
struct PeerRegion;
template <>
struct PeerRegion<double> {  // slots[2][kMaxRanks][kAccum]
  static constexpr int kStride = kAccum;
  __device__ __forceinline__ static double* base(const PeerView& v, int p) { return v.slots[p]; }
};
template <>
struct PeerRegion<unsigned long long> {  // words[2][kMaxRanks][kU64Words]
  static constexpr int kStride = kU64Words;
  __device__ __forceinline__ static unsigned long long* base(const PeerView& v, int p)
  {
    return reinterpret_cast<unsigned long long*>(reinterpret_cast<unsigned char*>(v.flags[p]) + kPeerWordsOffset);
  }
};

// Element-wise all-reduce of send[0..count) into recv[0..count) (send == recv is allowed; count <= blockDim.x, 0 = a
// barrier), called by every thread of ONE block on every rank with the same sequence number:
//   1. store this rank's elements into EVERY rank's region[seq & 1][rank][.]   (remote stores)
//   2. fence, then publish seq into every rank's flags[rank]
//   3. wait until all peers have published >= seq in OUR flags, then fold our region[seq & 1][.][i] in rank order,
//      acc = fold(acc, x_r) from acc = init: every rank folds the same numbers in the same order => bitwise identical
//      results everywhere.
// Two parities alternate.  Every rank draws its sequence numbers from one counter in the same order (comm.cu: next_seq),
// so a peer can be at most one exchange ahead (it needs our flag for seq + 1 before it can finish seq + 1) and never
// overwrites the parity we are still reading.
// seq, send, recv and d_error are references: inlined into an accumulate kernel they are read from its parameters where
// they are used, not ahead of the single-rank early return.
template <typename T, typename Fold>
__device__ __forceinline__ void peer_exchange(const PeerView& v, const unsigned long long& seq, const T* const& send,
                                              T* const& recv, int count, T init, Fold fold, int* const& d_error)
{
  typedef PeerRegion<T> R;
  if (v.nranks <= 1)
    return;
  __syncthreads();
  const int buf = (int)(seq & 1ull);
  if (threadIdx.x < (unsigned)count) {
    const T x = send[threadIdx.x];
    for (int p = 0; p < v.nranks; ++p)
      R::base(v, p)[((size_t)buf * kMaxRanks + v.rank) * R::kStride + threadIdx.x] = x;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x < v.nranks)
    *reinterpret_cast<volatile unsigned long long*>(&v.flags[threadIdx.x][v.rank]) = seq;
  __shared__ int timed_out;
  if (threadIdx.x == 0)
    timed_out = 0;
  __syncthreads();
  if (threadIdx.x < v.nranks) {
    const volatile unsigned long long* f = v.flags[v.rank] + threadIdx.x;
    const long long t0 = clock64();
    while (*f < seq) {
      if (clock64() - t0 > kPeerTimeoutCycles) {
        timed_out = 1;
        break;
      }
    }
  }
  __threadfence_system();
  __syncthreads();
  if (timed_out) {
    if (threadIdx.x == 0)
      atomicExch(d_error, kErrPeerTimeout);
  }
  else if (threadIdx.x < (unsigned)count) {
    T acc = init;
    const volatile T* mine = R::base(v, v.rank) + (size_t)buf * kMaxRanks * R::kStride;
    for (int r = 0; r < v.nranks; ++r)
      acc = fold(acc, mine[(size_t)r * R::kStride + threadIdx.x]);
    recv[threadIdx.x] = acc;
  }
}

}  // namespace pclb200
