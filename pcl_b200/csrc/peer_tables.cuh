// peer_tables.cuh — what a kernel reads out of the tables of comm.cu (comm_peer_tables, comm_scratch_tables,
// comm_segment_tables), and the layout of the exchanges that move segments through them (the halo of shard_normals.cu, the
// label answers of shard_cluster.cu, allgather_u64).
//   PeerTableSet       one table per rank, read at the same index: every rank's (peer path) or their NCCL reduction
//   PeerSegments       segments of tables read one after the other as one array
//   k_gather_segments  copies a PeerSegments set into a dense array (and a local array into a table, as one segment)
// Segment layout: rank s sends cnt[s R + r] elements to each other rank r (the diagonal is never sent).  Rank s's table
// holds its segments by destination, end to end, the one for r at the sum of cnt[s R + x] over x < r, x != s;
// comm_segment_tables gives every rank's table at read[s] on both paths.  The host functions below are the only copy of
// that arithmetic: the drivers and tests/host call them.  A header of its own, including only internal.cuh, so that the
// host tests compile it as they compile the kernel headers.
#pragma once
#include "internal.cuh"

namespace pclb200 {

template <typename T>
struct PeerTableSet {
  int n;
  const T* t[kMaxRanks];
};

// the tables a kernel reads from t: t.read[0 .. t.n_read)
template <typename T = unsigned long long>
inline PeerTableSet<T> peer_table_set(const PeerTables& t)
{
  PeerTableSet<T> s = {};
  s.n = t.n_read;
  for (int p = 0; p < t.n_read; ++p)
    s.t[p] = reinterpret_cast<const T*>(t.read[p]);
  return s;
}

// Segments read one after the other: segment s holds begin[s + 1] - begin[s] entries at src[s].
template <typename T>
struct PeerSegments {
  int n;
  const T* src[kMaxRanks];
  unsigned long long begin[kMaxRanks + 1];
};

// entry i of the concatenation (peer tables: read through to memory, never a stale cached line)
template <typename T>
__device__ __forceinline__ T peer_segment_read(const PeerSegments<T>& rs, unsigned long long i)
{
  int s = 0;
  while (i >= rs.begin[s + 1])
    ++s;
  return __ldcv(rs.src[s] + (i - rs.begin[s]));
}

template <typename T>
__global__ void __launch_bounds__(256)
k_gather_segments(const PeerSegments<T> rs, T* __restrict__ out)
{
  const unsigned long long total = rs.begin[rs.n];
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < total;
       i += (unsigned long long)gridDim.x * blockDim.x)
    out[i] = peer_segment_read(rs, i);
}

// ---- the segment layout (host) ----------------------------------------------------------------------------------------
// where rank s's segment for rank r starts in s's table (r == R: the size of s's table)
inline unsigned long long segment_start(const unsigned long long* cnt, int R, int s, int r)
{
  unsigned long long at = 0;
  for (int x = 0; x < r; ++x)
    if (x != s)
      at += cnt[(size_t)s * R + x];
  return at;
}

// every rank's table size, the counts comm_segment_tables takes
inline std::vector<unsigned long long> segment_table_sizes(const unsigned long long* cnt, int R)
{
  std::vector<unsigned long long> n(R);
  for (int s = 0; s < R; ++s)
    n[s] = segment_start(cnt, R, s, R);
  return n;
}

// comm_segment_tables' tables of n[s] elements of elem_bytes in u64 words: at[s] = where rank s's table starts when they
// lie end to end (NCCL path; at[R] = the whole); returns the largest (the size of each peer path table)
inline size_t segment_table_words(const unsigned long long* n, int R, size_t elem_bytes, size_t* at)
{
  size_t most = 0;
  at[0] = 0;
  for (int s = 0; s < R; ++s) {
    const size_t words = (size_t)((n[s] * elem_bytes + 7) / 8);
    at[s + 1] = at[s] + words;
    most = std::max(most, words);
  }
  return most;
}

// the counts of the answers: rank r answers the cnt[s R + r] points it received from s
inline std::vector<unsigned long long> segment_answers(const std::vector<unsigned long long>& cnt, int R)
{
  std::vector<unsigned long long> a((size_t)R * R);
  for (int s = 0; s < R; ++s)
    for (int r = 0; r < R; ++r)
      a[(size_t)r * R + s] = cnt[(size_t)s * R + r];
  return a;
}

// where rank me writes its segment for each other rank r into its table `mine` (dst[me] is left alone)
template <typename T>
inline void segment_writes(T* mine, const unsigned long long* cnt, int R, int me, T* dst[])
{
  for (int r = 0; r < R; ++r)
    if (r != me)
      dst[r] = mine + segment_start(cnt, R, me, r);
}

// the segments rank me receives, by sender, out of every rank's table
template <typename T>
inline PeerSegments<T> segment_reads(const PeerTables& t, const unsigned long long* cnt, int R, int me)
{
  PeerSegments<T> rs = {};
  for (int s = 0; s < R; ++s) {
    if (s == me)
      continue;
    rs.src[rs.n] = reinterpret_cast<const T*>(t.read[s]) + segment_start(cnt, R, s, me);
    rs.begin[rs.n + 1] = rs.begin[rs.n] + cnt[(size_t)s * R + me];
    ++rs.n;
  }
  return rs;
}

// the first n[s] elements of every rank's table, in rank order: an all-gather
template <typename T>
inline PeerSegments<T> table_runs(const PeerTables& t, const unsigned long long* n)
{
  PeerSegments<T> rs = {};
  rs.n = t.n_read;
  for (int s = 0; s < t.n_read; ++s) {
    rs.src[s] = reinterpret_cast<const T*>(t.read[s]);
    rs.begin[s + 1] = rs.begin[s] + n[s];
  }
  return rs;
}

// one array as a set of one segment (a copy into a table with k_gather_segments)
template <typename T>
inline PeerSegments<T> one_segment(const T* src, unsigned long long n)
{
  PeerSegments<T> rs = {};
  rs.n = 1;
  rs.src[0] = src;
  rs.begin[1] = n;
  return rs;
}

#ifdef __CUDACC__
// rs's segments one after the other into out, on the ctx stream (nothing when they are empty)
template <typename T>
void gather_segments(Ctx& c, const PeerSegments<T>& rs, T* out)
{
  const unsigned long long total = rs.begin[rs.n];
  if (!total)
    return;
  k_gather_segments<T><<<persistent_blocks(c, total), 256, 0, c.stream>>>(rs, out);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}
#endif

}  // namespace pclb200
