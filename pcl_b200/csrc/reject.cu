// reject.cu — correspondence rejectors on the device (SURVEY.md §8f #1): the stage between correspondence
// estimation and transformation estimation in the ICP loop (registration/include/pcl/registration/impl/icp.hpp:187-201).
//
//   CorrespondenceRejectorDistance        registration/src/correspondence_rejection_distance.cpp:44-68
//       keep distance < max_distance^2 (float, strict), order kept
//   CorrespondenceRejectorMedianDistance  registration/src/correspondence_rejection_median_distance.cpp:44-70
//       median = element n/2 of the sorted distances; keep distance <= median * factor (double), order kept
//   CorrespondenceRejectorOneToOne        registration/src/correspondence_rejection_one_to_one.cpp:44-71
//       sort by (index_match, distance), keep the first of every index_match; output in that order
//   CorrespondenceRejectorTrimmed         registration/src/correspondence_rejection_trimmed.cpp:44-63
//       keep = max(floor(overlap * float(n)), min); if keep < n: sort by distance, keep the first `keep`
// The reference sorts with the unstable std::sort; the canonical tie rule here (and in the oracle) is "earlier in the
// input first", obtained with stable radix sorts.  Inside the ICP loop the input of every rejector is the survivors in
// source-position order (the tie key is the source position), whatever the rejector before it emitted.
//
// All four work on flat per-correspondence arrays {d2, match, tie-break, accepted} so the same code serves the
// stand-alone C entry point (pclb200_reject) and the in-loop form (rejectors applied to the ICP's Match array with no
// host synchronisation: counts, the median and the trim length stay in device memory).
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>

#include "internal.cuh"
#include "reject_kernels.cuh"
#include "reject_sharded_kernels.cuh"

namespace pclb200 {

// TRIMMED's parameters as CorrespondenceRejectorTrimmed stores them (correspondence_rejection_trimmed.h:84, 103-106): the
// overlap ratio as min(1, max(0, float(p))) (NaN gives 0), the minimum count as the unsigned int setMinCorrespondences
// takes (the int32 field's bits, so -1 is 2^32 - 1)
static float trimmed_overlap(const pclb200_rejector& r)
{
  return std::min(1.0f, std::max(0.0f, (float)r.p));
}

static unsigned trimmed_min(const pclb200_rejector& r)
{
  return (unsigned)r.min_correspondences;
}

// Applies one rejector to the arrays.  perm / keep_sorted (nullable, n entries): for ONE_TO_ONE and TRIMMED the sorted
// order of the input positions and which of them survive, so a caller can emit the output in the reference's order.
// d_info (nullable, 2 doubles): [0] median distance.  trimmed_flag (nullable): 1 if TRIMMED actually cut the list.
void apply_rejector(Ctx& c, const pclb200_rejector& r, const RejectArrays& a, int* perm, int* keep_sorted,
                    double* d_info, int* trimmed_flag)
{
  cudaStream_t st = c.stream;
  const size_t n = a.n;
  if (n == 0)
    return;
  PCLB_REQUIRE(n < (size_t)0x7fffffff, PCLB200_ERR_INVALID, "too many correspondences for int32 positions");
  const unsigned g = grid_for(n, 256);
  if (r.kind == PCLB200_REJ_DISTANCE) {
    const float md = (float)r.p * (float)r.p;  // setMaximumDistance stores distance*distance in a float
    k_rej_distance<<<g, 256, 0, st>>>(a.d2, a.acc, n, md);
    ++c.launches;
    return;
  }
  DevBuf<unsigned long long> count;
  count.alloc(1, st);
  PCLB_CUDA(cudaMemsetAsync(count.p, 0, sizeof(unsigned long long), st));
  k_rej_count<<<std::min<unsigned>(g, (unsigned)c.sm_count * 8), 256, 0, st>>>(a.acc, n, count.p);
  ++c.launches;
  if (r.kind == PCLB200_REJ_MEDIAN) {
    DevBuf<unsigned> k_in, k_out;
    DevBuf<double> info;
    k_in.alloc(n, st);
    k_out.alloc(n, st);
    info.alloc(2, st);
    k_rej_keys32<<<g, 256, 0, st>>>(a.d2, a.acc, n, k_in.p);
    size_t tb = 0;
    PCLB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, k_in.p, k_out.p, (int)n, 0, 32, st));
    DevBuf<unsigned char> tmp;
    tmp.alloc(tb, st);
    PCLB_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, tb, k_in.p, k_out.p, (int)n, 0, 32, st));
    k_rej_median<<<1, 1, 0, st>>>(k_out.p, count.p, r.p, info.p);
    k_rej_threshold<<<g, 256, 0, st>>>(a.d2, a.acc, n, info.p);
    c.launches += 8;
    if (d_info)
      PCLB_CUDA(cudaMemcpyAsync(d_info, info.p, 2 * sizeof(double), cudaMemcpyDeviceToDevice, st));
    PCLB_CUDA(cudaGetLastError());
    return;
  }
  // ONE_TO_ONE and TRIMMED start from the (distance, input position) order
  DevBuf<unsigned long long> k64_in, k64_out;
  DevBuf<int> v_in, v_out;
  k64_in.alloc(n, st);
  k64_out.alloc(n, st);
  v_in.alloc(n, st);
  v_out.alloc(n, st);
  k_rej_keys64<<<g, 256, 0, st>>>(a.d2, a.tie, a.acc, n, k64_in.p, v_in.p);
  size_t tb = 0;
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, k64_in.p, k64_out.p, v_in.p, v_out.p, (int)n, 0, 64, st));
  DevBuf<unsigned char> tmp;
  tmp.alloc(tb, st);
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, k64_in.p, k64_out.p, v_in.p, v_out.p, (int)n, 0, 64, st));
  c.launches += 10;
  if (r.kind == PCLB200_REJ_TRIMMED) {
    k_rej_trim<<<g, 256, 0, st>>>(v_out.p, n, count.p, trimmed_overlap(r), trimmed_min(r), a.acc, keep_sorted,
                                  trimmed_flag);
    ++c.launches;
    if (perm)
      PCLB_CUDA(cudaMemcpyAsync(perm, v_out.p, n * sizeof(int), cudaMemcpyDeviceToDevice, st));
    PCLB_CUDA(cudaGetLastError());
    return;
  }
  PCLB_REQUIRE(r.kind == PCLB200_REJ_ONE_TO_ONE, PCLB200_ERR_INVALID, "unknown rejector kind");
  DevBuf<unsigned> m_in, m_out;
  DevBuf<int> v2;
  m_in.alloc(n, st);
  m_out.alloc(n, st);
  v2.alloc(n, st);
  k_rej_gather_match<<<g, 256, 0, st>>>(a.match, a.acc, v_out.p, n, m_in.p);
  size_t tb2 = 0;
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb2, m_in.p, m_out.p, v_out.p, v2.p, (int)n, 0, 32, st));
  DevBuf<unsigned char> tmp2;
  tmp2.alloc(tb2, st);
  PCLB_CUDA(cub::DeviceRadixSort::SortPairs(tmp2.p, tb2, m_in.p, m_out.p, v_out.p, v2.p, (int)n, 0, 32, st));  // stable
  k_rej_heads<<<g, 256, 0, st>>>(m_out.p, v2.p, n, count.p, a.acc, keep_sorted);
  c.launches += 7;
  if (perm)
    PCLB_CUDA(cudaMemcpyAsync(perm, v2.p, n * sizeof(int), cudaMemcpyDeviceToDevice, st));
  PCLB_CUDA(cudaGetLastError());
}

// ---- the same rejectors over the union of every rank's arrays (sharded source, DESIGN.md §5) ---------------------------
// DISTANCE and SURFACE_NORMAL are per correspondence: the caller applies them locally.  The others exchange only what
// their decision needs: MEDIAN 4 and TRIMMED 8 histogram sums (one per 8-bit digit of the 32- / 64-bit key); ONE_TO_ONE
// one table exchange (peer path: two barriers around the peer reads; NCCL: one min all-reduce of the table).  A rank with
// no accepted correspondence, or none at all, still takes part in every exchange.
void apply_rejector_sharded(Ctx& c, const pclb200_rejector& r, const RejectArrays& a, const ShardedRejectArgs& s)
{
  cudaStream_t st = c.stream;
  const size_t n = a.n;
  PCLB_REQUIRE(n < (size_t)0x7fffffff, PCLB200_ERR_INVALID, "too many correspondences for int32 positions");
  const unsigned g = std::max(1u, grid_for(n, 256));
  if (r.kind == PCLB200_REJ_MEDIAN || r.kind == PCLB200_REJ_TRIMMED) {
    const bool wide = r.kind == PCLB200_REJ_TRIMMED;
    const int passes = (wide ? 64 : 32) / kSelDigitBits;
    DevBuf<unsigned long long> hist;
    DevBuf<SelState> sel;
    DevBuf<double> info;
    hist.alloc(kSelBins, st);
    sel.alloc(1, st);
    info.alloc(2, st);
    PCLB_CUDA(cudaMemsetAsync(hist.p, 0, kSelBins * sizeof(unsigned long long), st));
    PCLB_CUDA(cudaMemsetAsync(sel.p, 0, sizeof(SelState), st));
    const unsigned hg = std::min<unsigned>(g, (unsigned)c.sm_count * 4);
    for (int p = 0; p < passes; ++p) {
      const int shift = (passes - 1 - p) * kSelDigitBits;
      if (wide)
        k_sel_hist<true><<<hg, 256, 0, st>>>(a.d2, a.tie, a.acc, n, s.offset, shift, p == 0, sel.p, hist.p);
      else
        k_sel_hist<false><<<hg, 256, 0, st>>>(a.d2, a.tie, a.acc, n, s.offset, shift, p == 0, sel.p, hist.p);
      comm_allreduce_u64(c, hist.p, hist.p, kSelBins, kU64Sum);
      k_sel_decide<<<1, 1, 0, st>>>(hist.p, shift, p == 0, p == passes - 1, r.kind, trimmed_overlap(r), trimmed_min(r),
                                    r.p, sel.p, info.p);
      c.launches += 2;
    }
    if (wide)
      k_sel_trim_apply<<<g, 256, 0, st>>>(a.d2, a.tie, a.acc, n, s.offset, sel.p);
    else
      k_rej_threshold<<<g, 256, 0, st>>>(a.d2, a.acc, n, info.p);
    ++c.launches;
    PCLB_CUDA(cudaGetLastError());
    return;
  }
  PCLB_REQUIRE(r.kind == PCLB200_REJ_ONE_TO_ONE, PCLB200_ERR_INVALID, "rejector kind has no sharded form");
  const PeerTables t = comm_peer_tables(c, *s.o2o, s.n_cloud);
  k_o2o_min<<<g, 256, 0, st>>>(a.d2, a.tie, a.match, a.acc, n, s.offset, s.tgt_pts, t.local);
  comm_tables_publish(c, t, kU64Min);
  k_o2o_keep<<<g, 256, 0, st>>>(a.d2, a.tie, a.match, a.acc, n, s.offset, s.tgt_pts, peer_table_set(t));
  comm_tables_release(c, t);  // no peer still reads this rank's table: the sparse reset may follow
  k_o2o_reset<<<g, 256, 0, st>>>(a.match, n, s.tgt_pts, t.local);
  c.launches += 3;
  PCLB_CUDA(cudaGetLastError());
}

// ---- stand-alone entry point -----------------------------------------------------------------------------------------
size_t reject_standalone(Ctx& c, const pclb200_rejector& r, const pclb200_corr* in, size_t n, pclb200_corr* out,
                         double* median_out)
{
  cudaStream_t st = c.stream;
  if (median_out)
    *median_out = 0.0;
  if (n == 0)
    return 0;
  DevBuf<pclb200_corr> d_in, staged;
  const pclb200_corr* din = on_device(c, in, n, d_in);
  DevBuf<float> d2;
  DevBuf<int> match, acc, perm, keep_sorted, trimmed;
  DevBuf<unsigned> tie;
  DevBuf<double> info;
  d2.alloc(n, st);
  match.alloc(n, st);
  acc.alloc(n, st);
  tie.alloc(n, st);
  perm.alloc(n, st);
  keep_sorted.alloc(n, st);
  trimmed.alloc(1, st);
  info.alloc(2, st);
  PCLB_CUDA(cudaMemsetAsync(trimmed.p, 0, sizeof(int), st));
  PCLB_CUDA(cudaMemsetAsync(info.p, 0, 2 * sizeof(double), st));
  k_rej_unpack<<<grid_for(n, 256), 256, 0, st>>>(din, n, d2.p, match.p, tie.p, acc.p,
                                                r.kind == PCLB200_REJ_ONE_TO_ONE ? 1 : 0);
  ++c.launches;
  RejectArrays a;
  a.n = n;
  a.d2 = d2.p;
  a.match = match.p;
  a.tie = tie.p;
  a.acc = acc.p;
  apply_rejector(c, r, a, perm.p, keep_sorted.p, info.p, trimmed.p);
  int h_trim = 0;
  double h_info[2] = {0, 0};
  PCLB_CUDA(cudaMemcpyAsync(&h_trim, trimmed.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaMemcpyAsync(h_info, info.p, sizeof(h_info), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  if (median_out)
    *median_out = h_info[0];
  // output order: input order for DISTANCE / MEDIAN (and an un-trimmed TRIMMED), sorted order otherwise
  const int use_perm = (r.kind == PCLB200_REJ_ONE_TO_ONE) || (r.kind == PCLB200_REJ_TRIMMED && h_trim);
  staged.alloc(n, st);
  DevBuf<unsigned char> flag;
  flag.alloc(n, st);
  k_rej_flag_in_order<<<grid_for(n, 256), 256, 0, st>>>(acc.p, perm.p, keep_sorted.p, n, use_perm, din, staged.p, flag.p);
  ++c.launches;
  const size_t m = compact_corr_to(c, staged.p, flag.p, n, out);
  PCLB_CUDA(cudaStreamSynchronize(st));
  return m;
}

}  // namespace pclb200
