// reject_twin.h — reject.cu's apply_rejector() on host memory: the kernels of pcl_b200/csrc/reject_kernels.cuh in the driver's
// sequence, std::stable_sort where the driver calls cub::DeviceRadixSort (both stable).  Shared by reject_host_test.cpp (the
// stand-alone entry point) and icp_host_test.cpp (the chain inside the ICP loop).  Include after host_index.h / warp_emu.h.
#pragma once
#include <numeric>

#ifndef PCLB_HOST_FLOAT_BITS
#define PCLB_HOST_FLOAT_BITS
static inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(unsigned u) { float f; std::memcpy(&f, &u, 4); return f; }
#endif

#include "../../pcl_b200/csrc/reject_kernels.cuh"

template <typename F> static void launch(unsigned grid, int block, F kernel)
{
  blockDim.x = block;
  gridDim.x = grid ? grid : 1;
  for (unsigned b = 0; b < gridDim.x; ++b) { blockIdx_storage.x = b; warp_emu::run_block(block, kernel); }
  blockIdx_storage.x = 0;
  gridDim.x = 1;
}
static unsigned grid_for(size_t n, int block) { return (unsigned)((n + block - 1) / block); }

struct Arrays { std::vector<float> d2; std::vector<int> match, acc; std::vector<unsigned> tie; };

// reject.cu: apply_rejector()
static void apply_rejector(const pclb200_rejector& r, Arrays& a, std::vector<int>& perm, std::vector<int>& keep_sorted, double info[2], int& trimmed_flag)
{
  using namespace pclb200;
  const size_t n = a.d2.size();
  if (n == 0) return;
  const unsigned g = grid_for(n, 256);
  if (r.kind == PCLB200_REJ_DISTANCE) {
    const float md = (float)r.p * (float)r.p;
    launch(g, 256, [&] { k_rej_distance(a.d2.data(), a.acc.data(), n, md); });
    return;
  }
  unsigned long long count = 0;
  launch(std::min<unsigned>(g, 132 * 8), 256, [&] { k_rej_count(a.acc.data(), n, &count); });
  if (r.kind == PCLB200_REJ_MEDIAN) {
    std::vector<unsigned> k_in(n), k_out;
    launch(g, 256, [&] { k_rej_keys32(a.d2.data(), a.acc.data(), n, k_in.data()); });
    k_out = k_in;
    std::stable_sort(k_out.begin(), k_out.end());
    k_rej_median(k_out.data(), &count, r.p, info);   // <<<1, 1>>>: no thread index, no collective
    launch(g, 256, [&] { k_rej_threshold(a.d2.data(), a.acc.data(), n, info); });
    return;
  }
  std::vector<unsigned long long> k64(n);
  std::vector<int> v_in(n), v_out(n);
  launch(g, 256, [&] { k_rej_keys64(a.d2.data(), a.tie.data(), a.acc.data(), n, k64.data(), v_in.data()); });
  {
    std::vector<int> order(n);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return k64[x] < k64[y]; });
    for (size_t j = 0; j < n; ++j) v_out[j] = v_in[order[j]];
  }
  if (r.kind == PCLB200_REJ_TRIMMED) {
    const float overlap = std::min(1.0f, std::max(0.0f, (float)r.p));  // reject.cu: trimmed_overlap / trimmed_min
    launch(g, 256, [&] { k_rej_trim(v_out.data(), n, &count, overlap, (unsigned)r.min_correspondences, a.acc.data(), keep_sorted.data(), &trimmed_flag); });
    perm = v_out;
    return;
  }
  std::vector<unsigned> m_in(n), m_out(n);
  std::vector<int> v2(n);
  launch(g, 256, [&] { k_rej_gather_match(a.match.data(), a.acc.data(), v_out.data(), n, m_in.data()); });
  {
    std::vector<int> order(n);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return m_in[x] < m_in[y]; });
    for (size_t j = 0; j < n; ++j) { m_out[j] = m_in[order[j]]; v2[j] = v_out[order[j]]; }
  }
  launch(g, 256, [&] { k_rej_heads(m_out.data(), v2.data(), n, &count, a.acc.data(), keep_sorted.data()); });
  perm = v2;
}

