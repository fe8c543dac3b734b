// shard_sim.h — what the host programs of the sharded map share (include after host_index.h, before the kernel headers):
// the shims of the two device intrinsics the exchange kernels add, the grid launch over the emulated block, the library's
// distance, and comm.cu's exchange tables over ranks simulated in one process.  The placement of the tables comes from
// peer_tables.cuh, as in comm.cu.
//   peer path  every rank's own table (sized to the largest); publish is the barrier
//   NCCL path  every rank's zeroed copy of one table; publish is the u64 sum all-reduce of the copies
#pragma once

template <typename T> static inline T __ldcv(const T* p) { return *p; }
static inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) { const unsigned long long o = *p; if (v < o) *p = v; return o; }

#include "../../pcl_b200/csrc/peer_tables.cuh"

template <typename F> static void launch(unsigned grid, int block, F kernel)
{
  blockDim.x = block;
  gridDim.x = grid ? grid : 1;
  for (unsigned b = 0; b < gridDim.x; ++b) { blockIdx_storage.x = b; warp_emu::run_block(block, kernel); }
  blockIdx_storage.x = 0;
  gridDim.x = 1;
}

// the library's squared distance: ((dx*dx) + dy*dy) + dz*dz, fp32, no fma
static float d2_of(const float4& q, const float4& p)
{
  const float dx = __fsub_rn(q.x, p.x), dy = __fsub_rn(q.y, p.y), dz = __fsub_rn(q.z, p.z);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}
static bool finite3(const float4& p) { return std::isfinite(p.x) && std::isfinite(p.y) && std::isfinite(p.z); }
static int id_of(const float4& p) { return __float_as_int(p.w); }
// a padding slot of a labelled index's point array
static const float4 kPad = make_float4(INFINITY, INFINITY, INFINITY, __int_as_float(kSentinelIndex));

enum { kPeer = 0, kNccl = 1 };

struct SimTables {
  int mode, R;
  bool segments = false;                  // comm_segment_tables (else comm_scratch_tables)
  size_t at[pclb200::kMaxRanks + 1] = {}; // NCCL segment tables: where rank s's table starts in the whole
  std::vector<std::vector<unsigned long long>> mem;  // per rank: its table (peer) or its copy of the whole (NCCL)
  std::vector<unsigned long long> sum;

  SimTables(int mode_, int R_, size_t words) : mode(mode_), R(R_) { alloc(words); }  // comm_scratch_tables
  SimTables(int mode_, int R_, const unsigned long long* n, size_t elem_bytes) : mode(mode_), R(R_), segments(true)
  {
    const size_t most = pclb200::segment_table_words(n, R, elem_bytes, at);
    alloc(mode == kPeer ? most : at[R]);
  }
  void alloc(size_t words)
  {
    mem.assign(R, std::vector<unsigned long long>(std::max<size_t>(words, 1), mode == kPeer ? ~0ull : 0ull));
  }
  // PeerTables::local of rank r
  unsigned long long* local(int r) { return mem[r].data() + (mode == kNccl && segments ? at[r] : 0); }
  // comm_tables_publish on every rank; returns the PeerTables every rank reads
  pclb200::PeerTables publish()
  {
    pclb200::PeerTables t;
    t.peer = mode == kPeer;
    if (mode == kNccl) {
      sum.assign(mem[0].size(), 0ull);
      for (int s = 0; s < R; ++s)
        for (size_t i = 0; i < sum.size(); ++i) sum[i] += mem[s][i];
    }
    t.n_read = mode == kPeer || segments ? R : 1;
    for (int s = 0; s < t.n_read; ++s) t.read[s] = mode == kPeer ? mem[s].data() : sum.data() + (segments ? at[s] : 0);
    return t;
  }
};
