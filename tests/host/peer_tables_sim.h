// peer_tables_sim.h — comm.cu's exchange tables over ranks simulated in one process, for the host tests of the sharded map
// (include after pcl_b200/csrc/peer_tables.cuh).  The placement of the tables comes from peer_tables.cuh, as in comm.cu.
//   peer path  every rank's own table (sized to the largest); publish is the barrier
//   NCCL path  every rank's zeroed copy of one table; publish is the u64 sum all-reduce of the copies
#pragma once

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
