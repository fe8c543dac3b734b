// shard_voxel.cu — VoxelGrid over a map sharded across the ranks of a communicator (pclb200_voxelgrid_sharded, capi.cu).
// Every rank passes its records and their ids; the output is voxelgrid() (voxel.cu) of the whole map with indices = the
// union of the ids in ascending order, byte for byte, each voxel returned by one rank (DESIGN.md §5, "VoxelGrid of a
// sharded map").
//
//   boxes      every rank checks its arguments and ids, and takes the min / max of its finite records (k_vg_minmax); its
//              verdict, its parameters and its box travel in one u64 minimum.  Every rank then knows every rank's box
//              and the union box, from which vg_grid gives the whole map's grid, guard included.  Every refusal happens
//              here, on every rank, before any record moves.
//   exchange   I_s = the voxel coordinates of rank s's box faces.  Every rank sends every finite record whose voxel lies
//              in I_s to rank s: one u64 sum of the R x R counts, then one segment per destination in the tables of
//              comm_segment_tables, publish, k_gather_segments, release (the protocol of the halo of shard_normals.cu).
//              A rank that holds a record of voxel v has v in its own I, so it receives every other rank's records of v.
//   centroids  own and received records sorted by (voxel << 32) | id, equal keys (one id held twice) dropped; per voxel
//              the mask of the ranks holding a record of it.  The owner, member v mod |mask| of the mask, returns the
//              voxel when its complete run has min_pts records: that run is the whole map's in id order, and the
//              unchanged k_vg_runs / k_vg_centroids / k_vg_normals reduce it in voxelgrid()'s order.
#include <cub/cub.cuh>

#include <cmath>
#include <vector>

#include "internal.cuh"
#include "peer_tables.cuh"
#include "shard_voxel_kernels.cuh"

namespace pclb200 {

bool comm_active(const Ctx& c);
int comm_nranks(const Ctx& c);
int comm_rank(const Ctx& c);

// the reason this rank refuses the call, or nullptr; d_ids receives the ids on the device when they are checked
static const char* local_fault(Ctx& c, const void* pts, size_t n, size_t stride, const int32_t* ids, const void* normals,
                               size_t stride_n,
                               const float leaf[3], const float* out_xyz1, const float* out_normal_curv,
                               const uint32_t* out_voxel, const size_t* n_out, DevBuf<int32_t>& staging,
                               const int32_t** d_ids)
{
  if (!leaf || !out_xyz1 || !out_voxel || !n_out || (n && (!pts || !ids)))
    return "NULL argument";
  for (int a = 0; a < 3; ++a)
    if (!(std::isfinite(leaf[a]) && leaf[a] > 0.f))
      return "leaf size must be positive and finite";
  if ((normals != nullptr) != (out_normal_curv != nullptr))
    return "out_normal_curv must be given exactly when normals are";
  if (n && (stride < 12 || stride % 4 != 0))  // an empty rank reads no record
    return "stride must be a multiple of 4 and >= 12";
  if (normals && n && (stride_n < 20 || stride_n % 4 != 0))
    return "normal stride must be a multiple of 4 and >= 20";
  if (n >= (size_t)0x7fffffff)
    return "more than 2^31 - 2 records on one rank";
  *d_ids = on_device(c, ids, n, staging);
  const int f = id_faults(c, *d_ids, n);
  if (f & kIdOutOfRange)
    return "every id must lie in [0, 2^31 - 2]";
  if (f & kIdRepeated)
    return "two records of this rank carry the same id";
  return nullptr;
}

size_t voxelgrid_sharded(Ctx& c, const void* pts, size_t n, size_t stride, const int32_t* ids, const void* normals,
                         size_t stride_n, const float leaf[3], unsigned min_pts, float* out_xyz1, float* out_normal_curv,
                         uint32_t* out_voxel, size_t* n_out)
{
  cudaStream_t st = c.stream;
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID,
               "voxelgrid_sharded needs an active communicator (pclb200_comm_init or pclb200_comm_export / _import)");
  const int R = comm_nranks(c), me = comm_rank(c);
  const bool with_normals = normals != nullptr;
  const int per = sv_units(with_normals);

  // ---- boxes --------------------------------------------------------------------------------------------------------
  DevBuf<float4> dense, nc;
  DevBuf<int32_t> ids_staging;
  const int32_t* d_ids = nullptr;
  SvBoxes boxes = {};
  float mn[3], mx[3];
  bool any = false;
  {
    ProfScope ps(c, "sharded_voxel_boxes");
    const char* fault = local_fault(c, pts, n, stride, ids, normals, stride_n, leaf, out_xyz1, out_normal_curv, out_voxel,
                                    n_out, ids_staging, &d_ids);
    MinMaxAcc h = vg_minmax(c, nullptr, 0);
    if (!fault && n) {
      dense.alloc(n, st);
      load_xyz_as_float4(c, pts, n, stride, nullptr, 0, dense.p, st);
      h = vg_minmax(c, dense.p, n);
      if (with_normals) {  // the fields of voxelgrid_normals, as it stages them
        nc.alloc(2 * n, st);
        vg_load_normals(c, normals, n, stride_n, nullptr, 0, nc.p);
      }
    }
    const size_t n_words = kSvHeadWords + (size_t)kSvBoxWords * R;
    std::vector<unsigned long long> w(n_words, ~0ull);
    w[kSvVerdict] = fault ? 0 : 1;
    unsigned lb[3] = {0, 0, 0};
    if (leaf)
      memcpy(lb, leaf, sizeof(lb));
    const unsigned long long p[3] = {((unsigned long long)lb[0] << 32) | lb[1], ((unsigned long long)lb[2] << 32) | min_pts,
                                     with_normals ? 1ull : 0ull};
    for (int i = 0; i < 3; ++i) {
      w[kSvParams + i] = p[i];
      w[kSvNotParams + i] = ~p[i];
    }
    sv_fold_box(h, w.data() + kSvHeadWords + (size_t)kSvBoxWords * me);
    DevBuf<unsigned long long> d_w;
    d_w.alloc(n_words, st);
    PCLB_CUDA(cudaMemcpyAsync(d_w.p, w.data(), n_words * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
    comm_allreduce_u64(c, d_w.p, d_w.p, n_words, kU64Min);
    PCLB_CUDA(cudaMemcpyAsync(w.data(), d_w.p, n_words * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    check_device_error(c);
    if (fault)
      throw Error(PCLB200_ERR_INVALID, std::string("voxelgrid_sharded: ") + fault);
    PCLB_REQUIRE(w[kSvVerdict] == 1, PCLB200_ERR_INVALID, "voxelgrid_sharded: another rank refused the call");
    PCLB_REQUIRE(w[kSvParams] == ~w[kSvNotParams] && w[kSvParams + 1] == ~w[kSvNotParams + 1], PCLB200_ERR_INVALID,
                 "voxelgrid_sharded: the ranks disagree on leaf or min_points_per_voxel");
    PCLB_REQUIRE(w[kSvParams + 2] == ~w[kSvNotParams + 2], PCLB200_ERR_INVALID,
                 "voxelgrid_sharded: normals given on some ranks and not on others");
    unsigned long long u[kSvBoxWords];  // the union box: the minimum of every rank's keys
    boxes.n = R;
    for (int a = 0; a < kSvBoxWords; ++a)
      u[a] = kSvNoBox;
    for (int s = 0; s < R; ++s) {
      const unsigned long long* ws = w.data() + kSvHeadWords + (size_t)kSvBoxWords * s;
      boxes.any[s] = sv_box(ws, boxes.lo[s], boxes.hi[s]);
      for (int a = 0; a < kSvBoxWords; ++a)
        u[a] = std::min(u[a], ws[a]);
    }
    any = sv_box(u, mn, mx);
  }
  *n_out = 0;
  if (!any)  // no rank holds a finite record
    return 0;
  VgParams gp;
  if (!vg_grid(mn, mx, leaf, gp))  // the same box and leaf on every rank: all of them throw
    throw Error(PCLB200_ERR_LEAF_TOO_SMALL, kVgLeafTooSmall);

  // ---- exchange -----------------------------------------------------------------------------------------------------
  DevBuf<float4> local;  // own records, then the received ones by sender; per float4s each
  size_t n_local = 0;
  SvSenders senders = {};
  {
    ProfScope ps(c, "sharded_voxel_exchange");
    DevBuf<SvRanges> rg;
    rg.alloc(1, st);
    k_sv_ranges<<<1, 32, 0, st>>>(boxes, gp, rg.p);
    ++c.launches;
    PCLB_CUDA(cudaGetLastError());
    DevBuf<unsigned long long> d_cnt, cursor;
    d_cnt.alloc((size_t)R * R, st);
    PCLB_CUDA(cudaMemsetAsync(d_cnt.p, 0, d_cnt.bytes(), st));
    SvOut count_only;
    memset(&count_only, 0, sizeof(count_only));
    count_only.count = d_cnt.p + (size_t)R * me;  // row `me`: what this rank sends to each rank
    const float4* d_nc = with_normals ? nc.p : nullptr;
    if (n) {
      k_sv_select<<<persistent_blocks(c, n), 256, 0, st>>>(dense.p, d_ids, d_nc, n, gp, rg.p, R, me, count_only);
      ++c.launches;
      PCLB_CUDA(cudaGetLastError());
    }
    comm_allreduce_u64(c, d_cnt.p, d_cnt.p, d_cnt.n, kU64Sum);
    std::vector<unsigned long long> cnt((size_t)R * R);
    PCLB_CUDA(cudaMemcpyAsync(cnt.data(), d_cnt.p, d_cnt.bytes(), cudaMemcpyDeviceToHost, st));
    check_device_error(c);
    for (int r = 0; r < R; ++r) {  // every rank sees every count: all of them refuse together
      unsigned long long held = 0;
      for (int s = 0; s < R; ++s)
        held += cnt[(size_t)s * R + r];
      PCLB_REQUIRE(held < 0x7fffffffull, PCLB200_ERR_INVALID,
                   "voxelgrid_sharded: a rank's records and the records it receives exceed 2^31 - 1");
    }
    std::vector<unsigned long long> units(cnt);  // the segments in float4s
    for (auto& x : units)
      x *= per;
    const std::vector<unsigned long long> n_table = segment_table_sizes(units.data(), R);
    unsigned long long all = 0;
    for (int s = 0; s < R; ++s)
      all += n_table[s];
    senders.n = 0;
    for (int s = -1; s < R; ++s) {  // this rank's own records first, then the senders in rank order
      const int from = s < 0 ? me : s;
      if (s == me)
        continue;
      senders.rank[senders.n] = from;
      senders.begin[senders.n + 1] = senders.begin[senders.n] + cnt[(size_t)from * R + me];
      ++senders.n;
    }
    n_local = senders.begin[senders.n];
    const size_t n_own = cnt[(size_t)me * R + me];
    local.alloc(n_local * per, st);
    cursor.alloc(R, st);
    PCLB_CUDA(cudaMemsetAsync(cursor.p, 0, cursor.bytes(), st));
    SvOut out;
    memset(&out, 0, sizeof(out));
    out.count = cursor.p;
    out.dst[me] = local.p;
    PeerTables t;
    if (all) {  // every rank knows every count: all of them take this branch or none
      t = comm_segment_tables(c, n_table.data(), sizeof(float4));
      segment_writes(reinterpret_cast<float4*>(t.local), units.data(), R, me, out.dst);
    }
    if (n) {
      k_sv_select<<<persistent_blocks(c, n), 256, 0, st>>>(dense.p, d_ids, d_nc, n, gp, rg.p, R, me, out);
      ++c.launches;
      PCLB_CUDA(cudaGetLastError());
    }
    if (all) {
      comm_tables_publish(c, t, kU64Sum);
      gather_segments(c, segment_reads<float4>(t, units.data(), R, me), local.p + n_own * per);
      comm_tables_release(c, t);
    }
  }
  dense.release();
  nc.release();

  // ---- centroids ----------------------------------------------------------------------------------------------------
  ProfScope ps(c, "sharded_voxel_centroids");
  if (n_local == 0)
    return 0;
  DevBuf<unsigned long long> keys_in, keys, ukeys;
  DevBuf<int32_t> vals_in, vals, uvals;
  DevBuf<unsigned char> holder, head, tmp;
  DevBuf<float4> pts_local, nc_local;
  keys_in.alloc(n_local, st);
  keys.alloc(n_local, st);
  ukeys.alloc(n_local, st);
  vals_in.alloc(n_local, st);
  vals.alloc(n_local, st);
  uvals.alloc(n_local, st);
  holder.alloc(n_local, st);
  head.alloc(n_local, st);
  if (with_normals) {
    pts_local.alloc(n_local, st);
    nc_local.alloc(2 * n_local, st);
  }
  k_sv_keys<<<grid_for(n_local, 256), 256, 0, st>>>(local.p, n_local, gp, senders, keys_in.p, vals_in.p, holder.p,
                                                   pts_local.p, nc_local.p);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
  const float4* d_pts = with_normals ? pts_local.p : local.p;
  const int ni = (int)n_local;
  DevBuf<size_t> d_num;
  d_num.alloc(3, st);
  DevBuf<int> d_m;
  d_m.alloc(1, st);
  cub::CountingInputIterator<unsigned> counting(0);
  DevBuf<unsigned> starts_all, starts_u;
  starts_all.alloc(n_local, st);
  starts_u.alloc(n_local, st);
  // 64-bit sort, equal keys dropped, the voxel runs of both: the same voxels in the same order
  auto cub_pass = [&](auto&& call) {
    size_t tb = 0;
    PCLB_CUDA(call(nullptr, tb));
    if (tb > tmp.n)
      tmp.alloc(tb, st);
    PCLB_CUDA(call(tmp.p, tb));
  };
  cub_pass([&](void* p, size_t& tb) {
    return cub::DeviceRadixSort::SortPairs(p, tb, keys_in.p, keys.p, vals_in.p, vals.p, ni, 0, kSvKeyBits, st);
  });
  cub_pass([&](void* p, size_t& tb) {
    return cub::DeviceSelect::UniqueByKey(p, tb, keys.p, vals.p, ukeys.p, uvals.p, d_m.p, ni, st);
  });
  k_sv_heads<<<grid_for(n_local, 256), 256, 0, st>>>(keys.p, n_local, head.p);
  cub_pass([&](void* p, size_t& tb) {
    return cub::DeviceSelect::Flagged(p, tb, counting, head.p, starts_all.p, d_num.p, ni, st);
  });
  int n_u = 0;
  PCLB_CUDA(cudaMemcpyAsync(&n_u, d_m.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  k_sv_heads<<<grid_for(n_u, 256), 256, 0, st>>>(ukeys.p, n_u, head.p);
  cub_pass([&](void* p, size_t& tb) {
    return cub::DeviceSelect::Flagged(p, tb, counting, head.p, starts_u.p, d_num.p + 1, n_u, st);
  });
  c.launches += 2 + 9;
  size_t n_vox[2] = {0, 0};
  PCLB_CUDA(cudaMemcpyAsync(n_vox, d_num.p, sizeof(n_vox), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  PCLB_REQUIRE(n_vox[0] == n_vox[1], PCLB200_ERR_INTERNAL, "voxelgrid_sharded: the voxel runs of the keys disagree");
  const size_t n_runs = n_vox[0];
  // ownership, the minimum-points rule on the complete run, the runs this rank returns
  DevBuf<unsigned char> mask, keep;
  DevBuf<RunRef> runs_all, runs;
  DevBuf<unsigned> voxel;
  mask.alloc(n_runs, st);
  keep.alloc(n_runs, st);
  runs_all.alloc(n_runs, st);
  runs.alloc(n_runs, st);
  voxel.alloc(n_runs, st);
  k_sv_holders<<<grid_for(n_runs, 256), 256, 0, st>>>(starts_all.p, n_runs, n_local, vals.p, holder.p, mask.p);
  vg_runs(c, starts_u.p, n_runs, (size_t)n_u, runs_all.p);
  k_sv_own<<<grid_for(n_runs, 256), 256, 0, st>>>(runs_all.p, ukeys.p, mask.p, n_runs, me, min_pts, keep.p, voxel.p);
  c.launches += 2;
  PCLB_CUDA(cudaGetLastError());
  DevBuf<unsigned> tv;
  unsigned* d_voxel = out_on_device(c, out_voxel, n_runs, tv);
  cub_pass([&](void* p, size_t& tb) {
    return cub::DeviceSelect::Flagged(p, tb, runs_all.p, keep.p, runs.p, d_num.p, (int)n_runs, st);
  });
  cub_pass([&](void* p, size_t& tb) {
    return cub::DeviceSelect::Flagged(p, tb, voxel.p, keep.p, d_voxel, d_num.p + 2, (int)n_runs, st);
  });
  c.launches += 4;
  size_t m = 0;
  PCLB_CUDA(cudaMemcpyAsync(&m, d_num.p, sizeof(size_t), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  copy_out(c, out_voxel, tv, m);
  if (m) {
    DevBuf<float4> tx, tn;
    float4* const caller_out = reinterpret_cast<float4*>(out_xyz1);
    float4* const caller_nout = reinterpret_cast<float4*>(out_normal_curv);
    vg_reduce(c, d_pts, with_normals ? nc_local.p : nullptr, uvals.p, runs.p, m, out_on_device(c, caller_out, m, tx),
              with_normals ? out_on_device(c, caller_nout, 2 * m, tn) : nullptr);
    copy_out(c, caller_out, tx, m);
    if (with_normals)
      copy_out(c, caller_nout, tn, 2 * m);
    PCLB_CUDA(cudaStreamSynchronize(st));
  }
  *n_out = m;
  return m;
}

}  // namespace pclb200
