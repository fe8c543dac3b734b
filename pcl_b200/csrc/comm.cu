// comm.cu — cross-GPU exchanges of a sharded source, and the tables of every exchange that moves whole arrays.
//
// The reference has no multi-GPU path.  Here the source cloud is sharded across ranks (one process per
// GPU, target index replicated); every ICP iteration sums kAccum (= 40) doubles, issued on the same stream as the
// iteration kernel so the solve kernel that follows sees the global sums, and a rejector chain adds u64 sums, minima
// and barriers (reject.cu).  Both run on every rank's IPC-mapped exchange block with one device protocol
// (peer_exchange.cuh): the accumulators inside the accumulate kernels, the u64 collectives in k_peer_u64.  Without the
// mappings they fall back to ncclAllReduce.  NCCL is bound at run time (dlopen of libnccl.so.2 — the copy torch
// already loaded, if any) so the library has no link-time dependency and single-GPU users never touch it.
//
// Arrays too large for the exchange block (the one-to-one rejector's table, the sharded target's matches, the halo and
// label answers of a sharded map, allgather_u64) go through PeerTables: one u64 table per rank, mapped into every rank,
// with a barrier to publish and one to release; or, under NCCL, one all-reduce to publish (internal.cuh).
#include <dlfcn.h>

#include <algorithm>
#include <cstdlib>
#include <vector>

#include "internal.cuh"
#include "peer_exchange.cuh"
#include "peer_tables.cuh"

namespace pclb200 {

typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { ncclSuccess = 0 };
enum { ncclFloat64 = 8 };
enum { ncclSum = 0 };

struct NcclApi {
  void* h = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};

static NcclApi& nccl()
{
  static NcclApi api;
  if (!api.h) {
    api.h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!api.h)
      api.h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    PCLB_REQUIRE(api.h != nullptr, PCLB200_ERR_NCCL, std::string("cannot load libnccl.so.2: ") + dlerror());
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(api.h, "ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(api.h, "ncclCommInitRank"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(api.h, "ncclCommDestroy"));
    api.AllReduce = reinterpret_cast<decltype(api.AllReduce)>(dlsym(api.h, "ncclAllReduce"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(dlsym(api.h, "ncclAllGather"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(api.h, "ncclGetErrorString"));
    PCLB_REQUIRE(api.GetUniqueId && api.CommInitRank && api.AllReduce, PCLB200_ERR_NCCL, "libnccl lacks expected symbols");
  }
  return api;
}

#define PCLB_NCCL(expr)                                                                                  \
  do {                                                                                                   \
    int _r = (expr);                                                                                     \
    if (_r != ncclSuccess)                                                                               \
      throw Error(PCLB200_ERR_NCCL, std::string(#expr) + ": " +                                          \
                                        (nccl().GetErrorString ? nccl().GetErrorString(_r) : "nccl error")); \
  } while (0)

enum { ncclUint8 = 1 };
enum { ncclUint32 = 3 };
enum { ncclUint64 = 5 };
enum { ncclMax = 2 };
enum { ncclMin = 3 };

// n u64 per rank, mapped into every rank: the one-to-one rejector table of one ICP session (reject.cu:
// apply_rejector_sharded, ~0 between iterations), the sharded-target exchange arrays (icp.cu) or a communicator's scratch
struct PeerTableEntry {
  unsigned long long comm_id = 0;       // the communicator it was made for
  int rank = 0, nranks = 0;
  size_t n = 0;
  unsigned long long* local = nullptr;  // cudaMalloc'ed (an IPC export needs its own allocation)
  unsigned long long* recv = nullptr;   // NCCL path: the min all-reduce lands here, so `local` keeps only this rank's writes
  void* peer[kMaxRanks] = {};           // peer path: every rank's table mapped here ([rank] = local)
  bool mapped = false;
  void release()
  {
    for (int p = 0; p < nranks && p < kMaxRanks; ++p)
      if (p != rank && peer[p])
        cudaIpcCloseMemHandle(peer[p]);
    if (local)
      cudaFree(local);
    if (recv)
      cudaFree(recv);
    local = recv = nullptr;
    for (auto& q : peer)
      q = nullptr;
    mapped = false;
    comm_id = 0;
  }
  ~PeerTableEntry() { release(); }
};

struct Comm {
  ncclComm_t comm = nullptr;  // nullptr: peer-memory exchange bootstrapped by the caller (comm_import), no NCCL at all
  int rank = 0, nranks = 1;
  int mode = PCLB200_REDUCE_FUSED;
  // fused peer-memory reduce (NVLink): one IPC-shared block per rank
  unsigned char* local_block = nullptr;
  void* peer_block[kMaxRanks] = {};
  PeerView view;
  bool peer_ok = false;
  unsigned long long seq = 0;         // the last sequence number drawn (next_seq)
  unsigned long long id = 0;          // distinct per communicator made in this process
  std::vector<std::weak_ptr<PeerTableEntry>> tables;  // the peer tables made for this communicator
  std::shared_ptr<PeerTableEntry> scratch;            // comm_scratch_tables
  Comm();
};

static unsigned long long g_comm_ids = 0;
Comm::Comm() : id(++g_comm_ids) {}

// The sequence number of the next peer exchange.  Every rank must draw them in the same order (peer_exchange.cuh): an
// iteration's rejector chain first, its accumulator exchange last.
static unsigned long long next_seq(Comm& cm) { return ++cm.seq; }

// Opens the IPC handles of the other ranks' allocations: ptr[p] = rank p's (ptr[rank] = mine).  Returns the first rank
// whose handle does not open (its CUDA error cleared, *err = the error, ptr[p] = nullptr), or -1 once all are open.
static int open_peers(const cudaIpcMemHandle_t* handles, int rank, int nranks, void* mine, void** ptr,
                      cudaError_t* err = nullptr)
{
  for (int p = 0; p < nranks; ++p) {
    if (p == rank) {
      ptr[p] = mine;
      continue;
    }
    const cudaError_t e = cudaIpcOpenMemHandle(&ptr[p], handles[p], cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      cudaGetLastError();
      ptr[p] = nullptr;
      if (err)
        *err = e;
      return p;
    }
  }
  return -1;
}

// every rank's block is mapped: switch to the peer exchange
static void use_peer_blocks(Comm& cm)
{
  cm.view.rank = cm.rank;
  cm.view.nranks = cm.nranks;
  for (int p = 0; p < cm.nranks; ++p) {
    unsigned char* b = static_cast<unsigned char*>(cm.peer_block[p]);
    cm.view.flags[p] = reinterpret_cast<unsigned long long*>(b);
    cm.view.slots[p] = reinterpret_cast<double*>(b + kPeerSlotsOffset);
  }
  cm.peer_ok = true;
}

// Maps every rank's exchange block into this process (CUDA IPC over NVLink / NVSwitch).  Any failure leaves
// peer_ok = false and the per-iteration reduce falls back to ncclAllReduce.
static void setup_peer_reduce(Ctx& c, Comm& cm)
{
  if (cm.nranks > kMaxRanks || !nccl().AllGather)
    return;
  cudaStream_t st = c.stream;
  if (cudaMalloc(reinterpret_cast<void**>(&cm.local_block), kPeerBlockBytes) != cudaSuccess) {
    cudaGetLastError();
    return;
  }
  cudaMemsetAsync(cm.local_block, 0, kPeerBlockBytes, st);
  cudaIpcMemHandle_t mine;
  bool ok = cudaIpcGetMemHandle(&mine, cm.local_block) == cudaSuccess;
  // exchange handles (+ an "ok" byte) through the communicator we already have
  struct Rec { cudaIpcMemHandle_t h; unsigned char ok; unsigned char pad[63]; };
  static_assert(sizeof(Rec) == 128, "record size");
  Rec r;
  memset(&r, 0, sizeof(r));
  r.h = mine;
  r.ok = ok ? 1 : 0;
  DevBuf<unsigned char> d_send, d_recv;
  d_send.alloc(sizeof(Rec), st);
  d_recv.alloc(sizeof(Rec) * cm.nranks, st);
  PCLB_CUDA(cudaMemcpyAsync(d_send.p, &r, sizeof(Rec), cudaMemcpyHostToDevice, st));
  PCLB_NCCL(nccl().AllGather(d_send.p, d_recv.p, sizeof(Rec), ncclUint8, cm.comm, st));
  std::vector<Rec> all(cm.nranks);
  PCLB_CUDA(cudaMemcpyAsync(all.data(), d_recv.p, sizeof(Rec) * cm.nranks, cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  bool all_ok = true;
  cudaIpcMemHandle_t handles[kMaxRanks];
  for (int p = 0; p < cm.nranks; ++p) {
    all_ok = all_ok && all[p].ok;
    handles[p] = all[p].h;
  }
  all_ok = all_ok && open_peers(handles, cm.rank, cm.nranks, cm.local_block, cm.peer_block) < 0;
  // every rank must take the same decision: agree through one more tiny all-reduce
  DevBuf<double> d_flag;
  d_flag.alloc(1, st);
  double hv = all_ok ? 0.0 : 1.0;
  PCLB_CUDA(cudaMemcpyAsync(d_flag.p, &hv, sizeof(double), cudaMemcpyHostToDevice, st));
  PCLB_NCCL(nccl().AllReduce(d_flag.p, d_flag.p, 1, ncclFloat64, ncclSum, cm.comm, st));
  PCLB_CUDA(cudaMemcpyAsync(&hv, d_flag.p, sizeof(double), cudaMemcpyDeviceToHost, st));
  PCLB_CUDA(cudaStreamSynchronize(st));
  if (hv == 0.0)
    use_peer_blocks(cm);
}

static void teardown_peer_reduce(Comm& cm)
{
  for (auto& w : cm.tables)
    if (auto e = w.lock())
      e->release();
  cm.tables.clear();
  for (int p = 0; p < cm.nranks && p < kMaxRanks; ++p)
    if (p != cm.rank && cm.peer_block[p])
      cudaIpcCloseMemHandle(cm.peer_block[p]);
  if (cm.local_block)
    cudaFree(cm.local_block);
  cm.local_block = nullptr;
  cm.peer_ok = false;
}

void comm_unique_id(void* out128)
{
  ncclUniqueId id;
  PCLB_NCCL(nccl().GetUniqueId(&id));
  memcpy(out128, &id, sizeof(id));
}

void comm_destroy(Ctx& c)
{
  if (c.comm) {
    teardown_peer_reduce(*c.comm);
    if (c.comm->comm)
      nccl().CommDestroy(c.comm->comm);
    delete c.comm;
    c.comm = nullptr;
  }
}

void comm_init(Ctx& c, int rank, int nranks, const void* unique_id)
{
  PCLB_REQUIRE(nranks >= 1 && rank >= 0 && rank < nranks, PCLB200_ERR_INVALID, "bad rank / nranks");
  comm_destroy(c);
  if (nranks == 1)
    return;
  ncclUniqueId id;
  memcpy(&id, unique_id, sizeof(id));
  Comm* cm = new Comm();
  cm->rank = rank;
  cm->nranks = nranks;
  PCLB_CUDA(cudaSetDevice(c.device));
  int r = nccl().CommInitRank(&cm->comm, nranks, id, rank);
  if (r != ncclSuccess) {
    delete cm;
    throw Error(PCLB200_ERR_NCCL, "ncclCommInitRank failed");
  }
  c.comm = cm;
  try {
    setup_peer_reduce(c, *cm);
  }
  catch (const Error&) {
    cm->peer_ok = false;  // keep the NCCL path
  }
}

// ---- caller-bootstrapped peer exchange (no NCCL): export the local block's IPC handle, import everybody's ----------------
// For deployments whose launcher already has a way to all-gather 64 bytes per rank (MPI, gloo, a file), and for
// ranks that share one GPU (NCCL refuses duplicate devices; CUDA IPC does not).
static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");

void comm_export(Ctx& c, void* out64)
{
  comm_destroy(c);
  Comm* cm = new Comm();
  c.comm = cm;
  PCLB_CUDA(cudaSetDevice(c.device));
  PCLB_CUDA(cudaMalloc(reinterpret_cast<void**>(&cm->local_block), kPeerBlockBytes));
  PCLB_CUDA(cudaMemsetAsync(cm->local_block, 0, kPeerBlockBytes, c.stream));
  PCLB_CUDA(cudaStreamSynchronize(c.stream));
  cudaIpcMemHandle_t h;
  PCLB_CUDA(cudaIpcGetMemHandle(&h, cm->local_block));
  memcpy(out64, &h, sizeof(h));
}

void comm_import(Ctx& c, int rank, int nranks, const void* handles)
{
  PCLB_REQUIRE(c.comm && c.comm->local_block && !c.comm->comm, PCLB200_ERR_INVALID, "comm_import: call comm_export first");
  PCLB_REQUIRE(nranks >= 2 && nranks <= kMaxRanks && rank >= 0 && rank < nranks, PCLB200_ERR_INVALID, "bad rank / nranks");
  Comm& cm = *c.comm;
  cm.rank = rank;
  cm.nranks = nranks;
  cudaError_t e = cudaSuccess;
  const int p = open_peers(static_cast<const cudaIpcMemHandle_t*>(handles), rank, nranks, cm.local_block, cm.peer_block, &e);
  if (p >= 0)
    throw Error(PCLB200_ERR_CUDA, std::string("comm_import: cudaIpcOpenMemHandle failed for rank ") + std::to_string(p) +
                                      ": " + cudaGetErrorString(e));
  use_peer_blocks(cm);
}

void comm_set_mode(Ctx& c, int mode)
{
  PCLB_REQUIRE(mode == PCLB200_REDUCE_FUSED || mode == PCLB200_REDUCE_NCCL, PCLB200_ERR_INVALID, "unknown reduce mode");
  PCLB_REQUIRE(c.comm != nullptr, PCLB200_ERR_INVALID, "no communicator");
  PCLB_REQUIRE(mode == PCLB200_REDUCE_FUSED || c.comm->comm != nullptr, PCLB200_ERR_INVALID,
               "the NCCL reduce needs a communicator made by pclb200_comm_init");
  c.comm->mode = mode;
}

bool comm_active(const Ctx& c) { return c.comm && c.comm->nranks > 1; }

int comm_nranks(const Ctx& c) { return comm_active(c) ? c.comm->nranks : 1; }

int comm_rank(const Ctx& c) { return comm_active(c) ? c.comm->rank : 0; }

bool comm_peer_fused(const Ctx& c) { return comm_active(c) && c.comm->peer_ok && c.comm->mode == PCLB200_REDUCE_FUSED; }

// view + next sequence number for a fused in-kernel exchange; returns false when the NCCL path must be used
bool comm_peer_view(Ctx& c, PeerView* view, unsigned long long* seq)
{
  if (!comm_peer_fused(c))
    return false;
  *view = c.comm->view;
  *seq = next_seq(*c.comm);
  return true;
}

void comm_allreduce_sum(Ctx& c, double* d_buf, int count)
{
  if (!comm_active(c))
    return;
  PCLB_REQUIRE(c.comm->comm != nullptr, PCLB200_ERR_NCCL, "no NCCL communicator for the library all-reduce");
  PCLB_NCCL(nccl().AllReduce(d_buf, d_buf, (size_t)count, ncclFloat64, ncclSum, c.comm->comm, c.stream));
  ++c.launches;
}

// ---- u64 collectives of the sharded rejectors ---------------------------------------------------------------------------
// One block of kU64Words threads runs peer_exchange on the u64 region: element-wise sum or min (identity ~0) of count
// <= kU64Words words; count == 0 is a barrier.
__global__ void __launch_bounds__(kU64Words)
k_peer_u64(const PeerView v, unsigned long long seq, const unsigned long long* send, unsigned long long* recv, int count,
           int op, int* d_error)
{
  const bool min = op == kU64Min;
  peer_exchange(v, seq, send, recv, count, min ? ~0ull : 0ull,
                [min](unsigned long long a, unsigned long long x) { return min ? (x < a ? x : a) : a + x; }, d_error);
}

static void peer_u64(Ctx& c, const unsigned long long* d_send, unsigned long long* d_recv, int count, int op)
{
  k_peer_u64<<<1, kU64Words, 0, c.stream>>>(c.comm->view, next_seq(*c.comm), d_send, d_recv, count, op, c.d_error);
  ++c.launches;
  PCLB_CUDA(cudaGetLastError());
}

void comm_allreduce_u64(Ctx& c, const unsigned long long* d_send, unsigned long long* d_recv, size_t count, int op)
{
  if (!comm_active(c)) {
    if (d_send != d_recv && count)
      PCLB_CUDA(cudaMemcpyAsync(d_recv, d_send, count * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, c.stream));
    return;
  }
  if (comm_peer_fused(c)) {
    PCLB_REQUIRE(count <= (size_t)kU64Words, PCLB200_ERR_INVALID, "peer-mapped u64 exchange: too many words");
    peer_u64(c, d_send, d_recv, (int)count, op);
    return;
  }
  PCLB_REQUIRE(c.comm->comm != nullptr, PCLB200_ERR_NCCL, "no NCCL communicator for the library all-reduce");
  PCLB_NCCL(nccl().AllReduce(d_send, d_recv, count, ncclUint64, op == kU64Min ? ncclMin : ncclSum, c.comm->comm, c.stream));
  ++c.launches;
}

unsigned long long comm_id(const Ctx& c) { return comm_active(c) ? c.comm->id : 0; }

unsigned long long comm_shard_offset(Ctx& c, unsigned long long n_q, unsigned long long* total)
{
  if (!comm_active(c)) {
    *total = n_q;
    return 0;
  }
  std::vector<unsigned long long> v(kMaxRanks, 0ull);
  v[c.comm->rank] = n_q;
  DevBuf<unsigned long long> d;
  d.alloc(kMaxRanks, c.stream);
  PCLB_CUDA(cudaMemcpyAsync(d.p, v.data(), kMaxRanks * sizeof(unsigned long long), cudaMemcpyHostToDevice, c.stream));
  comm_allreduce_u64(c, d.p, d.p, kMaxRanks, kU64Sum);
  PCLB_CUDA(cudaMemcpyAsync(v.data(), d.p, kMaxRanks * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c.stream));
  check_device_error(c);
  unsigned long long off = 0, tot = 0;
  for (int p = 0; p < c.comm->nranks; ++p) {
    if (p < c.comm->rank)
      off += v[p];
    tot += v[p];
  }
  *total = tot;
  return off;
}

// Maps every rank's table into this process: the IPC handles travel through the u64 region (one exchange), then every
// rank reports whether it could open all of them (a second one) so that all ranks take the same decision.  The caller
// releases the table when this throws.
static void map_peer_table(Ctx& c, PeerTableEntry& e)
{
  Comm& cm = *c.comm;
  cudaStream_t st = c.stream;
  constexpr int kWords = sizeof(cudaIpcMemHandle_t) / sizeof(unsigned long long);
  static_assert(kMaxRanks * kWords <= kU64Words, "IPC handles must fit the u64 region");
  std::vector<cudaIpcMemHandle_t> h(kMaxRanks);  // zero but for this rank's: the sum is every rank's handle
  PCLB_CUDA(cudaIpcGetMemHandle(&h[cm.rank], e.local));
  DevBuf<unsigned long long> d;
  d.alloc((size_t)kMaxRanks * kWords, st);
  PCLB_CUDA(cudaMemcpyAsync(d.p, h.data(), h.size() * sizeof(cudaIpcMemHandle_t), cudaMemcpyHostToDevice, st));
  comm_allreduce_u64(c, d.p, d.p, (size_t)cm.nranks * kWords, kU64Sum);
  PCLB_CUDA(cudaMemcpyAsync(h.data(), d.p, cm.nranks * sizeof(cudaIpcMemHandle_t), cudaMemcpyDeviceToHost, st));
  check_device_error(c);
  unsigned long long bad = open_peers(h.data(), cm.rank, cm.nranks, e.local, e.peer) >= 0 ? 1 : 0;
  PCLB_CUDA(cudaMemcpyAsync(d.p, &bad, sizeof(bad), cudaMemcpyHostToDevice, st));
  comm_allreduce_u64(c, d.p, d.p, 1, kU64Sum);
  PCLB_CUDA(cudaMemcpyAsync(&bad, d.p, sizeof(bad), cudaMemcpyDeviceToHost, st));
  check_device_error(c);
  PCLB_REQUIRE(!bad, PCLB200_ERR_CUDA, "one-to-one rejector: a rank could not map the peers' tables (CUDA IPC)");
  e.mapped = true;
}

PeerTables comm_scratch_tables(Ctx& c, size_t n_words)
{
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID, "no communicator");
  return comm_peer_tables(c, c.comm->scratch, n_words);
}

void comm_barrier(Ctx& c)
{
  if (comm_peer_fused(c))
    peer_u64(c, nullptr, nullptr, 0, kU64Sum);
}

void comm_allreduce_u32_max(Ctx& c, const unsigned* d_send, unsigned* d_recv, size_t count)
{
  PCLB_REQUIRE(comm_active(c) && c.comm->comm != nullptr, PCLB200_ERR_NCCL, "no NCCL communicator for the library all-reduce");
  PCLB_NCCL(nccl().AllReduce(d_send, d_recv, count, ncclUint32, ncclMax, c.comm->comm, c.stream));
  ++c.launches;
}

PeerTables comm_peer_tables(Ctx& c, std::shared_ptr<PeerTableEntry>& owner, size_t n_words)
{
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID, "no communicator");
  Comm& cm = *c.comm;
  if (!owner)
    owner = std::make_shared<PeerTableEntry>();
  PeerTableEntry* e = owner.get();
  const size_t n = std::max<size_t>(n_words, 1);
  if (e->local && (e->n != n || e->comm_id != cm.id))  // another size or another communicator: a new table
    e->release();
  if (!e->local) {
    e->comm_id = cm.id;
    e->rank = cm.rank;
    e->nranks = cm.nranks;
    e->n = n;
    cm.tables.erase(std::remove_if(cm.tables.begin(), cm.tables.end(),
                                   [](const std::weak_ptr<PeerTableEntry>& w) { return w.expired(); }),
                    cm.tables.end());
    cm.tables.push_back(owner);
    PCLB_CUDA(cudaMalloc(reinterpret_cast<void**>(&e->local), n * sizeof(unsigned long long)));
    PCLB_CUDA(cudaMemsetAsync(e->local, 0xff, n * sizeof(unsigned long long), c.stream));
  }
  PeerTables t;
  t.local = e->local;
  t.words = n;
  if (comm_peer_fused(c)) {
    if (!e->mapped) {
      try {
        map_peer_table(c, *e);
      }
      catch (const Error&) {
        e->release();
        throw;
      }
    }
    t.peer = true;
    t.n_read = cm.nranks;
    for (int p = 0; p < cm.nranks; ++p)
      t.read[p] = static_cast<const unsigned long long*>(e->peer[p]);
  }
  else {
    if (!e->recv)
      PCLB_CUDA(cudaMalloc(reinterpret_cast<void**>(&e->recv), n * sizeof(unsigned long long)));
    t.send = e->local;
    t.recv = e->recv;
    t.n_read = 1;
    t.read[0] = e->recv;
  }
  return t;
}

PeerTables comm_segment_tables(Ctx& c, const unsigned long long* n, size_t elem_bytes)
{
  PCLB_REQUIRE(comm_active(c), PCLB200_ERR_INVALID, "no communicator");
  const int R = c.comm->nranks;
  size_t at[kMaxRanks + 1];
  const size_t most = segment_table_words(n, R, elem_bytes, at);
  if (comm_peer_fused(c))
    return comm_scratch_tables(c, most);
  PeerTables t = comm_scratch_tables(c, at[R]);
  PCLB_CUDA(cudaMemsetAsync(t.send, 0, t.words * sizeof(unsigned long long), c.stream));
  t.local = t.send + at[c.comm->rank];
  t.n_read = R;
  for (int s = 0; s < R; ++s)
    t.read[s] = t.recv + at[s];
  return t;
}

void comm_tables_publish(Ctx& c, const PeerTables& t, int op)
{
  if (t.peer)
    peer_u64(c, nullptr, nullptr, 0, kU64Sum);  // every rank's writes to its table are complete
  else
    comm_allreduce_u64(c, t.send, t.recv, t.words, op);
}

void comm_tables_release(Ctx& c, const PeerTables& t)
{
  if (t.peer)
    peer_u64(c, nullptr, nullptr, 0, kU64Sum);  // no peer still reads this rank's table: it may be rewritten
}

size_t allgather_u64(Ctx& c, const unsigned long long* d_send, size_t n, DevBuf<unsigned long long>& out)
{
  cudaStream_t st = c.stream;
  const int R = comm_nranks(c), me = comm_rank(c);
  std::vector<unsigned long long> cnt(R, 0);  // every rank's count
  {
    DevBuf<unsigned long long> d_cnt;
    d_cnt.alloc(R, st);
    cnt[me] = n;
    PCLB_CUDA(cudaMemcpyAsync(d_cnt.p, cnt.data(), R * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
    comm_allreduce_u64(c, d_cnt.p, d_cnt.p, R, kU64Sum);
    PCLB_CUDA(cudaMemcpyAsync(cnt.data(), d_cnt.p, R * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    check_device_error(c);
  }
  unsigned long long total = 0;
  for (int s = 0; s < R; ++s)
    total += cnt[s];
  out.alloc(total, st);
  if (!total)
    return 0;
  const PeerTables t = comm_segment_tables(c, cnt.data(), sizeof(unsigned long long));
  gather_segments(c, one_segment(d_send, n), t.local);  // the write a peer reads after the barrier: a kernel
  comm_tables_publish(c, t, kU64Sum);
  gather_segments(c, table_runs<unsigned long long>(t, cnt.data()), out.p);
  comm_tables_release(c, t);
  return (size_t)total;
}

}  // namespace pclb200
