"""What the tests and tools of the sharded map share: the bootstrap of a torchrun rank and the launcher that starts the
ranks, the maps, partitions and queries of the normals and filters rank scripts, the halo box in numpy, the reference
rules of the two outlier filters, and the runner of the host-compiled test programs (tests/host).

Importing this module imports neither torch nor the library: the CPU-only tests import it too."""
import functools
import os
import shutil
import socket
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import pcl_b200 as P  # noqa: E402

# ---- ranks -----------------------------------------------------------------------------------------------------------------
NCCL_ENV = "PCLB_SHARDED_NCCL"  # "1": the ranks attach with pclb200_comm_init (torchrun(..., nccl=True) sets it)
NCCL = os.environ.get(NCCL_ENV) == "1"


class Rank:
    """One torchrun process: rank, world, device, nccl, ctx (attached to the communicator of the ranks) and ref (a Context
    with no communicator, made at first use: one process on the whole map)."""

    def __init__(self, rank, world, device, nccl, ctx):
        self.rank, self.world, self.device, self.nccl, self.ctx = rank, world, device, nccl, ctx

    @functools.cached_property
    def ref(self):
        return P.Context(self.device)

    def finish(self, tag, **counts):
        """The `<tag>_OK <protocol> <world> [name=count ...]` line every rank prints once all of them are done."""
        import torch.distributed as dist
        dist.barrier()
        words = [f"{tag}_OK", "nccl" if self.nccl else "export", str(self.world)] + [f"{k}={v}" for k, v in counts.items()]
        print(" ".join(words), flush=True)
        dist.barrier()
        dist.destroy_process_group()


def join(nccl=NCCL, device=None):
    """Start this torchrun rank: select its CUDA device, start gloo, and attach a Context to the communicator of the ranks,
    with pclb200_comm_init and PCLB200_REDUCE_NCCL when nccl, else with the peer exchange bootstrapped over gloo
    (comm_export / _import), which also serves ranks that share one GPU.  device None: the local rank's GPU under NCCL
    (it refuses two ranks on one device), cuda:0 for every rank otherwise.  One rank alone gets no communicator."""
    import torch
    import torch.distributed as dist
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    if device is None:
        device = int(os.environ["LOCAL_RANK"]) if nccl else 0
    torch.cuda.set_device(device)
    dist.init_process_group("gloo")
    ctx = P.Context(device)
    if world > 1 and nccl:
        uid = [P.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        ctx.comm_init(rank, world, uid[0])
        ctx.comm_set_mode(P.REDUCE_NCCL)
    elif world > 1:
        ctx.comm_import(rank, world, gathered(ctx.comm_export()))
    return Rank(rank, world, device, nccl, ctx)


def gathered(obj):
    """obj of every rank, in rank order"""
    import torch.distributed as dist
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, obj)
    return out


def refused(fn, word):
    """fn must raise ERR_INVALID with word in its message"""
    try:
        fn()
    except P.Pclb200Error as e:
        assert e.code == P.ERR_INVALID and word in str(e), e
        return
    raise SystemExit(f"accepted: {word}")


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def torchrun(script, nproc, nccl=False, timeout=1500):
    """Run tests/<script> as nproc ranks on this machine; returns the CompletedProcess (the tails of its output printed)."""
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                        "--master-addr", "127.0.0.1", "--master-port", str(free_port()), os.path.join(ROOT, "tests", script)],
                       capture_output=True, text=True, timeout=timeout, env=dict(os.environ, **{NCCL_ENV: "1" if nccl else "0"}))
    print(r.stdout[-4000:], r.stderr[-4000:])
    return r


# ---- the maps, partitions and queries of the normals and filters rank scripts (each draws from the caller's rng) -----------
def surface(rng, n):
    xy = rng.random((n, 2), dtype=np.float32) * 4
    z = (0.3 * np.sin(xy[:, 0]) * np.cos(xy[:, 1])).astype(np.float32)
    return np.c_[xy, z]


def volume(rng, n):
    return rng.random((n, 3), dtype=np.float32) * np.float32(0.6)


def with_extras(rng, xyz):
    """xyz1 rows, some non-finite, some points repeated under other ids (exact ties)"""
    w = P.xyz1(np.concatenate([xyz, xyz[rng.choice(len(xyz), 200, replace=False)]]))
    w[rng.choice(len(w), 30, replace=False), 1] = np.nan
    return w


def partitions(rng, whole, world):
    """(name, tiles as id arrays, the map they cut): slabs along x, a random partition, slabs whose points near a cut are
    held by both neighbours under one id, and slabs plus a far tile of two points of its own.  Every id of the map is
    held by some rank."""
    ids = np.arange(len(whole))
    x = np.nan_to_num(whole[:, 0], nan=0.0)
    span = x.max() + 1e-6
    slab = np.minimum((x / span * world).astype(int), world - 1)
    yield "slabs", [ids[slab == r] for r in range(world)], whole
    perm = rng.permutation(len(whole))
    yield "random", [np.sort(perm[r::world]) for r in range(world)], whole
    frac = x / span * world - slab
    yield "shared ids", [np.r_[ids[slab == r], ids[(slab == r + 1) & (frac < 0.1)]] for r in range(world)], whole
    far = [ids[slab == r] for r in range(world)]
    far[-2] = np.r_[far[-2], far[-1]]
    far[-1] = np.array([len(whole), len(whole) + 1])  # two far points, held by the last rank only
    yield "far tile", far, np.concatenate([whole, P.xyz1(np.array([[50, 50, 50], [50, 50.02, 50]], np.float32))])


def arbitrary_queries(rng, whole):
    """3000 points near the map's, a non-finite one and a far one; and a sorted subset of 1500 of them as indices"""
    q_any = P.xyz1(np.concatenate([whole[rng.choice(len(whole), 3000), :3] + np.float32(0.004),
                                   np.array([[np.nan, 0, 0], [100, 100, 100]], np.float32)]))
    sub = np.sort(rng.choice(len(q_any), 1500, replace=False)).astype(np.int32)
    return q_any, sub


def finite_rows(a):
    return np.isfinite(a[:, :3]).all(1)


# ---- the halo (DESIGN.md §5) -----------------------------------------------------------------------------------------------
def halo_box(queries, rho2):
    """The box of a rank's local map: every finite query widened by its reach rho (1 + 2^-20) + 2^-60, where rho2 is the
    squared reach per query or one for all, the faces rounded outward by one float step.  (lo, hi) as float32."""
    fin = finite_rows(queries)
    rho2 = np.asarray(rho2, np.float64)
    h = np.sqrt(rho2[fin] if rho2.ndim else rho2) * (1 + 2.0 ** -20) + 2.0 ** -60
    q = queries[fin, :3].astype(np.float64)
    h = h[:, None] if h.ndim else h
    lo = np.nextafter((q - h).min(0).astype(np.float32), np.float32(-np.inf))
    hi = np.nextafter((q + h).max(0).astype(np.float32), np.float32(np.inf))
    return lo, hi


def in_box(whole, lo, hi):
    with np.errstate(invalid="ignore"):
        return ((whole[:, :3] >= lo) & (whole[:, :3] <= hi)).all(1)


def local_ids(whole, parts, r, lo, hi):
    """Rank r's local map as ids, ascending (the id order): its tile, and every point of the other tiles inside the box."""
    inside = in_box(whole, lo, hi)
    sel = np.zeros(len(whole), bool)
    for s, p in enumerate(parts):
        if s != r:
            sel[p] |= inside[p]
    sel[parts[r]] = True
    return np.nonzero(sel)[0]


def halo_points(whole, tile_ids, lo, hi):
    """the number of points of the map outside the tile that lie in the box"""
    inside = in_box(whole, lo, hi)
    inside[tile_ids] = False
    return int(inside.sum())


# ---- the outlier filters' rules over one process's statistics --------------------------------------------------------------
def sor_rule(means, finite, std_mul, negative=False):
    """StatisticalOutlierRemoval (statistical_outlier_removal.hpp:100-135) over the mean distances in record order: sums
    in record order (np.cumsum is sequential), d * d in float.  (keep mask as uint8, (valid, mean, thr))."""
    valid = float(finite.sum())
    s = np.cumsum(means.astype(np.float64))[-1] if len(means) else 0.0
    sq = np.cumsum((means * means).astype(np.float64))[-1] if len(means) else 0.0
    mean = s / valid
    var = (sq - s * s / valid) / (valid - 1)
    thr = mean + std_mul * np.sqrt(var)
    m = means.astype(np.float64)
    return (~((m <= thr) if negative else (m > thr))).astype(np.uint8), (valid, mean, thr)


def ror_rule(kth, finite, is_dense, radius, negative=False):
    """RadiusOutlierRemoval::applyFilterIndices (radius_outlier_removal.hpp:86-150) on the k-th squared distances: keep
    mask as uint8"""
    kth = kth.astype(np.float64)
    if is_dense:
        fin = np.isfinite(kth)
        removed = np.where(fin, (radius * radius >= kth) if negative else (radius * radius < kth), not negative)
    else:
        enough = kth.astype(np.float32) < np.float32(radius * radius)
        removed = ~finite | (enough if negative else ~enough)
    return (~removed).astype(np.uint8)


# ---- host-compiled test programs -------------------------------------------------------------------------------------------
CUDA_INC = "/usr/local/cuda/include"
HOST = os.path.join(ROOT, "tests", "host")
needs_host_compiler = pytest.mark.skipif(
    not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")) or shutil.which("g++") is None,
    reason="needs g++ and the CUDA headers (vector types only; nothing is run on a device)")


def host_program(tmp_path, source, args=(), defines=(), link=(), timeout=None):
    """Compile tests/host/<source> for the host, run it with args, check that it exits 0 and prints PASSED; its stdout."""
    exe = str(tmp_path / (os.path.splitext(source)[0] + ("_dev" if defines else "")))
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-frounding-math", "-ffp-contract=off", "-fno-fast-math", *defines,
                           "-I" + CUDA_INC, "-I" + os.path.join(ROOT, "include"), "-I" + HOST,
                           "-I" + os.path.join(ROOT, "pcl_b200", "pcl_compat"), os.path.join(HOST, source), "-o", exe, *link])
    r = subprocess.run([exe, *args], capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]
    return r.stdout
