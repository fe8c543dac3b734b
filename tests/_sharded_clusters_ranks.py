"""Helper for tests/test_gpu_sharded_clusters.py (launched under torchrun, gloo): Euclidean clusters of a map sharded
across ranks (pclb200_cluster_labels_sharded).

Ranks on cuda:0 with the peer exchange bootstrapped over gloo (comm_export / _import), or, with PCLB_SHARDED_NCCL=1,
one GPU per rank with pclb200_comm_init and PCLB200_REDUCE_NCCL.  Scenes: a zig-zag chain crossing every slab boundary
many times, blobs straddling the boundaries with duplicated points and non-finite records, a lattice at exactly the
tolerance and just above it, tolerance 0, and a 1 M-point sheet with holes.  Partitions: slabs, random, and "special"
(points near a cut held by both neighbours under one id, a 1-point tile, tile records in no id order).  Labels must be
byte-equal to one process's cluster_labels on the whole map at the tile's ids, into host and device buffers; sizes
equal to a bincount of those labels; euclidean_clusters_sharded's parts, gathered over the ranks, equal
clusters_from_labels of the reference.  Last, the refusals (ERR_INVALID on every rank), after which the communicator
still works."""
import numpy as np
import torch

import _sharded as S
import pcl_b200 as P

me = S.join()
rank, world, dev, ctx, ref_ctx = me.rank, me.world, me.device, me.ctx, me.ref

rng = np.random.default_rng(29)


def zigzag():
    t = np.linspace(0, 4, 1600, dtype=np.float32)
    passes = [np.c_[t if p % 2 == 0 else 4 - t, np.full_like(t, 0.2 * p), np.zeros_like(t)] for p in range(10)]
    joins = [np.c_[np.full(79, 4.0 * (p % 2 == 0)), 0.2 * p + np.arange(1, 80) * 0.0025, np.zeros(79)] for p in range(9)]
    return P.xyz1(np.concatenate(passes + joins).astype(np.float32))


def blobs():
    c = rng.choice(np.linspace(0, 4, 13), size=(30000, 1)).astype(np.float32)
    xyz = (rng.normal(size=(30000, 3)) * 0.03 + c * [1, 0, 0] + rng.choice([0, 1, 2], size=(30000, 1)) * [0, 1, 0])
    w = P.xyz1(np.concatenate([xyz, xyz[rng.choice(len(xyz), 300, replace=False)]]).astype(np.float32))
    w[rng.choice(len(w), 25, replace=False), 1] = np.nan
    return w


def lattice():
    g = np.stack(np.meshgrid(np.arange(32), np.arange(32), np.arange(4), indexing="ij"), -1).reshape(-1, 3)
    return P.xyz1((g * 0.125).astype(np.float32))


def sheet():
    n = 1_000_000
    xy = rng.random((n, 2), dtype=np.float32) * 10
    keep = (np.sin(xy[:, 0] * 3) * np.cos(xy[:, 1] * 2.5)) < 0.55
    pts = np.zeros((keep.sum(), 3), np.float32)
    pts[:, :2] = xy[keep]
    pts[:, 2] = 0.3 * np.sin(pts[:, 0]) + rng.normal(0, 0.002, keep.sum()).astype(np.float32)
    return P.xyz1(pts)


SCENES = [("zig-zag", zigzag(), [0.004, 0.0025]), ("blobs", blobs(), [0.01, 0.0]),
          ("lattice", lattice(), [0.125, 0.125 * (1 + 1e-6)]), ("sheet", sheet(), [0.02])]


def partitions(whole):
    """Tiles as id arrays; every id of the map is held by some rank"""
    ids = np.arange(len(whole))
    x = np.nan_to_num(whole[:, 0], nan=0.0)
    span = x.max() + 1e-6
    slab = np.minimum((x / span * world).astype(int), world - 1)
    yield "slabs", [ids[slab == r] for r in range(world)]
    perm = rng.permutation(len(whole))
    yield "random", [np.sort(perm[r::world]) for r in range(world)]
    frac = x / span * world - slab
    special = [rng.permutation(np.r_[ids[slab == r], ids[(slab == r + 1) & (frac < 0.05)]]) for r in range(world)]
    special[-2] = rng.permutation(np.union1d(special[-2], special[-1][1:]))  # the last tile: 1 point
    special[-1] = special[-1][:1]
    yield "special", special


checked = 0
for sname, whole, tols in SCENES:
    ref_index = P.Index(ref_ctx, whole)
    for pname, parts in partitions(whole):
        ids = np.ascontiguousarray(parts[rank], dtype=np.int32)
        tile = np.ascontiguousarray(whole[ids])
        tindex = P.Index(ctx, tile, ids=ids)
        for tol in tols:
            want = ref_index.cluster_labels(tol)
            labels, sizes = tindex.cluster_labels_sharded(tol)
            assert labels.tobytes() == np.ascontiguousarray(want[ids]).tobytes(), (sname, pname, tol, rank)
            bc = np.bincount(want[want >= 0], minlength=len(whole))
            want_sizes = np.where(want[ids] >= 0, bc[np.maximum(want[ids], 0)], 0)
            assert np.array_equal(sizes, want_sizes), (sname, pname, tol, rank)
            # device buffers
            dl = torch.full((len(ids),), 7, dtype=torch.int32, device=f"cuda:{dev}")
            ds = torch.full((len(ids),), 7, dtype=torch.int64, device=f"cuda:{dev}")
            torch.cuda.synchronize()  # the fills run on torch's stream, the library writes on its own
            tindex.cluster_labels_sharded(tol, out=dl, sizes=ds)
            assert dl.cpu().numpy().tobytes() == labels.tobytes() and np.array_equal(ds.cpu().numpy(), sizes)
            # an id held by two ranks: one label everywhere
            seen = {}
            for r_ids, r_lab in S.gathered((ids, labels)):
                for i, l in zip(r_ids.tolist(), r_lab.tolist()):
                    assert seen.setdefault(i, l) == l, (sname, pname, tol, "shared id", i)
            checked += 1
        tol = tols[0]
        for lo, hi in ((1, 2 ** 32 - 1), (3, 500)):
            parts_here = tindex.euclidean_clusters_sharded(tol, ids, lo, hi)
            every = S.gathered(parts_here)
            assert len(set(len(e) for e in every)) == 1, (sname, pname, "lengths")
            union = [np.unique(np.concatenate([e[k] for e in every])).astype(np.int32) for k in range(len(every[0]))]
            want_cl = P.clusters_from_labels(ref_index.cluster_labels(tol), lo, hi)
            assert len(union) == len(want_cl) and all(np.array_equal(a, b) for a, b in zip(union, want_cl)), \
                (sname, pname, lo, hi, rank)
            checked += 1
        print(f"rank {rank}: {sname} {pname} ok", flush=True)


# ---- refusals: ERR_INVALID on every rank, and the communicator still works -------------------------------------------------
whole = SCENES[1][1]
ids = np.ascontiguousarray(next(partitions(whole))[1][rank], dtype=np.int32)
tile = np.ascontiguousarray(whole[ids])
tindex = P.Index(ctx, tile, ids=ids)
plain = P.Index(ctx, tile)
lone = P.Index(ref_ctx, tile, ids=ids)
short = np.empty(len(ids) - 1, np.int32)
S.refused(lambda: tindex.cluster_labels_sharded(-0.01), "negative cluster tolerance")
S.refused(lambda: plain.cluster_labels_sharded(0.01), "pclb200_index_build_ids")
S.refused(lambda: lone.cluster_labels_sharded(0.01), "communicator")
S.refused(lambda: P._check(P.lib().pclb200_cluster_labels_sharded(ctx.h, tindex.h, 0.01, short.ctypes.data, None,
                                                                    len(short))), "one entry per record")
S.refused(lambda: P._check(P.lib().pclb200_cluster_labels(ctx.h, tindex.h, 0.01, short.ctypes.data, len(ids))),
        "no cloud to size the labels by")  # the single-GPU call still refuses a tile
want = P.Index(ref_ctx, whole).cluster_labels(0.01)
assert tindex.cluster_labels_sharded(0.01)[0].tobytes() == np.ascontiguousarray(want[ids]).tobytes()
me.finish("SHARDED_CLUSTERS", checks=checked)
