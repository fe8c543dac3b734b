"""Helper for tests/test_gpu_sharded_normals.py (launched under torchrun, gloo): normals of a map sharded across ranks
(pclb200_normals_knn_sharded / pclb200_normals_radius_sharded).

Ranks on cuda:0 with the peer exchange bootstrapped over gloo (comm_export / _import), or, with SHARDED_NORMALS_NCCL=1, one
GPU per rank with pclb200_comm_init and PCLB200_REDUCE_NCCL.  Two maps (a 200 k-point surface and a volume cloud, both
with non-finite rows and duplicated points under other ids), four partitions (spatial slabs; a random partition; slabs
whose points near a cut are held by both neighbours under one id; slabs plus a far tile of 2 points), k = 3 / 16 / 40
and radius 0.03.  Queries: each tile's own records (non-finite ones included), and an arbitrary point set through an
indices subset.  out and is_dense must be byte-equal to one process's normals on an index of the whole map.  Then the
pipeline: the tiles' normals from the new call feed set_target_sharded, and point-to-plane / symmetric aligns must be
byte-equal to one process that used the whole map's normals.  Last, the refusals (ERR_INVALID on every rank), after
which the communicator still works."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pcl_b200 as P  # noqa: E402

NCCL = os.environ.get("SHARDED_NORMALS_NCCL") == "1"
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dev = rank if NCCL else 0
torch.cuda.set_device(dev)
dist.init_process_group("gloo")
ctx = P.Context(dev)
if NCCL:
    uid = [P.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    ctx.comm_init(rank, world, uid[0])
    ctx.comm_set_mode(P.REDUCE_NCCL)
else:
    handles = [None] * world
    dist.all_gather_object(handles, ctx.comm_export())
    ctx.comm_import(rank, world, handles)
ref_ctx = P.Context(dev)  # no communicator: one process on the whole map

rng = np.random.default_rng(17)


def surface(n):
    xy = rng.random((n, 2), dtype=np.float32) * 4
    z = (0.3 * np.sin(xy[:, 0]) * np.cos(xy[:, 1])).astype(np.float32)
    return np.c_[xy, z]


def volume(n):
    return rng.random((n, 3), dtype=np.float32) * np.float32(0.6)


def with_extras(xyz):
    """xyz1 rows, some non-finite, some points repeated under other ids (exact ties)"""
    w = P.xyz1(np.concatenate([xyz, xyz[rng.choice(len(xyz), 200, replace=False)]]))
    w[rng.choice(len(w), 30, replace=False), 1] = np.nan
    return w


SCENES = [("surface", with_extras(surface(200000))), ("volume", with_extras(volume(100000)))]


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
    yield "shared ids", [np.r_[ids[slab == r], ids[(slab == r + 1) & (frac < 0.1)]] for r in range(world)]
    far = [ids[slab == r] for r in range(world)]
    far[-2] = np.r_[far[-2], far[-1]]
    far[-1] = np.array([], np.int64)
    yield "far tile", far


def tile_of(whole, ids):
    return np.ascontiguousarray(whole[ids]), np.ascontiguousarray(ids, dtype=np.int32)


def same(a, b):
    return a[0].tobytes() == b[0].tobytes() and a[1] == b[1]


checked = 0
for sname, whole0 in SCENES:
    for pname, parts in partitions(whole0):
        whole = whole0
        if pname == "far tile":  # two far points of their own, held by the last rank only
            whole = np.concatenate([whole0, P.xyz1(np.array([[50, 50, 50], [50, 50.02, 50]], np.float32))])
            parts[-1] = np.array([len(whole0), len(whole0) + 1])
        ref_index = P.Index(ref_ctx, whole)
        tile, ids = tile_of(whole, parts[rank])
        tindex = P.Index(ctx, tile, ids=ids)
        q_any = P.xyz1(np.concatenate([whole[rng.choice(len(whole), 3000), :3] + np.float32(0.004),
                                       np.array([[np.nan, 0, 0], [100, 100, 100]], np.float32)]))
        sub = np.sort(rng.choice(len(q_any), 1500, replace=False)).astype(np.int32)
        for k in (3, 16, 40):
            got = tindex.normals_knn_sharded(tile, k, viewpoint=(1, 2, 3))
            want = ref_index.normals_knn(tile, k, viewpoint=(1, 2, 3))
            assert same(got, want), (sname, pname, "k", k, rank)
            got = tindex.normals_knn_sharded(q_any, k, indices=sub)
            want = ref_index.normals_knn(q_any, k, indices=sub)
            assert same(got, want), (sname, pname, "k, arbitrary queries", k, rank)
            checked += 2
        got = tindex.normals_radius_sharded(tile, 0.03)
        want = ref_index.normals_radius(tile, 0.03)
        assert same(got, want), (sname, pname, "radius", rank)
        got = tindex.normals_radius_sharded(q_any, 0.03, indices=sub)
        want = ref_index.normals_radius(q_any, 0.03, indices=sub)
        assert same(got, want), (sname, pname, "radius, arbitrary queries", rank)
        checked += 2
        print(f"rank {rank}: {sname} {pname} ok", flush=True)

# ---- the pipeline: sharded normals -> set_target_sharded -> point-to-plane / symmetric ----------------------------------
whole = SCENES[0][1]
parts = next(partitions(whole))[1]
ns = 40000
sel = rng.choice(len(whole), ns, replace=False)
a = np.deg2rad(2.0)
Rm = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
src = np.zeros((ns, 8), np.float32)
src[:, :3] = (np.nan_to_num(whole[sel, :3]).astype(np.float64) @ Rm.T + [0.02, -0.015, 0.01]).astype(np.float32)
src[:, 3] = 1
ref_index = P.Index(ref_ctx, whole)
src_n, _ = ref_index.normals_knn(src, 16)
src[:, 4:8] = src_n
whole_n, _ = ref_index.normals_knn(whole, 16)
tile, ids = tile_of(whole, parts[rank])
tindex = P.Index(ctx, tile, ids=ids)
tile_n, _ = tindex.normals_knn_sharded(tile, 16)
assert tile_n.tobytes() == np.ascontiguousarray(whole_n[ids]).tobytes()


def run(session_ctx, set_target, est):
    p = P.default_params(max_iterations=15, max_correspondence_distance=0.15, estimator=est, mse_threshold_absolute=0.0,
                         transformation_epsilon=1e-12, with_normals_transform=1)
    icp = P.Icp(session_ctx, p)
    set_target(icp)
    icp.set_source(src, normals=P.Field(src, 4), guess=None)
    st = icp.iterate()
    corr = icp.get_correspondences().tobytes()
    cloud = icp.get_cloud(stride_floats=8, normals=None).tobytes()
    icp.close()
    return (st["iterations"], st["state"], st["n_correspondences"], np.float64(st["mse"]).tobytes(),
            st["final"].tobytes()), corr, cloud


for est in (P.EST_POINT_TO_PLANE_LLS, P.EST_SYMMETRIC_POINT_TO_PLANE_LLS):
    want = run(ref_ctx, lambda icp: icp.set_target(ref_index, normals=whole_n), est)
    got = run(ctx, lambda icp: icp.set_target_sharded(tindex, normals=tile_n), est)
    assert got == want, ("pipeline", est, got[0], want[0])
    checked += 1
print(f"rank {rank}: pipeline ok", flush=True)


# ---- refusals: ERR_INVALID on every rank, and the communicator still works -------------------------------------------------
def refused(fn, word):
    try:
        fn()
    except P.Pclb200Error as e:
        assert e.code == P.ERR_INVALID and word in str(e), e
        return
    raise SystemExit(f"accepted: {word}")


plain = P.Index(ctx, tile)
lone = P.Index(ref_ctx, tile, ids=ids)
refused(lambda: tindex.normals_knn_sharded(tile, 0), "k must be positive")
refused(lambda: tindex.normals_radius_sharded(tile, 0.0), "radius must be positive")
refused(lambda: plain.normals_knn_sharded(tile, 8), "pclb200_index_build_ids")
refused(lambda: plain.normals_radius_sharded(tile, 0.03), "pclb200_index_build_ids")
refused(lambda: lone.normals_knn_sharded(tile, 8), "communicator")
refused(lambda: lone.normals_radius_sharded(tile, 0.03), "communicator")
assert tindex.normals_knn_sharded(tile, 16)[0].tobytes() == tile_n.tobytes()
dist.barrier()
print(f"SHARDED_NORMALS_OK {'nccl' if NCCL else 'export'} {world} checks={checked}", flush=True)
dist.barrier()
dist.destroy_process_group()
