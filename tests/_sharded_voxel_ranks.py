"""Helper for tests/test_gpu_sharded_voxel.py (launched under torchrun, gloo): VoxelGrid of a map sharded across ranks
(pclb200_voxelgrid_sharded).

Ranks on cuda:0 with the peer exchange bootstrapped over gloo (comm_export / _import), or, with PCLB_SHARDED_NCCL=1, one
GPU per rank with pclb200_comm_init and PCLB200_REDUCE_NCCL.  The map: a surface cloud of PointNormal records with a
lattice whose coordinates are multiples of the leaf, non-finite rows and points repeated under other ids.  Six
partitions: the four of _sharded.partitions (slabs, random, shared ids, a far tile), slabs cut exactly on voxel faces, and
one rank empty.  Leaves giving about 1 to 50 records per voxel, min_points_per_voxel 0, 1 and 3, with and without normals.
Every rank's rows, concatenated and stable-sorted by voxel index, must be byte-equal to one process's pclb200_voxelgrid
(_normals) on the whole map with the sorted union of the ids; no voxel on two ranks; n_out <= n on every rank.  Then
voxel indices at and above 2^31, device arrays in and out, ERR_LEAF_TOO_SMALL on every rank for a leaf only the union grid is too large for, every refusal
as ERR_INVALID on every rank (after which the communicator still works), and the down-sampled rows indexed under their
voxel indices answering pclb200_knn_sharded as pclb200_knn answers on the single-process output."""
import ctypes as C

import numpy as np
import torch

import _sharded as S
import pcl_b200 as P

me = S.join()
rank, world, dev, ctx, ref_ctx = me.rank, me.world, me.device, me.ctx, me.ref
rng = np.random.default_rng(41)
LEAF = 0.05


def point_normal(xyz1):
    """(n, 12) PointNormal rows: x y z 1 | unit normal, 0 | curvature 0 0 0"""
    out = np.zeros((len(xyz1), 12), np.float32)
    out[:, :4] = xyz1
    nrm = np.c_[np.cos(xyz1[:, 0]), np.sin(xyz1[:, 1]), np.ones(len(xyz1))].astype(np.float32)
    out[:, 4:7] = nrm / np.linalg.norm(nrm, axis=1, keepdims=True)
    out[:, 8] = rng.random(len(xyz1), dtype=np.float32) * np.float32(0.01)
    return out


def lattice(n, step):  # coordinates that are multiples of the leaf: points on voxel faces
    g = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float32) * np.float32(step)] * 2, indexing="ij"), -1).reshape(-1, 2)
    return np.c_[g, np.full(len(g), np.float32(2 * step))]


def partitions():
    """(name, tiles as id arrays, the map as PointNormal rows)"""
    for name, parts, whole in S.partitions(rng, np.ascontiguousarray(whole0[:, :4]), world):
        yield name, parts, whole0 if len(whole) == len(whole0) else np.concatenate([whole0, point_normal(whole[len(whole0):])])
    ids = np.arange(len(whole0))
    inv = np.float32(1) / np.float32(LEAF)
    ix = np.floor((np.nan_to_num(whole0[:, 0]) * inv).astype(np.float32)).astype(np.int64)
    cut = np.minimum(ix * world // (ix.max() + 1), world - 1)  # slabs whose cuts are voxel faces of the whole grid
    yield "voxel faces", [ids[cut == r] for r in range(world)], whole0
    yield "one rank empty", [ids[r::world - 1] for r in range(world - 1)] + [ids[:0]], whole0


def run(tile, tids, leaf, mp, normals):
    return ctx.voxelgrid_sharded(tile, tids, leaf, mp, normal_offset=4 if normals else None)


def outcome(fn):
    """fn's result, or its error as (code, message)"""
    try:
        return fn()
    except P.Pclb200Error as e:
        return e.code, str(e)


def check(name, whole, parts, leaf, mp, normals, got):
    """every rank's rows, sorted by voxel, against one process's output on the whole map (or its error on every rank)"""
    union = np.unique(np.concatenate(parts)).astype(np.int32)
    if normals:
        want = outcome(lambda: ref_ctx.voxelgrid_normals(whole, leaf, mp, indices=union, is_dense=False))
    else:
        want = outcome(lambda: (ref_ctx.voxelgrid(whole, leaf, mp, indices=union, is_dense=False), None))
    every = S.gathered(got)
    failed = [isinstance(g[0], int) for g in every]
    if isinstance(want[0], int):
        assert all(failed) and all(g[0] == want[0] for g in every), (name, leaf, mp, "errors", want, every)
        return 0
    assert not any(failed), (name, leaf, mp, normals, "refused", [g for g, f in zip(every, failed) if f])
    want, want_nc = want
    rows = np.concatenate([g[0] for g in every])
    vox = np.concatenate([g[1] for g in every])
    order = np.argsort(vox, kind="stable")
    assert len(np.unique(vox)) == len(vox), (name, "a voxel on two ranks")
    for r, g in enumerate(every):
        assert len(g[0]) <= len(parts[r]), (name, "n_out > n", r)
        assert (np.diff(g[1].astype(np.int64)) > 0).all(), (name, "rows not ordered by voxel", r)
    assert rows[order].tobytes() == want.tobytes(), (name, leaf, mp, normals, len(rows), len(want))
    if normals:
        nc = np.concatenate([g[2] for g in every])
        assert nc[order].tobytes() == want_nc.tobytes(), (name, leaf, mp, "normals")
    return len(want)


xyz = np.concatenate([S.surface(rng, 60000), lattice(64, LEAF)])
whole0 = point_normal(S.with_extras(rng, xyz))
checked = guarded = 0
for pname, parts, whole in partitions():
    tids = np.ascontiguousarray(parts[rank], dtype=np.int32)
    tile = np.ascontiguousarray(whole[tids])
    for leaf in (0.012, LEAF, 0.3):  # about 1, 10 and 50 records per voxel
        for mp in (0, 1, 3):
            for normals in (False, True):
                n_vox = check(pname, whole, parts, leaf, mp, normals, outcome(lambda: run(tile, tids, leaf, mp, normals)))
                checked += 1
                guarded += n_vox == 0
    print(f"rank {rank}: {pname} ok ({n_vox} voxels at leaf 0.3)", flush=True)
assert guarded == 6, guarded  # the far tile at leaf 0.012: the whole map's grid trips the guard

# ---- a voxel whose total passes min_points_per_voxel while no rank's share does -----------------------------------------
pts = P.xyz1(np.array([[0.01, 0.01, 0.01], [0.02, 0.02, 0.02], [0.03, 0.01, 0.02], [0.5, 0.5, 0.5]], np.float32))
mine = np.array([r for r in range(3) if r % world == rank] + ([3] if rank == 0 else []), np.int32)
got = ctx.voxelgrid_sharded(np.ascontiguousarray(pts[mine]), mine, 0.1, 3)
assert check("split voxel", pts, [np.array([r for r in range(3) if r % world == s] + ([3] if s == 0 else []))
                                  for s in range(world)], 0.1, 3, False, got) == 1
checked += 1

# ---- voxel indices at and above 2^31 while the guard passes ---------------------------------------------------------------
# leaf 1: int(extent) + 1 = 1290 per axis passes the guard, div_b = 1291 per axis; the far corner is voxel 2 151 685 170,
# whose low 31 bits are voxel 4 201 522.  Rank 0 holds records of both, the ids of the lower voxel on either side of the
# corner's; the other ranks hold records of the same voxels.
big = P.xyz1(np.array([[0, 0, 0], [608.5, 672.5, 2.5], [1290.4, 1290.4, 1290.4], [608.25, 672.75, 2.25], [0.5, 0.5, 0.5],
                       [0.7, 0.7, 0.7], [1290.3, 1290.3, 1290.3], [608.75, 672.25, 2.75], [1290.2, 1290.2, 1290.2]],
                      np.float32))
big_parts = [np.array([1, 2, 3, 4]), np.array([5, 6, 7]), np.array([8])]
big_parts = big_parts[:world - 1] + [np.concatenate(big_parts[world - 1:])]
bids = np.ascontiguousarray(big_parts[rank], dtype=np.int32)
got = ctx.voxelgrid_sharded(np.ascontiguousarray(big[bids]), bids, 1.0)
assert got[1].max(initial=0) >= 2 ** 31 or rank != 0, got[1]
assert check("voxels above 2^31", big, big_parts, 1.0, 0, False, got) == 3
checked += 1

# ---- device arrays in and out --------------------------------------------------------------------------------------------
_, parts, whole = next(partitions())
tids = np.ascontiguousarray(parts[rank], dtype=np.int32)
tile = np.ascontiguousarray(whole[tids])
d_tile = torch.from_numpy(tile).to(f"cuda:{dev}")
d_ids = torch.from_numpy(tids).to(f"cuda:{dev}")
n = len(tile)
o = torch.empty((n, 4), dtype=torch.float32, device=f"cuda:{dev}")
onc = torch.empty((n, 8), dtype=torch.float32, device=f"cuda:{dev}")
ov = torch.empty(n, dtype=torch.int32, device=f"cuda:{dev}")
m = C.c_size_t()
leaf3 = (C.c_float * 3)(LEAF, LEAF, LEAF)
P._check(P.lib().pclb200_voxelgrid_sharded(ctx.h, C.c_void_p(d_tile.data_ptr()), n, 48, C.c_void_p(d_ids.data_ptr()),
                                           C.c_void_p(d_tile.data_ptr() + 16), 48, leaf3, 2,
                                           C.c_void_p(o.data_ptr()), C.c_void_p(onc.data_ptr()),
                                           C.c_void_p(ov.data_ptr()), C.byref(m)))
host = ctx.voxelgrid_sharded(tile, tids, LEAF, 2, normal_offset=4)
k = m.value
assert o[:k].cpu().numpy().tobytes() == host[0].tobytes() and onc[:k].cpu().numpy().tobytes() == host[2].tobytes()
assert ov[:k].cpu().numpy().view(np.uint32).tobytes() == host[1].tobytes()
check("device arrays", whole, parts, LEAF, 2, True, host)
checked += 1

# ---- the union grid trips the guard, no tile's grid does: ERR_LEAF_TOO_SMALL on every rank --------------------------------
name, parts, whole = [p for p in partitions() if p[0] == "far tile"][0]
tids = np.ascontiguousarray(parts[rank], dtype=np.int32)
tile = np.ascontiguousarray(whole[tids])
try:
    ref_ctx.voxelgrid(tile, 0.005)  # this rank's tile alone is fine
    ctx.voxelgrid_sharded(tile, tids, 0.005)
    raise SystemExit("the union grid did not trip the guard")
except P.Pclb200Error as e:
    assert e.code == P.ERR_LEAF_TOO_SMALL, e
checked += 1

# ---- refusals: ERR_INVALID on every rank, and the communicator still works -------------------------------------------------
_, parts, whole = next(partitions())
tids = np.ascontiguousarray(parts[rank], dtype=np.int32)
tile = np.ascontiguousarray(whole[tids])
want = ctx.voxelgrid_sharded(tile, tids, LEAF, 0)
last = world - 1
other = "another rank refused"
S.refused(lambda: ref_ctx.voxelgrid_sharded(tile, tids, LEAF), "communicator")
S.refused(lambda: ctx.voxelgrid_sharded(tile, tids, 0.0), "leaf size")
S.refused(lambda: ctx.voxelgrid_sharded(tile, tids, float("nan")), "leaf size")
S.refused(lambda: ctx.voxelgrid_sharded(tile, tids, -LEAF if rank == 0 else LEAF), "leaf size" if rank == 0 else other)
S.refused(lambda: ctx.voxelgrid_sharded(tile, tids, float("inf") if rank == last else LEAF),
          "leaf size" if rank == last else other)
dup = tids.copy()
dup[-1] = dup[0]
S.refused(lambda: ctx.voxelgrid_sharded(tile, dup if rank == last else tids, LEAF), "same id" if rank == last else other)
bad = tids.copy()
bad[0] = 2 ** 31 - 1
S.refused(lambda: ctx.voxelgrid_sharded(tile, bad if rank == 0 else tids, LEAF), "[0, 2^31 - 2]" if rank == 0 else other)
S.refused(lambda: ctx.voxelgrid_sharded(tile, tids, LEAF * (1 + (rank == last))), "disagree")
S.refused(lambda: ctx.voxelgrid_sharded(tile, tids, LEAF, 3 if rank == 0 else 2), "disagree")
S.refused(lambda: ctx.voxelgrid_sharded(tile, tids, LEAF, normal_offset=4 if rank == 0 else None), "normals given")
h_out = np.empty((len(tile), 4), np.float32)
h_vox = np.empty(len(tile), np.uint32)
S.refused(lambda: P._check(P.lib().pclb200_voxelgrid_sharded(
    ctx.h, C.c_void_p(tile.ctypes.data), len(tile), 10 if rank == last else 48, C.c_void_p(tids.ctypes.data), None, 0,
    (C.c_float * 3)(LEAF, LEAF, LEAF), 0, C.c_void_p(h_out.ctypes.data), None, C.c_void_p(h_vox.ctypes.data),
    C.byref(C.c_size_t()))), "stride must be" if rank == last else other)
got = ctx.voxelgrid_sharded(tile, tids, LEAF, 0)
assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()
checked += 1

# ---- the output feeds the rest of the sharded pipeline: index the rows under their voxel indices ------------------------
union = np.unique(np.concatenate(parts)).astype(np.int32)
whole_out = ref_ctx.voxelgrid(whole, LEAF, 0, indices=union, is_dense=False)
every = S.gathered(got)
vox_sorted = np.sort(np.concatenate([g[1] for g in every]))
assert vox_sorted.max() <= 2 ** 31 - 2
q = np.ascontiguousarray(whole_out[rng.choice(len(whole_out), 2000)] + np.float32(0.003))
q[:, 3] = 1
tindex = P.Index(ctx, got[0], ids=got[1].astype(np.int32))
for kk in (1, 8, 20):
    gi, gd, keff = tindex.knn_sharded(q, kk)
    wi, wd, wkeff = P.Index(ref_ctx, whole_out).knn(q, kk)
    wi = np.where(wi >= 0, vox_sorted[np.maximum(wi, 0)].astype(np.int64), -1).astype(np.int32)
    assert gi.tobytes() == wi.tobytes() and gd.tobytes() == wd.tobytes() and keff == wkeff, ("knn on the output", kk)
    checked += 1
me.finish("SHARDED_VOXEL", checks=checked)
