"""VoxelGrid of a map sharded across ranks without a GPU: the kernels of pcl_b200/csrc/shard_voxel_kernels.cuh (driven by
shard_voxel.cu) compiled for the host against the host-compiled single-process VoxelGrid, and the rule they implement
stated in numpy against the numpy VoxelGrid of tests/test_consumers_reference.py, with the scenes shown to catch three
wrong rules.

The rule (DESIGN.md §5, "VoxelGrid of a sharded map"): the grid is the whole map's (the union of every rank's box).  Rank
s's voxel range I_s holds the voxels of its box's faces; every rank sends every finite record whose voxel lies in I_s to
rank s.  Each rank sorts its own and received records by (voxel, id), counts every id once and knows, per voxel, the ranks
holding a record of it.  The owner of voxel v, member v mod |holders| of the holders in rank order, returns it when the
whole run has min_points_per_voxel records, summed in id order."""
import numpy as np
import pytest

import _sharded as S
import test_consumers_reference as TC


@S.needs_host_compiler
def test_sharded_voxel_kernels_on_the_host(tmp_path):
    """1 / 2 / 3 / 5 / 8 simulated ranks, both exchange protocols, six partitions, three leaves, min_points_per_voxel
    0 / 1 / 3, with and without normals: every rank's rows sorted by voxel equal the single-process VoxelGrid of the whole
    map byte for byte; no voxel on two ranks; the guard trips on the union grid exactly when on the whole map's; a grid
    whose voxel indices reach 2^31 and beyond while the guard passes."""
    out = S.host_program(tmp_path, "shard_voxel_host_test.cpp", timeout=900)
    lines = out.splitlines()
    assert any(l.startswith("one rank empty") and "R=8 nccl" in l for l in lines)
    assert sum(l.startswith("far tile") and l.endswith("guard") for l in lines) == 8
    assert sum(l.startswith("voxels above 2^31") and l.endswith(" ok") for l in lines) == 4
    assert "DIFFERS" not in out


def sharded_rule(whole, parts, leaf, min_pts=0, normal=False, rank_order=False, float_box=False, share_min=False):
    """Per rank (voxel indices, centroids, normal rows or None) of the sharded VoxelGrid, or None where the whole map's
    grid trips the guard.  The wrong rules: rank_order sums a voxel's records in (rank, id) order; float_box sends a rank
    the records inside its float box instead of its voxel range; share_min applies min_pts to the owner's own share."""
    xyz = whole[:, :3].astype(np.float32)
    fin = np.isfinite(xyz).all(1)
    own = [np.asarray(p, np.int64)[fin[p]] for p in parts]
    held = np.unique(np.concatenate(own))
    empty = (np.zeros(0, np.uint32), np.zeros((0, 4), np.float32), np.zeros((0, 8), np.float32) if normal else None)
    if held.size == 0:
        return [empty] * len(parts)
    grid = TC.voxel_grid(xyz[held], leaf)
    if grid is None:
        return None
    inv, min_b = grid[0], grid[1]

    def ijk(v):
        return (np.floor((v * inv).astype(np.float32)) - min_b.astype(np.float32)).astype(np.int64)

    key = np.zeros(len(whole), np.uint32)
    key[held] = TC.voxel_keys(xyz[held], *grid)
    vox_ijk = np.zeros((len(whole), 3), np.int64)
    vox_ijk[held] = ijk(xyz[held])
    boxes = [(xyz[o].min(0), xyz[o].max(0)) if o.size else None for o in own]
    out = []
    for r in range(len(parts)):
        ids, holder = [own[r]], [np.full(own[r].size, r)]
        for s in range(len(parts)):
            if s == r or boxes[r] is None:
                continue
            lo, hi = boxes[r]
            if float_box:
                inside = ((xyz[own[s]] >= lo) & (xyz[own[s]] <= hi)).all(1)
            else:
                inside = ((vox_ijk[own[s]] >= ijk(lo)) & (vox_ijk[own[s]] <= ijk(hi))).all(1)
            ids.append(own[s][inside])
            holder.append(np.full(int(inside.sum()), s))
        ids, holder = np.concatenate(ids), np.concatenate(holder)
        if not ids.size:
            out.append(empty)
            continue
        k = key[ids].astype(np.int64)
        order = np.lexsort((ids, holder, k)) if rank_order else np.lexsort((holder, ids, k))
        ids, holder, k = ids[order], holder[order], k[order]
        starts = np.nonzero(np.r_[True, k[1:] != k[:-1]])[0]
        mask = np.bitwise_or.reduceat(np.left_shift(1, holder), starts)
        _, first = np.unique(ids * (1 << 32) + k, return_index=True)  # each (voxel, id) once, the first in this order
        keep_rec = np.zeros(ids.size, bool)
        keep_rec[first] = True
        ids, k, holder = ids[keep_rec], k[keep_rec], holder[keep_rec]
        starts = np.nonzero(np.r_[True, k[1:] != k[:-1]])[0]
        ends = np.r_[starts[1:], k.size]
        v = k[starts]
        count = ends - starts
        if share_min:
            count = np.add.reduceat((holder == r).astype(np.int64), starts)
        n_hold = np.array([bin(int(m)).count("1") for m in mask])
        nth = v % n_hold
        owner = np.array([[b for b in range(8) if (int(m) >> b) & 1][int(t)] for m, t in zip(mask, nth)], np.int64)
        keep = ((mask >> r) & 1).astype(bool) & (owner == r) & (count >= min_pts)
        starts, ends = starts[keep], ends[keep]
        fn = (ends - starts).astype(np.float32)[:, None]
        rows = np.ones((starts.size, 4), np.float32)
        rows[:, :3] = TC.sequential_sums(xyz[ids], np.arange(ids.size), starts, ends) / fn
        nc = None
        if normal:
            s = TC.sequential_sums(whole[ids, 4:9].astype(np.float32), np.arange(ids.size), starts, ends)
            n4 = s[:, :4]
            sq = ((n4[:, 0] * n4[:, 0] + n4[:, 1] * n4[:, 1]) + (n4[:, 2] * n4[:, 2] + n4[:, 3] * n4[:, 3])).astype(np.float32)
            nc = np.zeros((starts.size, 8), np.float32)
            nc[:, :4] = np.where((sq > 0)[:, None], n4 / np.where(sq > 0, np.sqrt(sq), 1)[:, None], n4)
            nc[:, 4] = s[:, 4] / fn[:, 0]
        out.append((v[keep].astype(np.uint32), rows, nc))
    return out


def _scene():
    rng = np.random.default_rng(43)
    xyz = np.concatenate([S.surface(rng, 20000),
                          np.c_[np.stack(np.meshgrid(*[np.arange(40, dtype=np.float32) * np.float32(0.05)] * 2,
                                                     indexing="ij"), -1).reshape(-1, 2), np.full(1600, np.float32(0.1))]])
    whole = TC.point_normal(S.with_extras(rng, xyz)[:, :3], rng.normal(size=(len(xyz) + 200, 3)).astype(np.float32),
                            rng.random(len(xyz) + 200, dtype=np.float32) * np.float32(0.01))
    return rng, whole


def _partitions(rng, whole, world):
    for name, parts, w in S.partitions(rng, np.ascontiguousarray(whole[:, :4]), world):
        yield name, parts, whole if len(w) == len(whole) else np.concatenate([whole, TC.point_normal(w[len(whole):, :3])])
    ids = np.arange(len(whole))
    ix = np.floor((np.nan_to_num(whole[:, 0]) * (np.float32(1) / np.float32(0.05))).astype(np.float32)).astype(np.int64)
    yield "voxel faces", [ids[np.minimum(ix * world // (ix.max() + 1), world - 1) == r] for r in range(world)], whole
    yield "one rank empty", [ids[r::world - 1] for r in range(world - 1)] + [ids[:0]], whole


def _joined(per_rank):
    vox = np.concatenate([p[0] for p in per_rank])
    order = np.argsort(vox, kind="stable")
    rows = np.concatenate([p[1] for p in per_rank])[order]
    nc = np.concatenate([p[2] for p in per_rank])[order] if per_rank[0][2] is not None else None
    return vox, rows, nc


CASES = [(0.012, 0, False), (0.05, 3, True), (0.3, 1, False), (0.3, 3, False)]


@pytest.mark.parametrize("world", [2, 3])
def test_the_rule_gives_the_whole_maps_voxelgrid(world):
    """The numpy rule on every partition and leaf: the ranks' rows sorted by voxel equal the numpy VoxelGrid of the whole
    map with the sorted union of the ids, byte for byte, each voxel on one rank and no rank with more rows than records."""
    rng, whole0 = _scene()
    for name, parts, whole in _partitions(rng, whole0, world):
        union = np.unique(np.concatenate(parts))
        for leaf, mp, normal in CASES:
            want = TC.voxel_ref(whole, leaf, mp, indices=union, normal=normal)
            got = sharded_rule(whole, parts, leaf, mp, normal)
            if want is None:
                assert got is None, (name, leaf)
                continue
            vox, rows, nc = _joined(got)
            assert len(np.unique(vox)) == len(vox), (name, leaf, mp)
            assert all(len(g[0]) <= len(p) for g, p in zip(got, parts)), (name, leaf, mp)
            assert rows.tobytes() == want[0].tobytes(), (name, leaf, mp)
            assert not normal or nc.tobytes() == want[1].tobytes(), (name, leaf, mp)


def test_the_scenes_catch_three_wrong_rules():
    """Summing a voxel in (rank, id) order, sending the records inside a rank's float box instead of its voxel range, and
    applying min_points_per_voxel to the owner's share each change the rows of at least one scene."""
    rng, whole0 = _scene()
    caught = {"rank_order": 0, "float_box": 0, "share_min": 0}
    for name, parts, whole in _partitions(rng, whole0, 3):
        union = np.unique(np.concatenate(parts))
        for leaf, mp, normal in CASES:
            want = TC.voxel_ref(whole, leaf, mp, indices=union)
            if want is None:
                continue
            for wrong in caught:
                vox, rows, _ = _joined(sharded_rule(whole, parts, leaf, mp, **{wrong: True}))
                caught[wrong] += rows.tobytes() != want[0].tobytes()
    print(caught)
    assert all(caught.values()), caught
