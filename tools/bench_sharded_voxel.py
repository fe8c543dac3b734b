"""VoxelGrid of a map sharded across ranks (pclb200_voxelgrid_sharded): per-stage device time, shared records and device
memory.

    torchrun --nproc-per-node=R tools/bench_sharded_voxel.py [--points N] [--leaf L] [--reps N] [--out F]

The map is bench.py's cfg3 surface (N points over [0, 10)^2, z = 0.5 sin x cos 0.7 y + N(0, 0.002^2)); the default leaf,
0.01, gives about 10^6 voxels.  Rank 0 first times one process's pclb200_voxelgrid on the whole map (the reference; a
communicator needs at least 2 ranks, so there is no single-rank sharded run).  Then every rank times the sharded call on
its tile for two partitions, spatial slabs along x and a random partition: the profile scopes of each stage
(sharded_voxel_boxes: id check, staging, min / max and the first exchange; sharded_voxel_exchange: voxel ranges, counts
and the record exchange; sharded_voxel_centroids: the 64-bit sort, ownership and the unchanged centroid kernels), averaged
over --reps calls after one warm-up call.  The records each rank receives are counted in numpy from the same rule (the
voxel range of its box) as a fraction of its tile.  Device memory in use is read after the last call (the ranks that share
a GPU see each other's).  The rows of every rank, sorted by voxel index, are compared with the reference byte for byte.
Ranks that share one GPU time-slice it: their times are stage costs under contention, not a scaling result.  One JSON
line per partition, with the card name and power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import _sharded as S  # noqa: E402
import pcl_b200 as P  # noqa: E402
from bench_sharded_filters import card, cfg3_surface  # noqa: E402

STAGES = ("sharded_voxel_boxes", "sharded_voxel_exchange", "sharded_voxel_centroids")


def received(whole, parts, leaf):
    """per rank: the records of the other ranks whose voxel lies in the voxel range of its box (float arithmetic of the
    kernels: floor(x * inv) - min_b in float)"""
    inv = np.float32(1) / np.float32(leaf)
    xyz = whole[:, :3]
    min_b = np.floor((xyz.min(0) * inv).astype(np.float32))
    ijk = (np.floor((xyz * inv).astype(np.float32)) - min_b).astype(np.int64)
    rng_ = []
    for p in parts:
        lo, hi = xyz[p].min(0), xyz[p].max(0)
        rng_.append(((np.floor((lo * inv).astype(np.float32)) - min_b).astype(np.int64),
                     (np.floor((hi * inv).astype(np.float32)) - min_b).astype(np.int64)))
    out = []
    for r, (lo, hi) in enumerate(rng_):
        out.append(int(sum(((ijk[p] >= lo) & (ijk[p] <= hi)).all(1).sum() for s, p in enumerate(parts) if s != r)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=20_000_000)
    ap.add_argument("--leaf", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    shared = torch.cuda.device_count() < world
    dev = 0 if shared else rank
    whole = cfg3_surface(a.points)
    ref_ms, ref_rows = None, None
    if rank == 0:  # the reference, before the communicator
        rctx = P.Context(dev)
        d_whole = torch.from_numpy(whole).to(f"cuda:{dev}")
        rctx.voxelgrid(d_whole, a.leaf)
        rctx.synchronize()
        rctx.profile(True)
        rctx.profile_reset()
        for _ in range(a.reps):
            ref_rows = rctx.voxelgrid(d_whole, a.leaf)
        ref_ms = rctx.profile_get("voxelgrid")[0] / a.reps
        rctx.profile(False)
        del d_whole
        rctx.close()
    ctx = S.join(nccl=False, device=dev).ctx  # the other ranks wait here while rank 0 takes its reference
    ids_all = np.arange(a.points)
    slab = np.minimum((whole[:, 0] / 10.0 * world).astype(np.int64), world - 1)
    perm = np.random.default_rng(5).permutation(a.points)
    for pname, parts in (("slabs", [ids_all[slab == r] for r in range(world)]),
                         ("random", [np.sort(perm[r::world]) for r in range(world)])):
        ids = parts[rank].astype(np.int32)
        d_tile = torch.from_numpy(np.ascontiguousarray(whole[ids])).to(f"cuda:{dev}")
        d_ids = torch.from_numpy(ids).to(f"cuda:{dev}")
        ctx.voxelgrid_sharded(d_tile, d_ids, a.leaf)  # warm-up: maps the tables, fills the cache
        ctx.synchronize()
        ctx.profile(True)
        ctx.profile_reset()
        dist.barrier()
        t0 = time.perf_counter()
        for _ in range(a.reps):
            rows, vox = ctx.voxelgrid_sharded(d_tile, d_ids, a.leaf)
        ctx.synchronize()
        wall_ms = (time.perf_counter() - t0) * 1e3 / a.reps
        stage = {s: round(ctx.profile_get(s)[0] / a.reps, 3) for s in STAGES}
        ctx.profile(False)
        free, total = torch.cuda.mem_get_info(dev)
        recv = received(whole, parts, a.leaf)[rank]
        mine = dict(rank=rank, tile_points=int(len(ids)), received_records=recv, received_fraction=round(recv / len(ids), 5),
                    voxels=int(len(vox)), stage_ms=stage, wall_ms=round(wall_ms, 3),
                    device_used_gb_after_call=round((total - free) / 2 ** 30, 3))
        every = S.gathered((mine, rows, vox))
        if rank == 0:
            v = np.concatenate([e[2] for e in every])
            got = np.concatenate([e[1] for e in every])[np.argsort(v, kind="stable")]
            rec = dict(workload="sharded_voxelgrid_cfg3_surface", partition=pname, ranks=world, gpus_shared=shared,
                       map_points=a.points, leaf=a.leaf, reps=a.reps, reference_voxelgrid_ms=round(ref_ms, 3),
                       reference_voxels=int(len(ref_rows)), rows_bytes_equal_to_reference=got.tobytes() == ref_rows.tobytes(),
                       per_rank=[e[0] for e in every],
                       note=("ranks time-slice one GPU: stage costs under contention, not scaling" if shared else ""),
                       device=torch.cuda.get_device_name(dev), card_power_limit=card())
            line = json.dumps(rec)
            print(line, flush=True)
            if a.out:
                with open(a.out, "a") as f:
                    f.write(line + "\n")
        del d_tile, d_ids
        dist.barrier()
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
