"""Statistical outlier removal of a map sharded across ranks (pclb200_statistical_outlier_sharded): per-stage device time
and halo size.

    torchrun --nproc-per-node=R tools/bench_sharded_filters.py [--points N] [--mean-k K] [--std-mul S] [--reps N] [--out F]

The map is bench.py's cfg3 surface (N points over [0, 10)^2, z = 0.5 sin x cos 0.7 y + N(0, 0.002^2)).  Rank 0 first times
one process's pclb200_knn_stats with k = mean_k + 1 on an index of the whole map (the reference; a communicator needs at
least 2 ranks, so there is no single-rank sharded run).  Then every rank times the sharded SOR on its tile's own records
for two partitions, spatial slabs along x and a random partition: the profile scopes of each stage
(sharded_filter_bound: the tile k-NN pass; sharded_filter_halo: boxes, counts and the exchange; sharded_filter_build:
sort, dedup and the index of tile + halo; sharded_filter_stats: the unchanged k-NN statistics on it; sharded_filter_sor:
partial sums, their exchange, the fold and the mask), averaged over --reps calls after one warm-up call.  The halo of
every rank is counted in numpy from the same bound (the tile's k-th nearest distances) as a fraction of the tile.  Rank 0
also checks its tile's mean distances against the reference byte for byte, and the threshold against the sequential sum
of the reference's means over every rank's tile in rank order.  Ranks that share one GPU time-slice it: their times are
stage costs under contention, not a scaling result.  One JSON line per partition, with the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import _sharded as S  # noqa: E402
import pcl_b200 as P  # noqa: E402

STAGES = ("sharded_filter_bound", "sharded_filter_halo", "sharded_filter_build", "sharded_filter_stats", "sharded_filter_sor")


def cfg3_surface(n, seed=7):
    r = np.random.default_rng(seed)
    xy = r.random((n, 2)) * 10.0
    pts = np.ones((n, 4), np.float32)
    pts[:, 0], pts[:, 1] = xy[:, 0], xy[:, 1]
    pts[:, 2] = 0.5 * np.sin(xy[:, 0]) * np.cos(0.7 * xy[:, 1]) + r.normal(0.0, 0.002, n)
    return pts


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=20_000_000)
    ap.add_argument("--mean-k", type=int, default=50)
    ap.add_argument("--std-mul", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    k = a.mean_k + 1
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    shared = torch.cuda.device_count() < world
    dev = 0 if shared else rank
    whole = cfg3_surface(a.points)
    ref_ms, ref_means = None, None
    if rank == 0:  # the reference, before the communicator
        rctx = P.Context(dev)
        d_whole = torch.from_numpy(whole).to(f"cuda:{dev}")
        rindex = P.Index(rctx, d_whole)
        rindex.knn_stats(d_whole, k)
        rctx.synchronize()
        rctx.profile(True)
        rctx.profile_reset()
        for _ in range(a.reps):
            ref_means, _ = rindex.knn_stats(d_whole, k)
        ref_ms = rctx.profile_get("knn_stats")[0] / a.reps
        rctx.profile(False)
        del rindex, d_whole
        rctx.close()
    ctx = S.join(nccl=False, device=dev).ctx  # the other ranks wait here while rank 0 takes its reference
    ids_all = np.arange(a.points)
    slab = np.minimum((whole[:, 0] / 10.0 * world).astype(np.int64), world - 1)
    perm = np.random.default_rng(5).permutation(a.points)
    for pname, parts in (("slabs", [ids_all[slab == r] for r in range(world)]),
                         ("random", [np.sort(perm[r::world]) for r in range(world)])):
        ids = parts[rank].astype(np.int32)
        d_tile = torch.from_numpy(np.ascontiguousarray(whole[ids])).to(f"cuda:{dev}")
        tindex = P.Index(ctx, d_tile, ids=ids)
        tindex.statistical_outlier_removal_sharded(d_tile, a.mean_k, a.std_mul)  # warm-up: maps the tables, fills the cache
        ctx.synchronize()
        ctx.profile(True)
        ctx.profile_reset()
        dist.barrier()
        t0 = time.perf_counter()
        for _ in range(a.reps):
            keep, st = tindex.statistical_outlier_removal_sharded(d_tile, a.mean_k, a.std_mul)
        ctx.synchronize()
        wall_ms = (time.perf_counter() - t0) * 1e3 / a.reps
        stage = {s: round(ctx.profile_get(s)[0] / a.reps, 3) for s in STAGES}
        ctx.profile(False)
        mean_exact, thr_rel = None, None
        if rank == 0:
            means, _ = tindex.knn_stats_sharded(d_tile, k)
            mean_exact = means.tobytes() == np.ascontiguousarray(ref_means[ids]).tobytes()
            every = np.concatenate(parts)
            _, (_, _, thr) = S.sor_rule(ref_means[every], S.finite_rows(whole[every]), a.std_mul)
            thr_rel = abs(st["thr"] - thr) / abs(thr)
        else:
            tindex.knn_stats_sharded(d_tile, k)
        _, kth = tindex.knn_stats(d_tile, k)
        halo = S.halo_points(whole, ids, *S.halo_box(whole[ids], kth))
        mine = dict(rank=rank, tile_points=int(len(ids)), halo_points=halo, halo_fraction=round(halo / len(ids), 5),
                    stage_ms=stage, wall_ms=round(wall_ms, 3), kept=int(keep.sum()), thr=st["thr"])
        allr = S.gathered(mine)
        if rank == 0:
            rec = dict(workload="sharded_sor_cfg3_surface", partition=pname, ranks=world, gpus_shared=shared,
                       map_points=a.points, mean_k=a.mean_k, std_mul=a.std_mul, reps=a.reps,
                       reference_knn_stats_ms=round(ref_ms, 3), rank0_means_bytes_equal_to_reference=mean_exact,
                       rank0_thr_rel_diff_from_sequential=thr_rel, per_rank=allr,
                       note=("ranks time-slice one GPU: stage costs under contention, not scaling" if shared else ""),
                       device=torch.cuda.get_device_name(dev), card_power_limit=card())
            line = json.dumps(rec)
            print(line, flush=True)
            if a.out:
                with open(a.out, "a") as f:
                    f.write(line + "\n")
        del tindex, d_tile
        dist.barrier()
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
