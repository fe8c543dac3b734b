"""Radius search and GICP covariances of a map sharded across ranks (pclb200_radius_into_sharded,
pclb200_gicp_covariances_sharded): per-stage device time, halo size and list totals.

    torchrun --nproc-per-node=R tools/bench_sharded_radius.py [--points N] [--neighbours M] [--k K] [--reps N] [--out F]

The map is bench.py's cfg3 surface (N points over [0, 10)^2, z = 0.5 sin x cos 0.7 y + N(0, 0.002^2)); the radius holds
about M neighbours on it (pi r^2 N / 100 = M).  Rank 0 first times one process's pclb200_radius_into (max_nn 0 and 16)
and pclb200_gicp_covariances (k) on an index of the whole map, with every point as a query (the reference, and the R = 1
row: a communicator needs at least 2 ranks).  Then every rank, for two partitions (spatial slabs along x and a random
partition), times on its tile's own records the sharded radius search with device buffers of the right size (one call
per repetition, all_fit 1) and the sharded covariances: the profile scopes of each stage (sharded_radius_halo: boxes,
counts and the exchange; sharded_radius_build: sort, dedup and the index of tile + halo; sharded_radius_search: the
unchanged radius search on it, the id mapping and the copy; likewise sharded_gicp_bound / _halo / _build and
sharded_gicp_covariances), averaged over --reps calls after one warm-up call.  The halo is counted in numpy from the same
box as a fraction of the tile.  Rank 0 checks its lists and covariances against the reference byte for byte.  Ranks that
share one GPU time-slice it: their times are stage costs under contention, not a scaling result.  One JSON line per
partition, with the card name and power limit."""
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

RADIUS_STAGES = ("sharded_radius_halo", "sharded_radius_build", "sharded_radius_search")
GICP_STAGES = ("sharded_gicp_bound", "sharded_gicp_halo", "sharded_gicp_build", "sharded_gicp_covariances")


def timed(ctx, reps, fn, stages):
    """fn once to warm up, then reps times under the profiler: (last result, mean wall ms, mean ms per stage)"""
    fn()
    ctx.synchronize()
    ctx.profile(True)
    ctx.profile_reset()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    ctx.synchronize()
    wall = (time.perf_counter() - t0) * 1e3 / reps
    st = {s: round(ctx.profile_get(s)[0] / reps, 3) for s in stages}
    ctx.profile(False)
    return out, round(wall, 3), st


def radius_into(index, sharded, q, r, max_nn, dev, cap):
    off = torch.empty(len(q) + 1, dtype=torch.int64, device=f"cuda:{dev}")
    ids = torch.empty(max(cap, 1), dtype=torch.int32, device=f"cuda:{dev}")
    d2 = torch.empty(max(cap, 1), dtype=torch.float32, device=f"cuda:{dev}")
    if sharded:
        total, fit = index.radius_into_sharded(q, r, off, ids, d2, max_nn)
    else:
        total, fit = index.radius_into(q, r, off, ids, d2, max_nn), True
    return off, ids[:total], d2[:total], total, fit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=2_000_000)
    ap.add_argument("--neighbours", type=float, default=30.0)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    radius = float(np.sqrt(a.neighbours * 100.0 / (np.pi * a.points)))
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    shared = torch.cuda.device_count() < world
    dev = 0 if shared else rank
    whole = cfg3_surface(a.points)
    ref = {}
    if rank == 0:  # the reference, before the communicator
        rctx = P.Context(dev)
        d_whole = torch.from_numpy(whole).to(f"cuda:{dev}")
        rindex = P.Index(rctx, d_whole)
        for max_nn in (0, 16):
            total = rindex.radius_into(d_whole, radius, torch.empty(a.points + 1, dtype=torch.int64,
                                                                    device=f"cuda:{dev}"), None, None, max_nn)
            (off, ids, d2, _, _), wall, st = timed(rctx, a.reps, lambda: radius_into(rindex, False, d_whole, radius, max_nn,
                                                                                     dev, total),
                                                   ("radius_count", "radius", "radius_knn"))
            ref[max_nn] = dict(total=total, wall_ms=wall, stage_ms=st, lists=(off.cpu().numpy(), ids.cpu().numpy(),
                                                                             d2.cpu().numpy()))
        cov, wall, st = timed(rctx, a.reps, lambda: rindex.gicp_covariances(d_whole, k=a.k), ("gicp_covariances",))
        ref["gicp"] = dict(wall_ms=wall, stage_ms=st, cov=cov.reshape(-1, 9))
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
        mine = dict(rank=rank, tile_points=int(len(ids)),
                    halo_points=S.halo_points(whole, ids, *S.halo_box(whole[ids], np.float32(radius * radius))))
        mine["halo_fraction"] = round(mine["halo_points"] / len(ids), 5)
        exact = {}
        for max_nn in (0, 16):
            total, _ = tindex.radius_into_sharded(d_tile, radius, torch.empty(len(ids) + 1, dtype=torch.int64,
                                                                              device=f"cuda:{dev}"), None, None, max_nn)
            dist.barrier()
            (off, lid, ld2, total, fit), wall, st = timed(
                ctx, a.reps, lambda: radius_into(tindex, True, d_tile, radius, max_nn, dev, total), RADIUS_STAGES)
            mine[f"radius_max_nn_{max_nn}"] = dict(total=int(total), all_fit=bool(fit), wall_ms=wall, stage_ms=st)
            if rank == 0:
                r_off, r_ids, r_d2 = ref[max_nn]["lists"]
                rows = np.concatenate([np.arange(r_off[i], r_off[i + 1]) for i in ids]) if len(ids) else np.zeros(0, int)
                exact[max_nn] = (np.diff(off.cpu().numpy()).tobytes() == np.diff(r_off)[ids].tobytes()
                                 and lid.cpu().numpy().tobytes() == r_ids[rows].tobytes()
                                 and ld2.cpu().numpy().tobytes() == r_d2[rows].tobytes())
        dist.barrier()
        cov, wall, st = timed(ctx, a.reps, lambda: tindex.gicp_covariances_sharded(d_tile, k=a.k), GICP_STAGES)
        mine["gicp"] = dict(wall_ms=wall, stage_ms=st)
        if rank == 0:
            exact["gicp"] = cov.reshape(-1, 9).tobytes() == np.ascontiguousarray(ref["gicp"]["cov"][ids]).tobytes()
        allr = S.gathered(mine)
        if rank == 0:
            rec = dict(workload="sharded_radius_cfg3_surface", partition=pname, ranks=world, gpus_shared=shared,
                       map_points=a.points, radius=radius, neighbours_target=a.neighbours, k=a.k, reps=a.reps,
                       reference={str(m): dict(total=ref[m]["total"], wall_ms=ref[m]["wall_ms"],
                                               stage_ms=ref[m]["stage_ms"]) for m in (0, 16)},
                       reference_gicp=dict(wall_ms=ref["gicp"]["wall_ms"], stage_ms=ref["gicp"]["stage_ms"]),
                       rank0_bytes_equal_to_reference={str(k): v for k, v in exact.items()}, per_rank=allr,
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
