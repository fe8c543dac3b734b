"""Scan-to-map registration against a map sharded across ranks (pclb200_index_build_ids + pclb200_icp_set_target_sharded).

    torchrun --nproc-per-node=R tools/bench_sharded_target.py [--map-points M] [--source-points S] [--aligns K] [--out F]

The map is a surface of M points cut into R spatial slabs, one per rank; every rank holds the whole source (S points, a
moved sample of the surface).  One process per GPU when the box has R GPUs (peer exchange through CUDA IPC, bootstrapped
over gloo); with fewer GPUs the ranks share cuda:0 and the run checks correctness only (no rate is printed).  Per align it
reports the total and the profile scopes (search, exchange, accumulate, solve), and the memory the tile's index takes:
pclb200_index_stats()[2] per point, and the device memory the build left in use (the index plus the library's block cache,
i.e. the build's peak) per point, from which the largest map that fits one GPU's free memory follows.  One JSON line per
rank 0 run, with the card name and its power limit."""
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


def surface(n, seed, extent):
    rng = np.random.default_rng(seed)
    pts = np.ones((n, 4), np.float32)
    pts[:, :2] = rng.random((n, 2), dtype=np.float32) * extent
    pts[:, 2] = 0.5 * np.sin(pts[:, 0] * 0.7) * np.cos(pts[:, 1] * 0.5)
    return pts


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--map-points", type=int, default=20_000_000)
    ap.add_argument("--source-points", type=int, default=1_000_000)
    ap.add_argument("--aligns", type=int, default=5)
    ap.add_argument("--max-correspondence-distance", type=float, default=0.0, help="0 = unbounded (the default gate)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    shared = torch.cuda.device_count() < world
    dev = 0 if shared else rank
    ctx = S.join(nccl=False, device=dev).ctx
    extent = 100.0
    whole = surface(a.map_points, 1, extent)
    cut = np.minimum((whole[:, 0] / extent * world).astype(np.int64), world - 1)
    ids = np.nonzero(cut == rank)[0].astype(np.int32)
    tile = np.ascontiguousarray(whole[ids])
    del whole
    free0, total = torch.cuda.mem_get_info(dev)
    t0 = time.perf_counter()
    # one rank: the single-GPU session on the whole map (a sharded target needs a communicator), the baseline of the rates
    index = P.Index(ctx, tile, ids=ids) if world > 1 else P.Index(ctx, tile)
    ctx.synchronize()
    build_s = time.perf_counter() - t0
    free1, _ = torch.cuda.mem_get_info(dev)
    stats = index.stats
    rng = np.random.default_rng(2)
    src = surface(a.source_points, 3, extent)
    ang = np.deg2rad(1.0)
    Rm = np.array([[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1]])
    src[:, :3] = (src[:, :3].astype(np.float64) @ Rm.T + [0.05, -0.03, 0.02]).astype(np.float32)
    src[:, :3] += rng.normal(0, 0.002, (a.source_points, 3)).astype(np.float32)
    kw = dict(max_iterations=20, transformation_epsilon=1e-10)
    if a.max_correspondence_distance > 0:
        kw["max_correspondence_distance"] = a.max_correspondence_distance
    icp = P.Icp(ctx, P.default_params(**kw))
    if world > 1:
        icp.set_target_sharded(index)
    else:
        icp.set_target(index)
    scopes = ("icp_search", "icp_exchange", "icp_accum", "solve")
    times, per_scope, iters = [], {s: 0.0 for s in scopes}, 0
    for k in range(a.aligns + 1):
        icp.set_source(src)
        ctx.profile(k > 0)
        ctx.profile_reset()
        dist.barrier()
        t0 = time.perf_counter()
        st = icp.iterate()
        ctx.synchronize()
        dt = time.perf_counter() - t0
        if k > 0:  # the first align maps the exchange arrays and warms the block cache
            times.append(dt * 1e3)
            for s in scopes:
                per_scope[s] += ctx.profile_get(s)[0] / a.aligns
            iters = st["iterations"]
    ctx.profile(False)
    finals = S.gathered(st["final"].tobytes())
    assert all(f == finals[0] for f in finals), "ranks disagree on the transform"
    per_pt_index = stats["bytes"] / max(len(ids), 1)
    per_pt_peak = (free0 - free1) / max(len(ids), 1)
    rec = dict(workload="sharded_target_scan_to_map", ranks=world, gpus_shared=shared, map_points=a.map_points,
               tile_points=int(len(ids)), source_points=a.source_points,
               gate=a.max_correspondence_distance or "unbounded", iterations=iters, build_s=round(build_s, 3),
               index_bytes_per_point=round(per_pt_index, 2), build_peak_bytes_per_point=round(per_pt_peak, 2),
               largest_map_one_gpu_points=int(free0 / per_pt_peak) if per_pt_peak > 0 else None,
               largest_map_r_gpus_points=int(world * free0 / per_pt_peak) if per_pt_peak > 0 and not shared else None,
               device=torch.cuda.get_device_name(dev), card_power_limit=power_limit())
    if not shared:
        rec.update(align_ms_median=round(float(np.median(times)), 3),
                   scope_ms_per_align={s: round(v, 3) for s, v in per_scope.items()})
    if rank == 0:
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
