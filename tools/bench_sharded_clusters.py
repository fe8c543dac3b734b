"""Euclidean clusters of a map sharded across ranks (pclb200_cluster_labels_sharded): per-stage device time, halo size
and device memory.

    torchrun --nproc-per-node=R tools/bench_sharded_clusters.py [--points N] [--tolerance T] [--reps N] [--out F]

The map is a scene of separated objects in the manner of bench.py's cfg4 (planar patches, N(0, 0.002^2) noise), laid on a
4 x 4 x 2 grid of 10 m cells so that no two objects touch: planar 6 m x 6 m patches and the surfaces of 4 m boxes,
alternately, points in proportion to area.  At 20 M points the spacing is about 1 cm and the default tolerance is 2 cm.
Rank 0 first times one process's pclb200_cluster_labels on an index of the whole map (CUDA-synchronised wall time).  Then
every rank times the sharded call on its tile for spatial slabs of [0, 30) along x (cut through a column of
objects) and a random partition: the profile scopes of
each stage (sharded_cluster_halo: boxes, counts, the exchange, sort and index of tile + halo; _local: the unchanged
clustering of it; _stitch: answers, edges, their all-gather and the union-find; _labels: sizes and output), averaged
over --reps calls after one warm-up call.  The halo is counted in numpy from the same box as a fraction of the tile;
cross-rank components are the labels more than one rank returns.  Device memory: the drop of free memory on the card
over the warm-up call (the library's block cache keeps the peak), per map point.  Rank 0 checks its labels against the
reference byte for byte.  Ranks that share one GPU time-slice it: their times are stage costs under contention, not a
scaling result.  One JSON line per partition, with the card name and power limit."""
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

STAGES = ("sharded_cluster_halo", "sharded_cluster_local", "sharded_cluster_stitch", "sharded_cluster_labels")


def scene(n, seed=11):
    r = np.random.default_rng(seed)
    objs = []  # (origin, list of (corner, u, v) faces)
    for i in range(32):
        o = np.array([10.0 * (i % 4) + 2, 10.0 * (i // 4 % 4) + 2, 10.0 * (i // 16) + 2])
        if i % 2 == 0:
            objs.append([(o, np.array([6.0, 0, 0]), np.array([0, 6.0, 0]))])
        else:
            e = np.eye(3) * 4.0
            faces = []
            for a in range(3):
                u, v = e[(a + 1) % 3], e[(a + 2) % 3]
                faces += [(o, u, v), (o + e[a], u, v)]
            objs.append(faces)
    faces = [f for ob in objs for f in ob]
    area = np.array([np.linalg.norm(np.cross(u, v)) for (_, u, v) in faces])
    counts = np.floor(n * area / area.sum()).astype(np.int64)
    counts[0] += n - counts.sum()
    out = np.ones((n, 4), np.float32)
    k = 0
    for (c, u, v), m in zip(faces, counts):
        ab = r.random((m, 2))
        out[k:k + m, :3] = (c + ab[:, :1] * u + ab[:, 1:] * v + r.normal(0.0, 0.002, (m, 3))).astype(np.float32)
        k += m
    return out


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
    ap.add_argument("--tolerance", type=float, default=0.02)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    shared = torch.cuda.device_count() < world
    dev = 0 if shared else rank
    whole = scene(a.points)
    ref_ms, ref_labels, n_clusters = None, None, None
    if rank == 0:  # the reference, before the communicator
        rctx = P.Context(dev)
        d_whole = torch.from_numpy(whole).to(f"cuda:{dev}")
        rindex = P.Index(rctx, d_whole)
        out = torch.empty(a.points, dtype=torch.int32, device=f"cuda:{dev}")
        rindex.cluster_labels(a.tolerance, out=out)
        rctx.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.reps):
            rindex.cluster_labels(a.tolerance, out=out)
        rctx.synchronize()
        ref_ms = (time.perf_counter() - t0) * 1e3 / a.reps
        ref_labels = out.cpu().numpy()
        n_clusters = int(len(np.unique(ref_labels[ref_labels >= 0])))
        del rindex, d_whole, out
        rctx.close()
    ctx = S.join(nccl=False, device=dev).ctx  # the other ranks wait here while rank 0 takes its reference
    ids_all = np.arange(a.points)
    slab = np.minimum((whole[:, 0] / 30.0 * world).astype(np.int64), world - 1)  # R = 2: cut at x = 15 m, through objects
    perm = np.random.default_rng(5).permutation(a.points)
    for pname, ids in (("slabs", ids_all[slab == rank]), ("random", np.sort(perm[rank::world]))):
        ids = ids.astype(np.int32)
        d_tile = torch.from_numpy(np.ascontiguousarray(whole[ids])).to(f"cuda:{dev}")
        tindex = P.Index(ctx, d_tile, ids=ids)
        labels = torch.empty(len(ids), dtype=torch.int32, device=f"cuda:{dev}")
        sizes = torch.empty(len(ids), dtype=torch.int64, device=f"cuda:{dev}")
        ctx.synchronize()
        dist.barrier()
        free0, _ = torch.cuda.mem_get_info(dev)
        dist.barrier()
        tindex.cluster_labels_sharded(a.tolerance, out=labels, sizes=sizes)  # warm-up: maps the tables, fills the cache
        ctx.synchronize()
        dist.barrier()
        free1, _ = torch.cuda.mem_get_info(dev)
        ctx.profile(True)
        ctx.profile_reset()
        dist.barrier()
        t0 = time.perf_counter()
        for _ in range(a.reps):
            tindex.cluster_labels_sharded(a.tolerance, out=labels, sizes=sizes)
        ctx.synchronize()
        wall_ms = (time.perf_counter() - t0) * 1e3 / a.reps
        stage = {s: round(ctx.profile_get(s)[0] / a.reps, 3) for s in STAGES}
        ctx.profile(False)
        lab = labels.cpu().numpy()
        exact = None
        if rank == 0:
            exact = lab.tobytes() == np.ascontiguousarray(ref_labels[ids]).tobytes()
        r2 = np.float32(np.float64(np.float32(a.tolerance)) ** 2)  # the tile widened by the reach of r2
        halo = S.halo_points(whole, ids, *S.halo_box(whole[ids], r2))
        mine = dict(rank=rank, tile_points=int(len(ids)), halo_points=halo, halo_fraction=round(halo / len(ids), 5),
                    stage_ms=stage, wall_ms=round(wall_ms, 3))
        allr = S.gathered(mine)
        labs = S.gathered(np.unique(lab))
        if rank == 0:
            seen = np.concatenate(labs)
            _, times = np.unique(seen, return_counts=True)
            rec = dict(workload="sharded_clusters_separated_objects", partition=pname, ranks=world, gpus_shared=shared,
                       map_points=a.points, tolerance=a.tolerance, clusters=n_clusters, reps=a.reps,
                       reference_cluster_labels_ms=round(ref_ms, 3), rank0_bytes_equal_to_reference=exact,
                       cross_rank_components=int((times > 1).sum()),
                       card_bytes_per_map_point_over_first_call=round((free0 - free1) / a.points, 2),
                       per_rank=allr,
                       note=("ranks time-slice one GPU: stage costs under contention, not scaling" if shared else ""),
                       device=torch.cuda.get_device_name(dev), card_power_limit=card())
            line = json.dumps(rec)
            print(line, flush=True)
            if a.out:
                with open(a.out, "a") as f:
                    f.write(line + "\n")
        del tindex, d_tile, labels, sizes
        dist.barrier()
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
