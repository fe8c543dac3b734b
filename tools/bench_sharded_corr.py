"""Correspondences, inliers and validation against a map sharded across ranks (pclb200_correspondences_sharded,
pclb200_correspondences_normals_sharded, pclb200_inliers_sharded, pclb200_validate_transformation_sharded), against one
process on the whole map.

    torchrun --nproc-per-node=R tools/bench_sharded_corr.py [--map-points M] [--source-points S] [--calls K] [--out F]

The map is a surface of M points cut into R spatial slabs, one per rank; every rank holds the whole source (S points, a
moved sample of the surface).  Each call is timed on the host around a device synchronise, after one warm-up call (which
maps the exchange tables), and its profile scopes are averaged: shard_corr_keys (tile search, key exchange, list),
shard_corr_records (record exchange and rows), shard_corr_knn (the tile's k-NN rows, their exchange and merge) and
shard_corr_select (candidate scores, their exchange, the choice).  Then rank 0 times the single-GPU calls on one index
of the whole map while the other ranks wait.  When the ranks share one GPU the sharded times are costs under time-slicing, not a scaling.  One
JSON line from rank 0, with the card's name and power limit read in the same run."""
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
from bench_sharded_target import power_limit, surface  # noqa: E402


def timed(ctx, fn, calls, scopes=()):
    fn()
    ctx.synchronize()
    ctx.profile(True)
    ctx.profile_reset()
    ts = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        ctx.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    out = dict(call_ms_median=round(float(np.median(ts)), 3))
    for s in scopes:
        out[s + "_ms"] = round(ctx.profile_get(s)[0] / calls, 3)
    ctx.profile(False)
    return out


def raw_inliers(index, src, T, thr):
    """pclb200_inliers itself (Index.inliers also sums the fitness in Python, one float at a time)"""
    b = P._Buf(src)
    T = np.ascontiguousarray(T, np.float64)
    out = np.empty(len(src), P.CORR_DTYPE)
    m = P.C.c_size_t()
    P._check(P.lib().pclb200_inliers(index.ctx.h, index.h, b.ptr, b.rows, b.stride, T.ctypes.data_as(P.C.POINTER(P.C.c_double)),
                                     float(thr), P.C.c_void_p(out.ctypes.data), P.C.byref(m)))
    return out[:m.value]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--map-points", type=int, default=20_000_000)
    ap.add_argument("--source-points", type=int, default=1_000_000)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--max-correspondence-distance", type=float, default=0.25)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    shared = torch.cuda.device_count() < world
    dev = 0 if shared else rank
    me = S.join(nccl=False, device=dev)
    ctx = me.ctx
    extent = 100.0
    whole = surface(a.map_points, 1, extent)
    nrm = np.zeros((a.map_points, 4), np.float32)
    nrm[:, 2] = 1
    cut = np.minimum((whole[:, 0] / extent * world).astype(np.int64), world - 1)
    ids = np.nonzero(cut == rank)[0].astype(np.int32)
    tile, tnrm = np.ascontiguousarray(whole[ids]), np.ascontiguousarray(nrm[ids])
    tindex = P.Index(ctx, tile, ids=ids)
    rng = np.random.default_rng(2)
    src = surface(a.source_points, 3, extent)
    ang = np.deg2rad(1.0)
    Rm = np.array([[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1]])
    src[:, :3] = (src[:, :3].astype(np.float64) @ Rm.T + [0.05, -0.03, 0.02]).astype(np.float32)
    src[:, :3] += rng.normal(0, 0.002, (a.source_points, 3)).astype(np.float32)
    src_index = P.Index(ctx, src)
    snrm = np.zeros((a.source_points, 4), np.float32)
    snrm[:, 2] = 1
    md, T = a.max_correspondence_distance, np.eye(4)
    T[:3, :3] = Rm.T
    keys, recs = ("shard_corr_keys",), ("shard_corr_keys", "shard_corr_records")
    dist.barrier()
    sharded = dict(
        nearest=timed(ctx, lambda: tindex.correspondences_sharded(src, md), a.calls, keys),
        nearest_rows_normals=timed(ctx, lambda: tindex.correspondences_sharded(src, md, tgt_normals=tnrm, rows=True,
                                                                               normal_rows=True), a.calls, recs),
        reciprocal=timed(ctx, lambda: tindex.correspondences_sharded(src, md, src_index=src_index), a.calls, keys),
        inliers=timed(ctx, lambda: tindex.inliers_sharded(src, T, 0.1), a.calls, keys),
        normal_shooting_k10=timed(ctx, lambda: tindex.correspondences_normals_sharded(P.CORR_NORMAL_SHOOTING, src, snrm, k=10,
                                                                                     max_distance=md), a.calls,
                                  ("shard_corr_knn", "shard_corr_select")),
        validate=timed(ctx, lambda: tindex.validate_transformation_sharded(src, T), a.calls))
    n_pairs = S.gathered(len(tindex.correspondences_sharded(src, md)))
    assert all(x == n_pairs[0] for x in n_pairs), n_pairs
    dist.barrier()
    single = None
    if rank == 0:  # one process on the whole map, the other ranks idle
        ref = me.ref
        index = P.Index(ref, whole)
        rsrc = P.Index(ref, src)
        single = dict(nearest=timed(ref, lambda: index.correspondences(src, md), a.calls),
                      reciprocal=timed(ref, lambda: index.correspondences(src, md, src_index=rsrc), a.calls),
                      inliers=timed(ref, lambda: raw_inliers(index, src, T, 0.1), a.calls),
                      normal_shooting_k10=timed(ref, lambda: index.correspondences_normals(P.CORR_NORMAL_SHOOTING, src, snrm,
                                                                                           k=10, max_distance=md), a.calls),
                      validate=timed(ref, lambda: index.validate_transformation(src, T), a.calls))
        assert len(index.correspondences(src, md)) == n_pairs[0]
    dist.barrier()
    if rank == 0:
        rec = dict(workload="sharded_corr", ranks=world, gpus_shared=shared, map_points=a.map_points,
                   source_points=a.source_points, gate=md, pairs=n_pairs[0], sharded=sharded, single_process=single,
                   r_gpu_rates="not measured", nccl_path="not measured",
                   device=torch.cuda.get_device_name(dev), card_power_limit=power_limit())
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
