"""Index-build throughput on one GPU: one batch build of B clouds (pclb200_index_build_batch) against a loop of B single
builds (pclb200_index_build), and what that does to scan pairs with their builds counted.

    python tools/bench_index_batch.py [--out profiles/h100_index_batch.jsonl] [--reps 3]

The clouds are the target windows of the odometry chain of bench_icp_pairs.py (make_chain): B + 1 windows of n points,
pair k aligning window k + 1 to window k.  Grid: n in {8 k, 32 k, 128 k} x B in {1, 8, 64, 256}.  Each row reports
  * build: the loop of single builds and the batch build, seconds and clouds/s;
  * normals_s: the k = 16 normals of every window, one normals_knn per handle, timed on its own (the batch build does not
    batch them);
  * pairs: point-to-plane pairs/s with everything a pair needs counted, the batch build + normals + one batch align
    (set_target_batch) against single builds + normals + a loop of single aligns.
Before anything is timed, every batch-built handle is checked against its window's single build: size and stats equal, the
k = 1 and k = 16 nearest neighbours of a sample of the window and its k = 16 normals byte-equal; and the batch align on
batch-built targets byte-equal (stats, correspondences, aligned records) to the loop on single-built targets.  Every mode
reads the same host memory: the B target windows and the B source windows are each laid end to end in one array before
anything is timed, the batch calls take those arrays, and the single calls take views of them, so no timed run copies or
allocates a cloud on the host.  Each timed call ends in the library's stream synchronisation, so a host clock around it times the device work (best of --reps after
a warm-up of the same shape).  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_icp_batch import GATE, MAX_ITERS, card, timed  # noqa: E402
from bench_icp_pairs import make_chain, run_loop  # noqa: E402


def single_builds(P, ctx, wins):
    idx = [P.Index(ctx, w) for w in wins]
    ctx.synchronize()
    return idx


def batch_build(ctx, all_tg, off):
    idx = ctx.index_build_batch(all_tg, off)
    ctx.synchronize()
    return idx


def run_batch(b, idx, nrm, all_src, off, outputs=False):
    """bench_icp_pairs.run_batch on sources already laid end to end"""
    B = len(idx)
    b.set_target_batch(idx, normals=nrm)
    b.set_source_batch(all_src, off)
    st = b.iterate_batch()
    if not outputs:
        return st
    corr, cloud = b.get_correspondences_batch(), b.get_cloud()
    return [(st[p], corr[p], cloud[off[p]:off[p + 1]]) for p in range(B)]


def normals(ctx, idx, wins):
    nrm = [i.normals_knn(w, 16)[0] for i, w in zip(idx, wins)]
    ctx.synchronize()
    return nrm


def close(idx):
    for i in idx:
        i.close()


def check_handles(bidx, sidx, wins, seed):
    r = np.random.default_rng(seed)
    for b, s, w in zip(bidx, sidx, wins):
        assert b.size == s.size and b.stats == s.stats
        q = np.ascontiguousarray(w[r.choice(len(w), min(len(w), 2000), replace=False)])
        for k in (1, 16):
            for x, y in zip(b.knn(q, k)[:2], s.knn(q, k)[:2]):
                assert x.tobytes() == y.tobytes()
        assert b.normals_knn(w, 16)[0].tobytes() == s.normals_knn(w, 16)[0].tobytes()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_index_batch.jsonl"))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="8192,32768,131072")
    ap.add_argument("--batches", default="1,8,64,256")
    args = ap.parse_args()
    import pcl_b200 as P
    P.lib()
    name, power, clock = card()
    ctx = P.Context(0)
    params = P.default_params(estimator=1, max_iterations=MAX_ITERS, max_correspondence_distance=GATE,
                              transformation_epsilon=1e-8)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "a") as f:
        for n in [int(x) for x in args.sizes.split(",")]:
            for B in [int(x) for x in args.batches.split(",")]:
                wins = make_chain(B, n, 300 + B + n)
                off = np.arange(B + 1, dtype=np.int64) * n
                # every window once in host memory: the batch reads the two arrays, the loop views of them
                all_tg, all_src = np.concatenate(wins[:B]), np.concatenate(wins[1:B + 1])
                tg = [all_tg[off[k]:off[k + 1]] for k in range(B)]
                chain = tg[:1] + [all_src[off[k]:off[k + 1]] for k in range(B)]  # run_loop aligns chain[p + 1] to tg[p]
                # warm-up of every shape, and the outputs checked byte-equal before any timing
                sidx, bidx = single_builds(P, ctx, tg), batch_build(ctx, all_tg, off)
                check_handles(bidx, sidx, tg, n + B)
                snrm, bnrm = normals(ctx, sidx, tg), normals(ctx, bidx, tg)
                s, bs = P.Icp(ctx, params), P.Icp(ctx, params)
                ref = run_loop(s, sidx, snrm, chain, B, True)
                got = run_batch(bs, bidx, bnrm, all_src, off, True)
                for (sa, ca, xa), (sb, cb, xb) in zip(ref, got):
                    for k in sa:
                        va, vb = sa[k], sb[k]
                        assert (va.tobytes() == vb.tobytes()) if isinstance(va, np.ndarray) else (va == vb or va != va)
                    assert ca.tobytes() == cb.tobytes() and xa.tobytes() == xb.tobytes()
                close(sidx + bidx)

                t_loop, _ = timed(lambda: close(single_builds(P, ctx, tg)), args.reps)
                t_batch, _ = timed(lambda: close(batch_build(ctx, all_tg, off)), args.reps)
                bidx = batch_build(ctx, all_tg, off)
                t_normals, _ = timed(lambda: normals(ctx, bidx, tg), args.reps)
                close(bidx)

                def pairs_loop():
                    idx = single_builds(P, ctx, tg)
                    run_loop(s, idx, normals(ctx, idx, tg), chain, B)
                    close(idx)

                def pairs_batch():
                    idx = batch_build(ctx, all_tg, off)
                    run_batch(bs, idx, normals(ctx, idx, tg), all_src, off)
                    close(idx)

                t_pl, _ = timed(pairs_loop, args.reps)
                t_pb, _ = timed(pairs_batch, args.reps)
                s.close()
                bs.close()
                row = dict(tool="bench_index_batch", gpu=name, power_limit=power, max_sm_clock=clock, n=n, B=B,
                           outputs_byte_equal=True,
                           build_loop_s=round(t_loop, 6), build_batch_s=round(t_batch, 6),
                           build_loop_clouds_per_s=round(B / t_loop, 2), build_batch_clouds_per_s=round(B / t_batch, 2),
                           build_batch_over_loop=round(t_loop / t_batch, 3),
                           normals_s=round(t_normals, 6),
                           pairs_loop_with_builds_s=round(t_pl, 6), pairs_batch_with_builds_s=round(t_pb, 6),
                           pairs_loop_with_builds_per_s=round(B / t_pl, 2),
                           pairs_batch_with_builds_per_s=round(B / t_pb, 2),
                           pairs_batch_over_loop=round(t_pl / t_pb, 3))
                print(json.dumps(row), flush=True)
                f.write(json.dumps(row) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
