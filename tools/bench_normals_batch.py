"""k-NN normals throughput on one GPU: one pclb200_normals_knn_batch call over B indexed clouds against a loop of B
pclb200_normals_knn calls, and what that does to point-to-plane scan pairs with their builds and normals counted.

    python tools/bench_normals_batch.py [--out profiles/h100_normals_batch.jsonl] [--reps 3]

The clouds are the target windows of the odometry chain of bench_icp_pairs.py (make_chain): B + 1 windows of n points,
pair k aligning window k + 1 to window k.  Grid: n in {8 k, 32 k, 128 k} x B in {1, 8, 64, 256}, k = 16.  Each row reports
  * normals: the loop of B normals_knn calls and the one batch call on the same batch-built handles, seconds and clouds/s;
  * pairs: point-to-plane pairs/s with the builds and normals counted, for three pipelines:
      batch build + batch normals + batch align,
      batch build + a loop of normals + batch align (the best pipeline without the batch normals),
      a loop of single builds, single normals and single aligns.
Before anything is timed, every window's batch normals are checked byte-equal (rows and is_dense) to its own normals_knn,
and the all-batch pipeline's stats, correspondences and aligned records byte-equal to the all-single loop's.  Every mode
reads the same host memory: the B target windows and the B source windows are each laid end to end in one array before
anything is timed; batch calls take those arrays and single calls views of them.  The normals go to one host array per
mode, allocated and touched before anything is timed, which the batch call fills whole and the loop view by view.  Each
timed call ends in the library's stream synchronisation, so a host clock around it times the device work (best of --reps
after a warm-up of the same shape).  The card's name and power limit are read in the same run."""
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
from bench_index_batch import batch_build, close, run_batch, single_builds  # noqa: E402

K = 16


def loop_normals(ctx, idx, wins, out, off):
    """one normals_knn per window, each into its view of `out`"""
    for p, (i, w) in enumerate(zip(idx, wins)):
        i.normals_knn(w, K, out=out[off[p]:off[p + 1]])
    ctx.synchronize()
    return [out[off[p]:off[p + 1]] for p in range(len(idx))]


def batch_normals(ctx, idx, all_tg, out, off):
    _, dense = ctx.normals_knn_batch(idx, all_tg, off, K, out=out)
    ctx.synchronize()
    return [out[off[p]:off[p + 1]] for p in range(len(idx))], dense


def same_stats(a, b):
    for k in a:
        va, vb = a[k], b[k]
        if not ((va.tobytes() == vb.tobytes()) if isinstance(va, np.ndarray) else (va == vb or va != va)):
            return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_normals_batch.jsonl"))
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
                # the normals of every mode go to one host array, allocated and touched once: a fresh array per call
                # would time the host's page faults on its first touch (a 128 MB array at 128 k, B = 64)
                lout, bout = np.zeros((B * n, 4), np.float32), np.zeros((B * n, 4), np.float32)
                # warm-up of every shape, and the outputs checked byte-equal before any timing
                sidx, bidx = single_builds(P, ctx, tg), batch_build(ctx, all_tg, off)
                snrm = loop_normals(ctx, sidx, tg, lout, off)
                bnrm, dense = batch_normals(ctx, bidx, all_tg, bout, off)
                for p in range(B):
                    ref, d = bidx[p].normals_knn(tg[p], K)
                    assert bnrm[p].tobytes() == ref.tobytes() and bool(dense[p]) == d, p
                s, bs = P.Icp(ctx, params), P.Icp(ctx, params)
                ref = run_loop(s, sidx, snrm, chain, B, True)
                got = run_batch(bs, bidx, bnrm, all_src, off, True)
                for (sa, ca, xa), (sb, cb, xb) in zip(ref, got):
                    assert same_stats(sa, sb) and ca.tobytes() == cb.tobytes() and xa.tobytes() == xb.tobytes()
                close(sidx)

                t_loop, _ = timed(lambda: loop_normals(ctx, bidx, tg, lout, off), args.reps)
                t_batch, _ = timed(lambda: batch_normals(ctx, bidx, all_tg, bout, off), args.reps)
                close(bidx)

                def pairs_all_batch():
                    idx = batch_build(ctx, all_tg, off)
                    run_batch(bs, idx, batch_normals(ctx, idx, all_tg, bout, off)[0], all_src, off)
                    close(idx)

                def pairs_loop_normals():
                    idx = batch_build(ctx, all_tg, off)
                    run_batch(bs, idx, loop_normals(ctx, idx, tg, lout, off), all_src, off)
                    close(idx)

                def pairs_all_single():
                    idx = single_builds(P, ctx, tg)
                    run_loop(s, idx, loop_normals(ctx, idx, tg, lout, off), chain, B)
                    close(idx)

                t_ab, _ = timed(pairs_all_batch, args.reps)
                t_ln, _ = timed(pairs_loop_normals, args.reps)
                t_as, _ = timed(pairs_all_single, args.reps)
                s.close()
                bs.close()
                row = dict(tool="bench_normals_batch", gpu=name, power_limit=power, max_sm_clock=clock, n=n, B=B, k=K,
                           outputs_byte_equal=True,
                           normals_loop_s=round(t_loop, 6), normals_batch_s=round(t_batch, 6),
                           normals_loop_clouds_per_s=round(B / t_loop, 2),
                           normals_batch_clouds_per_s=round(B / t_batch, 2),
                           normals_batch_over_loop=round(t_loop / t_batch, 3),
                           pairs_all_batch_s=round(t_ab, 6), pairs_loop_normals_s=round(t_ln, 6),
                           pairs_all_single_s=round(t_as, 6),
                           pairs_all_batch_per_s=round(B / t_ab, 2), pairs_loop_normals_per_s=round(B / t_ln, 2),
                           pairs_all_single_per_s=round(B / t_as, 2),
                           pairs_all_batch_over_loop_normals=round(t_ln / t_ab, 3))
                print(json.dumps(row), flush=True)
                f.write(json.dumps(row) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
