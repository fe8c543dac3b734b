"""Fitness score throughput on one GPU: one pclb200_fitness_score_batch call (and the session form,
pclb200_icp_fitness_score_batch) over B aligned scan pairs against a loop of B pclb200_fitness_score calls, and what that
does to point-to-plane pairs aligned and scored.

    python tools/bench_fitness_batch.py [--out profiles/h100_fitness_batch.jsonl] [--reps 3]

The pairs are those of bench_icp_pairs.py's odometry chain (make_chain): B + 1 windows of n points, pair k aligning window
k + 1 to window k.  Grid: n in {8 k, 32 k, 128 k} x B in {1, 8, 64, 256}.  The targets are built as one batch and their
normals estimated as one batch, once, outside every timed region.  Each row reports
  * scores: the loop of B fitness_score calls, the free batch call and the session form, each scoring every pair under
    its final transformation from one batch align; seconds and pairs scored per second;
  * pairs: point-to-plane pairs aligned and scored per second, batch align + session score against batch align + a loop
    of fitness_score.
Before anything is timed, the free batch scores and the session's scores are checked byte-equal to the loop's.  Every
mode reads the same host memory: the B source windows are laid end to end in one array, which the batch calls take and
the loop takes views of.  Each timed call ends in the library's stream synchronisation, so a host clock around it times
the device work (best of --reps after a warm-up of the same shape).  The card's name and power limit are read in the same
run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_icp_batch import GATE, MAX_ITERS, card, timed  # noqa: E402
from bench_icp_pairs import make_chain  # noqa: E402
from bench_index_batch import batch_build, close, run_batch  # noqa: E402


def loop_scores(ctx, idx, src, finals):
    out = np.array([i.fitness_score(s, T) for i, s, T in zip(idx, src, finals)])
    ctx.synchronize()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_fitness_batch.jsonl"))
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
                wins = make_chain(B, n, 500 + B + n)
                off = np.arange(B + 1, dtype=np.int64) * n
                all_tg, all_src = np.concatenate(wins[:B]), np.concatenate(wins[1:B + 1])
                src = [all_src[off[k]:off[k + 1]] for k in range(B)]
                idx = batch_build(ctx, all_tg, off)
                bn, _ = ctx.normals_knn_batch(idx, all_tg, off, 16)
                nrm = [bn[off[p]:off[p + 1]] for p in range(B)]
                bs = P.Icp(ctx, params)
                st = run_batch(bs, idx, nrm, all_src, off)
                finals = np.array([x["final"] for x in st])
                # warm-up of every shape, and the scores checked byte-equal before any timing
                ref = loop_scores(ctx, idx, src, finals)
                got = ctx.fitness_score_batch(idx, all_src, off, finals)
                ses = bs.fitness_score_batch()
                assert got.tobytes() == ref.tobytes() and ses.tobytes() == ref.tobytes()

                t_loop, _ = timed(lambda: loop_scores(ctx, idx, src, finals), args.reps)
                t_batch, _ = timed(lambda: ctx.fitness_score_batch(idx, all_src, off, finals), args.reps)
                t_session, _ = timed(bs.fitness_score_batch, args.reps)

                def pairs_batch_score():
                    run_batch(bs, idx, nrm, all_src, off)
                    return bs.fitness_score_batch()

                def pairs_loop_score():
                    s = run_batch(bs, idx, nrm, all_src, off)
                    return loop_scores(ctx, idx, src, [x["final"] for x in s])

                t_pb, _ = timed(pairs_batch_score, args.reps)
                t_pl, _ = timed(pairs_loop_score, args.reps)
                bs.close()
                close(idx)
                row = dict(tool="bench_fitness_batch", gpu=name, power_limit=power, max_sm_clock=clock, n=n, B=B,
                           scores_byte_equal=True,
                           score_loop_s=round(t_loop, 6), score_batch_s=round(t_batch, 6),
                           score_session_s=round(t_session, 6),
                           score_loop_per_s=round(B / t_loop, 2), score_batch_per_s=round(B / t_batch, 2),
                           score_session_per_s=round(B / t_session, 2),
                           score_batch_over_loop=round(t_loop / t_batch, 3),
                           score_session_over_loop=round(t_loop / t_session, 3),
                           pairs_batch_score_s=round(t_pb, 6), pairs_loop_score_s=round(t_pl, 6),
                           pairs_batch_score_per_s=round(B / t_pb, 2), pairs_loop_score_per_s=round(B / t_pl, 2),
                           pairs_batch_over_loop=round(t_pl / t_pb, 3))
                print(json.dumps(row), flush=True)
                f.write(json.dumps(row) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
