"""VoxelGrid throughput on one GPU: one pclb200_voxelgrid_batch call over B raw clouds against a loop of B pclb200_voxelgrid
calls, and what that does to point-to-plane scan pairs from raw scans to aligned pairs.

    python tools/bench_voxel_batch.py [--out profiles/h100_voxel_batch.jsonl] [--reps 3] [--sizes ...] [--batches ...]

The clouds are the raw windows of the odometry chain of bench_icp_pairs.py (make_chain): B + 1 windows of n records, pair
k aligning window k + 1 to window k.  Grid: n in {32 k, 128 k, 512 k} x B in {1, 8, 64, 256}.  The leaf is chosen per n
on window 0 so that VoxelGrid keeps about a quarter of the records, and every row records it.  Each row reports
  * voxel: the loop of B voxelgrid calls and the one batch call over the B target windows, seconds and clouds/s;
  * pairs: raw-to-aligned point-to-plane pairs/s (both windows of every pair down-sampled, the targets indexed, their
    k = 16 normals estimated, the pairs aligned), for three pipelines:
      batch voxel + batch build + batch normals + batch align,
      a loop of voxelgrid + batch build + batch normals + batch align (the best pipeline without the batch VoxelGrid),
      a loop of single voxelgrid, builds, normals and aligns.
Before anything is timed, every window's batch rows are checked byte-equal to its own voxelgrid, and the all-batch
pipeline's stats, correspondences and aligned records byte-equal to the all-single loop's.  Every mode reads the same
host memory: the B target windows and the B source windows are each laid end to end in one array before anything is
timed; batch calls take those arrays and single calls views of them.  The down-sampled rows go to host arrays allocated and
touched before anything is timed; the loop packs each window's rows right after the previous window's, as a caller
feeding index_build_batch would.  Each timed call ends in the library's stream synchronisation, so a host clock around it
times the device work (best of --reps after a warm-up of the same shape).  The card's name and power limit are read in the
same run."""
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
from bench_normals_batch import same_stats  # noqa: E402

K = 16
KEEP = 0.25


def pick_leaf(ctx, w):
    """a cubic leaf that keeps about KEEP of the window's records (bisection on the log of the leaf)"""
    lo, hi = 1e-3, 3.0
    for _ in range(24):
        mid = float(np.sqrt(lo * hi))
        if len(ctx.voxelgrid(w, mid)) > KEEP * len(w):
            lo = mid
        else:
            hi = mid
    return float(np.float32(hi))


def loop_voxel(ctx, wins, leaf, out):
    """one voxelgrid per window, each window's rows packed after the previous window's in `out`; (rows, offsets)"""
    off = [0]
    for w in wins:
        off.append(off[-1] + len(ctx.voxelgrid(w, leaf, out=out[off[-1]:off[-1] + len(w)])))
    ctx.synchronize()
    return out[:off[-1]], np.array(off, np.int64)


def batch_voxel(ctx, all_w, off, leaf, out):
    rows, oo = ctx.voxelgrid_batch(all_w, off, leaf, out=out)
    ctx.synchronize()
    return rows, oo


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_voxel_batch.jsonl"))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="32768,131072,524288")
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
            leaf = None
            for B in [int(x) for x in args.batches.split(",")]:
                wins = make_chain(B, n, 300 + B + n)
                if leaf is None:
                    leaf = pick_leaf(ctx, wins[0])
                off = np.arange(B + 1, dtype=np.int64) * n
                # every window once in host memory: the batch reads the two arrays, the loop views of them
                all_tg, all_src = np.concatenate(wins[:B]), np.concatenate(wins[1:B + 1])
                tg = [all_tg[off[k]:off[k + 1]] for k in range(B)]
                src = [all_src[off[k]:off[k + 1]] for k in range(B)]
                del wins
                # the rows of every mode go to host arrays allocated and touched once (first-touch page faults would
                # otherwise be timed as device work)
                outs = {k: np.zeros((B * n, 4), np.float32) for k in ("lt", "ls", "bt", "bs")}
                nout = np.zeros((B * n, 4), np.float32)
                # warm-up of every shape, and the outputs checked byte-equal before any timing
                lrows, loff = loop_voxel(ctx, tg, leaf, outs["lt"])
                brows, boff = batch_voxel(ctx, all_tg, off, leaf, outs["bt"])
                assert np.array_equal(loff, boff) and lrows.tobytes() == brows.tobytes()
                kept = float(boff[-1]) / (B * n)
                srows, soff = batch_voxel(ctx, all_src, off, leaf, outs["bs"])
                trows_s = [lrows[loff[p]:loff[p + 1]] for p in range(B)]
                chain = trows_s[:1] + [srows[soff[p]:soff[p + 1]] for p in range(B)]
                sidx = single_builds(P, ctx, trows_s)
                snrm = [i.normals_knn(w, K)[0] for i, w in zip(sidx, trows_s)]
                bidx = batch_build(ctx, brows, boff)
                bn, _ = ctx.normals_knn_batch(bidx, brows, boff, K, out=nout)
                bnrm = [bn[boff[p]:boff[p + 1]] for p in range(B)]
                s, bs = P.Icp(ctx, params), P.Icp(ctx, params)
                ref = run_loop(s, sidx, snrm, chain, B, True)
                got = run_batch(bs, bidx, bnrm, srows, soff, True)
                for (sa, ca, xa), (sb, cb, xb) in zip(ref, got):
                    assert same_stats(sa, sb) and ca.tobytes() == cb.tobytes() and xa.tobytes() == xb.tobytes()
                close(sidx)
                close(bidx)

                t_loop, _ = timed(lambda: loop_voxel(ctx, tg, leaf, outs["lt"]), args.reps)
                t_batch, _ = timed(lambda: batch_voxel(ctx, all_tg, off, leaf, outs["bt"]), args.reps)

                def align_batch(trows, toff, srows, soff):
                    idx = batch_build(ctx, trows, toff)
                    nrm, _ = ctx.normals_knn_batch(idx, trows, toff, K, out=nout)
                    run_batch(bs, idx, [nrm[toff[p]:toff[p + 1]] for p in range(B)], srows, soff)
                    close(idx)

                def pairs_all_batch():
                    align_batch(*batch_voxel(ctx, all_tg, off, leaf, outs["bt"]),
                                *batch_voxel(ctx, all_src, off, leaf, outs["bs"]))

                def pairs_loop_voxel():
                    align_batch(*loop_voxel(ctx, tg, leaf, outs["lt"]), *loop_voxel(ctx, src, leaf, outs["ls"]))

                def pairs_all_single():
                    trows, toff = loop_voxel(ctx, tg, leaf, outs["lt"])
                    srows, soff = loop_voxel(ctx, src, leaf, outs["ls"])
                    ts = [trows[toff[p]:toff[p + 1]] for p in range(B)]
                    idx = single_builds(P, ctx, ts)
                    nrm = [i.normals_knn(w, K)[0] for i, w in zip(idx, ts)]
                    run_loop(s, idx, nrm, ts[:1] + [srows[soff[p]:soff[p + 1]] for p in range(B)], B)
                    close(idx)

                t_ab, _ = timed(pairs_all_batch, args.reps)
                t_lv, _ = timed(pairs_loop_voxel, args.reps)
                t_as, _ = timed(pairs_all_single, args.reps)
                s.close()
                bs.close()
                row = dict(tool="bench_voxel_batch", gpu=name, power_limit=power, max_sm_clock=clock, n=n, B=B,
                           leaf=leaf, kept_fraction=round(kept, 4), k=K, outputs_byte_equal=True,
                           voxel_loop_s=round(t_loop, 6), voxel_batch_s=round(t_batch, 6),
                           voxel_loop_clouds_per_s=round(B / t_loop, 2),
                           voxel_batch_clouds_per_s=round(B / t_batch, 2),
                           voxel_batch_over_loop=round(t_loop / t_batch, 3),
                           pairs_all_batch_s=round(t_ab, 6), pairs_loop_voxel_s=round(t_lv, 6),
                           pairs_all_single_s=round(t_as, 6),
                           pairs_all_batch_per_s=round(B / t_ab, 2), pairs_loop_voxel_per_s=round(B / t_lv, 2),
                           pairs_all_single_per_s=round(B / t_as, 2),
                           pairs_all_batch_over_loop_voxel=round(t_lv / t_ab, 3))
                print(json.dumps(row), flush=True)
                f.write(json.dumps(row) + "\n")
                del outs, nout, all_tg, all_src, tg, src
    ctx.close()


if __name__ == "__main__":
    main()
