"""Scan-pair ICP throughput on one GPU: a batch session with one target per pair (pclb200_icp_set_target_batch) against
a loop of single sessions (set_target + set_source + iterate per pair) on one context and against two contexts in
flight (two host threads, half the pairs each).

    python tools/bench_icp_pairs.py [--out profiles/h100_icp_pairs.jsonl] [--reps 3]

The workload is an odometry chain: B + 1 overlapping 3 x 3 windows of the cfg3-style surface of bench_icp_batch.py, each
window a fresh sample of n points moved by its own small rigid motion, the windows 0.3 apart along x in rows of 20.
Pair k aligns window k + 1 to window k, with k = 16 target normals from the library.  Grid: B in {1, 8, 64, 256} pairs x n in
{8 k, 32 k, 128 k} points x {point-to-plane, SVD}.  The B index builds and normal estimations are timed on their own
(build_s) and reported in the same line, since every mode needs them.  Before anything is timed, every pair's stats
(final transform included), last correspondences and aligned cloud are checked byte-equal across the three modes.  A timed
run sets the targets (the batch: one set_target_batch) and the sources and iterates; each call ends in the library's
stream synchronisation, so a host clock around the run times the device work (best of --reps after a warm-up of the same
shape).  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_icp_batch import GATE, MAX_ITERS, card, surface_xy, timed  # noqa: E402


def make_chain(B, n, seed):
    """B + 1 windows (n, 4) along x, each moved by a small rigid motion about its centre"""
    r = np.random.default_rng(seed)
    out = []
    for k in range(B + 1):
        lo = np.array([0.3 * (k % 20), 1.0 + 0.15 * (k // 20 % 20)])
        xy = lo + r.random((n, 2)) * 3.0
        z = surface_xy(xy, r)
        a = np.deg2rad(r.uniform(-1.0, 1.0))
        c, s = np.cos(a), np.sin(a)
        cx, cy = lo + 1.5
        x0, y0 = xy[:, 0] - cx, xy[:, 1] - cy
        rec = np.zeros((n, 4), np.float32)
        rec[:, 0] = c * x0 - s * y0 + cx + r.uniform(-0.02, 0.02)
        rec[:, 1] = s * x0 + c * y0 + cy + r.uniform(-0.02, 0.02)
        rec[:, 2] = z + r.uniform(-0.01, 0.01)
        rec[:, 3] = 1.0
        out.append(rec)
    return out


def build_targets(P, ctx, wins, with_normals):
    """the index (and k = 16 normals) of every target window; synchronised, so a host clock times it"""
    idx = [P.Index(ctx, w) for w in wins]
    nrm = [i.normals_knn(w, 16)[0] for i, w in zip(idx, wins)] if with_normals else [None] * len(wins)
    ctx.synchronize()
    return idx, nrm


def run_single(s, idx, nrm, src, outputs=False):
    s.set_target(idx, normals=nrm)
    s.set_source(src)
    st = s.iterate()
    return (st, s.get_correspondences(), s.get_cloud()) if outputs else st


def run_loop(s, idx, nrm, wins, B, outputs=False):
    return [run_single(s, idx[p], nrm[p], wins[p + 1], outputs) for p in range(B)]


def run_batch(b, idx, nrm, wins, B, n, outputs=False):
    b.set_target_batch(idx[:B], normals=None if nrm[0] is None else nrm[:B])
    off = np.arange(B + 1, dtype=np.int64) * n
    src = np.concatenate(wins[1:B + 1])
    b.set_source_batch(src, off)
    st = b.iterate_batch()
    if not outputs:
        return st
    corr, cloud = b.get_correspondences_batch(), b.get_cloud()
    return [(st[p], corr[p], cloud[off[p]:off[p + 1]]) for p in range(B)]


def run_two(ss, targets, wins, B, outputs=False):
    res = [None, None]

    def work(k):
        idx, nrm = targets[k]
        res[k] = [(p, run_single(ss[k], idx[p], nrm[p], wins[p + 1], outputs)) for p in range(k, B, 2)]

    th = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    return [st for _, st in sorted(res[0] + res[1], key=lambda x: x[0])]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_icp_pairs.jsonl"))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="8192,32768,131072")
    ap.add_argument("--batches", default="1,8,64,256")
    ap.add_argument("--estimators", default="point_to_plane,svd")
    args = ap.parse_args()
    import pcl_b200 as P
    P.lib()
    name, power, clock = card()
    ctxs = [P.Context(0), P.Context(0)]
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "a") as f:
        for n in [int(x) for x in args.sizes.split(",")]:
            for B in [int(x) for x in args.batches.split(",")]:
                wins = make_chain(B, n, 300 + B + n)
                build_targets(P, ctxs[0], wins[:B], True)  # warm-up of the build shapes
                t0 = time.perf_counter()
                targets0 = build_targets(P, ctxs[0], wins[:B], True)
                t_build = time.perf_counter() - t0
                targets = [targets0, build_targets(P, ctxs[1], wins[:B], True)]
                for est_name in args.estimators.split(","):
                    est = {"point_to_plane": 1, "svd": 0}[est_name]
                    params = P.default_params(estimator=est, max_iterations=MAX_ITERS, max_correspondence_distance=GATE,
                                              transformation_epsilon=1e-8)
                    tg = [(i, nr if est == 1 else [None] * B) for i, nr in targets]
                    ss = [P.Icp(c, params) for c in ctxs]
                    bs = P.Icp(ctxs[0], params)
                    # warm-up of every shape, and the outputs checked byte-equal before any timing
                    ref = run_loop(ss[0], *tg[0], wins, B, True)
                    got = run_batch(bs, *tg[0], wins, B, n, True)
                    two = run_two(ss, tg, wins, B, True)
                    for (sa, ca, xa), (sb, cb, xb), (sc, cc, xc) in zip(ref, got, two):
                        for k in sa:
                            va, vb, vc = sa[k], sb[k], sc[k]
                            if isinstance(va, np.ndarray):
                                assert va.tobytes() == vb.tobytes() == vc.tobytes(), (k, va, vb)
                            else:
                                assert va == vb == vc or va != va, (k, va, vb, vc)
                        assert ca.tobytes() == cb.tobytes() == cc.tobytes()
                        assert xa.tobytes() == xb.tobytes() == xc.tobytes()
                    corr = sum(s["total_correspondences"] for s, _, _ in ref)
                    iters = sum(s["iterations"] for s, _, _ in ref)
                    t_loop, _ = timed(lambda: run_loop(ss[0], *tg[0], wins, B), args.reps)
                    t_batch, _ = timed(lambda: run_batch(bs, *tg[0], wins, B, n), args.reps)
                    t_two, _ = timed(lambda: run_two(ss, tg, wins, B), args.reps)
                    row = dict(tool="bench_icp_pairs", gpu=name, power_limit=power, max_sm_clock=clock,
                               estimator=est_name, n=n, B=B, iterations_total=iters, correspondences_total=corr,
                               outputs_byte_equal=True, build_s=round(t_build, 6))
                    for mode, t in (("batch", t_batch), ("loop", t_loop), ("two_contexts", t_two)):
                        row[mode + "_s"] = round(t, 6)
                        row[mode + "_pairs_per_s"] = round(B / t, 2)
                        row[mode + "_with_builds_pairs_per_s"] = round(B / (t + t_build), 2)
                    row["batch_over_loop"] = round(t_loop / t_batch, 3)
                    row["batch_over_two_contexts"] = round(t_two / t_batch, 3)
                    print(json.dumps(row), flush=True)
                    f.write(json.dumps(row) + "\n")
                    for s in ss + [bs]:
                        s.close()
    for c in ctxs:
        c.close()


if __name__ == "__main__":
    main()
