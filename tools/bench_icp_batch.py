"""Small-scan ICP throughput on one GPU: a batch session (include/pclb200_batch.h) against a loop of single sessions on
one context and against two contexts in flight (two host threads, half the scans each).  Every mode holds one session
per context whose target (index and normals) is set once, as a program that calls setInputTarget once and align() per
scan does.

    python tools/bench_icp_batch.py [--out profiles/h100_icp_batch.jsonl] [--reps 2]

The map is a cfg3-style Gaussian surface of 2 M points (bench.py's generator) with k = 16 normals from the library;
the scans are re-samples of 3 x 3 windows of the same surface, each moved by its own small rigid motion.  Grid:
B in {1, 8, 64, 256} scans x n in {8 k, 32 k, 128 k} points x {point-to-plane, SVD}.  Before anything is timed, every
scan's stats (final transform included), last correspondences and aligned cloud from the batch are checked byte-equal to
its single session's.  A timed run is set_source + iterate per scan (the batch: one set_source_batch + iterate_batch) on
the prepared sessions; each call ends in the library's stream synchronisation, so a host clock around the run times the
device work (best of --reps after a warm-up of the same shape).  The card's name and power limit are read in the same
run.  One JSON line per (estimator, n,
B) with aligns/s and correspondences/s of each mode, and the batch's ratio to the other two."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_MAP = 2_000_000
GATE = 0.3
MAX_ITERS = 30


def surface_xy(xy, r):
    return 0.5 * np.sin(xy[:, 0]) * np.cos(0.7 * xy[:, 1]) + r.normal(0.0, 0.002, len(xy))


def make_map():
    r = np.random.default_rng(7)
    xy = r.random((N_MAP, 2)) * 10.0
    t = np.zeros((N_MAP, 4), np.float32)
    t[:, 0:2], t[:, 2], t[:, 3] = xy, surface_xy(xy, r), 1.0
    return t


def make_scans(B, n, seed):
    r = np.random.default_rng(seed)
    out = np.zeros((B * n, 4), np.float32)
    for p in range(B):
        lo = r.uniform(1.0, 6.0, 2)
        xy = lo + r.random((n, 2)) * 3.0
        z = surface_xy(xy, r)
        a = np.deg2rad(r.uniform(-1.5, 1.5))
        c, s = np.cos(a), np.sin(a)
        cx, cy = lo + 1.5
        x0, y0 = xy[:, 0] - cx, xy[:, 1] - cy
        rec = out[p * n:(p + 1) * n]
        rec[:, 0] = c * x0 - s * y0 + cx + r.uniform(-0.03, 0.03)
        rec[:, 1] = s * x0 + c * y0 + cy + r.uniform(-0.03, 0.03)
        rec[:, 2] = z + r.uniform(-0.02, 0.02)
        rec[:, 3] = 1.0
    return out


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                     "--format=csv,noheader"], text=True).strip().splitlines()[0]
        return [x.strip() for x in q.split(",")]
    except Exception as e:  # the numbers still carry the device name torch reports
        return [str(e), "unknown", "unknown"]


def session(P, ctx, params, idx, tnrm):
    s = P.Icp(ctx, params)
    s.set_target(idx, normals=tnrm)
    return s


def run_single(s, src, outputs=False):
    s.set_source(src)
    st = s.iterate()
    return (st, s.get_correspondences(), s.get_cloud()) if outputs else st


def run_loop(s, scans, n, B, outputs=False):
    return [run_single(s, scans[p * n:(p + 1) * n], outputs) for p in range(B)]


def run_batch(b, scans, n, B, outputs=False):
    off = np.arange(B + 1, dtype=np.int64) * n
    b.set_source_batch(scans, off)
    st = b.iterate_batch()
    if not outputs:
        return st
    corr, cloud = b.get_correspondences_batch(), b.get_cloud()
    return [(st[p], corr[p], cloud[off[p]:off[p + 1]]) for p in range(B)]


def run_two(ss, scans, n, B, outputs=False):
    res = [None, None]

    def work(k):
        ps = range(k, B, 2)
        res[k] = [(p, run_single(ss[k], scans[p * n:(p + 1) * n], outputs)) for p in ps]

    th = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    return [st for _, st in sorted(res[0] + res[1], key=lambda x: x[0])]


def timed(fn, reps):
    best = None
    out = None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_icp_batch.jsonl"))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="8192,32768,131072")
    ap.add_argument("--batches", default="1,8,64,256")
    ap.add_argument("--estimators", default="point_to_plane,svd")
    args = ap.parse_args()
    import pcl_b200 as P
    P.lib()
    name, power, clock = card()
    tgt = make_map()
    ctxs = [P.Context(0), P.Context(0)]
    idxs = [P.Index(c, tgt) for c in ctxs]
    tnrm, _ = idxs[0].normals_knn(tgt, 16)
    tnrms = [tnrm, tnrm]
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "a") as f:
        for est_name in args.estimators.split(","):
            est = {"point_to_plane": 1, "svd": 0}[est_name]
            params = P.default_params(estimator=est, max_iterations=MAX_ITERS, max_correspondence_distance=GATE,
                                      transformation_epsilon=1e-8)
            tn = tnrm if est == 1 else None
            ss = [session(P, c, params, i, tn) for c, i in zip(ctxs, idxs)]  # the target is set once per context
            bs = session(P, ctxs[0], params, idxs[0], tn)
            for n in [int(x) for x in args.sizes.split(",")]:
                for B in [int(x) for x in args.batches.split(",")]:
                    scans = make_scans(B, n, 100 + B + n)
                    # warm-up of every shape, and the outputs checked byte-equal before any timing
                    ref = run_loop(ss[0], scans, n, B, True)
                    got = run_batch(bs, scans, n, B, True)
                    two = run_two(ss, scans, n, B, True)
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
                    t_loop, _ = timed(lambda: run_loop(ss[0], scans, n, B), args.reps)
                    t_batch, _ = timed(lambda: run_batch(bs, scans, n, B), args.reps)
                    t_two, _ = timed(lambda: run_two(ss, scans, n, B), args.reps)
                    row = dict(tool="bench_icp_batch", gpu=name, power_limit=power, max_sm_clock=clock,
                               estimator=est_name, n=n, B=B, iterations_total=iters, correspondences_total=corr,
                               outputs_byte_equal=True)
                    for mode, t in (("batch", t_batch), ("loop", t_loop), ("two_contexts", t_two)):
                        row[mode + "_s"] = round(t, 6)
                        row[mode + "_aligns_per_s"] = round(B / t, 2)
                        row[mode + "_corr_per_s"] = round(corr / t, 1)
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
