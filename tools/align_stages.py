#!/usr/bin/env python
"""Where one cfg3 align's time goes, stage by stage: bench.py's value leg (device-resident pcl::PointNormal records,
set_source / iterate / get_cloud through the C-ABI) under torch.profiler with CUDA activities.

    python tools/align_stages.py [--steps K] [--warmup W] [--points N] [--out DIR]

Prints one JSON object: per align, the device time of every kernel (by name), memcpy (by kind) and memset, the time the
device sat idle between them (launch latency and host round trips), the CUDA runtime calls that block the host
(stream / device synchronisations, blocking copies) and the card's name and power limit.  The profiler's trace is written
to DIR/align_stages_trace.json and the object to DIR/align_stages.json.  The timings come from a traced run: take step times from bench.py, not from here."""
import argparse
import collections
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
import pcl_b200 as P  # noqa: E402

# runtime calls that return only once the device has caught up with the host
BLOCKING = ("cudaStreamSynchronize", "cudaDeviceSynchronize", "cudaEventSynchronize", "cudaMemcpy", "cudaMemcpy2D",
            "cudaMemcpyFromSymbol", "cudaMemcpyToSymbol", "cudaMemset")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--points", type=int, default=None)
    ap.add_argument("--out", default=None, help="output directory (default: a new temporary directory)")
    a = ap.parse_args()
    a.out = a.out or tempfile.mkdtemp(prefix="align_stages_")
    W = bench.WORKLOADS["cfg3"]
    n = a.points or W["n"]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ctx = P.Context(0)
    tgt, src = bench.gen_clouds("cfg3", n, 0, False)
    tidx = P.Index(ctx, tgt)
    tgt_dev = torch.from_numpy(tgt).to(dev)
    nrm = torch.empty((tgt.shape[0], 4), dtype=torch.float32, device=dev)
    tidx.normals_knn(tgt_dev, W["normals_k"], viewpoint=(5.0, 5.0, 10.0), out=nrm)
    del tgt_dev
    src_dev = torch.from_numpy(src).to(dev)
    out_dev = torch.empty_like(src_dev)
    params = P.default_params(max_iterations=W["iters"], max_correspondence_distance=W["gate"],
                              estimator=P.EST_POINT_TO_PLANE_LLS, with_normals_transform=1, mse_threshold_absolute=0.0,
                              transformation_epsilon=0.0)
    obj = P.Icp(ctx, params=params)
    obj.set_target(tidx, normals=nrm)

    def align():
        obj.set_source(src_dev, normals=P.Field(src_dev, 4))
        obj.iterate()
        obj.get_cloud(out_dev, normals=P.Field(out_dev, 4))

    for _ in range(a.warmup):
        align()
    torch.cuda.synchronize()
    os.makedirs(a.out, exist_ok=True)
    trace = os.path.join(a.out, "align_stages_trace.json")
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for _ in range(a.steps):
            align()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    ev = json.load(open(trace))["traceEvents"]

    K = float(a.steps)
    gpu = sorted((e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")),
                 key=lambda e: e["ts"])
    per = collections.defaultdict(lambda: [0.0, 0])
    for e in gpu:
        name = e["name"] if e["cat"] == "kernel" else e["cat"] + ":" + e["name"].split(" ")[0]
        per[name][0] += e["dur"]
        per[name][1] += 1
    # idle device time between consecutive activities (one stream: the library issues everything on the ctx stream)
    busy_end, idle = None, 0.0
    for e in gpu:
        if busy_end is not None and e["ts"] > busy_end:
            idle += e["ts"] - busy_end
        busy_end = max(busy_end or 0.0, e["ts"] + e["dur"])
    span = (busy_end - gpu[0]["ts"]) if gpu else 0.0
    runtime = collections.Counter(e["name"] for e in ev if e.get("ph") == "X" and e.get("cat") == "cuda_runtime")
    blocking = {k: v / K for k, v in runtime.items() if k in BLOCKING}
    by_time = sorted(per.items(), key=lambda kv: -kv[1][0])
    iter_kernels = ("k_search", "k_accum", "k_solve")
    outside = sum(v[0] for k, v in per.items() if not any(t in k for t in iter_kernels))
    res = {
        "workload": W["name"], "points": n, "steps": a.steps,
        "device": bench.device_info(0),
        "ms_per_align_span": span / K / 1e3,
        "ms_per_align_device_busy": sum(v[0] for v in per.values()) / K / 1e3,
        "ms_per_align_device_idle": idle / K / 1e3,
        "ms_per_align_outside_iterations": outside / K / 1e3,
        "stages_ms_per_align": {k: round(v[0] / K / 1e3, 4) for k, v in by_time},
        "launches_per_align": {k: v[1] / K for k, v in by_time},
        "blocking_runtime_calls_per_align": blocking,
        "how": ("torch.profiler (CUPTI) over K aligns of bench.py's cfg3 value leg after W warm-up aligns; "
                "idle = device time between consecutive activities of the trace"),
    }
    print(json.dumps(res, indent=1))
    with open(os.path.join(a.out, "align_stages.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
