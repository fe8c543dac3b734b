"""Cost of the rejector chain on a sharded source: the `icp_reject` stage per iteration (CUDA events, pclb200 profiling)
with the four-rejector chain (median 3.0, one-to-one, trimmed 0.9 / 100, distance 0.2) on a ~2 M-point source, for two
processes SHARING ONE GPU (comm_export / _import over gloo) against one process on the whole cloud.  Two processes on one
device take turns on it, so this measures the exchange latency and the kernels' cost, not multi-GPU scaling.

usage: python -m torch.distributed.run --nproc-per-node=2 tools/sharded_reject_times.py [out.jsonl]"""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import _sharded as S  # noqa: E402
import pcl_b200 as P  # noqa: E402

CHAIN4 = [(P.REJ_MEDIAN, 3.0, 0), (P.REJ_ONE_TO_ONE, 0.0, 0), (P.REJ_TRIMMED, 0.9, 100), (P.REJ_DISTANCE, 0.2, 0)]
N = 2_000_000
ITERS = 10


def cloud():
    rng = np.random.default_rng(7)
    tgt = rng.random((N, 3), dtype=np.float32) * np.float32(4)
    tgt[:, 2] = 0.3 * np.sin(tgt[:, 0]) * np.cos(tgt[:, 1])
    a = np.deg2rad(2.0)
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    src = (tgt.astype(np.float64) @ R.T + [0.01, -0.01, 0.004] + rng.normal(0, 0.002, (N, 3))).astype(np.float32)
    src[: N // 50] += np.float32(0.3)
    return P.xyz1(tgt), P.xyz1(src)


def reject_ms(ctx, idx, src):
    s = P.Icp(ctx, max_iterations=ITERS, transformation_epsilon=0.0, mse_threshold_absolute=0.0)
    s.set_rejectors(CHAIN4)
    s.set_target(idx)
    s.set_source(src)
    s.iterate(1)  # first iteration: one-time table set-up and offsets
    ctx.synchronize()
    ctx.profile(True)
    ctx.profile_reset()
    st = s.iterate()
    ms, n = ctx.profile_get("icp_reject")
    ctx.profile(False)
    s.close()
    return ms / max(n, 1), n, st


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else None
    me = S.join(nccl=False, device=0)
    rank, world, ctx = me.rank, me.world, me.ctx
    tgt, src = cloud()
    idx = P.Index(ctx, tgt)
    lo, hi = rank * N // world, (rank + 1) * N // world
    ms, n, st = reject_ms(ctx, idx, np.ascontiguousarray(src[lo:hi]))
    got = S.gathered((ms, n))
    dist.barrier()
    if rank == 0:
        single = me.ref
        ms1, n1, st1 = reject_ms(single, P.Index(single, tgt), src)
        props = torch.cuda.get_device_properties(0)
        power = os.popen("nvidia-smi --query-gpu=power.limit --format=csv,noheader -i 0").read().strip()
        rec = dict(card=props.name, power_limit=power, setup="two processes sharing one GPU (comm_export / _import)",
                   points=N, chain="median 3.0, one-to-one, trimmed 0.9/100, distance 0.2", iterations_timed=n,
                   icp_reject_ms_per_iter_by_rank=[g[0] for g in got], icp_reject_ms_per_iter_one_process=ms1,
                   correspondences_sharded=st["n_correspondences"], correspondences_one_process=st1["n_correspondences"])
        line = json.dumps(rec)
        print(line)
        if out:
            with open(out, "a") as f:
                f.write(line + "\n")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
