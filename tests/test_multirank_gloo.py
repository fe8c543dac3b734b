"""World-size-2 checks of the N>1 path's host-side logic on CPU (gloo).

What the multi-GPU design relies on (SURVEY.md §8e, pcl_b200/csrc/comm.cu + icp.cu): every rank accumulates the
origin-shifted fp64 sums of ITS source shard, the 40 doubles are all-reduced (sum), and every rank then solves the
identical 3x3 / 6x6 system.  These tests run that algebra over a real torch.distributed all_reduce and compare with
the oracle's single-process estimator on the whole cloud, and exercise the unique-id broadcast plumbing bench.py uses."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import _sharded as S


def _svd_accumulators(p, q, o):
    """icp.cu accumulator layout: [0] n, [1] sum d2, [2:5] sum(p-o), [5:8] sum(q-o), [8:17] sum (q-o)(p-o)^T."""
    a = np.zeros(40)
    pp, qq = p.astype(np.float64) - o, q.astype(np.float64) - o
    a[0] = len(p)
    a[1] = float(((p.astype(np.float32) - q.astype(np.float32)) ** 2).sum())
    a[2:5] = pp.sum(0)
    a[5:8] = qq.sum(0)
    a[8:17] = (qq.T @ pp).ravel()
    return a


def _solve_svd(a, o):
    """k_solve, Umeyama branch."""
    n = a[0]
    mp_, mq = a[2:5] / n, a[5:8] / n
    sig = a[8:17].reshape(3, 3) / n - np.outer(mq, mp_)
    U, s, Vt = np.linalg.svd(sig)
    S = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2, 2] = -1
    R = U @ S @ Vt
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = (mq + o) - R @ (mp_ + o)
    return T


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import bench
    # 1. unique-id plumbing: rank 0's 128 bytes reach every rank unchanged
    uid = [bytes(range(128)) if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    assert uid[0] == bytes(range(128))
    # 2. shards are rank-specific but deterministic (bench.make_source(n, rank))
    s_a, s_b = bench.make_source(2000, rank), bench.make_source(2000, rank)
    assert np.array_equal(s_a, s_b)
    other = bench.make_source(2000, 1 - rank)
    assert not np.array_equal(s_a, other)
    # 3. sharded accumulation + all-reduce == whole-cloud estimate
    rng = np.random.default_rng(123)
    n = 5000
    tgt = rng.random((n, 3)).astype(np.float32) * 4
    ang = 0.05
    R = np.array([[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1]])
    src = ((tgt.astype(np.float64) - 0.01) @ R).astype(np.float32)
    o = 0.5 * (tgt.min(0) + tgt.max(0)).astype(np.float64)
    lo, hi = rank * n // world, (rank + 1) * n // world
    acc = torch.from_numpy(_svd_accumulators(src[lo:hi], tgt[lo:hi], o))
    dist.all_reduce(acc, op=dist.ReduceOp.SUM)
    T = _solve_svd(acc.numpy(), o)
    gathered = [None] * world
    dist.all_gather_object(gathered, T.tobytes())
    assert all(g == gathered[0] for g in gathered), "ranks disagree on the transform"
    if rank == 0:
        q.put((T, src, tgt, float(acc[0])))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_accumulators_match_whole_cloud(orc):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = S.free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    T, src, tgt, n = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert n == 5000
    To = orc.estimate_svd(orc.to_xyz1(src), orc.to_xyz1(tgt), scalar_is_double=True)
    assert np.linalg.norm(T - To) < 1e-10, np.linalg.norm(T - To)


@pytest.mark.gpu
def test_two_gpu_icp_matches_single_gpu():
    """Needs 2 GPUs: the sharded ICP (NCCL all-reduce per iteration) reaches the single-GPU transform."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (VISIBLE SKIP: the same product path runs on one GPU in test_two_ranks_share_one_gpu)")
    r = S.torchrun("_two_gpu_icp.py", 2, timeout=600)
    assert r.returncode == 0 and "TWO_GPU_OK" in r.stdout


@pytest.mark.gpu
def test_two_ranks_share_one_gpu():
    """The N > 1 product path on ANY box with one GPU: two processes on cuda:0, the peer exchange bootstrapped over gloo
    (pclb200_comm_export / _import), 40 accumulators per iteration crossing between the processes inside the iteration
    kernel.  Sharded == whole-cloud result; reciprocal + communicator is refused (tests/_two_rank_one_gpu.py)."""
    r = S.torchrun("_two_rank_one_gpu.py", 2, timeout=600)
    assert r.returncode == 0 and "TWO_RANK_ONE_GPU_OK" in r.stdout
