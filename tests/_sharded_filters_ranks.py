"""Helper for tests/test_gpu_sharded_filters.py (launched under torchrun, gloo): k-NN queries, k-NN statistics and the two
outlier filters of a map sharded across ranks (pclb200_knn_sharded, pclb200_knn_stats_sharded,
pclb200_statistical_outlier_sharded, pclb200_radius_outlier_sharded).

Ranks on cuda:0 with the peer exchange bootstrapped over gloo (comm_export / _import), or, with PCLB_SHARDED_NCCL=1, one
GPU per rank with pclb200_comm_init and PCLB200_REDUCE_NCCL.  Two maps (a surface and a volume cloud, both with an
exact-tie lattice, non-finite rows and duplicated points under other ids), four partitions (spatial slabs; a random
partition; slabs whose points near a cut are held by both neighbours under one id; slabs plus a far tile of 2 points).
Queries: each tile's own records (non-finite ones included), and an arbitrary point set through an indices subset.
k-NN rows, k_eff, mean and kth must be byte-equal to one process's pclb200_knn / pclb200_knn_stats on an index of the
whole map; the ROR masks byte-equal (dense and not, negative both ways); the SOR threshold the same on every rank and
within 1e-12 relative of the sequential threshold over one process's means, no query within that band of it, and the
SOR masks byte-equal; both masks equal the CPU oracle's.  Last, the refusals (ERR_INVALID on every rank), after which the
communicator still works."""
import numpy as np
import torch

import _sharded as S
import oracle
import pcl_b200 as P

me = S.join()
rank, world, dev, ctx, ref_ctx = me.rank, me.world, me.device, me.ctx, me.ref

rng = np.random.default_rng(23)
REL = 1e-12


def lattice(origin, n, step):
    g = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float32) * np.float32(step)] * 2, indexing="ij"), -1).reshape(-1, 2)
    return np.c_[g, np.zeros(len(g), np.float32)] + np.asarray(origin, np.float32)


SCENES = [("surface", S.with_extras(rng, np.concatenate([S.surface(rng, 150000), lattice((0.5, 0.5, 1.0), 64, 1 / 32)]))),
          ("volume", S.with_extras(rng, np.concatenate([S.volume(rng, 80000), lattice((0.0, 0.0, 0.3), 32, 1 / 64)])))]

checked = 0
for sname, whole0 in SCENES:
    orc_index = None
    for pname, parts, whole in S.partitions(rng, whole0, world):
        ref_index = P.Index(ref_ctx, whole)
        tile = np.ascontiguousarray(whole[parts[rank]])
        tindex = P.Index(ctx, tile, ids=np.ascontiguousarray(parts[rank], dtype=np.int32))
        q_any, sub = S.arbitrary_queries(rng, whole)
        for k in (2, 16, 51):
            for q in (tile, q_any[sub]):
                got, want = tindex.knn_sharded(q, k), ref_index.knn(q, k)
                assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes(), \
                    (sname, pname, "knn", k, rank)
                assert got[2] == want[2], (sname, pname, "k_eff", k, got[2], want[2])
            for q, ind in ((tile, None), (q_any, sub)):
                got, want = tindex.knn_stats_sharded(q, k, indices=ind), ref_index.knn_stats(q, k, indices=ind)
                assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes(), \
                    (sname, pname, "knn_stats", k, rank)
            checked += 4
        # RadiusOutlierRemoval: both rules, negative both ways, on the tile and on a subset of arbitrary queries
        for q, ind in ((tile, None), (q_any, sub)):
            rows = q if ind is None else q[ind]
            for min_pts, radius in ((3, 0.02), (40, 0.05)):
                _, kth = ref_index.knn_stats(q, min_pts + 1, indices=ind)
                for is_dense in (True, False):
                    for negative in (False, True):
                        got = tindex.radius_outlier_removal_sharded(q, radius, min_pts, negative, is_dense, indices=ind)
                        want = S.ror_rule(kth, S.finite_rows(rows), is_dense, radius, negative)
                        assert got.tobytes() == want.tobytes(), (sname, pname, "ror", min_pts, is_dense, negative, rank)
                        checked += 1
        # one rank not dense: the radius rule on every rank
        got = tindex.radius_outlier_removal_sharded(tile, 0.02, 3, False, is_dense=rank != world - 1)
        _, kth = ref_index.knn_stats(tile, 4)
        assert got.tobytes() == S.ror_rule(kth, S.finite_rows(tile), False, 0.02).tobytes(), (sname, pname, "ror mixed")
        # StatisticalOutlierRemoval over the concatenation of every rank's queries in rank order
        every = np.concatenate(parts).astype(np.int32)
        at = int(sum(len(p) for p in parts[:rank]))
        for mean_k, std_mul in ((8, 1.0), (50, 0.5)):
            means, _ = ref_index.knn_stats(whole, mean_k + 1, indices=every)
            for negative in (False, True):
                want, (valid, mean, thr) = S.sor_rule(means, S.finite_rows(whole[every]), std_mul, negative)
                band = REL * abs(thr)
                assert not (np.abs(means.astype(np.float64) - thr) <= band).any(), (sname, pname, "a mean in the band")
                keep, st = tindex.statistical_outlier_removal_sharded(tile, mean_k, std_mul, negative)
                assert st["valid"] == valid and abs(st["thr"] - thr) <= band and abs(st["mean"] - mean) <= REL * abs(mean), \
                    (sname, pname, "sor stats", st, (valid, mean, thr))
                every_thr = S.gathered(st["thr"])
                assert len(set(every_thr)) == 1, (sname, pname, "thr differs between ranks", every_thr)
                assert keep.tobytes() == want[at:at + len(parts[rank])].tobytes(), (sname, pname, "sor", mean_k, negative, rank)
                checked += 1
        # an indices subset of arbitrary queries: each rank its own slice
        mine = sub[rank::world]
        keep, st = tindex.statistical_outlier_removal_sharded(q_any, 8, 1.0, False, indices=mine)
        allq = np.concatenate([sub[r::world] for r in range(world)])
        means, _ = ref_index.knn_stats(q_any, 9, indices=allq)
        want, (valid, mean, thr) = S.sor_rule(means, S.finite_rows(q_any[allq]), 1.0)
        assert st["valid"] == valid and abs(st["thr"] - thr) <= REL * abs(thr), (sname, pname, "sor subset", st, thr)
        off = int(sum(len(sub[r::world]) for r in range(rank)))
        assert not (np.abs(means.astype(np.float64) - thr) <= REL * abs(thr)).any()
        assert keep.tobytes() == want[off:off + len(mine)].tobytes(), (sname, pname, "sor subset", rank)
        checked += 1
        # the CPU oracle (PCL's own arithmetic): the slab partition of each scene, the tile's records as queries
        if pname == "slabs":
            orc_index = oracle.Index(whole)
            kept = orc_index.statistical_outlier_removal(np.ascontiguousarray(whole[every]), 50, 0.5)
            want = np.zeros(len(every), np.uint8)
            want[kept] = 1
            keep, _ = tindex.statistical_outlier_removal_sharded(tile, 50, 0.5)
            assert keep.tobytes() == want[at:at + len(parts[rank])].tobytes(), (sname, "sor vs oracle", rank)
            for is_dense in (True, False):
                kept = orc_index.radius_outlier_removal(tile, 0.02, 3, is_dense=is_dense)
                want = np.zeros(len(tile), np.uint8)
                want[kept] = 1
                got = tindex.radius_outlier_removal_sharded(tile, 0.02, 3, is_dense=is_dense)
                assert got.tobytes() == want.tobytes(), (sname, "ror vs oracle", is_dense, rank)
            checked += 3
        print(f"rank {rank}: {sname} {pname} ok", flush=True)

# ---- a map smaller than k: k_eff counts its distinct finite ids; id 0 is held by every rank; the last rank asks nothing --
tiny = P.xyz1(rng.random((12, 3), dtype=np.float32))
tiny[5, 0] = np.nan
tids = np.unique(np.r_[0, np.arange(12)[rank::world]]).astype(np.int32)
tt = P.Index(ctx, np.ascontiguousarray(tiny[tids]), ids=tids)
tq = np.ascontiguousarray(tiny[tids]) if rank != world - 1 else np.zeros((0, 4), np.float32)
got, want = tt.knn_sharded(tq, 16), P.Index(ref_ctx, tiny).knn(tq, 16)
assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes() and got[2] == want[2] == 11, \
    ("tiny map", got[2], want[2])
checked += 1

# ---- device arrays in and out --------------------------------------------------------------------------------------------
whole = SCENES[0][1]
parts = next(S.partitions(rng, whole, world))[1]
tile = np.ascontiguousarray(whole[parts[rank]])
tindex = P.Index(ctx, tile, ids=np.ascontiguousarray(parts[rank], dtype=np.int32))
ref_index = P.Index(ref_ctx, whole)
qd = torch.from_numpy(tile).to(f"cuda:{dev}")
oi = torch.empty((len(tile), 16), dtype=torch.int32, device=f"cuda:{dev}")
od = torch.empty((len(tile), 16), dtype=torch.float32, device=f"cuda:{dev}")
_, _, keff = tindex.knn_sharded(qd, 16, out_idx=oi, out_d2=od)
want = ref_index.knn(tile, 16)
assert oi.cpu().numpy().tobytes() == want[0].tobytes() and od.cpu().numpy().tobytes() == want[1].tobytes() and keff == 16
checked += 1


# ---- refusals: ERR_INVALID on every rank, and the communicator still works -------------------------------------------------
plain = P.Index(ctx, tile)
lone = P.Index(ref_ctx, tile, ids=np.ascontiguousarray(parts[rank], dtype=np.int32))
S.refused(lambda: tindex.knn_sharded(tile, 0), "k must be positive")
S.refused(lambda: tindex.knn_stats_sharded(tile, 0), "k must be positive")
S.refused(lambda: tindex.statistical_outlier_removal_sharded(tile, 0, 1.0), "mean_k must be positive")
S.refused(lambda: tindex.radius_outlier_removal_sharded(tile, 0.0, 3), "radius must be positive")
S.refused(lambda: tindex.radius_outlier_removal_sharded(tile, 0.02, -1), "min_pts must not be negative")
S.refused(lambda: plain.knn_sharded(tile, 8), "pclb200_index_build_ids")
S.refused(lambda: plain.knn_stats_sharded(tile, 8), "pclb200_index_build_ids")
S.refused(lambda: plain.statistical_outlier_removal_sharded(tile, 8, 1.0), "pclb200_index_build_ids")
S.refused(lambda: plain.radius_outlier_removal_sharded(tile, 0.02, 3), "pclb200_index_build_ids")
S.refused(lambda: lone.knn_sharded(tile, 8), "communicator")
S.refused(lambda: lone.knn_stats_sharded(tile, 8), "communicator")
S.refused(lambda: lone.statistical_outlier_removal_sharded(tile, 8, 1.0), "communicator")
S.refused(lambda: lone.radius_outlier_removal_sharded(tile, 0.02, 3), "communicator")
got = tindex.knn_sharded(tile, 16)
assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()
me.finish("SHARDED_FILTERS", checks=checked)
