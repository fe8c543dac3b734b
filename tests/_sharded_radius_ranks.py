"""Helper for tests/test_gpu_sharded_radius.py (launched under torchrun, gloo): radius search and GICP covariances of a map
sharded across ranks (pclb200_radius_sharded, pclb200_radius_into_sharded, pclb200_gicp_covariances_sharded).

Ranks on cuda:0 with the peer exchange bootstrapped over gloo (comm_export / _import), or, with PCLB_SHARDED_NCCL=1, one
GPU per rank with pclb200_comm_init and PCLB200_REDUCE_NCCL.  Two maps (a surface and a volume cloud, both with an
exact-tie lattice, non-finite rows and duplicated points under other ids), four partitions (spatial slabs; a random
partition; slabs whose points near a cut are held by both neighbours under one id; slabs plus a far tile of 2 points).
Queries: each tile's own records, arbitrary points and NaN points; the last rank passes none in one case.  Radii: 0, NaN,
~10 and ~300 neighbours, and one whose square overflows; max_nn 0, 1, 5, 32 (the register k-NN path), 40 and larger than
the map; ranks pass different radii in one case.  Offsets, ids and d2 of both calls, with host and device buffers, must be
byte-equal to one process's pclb200_radius / pclb200_radius_into on an index of the whole map; the GICP covariances, as
rows at the ids, byte-equal to pclb200_gicp_covariances on the whole map.  The collective retry: only one rank's capacity
is short, all_fit is 0 on every rank, then 1 after one grown call, with the same bytes.  Last, the refusals (ERR_INVALID
on every rank, also when only one rank passes the bad argument), after which the communicator still works."""
import ctypes as C

import numpy as np
import torch

import _sharded as S
import pcl_b200 as P

me = S.join()
rank, world, dev, ctx, ref_ctx = me.rank, me.world, me.device, me.ctx, me.ref

rng = np.random.default_rng(29)


def lattice(origin, n, step):
    g = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float32) * np.float32(step)] * 2, indexing="ij"), -1).reshape(-1, 2)
    return np.c_[g, np.zeros(len(g), np.float32)] + np.asarray(origin, np.float32)


# radii of ~10 and ~300 neighbours on each map (surface: 150k points on 4 x 4; volume: 80k points in 0.6^3)
SCENES = [("surface", S.with_extras(rng, np.concatenate([S.surface(rng, 150000), lattice((0.5, 0.5, 1.0), 64, 1 / 32)])),
           (0.016, 0.08)),
          ("volume", S.with_extras(rng, np.concatenate([S.volume(rng, 80000), lattice((0.0, 0.0, 0.3), 32, 1 / 64)])),
           (0.0125, 0.04))]


def same(got, want, what):
    for g, w, name in zip(got, want, ("offsets", "ids", "d2")):
        assert np.asarray(g).tobytes() == np.asarray(w).tobytes(), (what, name, rank)


def into(index, q, r, max_nn, cap, device=False):
    """radius_into_sharded with buffers of cap entries: (offsets, ids, d2, total, all_fit)"""
    n = len(q)
    if device:
        d = f"cuda:{dev}"
        qq = torch.from_numpy(np.ascontiguousarray(q)).to(d)
        off, ids, d2 = (torch.empty(n + 1, dtype=torch.int64, device=d), torch.empty(max(cap, 1), dtype=torch.int32, device=d),
                        torch.empty(max(cap, 1), dtype=torch.float32, device=d))
        ids, d2 = ids[:cap], d2[:cap]
    else:
        qq = q
        off, ids, d2 = np.empty(n + 1, np.int64), np.empty(cap, np.int32), np.empty(cap, np.float32)
    total, fit = index.radius_into_sharded(qq, r, off, ids, d2, max_nn)
    if device:
        off, ids, d2 = off.cpu().numpy(), ids.cpu().numpy(), d2.cpu().numpy()
    return off, ids[:min(total, cap)], d2[:min(total, cap)], total, fit


def grown_into(index, q, r, max_nn, device=False):
    """the caller's loop: start with no room, grow to the total while some rank's lists do not fit"""
    cap, calls = 0, 0
    while True:
        off, ids, d2, total, fit = into(index, q, r, max_nn, cap, device)
        calls += 1
        if fit:
            return (off, ids, d2), calls
        cap = max(cap, total)


checked = 0
for sname, whole0, (r_small, r_large) in SCENES:
    for pname, parts, whole in S.partitions(rng, whole0, world):
        ref_index = P.Index(ref_ctx, whole)
        tile = np.ascontiguousarray(whole[parts[rank]])
        tindex = P.Index(ctx, tile, ids=np.ascontiguousarray(parts[rank], dtype=np.int32))
        q_any, sub = S.arbitrary_queries(rng, whole)
        q_any = np.ascontiguousarray(q_any[sub])
        huge = float(np.sqrt(np.finfo(np.float32).max)) * 2.0  # its square overflows float: the whole map
        cases = [(tile, r_small, 0), (tile, r_large, 0), (tile, r_small, 1), (tile, r_large, 5), (tile, r_large, 32),
                 (tile, r_large, 40), (q_any, r_small, 0), (q_any, r_large, 32), (q_any, r_small, len(whole) + 5),
                 (tile, 0.0, 0), (q_any, float("nan"), 0)]
        if pname == "far tile":
            cases.append((tile, huge, 7))  # a radius over the whole map: 2 queries on the last rank, ~n on the others
        # ranks pass different radii and max_nn in one case
        cases.append((tile, (r_small, r_large, r_small * 2)[rank % 3], (0, 32, 3)[rank % 3]))
        if pname == "slabs":  # the last rank passes no query
            cases.append((tile if rank != world - 1 else np.zeros((0, 4), np.float32), r_small, 0))
        for q, r, max_nn in cases:
            if r == huge and rank != world - 1:
                q = q[:3]
            # pclb200_radius on no query: offsets [0] and no list (Index.radius reads the lists it allocates)
            want = ref_index.radius(q, r, max_nn) if len(q) else (np.zeros(1, np.int64), np.zeros(0, np.int32),
                                                                   np.zeros(0, np.float32))
            got = tindex.radius_sharded(q, r, max_nn)
            same(got, want, (sname, pname, "radius", r, max_nn))
            if len(q) == 0:
                assert got[1].size == 0
            got, calls = grown_into(tindex, q, r, max_nn, device=(checked % 2 == 1))
            same(got, want, (sname, pname, "radius_into", r, max_nn))
            checked += 2
        # GICP covariances of the tile's records: rows at the ids
        for k in (20, 64):
            want = ref_index.gicp_covariances(whole, k=k)[parts[rank]]
            got = tindex.gicp_covariances_sharded(tile, k=k)
            assert got.tobytes() == want.tobytes(), (sname, pname, "gicp", k, rank)
            checked += 1
        print(f"rank {rank}: {sname} {pname} ok", flush=True)

# ---- the collective retry: only rank 0's capacity is short ------------------------------------------------------------------
whole, (r_small, _) = SCENES[0][1], SCENES[0][2]
parts = next(S.partitions(rng, whole, world))[1]
tile = np.ascontiguousarray(whole[parts[rank]])
tindex = P.Index(ctx, tile, ids=np.ascontiguousarray(parts[rank], dtype=np.int32))
ref_index = P.Index(ref_ctx, whole)
want = ref_index.radius(tile, r_small)
need = int(want[0][-1])
for device in (False, True):
    cap = need - 1 if rank == 0 else need + 10
    off, ids, d2, total, fit = into(tindex, tile, r_small, 0, cap, device)
    assert total == need and not fit, ("retry", rank, total, need, fit)
    assert off.tobytes() == want[0].tobytes(), ("retry offsets", rank)
    if rank != 0:
        assert ids.tobytes() == want[1].tobytes() and d2.tobytes() == want[2].tobytes(), ("retry: fitted lists", rank)
    off, ids, d2, total, fit = into(tindex, tile, r_small, 0, max(cap, total), device)
    assert fit, ("retry: grown", rank)
    same((off, ids, d2), want, ("retry: grown", device))
    checked += 1
# all_fit is the same on every rank
_, _, _, _, fit = into(tindex, tile, r_small, 0, 0 if rank == world - 1 else need)
assert S.gathered(fit) == [False] * world

# ---- GICP covariances of a map smaller than k; id 0 held by every rank -----------------------------------------------------
tiny = P.xyz1(rng.random((12, 3), dtype=np.float32))
tiny[5, 0] = np.nan
tids = np.unique(np.r_[0, np.arange(12)[rank::world]]).astype(np.int32)
tt = P.Index(ctx, np.ascontiguousarray(tiny[tids]), ids=tids)
want = P.Index(ref_ctx, tiny).gicp_covariances(tiny, k=16)[tids]
assert tt.gicp_covariances_sharded(np.ascontiguousarray(tiny[tids]), k=16).tobytes() == want.tobytes(), "tiny gicp"
# device output
out = torch.empty((len(tids), 9), dtype=torch.float64, device=f"cuda:{dev}")
tt.gicp_covariances_sharded(torch.from_numpy(np.ascontiguousarray(tiny[tids])).to(f"cuda:{dev}"), k=16, out=out)
assert out.cpu().numpy().tobytes() == want.reshape(-1, 9).tobytes(), "tiny gicp on the device"
checked += 2

# ---- refusals: ERR_INVALID on every rank, also when one rank alone passes the bad argument ----------------------------------
plain = P.Index(ctx, tile)
lone = P.Index(ref_ctx, tile, ids=np.ascontiguousarray(parts[rank], dtype=np.int32))
S.refused(lambda: plain.radius_sharded(tile, r_small), "pclb200_index_build_ids")
S.refused(lambda: plain.radius_into_sharded(tile, r_small, np.empty(len(tile) + 1, np.int64), np.empty(0, np.int32),
                                            np.empty(0, np.float32)), "pclb200_index_build_ids")
S.refused(lambda: plain.gicp_covariances_sharded(tile), "pclb200_index_build_ids")
S.refused(lambda: tindex.gicp_covariances_sharded(tile, k=0), "k must be positive")
S.refused(lambda: tindex.gicp_covariances_sharded(tile[:-1]), "record count")
S.refused(lambda: lone.radius_sharded(tile, r_small), "communicator")
S.refused(lambda: lone.radius_into_sharded(tile, r_small, np.empty(len(tile) + 1, np.int64), np.empty(0, np.int32),
                                           np.empty(0, np.float32)), "communicator")
S.refused(lambda: lone.gicp_covariances_sharded(tile), "communicator")
bad = world - 1  # one rank alone refuses its own arguments: every rank refuses
word = "refused its arguments" if rank != bad else "k must be positive"
S.refused(lambda: tindex.gicp_covariances_sharded(tile, k=0 if rank == bad else 20), word)
word = "refused its arguments" if rank != bad else "pclb200_index_build_ids"
S.refused(lambda: (plain if rank == bad else tindex).radius_sharded(tile, r_small), word)
word = "refused its arguments" if rank != bad else "NULL output buffers"
off = np.empty(len(tile) + 1, np.int64)
S.refused(lambda: P._check(P.lib().pclb200_radius_into_sharded(
    ctx.h, tindex.h, tile.ctypes.data, len(tile), 16, r_small, 0, off.ctypes.data, None, None, 10 if rank == bad else 0,
    C.byref(C.c_size_t()), None)), word)
# device out_offsets given to pclb200_radius_sharded
doff = torch.empty(len(tile) + 1, dtype=torch.int64, device=f"cuda:{dev}")
pi, pd = C.POINTER(C.c_int32)(), C.POINTER(C.c_float)()
word = "refused its arguments" if rank != bad else "host memory"
S.refused(lambda: P._check(P.lib().pclb200_radius_sharded(
    ctx.h, tindex.h, tile.ctypes.data, len(tile), 16, r_small, 0, 1,
    C.cast(C.c_void_p(doff.data_ptr() if rank == bad else off.ctypes.data), C.POINTER(C.c_int64)),
    C.byref(pi), C.byref(pd))), word)
checked += 12
got = tindex.radius_sharded(tile, r_small)
same(got, ref_index.radius(tile, r_small), "after the refusals")
me.finish("SHARDED_RADIUS", checks=checked)
