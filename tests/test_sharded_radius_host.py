"""Radius search and GICP covariances of a map sharded across ranks without a GPU: the exactness argument checked on the
CPU oracle (radius lists and GICP neighbour rows over one rank's tile plus its halo, indexed in id order, equal the whole
map's bit for bit), the id mapping and the exchanges of pcl_b200/csrc/shard_filter.cu compiled for the host, and the
pairing of every index consumer of include/pclb200.h with a sharded form in include/pclb200_sharded.h."""
import os
import re

import numpy as np
import pytest

import _sharded as S

# the entry points of include/pclb200.h that take a pclb200_index but do not consume it as a search: its lifecycle, and
# the one-call wrapper of the ICP session (whose sharded form is the session itself, pclb200_icp_set_target_sharded)
NOT_CONSUMERS = {"pclb200_index_build", "pclb200_index_destroy", "pclb200_index_size", "pclb200_index_stats",
                 "pclb200_icp_align"}


def _entry_points(name):
    """{function: its parameter list} of every PCLB200_API declaration in include/<name>"""
    h = open(os.path.join(S.ROOT, "include", name)).read()
    return dict(re.findall(r"PCLB200_API\s+[\w\s\*]+?\b(pclb200_\w+)\s*\(([^;]*?)\)\s*;", h, re.S))


def test_every_index_consumer_has_a_sharded_form():
    """Every entry point of pclb200.h that reads a pclb200_index, other than the index lifecycle and pclb200_icp_align,
    has a <name>_sharded in pclb200_sharded.h (pclb200_icp_set_target: pclb200_icp_set_target_sharded)."""
    single, sharded = _entry_points("pclb200.h"), _entry_points("pclb200_sharded.h")
    consumers = sorted(f for f, params in single.items() if "pclb200_index*" in params.replace(" *", "*")
                       and f not in NOT_CONSUMERS)
    assert "pclb200_radius" in consumers and "pclb200_gicp_covariances" in consumers, consumers
    missing = [f for f in consumers if f + "_sharded" not in sharded]
    assert not missing, missing


@S.needs_host_compiler
def test_sharded_radius_kernels_on_the_host(tmp_path):
    """1 / 2 / 3 / 5 / 8 simulated ranks, both exchange protocols: the id mapping of the sorted-keys and register-rows
    lists against brute force on the whole map, the verdict and all_fit exchanges, a rank with no query, a rank whose
    capacity alone is short."""
    out = S.host_program(tmp_path, "shard_radius_host_test.cpp", timeout=900)
    assert any(l.startswith("overlapping") and "R=8 nccl" in l for l in out.splitlines())
    assert "DIFFERS" not in out


def _layouts(whole, R, rng):
    ids = np.arange(len(whole))
    x = np.nan_to_num(whole[:, 0])
    slab = np.minimum((x * R).astype(int), R - 1)
    yield "slabs", [ids[slab == r] for r in range(R)], whole
    perm = rng.permutation(len(whole))
    yield "random", [np.sort(perm[r::R]) for r in range(R)], whole
    frac = x * R - slab
    yield "shared ids", [np.r_[ids[slab == r], ids[(slab == r + 1) & (frac < 0.1)]] for r in range(R)], whole
    far = np.concatenate([whole, np.array([[9, 9, 9, 1], [9, 9.25, 9, 1]], np.float32)])
    parts = [ids[slab == r] for r in range(R)]
    parts[-2] = np.r_[parts[-2], parts[-1]]
    parts[-1] = np.array([len(whole), len(whole) + 1])
    yield "a far tile of 2 points", parts, far


def _rows_by_d2_id(offs, idx, d2):
    """every row of a radius list in (d2, id) order (the oracle's kd-tree orders ties by its own walk)"""
    out_i, out_d = idx.copy(), d2.copy()
    for a, b in zip(offs[:-1], offs[1:]):
        o = np.lexsort((idx[a:b], d2[a:b]))
        out_i[a:b], out_d[a:b] = idx[a:b][o], d2[a:b][o]
    return out_i, out_d


@pytest.mark.parametrize("layout", ["slabs", "random", "shared ids", "a far tile of 2 points"])
def test_oracle_radius_and_gicp_over_tile_and_halo_equal_the_whole_map(orc, layout):
    """The oracle's radius lists over a rank's tile plus its numpy-selected halo (the box of its queries widened by the
    reach of r^2), as a cloud in id order, mapped back to ids, equal the oracle's on the whole map bit for bit, for radii
    of 0, a few and many neighbours; with max_nn 1, 16, 33 and more than the map, under the library's (d2, index) rule
    (brute-force k-NN rows cut at d2 < r^2).  The GICP neighbour rows of the tile's records over tile plus the halo of
    their k-th distance equal the whole map's (k = 20, and k above the map's size, where the halo is the whole map)."""
    rng = np.random.default_rng(37)
    n = 6000
    xy = rng.random((n, 2), dtype=np.float32)
    surf = np.stack([xy[:, 0], xy[:, 1], (0.1 * np.sin(6 * xy[:, 0]) * np.cos(5 * xy[:, 1])).astype(np.float32)], 1)
    g = np.stack(np.meshgrid(*[np.arange(8, dtype=np.float32) / 8] * 2, indexing="ij"), -1).reshape(-1, 2)
    lattice = np.c_[g, np.full(len(g), 0.5, np.float32)]          # exact ties
    base = orc.to_xyz1(np.concatenate([surf, lattice, surf[:50]]))  # and duplicated points under other ids
    base[7, 1] = np.nan
    R = 3
    _, parts, whole = next(l for l in _layouts(base, R, rng) if l[0] == layout)
    ref_index = orc.Index(whole)
    fin = S.finite_rows(whole)
    for r in range(R):
        tile_q = np.ascontiguousarray(whole[parts[r]])
        extra = orc.to_xyz1(np.array([[0.125, 0.375, 0.5], [0.5, 0.5, 0.5], [5, 5, 5], [np.nan, 0, 0]], np.float32))
        queries = np.ascontiguousarray(np.concatenate([tile_q[::4], extra]))
        for radius in (0.0, 0.01, 0.125, 0.06):
            r2 = np.float32(radius * radius)
            local = S.local_ids(whole, parts, r, *S.halo_box(queries, r2)) if r2 > 0 else np.sort(parts[r])
            cr = orc.Index(np.ascontiguousarray(whole[local]))
            got = cr.radius(queries, radius)
            want = ref_index.radius(queries, radius)
            assert got[0].tobytes() == want[0].tobytes(), (layout, r, radius, "offsets")
            gi, gd = _rows_by_d2_id(got[0], local[got[1]].astype(np.int32), got[2])
            wi, wd = _rows_by_d2_id(*want)
            assert gi.tobytes() == wi.tobytes() and gd.tobytes() == wd.tobytes(), (layout, r, radius)
            if radius == 0.06:  # max_nn: the nearest max_nn of the ball in (d2, id) order
                fq = np.ascontiguousarray(queries[S.finite_rows(queries)][:300])
                for max_nn in (1, 16, 33, int(fin.sum()) + 5):
                    li, ld, _ = orc.knn_bruteforce(whole[local], fq, max_nn)
                    li = np.where((li >= 0) & (ld < r2), local[np.maximum(li, 0)], -1).astype(np.int32)
                    wi, wd, _ = orc.knn_bruteforce(whole, fq, max_nn)
                    wi = np.where((wi >= 0) & (wd < r2), wi, -1).astype(np.int32)
                    assert li.tobytes() == wi.tobytes(), (layout, r, max_nn)
                    assert ld[li >= 0].tobytes() == wd[wi >= 0].tobytes(), (layout, r, max_nn)
        # GICP covariances: the tile's records, their k nearest
        fq = np.ascontiguousarray(tile_q[S.finite_rows(tile_q)])
        for k in (20, int(fin.sum()) + 3):
            rho2 = orc.Index(whole[parts[r]]).knn_stats(fq, k)[1] if k <= len(fq) else np.float32(np.inf)
            local = S.local_ids(whole, parts, r, *S.halo_box(fq, rho2))
            keff = min(k, int(S.finite_rows(whole[local]).sum()))
            assert keff == min(k, int(fin.sum())), (layout, r, k)
            qq = fq[:400]
            li, ld, _ = orc.knn_bruteforce(whole[local], qq, keff)
            li = np.where(li >= 0, local[np.maximum(li, 0)], -1).astype(np.int32)
            wi, wd, _ = orc.knn_bruteforce(whole, qq, keff)
            assert li.tobytes() == wi.tobytes() and ld.tobytes() == wd.tobytes(), (layout, r, k)
