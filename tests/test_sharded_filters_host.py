"""k-NN queries and outlier filters of a map sharded across ranks without a GPU: the exactness argument checked on the CPU
oracle (k-NN rows and statistics over one rank's tile plus its halo, indexed in id order, equal the whole map's bit for
bit, and the filters' rules applied to the ranks' concatenated statistics give the whole map's masks), and the kernels of
pcl_b200/csrc/shard_filter_kernels.cuh (driven by shard_filter.cu) compiled for the host."""
import numpy as np
import pytest

import _sharded as S


@S.needs_host_compiler
def test_sharded_filter_kernels_on_the_host(tmp_path):
    """1 / 2 / 3 / 5 / 8 simulated ranks, both exchange protocols: the id mapping of k-NN rows, the SOR partial sums, their
    exchange and the rank-order fold (every rank the same threshold, within 1e-12 of the sequential one), and both mask
    rules against the facade's."""
    out = S.host_program(tmp_path, "shard_filter_host_test.cpp", timeout=900)
    assert any(l.startswith("random, one rank empty") and "R=8 nccl" in l for l in out.splitlines())
    assert "DIFFERS" not in out


def _halo_ids(orc, whole, parts, r, queries, k, radius):
    """Rank r's local map as ids: the box of its queries widened by their reach (the k-th nearest distance in its own
    tile, or the radius) over every tile."""
    q = queries[S.finite_rows(queries)]
    rho2 = orc.Index(whole[parts[r]]).knn_stats(q, k)[1] if k else np.float32(radius * radius)
    return S.local_ids(whole, parts, r, *S.halo_box(q, rho2))


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


def _mask(kept, n):
    m = np.zeros(n, np.uint8)
    m[kept] = 1
    return m


@pytest.mark.parametrize("layout", ["slabs", "random", "shared ids", "a far tile of 2 points"])
def test_oracle_knn_and_filters_over_tile_and_halo_equal_the_whole_map(orc, layout):
    """The oracle's k-NN rows (record numbers mapped back to ids) and k-NN statistics over a rank's tile plus its
    numpy-selected halo, as a cloud in id order, equal the oracle's on the whole map bit for bit for k = 2, 9, 16, 33, 51;
    SOR's rule over the ranks' concatenated means and ROR's over each rank's k-th distances give orc_sor's and orc_ror's
    masks on the whole map."""
    rng = np.random.default_rng(31)
    n = 12000
    xy = rng.random((n, 2), dtype=np.float32)
    surf = np.stack([xy[:, 0], xy[:, 1], (0.1 * np.sin(6 * xy[:, 0]) * np.cos(5 * xy[:, 1])).astype(np.float32)], 1)
    g = np.stack(np.meshgrid(*[np.arange(8, dtype=np.float32) / 8] * 2, indexing="ij"), -1).reshape(-1, 2)
    lattice = np.c_[g, np.full(len(g), 0.5, np.float32)]          # exact ties
    base = orc.to_xyz1(np.concatenate([surf, lattice, surf[:50]]))  # and duplicated points under other ids
    base[7, 1] = np.nan
    R = 3
    _, parts, whole = next(l for l in _layouts(base, R, rng) if l[0] == layout)
    ref_index = orc.Index(whole)
    fin_all = np.isfinite(whole[:, :3]).all(1)
    for k in (2, 9, 16, 33, 51):
        means = []
        for r in range(R):
            queries = np.ascontiguousarray(whole[parts[r]])
            local = _halo_ids(orc, whole, parts, r, queries, k, 0)
            cr = orc.Index(np.ascontiguousarray(whole[local]))
            # rows under the (d2, index) rule of the library (the brute force's; the kd-tree orders ties by its own
            # walk), for the finite queries (the library's rows of non-finite queries are checked on the GPU)
            fq = np.ascontiguousarray(queries[np.isfinite(queries[:, :3]).all(1)])
            got_i, got_d, _ = orc.knn_bruteforce(whole[local], fq, k)
            got_i = np.where(got_i >= 0, local[np.maximum(got_i, 0)], -1).astype(np.int32)
            want_i, want_d, _ = orc.knn_bruteforce(whole, fq, k)
            assert got_i.tobytes() == want_i.tobytes() and got_d.tobytes() == want_d.tobytes(), (layout, r, k)
            gm, gk = cr.knn_stats(queries, k)
            wm, wk = ref_index.knn_stats(queries, k)
            assert gm.tobytes() == wm.tobytes() and gk.tobytes() == wk.tobytes(), (layout, r, k)
            means.append(gm)
            if k in (2, 9):  # ROR with min_pts = k - 1
                for is_dense in (True, False):
                    want = _mask(ref_index.radius_outlier_removal(queries, 0.02, k - 1, is_dense=is_dense), len(queries))
                    assert S.ror_rule(gk, fin_all[parts[r]], is_dense, 0.02).tobytes() == want.tobytes(), (layout, r, k)
            assert len(local) < len(whole) or layout == "random" or (layout.startswith("a far") and r == R - 1), \
                (layout, r, k, len(local))
        if k in (9, 51):  # SOR with mean_k = k - 1 over the concatenation of the ranks' queries in rank order
            every = np.concatenate(parts)
            want = _mask(ref_index.statistical_outlier_removal(np.ascontiguousarray(whole[every]), k - 1, 1.0), len(every))
            assert S.sor_rule(np.concatenate(means), fin_all[every], 1.0)[0].tobytes() == want.tobytes(), (layout, k)
