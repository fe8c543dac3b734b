"""Normals of a map sharded across ranks without a GPU: the halo kernels (pcl_b200/csrc/shard_normals_kernels.cuh, driven
by shard_normals.cu) compiled for the host, and the exactness argument checked on the CPU oracle: the normals of the
whole map equal, bit for bit, the normals over one rank's tile plus its halo, indexed in id order."""
import numpy as np
import pytest

import _sharded as S


@S.needs_host_compiler
def test_sharded_normals_halo_layout_on_the_host(tmp_path):
    """1 / 2 / 3 / 5 / 8 simulated ranks, both exchange protocols, the segments placed and read with the layout functions
    of peer_tables.cuh that the driver calls: every rank's box is the outward-rounded union of its
    queries' reaches, its halo is exactly the other tiles' points inside that box, and every whole-map neighbour of every
    query (ties at the k-th distance included; radius: d2 <= r^2) lies in the tile plus the halo — slabs, a random
    partition, overlapping tiles sharing ids, a far tile with fewer than k points, k = 3 / 16 / 40 and a radius."""
    out = S.host_program(tmp_path, "shard_normals_host_test.cpp", timeout=900)
    assert any(l.startswith("a far tile of 2 points") and "R=8 nccl" in l for l in out.splitlines())
    assert "DIFFERS" not in out


def _halo_ids(orc, whole, parts, r, queries, k, radius):
    """Rank r's local map as ids: the box of its queries widened by their reach (the k-th nearest distance in its own
    tile, or the radius) over every tile."""
    q = queries[S.finite_rows(queries)]
    rho2 = orc.Index(whole[parts[r]]).knn_stats(q, k)[1] if k else np.float32(radius * radius)
    return S.local_ids(whole, parts, r, *S.halo_box(q, rho2))


@pytest.mark.parametrize("layout", ["slabs", "random"])
def test_oracle_normals_over_tile_and_halo_equal_the_whole_map(orc, layout):
    """The oracle's normals over a rank's tile plus its numpy-selected halo, as a cloud in id order, equal the oracle's
    normals over the whole map bit for bit (NaN rows included) for k = 3, 16, 40 and a radius: the claim that lets the
    library answer sharded normals with its unchanged single-GPU kernels."""
    rng = np.random.default_rng(21)
    n = 12000
    xy = rng.random((n, 2), dtype=np.float32)
    surf = np.stack([xy[:, 0], xy[:, 1], (0.1 * np.sin(6 * xy[:, 0]) * np.cos(5 * xy[:, 1])).astype(np.float32)], 1)
    g = np.stack(np.meshgrid(*[np.arange(8, dtype=np.float32) / 8] * 2, indexing="ij"), -1).reshape(-1, 2)
    lattice = np.c_[g, np.full(len(g), 0.5, np.float32)]          # exact ties
    whole = orc.to_xyz1(np.concatenate([surf, lattice, surf[:50]]))  # and duplicated points under other ids
    whole[7, 1] = np.nan
    R = 3
    ids = np.arange(len(whole))
    if layout == "slabs":
        parts = [ids[np.minimum((np.nan_to_num(whole[:, 0]) * R).astype(int), R - 1) == r] for r in range(R)]
    else:
        perm = rng.permutation(len(whole))
        parts = [np.sort(perm[r::R]) for r in range(R)]
    ref_index = orc.Index(whole)
    for r in range(R):
        # the oracle reads the neighbours out of the cloud it is given, as NormalEstimation does with its search
        # surface: the queries are the tile's points, addressed by indices into the whole map or into the local map;
        # is_dense=False so that the non-finite map point gets a NaN row, as in the library, not a search from NaN
        queries = whole[parts[r]]
        for k, radius in ((3, 0), (16, 0), (40, 0), (0, 0.05)):
            local = _halo_ids(orc, whole, parts, r, queries, k, radius)
            cloud = np.ascontiguousarray(whole[local])
            cr = orc.Index(cloud)
            at = np.searchsorted(local, parts[r])
            if k:
                want, dw = ref_index.normals_knn(whole, k, indices=parts[r], is_dense=False)
                got, dg = cr.normals_knn(cloud, k, indices=at, is_dense=False)
            else:
                want, dw = ref_index.normals_radius(whole, radius, indices=parts[r], is_dense=False)
                got, dg = cr.normals_radius(cloud, radius, indices=at, is_dense=False)
            assert got.tobytes() == want.tobytes() and dg == dw, (layout, r, k, radius)
            assert len(local) < len(whole) or layout == "random", (layout, r, k, len(local))
