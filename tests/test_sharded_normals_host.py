"""Normals of a map sharded across ranks without a GPU: the halo kernels (pcl_b200/csrc/shard_normals_kernels.cuh, driven
by shard_normals.cu) compiled for the host, and the exactness argument checked on the CPU oracle: the normals of the
whole map equal, bit for bit, the normals over one rank's tile plus its halo, indexed in id order."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"
HOST = os.path.join(ROOT, "tests", "host")


@pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")) or shutil.which("g++") is None,
                    reason="needs g++ and the CUDA headers (vector types only; nothing is run on a device)")
def test_sharded_normals_halo_layout_on_the_host(tmp_path):
    """1 / 2 / 3 / 5 / 8 simulated ranks, both exchange protocols, the segments placed and read with the layout functions
    of peer_tables.cuh that the driver calls: every rank's box is the outward-rounded union of its
    queries' reaches, its halo is exactly the other tiles' points inside that box, and every whole-map neighbour of every
    query (ties at the k-th distance included; radius: d2 <= r^2) lies in the tile plus the halo — slabs, a random
    partition, overlapping tiles sharing ids, a far tile with fewer than k points, k = 3 / 16 / 40 and a radius."""
    exe = str(tmp_path / "shard_normals_host_test")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-frounding-math", "-ffp-contract=off", "-fno-fast-math",
                           "-I" + CUDA_INC, "-I" + os.path.join(ROOT, "include"), "-I" + HOST,
                           os.path.join(HOST, "shard_normals_host_test.cpp"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]
    assert any(l.startswith("a far tile of 2 points") and "R=8 nccl" in l for l in r.stdout.splitlines())
    assert "DIFFERS" not in r.stdout


def _halo_ids(orc, whole, parts, r, queries, k, radius):
    """Rank r's local map as ids, selected in numpy: the box of its queries widened by their reach (the k-th nearest
    distance in its own tile, or the radius), rounded outward by a float step, over every tile."""
    tile = whole[parts[r]]
    fin = np.isfinite(queries[:, :3]).all(1)
    q = queries[fin, :3].astype(np.float64)
    if k:
        _, kth = orc.Index(tile).knn_stats(queries[fin], k)
        rho = np.sqrt(kth.astype(np.float64))
    else:
        rho = np.full(len(q), radius * radius, np.float32).astype(np.float64) ** 0.5
    h = rho * (1 + 2.0 ** -20) + 2.0 ** -60
    lo = np.nextafter((q - h[:, None]).min(0).astype(np.float32), np.float32(-np.inf))
    hi = np.nextafter((q + h[:, None]).max(0).astype(np.float32), np.float32(np.inf))
    pts = whole[:, :3]
    inside = (pts >= lo).all(1) & (pts <= hi).all(1)
    sel = np.zeros(len(whole), bool)
    for s, p in enumerate(parts):
        if s != r:
            sel[p] |= inside[p]
    sel[parts[r]] = True
    return np.nonzero(sel)[0]  # ascending: the id order


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
