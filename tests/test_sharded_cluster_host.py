"""Euclidean clusters of a map sharded across ranks without a GPU: the stitching kernels (pcl_b200/csrc/
shard_cluster_kernels.cuh, driven by shard_cluster.cu) compiled for the host, and the exactness argument restated on the
CPU oracle: per-rank clusters of tile plus halo, joined by the edges of the points the halo shares, are the whole map's
clusters."""
import numpy as np
import pytest

import _sharded as S


@S.needs_host_compiler
def test_sharded_cluster_kernels_and_layout_on_the_host(tmp_path):
    """1 / 2 / 3 / 5 / 8 simulated ranks, both exchange protocols, the halo, the answers and the edges placed and read with
    the layout functions of peer_tables.cuh that the driver calls: every rank's labels and sizes equal a brute-force
    connected-components of the whole map — a zig-zag chain crossing every slab boundary many times, blobs on the
    boundaries, a lattice at and just above the tolerance, duplicated points, non-finite records, ids near 2^31 - 2,
    tolerance 0; slabs, a random partition, overlapping tiles sharing ids and a 1-point tile."""
    out = S.host_program(tmp_path, "shard_cluster_host_test.cpp", timeout=900)
    lines = out.splitlines()
    for want in ("zig-zag chain          slabs        R=8 nccl", "1-point tile R=8 peer", "overlapping  R=5 nccl",
                 "lattice above", "blobs, tolerance 0"):
        assert any(want in l for l in lines), want
    assert "DIFFERS" not in out


def _local_ids(whole, parts, r, tol):
    """Rank r's local map as ids: the box of its tile's finite points widened by the reach of r2, over every tile."""
    r2 = np.float32(np.float64(np.float32(tol)) ** 2)
    return S.local_ids(whole, parts, r, *S.halo_box(whole[parts[r]], r2))


def _stitched_labels(orc, whole, parts, tol):
    """The protocol of shard_cluster.cu in numpy: per-rank local labels, the edges of every point one rank's tile shares
    with another rank's local map, the smallest label of each connected set of labels.  Returns id -> final label."""
    R = len(parts)
    local, lab = [], []
    for r in range(R):
        ids = _local_ids(whole, parts, r, tol)
        l = orc.Index(np.ascontiguousarray(whole[ids])).cluster_labels(tol)
        local.append(ids)
        lab.append(np.where(l >= 0, ids[np.maximum(l, 0)], -1))  # as ids: the smallest id of the local component
    parent = {}

    def find(x):
        while parent.setdefault(x, x) != x:
            x = parent[x]
        return x

    for s in range(R):
        own = parts[s][np.isfinite(whole[parts[s], :3]).all(1)]
        for r in range(R):
            if r == s:
                continue
            shared = np.intersect1d(own, local[r])  # what s sent to r
            a = lab[s][np.searchsorted(local[s], shared)]
            b = lab[r][np.searchsorted(local[r], shared)]
            for x, y in zip(a.tolist(), b.tolist()):
                fx, fy = find(x), find(y)
                parent[max(fx, fy)] = min(fx, fy)
    final = {}
    for r in range(R):
        for i, l in zip(local[r].tolist(), lab[r].tolist()):
            f = find(l) if l >= 0 else -1
            assert final.setdefault(i, f) == f, ("two ranks disagree", i)
    return final


@pytest.mark.parametrize("layout", ["slabs", "random", "overlapping"])
def test_oracle_stitched_clusters_equal_the_whole_map(orc, layout):
    """The oracle's clusters of each rank's tile plus its numpy-selected halo, joined by one round of label edges over
    the shared points, equal the oracle's clusters of the whole map for every id: the claim that lets the library cluster
    a sharded map with its unchanged single-GPU kernels and one label exchange."""
    rng = np.random.default_rng(23)
    t = np.linspace(0, 1, 400, dtype=np.float32)
    chain = np.concatenate([np.c_[t if p % 2 == 0 else 1 - t, np.full_like(t, 0.05 * p), np.zeros_like(t)]
                            for p in range(8)])                               # 8 passes, 0.05 apart
    joins = np.concatenate([np.c_[np.full(20, float(p % 2 == 0)), 0.05 * p + np.arange(1, 21) * 0.0025, np.zeros(20)]
                            for p in range(7)]).astype(np.float32)            # joined alternately at x = 1 and x = 0
    blobs = (rng.normal(size=(3000, 3)) * 0.015 + rng.choice([0.25, 0.5, 0.75], size=(3000, 1))
             + [0, 0.6, 0]).astype(np.float32)
    xyz = np.concatenate([chain, joins, blobs, blobs[:40]])  # and duplicated points under other ids
    whole = orc.to_xyz1(xyz)
    whole[11, 2] = np.nan
    R = 3
    ids = np.arange(len(whole))
    x = np.nan_to_num(whole[:, 0])
    slab = np.minimum((x * R).astype(int), R - 1)
    if layout == "slabs":
        parts = [ids[slab == r] for r in range(R)]
    elif layout == "random":
        perm = rng.permutation(len(whole))
        parts = [np.sort(perm[r::R]) for r in range(R)]
    else:
        parts = [np.union1d(ids[slab == r], ids[(slab == r + 1) & (x * R - slab < 0.15)]) for r in range(R)]
    for tol in (0.003, 0.01, 0.04):
        want = orc.Index(whole).cluster_labels(tol)
        got = _stitched_labels(orc, whole, parts, tol)
        for r in range(R):
            lab = np.array([got[i] for i in parts[r].tolist()])
            assert np.array_equal(lab, want[parts[r]]), (layout, tol, r)
        n_comp = len(np.unique(want[want >= 0]))
        assert n_comp > 1 or tol == 0.04, (layout, tol, n_comp)
