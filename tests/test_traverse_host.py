"""The DEVICE code compiled for the HOST (tests/host/*.cpp) — CPU only; nothing runs on a GPU.

g++ sees the same headers the kernels are built from (pcl_b200/csrc/traverse.cuh, knn_warp.cuh, search_kernels.cuh,
icp_kernels.cuh, lbvh_kernels.cuh, voxel_kernels.cuh, reject_kernels.cuh, normals_corr_kernels.cuh, cluster_kernels.cuh); the CUDA intrinsics are supplied with the same rounding, warp- and block-synchronous
primitives by a lock-step emulation of one thread block (tests/host/warp_emu.h: one fiber per thread, every *_sync
primitive a rendezvous; the m8n8k4 fp64 MMA emulated fragment by fragment).  Each program checks against brute force
under the library's own distance expression and tie rule, against the facade's host-side PCL functions, or against the
CPU oracle.  The search programs run twice: on an index built by a small reference builder (tests/host/host_index.h) and on
the index the REAL build kernels produce (tests/host/device_build.h replays lbvh.cu's sequence)."""
import os

import pytest

from _sharded import ROOT, host_program, needs_host_compiler

pytestmark = needs_host_compiler

DEVICE_BUILD = ["-DPCLB_TEST_DEVICE_BUILD", "-DPCLB_HOST_EMULATION", '-DPCLB_HOST_EXTRA_SHIMS="warp_emu.h"']


def test_index_build_kernels_on_the_host(tmp_path):
    """lbvh_kernels.cuh in lbvh.cu's sequence: every point in exactly one leaf slot, leaves of 1..8 points in Morton order,
    child boxes exact, subtree leaf ranges, and the cell table — every occupied cell of every level maps to a subtree that
    holds all of (and, for a node, only) its points — on fifteen clouds incl. duplicates, a lattice, degenerate frames and
    map-scale frames (a map at 1e5, a frame straddling zero, a cube stretched by one outlier 1e6 away)."""
    out = host_program(tmp_path, "lbvh_host_test.cpp", ["2"])
    assert "cell table levels 1.." in out and "map at 1e5" in out and "straddling zero" in out and "one outlier 1e6 away" in out


@pytest.mark.parametrize("device_built", [False, True], ids=["reference-index", "device-built-index"])
def test_device_traversal_header_on_the_host(tmp_path, device_built):
    """traverse.cuh (walk, nearest1, the cell-table look-ups and their conservative bounds, still_nearest): ~7e5 query
    variants on twelve scene families (map-scale frames among them) against brute force — with and without the table, no / the true / a random seed,
    the TRACK visitor's lower bound — and the temporal-coherence chain of k_search over drifting queries: a skipped walk
    never keeps a match that stopped being the nearest.  Five seeded mutations of the header are caught by this program."""
    out = host_program(tmp_path, "traverse_host_test.cpp", ["2"], DEVICE_BUILD if device_built else ())
    assert "map at 1e5" in out and "straddling zero" in out and "one outlier 1e6 away" in out


@pytest.mark.parametrize("device_built", [False, True], ids=["reference-index", "device-built-index"])
def test_per_thread_search_kernels_on_the_host(tmp_path, device_built):
    """search_kernels.cuh — k_knn<K> for every compiled list size, k_knn_any, k_knn_stats, k_radius_count / k_radius_fill,
    k_normals<K>, and the list-based forms k_stats_from_lists / k_normals_from_lists (k > 32) / k_normals_from_csr (radius
    normals) — block by block against brute force (lists bit for bit, ties and duplicates included) and, for the normals,
    against the host computePointNormal."""
    host_program(tmp_path, "search_host_test.cpp", ["2"], DEVICE_BUILD if device_built else ())


@pytest.mark.parametrize("device_built", [False, True], ids=["reference-index", "device-built-index"])
def test_warp_knn_kernel_on_an_emulated_warp(tmp_path, device_built):
    """knn_warp.cuh (k_knn_warp<false|true>, the shuffled bitonic sort / merge, the ranked insertion, the certification rule,
    the normals epilogue) on an emulated warp: every certified row equals brute force bit for bit, every normal equals the
    host computePointNormal on the brute-force list, and (reference index) the constructed shared-leaf scene — the bug the
    10 M-row comparison found on the device — passes; it fails on the kernel as it was before the fix."""
    out = host_program(tmp_path, "knn_warp_host_test.cpp", ["1"], DEVICE_BUILD if device_built else ())
    assert "shared leaf, constructed #5" in out and "map at 1e5" in out and "straddling zero" in out and "one outlier 1e6 away" in out


@pytest.mark.parametrize("device_built", [False, True], ids=["reference-index", "device-built-index"])
def test_whole_icp_iterations_about_the_svd_origin_on_an_emulated_block(tmp_path, device_built):
    """icp_kernels.cuh — k_search, k_accum_dmma (the m8n8k4 fp64 MMA emulated fragment by fragment), k_accum, k_solve with the
    convergence criteria in its tail, k_seed_origin — on an emulated 256-thread block, driven like icp.cu's icp_iterate
    (the SVD sums about the loop's device-side origin, which k_solve moves every iteration): every iteration's
    correspondences equal brute force, the accumulated normal equations equal plain fp64 sums, and iterations /
    state / counts / final transform of twelve aligns (SVD, point-to-plane, the symmetric objective, ICPWithNormals,
    reciprocal correspondences; float and double; gates; tracking off / on / automatic; rejector chains inside the loop —
    median + one-to-one, distance + trimmed, surface-normal + one-to-one; normal-shooting and back-projection
    correspondences; a 10 cm patch 500 m from the centre of its map) equal the oracle's loop (1e-5 float, 1e-9 double); the
    four stand-alone estimators against the oracle's."""
    import oracle
    oracle.build()
    odir = os.path.join(ROOT, "oracle")
    out = host_program(tmp_path, "icp_host_test.cpp", (), DEVICE_BUILD if device_built else (), ["-L" + odir, "-lpcl_oracle", "-Wl,-rpath," + odir])
    assert "tracking automatic" in out and "point-to-plane LLS double" in out and "reciprocal" in out and "trimmed rejectors" in out and "back-projection" in out and "500 m out" in out


def test_voxelgrid_kernels_on_the_host(tmp_path):
    """voxel_kernels.cuh in voxel.cu's sequence (bounds -> cell keys -> stable sort -> run heads -> runs -> minimum-points
    filter -> centroids -> normal / curvature planes), against the oracle's VoxelGrid: the same voxels in the same order,
    every centroid and every PointNormal plane bit for bit; anisotropic leaves, a far-from-origin sweep, non-finite points,
    an index subset, the minimum-points filter, and the overflow guard."""
    import oracle
    oracle.build()
    odir = os.path.join(ROOT, "oracle")
    out = host_program(tmp_path, "voxel_host_test.cpp", ["2"], (), ["-L" + odir, "-lpcl_oracle", "-Wl,-rpath," + odir])
    assert "overflow guard" in out and "PointNormal, min 2 points" in out


def test_rejector_kernels_on_the_host(tmp_path):
    """reject_kernels.cuh in reject.cu's sequence (stable sorts where the driver calls CUB) against the oracle's rejectors:
    survivors, their order and the median bit for bit for Distance / MedianDistance / OneToOne / Trimmed on eleven lists
    (ties, shared and negative matches, 0 / 1 / 2 / 256 / 257 records) and three chains."""
    import oracle
    oracle.build()
    odir = os.path.join(ROOT, "oracle")
    out = host_program(tmp_path, "reject_host_test.cpp", ["2"], (), ["-L" + odir, "-lpcl_oracle", "-Wl,-rpath," + odir])
    assert "every distance equal" in out and "DIFFERS" not in out


def test_searcher_consumer_kernels_on_the_host(tmp_path):
    """icp_kernels.cuh: k_corr (pclb200_correspondences, plain and reciprocal), k_fitness (getFitnessScore) and k_gicp_cov;
    normals_corr_kernels.cuh: normal shooting / back projection over k-NN rows and the surface-normal rejector;
    cluster_kernels.cuh: the union-find clustering — on the emulated block over the device-built index, against the oracle:
    correspondence lists bit for bit (gates incl. 0 and none, a descending index subset, non-finite source points, duplicated
    target points), fitness to 1e-12 in float and double, the regularised GICP covariances to 1e-9, cluster labels equal at
    five tolerances (2 ... 4 940 components)."""
    import oracle
    oracle.build()
    odir = os.path.join(ROOT, "oracle")
    out = host_program(tmp_path, "consumers_host_test.cpp", (), DEVICE_BUILD, ["-L" + odir, "-lpcl_oracle", "-Wl,-rpath," + odir])
    assert "reciprocal, index subset" in out and "GICP covariances" in out and "back projection" in out and "Euclidean clustering" in out
