"""The batch VoxelGrid kernels (voxel_kernels.cuh: k_vg_keys_batch, k_vg_heads_batch, k_vg_offsets_batch; lbvh_kernels.cuh:
k_bbox_batch) compiled for the HOST and run on emulated blocks in voxel.cu's voxelgrid_batch sequence, with the single
call's run, filter and reduce kernels, against the oracle's VoxelGrid of each cloud alone
(tests/host/voxel_batch_host_test.cpp) — CPU only; nothing runs on a GPU."""
import os

from _sharded import ROOT, host_program, needs_host_compiler

pytestmark = needs_host_compiler


def test_batch_voxelgrid_equals_each_cloud_alone(tmp_path):
    """Batches of 1, 3 and 37 clouds (two clouds with identical coordinates, NaN and Inf records, an all-NaN cloud, one
    point, a cloud the minimum empties, a zero-extent axis, points on voxel faces, a cloud 1e4 away) for fine, coarse and
    anisotropic leaves and min_points_per_voxel 0, 1 and 3, xyz1 and PointNormal records: every cloud's count, rows and
    normal / curvature rows byte-equal to the oracle's VoxelGrid of that cloud alone; the guard names the first cloud
    that trips it."""
    import oracle
    oracle.build()
    odir = os.path.join(ROOT, "oracle")
    out = host_program(tmp_path, "voxel_batch_host_test.cpp", (), (), ["-L" + odir, "-lpcl_oracle", "-Wl,-rpath," + odir],
                       timeout=1800)
    assert "B = 37: 37 clouds compared" in out and "PointNormal, overflow guard" in out and "cloud 2 trips the guard" in out
