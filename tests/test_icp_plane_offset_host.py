"""The point-to-plane accumulation's one-record rows (icp_kernels.cuh: pair_rows, k_accum_dmma) compiled for the HOST and
run on an emulated thread block (tests/host/icp_plane_offset_host_test.cpp) — CPU only; nothing runs on a GPU."""
from _sharded import host_program, needs_host_compiler

pytestmark = needs_host_compiler


def test_point_to_plane_rows_from_one_record_equal_the_two_gathers(tmp_path):
    """Target normals with plane_offset in w, on a target with NaN and infinite normal components and an index with
    padding slots: every row equals the row of the matched point and its normal bit for bit, the two accumulations are
    bit-identical and equal plain fp64 sums; the one-record run reads no target point."""
    out = host_program(tmp_path, "icp_plane_offset_host_test.cpp")
    assert "point-to-plane rows from one record" in out
