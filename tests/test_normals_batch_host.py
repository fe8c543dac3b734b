"""The batch k-NN normals kernels (knn_warp.cuh: k_knn_warp_batch; search_kernels.cuh: k_normals_batch<K>, k_knn_any_batch,
k_normals_from_lists_batch) compiled for the HOST and run on emulated blocks in search.cu's launch_normals_batch sequence,
against the single kernels run set by set (tests/host/normals_batch_host_test.cpp) — CPU only; nothing runs on a GPU."""
from _sharded import host_program, needs_host_compiler

pytestmark = needs_host_compiler


def test_batch_normals_equal_single_calls(tmp_path):
    """Batches of 1, 3 and 37 sets (1, 2, 8 and 9 points, NaN and Inf records, identical points, zero extent, a planar
    cloud, frames 1e-3 and 1e4 wide far from the origin, clouds smaller than k, a repeated handle, a query set that is not
    the handle's cloud, per-set viewpoints and warp start levels) for k = 3, 8, 10, 16, 20, 32 and 40: every row and every
    set's not-dense flag byte-equal to the single kernels' on that set alone."""
    out = host_program(tmp_path, "normals_batch_host_test.cpp", timeout=1800)
    assert "B = 37: 37 sets compared" in out
