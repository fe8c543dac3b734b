"""The batch index build (lbvh_kernels.cuh: the *_batch kernels, in lbvh.cu's build_index_batch sequence) compiled for the
HOST and run on emulated thread blocks against the single build of each cloud alone (tests/host/lbvh_batch_host_test.cpp)
— CPU only; nothing runs on a GPU."""
from _sharded import host_program, needs_host_compiler

pytestmark = needs_host_compiler


def test_batch_build_equals_single_builds(tmp_path):
    """Batches of 1, 3 and 37 clouds (1, 8 and 9 points, 255 and 256 finite points, NaN and Inf records, identical points,
    zero-extent and planar frames, frames 1e-3 and 1e4 wide far from the origin): every handle's counts, frame, points,
    nodes, leaf ranges and cell-table shape are byte-equal to its cloud's single build, and its cell-table entries equal
    as a set."""
    out = host_program(tmp_path, "lbvh_batch_host_test.cpp", timeout=1800)
    assert "B = 37: 37 clouds compared" in out
