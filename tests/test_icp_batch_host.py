"""The batch ICP kernels (icp_kernels.cuh: k_search_batch, k_accum_dmma_batch, k_accum_batch, k_solve_batch over
batch_blocks's table) compiled for the HOST and run on emulated thread blocks against the single-problem kernels on each
problem alone (tests/host/icp_batch_host_test.cpp) — CPU only; nothing runs on a GPU."""
from _sharded import host_program, needs_host_compiler

pytestmark = needs_host_compiler


def test_batch_kernels_equal_single_problem_kernels(tmp_path):
    """1, 3 and 7 problems (1- and 2-point problems, sizes off multiples of 32 and 256), SVD, point-to-plane and symmetric,
    float and double, tracking off / on / auto: the block tables cover each problem's grid exactly once, and after every
    iteration each problem's matches, queries, accumulators, loop state, pending transform and solve output are byte-equal
    to its single run; so are the final transforms."""
    out = host_program(tmp_path, "icp_batch_host_test.cpp", timeout=1800)
    assert out.count("B = 7") == 18
