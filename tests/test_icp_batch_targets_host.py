"""The batch ICP kernels with one target per problem (icp_kernels.cuh: k_search_batch, k_accum_dmma_batch, k_accum_batch
with a BatchTarget table, k_solve_batch with each target's rmax; lbvh_kernels.cuh: k_problem_frame_keys) compiled for the
HOST and run on emulated thread blocks against the single-problem kernels on each problem against its own target
(tests/host/icp_batch_targets_host_test.cpp) — CPU only; nothing runs on a GPU."""
from _sharded import host_program, needs_host_compiler

pytestmark = needs_host_compiler


def test_batch_of_targets_equals_single_problem_kernels(tmp_path):
    """1, 3 and 7 problems over three targets whose boxes differ by orders of magnitude, SVD, point-to-plane and
    symmetric, float and double, tracking off / on / auto: each problem's query keys and order are k_stage_records's in
    its own target's frame, and after every iteration its matches, queries, accumulators, loop state, pending transform
    and solve output are byte-equal to its single run against its own target; so are the final transforms."""
    out = host_program(tmp_path, "icp_batch_targets_host_test.cpp", timeout=1800)
    assert out.count("B = 7") == 18
