"""The batch fitness score kernels (icp_kernels.cuh: k_transform_batch, k_fitness_batch) compiled for the HOST and run on
emulated blocks in icp.cu's fitness_batch sequence, against k_fitness run problem by problem as fitness_score runs it
(tests/host/fitness_batch_host_test.cpp) — CPU only; nothing runs on a GPU."""
from _sharded import host_program, needs_host_compiler

pytestmark = needs_host_compiler


def test_batch_fitness_sums_equal_single_calls(tmp_path):
    """Batches of 1, 3 and 37 problems (1, 255, 256 and 257 points, a problem whose grid is capped, NaN and Inf records,
    an all-NaN problem, a problem moved beyond max_range, targets shared by several problems) in the fitness and the
    validation operation orders, float and double, with max_range = DBL_MAX, 2e-3 and 0: every problem's accumulators
    and counter byte-equal to the single kernel's on that problem alone."""
    out = host_program(tmp_path, "fitness_batch_host_test.cpp", timeout=1800)
    assert "B = 37: 37 problems compared" in out
