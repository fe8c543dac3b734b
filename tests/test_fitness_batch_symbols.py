"""CPU-side check of pclb200_fitness_score_batch, pclb200_validate_transformation_batch and
pclb200_icp_fitness_score_batch (include/pclb200_batch.h): their declarations compile in a C translation unit with the
signatures the ctypes binding uses.  No compute calls."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["pclb200_fitness_score_batch", "pclb200_validate_transformation_batch", "pclb200_icp_fitness_score_batch"]


def test_fitness_batch_declarations_compile_as_c(tmp_path):
    src = tmp_path / "use.c"
    score = ("int (*{})(pclb200_ctx*, const pclb200_index* const*, int32_t, const void*, size_t, size_t, const int64_t*, "
             "const double*, int, double, double*) = {};\n")
    src.write_text('#include "pclb200_batch.h"\n'
                   + score.format("f", "pclb200_fitness_score_batch")
                   + score.format("v", "pclb200_validate_transformation_batch")
                   + "int (*s)(pclb200_icp*, double, double*) = pclb200_icp_fitness_score_batch;\n")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-c", "-I" + os.path.join(ROOT, "include"), str(src),
                           "-o", str(tmp_path / "use.o")])


def test_binding_declares_fitness_batch():
    import pcl_b200
    for name in NAMES:
        assert name in pcl_b200.BATCH_SYMBOLS
