"""CPU-side check of pclb200_voxelgrid_batch (include/pclb200_batch.h): its declaration compiles in a C translation unit
with the signature the ctypes binding uses.  No compute calls."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_voxelgrid_batch_compiles_as_c(tmp_path):
    src = tmp_path / "use.c"
    src.write_text('#include "pclb200_batch.h"\n'
                   "int (*f)(pclb200_ctx*, const void*, size_t, size_t, const int64_t*, int32_t, const float*, unsigned, "
                   "const void*, size_t, float*, float*, int64_t*) = pclb200_voxelgrid_batch;\n")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-c", "-I" + os.path.join(ROOT, "include"), str(src),
                           "-o", str(tmp_path / "use.o")])


def test_binding_declares_voxelgrid_batch():
    import pcl_b200
    assert "pclb200_voxelgrid_batch" in pcl_b200.BATCH_SYMBOLS
