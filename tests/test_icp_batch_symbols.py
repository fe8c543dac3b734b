"""CPU-side checks of the batch extension of the C-ABI (include/pclb200_batch.h): its header, the ctypes binding and the
library agree, it declares nothing include/pclb200.h or include/pclb200_sharded.h already does, and it compiles alone in
a C translation unit.  No compute calls."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared(name):
    h = open(os.path.join(ROOT, "include", name)).read()
    return sorted(set(re.findall(r"PCLB200_API\s+[\w\s\*]+?\b(pclb200_\w+)\s*\(", h)))


@pytest.fixture(scope="module")
def built():
    from pcl_b200 import build
    return build.build()


def test_batch_header_and_binding_agree():
    import pcl_b200
    assert _declared("pclb200_batch.h") == sorted(pcl_b200.BATCH_SYMBOLS)
    assert not set(_declared("pclb200_batch.h")) & set(_declared("pclb200.h"))
    assert not set(_declared("pclb200_batch.h")) & set(_declared("pclb200_sharded.h"))


def test_library_exports_the_batch_symbols(built):
    out = subprocess.check_output(["nm", "-D", "--defined-only", built], text=True)
    exported = set(re.findall(r"\bT (pclb200_\w+)", out))
    missing = [s for s in _declared("pclb200_batch.h") if s not in exported]
    assert not missing, missing
    import pcl_b200
    pcl_b200.lib()  # binds and checks every symbol of the three headers


def test_batch_header_compiles_as_c(tmp_path):
    """The extension header stands on its own in a C translation unit (it includes pclb200.h itself)."""
    src = tmp_path / "use.c"
    src.write_text('#include "pclb200_batch.h"\n'
                   "int (*f)(pclb200_icp*, const void*, size_t, size_t, const void*, size_t, const int64_t*, int32_t, "
                   "const double*) = pclb200_icp_set_source_batch;\n"
                   "int (*g)(pclb200_icp*, int, pclb200_icp_stats*) = pclb200_icp_iterate_batch;\n"
                   "int (*h)(pclb200_icp*, pclb200_corr*, int64_t*) = pclb200_icp_get_correspondences_batch;\n")
    subprocess.check_call(["gcc", "-std=c99", "-c", "-I" + os.path.join(ROOT, "include"), str(src), "-o",
                           str(tmp_path / "use.o")])
