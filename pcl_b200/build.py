"""Builds pcl_b200/libpclb200.so in-tree with nvcc for sm_90a (H100) (cross-compiles without a GPU).

    python -m pcl_b200.build [--force] [--verbose]

-fmad=false: device arithmetic must round like the reference's scalar C++ (no fused multiply-add), because
parity with the CPU path is bit-exact for indices and distances (see DESIGN.md "numerics").
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
SO = os.path.join(HERE, "libpclb200.so")
SOURCES = ["alloc.cu", "lbvh.cu", "search.cu", "icp.cu", "voxel.cu", "reject.cu", "normals_corr.cu", "cluster.cu", "comm.cu", "shard_normals.cu", "shard_cluster.cu", "shard_filter.cu", "shard_voxel.cu", "capi.cu"]
HEADERS = ["internal.cuh", "traverse.cuh", "knn_warp.cuh", "search_kernels.cuh", "lbvh_kernels.cuh", "voxel_grid.cuh", "voxel_kernels.cuh", "reject_kernels.cuh", "reject_sharded_kernels.cuh", "normals_corr_kernels.cuh", "cluster_kernels.cuh", "union_find.cuh", "icp_kernels.cuh", "grid_sum.cuh", "shard_target_kernels.cuh", "shard_normals_kernels.cuh", "shard_cluster_kernels.cuh", "shard_filter_kernels.cuh", "shard_voxel_kernels.cuh", "corr_select.cuh", "solve_body.inc", "assemble_body.inc", "karras_points_body.inc", "mark_cells_body.inc", "link_cells_body.inc", "knn_warp_body.inc", "normals_body.inc", "knn_any_body.inc", "normals_from_lists_body.inc", "fitness_body.inc", "peer_exchange.cuh", "peer_tables.cuh", os.path.join("..", "..", "include", "pclb200.h"), os.path.join("..", "..", "include", "pclb200_sharded.h"), os.path.join("..", "..", "include", "pclb200_batch.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = GENCODE + ["-lineinfo", "-O3", "-std=c++17", "-fmad=false",
                   "-Xcompiler", "-fPIC,-fvisibility=hidden", "-Xptxas", "-v", "--expt-relaxed-constexpr",
                   "-ccbin", "/usr/bin/g++"]


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, leaf=None, tag=None, defines=()):
    """leaf/tag: build an experimental variant (libpclb200_<tag>.so with -DPCLB_LEAF=<leaf>) next to the default."""
    global OBJ, SO
    flags = list(FLAGS)
    if tag:
        OBJ = os.path.join(HERE, "build_" + tag)
        SO = os.path.join(HERE, f"libpclb200_{tag}.so")
    if leaf:
        flags += [f"-DPCLB_LEAF={int(leaf)}"]
    flags += [f"-D{d}" for d in defines]
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.normpath(os.path.join(CSRC, h)) for h in HEADERS]
    jobs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s.replace(".cu", ".o"))
        if force or _newer(obj, [src] + hdrs):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        r = subprocess.run([NVCC] + flags + ["-c", src, "-o", obj], capture_output=True, text=True)
        if verbose or r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
        else:
            with open(obj + ".ptxas.log", "w") as f:
                f.write(r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed on " + src)
        return obj

    with ThreadPoolExecutor(max_workers=min(6, os.cpu_count() or 1)) as ex:
        list(ex.map(compile_one, jobs))
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _newer(SO, objs):
        r = subprocess.run([NVCC, "-shared", "-o", SO] + objs + GENCODE + [
                           "-ccbin", "/usr/bin/g++", "-Xcompiler", "-fPIC", "-ldl"], capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return SO


if __name__ == "__main__":
    kw = {}
    for a in sys.argv[1:]:
        if a.startswith("--leaf="):
            kw["leaf"] = int(a.split("=")[1])
        if a.startswith("--tag="):
            kw["tag"] = a.split("=")[1]
        if a.startswith("--define="):
            kw.setdefault("defines", []).append(a.split("=", 1)[1])
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv, **kw))
