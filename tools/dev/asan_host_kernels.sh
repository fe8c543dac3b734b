#!/bin/bash
# The host-compiled DEVICE kernels (tests/host/*_host_test.cpp, on the device-built index) under -fsanitize=address,undefined:
# every global-memory access of the kernels goes to a std::vector of the test, so an out-of-bounds read or write, a misaligned
# access, a signed overflow or an invalid shift in the device code is reported — a memcheck of the kernels without a GPU.
# usage: tools/dev/asan_host_kernels.sh [workdir]
set -u
ROOT=$(cd "$(dirname "$0")/../.." && pwd)
W=${1:-/tmp/pclb_asan_kernels}
mkdir -p "$W" && cd "$W"
FL="-O1 -g -std=c++17 -frounding-math -ffp-contract=off -fno-fast-math -fsanitize=address,undefined -fno-omit-frame-pointer -I/usr/local/cuda/include -I$ROOT/include -I$ROOT/tests/host -I$ROOT/pcl_b200/pcl_compat"
DEV='-DPCLB_TEST_DEVICE_BUILD -DPCLB_HOST_EMULATION -DPCLB_HOST_EXTRA_SHIMS=\"warp_emu.h\"'
LINK="-L$ROOT/oracle -lpcl_oracle -Wl,-rpath,$ROOT/oracle"
export ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0 UBSAN_OPTIONS=print_stacktrace=1:halt_on_error=0
bad=0
for t in lbvh lbvh_batch normals_batch fitness_batch loop traverse search knn_warp icp icp_batch_targets consumers voxel voxel_batch reject reject_sharded shard_target shard_normals shard_cluster shard_filter shard_voxel shard_corr shard_radius; do
  case $t in lbvh|voxel|voxel_batch|reject|reject_sharded|shard_*) D="";; *) D=$DEV;; esac
  eval g++ $FL $D "$ROOT/tests/host/${t}_host_test.cpp" -o k_$t $LINK 2> build_$t.log || { echo "BUILD FAILED $t"; tail -5 build_$t.log; bad=1; continue; }
  case $t in icp|icp_batch_targets|lbvh_batch|normals_batch|fitness_batch|loop|consumers|shard_*) args="";; *) args="1";; esac
  ./k_$t $args > run_$t.log 2>&1
  rc=$?
  reports=$(grep -c -i -E "AddressSanitizer|runtime error" run_$t.log)
  echo "$t: exit $rc, $(grep -E 'checks, [0-9]+ failures' run_$t.log | tail -1), sanitizer reports: $reports"
  [ $rc -ne 0 ] || [ "$reports" -ne 0 ] && bad=1
done
[ $bad -eq 0 ] && echo "all kernel programs clean under ASan + UBSan" || echo "PROBLEMS — see $W/run_*.log"
