#!/bin/bash
# The host-compiled device kernels under several THREAD SCHEDULES of the block emulation (PCLB_EMU_ORDER: ascending thread
# index, descending, and fixed strided permutations).  A kernel that is only correct under one order — a missing __syncthreads /
# __syncwarp between one thread's write and another's read of shared or global memory — produces different results under the
# others and fails its checks; removing the first barrier of block_reduce_and_publish is caught by two of three orders.
# usage: tools/dev/racecheck_host_kernels.sh [workdir]
set -u
ROOT=$(cd "$(dirname "$0")/../.." && pwd)
W=${1:-/tmp/pclb_racecheck}
mkdir -p "$W" && cd "$W"
FL="-O1 -std=c++17 -frounding-math -ffp-contract=off -fno-fast-math -I/usr/local/cuda/include -I$ROOT/include -I$ROOT/tests/host -I$ROOT/pcl_b200/pcl_compat"
DEV='-DPCLB_TEST_DEVICE_BUILD -DPCLB_HOST_EMULATION -DPCLB_HOST_EXTRA_SHIMS=\"warp_emu.h\"'
LINK="-L$ROOT/oracle -lpcl_oracle -Wl,-rpath,$ROOT/oracle"
bad=0
for t in lbvh lbvh_batch normals_batch fitness_batch loop traverse search knn_warp icp icp_batch_targets consumers voxel voxel_batch reject reject_sharded shard_target shard_normals shard_cluster shard_filter shard_voxel shard_corr shard_radius; do
  case $t in lbvh|voxel|voxel_batch|reject|reject_sharded|shard_*) D="";; *) D=$DEV;; esac
  eval g++ $FL $D "$ROOT/tests/host/${t}_host_test.cpp" -o r_$t $LINK 2> build_$t.log || { echo "BUILD FAILED $t"; bad=1; continue; }
  case $t in icp|icp_batch_targets|lbvh_batch|normals_batch|fitness_batch|loop|consumers|shard_*) args="";; *) args="1";; esac
  line="$t:"
  for order in "" reverse 3 7 123; do
    if PCLB_EMU_ORDER=$order ./r_$t $args > run_${t}_${order:-ascending}.log 2>&1; then line="$line ${order:-ascending}=ok"; else line="$line ${order:-ascending}=FAILED"; bad=1; fi
  done
  echo "$line"
done
[ $bad -eq 0 ] && echo "every program passes under all five schedules" || echo "PROBLEMS — see $W"
