#!/bin/bash
# Re-runs the host-compiled device tests (tests/host/*_host_test.cpp) with other random scenes: PCLB_TEST_SEED perturbs
# every generator seed of the programs.  CPU only.  usage: tools/dev/fuzz_host_tests.sh <first seed> <last seed> [outdir]
set -u
ROOT=$(cd "$(dirname "$0")/../.." && pwd)
OUT=${3:-/tmp/pclb_fuzz}
mkdir -p "$OUT"
FLAGS="-O1 -std=c++17 -frounding-math -ffp-contract=off -fno-fast-math -I/usr/local/cuda/include -I$ROOT/include -I$ROOT/tests/host -I$ROOT/pcl_b200/pcl_compat"
LINK="-L$ROOT/oracle -lpcl_oracle -Wl,-rpath,$ROOT/oracle"
declare -A ARGS=([traverse]="1" [knn_warp]="1" [search]="1" [lbvh]="1" [voxel]="1" [reject]="1" [reject_sharded]="" [icp]="" [consumers]="" [lbvh_batch]="" [normals_batch]="" [fitness_batch]="" [voxel_batch]="" [loop]=""
          [shard_target]="" [shard_normals]="" [shard_cluster]="" [shard_filter]="" [shard_voxel]="" [shard_corr]="" [shard_radius]="")
for t in "${!ARGS[@]}"; do
  for variant in ref dev; do
    [ $variant = dev ] && D="-DPCLB_TEST_DEVICE_BUILD -DPCLB_HOST_EMULATION -DPCLB_HOST_EXTRA_SHIMS=\"warp_emu.h\"" || D=""
    case $t in lbvh|voxel|voxel_batch|reject|reject_sharded|shard_*) [ $variant = dev ] && continue;; consumers|lbvh_batch|normals_batch|fitness_batch|loop) [ $variant = ref ] && continue;; esac
    g++ $FLAGS $D "$ROOT/tests/host/${t}_host_test.cpp" -o "$OUT/${t}_$variant" $LINK 2> "$OUT/${t}_$variant.build.log" || { echo "BUILD FAILED $t $variant"; exit 1; }
  done
done
fail=0
for seed in $(seq "$1" "$2"); do
  for exe in "$OUT"/*_ref "$OUT"/*_dev; do
    t=$(basename "$exe"); t=${t%_*}
    if ! PCLB_TEST_SEED=$seed "$exe" ${ARGS[$t]} > "$OUT/last.log" 2>&1; then
      cp "$OUT/last.log" "$OUT/FAIL_$(basename "$exe")_seed$seed.log"
      echo "FAIL $(basename "$exe") seed $seed"
      fail=$((fail + 1))
    fi
  done
  echo "seed $seed done, failures so far: $fail"
done
echo "fuzz finished: $fail failing runs"
