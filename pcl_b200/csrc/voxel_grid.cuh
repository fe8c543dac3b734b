// voxel_grid.cuh — what the VoxelGrid kernels (voxel_kernels.cuh) and the VoxelGrid of a sharded map
// (shard_voxel_kernels.cuh) share without defining a kernel: the min / max accumulator, the grid rule, the voxel of a point
// and the run of a voxel.  A header of its own so that two translation units can include it (the kernels of
// voxel_kernels.cuh are defined once, in voxel.cu).
#pragma once
#include <cmath>
#include <limits>

#include "internal.cuh"

namespace pclb200 {

struct MinMaxAcc {
  int lo[3];
  int hi[3];
  unsigned long long count;
};

__device__ __forceinline__ int vf2ord(float f)
{
  int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
static inline float vord2f(int i)
{
  int j = i >= 0 ? i : i ^ 0x7fffffff;
  float f;
  memcpy(&f, &j, 4);
  return f;
}

struct VgParams {
  float inv[3];
  int min_b[3];
  int mul[3];
};

// The grid of the box [mn, mx] (voxel_grid.hpp:617-644) in the reference's float arithmetic: inverse leaf, min_b and the
// key multipliers.  False when the int32 guard of :620-629 trips.  The one copy of the grid rule: voxelgrid() (voxel.cu)
// takes it over its own points' box, voxelgrid_sharded() (shard_voxel.cu) over the union of every rank's box.
constexpr const char* kVgLeafTooSmall =
    "VoxelGrid: leaf size is too small for the input dataset, integer indices would overflow (voxel_grid.hpp:620-629)";
inline bool vg_grid(const float mn[3], const float mx[3], const float leaf[3], VgParams& gp)
{
  float inv[3];
  for (int d = 0; d < 3; ++d)
    inv[d] = 1.0f / leaf[d];  // inverse_leaf_size_ = 1 / leaf_size_ (voxel_grid.h:266,282)
  volatile float e0 = (mx[0] - mn[0]) * inv[0], e1 = (mx[1] - mn[1]) * inv[1], e2 = (mx[2] - mn[2]) * inv[2];
  const int64_t dx = (int64_t)e0 + 1, dy = (int64_t)e1 + 1, dz = (int64_t)e2 + 1;
  if (dx * dy * dz > (int64_t)std::numeric_limits<int32_t>::max())
    return false;
  int div_b[3];
  for (int d = 0; d < 3; ++d) {
    volatile float lo_s = mn[d] * inv[d], hi_s = mx[d] * inv[d];
    gp.inv[d] = inv[d];
    gp.min_b[d] = (int)std::floor(lo_s);
    div_b[d] = (int)std::floor(hi_s) - gp.min_b[d] + 1;
  }
  gp.mul[0] = 1;
  gp.mul[1] = div_b[0];
  gp.mul[2] = div_b[0] * div_b[1];
  return true;
}

// voxel coordinate of a finite point on one axis (voxel_grid.hpp:705-719): non-decreasing in v, so the voxels of the
// points of a box lie between the coordinates of its faces
__device__ __forceinline__ int vg_ijk(float v, float inv, int min_b)
{
  return (int)(floorf(__fmul_rn(v, inv)) - (float)min_b);
}
// linear index of a voxel: ijk . mul, in int
__device__ __forceinline__ unsigned vg_linear(int ijk0, int ijk1, int ijk2, const VgParams& g)
{
  return (unsigned)(ijk0 * g.mul[0] + ijk1 * g.mul[1] + ijk2 * g.mul[2]);
}

struct RunRef {
  unsigned begin, end;
};

}  // namespace pclb200
