// GlobalRotScaleTrans + RandomFlip3D on one row (include/bevfusion_b200.h, bevb200_lidar_aug_t), shared by the sweep
// assemblers and the box kernel.  Internal header.
//
// torch's fp32 [n, 3] @ [3, 3] on the CPU evaluates each output as the FMA chain in k order from a +0 accumulator
// (DESIGN.md section 4.29); the _rn intrinsics keep nvcc from contracting or reordering any of it.
#pragma once
#include "common.cuh"

static_assert(sizeof(bevb200_lidar_aug_t) == BEVB200_LIDAR_AUG_BYTES, "aug record layout");

namespace bevb200 {

// p @ R[:, j] for R row-major [3, 3] (rot_mat_T): fma(p2, R[2][j], fma(p1, R[1][j], fma(p0, R[0][j], +0)))
__device__ __forceinline__ float aug_chain3(float p0, float p1, float p2, const float *R, int j) {
  return __fmaf_rn(p2, R[6 + j], __fmaf_rn(p1, R[3 + j], __fmaf_rn(p0, R[j], 0.0f)));
}

// [p0, p1] @ R[:2, :2][:, j]
__device__ __forceinline__ float aug_chain2(float p0, float p1, const float *R, int j) {
  return __fmaf_rn(p1, R[3 + j], __fmaf_rn(p0, R[j], 0.0f));
}

// BasePoints.rotate(-theta), translate, scale, then LiDARPoints.flip; v[0..2] are x, y, z.  With radar, also
// RadarPoints' columns 3:5 (rotated by the 2 x 2 block, scaled, negated with the flips); v needs 5 entries then.
template <bool kRadar>
__device__ __forceinline__ void aug_point(const bevb200_lidar_aug_t &a, float *v) {
  if (!a.enabled) return;
  if (a.rot_scale_trans) {
    const float x = v[0], y = v[1], z = v[2];
#pragma unroll
    for (int j = 0; j < 3; ++j)
      v[j] = __fmul_rn(__fadd_rn(aug_chain3(x, y, z, a.point_rot, j), a.translation[j]), a.scale);
    if (kRadar) {
      const float c3 = v[3], c4 = v[4];
      v[3] = __fmul_rn(aug_chain2(c3, c4, a.point_rot, 0), a.scale);
      v[4] = __fmul_rn(aug_chain2(c3, c4, a.point_rot, 1), a.scale);
    }
  }
  if (a.flip_horizontal) {
    v[1] = -v[1];
    if (kRadar) v[4] = -v[4];
  }
  if (a.flip_vertical) {
    v[0] = -v[0];
    if (kRadar) v[3] = -v[3];
  }
}

// the record of sample b, or a disabled one when there is none
__device__ __forceinline__ bevb200_lidar_aug_t aug_record(const bevb200_lidar_aug_t *aug, int b) {
  bevb200_lidar_aug_t a;
  if (aug) {
    a = aug[b];
  } else {
    a.enabled = 0;
  }
  return a;
}

}  // namespace bevb200
