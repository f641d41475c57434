// GlobalRotScaleTrans + RandomFlip3D on the GT boxes, then ObjectRangeFilter and ObjectNameFilter
// (transforms_3d.py:195-232, 323-353, 534-636; lidar_box3d.py:140-205, base_box3d.py:148-232, utils.py:6-19) on the
// device, bit-exact to the reference's torch CPU lines, over the padded (boxes, labels, counts) of
// head_targets.pad_gt.  One CTA per sample walks its boxes in order, 256 at a time; each survivor's position is the
// CTA's running count plus its ballot rank, so the output keeps the input order with no atomics.
#include <math.h>

#include "lidar_aug.cuh"

namespace bevb200 {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxBoxes = BEVB200_HEAD_TARGETS_MAX_BOXES;
constexpr float kPi = 3.14159265358979323846f;      // fl32(np.pi): torch adds the Python float in fp32
constexpr float kTwoPi = 6.28318530717958647692f;   // fl32(2 * np.pi), limit_yaw's period

// LiDARInstance3DBoxes.rotate(theta), translate, scale, flip on one box; v[7..8] is the velocity when vel
__device__ __forceinline__ void aug_box(const bevb200_lidar_aug_t &a, float v[9], bool vel) {
  if (!a.enabled) return;
  if (a.rot_scale_trans) {
    const float x = v[0], y = v[1], z = v[2], vx = v[7], vy = v[8];
#pragma unroll
    for (int j = 0; j < 3; ++j) v[j] = aug_chain3(x, y, z, a.box_rot, j);
    v[6] = __fadd_rn(v[6], a.yaw_inc);
    if (vel) {
      v[7] = aug_chain2(vx, vy, a.box_rot, 0);
      v[8] = aug_chain2(vx, vy, a.box_rot, 1);
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) v[j] = __fadd_rn(v[j], a.translation[j]);
#pragma unroll
    for (int c = 0; c < 6; ++c) v[c] = __fmul_rn(v[c], a.scale);   // tensor[:, :6] *= scale
    v[7] = __fmul_rn(v[7], a.scale);                                 // tensor[:, 7:] *= scale
    v[8] = __fmul_rn(v[8], a.scale);
  }
  if (a.flip_horizontal) {   // tensor[:, 1::7] = -tensor[:, 1::7]; yaw = -yaw + pi
    v[1] = -v[1];
    v[8] = -v[8];
    v[6] = __fadd_rn(-v[6], kPi);
  }
  if (a.flip_vertical) {     // tensor[:, 0::7] = -tensor[:, 0::7]; yaw = -yaw
    v[0] = -v[0];
    v[7] = -v[7];
    v[6] = -v[6];
  }
}

__global__ void __launch_bounds__(kThreads)
box_aug_kernel(const float *__restrict__ boxes, const int32_t *__restrict__ labels, const int32_t *__restrict__ counts,
               int nmax, int D, const bevb200_lidar_aug_t *__restrict__ aug, float4 range, int num_classes,
               float *__restrict__ out_boxes, int32_t *__restrict__ out_labels, int32_t *__restrict__ out_counts,
               int32_t *__restrict__ status) {
  __shared__ int warp_sum[kThreads / 32];
  const int b = blockIdx.x;
  const bevb200_lidar_aug_t a = aug_record(aug, b);
  const int given = counts[b], n = min(max(given, 0), nmax);
  if (threadIdx.x == 0 && n != given) atomicOr(status, BEVB200_BOX_AUG_BAD_COUNT);
  const float *src = boxes + (size_t)b * nmax * D;
  float *dst = out_boxes + (size_t)b * nmax * D;
  const int32_t *lab = labels + (size_t)b * nmax;
  int32_t *dlab = out_labels + (size_t)b * nmax;
  const bool vel = D == 9;
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  int off = 0;
  for (int base = 0; base < n; base += kThreads) {
    const int i = base + threadIdx.x;
    float v[9];
    int label = 0;
    bool keep = false;
    if (i < n) {
#pragma unroll
      for (int c = 0; c < 9; ++c) v[c] = c < D ? src[(size_t)i * D + c] : 0.0f;
      label = lab[i];
      aug_box(a, v, vel);
      // ObjectRangeFilter: strict fp32 in_range_bev (NaN fails), then limit_yaw(0.5, 2 pi); ObjectNameFilter
      keep = v[0] > range.x && v[1] > range.y && v[0] < range.z && v[1] < range.w && label >= 0 &&
             label < num_classes;
      v[6] = __fsub_rn(v[6], __fmul_rn(floorf(__fadd_rn(__fdiv_rn(v[6], kTwoPi), 0.5f)), kTwoPi));
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_sum[warp] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
      before += w < warp ? warp_sum[w] : 0;
      total += warp_sum[w];
    }
    if (keep) {
      const int pos = off + before + __popc(m & ((1u << lane) - 1));
#pragma unroll
      for (int c = 0; c < 9; ++c)
        if (c < D) dst[(size_t)pos * D + c] = v[c];
      dlab[pos] = label;
    }
    off += total;
    __syncthreads();
  }
  for (size_t k = (size_t)off * D + threadIdx.x; k < (size_t)nmax * D; k += kThreads) dst[k] = 0.0f;
  for (int k = off + threadIdx.x; k < nmax; k += kThreads) dlab[k] = 0;
  if (threadIdx.x == 0) out_counts[b] = off;
}

bool overlap(const void *a, const void *b, size_t bytes) {
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return bytes && x < y + bytes && y < x + bytes;
}

}  // namespace
}  // namespace bevb200

using namespace bevb200;

extern "C" {

int bevb200_box_aug(const float *boxes, const int32_t *labels, const int32_t *counts, int batch, int nmax, int box_dim,
                    const bevb200_lidar_aug_t *aug, float range_x_min, float range_y_min, float range_x_max,
                    float range_y_max, int num_classes, float *out_boxes, int32_t *out_labels, int32_t *out_counts,
                    int32_t *status, void *stream) {
  BEVB200_REQUIRE(batch >= 0 && batch <= 65535 && nmax >= 0 && nmax <= kMaxBoxes,
                  "sizes out of range (0 <= batch <= 65535, 0 <= nmax <= BEVB200_HEAD_TARGETS_MAX_BOXES)");
  BEVB200_REQUIRE(box_dim == 7 || box_dim == 9, "box_dim must be 7 or 9");
  BEVB200_REQUIRE(num_classes >= 0, "num_classes must not be negative");
  BEVB200_REQUIRE(status, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (batch == 0) {
    BEVB200_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
    return BEVB200_OK;
  }
  BEVB200_REQUIRE(counts && out_counts && (nmax == 0 || (boxes && labels && out_boxes && out_labels)),
                  "null pointer");
  BEVB200_REQUIRE((uintptr_t)aug % alignof(bevb200_lidar_aug_t) == 0, "misaligned augmentation records");
  const size_t box_bytes = (size_t)batch * nmax * box_dim * sizeof(float), label_bytes = (size_t)batch * nmax * 4;
  BEVB200_REQUIRE(!overlap(boxes, out_boxes, box_bytes) && !overlap(labels, out_labels, label_bytes),
                  "the outputs overlap the inputs");
  BEVB200_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
  BEVB200_LAUNCH(box_aug_kernel, batch, kThreads, 0, st, boxes, labels, counts, nmax, box_dim, aug,
                 make_float4(range_x_min, range_y_min, range_x_max, range_y_max), num_classes, out_boxes, out_labels,
                 out_counts, status);
  return BEVB200_OK;
}

}  // extern "C"
