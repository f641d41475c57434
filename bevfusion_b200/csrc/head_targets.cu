// Heatmap training targets of CenterHead and TransFusionHead on the device (the semantics of
// models/heads/bbox/centerpoint.py:432-582 get_targets_single, the heatmap block of transfusion.py:526-573, and
// core/utils/gaussian.py), with no per-object host loop.
//
// Three launches per call, whatever B and the box counts are:
//   head_targets_zero_kernel    zeroes the heatmap and the status word
//   head_targets_assign_kernel  one CTA per sample: label -> (task, channel) through the caller's table, the
//                               CenterHead slot order (by class in task order, then by original index), the fp32
//                               size / radius / centre arithmetic of the reference, one draw record per object,
//                               and for CenterHead anno_box / ind / mask of every slot
//   head_targets_draw_kernel    one CTA per draw record: the (2r+1)^2 window clipped to the map, the gaussian in
//                               double rounded to fp32, applied with atomicMax on the int bits (values >= 0, so the
//                               max is exact in any order and the heatmap is bit-reproducible)
// The fp32 arithmetic uses explicit round-to-nearest intrinsics: no FMA contraction, one rounding per op in the
// reference's order.
#include <float.h>

#include "common.cuh"

namespace bevb200 {
namespace {

constexpr int kMaxBoxes = BEVB200_HEAD_TARGETS_MAX_BOXES;
constexpr int kMaxLabels = BEVB200_HEAD_TARGETS_MAX_LABELS;
constexpr int kMaxTasks = BEVB200_HEAD_TARGETS_MAX_TASKS;
constexpr int kAssignThreads = 256;
constexpr int kDrawThreads = 128;
constexpr int kZeroThreads = 256;
// int(radius) must fit an int32 with room for centre +- radius; larger radii are counted in status and skipped.
constexpr float kMaxRadius = 1073741824.f;   // 2^30

struct HeadParams {
  int B, nmax, box_dim, anno_dim, mode, num_labels, num_tasks;
  int fmap_x, fmap_y, min_radius, max_objs, norm_bbox;
  float pc_x, pc_y, vs_x, vs_y, osf;
  // gaussian_overlap's Python constants, each rounded to fp32 where it meets a tensor (gaussian.py:55-84)
  float one_minus, one_plus, b3k, c3k, a3x4;
  int table[kMaxLabels];        // task << 16 | channel, or -1: the label belongs to no task
  int plane0[kMaxTasks];        // first heatmap plane of each task: B * (classes of the earlier tasks)
  int ncls[kMaxTasks];
};

// gaussian_radius((height, width), min_overlap) in fp32, op for op (gaussian.py:55-84); Python's min(r1, r2, r3).
__device__ __forceinline__ float gaussian_radius_f32(float height, float width, const HeadParams &p) {
  const float hw = __fadd_rn(height, width);
  const float b1 = hw;
  const float c1 = __fdiv_rn(__fmul_rn(__fmul_rn(width, height), p.one_minus), p.one_plus);
  const float r1 = __fdiv_rn(__fadd_rn(b1, __fsqrt_rn(__fsub_rn(__fmul_rn(b1, b1), __fmul_rn(4.f, c1)))), 2.f);
  const float b2 = __fmul_rn(2.f, hw);
  const float c2 = __fmul_rn(__fmul_rn(p.one_minus, width), height);
  const float r2 = __fdiv_rn(__fadd_rn(b2, __fsqrt_rn(__fsub_rn(__fmul_rn(b2, b2), __fmul_rn(16.f, c2)))), 2.f);
  const float b3 = __fmul_rn(p.b3k, hw);
  const float c3 = __fmul_rn(__fmul_rn(p.c3k, width), height);
  const float r3 = __fdiv_rn(__fadd_rn(b3, __fsqrt_rn(__fsub_rn(__fmul_rn(b3, b3), __fmul_rn(p.a3x4, c3)))), 2.f);
  float r = r1;
  if (r2 < r) r = r2;
  if (r3 < r) r = r3;
  return r;
}

__global__ void __launch_bounds__(kZeroThreads)
    head_targets_zero_kernel(float *__restrict__ heatmap, long long n, int32_t *__restrict__ status) {
  if (blockIdx.x == 0 && threadIdx.x == 0) *status = 0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (((uintptr_t)heatmap & 15) == 0) {
    const long long n4 = n >> 2;
    for (long long j = i; j < n4; j += stride) reinterpret_cast<float4 *>(heatmap)[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long j = (n4 << 2) + i; j < n; j += stride) heatmap[j] = 0.f;
  } else {
    for (long long j = i; j < n; j += stride) heatmap[j] = 0.f;
  }
}

__global__ void __launch_bounds__(kAssignThreads)
    head_targets_assign_kernel(const float *__restrict__ boxes, const int32_t *__restrict__ labels,
                               const int32_t *__restrict__ counts, const __grid_constant__ HeadParams p,
                               float *__restrict__ anno, int64_t *__restrict__ ind, uint8_t *__restrict__ mask,
                               int4 *__restrict__ rec, int32_t *__restrict__ status) {
  __shared__ int key[kMaxBoxes];
  const int b = blockIdx.x, tid = threadIdx.x;
  int n = counts ? counts[b] : p.nmax;
  n = n < 0 ? 0 : (n > p.nmax ? p.nmax : n);
  const bool center = p.mode == BEVB200_HEAD_TARGETS_CENTERHEAD;
  for (int i = tid; i < n; i += kAssignThreads) {
    const int l = labels[(long long)b * p.nmax + i];
    key[i] = (l >= 0 && l < p.num_labels) ? p.table[l] : -1;
  }
  if (center) {   // every slot of this sample starts empty
    for (int t = 0; t < p.num_tasks; ++t) {
      const long long s0 = ((long long)t * p.B + b) * p.max_objs;
      for (long long e = tid; e < (long long)p.max_objs * p.anno_dim; e += kAssignThreads) anno[s0 * p.anno_dim + e] = 0.f;
      for (int s = tid; s < p.max_objs; s += kAssignThreads) {
        ind[s0 + s] = 0;
        mask[s0 + s] = 0;
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < p.nmax; i += kAssignThreads) {
    int4 r = make_int4(0, 0, 0, -1);
    const int k = i < n ? key[i] : -1;
    bool live = i < n && (k >= 0 || !center);
    int slot = i;
    if (live && center) {
      // task_masks / torch.cat(task_box) (centerpoint.py:463-486): by class in task order, then by index
      const int t = k >> 16, c = k & 0xffff;
      slot = 0;
      for (int j = 0; j < n; ++j) {
        const int kj = key[j];
        slot += kj >= 0 && (kj >> 16) == t && ((kj & 0xffff) < c || (kj == k && j < i));
      }
      live = slot < p.max_objs;   // num_objs = min(len(task_boxes), max_objs)
    }
    if (live) {
      const float *bx = boxes + ((long long)b * p.nmax + i) * p.box_dim;
      const float width = __fdiv_rn(__fdiv_rn(bx[3], p.vs_x), p.osf);
      const float length = __fdiv_rn(__fdiv_rn(bx[4], p.vs_y), p.osf);
      if (width > 0.f && length > 0.f) {   // false for NaN
        const float rf = gaussian_radius_f32(length, width, p);
        if (!(rf >= 0.f && rf < kMaxRadius) || k < 0) {
          // int(radius) raises on inf / NaN; TransFusion would wrap or raise on the label (heatmap[label])
          atomicAdd(status, 1);
        } else {
          const int radius = max(p.min_radius, (int)rf);
          const float coor_x = __fdiv_rn(__fdiv_rn(__fsub_rn(bx[0], p.pc_x), p.vs_x), p.osf);
          const float coor_y = __fdiv_rn(__fdiv_rn(__fsub_rn(bx[1], p.pc_y), p.vs_y), p.osf);
          if (isfinite(coor_x) && isfinite(coor_y)) {
            const int cx = __float2int_rz(coor_x), cy = __float2int_rz(coor_y);
            const int t = k >> 16, c = k & 0xffff;
            const int plane = p.plane0[t] + b * p.ncls[t] + c;
            if (!center) {
              r = make_int4(plane, cx, cy, radius);
            } else if (cx >= 0 && cx < p.fmap_x && cy >= 0 && cy < p.fmap_y) {
              r = make_int4(plane, cx, cy, radius);
              const long long s = ((long long)t * p.B + b) * p.max_objs + slot;
              ind[s] = (int64_t)cx * p.fmap_y + cy;
              mask[s] = 1;
              float *a = anno + s * p.anno_dim;
              a[0] = __fsub_rn(coor_x, (float)cx);
              a[1] = __fsub_rn(coor_y, (float)cy);
              a[2] = __fadd_rn(bx[2], __fmul_rn(bx[5], 0.5f));   // gravity centre z
#pragma unroll
              for (int d = 0; d < 3; ++d) a[3 + d] = p.norm_bbox ? logf(bx[3 + d]) : bx[3 + d];
              float sn, cs;
              sincosf(bx[6], &sn, &cs);
              a[6] = sn;
              a[7] = cs;
              if (p.anno_dim == 10) {
                a[8] = bx[7];
                a[9] = bx[8];
              }
            }
          }
        }
      }
    }
    rec[(long long)b * p.nmax + i] = r;
  }
}

// Record (plane, row, col, radius): the window rows [row - r, row + r] x cols [col - r, col + r] clipped to the
// [height, width] map, which is what draw_heatmap_gaussian's slicing draws (gaussian.py:24-52), also for a centre
// outside the map.  radius < 0: no record.
// With records (the targets), many records may share a cell of a zeroed heatmap and every value is >= 0, so the
// cells take atomicMax on the int bits and zeros are skipped.  With one record (`one`, rec == nullptr: the
// draw_heatmap_gaussian mirror) each cell of the window is visited by exactly one thread, which stores
// torch.max(old, k * g) over the whole window: zeros and negative k included, NaN propagated.
__global__ void __launch_bounds__(kDrawThreads)
    head_targets_draw_kernel(const int4 *__restrict__ rec, int4 one, float *__restrict__ heatmap, int height,
                             int width, float k) {
  const int4 d = rec ? rec[blockIdx.x] : one;
  if (d.w < 0) return;
  const long long r = d.w;
  const long long r0 = max((long long)d.y - r, 0ll), r1 = min((long long)d.y + r, (long long)height - 1);
  const long long c0 = max((long long)d.z - r, 0ll), c1 = min((long long)d.z + r, (long long)width - 1);
  if (r0 > r1 || c0 > c1) return;
  const int nc = (int)(c1 - c0 + 1), cells = (int)(r1 - r0 + 1) * nc;
  const double sigma = (double)(2 * r + 1) / 6.0;
  const double q = __dmul_rn(__dmul_rn(2.0, sigma), sigma);
  float *plane = heatmap + (long long)d.x * height * width;
  for (int e = threadIdx.x; e < cells; e += kDrawThreads) {
    const long long row = r0 + e / nc, col = c0 + e % nc;
    const double dy = (double)(row - d.y), dx = (double)(col - d.z);
    double v = exp(-__ddiv_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), q));
    if (v < DBL_EPSILON) v = 0.0;   // h[h < eps * h.max()] = 0, h.max() = 1
    const float f = __fmul_rn(__double2float_rn(v), k);
    float *cell = plane + row * width + col;
    if (rec) {
      if (f > 0.f) atomicMax(reinterpret_cast<int *>(cell), __float_as_int(f));
    } else {
      const float old = *cell;
      *cell = isnan(old) ? old : (isnan(f) ? f : (old < f ? f : old));
    }
  }
}

size_t records_bytes(int B, int nmax) { return align_up((size_t)B * (size_t)nmax * sizeof(int4)); }

}  // namespace
}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_head_targets_workspace_bytes(int B, int nmax) {
  if (B < 0 || nmax < 0 || nmax > kMaxBoxes) return 0;
  return records_bytes(B, nmax);
}

int bevb200_head_targets(const float *boxes, const int32_t *labels, const int32_t *counts, int B, int nmax,
                         int box_dim, const int32_t *label_table_host, int num_labels,
                         const int32_t *task_classes_host, int num_tasks, float pc_x, float pc_y, float vs_x,
                         float vs_y, int out_size_factor, int fmap_x, int fmap_y, double gaussian_overlap,
                         int min_radius, int mode, int max_objs, int norm_bbox, float *heatmap, float *anno_box,
                         int64_t *ind, uint8_t *mask, int32_t *status, void *workspace, size_t workspace_bytes,
                         void *stream) {
  BEVB200_REQUIRE(mode == BEVB200_HEAD_TARGETS_CENTERHEAD || mode == BEVB200_HEAD_TARGETS_TRANSFUSION,
                  "mode must be BEVB200_HEAD_TARGETS_CENTERHEAD or _TRANSFUSION");
  const bool center = mode == BEVB200_HEAD_TARGETS_CENTERHEAD;
  BEVB200_REQUIRE(B >= 0 && nmax >= 0, "negative size");
  BEVB200_REQUIRE((long long)B * nmax <= 0x7fffffffll, "too many boxes");
  if (nmax > kMaxBoxes) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: at most %d boxes per sample (got %d)", __func__, kMaxBoxes,
             nmax);
    return BEVB200_EUNSUPPORTED;
  }
  BEVB200_REQUIRE(box_dim == 7 || box_dim == 9, "box_dim must be 7 or 9");
  BEVB200_REQUIRE(num_tasks >= 1 && num_tasks <= kMaxTasks, "num_tasks out of range");
  BEVB200_REQUIRE(center || num_tasks == 1, "TransFusion mode takes one task");
  BEVB200_REQUIRE(num_labels >= 0 && num_labels <= kMaxLabels, "num_labels out of range");
  BEVB200_REQUIRE(task_classes_host && (label_table_host || num_labels == 0), "null table");
  BEVB200_REQUIRE(fmap_x >= 1 && fmap_y >= 1 && (long long)fmap_x * fmap_y <= 0x7fffffffll, "bad feature map size");
  BEVB200_REQUIRE(out_size_factor >= 1 && min_radius >= 0, "bad out_size_factor or min_radius");
  BEVB200_REQUIRE(!center || max_objs >= 0, "negative max_objs");
  BEVB200_REQUIRE(status, "null status");
  HeadParams p;
  memset(&p, 0, sizeof(p));
  long long planes = 0;
  for (int t = 0; t < num_tasks; ++t) {
    BEVB200_REQUIRE(task_classes_host[t] >= 1 && task_classes_host[t] <= 0xffff, "task class count out of range");
    p.ncls[t] = task_classes_host[t];
    BEVB200_REQUIRE(planes <= 0x7fffffffll, "too many heatmap planes");
    p.plane0[t] = (int)planes;
    planes += (long long)B * task_classes_host[t];
  }
  BEVB200_REQUIRE(planes <= 0x7fffffffll, "too many heatmap planes");
  for (int l = 0; l < num_labels; ++l) {
    const int t = label_table_host[2 * l], c = label_table_host[2 * l + 1];
    BEVB200_REQUIRE(t == -1 || (t >= 0 && t < num_tasks && c >= 0 && c < p.ncls[t]), "bad label table entry");
    p.table[l] = t < 0 ? -1 : (t << 16 | c);
  }
  const size_t need = records_bytes(B, nmax);
  if (workspace_bytes < need || (need && !workspace)) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace %zu < %zu bytes", __func__, workspace_bytes, need);
    return BEVB200_EWORKSPACE;
  }
  const long long cells = planes * fmap_x * fmap_y;
  BEVB200_REQUIRE(heatmap || cells == 0, "null heatmap");
  BEVB200_REQUIRE((boxes && labels) || (long long)B * nmax == 0, "null boxes or labels");
  BEVB200_REQUIRE(!center || (long long)B * max_objs == 0 || (anno_box && ind && mask), "null CenterHead outputs");
  p.B = B;
  p.nmax = nmax;
  p.box_dim = box_dim;
  p.anno_dim = box_dim == 9 ? 10 : 8;
  p.mode = mode;
  p.num_labels = num_labels;
  p.num_tasks = num_tasks;
  p.fmap_x = fmap_x;
  p.fmap_y = fmap_y;
  p.min_radius = min_radius;
  p.max_objs = center ? max_objs : 0;
  p.norm_bbox = norm_bbox != 0;
  p.pc_x = pc_x;
  p.pc_y = pc_y;
  p.vs_x = vs_x;
  p.vs_y = vs_y;
  p.osf = (float)out_size_factor;
  p.one_minus = (float)(1.0 - gaussian_overlap);
  p.one_plus = (float)(1.0 + gaussian_overlap);
  p.b3k = (float)(-2.0 * gaussian_overlap);
  p.c3k = (float)(gaussian_overlap - 1.0);
  p.a3x4 = (float)(4.0 * (4.0 * gaussian_overlap));
  cudaStream_t st = (cudaStream_t)stream;
  BEVB200_LAUNCH(head_targets_zero_kernel, grid_for((cells + 3) / 4, kZeroThreads), kZeroThreads, 0, st, heatmap,
                 cells, status);
  if (B == 0) return BEVB200_OK;
  int4 *rec = (int4 *)workspace;
  BEVB200_LAUNCH(head_targets_assign_kernel, B, kAssignThreads, 0, st, boxes, labels, counts, p, anno_box, ind, mask,
                 rec, status);
  if (nmax > 0)
    BEVB200_LAUNCH(head_targets_draw_kernel, B * nmax, kDrawThreads, 0, st, (const int4 *)rec, make_int4(0, 0, 0, -1),
                   heatmap, fmap_y, fmap_x, 1.f);
  return BEVB200_OK;
}

int bevb200_draw_heatmap_gaussian(float *heatmap, int height, int width, int x, int y, int radius, float k,
                                  void *stream) {
  BEVB200_REQUIRE(height >= 0 && width >= 0 && radius >= 0, "negative size");
  BEVB200_REQUIRE(radius < (int)kMaxRadius, "radius too large");
  if (height == 0 || width == 0) return BEVB200_OK;
  BEVB200_REQUIRE(heatmap, "null heatmap");
  BEVB200_LAUNCH(head_targets_draw_kernel, 1, kDrawThreads, 0, (cudaStream_t)stream, (const int4 *)nullptr,
                 make_int4(0, y, x, radius), heatmap, height, width, k);
  return BEVB200_OK;
}

}  // extern "C"
