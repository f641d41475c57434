// Rotated BEV IoU, rotated / axis-aligned / circle NMS for the CenterHead box post-processing
// (the semantics of mmdet3d/ops/iou3d and core/post_processing/box3d_nms.py:circle_nms).
//
// Boxes are [x1, y1, x2, y2, ry] fp32.  A box is the axis-aligned extent turned by ry about its centre:
//   x' = (x - cx) cos r + (y - cy) sin r + cx,   y' = -(x - cx) sin r + (y - cy) cos r + cy.
// The overlap of two boxes is the area of one clipped by the other, in the other's own frame (rot_overlap.cuh).
// iou = overlap / max(sa + sb - overlap, 1e-8), sa and sb the unrotated extents' areas; a pair is suppressed when
// iou > thresh.
//
// NMS runs over S segments of up to Nmax boxes each (device-side counts), sorted by descending score:
//   nms_mask_kernel      bit j of mask row i (j > i) = pair (i, j) is suppressed; upper-triangle 64x64 tiles only
//   nms_suppress_kernel  one warp per segment walks 64-box blocks: the diagonal word is resolved serially in
//                        registers, then the lanes OR every kept row into the later words of the remv bitmap
//                        (shared memory), which is the reference's host loop (iou3d.cpp:132-145) bit for bit.
//                        The walk stops once post_max boxes are kept.
#include "common.cuh"
#include "rot_overlap.cuh"

namespace bevb200 {
namespace {

constexpr int kNmsBlock = 64;                                // boxes per mask word
constexpr int kNmsMaxBoxes = BEVB200_NMS_MAX_BOXES;
constexpr int kNmsMaxSegments = BEVB200_NMS_MAX_SEGMENTS;
constexpr int kNmsMaxWords = kNmsMaxBoxes / kNmsBlock;       // remv bitmap words in shared memory
constexpr float kIouEps = 1e-8f;
constexpr int kDenseTile = 16;
constexpr int kMaskSplit = 8;                                // lanes per mask row

__device__ __forceinline__ float iou_of_overlap(const float *pa, const float *pb, float ov) {
  const float sa = __fmul_rn(pa[2] - pa[0], pa[3] - pa[1]), sb = __fmul_rn(pb[2] - pb[0], pb[3] - pb[1]);
  return ov / fmaxf(sa + sb - ov, kIouEps);
}

__device__ __forceinline__ float rot_iou(const float *pa, const float *pb) {
  return iou_of_overlap(pa, pb, rot_overlap(load_rot(pa), load_rot(pb)));
}

// Axis-aligned IoU of nms_normal (iou3d_kernel.cu:335-343): the angle is ignored.
__device__ __forceinline__ float normal_iou(const float *a, const float *b) {
  const float w = fmaxf(fminf(a[2], b[2]) - fmaxf(a[0], b[0]), 0.f);
  const float h = fmaxf(fminf(a[3], b[3]) - fmaxf(a[1], b[1]), 0.f);
  const float inter = __fmul_rn(w, h);
  const float sa = __fmul_rn(a[2] - a[0], a[3] - a[1]), sb = __fmul_rn(b[2] - b[0], b[3] - b[1]);
  return inter / fmaxf(sa + sb - inter, kIouEps);
}

// circle_nms (box3d_nms.py:210-216): fp32 dx^2 + dy^2 (no FMA), compared in double with the radius itself.
__device__ __forceinline__ bool circle_hit(const float *a, const float *b, double thresh) {
  const float dx = __fsub_rn(a[0], b[0]), dy = __fsub_rn(a[1], b[1]);
  return (double)__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) <= thresh;
}

__global__ void __launch_bounds__(kDenseTile *kDenseTile)
    boxes_bev_dense_kernel(const float *__restrict__ a, int na, const float *__restrict__ b, int nb,
                           float *__restrict__ out, bool iou) {
  const int i = blockIdx.y * kDenseTile + threadIdx.y, j = blockIdx.x * kDenseTile + threadIdx.x;
  if (i >= na || j >= nb) return;
  const float *pa = a + 5ll * i, *pb = b + 5ll * j;
  const float ov = rot_overlap(load_rot(pa), load_rot(pb));
  out[(long long)i * nb + j] = iou ? iou_of_overlap(pa, pb, ov) : ov;
}

__device__ __forceinline__ int segment_count(const int32_t *counts, int s, int nmax) {
  const int n = counts ? counts[s] : nmax;
  return n < 0 ? 0 : (n > nmax ? nmax : n);
}

// One CTA per upper-triangle 64x64 tile (row block <= column block) of one segment; tiles are numbered column
// by column, t = col * (col + 1) / 2 + row.  kMaskSplit consecutive lanes share a row, each testing every
// kMaskSplit-th column, and OR their bits together, so that a tile is kMaskSplit times wider than its rows.
template <int kMode>
__global__ void __launch_bounds__(kNmsBlock *kMaskSplit)
    nms_mask_kernel(const float *__restrict__ boxes, const int32_t *__restrict__ counts, int nmax, int words,
                    float fthresh, double dthresh, unsigned long long *__restrict__ mask) {
  constexpr int D = kMode == BEVB200_NMS_CIRCLE ? 2 : 5;
  const int s = blockIdx.y, t = blockIdx.x;
  int col = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while (col * (col + 1) / 2 > t) --col;
  while ((col + 1) * (col + 2) / 2 <= t) ++col;
  const int row = t - col * (col + 1) / 2;
  const int n = segment_count(counts, s, nmax);
  if (col * kNmsBlock >= n) return;                   // uniform over the CTA
  const float *seg = boxes + (long long)s * nmax * D;
  __shared__ float cb[kNmsBlock * D];
  const int col_size = min(kNmsBlock, n - col * kNmsBlock);
  for (int e = threadIdx.x; e < col_size * D; e += kNmsBlock * kMaskSplit)
    cb[e] = seg[(long long)col * kNmsBlock * D + e];
  __syncthreads();
  const int r = threadIdx.x / kMaskSplit, part = threadIdx.x % kMaskSplit;
  const int i = row * kNmsBlock + r;
  unsigned long long bits = 0;
  if (i < n) {
    float me[D];
#pragma unroll
    for (int d = 0; d < D; ++d) me[d] = seg[(long long)i * D + d];
    const int k0 = row == col ? r + 1 : 0;
    for (int k = k0 + (part - k0 % kMaskSplit + kMaskSplit) % kMaskSplit; k < col_size; k += kMaskSplit) {
      bool hit;
      if (kMode == BEVB200_NMS_ROTATE) {
        hit = rot_iou(me, cb + k * D) > fthresh;
      } else if (kMode == BEVB200_NMS_NORMAL) {
        hit = normal_iou(me, cb + k * D) > fthresh;
      } else {
        hit = circle_hit(me, cb + k * D, dthresh);
      }
      bits |= (unsigned long long)hit << k;
    }
  }
#pragma unroll
  for (int o = 1; o < kMaskSplit; o <<= 1) bits |= __shfl_xor_sync(0xffffffffu, bits, o);
  if (i < n && part == 0) mask[((long long)s * nmax + i) * words + col] = bits;
}

__global__ void __launch_bounds__(32)
    nms_suppress_kernel(const unsigned long long *__restrict__ mask, const int32_t *__restrict__ counts, int nmax,
                        int words, const int64_t *__restrict__ order, int post_max, int64_t *__restrict__ keep,
                        int32_t *__restrict__ keep_count) {
  __shared__ unsigned long long remv[kNmsMaxWords];
  const int s = blockIdx.x, lane = threadIdx.x;
  const int n = segment_count(counts, s, nmax);
  const int nw = (n + kNmsBlock - 1) / kNmsBlock;
  for (int w = lane; w < nw; w += 32) remv[w] = 0ull;
  __syncwarp();
  const unsigned long long *m = mask + (long long)s * nmax * words;
  const int64_t *ord = order ? order + (long long)s * nmax : nullptr;
  int64_t *kp = keep + (long long)s * post_max;
  int nk = 0;
  for (int blk = 0; blk < nw && nk < post_max; ++blk) {
    const int row0 = blk * kNmsBlock, rows = min(kNmsBlock, n - row0);
    const unsigned long long d0 = lane < rows ? m[(long long)(row0 + lane) * words + blk] : 0ull;
    const unsigned long long d1 = lane + 32 < rows ? m[(long long)(row0 + lane + 32) * words + blk] : 0ull;
    unsigned long long r = remv[blk], kept = 0ull;
    for (int i = 0; i < rows; ++i) {             // the diagonal word, serially (warp-uniform)
      const unsigned long long di = __shfl_sync(0xffffffffu, i < 32 ? d0 : d1, i & 31);
      if (!((r >> i) & 1ull)) {
        kept |= 1ull << i;
        r |= di;
      }
    }
    while (nk + __popcll(kept) > post_max) kept &= ~(1ull << (63 - __clzll(kept)));
    for (int i = lane; i < kNmsBlock; i += 32) {
      if ((kept >> i) & 1ull) {
        const int idx = row0 + i, rank = __popcll(kept & ((1ull << i) - 1ull));
        kp[nk + rank] = ord ? ord[idx] : (int64_t)idx;
      }
    }
    nk += __popcll(kept);
    if (nk >= post_max) break;
    // OR the kept rows into the later words: g lanes (a power of two, as many as the words left allow) share
    // a word, each reading every g-th row of the block, and combine their words with shuffles.
    const int rem = nw - blk - 1;
    if (rem > 0) {
      const int g = 1 << (31 - __clz(max(32 / rem, 1)));
      const int groups = 32 / g, grp = lane / g, sub = lane % g;
      for (int w0 = blk + 1; w0 < nw; w0 += groups) {   // warp-uniform: every lane takes the shuffles
        const int w = w0 + grp;
        unsigned long long acc = 0ull;
        if (w < nw) {
#pragma unroll 8
          for (int i = sub; i < kNmsBlock; i += g)
            if ((kept >> i) & 1ull) acc |= m[(long long)(row0 + i) * words + w];
        }
        for (int o = 1; o < g; o <<= 1) acc |= __shfl_xor_sync(0xffffffffu, acc, o);
        if (w < nw && sub == 0) remv[w] |= acc;
      }
    }
    __syncwarp();
  }
  for (int i = nk + lane; i < post_max; i += 32) kp[i] = -1;
  if (lane == 0) keep_count[s] = nk;
}

int dense_bev(const float *a, int na, const float *b, int nb, float *out, void *stream, bool iou) {
  BEVB200_REQUIRE(na >= 0 && nb >= 0, "negative box count");
  BEVB200_REQUIRE((long long)na <= 65535ll * kDenseTile, "too many boxes_a");
  if (na == 0 || nb == 0) return BEVB200_OK;
  BEVB200_REQUIRE(a && b && out, "null argument");
  const dim3 grid((nb + kDenseTile - 1) / kDenseTile, (na + kDenseTile - 1) / kDenseTile);
  BEVB200_LAUNCH(boxes_bev_dense_kernel, grid, dim3(kDenseTile, kDenseTile), 0, (cudaStream_t)stream, a, na, b, nb,
                 out, iou);
  return BEVB200_OK;
}

size_t mask_bytes(int S, int nmax) {
  const long long words = (nmax + kNmsBlock - 1) / kNmsBlock;
  return align_up((size_t)S * (size_t)nmax * (size_t)words * sizeof(unsigned long long));
}

}  // namespace
}  // namespace bevb200

using namespace bevb200;

extern "C" {

int bevb200_boxes_iou_bev(const float *a, int na, const float *b, int nb, float *out, void *stream) {
  return dense_bev(a, na, b, nb, out, stream, true);
}

int bevb200_boxes_overlap_bev(const float *a, int na, const float *b, int nb, float *out, void *stream) {
  return dense_bev(a, na, b, nb, out, stream, false);
}

size_t bevb200_nms_workspace_bytes(int S, int nmax) {
  if (S < 0 || S > kNmsMaxSegments || nmax < 0 || nmax > kNmsMaxBoxes) return 0;
  return mask_bytes(S, nmax);
}

int bevb200_nms(const float *boxes, const int32_t *counts, int S, int nmax, int mode, double thresh, int post_max,
                const int64_t *order, int64_t *keep, int32_t *keep_count, void *workspace, size_t workspace_bytes,
                void *stream) {
  BEVB200_REQUIRE(mode == BEVB200_NMS_ROTATE || mode == BEVB200_NMS_NORMAL || mode == BEVB200_NMS_CIRCLE,
                  "mode must be BEVB200_NMS_ROTATE, _NORMAL or _CIRCLE");
  BEVB200_REQUIRE(S >= 0 && nmax >= 0 && post_max >= 0, "negative size");
  if (nmax > kNmsMaxBoxes || S > kNmsMaxSegments) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: at most %d boxes per segment and %d segments (got %d, %d)",
             __func__, kNmsMaxBoxes, kNmsMaxSegments, nmax, S);
    return BEVB200_EUNSUPPORTED;
  }
  if (S == 0) return BEVB200_OK;
  BEVB200_REQUIRE(keep_count && (keep || post_max == 0), "null output");
  BEVB200_REQUIRE(boxes || nmax == 0, "null boxes");
  const size_t need = mask_bytes(S, nmax);
  if (workspace_bytes < need || (need && !workspace)) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace %zu < %zu bytes", __func__, workspace_bytes, need);
    return BEVB200_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int words = (nmax + kNmsBlock - 1) / kNmsBlock;
  auto *mask = (unsigned long long *)workspace;
  if (words > 0) {
    const dim3 grid(words * (words + 1) / 2, S);
    const float ft = (float)thresh;
    if (mode == BEVB200_NMS_ROTATE) {
      BEVB200_LAUNCH(nms_mask_kernel<BEVB200_NMS_ROTATE>, grid, kNmsBlock * kMaskSplit, 0, st, boxes, counts, nmax, words, ft,
                     thresh, mask);
    } else if (mode == BEVB200_NMS_NORMAL) {
      BEVB200_LAUNCH(nms_mask_kernel<BEVB200_NMS_NORMAL>, grid, kNmsBlock * kMaskSplit, 0, st, boxes, counts, nmax, words, ft,
                     thresh, mask);
    } else {
      BEVB200_LAUNCH(nms_mask_kernel<BEVB200_NMS_CIRCLE>, grid, kNmsBlock * kMaskSplit, 0, st, boxes, counts, nmax, words, ft,
                     thresh, mask);
    }
  }
  BEVB200_LAUNCH(nms_suppress_kernel, S, 32, 0, st, mask, counts, nmax, words, order, post_max, keep, keep_count);
  return BEVB200_OK;
}

}  // extern "C"
