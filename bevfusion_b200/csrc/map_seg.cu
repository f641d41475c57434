// BEV map segmentation on the device: BEVSegmentationHead (models/heads/segm/vanilla.py) -- the BEVGridTransform
// resampling forward and backward, the per-class sigmoid focal / xent losses with their gradients -- and the IoU
// counts of NuScenesDataset.evaluate_map (datasets/nuscenes_dataset.py:498-530).
//
// Grid transform.  The optional bilinear prescale and the bilinear grid_sample are both separable and the same for
// every sample, so the whole transform is dst[i][j] = sum_(r, wy) in rows[i] wy * sum_(c, wx) in cols[j] wx * src[r][c]
// with per-axis CSR tables built once on the host (bevfusion_b200/map_seg.py).  One kernel runs both directions:
//   forward    rows / cols are the <= 4 composite taps of each output row / column (zeros padding: taps outside the
//              input are absent);
//   backward   the transposed tables -- for each input row / column its (output index, weight) list in ascending
//              output order -- applied to grad_output.  Every grad_input element is written once, in a fixed order,
//              with no atomics and no memset: rows and columns that no tap reaches get an empty sum, 0.
// One CTA per (plane = sample x channel, block of rows_per_block destination rows) stages the column table and the
// source rows its block reads [block_lo, block_lo + block_rows) in shared memory with coalesced loads, interpolates
// horizontally into a second shared buffer, then vertically, and stores whole destination rows.  fp32 accumulation,
// fp32 or fp16 I/O.
//
// Losses.  Forward: seg_loss_kernel writes one double partial per (tile of 1024 elements, class, sample) to its own
// workspace slot, seg_reduce_kernel adds each class's slots in a fixed order and divides by B * H * W.  Backward:
// seg_loss_grad_kernel writes every logit gradient once.  No atomics: bit-reproducible.
//
// Counts.  seg_counts_kernel: per-thread tp / predicted-positive / positive counters, warp sums, shared-memory
// counters, then one 64-bit integer atomic per counter per CTA -- exact and independent of the order of the CTAs.
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace bevb200 {
namespace {

constexpr int kThreads = 256;
constexpr int kLossTile = 1024;                       // elements per loss CTA: 4 per thread
constexpr int kCountTile = 2048;                      // elements per count CTA: 8 per thread
constexpr int kMaxThr = BEVB200_MAP_MAX_THRESHOLDS;
constexpr size_t kGridSmemLimit = 48 * 1024;

template <typename T>
__device__ __forceinline__ float ldf(const T *p) {
  if constexpr (sizeof(T) == 2) return __half2float(__ldg(p));
  else return (float)__ldg(p);
}

template <typename T>
__device__ __forceinline__ void stf(T *p, float v) {
  if constexpr (sizeof(T) == 2) *p = __float2half_rn(v);
  else *p = v;
}

// ---- grid transform ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ size_t al16(size_t x) { return (x + 15) / 16 * 16; }

// Shared memory: column ptr, column (index, weight), staged source rows, horizontally interpolated rows.
size_t grid_smem(int src_w, int dst_w, int col_nnz, int max_block_rows) {
  return al16((size_t)(dst_w + 1) * 4) + al16((size_t)col_nnz * 8) +
         (size_t)max_block_rows * (src_w + dst_w) * 4;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) grid_apply_kernel(
    const T *__restrict__ src, T *__restrict__ dst, int Hs, int Ws, int Hd, int Wd, const int *__restrict__ rptr,
    const int *__restrict__ ridx, const float *__restrict__ rw, const int *__restrict__ cptr,
    const int *__restrict__ cidx, const float *__restrict__ cw, int c_nnz, const int *__restrict__ blk_lo,
    const int *__restrict__ blk_rows, int R, int n_max) {
  extern __shared__ __align__(16) unsigned char smem[];
  int *s_cptr = (int *)smem;
  int *s_cidx = (int *)(smem + al16((size_t)(Wd + 1) * 4));
  float *s_cw = (float *)(s_cidx + c_nnz);
  float *s_in = (float *)((unsigned char *)s_cidx + al16((size_t)c_nnz * 8));
  float *s_h = s_in + (size_t)n_max * Ws;

  const long long plane = blockIdx.x;
  const int i0 = blockIdx.y * R;
  const int lo = __ldg(blk_lo + blockIdx.y);
  int n = min(__ldg(blk_rows + blockIdx.y), n_max);
  if (lo < 0 || lo + n > Hs) n = 0;                    // a malformed block reads nothing

  for (int k = threadIdx.x; k <= Wd; k += kThreads) s_cptr[k] = min(max(__ldg(cptr + k), 0), c_nnz);
  for (int k = threadIdx.x; k < c_nnz; k += kThreads) {
    s_cidx[k] = __ldg(cidx + k);
    s_cw[k] = __ldg(cw + k);
  }
  const T *sp = src + plane * Hs * Ws + (long long)lo * Ws;
  for (int k = threadIdx.x; k < n * Ws; k += kThreads) s_in[k] = ldf(sp + k);
  __syncthreads();

  for (int k = threadIdx.x; k < n * Wd; k += kThreads) {
    const int r = k / Wd, j = k - r * Wd;
    const float *row = s_in + (size_t)r * Ws;
    float a = 0.f;
    for (int e = s_cptr[j]; e < s_cptr[j + 1]; ++e) {
      const int c = s_cidx[e];
      if ((unsigned)c < (unsigned)Ws) a += s_cw[e] * row[c];
    }
    s_h[k] = a;
  }
  __syncthreads();

  T *dp = dst + plane * Hd * Wd;
  const int rows = min(R, Hd - i0);
  for (int k = threadIdx.x; k < rows * Wd; k += kThreads) {
    const int ii = k / Wd, j = k - ii * Wd, i = i0 + ii;
    float a = 0.f;
    const int e1 = __ldg(rptr + i + 1);
    for (int e = __ldg(rptr + i); e < e1; ++e) {
      const int r = __ldg(ridx + e) - lo;
      if ((unsigned)r < (unsigned)n) a += __ldg(rw + e) * s_h[(size_t)r * Wd + j];
    }
    stf(dp + (long long)i * Wd + j, a);
  }
}

// ---- losses -----------------------------------------------------------------------------------------------------
// Elementwise loss in double of fp32 logit x against target t; *d = d loss / d x.
//   ce = (1 - t) x + log(1 + e^-x)              (binary_cross_entropy_with_logits)
//   focal: m = 1 - p_t = t (1 - p) + (1 - t) p, loss = ce m^2  (alpha < 0: no alpha_t, gamma = 2)
__device__ __forceinline__ double seg_elem(float xf, float tf, int focal, double *d) {
  const double x = xf, t = tf;
  const double sp = x > 0.0 ? log1p(exp(-x)) : -x + log1p(exp(x));
  const double p = 1.0 / (1.0 + exp(-x)), q = 1.0 / (1.0 + exp(x));
  const double ce = (1.0 - t) * x + sp;
  const double dce = (1.0 - t) * p - t * q;          // p - t without cancellation at saturated logits
  if (!focal) {
    if (d) *d = dce;
    return ce;
  }
  const double m = t * q + (1.0 - t) * p;
  if (d) *d = dce * m * m + ce * 2.0 * m * (1.0 - 2.0 * t) * p * q;
  return ce * m * m;
}

template <typename TT>
__device__ __forceinline__ float ld_target(const TT *p) {
  return (float)__ldg(p);                             // int64 / uint8 / fp32 -> fp32, as the reference's .float()
}

template <typename TX, typename TT>
__global__ void __launch_bounds__(kThreads) seg_loss_kernel(const TX *__restrict__ x, const TT *__restrict__ t,
                                                            int K, long long HW, int focal, double *__restrict__ part) {
  const int tile = blockIdx.x, k = blockIdx.y, b = blockIdx.z;
  const long long base = ((long long)b * K + k) * HW;
  double s = 0.0;
#pragma unroll
  for (int r = 0; r < kLossTile / kThreads; ++r) {
    const long long e = (long long)tile * kLossTile + r * kThreads + threadIdx.x;
    if (e < HW) s += seg_elem(ldf(x + base + e), ld_target(t + base + e), focal, nullptr);
  }
  __shared__ double ws[kThreads / 32];
  for (int o = 16; o; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double r = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) r += ws[w];
    part[((long long)k * gridDim.z + b) * gridDim.x + tile] = r;
  }
}

// One warp per class: its B * tiles slots in lane-strided order, then a shuffle tree.
__global__ void seg_reduce_kernel(const double *__restrict__ part, long long slots, double inv_n,
                                  float *__restrict__ losses) {
  const int k = blockIdx.x;
  double s = 0.0;
  for (long long i = threadIdx.x; i < slots; i += 32) s += part[k * slots + i];
  for (int o = 16; o; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if (threadIdx.x == 0) losses[k] = (float)(s * inv_n);
}

template <typename TX, typename TT>
__global__ void __launch_bounds__(kThreads) seg_loss_grad_kernel(const TX *__restrict__ x, const TT *__restrict__ t,
                                                                 int K, long long HW, int focal, double inv_n,
                                                                 const float *__restrict__ grad_losses,
                                                                 TX *__restrict__ g) {
  const int tile = blockIdx.x, k = blockIdx.y, b = blockIdx.z;
  const long long base = ((long long)b * K + k) * HW;
  const double G = (double)__ldg(grad_losses + k) * inv_n;
  double d;
#pragma unroll
  for (int r = 0; r < kLossTile / kThreads; ++r) {
    const long long e = (long long)tile * kLossTile + r * kThreads + threadIdx.x;
    if (e < HW) {
      seg_elem(ldf(x + base + e), ld_target(t + base + e), focal, &d);
      stf(g + base + e, (float)(G * d));
    }
  }
}

// ---- IoU counts -------------------------------------------------------------------------------------------------
struct Thresholds {
  float v[kMaxThr];
};

template <typename TP, typename TG>
__global__ void __launch_bounds__(kThreads) seg_counts_kernel(const TP *__restrict__ pred, const TG *__restrict__ gt,
                                                              int K, long long HW, Thresholds th, int T,
                                                              unsigned long long *__restrict__ out) {
  const int tile = blockIdx.x, k = blockIdx.y, b = blockIdx.z;
  const long long base = ((long long)b * K + k) * HW;
  int pos = 0, tp[kMaxThr], pp[kMaxThr];
#pragma unroll
  for (int i = 0; i < kMaxThr; ++i) tp[i] = pp[i] = 0;
#pragma unroll
  for (int r = 0; r < kCountTile / kThreads; ++r) {
    const long long e = (long long)tile * kCountTile + r * kThreads + threadIdx.x;
    if (e < HW) {
      const float v = ldf(pred + base + e);
      const int lab = __ldg(gt + base + e) != (TG)0;  // NaN != 0: positive, as bool(NaN)
      pos += lab;
#pragma unroll
      for (int i = 0; i < kMaxThr; ++i) {
        if (i < T) {
          const int pr = v >= th.v[i];                // NaN: negative
          tp[i] += pr & lab;
          pp[i] += pr;
        }
      }
    }
  }
  __shared__ int s_cnt[1 + 2 * kMaxThr];
  for (int i = threadIdx.x; i < 1 + 2 * kMaxThr; i += kThreads) s_cnt[i] = 0;
  __syncthreads();
  pos = __reduce_add_sync(0xffffffffu, pos);
#pragma unroll
  for (int i = 0; i < kMaxThr; ++i) {
    tp[i] = __reduce_add_sync(0xffffffffu, tp[i]);
    pp[i] = __reduce_add_sync(0xffffffffu, pp[i]);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&s_cnt[0], pos);
#pragma unroll
    for (int i = 0; i < kMaxThr; ++i) {
      if (i < T) {
        atomicAdd(&s_cnt[1 + i], tp[i]);
        atomicAdd(&s_cnt[1 + kMaxThr + i], pp[i]);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < 3 * T) {
    const int which = threadIdx.x / T, i = threadIdx.x - which * T;
    const int tpi = s_cnt[1 + i], ppi = s_cnt[1 + kMaxThr + i];
    const int v = which == 0 ? tpi : (which == 1 ? ppi - tpi : s_cnt[0] - tpi);
    if (v) atomicAdd(out + ((long long)which * gridDim.y + k) * T + i, (unsigned long long)(long long)v);
  }
}

int check_map(const void *a, const void *b, int B, int K, int H, int W) {
  BEVB200_REQUIRE(a && b, "null pointer");
  BEVB200_REQUIRE(B >= 1 && K >= 1 && H >= 1 && W >= 1, "sizes must be >= 1");
  BEVB200_REQUIRE(B <= 65535 && K <= 65535, "B and K must be <= 65535");
  return 0;
}

int tiles_of(long long HW, int tile) { return (int)((HW + tile - 1) / tile); }

template <typename TX>
int loss_dispatch(const void *x, const void *t, int ttype, dim3 grid, int K, long long HW, int focal, double *part,
                  cudaStream_t s) {
  switch (ttype) {
    case BEVB200_MAP_TARGET_F32:
      BEVB200_LAUNCH(seg_loss_kernel, grid, kThreads, 0, s, (const TX *)x, (const float *)t, K, HW, focal, part);
      return 0;
    case BEVB200_MAP_TARGET_U8:
      BEVB200_LAUNCH(seg_loss_kernel, grid, kThreads, 0, s, (const TX *)x, (const uint8_t *)t, K, HW, focal, part);
      return 0;
    case BEVB200_MAP_TARGET_I64:
      BEVB200_LAUNCH(seg_loss_kernel, grid, kThreads, 0, s, (const TX *)x, (const int64_t *)t, K, HW, focal, part);
      return 0;
  }
  BEVB200_REQUIRE(false, "unknown target type");
  return 0;
}

template <typename TX>
int grad_dispatch(const void *x, const void *t, int ttype, dim3 grid, int K, long long HW, int focal, double inv_n,
                  const float *gl, void *g, cudaStream_t s) {
  switch (ttype) {
    case BEVB200_MAP_TARGET_F32:
      BEVB200_LAUNCH(seg_loss_grad_kernel, grid, kThreads, 0, s, (const TX *)x, (const float *)t, K, HW, focal, inv_n,
                     gl, (TX *)g);
      return 0;
    case BEVB200_MAP_TARGET_U8:
      BEVB200_LAUNCH(seg_loss_grad_kernel, grid, kThreads, 0, s, (const TX *)x, (const uint8_t *)t, K, HW, focal,
                     inv_n, gl, (TX *)g);
      return 0;
    case BEVB200_MAP_TARGET_I64:
      BEVB200_LAUNCH(seg_loss_grad_kernel, grid, kThreads, 0, s, (const TX *)x, (const int64_t *)t, K, HW, focal,
                     inv_n, gl, (TX *)g);
      return 0;
  }
  BEVB200_REQUIRE(false, "unknown target type");
  return 0;
}

template <typename TP>
int counts_dispatch(const void *p, const void *g, int gtype, dim3 grid, int K, long long HW, const Thresholds &th,
                    int T, int64_t *out, cudaStream_t s) {
  unsigned long long *o = (unsigned long long *)out;
  switch (gtype) {
    case BEVB200_MAP_TARGET_F32:
      BEVB200_LAUNCH(seg_counts_kernel, grid, kThreads, 0, s, (const TP *)p, (const float *)g, K, HW, th, T, o);
      return 0;
    case BEVB200_MAP_TARGET_U8:
      BEVB200_LAUNCH(seg_counts_kernel, grid, kThreads, 0, s, (const TP *)p, (const uint8_t *)g, K, HW, th, T, o);
      return 0;
    case BEVB200_MAP_TARGET_I64:
      BEVB200_LAUNCH(seg_counts_kernel, grid, kThreads, 0, s, (const TP *)p, (const int64_t *)g, K, HW, th, T, o);
      return 0;
  }
  BEVB200_REQUIRE(false, "unknown target type");
  return 0;
}

}  // namespace
}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_map_grid_smem_bytes(int src_w, int dst_w, int col_nnz, int max_block_rows) {
  if (src_w < 1 || dst_w < 1 || col_nnz < 0 || max_block_rows < 0) return 0;
  return grid_smem(src_w, dst_w, col_nnz, max_block_rows);
}

int bevb200_map_grid_transform(const void *src, void *dst, int half, long long planes, int src_h, int src_w,
                               int dst_h, int dst_w, const int32_t *row_ptr, const int32_t *row_idx,
                               const float *row_w, const int32_t *col_ptr, const int32_t *col_idx, const float *col_w,
                               int col_nnz, const int32_t *block_lo, const int32_t *block_rows, int rows_per_block,
                               int max_block_rows, void *stream) {
  BEVB200_REQUIRE(src && dst && row_ptr && col_ptr && block_lo && block_rows, "null pointer");
  BEVB200_REQUIRE(col_nnz == 0 || (col_idx && col_w), "null column table");
  BEVB200_REQUIRE(row_idx && row_w, "null row table");
  BEVB200_REQUIRE(planes >= 1 && planes <= 0x7fffffffLL, "planes must be in 1..2^31-1");
  BEVB200_REQUIRE(src_h >= 1 && src_w >= 1 && dst_h >= 1 && dst_w >= 1, "sizes must be >= 1");
  BEVB200_REQUIRE(col_nnz >= 0 && max_block_rows >= 0 && max_block_rows <= src_h, "bad table sizes");
  BEVB200_REQUIRE(rows_per_block >= 1, "rows_per_block must be >= 1");
  const long long nblk = ((long long)dst_h + rows_per_block - 1) / rows_per_block;
  BEVB200_REQUIRE(nblk <= 65535, "too many row blocks");
  const size_t smem = grid_smem(src_w, dst_w, col_nnz, max_block_rows);
  if (smem > kGridSmemLimit) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: %zu bytes of shared memory exceed %zu", __func__, smem,
             kGridSmemLimit);
    return BEVB200_EUNSUPPORTED;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid((unsigned)planes, (unsigned)nblk);
  if (half)
    BEVB200_LAUNCH(grid_apply_kernel<__half>, grid, kThreads, smem, s, (const __half *)src, (__half *)dst, src_h,
                   src_w, dst_h, dst_w, row_ptr, row_idx, row_w, col_ptr, col_idx, col_w, col_nnz, block_lo,
                   block_rows, rows_per_block, max_block_rows);
  else
    BEVB200_LAUNCH(grid_apply_kernel<float>, grid, kThreads, smem, s, (const float *)src, (float *)dst, src_h, src_w,
                   dst_h, dst_w, row_ptr, row_idx, row_w, col_ptr, col_idx, col_w, col_nnz, block_lo, block_rows,
                   rows_per_block, max_block_rows);
  return 0;
}

size_t bevb200_map_seg_loss_workspace_bytes(int B, int K, int H, int W) {
  if (B < 1 || K < 1 || H < 1 || W < 1) return 0;
  return align_up((size_t)K * B * tiles_of((long long)H * W, kLossTile) * sizeof(double));
}

int bevb200_map_seg_loss(const void *logits, int logits_half, const void *target, int target_type, int B, int K,
                         int H, int W, int focal, float *losses, void *workspace, size_t workspace_bytes,
                         void *stream) {
  if (int rc = check_map(logits, target, B, K, H, W)) return rc;
  BEVB200_REQUIRE(losses && workspace, "null pointer");
  const long long HW = (long long)H * W;
  const int tiles = tiles_of(HW, kLossTile);
  if (workspace_bytes < bevb200_map_seg_loss_workspace_bytes(B, K, H, W)) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace too small", __func__);
    return BEVB200_EWORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  double *part = (double *)workspace;
  const dim3 grid(tiles, K, B);
  const int rc = logits_half ? loss_dispatch<__half>(logits, target, target_type, grid, K, HW, focal != 0, part, s)
                             : loss_dispatch<float>(logits, target, target_type, grid, K, HW, focal != 0, part, s);
  if (rc) return rc;
  BEVB200_LAUNCH(seg_reduce_kernel, K, 32, 0, s, part, (long long)B * tiles, 1.0 / ((double)B * HW), losses);
  return 0;
}

int bevb200_map_seg_loss_backward(const void *logits, int logits_half, const void *target, int target_type, int B,
                                  int K, int H, int W, int focal, const float *grad_losses, void *grad_logits,
                                  void *stream) {
  if (int rc = check_map(logits, target, B, K, H, W)) return rc;
  BEVB200_REQUIRE(grad_losses && grad_logits, "null pointer");
  const long long HW = (long long)H * W;
  const dim3 grid(tiles_of(HW, kLossTile), K, B);
  const double inv_n = 1.0 / ((double)B * HW);
  cudaStream_t s = (cudaStream_t)stream;
  return logits_half ? grad_dispatch<__half>(logits, target, target_type, grid, K, HW, focal != 0, inv_n, grad_losses,
                                             grad_logits, s)
                     : grad_dispatch<float>(logits, target, target_type, grid, K, HW, focal != 0, inv_n, grad_losses,
                                            grad_logits, s);
}

int bevb200_map_seg_counts(const void *pred, int pred_half, const void *gt, int gt_type, int B, int K, int H, int W,
                           const float *thresholds_host, int T, int64_t *counts, void *stream) {
  if (int rc = check_map(pred, gt, B, K, H, W)) return rc;
  BEVB200_REQUIRE(thresholds_host && counts, "null pointer");
  BEVB200_REQUIRE(T >= 1 && T <= kMaxThr, "1..BEVB200_MAP_MAX_THRESHOLDS thresholds");
  Thresholds th;
  for (int i = 0; i < kMaxThr; ++i) th.v[i] = i < T ? thresholds_host[i] : 0.f;
  const long long HW = (long long)H * W;
  const dim3 grid(tiles_of(HW, kCountTile), K, B);
  cudaStream_t s = (cudaStream_t)stream;
  return pred_half ? counts_dispatch<__half>(pred, gt, gt_type, grid, K, HW, th, T, counts, s)
                   : counts_dispatch<float>(pred, gt, gt_type, grid, K, HW, th, T, counts, s);
}

}  // extern "C"
