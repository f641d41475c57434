// TransFusion query proposals on the device: the query initialisation of TransFusionHead.forward_single
// (models/heads/bbox/transfusion.py:237-281 and :322-325) -- sigmoid of the dense heatmap, the k x k peak mask with
// its exempt classes, the top num_proposals of the masked plane and the query_heatmap_score gather -- with no host
// synchronisation, no allocation and no full sort.
//
// Two launches per call:
//   tf_peak_kernel    one CTA per tile of 1024 consecutive flat cells (c * H * W + h * W + w) of a sample: sigmoid,
//                     peak test and the order-preserving 64-bit key of every cell whose masked value m is > 0 or NaN,
//                     written in index order to the tile's own slice of the workspace with the tile's count.  Most
//                     cells are masked zeros and write nothing; no counter needs zeroing beforehand.
//   tf_select_kernel  one CTA per sample: an MSD radix select (8-bit digits) of the K-th largest key over the
//                     candidates.  As soon as the keys under the current prefix fit in shared memory (4096) they are
//                     moved there in one pass, so the global list is typically read twice.  The K winners (or every
//                     candidate plus the lowest-index masked zeros when there are fewer than K) are bitonic-sorted in
//                     shared memory, then labels, index and query_heatmap_score are written, the masked values
//                     recomputed from the logits at the K selected cells.
//
// key(m) is the float's order-preserving unsigned image with every NaN mapped to the top, and the 64-bit key is
// key(m) << 32 | ~flat, so descending 64-bit order is (m descending, NaN first; ties by ascending flat index):
// argsort(descending=True, stable=True).  Every key is distinct, so the selected set and its order are fixed and the
// result is the same bit for bit on every run, whatever order the candidates were counted in.
//
// The sigmoid is torch's on CUDA: 1 / (1 + expf(-x)) in fp32 with IEEE division and the full-precision expf, rounded
// to fp16 for fp16 input; the peak test compares those rounded values.  The window maximum propagates NaN as
// max_pool2d does.  Built without fast-math, as the whole library is.  The keys, the candidate tiles and the select
// are topk_select.cuh's, shared with the CenterHead box decode.
#include <cuda_fp16.h>
#include <math.h>

#include "topk_select.cuh"

namespace bevb200 {
namespace {

using namespace topk;   // the key helpers, the candidate tiles and the select (topk_select.cuh)

constexpr int kPeakThreads = 256;
constexpr int kCellsPerThread = kTile / kPeakThreads;
constexpr int kMaxK = BEVB200_PROPOSALS_MAX_K;

struct PropParams {
  int B, C, H, W, K, pad;
  int ex0, ex1;        // exempt classes, -1 for none
  int hw, chw, tiles;  // H * W, C * H * W, ceil(chw / kTile)
};

template <typename T>
__device__ __forceinline__ float load_logit(const T *p);
template <>
__device__ __forceinline__ float load_logit<float>(const float *p) {
  return __ldg(p);
}
template <>
__device__ __forceinline__ float load_logit<__half>(const __half *p) {
  return __half2float(__ldg(p));
}

// m = s * (s == local_max) at (c, h, w) of one sample's [C, H, W] logits, as a float (exact for fp16)
template <typename T>
__device__ __forceinline__ float masked_value(const T *__restrict__ xs, const PropParams &p, int c, int h, int w) {
  const T *plane = xs + (long long)c * p.hw;
  const float s = sigmoid_as<T>(load_logit(plane + h * p.W + w));
  float lm;
  if (c == p.ex0 || c == p.ex1) {
    lm = s;                                       // max_pool2d with kernel 1
  } else if (h < p.pad || h >= p.H - p.pad || w < p.pad || w >= p.W - p.pad) {
    lm = 0.f;                                     // the zeroed border band of local_max
  } else {
    lm = -INFINITY;                               // max_pool2d: (val > maxval) || isnan(val)
    for (int dy = -p.pad; dy <= p.pad; ++dy) {
      const T *row = plane + (h + dy) * p.W + w;
      for (int dx = -p.pad; dx <= p.pad; ++dx) {
        const float v = sigmoid_as<T>(load_logit(row + dx));
        if (v > lm || isnan(v)) lm = v;
      }
    }
  }
  return __fmul_rn(s, s == lm ? 1.f : 0.f);      // NaN * 0 stays NaN
}

// Thread tid handles cells tile * kTile + r * kPeakThreads + tid, r = 0..kCellsPerThread-1; the tile's keepers are
// written in that (flat index) order.
template <typename T>
__global__ void __launch_bounds__(kPeakThreads, 1)
    tf_peak_kernel(const T *__restrict__ x, const __grid_constant__ PropParams p, uint64_t *__restrict__ cand,
                   int32_t *__restrict__ tile_count) {
  const int b = blockIdx.y, tile = blockIdx.x, tid = threadIdx.x;
  const T *xs = x + (long long)b * p.chw;
  uint64_t key[kCellsPerThread];
  unsigned bal[kCellsPerThread];
#pragma unroll
  for (int r = 0; r < kCellsPerThread; ++r) {
    const int flat = tile * kTile + r * kPeakThreads + tid;
    bool keep = false;
    key[r] = 0;
    if (flat < p.chw) {
      const int c = flat / p.hw, cell = flat - c * p.hw;
      const int h = cell / p.W, w = cell - h * p.W;
      const float m = masked_value(xs, p, c, h, w);
      keep = m > 0.f || isnan(m);
      key[r] = full_key(m, flat);
    }
    bal[r] = __ballot_sync(0xffffffffu, keep);
  }
  const long long slot = (long long)b * p.tiles + tile;
  write_tile_keys<kPeakThreads>(key, bal, cand + slot * kTile, tile_count + slot);
}

template <typename T>
__global__ void __launch_bounds__(kSelectThreads, 1)
    tf_select_kernel(const T *__restrict__ x, const __grid_constant__ PropParams p,
                     const uint64_t *__restrict__ cand_all, const int32_t *__restrict__ count_all, int sort_n,
                     int64_t *__restrict__ labels, int64_t *__restrict__ index, T *__restrict__ score) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint64_t *sel = (uint64_t *)smem;               // [sort_n]
  uint64_t *buf = sel + sort_n;                   // [kBufCap] the keys under the current prefix, once they fit
  uint32_t *win = (uint32_t *)(buf + kBufCap);    // [K] selected flat indices in output order
  const int b = blockIdx.x, tid = threadIdx.x;
  const int K = p.K;
  const int nsel = select_top_keys(cand_all + (long long)b * p.tiles * kTile, count_all + (long long)b * p.tiles,
                                   p.tiles, K, sort_n, sel, buf);
  for (int i = tid; i < nsel; i += kSelectThreads) win[i] = key_flat(sel[i]);
  __syncthreads();

  if (nsel < K) {
    // fewer than K candidates: the rest are masked zeros in ascending flat index, skipping candidates.  With the
    // candidates' indices a_0 < a_1 < ... sorted, the j-th non-candidate is j + #{i : a_i - i <= j}.
    for (int i = tid; i < sort_n; i += kSelectThreads) sel[i] = i < nsel ? ~(uint64_t)win[i] : 0;
    __syncthreads();
    bitonic_desc(sel, sort_n);                    // ~a descending: a ascending
    for (int j = tid; j < K - nsel; j += kSelectThreads) {
      int lo = 0, hi = nsel;                      // first i with a_i - i > j
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const int gap = (int)(uint32_t)~sel[mid] - mid;
        if (gap <= j) lo = mid + 1;
        else hi = mid;
      }
      win[nsel + j] = (uint32_t)(j + lo);
    }
    __syncthreads();
  }

  for (int j = tid; j < K; j += kSelectThreads) {
    const int f = (int)win[j];
    labels[(long long)b * K + j] = f / p.hw;
    index[(long long)b * K + j] = f % p.hw;
  }
  const T *xs = x + (long long)b * p.chw;
  for (int q = tid; q < p.C * K; q += kSelectThreads) {
    const int c = q / K, j = q - c * K;
    const int cell = (int)win[j] % p.hw;
    const int h = cell / p.W, w = cell - h * p.W;
    const float m = masked_value(xs, p, c, h, w);
    if constexpr (sizeof(T) == 2)
      score[(long long)b * p.C * K + q] = __float2half_rn(m);
    else
      score[(long long)b * p.C * K + q] = m;
  }
}

size_t select_smem_bytes(int K) {
  return (size_t)(sort_size(K) + kBufCap) * sizeof(uint64_t) + (size_t)K * sizeof(uint32_t);
}

bool sizes_ok(int B, int C, int H, int W) {
  return B >= 1 && C >= 1 && H >= 1 && W >= 1 && B <= BEVB200_PROPOSALS_MAX_BATCH &&
         C <= BEVB200_PROPOSALS_MAX_CLASSES && (long long)C * H * W <= BEVB200_PROPOSALS_MAX_CELLS;
}

size_t ws_bytes(int B, int C, int H, int W) {
  const long long tiles = ((long long)C * H * W + kTile - 1) / kTile;
  return align_up((size_t)B * tiles * kTile * sizeof(uint64_t)) + align_up((size_t)B * tiles * sizeof(int32_t));
}

template <typename T>
int launch(const void *x, const PropParams &p, int64_t *labels, int64_t *index, void *score, uint64_t *cand,
           int32_t *counts, cudaStream_t st) {
  const dim3 grid((unsigned)p.tiles, (unsigned)p.B);
  BEVB200_LAUNCH(tf_peak_kernel<T>, grid, kPeakThreads, 0, st, (const T *)x, p, cand, counts);
  const size_t smem = select_smem_bytes(p.K);
  if (smem > 44 * 1024)   // the shipped K = 200 (36 KB) stays below the default limit
    BEVB200_CUDA(cudaFuncSetAttribute(tf_select_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  BEVB200_LAUNCH(tf_select_kernel<T>, p.B, kSelectThreads, smem, st, (const T *)x, p, cand, counts,
                 sort_size(p.K), labels, index, (T *)score);
  return BEVB200_OK;
}

}  // namespace
}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_transfusion_proposals_workspace_bytes(int B, int C, int H, int W) {
  if (!sizes_ok(B, C, H, W)) return 0;
  return ws_bytes(B, C, H, W);
}

int bevb200_transfusion_proposals(const void *heatmap, int dtype, int B, int C, int H, int W, int num_proposals,
                                  int kernel_size, int exempt0, int exempt1, int64_t *labels, int64_t *index,
                                  void *query_heatmap_score, void *workspace, size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(B >= 1 && C >= 1 && H >= 1 && W >= 1, "bad size");
  BEVB200_REQUIRE(kernel_size >= 3 && kernel_size % 2 == 1, "kernel_size must be odd and at least 3");
  BEVB200_REQUIRE(H >= kernel_size && W >= kernel_size, "the map is smaller than the kernel");
  BEVB200_REQUIRE(exempt0 >= -1 && exempt0 < C && exempt1 >= -1 && exempt1 < C, "exempt class out of range");
  BEVB200_REQUIRE(num_proposals >= 1 && (long long)num_proposals <= (long long)C * H * W,
                  "num_proposals must be in 1..C * H * W");
  if (dtype != BEVB200_PROPOSALS_F32 && dtype != BEVB200_PROPOSALS_F16) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: dtype %d is neither fp32 nor fp16", __func__, dtype);
    return BEVB200_EUNSUPPORTED;
  }
  if (!sizes_ok(B, C, H, W) || num_proposals > kMaxK || kernel_size > BEVB200_PROPOSALS_MAX_KERNEL) {
    snprintf(g_last_error, sizeof(g_last_error),
             "%s: at most %d samples, %d classes, %d cells per sample, %d proposals and kernel %d (got B %d, C %d, "
             "H %d, W %d, K %d, k %d)",
             __func__, BEVB200_PROPOSALS_MAX_BATCH, BEVB200_PROPOSALS_MAX_CLASSES, BEVB200_PROPOSALS_MAX_CELLS, kMaxK,
             BEVB200_PROPOSALS_MAX_KERNEL, B, C, H, W, num_proposals, kernel_size);
    return BEVB200_EUNSUPPORTED;
  }
  BEVB200_REQUIRE(heatmap && labels && index && query_heatmap_score, "null pointer");
  const size_t need = ws_bytes(B, C, H, W);
  if (workspace_bytes < need || !workspace) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace %zu < %zu bytes", __func__, workspace_bytes, need);
    return BEVB200_EWORKSPACE;
  }
  PropParams p;
  p.B = B;
  p.C = C;
  p.H = H;
  p.W = W;
  p.K = num_proposals;
  p.pad = kernel_size / 2;
  p.ex0 = exempt0;
  p.ex1 = exempt1;
  p.hw = H * W;
  p.chw = C * H * W;
  p.tiles = (p.chw + kTile - 1) / kTile;
  Arena ar(workspace, workspace_bytes);
  uint64_t *cand = ar.take<uint64_t>((size_t)B * p.tiles * kTile);
  int32_t *counts = ar.take<int32_t>((size_t)B * p.tiles);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == BEVB200_PROPOSALS_F16)
    return launch<__half>(heatmap, p, labels, index, query_heatmap_score, cand, counts, st);
  return launch<float>(heatmap, p, labels, index, query_heatmap_score, cand, counts, st);
}

}  // extern "C"
