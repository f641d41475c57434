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
// max_pool2d does.  Built without fast-math, as the whole library is.
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace bevb200 {
namespace {

constexpr int kPeakThreads = 256;
constexpr int kCellsPerThread = 4;
constexpr int kTile = kPeakThreads * kCellsPerThread;   // cells per peak CTA, and key slots per tile
constexpr int kSelectThreads = 1024;
constexpr int kBufCap = 4096;          // keys of the threshold bin the select moves to shared memory
constexpr int kSelectWarps = kSelectThreads / 32;
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

// torch's sigmoid_kernel_cuda: opmath (fp32) 1 / (1 + exp(-x)), returned in the input's dtype
template <typename T>
__device__ __forceinline__ float sigmoid_as(float x) {
  const float s = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x)));
  if constexpr (sizeof(T) == 2) return __half2float(__float2half_rn(s));
  return s;
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

__device__ __forceinline__ uint32_t order_key(float m) {
  if (isnan(m)) return 0xffffffffu;
  const uint32_t u = __float_as_uint(m);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ uint64_t full_key(float m, int flat) {
  return ((uint64_t)order_key(m) << 32) | (uint32_t)~(uint32_t)flat;
}

// Thread tid handles cells tile * kTile + r * kPeakThreads + tid, r = 0..kCellsPerThread-1; the tile's keepers are
// written in that (flat index) order.
template <typename T>
__global__ void __launch_bounds__(kPeakThreads, 1)
    tf_peak_kernel(const T *__restrict__ x, const __grid_constant__ PropParams p, uint64_t *__restrict__ cand,
                   int32_t *__restrict__ tile_count) {
  constexpr int kWarps = kPeakThreads / 32, kSlots = kCellsPerThread * kWarps;
  __shared__ int base[kSlots + 1];
  const int b = blockIdx.y, tile = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
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
    if (lane == 0) base[r * kWarps + warp] = __popc(bal[r]);
  }
  __syncthreads();
  if (warp == 0) {                                // exclusive scan of the kSlots = 32 warp counts
    const int v = lane < kSlots ? base[lane] : 0;
    int incl = v;
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    if (lane < kSlots) base[lane] = incl - v;
    if (lane == 31) base[kSlots] = incl;
  }
  __syncthreads();
  uint64_t *dst = cand + ((long long)b * p.tiles + tile) * kTile;
#pragma unroll
  for (int r = 0; r < kCellsPerThread; ++r)
    if ((bal[r] >> lane) & 1u) dst[base[r * kWarps + warp] + __popc(bal[r] & ((1u << lane) - 1u))] = key[r];
  if (tid == 0) tile_count[(long long)b * p.tiles + tile] = base[kSlots];
}

// Visits every candidate key of one sample: each warp takes whole tiles, its lanes the tile's entries, four loads
// in flight per lane.
template <typename F>
__device__ __forceinline__ void for_each_candidate(const uint64_t *__restrict__ cand,
                                                   const int32_t *__restrict__ count, int tiles, F f) {
  constexpr int kUnroll = 4;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t = warp; t < tiles; t += kSelectWarps) {
    const int n = count[t];
    const uint64_t *src = cand + (long long)t * kTile;
    for (int base = 0; base < n; base += 32 * kUnroll) {
      uint64_t v[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const int i = base + u * 32 + lane;
        v[u] = i < n ? src[i] : 0;
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u)
        if (base + u * 32 + lane < n) f(v[u]);
    }
  }
}

// Descending bitonic sort of s[0, n), n a power of two, by the whole CTA.
__device__ void bitonic_desc(uint64_t *s, int n) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const uint64_t a = s[i], c = s[ixj];
          if ((i & k) == 0 ? a < c : a > c) {
            s[i] = c;
            s[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  }
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
  __shared__ uint32_t hist[256];
  __shared__ int red[kSelectWarps];
  __shared__ int sh_n, sh_count, sh_nbuf, sh_digit, sh_above, sh_bin;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int K = p.K;
  const uint64_t *cand = cand_all + (long long)b * p.tiles * kTile;
  const int32_t *count = count_all + (long long)b * p.tiles;

  int local = 0;
  for (int t = tid; t < p.tiles; t += kSelectThreads) local += count[t];
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if (lane == 0) red[warp] = local;
  if (tid == 0) {
    sh_count = 0;
    sh_nbuf = 0;
  }
  __syncthreads();
  if (tid == 0) {
    int n = 0;
    for (int i = 0; i < kSelectWarps; ++i) n += red[i];
    sh_n = n;
  }
  __syncthreads();
  const int n = sh_n;

  // the keys still in play: every candidate, or (in_buf) the ones under the prefix moved to shared memory
  bool in_buf = false;
  auto visit = [&](auto f) {
    if (in_buf) {
      const int nb = sh_nbuf;
      for (int i = tid; i < nb; i += kSelectThreads) f(buf[i]);
    } else {
      for_each_candidate(cand, count, p.tiles, f);
    }
  };
  // gathers a winner; `sel` has room for K
  auto take = [&](uint64_t e) {
    const int pos = atomicAdd(&sh_count, 1);
    if (pos < sort_n) sel[pos] = e;
  };

  // the K-th largest key: keys whose masked top bits exceed `prefix` are in, and so are those equal to it
  uint64_t prefix = 0, mask = 0;
  if (n > K) {
    int remaining = K;
    for (int shift = 56; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += kSelectThreads) hist[i] = 0;
      __syncthreads();
      visit([&](uint64_t e) {
        const int d = (e & mask) == prefix ? (int)((e >> shift) & 255u) : 256;
        const unsigned peers = __match_any_sync(__activemask(), d);
        if (d < 256 && (int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&hist[d], (uint32_t)__popc(peers));
      });
      __syncthreads();
      if (warp == 0) {                            // lane l holds bins 255 - 8 l - j, j = 0..7, top down
        uint32_t mine[8], sum = 0;
        for (int j = 0; j < 8; ++j) {
          mine[j] = hist[255 - 8 * lane - j];
          sum += mine[j];
        }
        uint32_t incl = sum;
        for (int o = 1; o < 32; o <<= 1) {
          const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += v;
        }
        uint32_t above = incl - sum;
        if (above < (uint32_t)remaining && (uint32_t)remaining <= incl) {
          for (int j = 0; j < 8; ++j) {
            if ((uint32_t)remaining <= above + mine[j]) {
              sh_digit = 255 - 8 * lane - j;
              sh_above = (int)above;
              sh_bin = (int)mine[j];
              break;
            }
            above += mine[j];
          }
        }
      }
      __syncthreads();
      remaining -= sh_above;
      prefix |= (uint64_t)sh_digit << shift;
      mask |= (uint64_t)0xff << shift;
      const bool done = sh_bin == remaining;      // every key under this prefix is selected
      const bool fits = !in_buf && sh_bin <= kBufCap;
      __syncthreads();
      if (done) break;
      if (fits) {
        // one more pass over the candidates: the keys above the prefix are winners, the ones under it go to
        // shared memory, and the remaining digits are resolved there
        visit([&](uint64_t e) {
          const uint64_t top = e & mask;
          if (top > prefix) take(e);
          else if (top == prefix) buf[atomicAdd(&sh_nbuf, 1)] = e;
        });
        in_buf = true;
        __syncthreads();
      }
    }
  }

  // gather the (remaining) winners -- all candidates when there are at most K -- then sort them
  visit([&](uint64_t e) {
    if ((e & mask) >= prefix) take(e);
  });
  __syncthreads();
  const int nsel = min(sh_count, K);
  for (int i = nsel + tid; i < sort_n; i += kSelectThreads) sel[i] = 0;   // below every real key
  __syncthreads();
  bitonic_desc(sel, sort_n);
  for (int i = tid; i < nsel; i += kSelectThreads) win[i] = ~(uint32_t)sel[i];
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

int sort_size(int K) {
  int n = 32;
  while (n < K) n <<= 1;
  return n;
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
