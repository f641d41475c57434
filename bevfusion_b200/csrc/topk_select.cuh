// Exact top-K of a sample's candidate keys, shared by the TransFusion query proposals (transfusion_proposals.cu) and
// the CenterHead box decode (centerhead_decode.cu).  Internal header.
//
// A first kernel of each user writes, per tile of kTile consecutive flat cells, the 64-bit keys of the tile's
// candidate cells to the tile's slice of the workspace ([tiles, kTile] keys) and the tile's count ([tiles]).
// key(v) is the float's order-preserving unsigned image with every NaN mapped to the top, and the 64-bit key is
// key(v) << 32 | ~flat, so descending 64-bit order is (v descending, NaN first; ties by ascending flat index):
// argsort(descending=True, stable=True).  Every key is distinct, so the selected set and its order are fixed and the
// result is the same bit for bit on every run, whatever order the candidates were counted in.
//
// select_top_keys, called by a whole CTA of kSelectThreads threads, leaves the min(n, K) largest keys in descending
// order in shared memory: an MSD radix select (8-bit digits) of the K-th largest key over the candidates, which moves
// the keys under the current prefix to shared memory as soon as they fit (kBufCap), so the global list is typically
// read twice, then a bitonic sort of the winners.
#pragma once
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace bevb200 {
namespace topk {

constexpr int kTile = 1024;            // cells per candidate tile, and key slots per tile
constexpr int kSelectThreads = 1024;
constexpr int kBufCap = 4096;          // keys of the threshold bin the select moves to shared memory
constexpr int kSelectWarps = kSelectThreads / 32;

// torch's sigmoid_kernel_cuda: opmath (fp32) 1 / (1 + exp(-x)), returned in the input's dtype
template <typename T>
__device__ __forceinline__ float sigmoid_as(float x) {
  const float s = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x)));
  if constexpr (sizeof(T) == 2) return __half2float(__float2half_rn(s));
  return s;
}

__device__ __forceinline__ uint32_t order_key(float m) {
  if (isnan(m)) return 0xffffffffu;
  const uint32_t u = __float_as_uint(m);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ uint64_t full_key(float m, int flat) {
  return ((uint64_t)order_key(m) << 32) | (uint32_t)~(uint32_t)flat;
}

// The flat cell index of a key.
__device__ __forceinline__ uint32_t key_flat(uint64_t key) { return ~(uint32_t)key; }

// Writes a tile's kept keys, in the order (r, thread), to its workspace slice and the tile's count.  Thread tid
// holds kCells keys; `keep` of each is given as the warp's ballot bal[r].  Called by a whole CTA of kThreads threads.
template <int kThreads, int kCells>
__device__ __forceinline__ void write_tile_keys(const uint64_t (&key)[kCells], const unsigned (&bal)[kCells],
                                                uint64_t *__restrict__ dst, int32_t *__restrict__ tile_count) {
  constexpr int kWarps = kThreads / 32, kSlots = kCells * kWarps;
  static_assert(kSlots <= 32, "one warp scans the slot counts");
  __shared__ int base[kSlots + 1];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int r = 0; r < kCells; ++r)
    if (lane == 0) base[r * kWarps + warp] = __popc(bal[r]);
  __syncthreads();
  if (warp == 0) {                                // exclusive scan of the kSlots warp counts
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
#pragma unroll
  for (int r = 0; r < kCells; ++r)
    if ((bal[r] >> lane) & 1u) dst[base[r * kWarps + warp] + __popc(bal[r] & ((1u << lane) - 1u))] = key[r];
  if (tid == 0) *tile_count = base[kSlots];
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
__device__ inline void bitonic_desc(uint64_t *s, int n) {
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

// The K largest of one sample's candidate keys (all of them when there are at most K), sorted descending into
// sel[0, nsel) with sel[nsel, sort_n) = 0; returns nsel = min(n, K).  sel [sort_n] and buf [kBufCap] are shared
// memory, sort_n = sort_size(K).  Called by a whole CTA of kSelectThreads threads; ends with a barrier.
__device__ inline int select_top_keys(const uint64_t *__restrict__ cand, const int32_t *__restrict__ count,
                                      int tiles, int K, int sort_n, uint64_t *sel, uint64_t *buf) {
  __shared__ uint32_t hist[256];
  __shared__ int red[kSelectWarps];
  __shared__ int sh_n, sh_count, sh_nbuf, sh_digit, sh_above, sh_bin;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  int local = 0;
  for (int t = tid; t < tiles; t += kSelectThreads) local += count[t];
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
      for_each_candidate(cand, count, tiles, f);
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
  return nsel;
}

inline int sort_size(int K) {
  int n = 32;
  while (n < K) n <<= 1;
  return n;
}

}  // namespace topk
}  // namespace bevb200
