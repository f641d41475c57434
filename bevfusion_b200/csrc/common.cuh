// Shared helpers for libbevfusion_b200 (sm_90a).  Internal header.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/bevfusion_b200.h"

namespace bevb200 {

constexpr int kNumSMs = 132;  // H100 SXM; grids are sized in multiples of this

// ---- error plumbing -------------------------------------------------------------------
extern thread_local char g_last_error[512];
extern thread_local long long g_launch_count;

#define BEVB200_REQUIRE(cond, msg)                                                      \
  do {                                                                                  \
    if (!(cond)) {                                                                      \
      snprintf(::bevb200::g_last_error, sizeof(::bevb200::g_last_error), "%s: %s [%s]", \
               __func__, msg, #cond);                                                   \
      return BEVB200_EINVAL;                                                            \
    }                                                                                   \
  } while (0)

#define BEVB200_CUDA(expr)                                                              \
  do {                                                                                  \
    cudaError_t e__ = (expr);                                                           \
    if (e__ != cudaSuccess) {                                                           \
      snprintf(::bevb200::g_last_error, sizeof(::bevb200::g_last_error), "%s: %s -> %s", \
               __func__, #expr, cudaGetErrorString(e__));                               \
      return BEVB200_ECUDA;                                                             \
    }                                                                                   \
  } while (0)

// Every kernel launch of the library goes through this so the launch counter is exact.
#define BEVB200_LAUNCH(kernel, grid, block, smem, stream, ...)                          \
  do {                                                                                  \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);                         \
    ++::bevb200::g_launch_count;                                                        \
    BEVB200_CUDA(cudaGetLastError());                                                   \
  } while (0)

inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// Bump allocator over a caller-provided workspace.
struct Arena {
  char *base;
  size_t size, off;
  Arena(void *p, size_t n) : base((char *)p), size(n), off(0) {}
  template <typename T>
  T *take(size_t count) {
    size_t bytes = align_up(count * sizeof(T));
    char *p = base ? base + off : nullptr;
    off += bytes;
    return (T *)p;
  }
  bool ok() const { return off <= size; }
};

inline int grid_for(long long work_items, int block, int max_blocks = kNumSMs * 16) {
  long long g = (work_items + block - 1) / block;
  if (g < 1) g = 1;
  if (g > max_blocks) g = max_blocks;
  return (int)g;
}

// ---- device helpers -------------------------------------------------------------------
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ void stg_stream_f4(float4 *p, const float4 &v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// Exclusive prefix sum of `count` uint32 values (in place allowed: out may alias in), total
// written to *total.  Three launches (tile sums, scan of tile sums, apply); `tile_sums` is
// scratch of scan_scratch_elems(count) uint32.
constexpr int kScanTile = 4096;  // elements per CTA (256 threads x 16)
inline size_t scan_scratch_elems(size_t count) { return (count + kScanTile - 1) / kScanTile + 1; }
int exclusive_scan_u32(const uint32_t *in, uint32_t *out, size_t count, uint32_t *tile_sums,
                       uint32_t *total, bool popc_input, cudaStream_t stream);

}  // namespace bevb200
