// BEV pooling and the fused LSS lift: everything bevpool.cu and bevpool_lift.cu share.  Internal header.
//
//   bevpool.cu       pooling forward / backward, the row form of the fused lift, the prepare_* tables
//   bevpool_lift.cu  column form of the fused lift and both lift backwards
#pragma once
#include <type_traits>

#include "common.cuh"

namespace bevb200 {

struct PoolDims {
  int b, d, h, w;
};

__device__ __forceinline__ long long cell_of(const int32_t *__restrict__ geom_feats, int row,
                                             const PoolDims dm) {
  // flat index into out[b][d][h][w] from (x, y, z, b) = geom_feats[row] (bev_pool_cuda.cu:34-36)
  int4 g = *reinterpret_cast<const int4 *>(geom_feats + 4ll * row);
  if ((unsigned)g.x >= (unsigned)dm.h || (unsigned)g.y >= (unsigned)dm.w ||
      (unsigned)g.z >= (unsigned)dm.d || (unsigned)g.w >= (unsigned)dm.b)
    return -1;
  return (((long long)g.w * dm.d + g.z) * dm.h + g.x) * dm.w + g.y;
}

// cell of the interval that starts at sorted row s; -1 outside the grid or when s is outside [0, n).
// The entries refuse grids of 2^31 cells or more, so the cell fits in an int32.
__device__ __forceinline__ int32_t interval_cell(const int32_t *__restrict__ geom_feats, int s, int n,
                                                 const PoolDims dm) {
  return (int32_t)(s >= 0 && s < n ? cell_of(geom_feats, s, dm) : -1);
}

// Sync-free plans (the *_dev entries): the kernels take a nullable `counts` = {n_kept, n_intervals} in device memory
// that replaces the host n / n_intervals they were sized for, and the fused-lift kernels a nullable `lift_form`, the
// status word of bevb200_bev_pool_lift_prepare_dev: a kernel whose form it does not name exits at once, so both forms
// can be launched and the device picks one.
__device__ __forceinline__ void device_counts(const int32_t *counts, int &n, int &n_intervals) {
  if (counts) {
    n = __ldg(counts);
    n_intervals = __ldg(counts + 1);
  }
}
__device__ __forceinline__ bool form_off(const int32_t *lift_form, int32_t form) {
  return lift_form != nullptr && __ldg(lift_form) != form;
}

// cells[i] = interval_cell(starts[i]) for every interval (defined in bevpool.cu)
__global__ void pool_interval_cells_kernel(const int32_t *__restrict__ geom_feats,
                                           const int32_t *__restrict__ starts, int n, int n_intervals,
                                           PoolDims dm, int32_t *__restrict__ cells,
                                           const int32_t *__restrict__ counts);

// out[0 .. n_floats) = 0 unless `lift_form` names another form or, given `only_if_empty` = device {n_kept,
// n_intervals}, the tables are not empty (defined in bevpool.cu)
int zero_fill(float *out, size_t n_floats, const int32_t *lift_form, int32_t form, cudaStream_t st,
              const int32_t *only_if_empty = nullptr);

// BEVB200_EWORKSPACE, with the error text, when the caller's workspace is smaller than `need` bytes
inline int workspace_check(const char *who, const void *ws, size_t ws_bytes, size_t need) {
  if (ws != nullptr && ws_bytes >= need) return BEVB200_OK;
  snprintf(g_last_error, sizeof(g_last_error), "%s: workspace too small (%zu < %zu)", who, ws_bytes, need);
  return BEVB200_EWORKSPACE;
}

// The channel widths C that have tuned kernels; each runs with Q = C / 4 float4 per row.
template <int... C>
struct ChannelWidths {
  static constexpr bool has(int c) { return ((c == C) || ...); }
  // f(std::integral_constant<int, c / 4>{}) and the status it returns; a width without a kernel sets the error text
  // and gives BEVB200_EINVAL
  template <typename F>
  static int dispatch(int c, F &&f) {
    int rc = BEVB200_EINVAL;
    const bool tuned = ((c == C && ((rc = f(std::integral_constant<int, C / 4>{})), true)) || ...);
    if (!tuned) snprintf(g_last_error, sizeof(g_last_error), "no tuned BEV pooling kernel for %d channels", c);
    return rc;
  }
};
using TunedWidths = ChannelWidths<16, 32, 64, 80, 96, 128, 160, 256>;

}  // namespace bevb200
