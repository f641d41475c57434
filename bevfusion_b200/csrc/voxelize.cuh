// Hard-voxelizer front (K1-K4 of voxelize.cu) shared with the fused consumers of its per-voxel slot
// lists: the mean reduce (voxelize.cu) and the pillar feature net (pillars.cu).  Internal header.
#pragma once
#include "common.cuh"

namespace bevb200 {

struct VoxParams {
  float vs[3], lo[3];
  int grid[3];
};

__device__ __forceinline__ bool point_coords(const float *__restrict__ p, const VoxParams &vp,
                                             int c[3]) {
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    // voxelization_cuda.cu:37,43,50: floor((p - min) / voxel) evaluated in fp32
    float v = floorf(__fdiv_rn(__fsub_rn(p[k], vp.lo[k]), vp.vs[k]));
    // out-of-range (and NaN) points are dropped; compare in float so huge values cannot wrap
    ok = ok && (v >= 0.f) && (v < (float)vp.grid[k]);
    c[k] = ok ? (int)v : -1;
  }
  return ok;
}

// After K1-K4: a voxel is named by its provisional id pv; lists[pv * P + s] is the point index in
// slot s (sorted, the first min(counts[pv], P) entries are valid).  Point i is the first point of
// its voxel iff bit i of first_bits is set; the voxel's final id is then word_prefix[i / 32] plus the
// set bits below i in its word, and *total is the number of distinct voxels.
struct VoxWs {
  unsigned long long *keys;
  int32_t *slot_pvid, *point_slot, *point_pvid, *lists, *counts, *pvid_counter;
  uint32_t *first_bits, *word_prefix, *tiles, *total;
  uint32_t table_size;
  size_t nwords;
};

int make_params(const float *vs, const float *range, VoxParams *vp);

// K1-K4 on n > 0 points, or on the first min(*n_dev, n) of them when n_dev (device int32) is not null;
// BEVB200_EWORKSPACE when the workspace is smaller than bevb200_hard_voxelize_workspace_bytes(n, max_points)
int vox_front(const char *who, const float *points, int n, const int32_t *n_dev, int num_features,
              const VoxParams &vp, int max_points, void *workspace, size_t workspace_bytes, cudaStream_t st,
              VoxWs *wout);

}  // namespace bevb200
