// PointPillars pillar feature net for sm_90a: decoration + PFN layer 1 (F+5 -> 32, BN, ReLU, max, concat)
// + PFN layer 2 (64 -> 64, BN, ReLU, max) of mmdet3d/models/backbones/pillar_encoder.py:43-176, one warp
// per pillar, nothing but the [64] result per pillar leaves the chip.
//
// Semantics kept from the reference (DESIGN 4.11):
//   - mean_xyz = (sum over all P slots) / n; slots s >= n are zero rows after decoration (:141-176)
//   - both layers run on all P slots, so a pillar with n < P has one extra "virtual" row (a zero input
//     row: layer 1 gives relu(shift1)) that takes part in both maxes; a pillar with n == P has none
//   - BN is folded per channel (eval statistics) and applied per row before the max, so negative BN
//     scales need no special case
//   - the layer-2 linear over [x1, max1] is split into W2a * x1 (per row) + W2b * max1 (per pillar)
//
// Lane c owns layer-1 channel c and layer-2 channels c and c + 32, so both maxes are lane-local and
// the weights of a lane stay in registers for the whole kernel.  The pillar's rows go through shared
// memory (broadcast reads).  Exact fp32 FMA arithmetic, no atomics: the output is bit-reproducible
// and does not depend on which warp handles which pillar.
//
// Two row sources share that core: the [M, P, F] voxel tensor (PillarFeatureNet contract, rows out)
// and the hard voxelizer's per-voxel slot lists (K1-K4 of voxelize.cu), which never writes [M, P, F]
// and stores straight into the channels-first BEV canvas.
#include "pillars.cuh"
#include "voxelize.cuh"

namespace bevb200 {

// rows source: the [M, P, F] voxel tensor; out [M, 64]
__global__ void __launch_bounds__(kPfnWarps * 32)
    pillar_rows_kernel(const float *__restrict__ voxels, const int32_t *__restrict__ num_points,
                       const int32_t *__restrict__ coords4, int cap, const int32_t *__restrict__ n_dev, int P,
                       int F, PfnGeom g, const float *__restrict__ packed, float *__restrict__ out) {
  __shared__ PfnWarpSmem sm[kPfnWarps];
  __shared__ float w2bT[kPfnC1 * kPfnC2];
  PfnLane w;
  pfn_block_setup(packed, w2bT, w);
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  PfnWarpSmem &s = sm[warp];
  const int m = n_dev ? min(*n_dev, cap) : cap;
  for (int v = blockIdx.x * kPfnWarps + warp; v < m; v += gridDim.x * kPfnWarps) {
    const int n = num_points[v];
    float3 p = make_float3(0.f, 0.f, 0.f);
    if (lane < P) p = pfn_stage_row(s, lane, voxels + ((long long)v * P + lane) * F, F);  // all P slots
    const float sx = warp_sum(p.x), sy = warp_sum(p.y), sz = warp_sum(p.z);
    __syncwarp();
    const int cnt = min(n, P);
    float o0, o1;
    pfn_pillar(s, w2bT, w, lane, n, cnt, cnt < P, sx, sy, sz, coords4[4ll * v + 1], coords4[4ll * v + 2], g, o0,
               o1);
    out[(long long)v * kPfnC2 + lane] = o0;
    out[(long long)v * kPfnC2 + lane + 32] = o1;
  }
}

// rows source: the voxelizer's slot lists (after K1-K4); one warp per 32-point word of first-point
// flags, every voxel whose first point lies in the word in turn.  canvas [64, grid_x, grid_y].
__global__ void __launch_bounds__(kPfnWarps * 32)
    pillar_canvas_kernel(const float *__restrict__ points, int F, VoxParams vp, int P, int max_voxels, PfnGeom g,
                         const int32_t *__restrict__ point_pvid, const int32_t *__restrict__ lists,
                         const int32_t *__restrict__ counts, const uint32_t *__restrict__ first_bits,
                         const uint32_t *__restrict__ word_prefix, const uint32_t *__restrict__ total_voxels,
                         long long nwords, const float *__restrict__ packed, float *__restrict__ canvas,
                         int32_t *__restrict__ voxel_num) {
  __shared__ PfnWarpSmem sm[kPfnWarps];
  __shared__ float w2bT[kPfnC1 * kPfnC2];
  if (blockIdx.x == 0 && threadIdx.x == 0)
    *voxel_num = (int32_t)min(*total_voxels, (uint32_t)max_voxels);
  PfnLane w;
  pfn_block_setup(packed, w2bT, w);
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  PfnWarpSmem &s = sm[warp];
  const long long plane = (long long)vp.grid[0] * vp.grid[1];
  for (long long wd = blockIdx.x * kPfnWarps + warp; wd < nwords; wd += (long long)gridDim.x * kPfnWarps) {
    uint32_t bits = first_bits[wd];
    const uint32_t vid0 = word_prefix[wd];
    for (uint32_t rank = 0; bits != 0u; ++rank, bits &= bits - 1u) {
      if (vid0 + rank >= (uint32_t)max_voxels) break;  // voxel ids grow with the first point index
      const int i = (int)(wd * 32 + __ffs(bits) - 1);
      const int pv = point_pvid[i];
      const int cnt = min(counts[pv], P);
      float3 p = make_float3(0.f, 0.f, 0.f);
      if (lane < cnt) p = pfn_stage_row(s, lane, points + (long long)lists[(long long)pv * P + lane] * F, F);
      const float sx = warp_sum(p.x), sy = warp_sum(p.y), sz = warp_sum(p.z);
      int c[3];
      point_coords(points + (long long)i * F, vp, c);
      __syncwarp();
      float o0, o1;
      pfn_pillar(s, w2bT, w, lane, cnt, cnt, cnt < P, sx, sy, sz, c[0], c[1], g, o0, o1);
      float *o = canvas + (long long)c[0] * vp.grid[1] + c[1];
      o[lane * plane] = o0;
      o[(lane + 32) * plane] = o1;
    }
  }
}

}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_pillar_packed_bytes(int in_channels, int c1, int c2) {
  if (in_channels < 3 || in_channels > kPfnMaxF || c1 != kPfnC1 || c2 != kPfnC2) return 0;
  return kPfnPacked * sizeof(float);
}

int bevb200_pillar_pack_weights(const float *w1, const float *scale1, const float *shift1, const float *w2,
                                const float *scale2, const float *shift2, int in_channels, int c1, int c2,
                                float *packed, void *stream) {
  BEVB200_UNSUPPORTED(bevb200_pillar_packed_bytes(in_channels, c1, c2) > 0,
                      "native pillar net: in_channels 3..8, feat_channels [64, 64]");
  BEVB200_REQUIRE(w1 && scale1 && shift1 && w2 && scale2 && shift2 && packed, "null argument");
  BEVB200_LAUNCH(pillar_pack_kernel, grid_for(kPfnPacked, 256), 256, 0, (cudaStream_t)stream, w1, scale1, shift1,
                 w2, scale2, shift2, in_channels, packed);
  return BEVB200_OK;
}

int bevb200_pillar_features(const float *voxels, const int32_t *num_points, const int32_t *coords4, int cap,
                            const int32_t *n_dev, int max_points, int num_features, float vx, float vy, float x_off,
                            float y_off, const float *packed, float *out_rows, void *stream) {
  BEVB200_UNSUPPORTED(pfn_native(num_features, max_points), "native pillar net: F 3..8, P 1..32");
  BEVB200_REQUIRE(cap >= 0, "bad sizes");
  if (cap == 0) return BEVB200_OK;
  BEVB200_REQUIRE(voxels && num_points && coords4 && packed && out_rows, "null argument");
  const PfnGeom g{vx, vy, x_off, y_off};
  BEVB200_LAUNCH(pillar_rows_kernel, grid_for(cap, kPfnWarps), kPfnWarps * 32, 0, (cudaStream_t)stream, voxels,
                 num_points, coords4, cap, n_dev, max_points, num_features, g, packed, out_rows);
  return BEVB200_OK;
}

int bevb200_hard_voxelize_pillars(const float *points, int num_points, int num_features,
                                  const float *voxel_size_host, const float *coors_range_host, int max_points,
                                  int max_voxels, float vx, float vy, float x_off, float y_off, const float *packed,
                                  float *canvas, int nx, int ny, int32_t *voxel_num, void *workspace,
                                  size_t workspace_bytes, void *stream) {
  BEVB200_UNSUPPORTED(pfn_native(num_features, max_points), "native pillar net: F 3..8, P 1..32");
  BEVB200_REQUIRE(num_points >= 0 && max_voxels > 0, "bad sizes");
  BEVB200_REQUIRE(voxel_size_host && coors_range_host && voxel_num, "null argument");
  VoxParams vp;
  BEVB200_REQUIRE(make_params(voxel_size_host, coors_range_host, &vp) == 0, "bad voxel grid");
  BEVB200_UNSUPPORTED(vp.grid[2] == 1, "pillars need a voxel grid one cell high");
  BEVB200_REQUIRE(vp.grid[0] == nx && vp.grid[1] == ny, "canvas shape differs from the voxel grid");
  cudaStream_t st = (cudaStream_t)stream;
  const int n = num_points;
  if (n == 0) {
    BEVB200_CUDA(cudaMemsetAsync(voxel_num, 0, sizeof(int32_t), st));
    return BEVB200_OK;
  }
  BEVB200_REQUIRE(points && packed && canvas, "null argument");
  VoxWs w;
  int rc = vox_front("hard_voxelize_pillars", points, n, nullptr, num_features, vp, max_points, workspace, workspace_bytes,
                     st, &w);
  if (rc) return rc;
  const PfnGeom g{vx, vy, x_off, y_off};
  BEVB200_LAUNCH(pillar_canvas_kernel, grid_for((long long)w.nwords, kPfnWarps), kPfnWarps * 32, 0, st, points,
                 num_features, vp, max_points, max_voxels, g, w.point_pvid, w.lists, w.counts, w.first_bits,
                 w.word_prefix, w.total, (long long)w.nwords, packed, canvas, voxel_num);
  return BEVB200_OK;
}

}  // extern "C"
