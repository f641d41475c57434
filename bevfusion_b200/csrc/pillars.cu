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
#include "voxelize.cuh"

namespace bevb200 {

constexpr int kPfnMaxF = 8, kPfnMaxP = 32, kPfnC1 = 32, kPfnC2 = 64;
constexpr int kPfnK1 = 16;  // layer-1 input columns: raw 0..7, cluster offset 8..10, centre offset 11..12
// packed fp32 image: w1 [32][16] | s1 [32] | t1 [32] | w2a [64][32] | w2b^T [32][64] | s2 [64] | t2 [64]
constexpr int kPfnW1 = 0, kPfnS1 = kPfnW1 + kPfnC1 * kPfnK1, kPfnT1 = kPfnS1 + kPfnC1,
              kPfnW2a = kPfnT1 + kPfnC1, kPfnW2b = kPfnW2a + kPfnC2 * kPfnC1,
              kPfnS2 = kPfnW2b + kPfnC1 * kPfnC2, kPfnT2 = kPfnS2 + kPfnC2, kPfnPacked = kPfnT2 + kPfnC2;
constexpr int kPfnWarps = 4;

struct PfnGeom {
  float vx, vy, x_off, y_off;  // pillar centre = idx * v + off (pillar_encoder.py:135-138)
};

struct __align__(16) PfnWarpSmem {
  float pts[kPfnMaxP][kPfnMaxF];  // raw point rows, columns >= F zero
  float x1[kPfnMaxP][kPfnC1];     // layer-1 output rows (the virtual row last)
  float m1[kPfnC1];               // layer-1 max
};

struct PfnLane {
  float w1[kPfnK1], s1, t1;
  float w2a0[kPfnC1], w2a1[kPfnC1], s20, t20, s21, t21;
};

__device__ __forceinline__ void pfn_load_lane(const float *__restrict__ pk, int lane, PfnLane &w) {
#pragma unroll
  for (int k = 0; k < kPfnK1; ++k) w.w1[k] = pk[kPfnW1 + lane * kPfnK1 + k];
  w.s1 = pk[kPfnS1 + lane];
  w.t1 = pk[kPfnT1 + lane];
#pragma unroll
  for (int k = 0; k < kPfnC1; ++k) {
    w.w2a0[k] = pk[kPfnW2a + lane * kPfnC1 + k];
    w.w2a1[k] = pk[kPfnW2a + (lane + 32) * kPfnC1 + k];
  }
  w.s20 = pk[kPfnS2 + lane];
  w.t20 = pk[kPfnT2 + lane];
  w.s21 = pk[kPfnS2 + lane + 32];
  w.t21 = pk[kPfnT2 + lane + 32];
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One pillar on one warp.  s.pts holds rows 0..cnt-1; (sx, sy, sz) is the xyz sum over its slots, n the
// reference's num_voxels.  Returns layer-2 channels lane and lane + 32.
__device__ __forceinline__ void pfn_pillar(PfnWarpSmem &s, const float *__restrict__ w2bT, const PfnLane &w,
                                           int lane, int n, int cnt, bool virt, float sx, float sy, float sz,
                                           int cx, int cy, const PfnGeom &g, float &o0, float &o1) {
  const float fn = (float)n;
  const float mx = __fdiv_rn(sx, fn), my = __fdiv_rn(sy, fn), mz = __fdiv_rn(sz, fn);
  // coors * v + offset, two roundings as in the reference (no contraction into an FMA)
  const float xc = __fadd_rn(__fmul_rn((float)cx, g.vx), g.x_off);
  const float yc = __fadd_rn(__fmul_rn((float)cy, g.vy), g.y_off);
  float best = -INFINITY;
  for (int r = 0; r < cnt; ++r) {
    const float4 a = *reinterpret_cast<const float4 *>(&s.pts[r][0]);
    const float4 b = *reinterpret_cast<const float4 *>(&s.pts[r][4]);
    const float d[13] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w,
                         __fsub_rn(a.x, mx), __fsub_rn(a.y, my), __fsub_rn(a.z, mz),
                         __fsub_rn(a.x, xc), __fsub_rn(a.y, yc)};
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 13; ++k) acc = fmaf(w.w1[k], d[k], acc);
    const float y = fmaxf(fmaf(acc, w.s1, w.t1), 0.f);
    s.x1[r][lane] = y;
    best = fmaxf(best, y);
  }
  if (virt) {  // the padded slots: zero input row
    const float y = fmaxf(w.t1, 0.f);
    s.x1[cnt][lane] = y;
    best = fmaxf(best, y);
  }
  s.m1[lane] = best;
  __syncwarp();
  float b0 = 0.f, b1 = 0.f;
#pragma unroll 8
  for (int k = 0; k < kPfnC1; ++k) {
    const float m = s.m1[k];
    b0 = fmaf(w2bT[k * kPfnC2 + lane], m, b0);
    b1 = fmaf(w2bT[k * kPfnC2 + lane + 32], m, b1);
  }
  float best0 = -INFINITY, best1 = -INFINITY;
  const int rows = cnt + (virt ? 1 : 0);
  for (int r = 0; r < rows; ++r) {
    float a0 = b0, a1 = b1;
#pragma unroll
    for (int k = 0; k < kPfnC1; k += 4) {
      const float4 x = *reinterpret_cast<const float4 *>(&s.x1[r][k]);
      a0 = fmaf(w.w2a0[k], x.x, a0); a1 = fmaf(w.w2a1[k], x.x, a1);
      a0 = fmaf(w.w2a0[k + 1], x.y, a0); a1 = fmaf(w.w2a1[k + 1], x.y, a1);
      a0 = fmaf(w.w2a0[k + 2], x.z, a0); a1 = fmaf(w.w2a1[k + 2], x.z, a1);
      a0 = fmaf(w.w2a0[k + 3], x.w, a0); a1 = fmaf(w.w2a1[k + 3], x.w, a1);
    }
    best0 = fmaxf(best0, fmaf(a0, w.s20, w.t20));
    best1 = fmaxf(best1, fmaf(a1, w.s21, w.t21));
  }
  o0 = fmaxf(best0, 0.f);  // relu commutes with max
  o1 = fmaxf(best1, 0.f);
  __syncwarp();  // the next pillar overwrites s
}

// load one point row (F <= 8) into s.pts[lane], zero-padded to 8 columns; returns its xyz
__device__ __forceinline__ float3 pfn_stage_row(PfnWarpSmem &s, int lane, const float *__restrict__ row, int F) {
  float r[kPfnMaxF];
#pragma unroll
  for (int k = 0; k < kPfnMaxF; ++k) r[k] = k < F ? row[k] : 0.f;
  *reinterpret_cast<float4 *>(&s.pts[lane][0]) = make_float4(r[0], r[1], r[2], r[3]);
  *reinterpret_cast<float4 *>(&s.pts[lane][4]) = make_float4(r[4], r[5], r[6], r[7]);
  return make_float3(r[0], r[1], r[2]);
}

__device__ __forceinline__ void pfn_block_setup(const float *__restrict__ packed, float *w2bT, PfnLane &w) {
  for (int i = threadIdx.x; i < kPfnC1 * kPfnC2; i += blockDim.x) w2bT[i] = packed[kPfnW2b + i];
  pfn_load_lane(packed, lane_id(), w);
  __syncthreads();
}

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

// W1 [32, F+5], W2 [64, 64] row-major (nn.Linear layout); s/t the folded BN scale / shift
__global__ void pillar_pack_kernel(const float *__restrict__ W1, const float *__restrict__ s1,
                                   const float *__restrict__ t1, const float *__restrict__ W2,
                                   const float *__restrict__ s2, const float *__restrict__ t2, int F,
                                   float *__restrict__ packed) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kPfnPacked; i += gridDim.x * blockDim.x) {
    float v;
    if (i < kPfnS1) {
      const int c = i / kPfnK1, k = i % kPfnK1;
      const int col = k < kPfnMaxF ? (k < F ? k : -1) : (k < 13 ? F + k - kPfnMaxF : -1);
      v = col >= 0 ? W1[c * (F + 5) + col] : 0.f;
    } else if (i < kPfnT1) {
      v = s1[i - kPfnS1];
    } else if (i < kPfnW2a) {
      v = t1[i - kPfnT1];
    } else if (i < kPfnW2b) {
      const int o = (i - kPfnW2a) / kPfnC1, k = (i - kPfnW2a) % kPfnC1;
      v = W2[o * kPfnC2 + k];
    } else if (i < kPfnS2) {
      const int k = (i - kPfnW2b) / kPfnC2, o = (i - kPfnW2b) % kPfnC2;
      v = W2[o * kPfnC2 + kPfnC1 + k];
    } else if (i < kPfnT2) {
      v = s2[i - kPfnS2];
    } else {
      v = t2[i - kPfnT2];
    }
    packed[i] = v;
  }
}

static bool pfn_native(int F, int P) { return F >= 3 && F <= kPfnMaxF && P >= 1 && P <= kPfnMaxP; }

#define BEVB200_UNSUPPORTED(cond, msg)                                                  \
  do {                                                                                  \
    if (!(cond)) {                                                                      \
      snprintf(::bevb200::g_last_error, sizeof(::bevb200::g_last_error), "%s: %s [%s]", \
               __func__, msg, #cond);                                                   \
      return BEVB200_EUNSUPPORTED;                                                      \
    }                                                                                   \
  } while (0)

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
  int rc = vox_front("hard_voxelize_pillars", points, n, num_features, vp, max_points, workspace, workspace_bytes,
                     st, &w);
  if (rc) return rc;
  const PfnGeom g{vx, vy, x_off, y_off};
  BEVB200_LAUNCH(pillar_canvas_kernel, grid_for((long long)w.nwords, kPfnWarps), kPfnWarps * 32, 0, st, points,
                 num_features, vp, max_points, max_voxels, g, w.point_pvid, w.lists, w.counts, w.first_bits,
                 w.word_prefix, w.total, (long long)w.nwords, packed, canvas, voxel_num);
  return BEVB200_OK;
}

}  // extern "C"
