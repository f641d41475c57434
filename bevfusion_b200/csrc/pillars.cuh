// PointPillars pillar feature net: the per-pillar arithmetic shared by the eval kernels (pillars.cu) and the
// training passes (pillars_train.cu).  Internal header.
#pragma once
#include "common.cuh"

namespace bevb200 {

constexpr int kPfnMaxF = 8, kPfnMaxP = 32, kPfnC1 = 32, kPfnC2 = 64;
constexpr int kPfnK1 = 16;  // layer-1 input columns: raw 0..7, cluster offset 8..10, centre offset 11..12
constexpr int kPfnD = 13;   // used layer-1 input columns
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

// the pillar's decoration constants: xyz mean over n points and the pillar centre
struct PfnCentre {
  float mx, my, mz, xc, yc;
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

__device__ __forceinline__ PfnCentre pfn_centre(int n, float sx, float sy, float sz, int cx, int cy,
                                                const PfnGeom &g) {
  const float fn = (float)n;
  PfnCentre c;
  c.mx = __fdiv_rn(sx, fn);
  c.my = __fdiv_rn(sy, fn);
  c.mz = __fdiv_rn(sz, fn);
  // coors * v + offset, two roundings as in the reference (no contraction into an FMA)
  c.xc = __fadd_rn(__fmul_rn((float)cx, g.vx), g.x_off);
  c.yc = __fadd_rn(__fmul_rn((float)cy, g.vy), g.y_off);
  return c;
}

// the 13 decorated columns of one staged point row
__device__ __forceinline__ void pfn_decorate(const float *row, const PfnCentre &c, float (&d)[kPfnD]) {
  const float4 a = *reinterpret_cast<const float4 *>(row);
  const float4 b = *reinterpret_cast<const float4 *>(row + 4);
  d[0] = a.x; d[1] = a.y; d[2] = a.z; d[3] = a.w; d[4] = b.x; d[5] = b.y; d[6] = b.z; d[7] = b.w;
  d[8] = __fsub_rn(a.x, c.mx); d[9] = __fsub_rn(a.y, c.my); d[10] = __fsub_rn(a.z, c.mz);
  d[11] = __fsub_rn(a.x, c.xc); d[12] = __fsub_rn(a.y, c.yc);
}

// layer-1 pre-BN value of one staged row for the lane's channel
__device__ __forceinline__ float pfn_z1(const float *row, const PfnCentre &c, const float (&w1)[kPfnK1]) {
  float d[kPfnD];
  pfn_decorate(row, c, d);
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < kPfnD; ++k) acc = fmaf(w1[k], d[k], acc);
  return acc;
}

// per-pillar part of layer 2: W2b * max1 for channels lane and lane + 32
__device__ __forceinline__ void pfn_w2b_max(const float *w2bT, const float *m1, int lane, float &b0, float &b1) {
  b0 = 0.f;
  b1 = 0.f;
#pragma unroll 8
  for (int k = 0; k < kPfnC1; ++k) {
    const float m = m1[k];
    b0 = fmaf(w2bT[k * kPfnC2 + lane], m, b0);
    b1 = fmaf(w2bT[k * kPfnC2 + lane + 32], m, b1);
  }
}

// layer-2 pre-BN values of one layer-1 row: a0 / a1 enter as the per-pillar part
__device__ __forceinline__ void pfn_z2(const float *x1row, const PfnLane &w, float &a0, float &a1) {
#pragma unroll
  for (int k = 0; k < kPfnC1; k += 4) {
    const float4 x = *reinterpret_cast<const float4 *>(x1row + k);
    a0 = fmaf(w.w2a0[k], x.x, a0); a1 = fmaf(w.w2a1[k], x.x, a1);
    a0 = fmaf(w.w2a0[k + 1], x.y, a0); a1 = fmaf(w.w2a1[k + 1], x.y, a1);
    a0 = fmaf(w.w2a0[k + 2], x.z, a0); a1 = fmaf(w.w2a1[k + 2], x.z, a1);
    a0 = fmaf(w.w2a0[k + 3], x.w, a0); a1 = fmaf(w.w2a1[k + 3], x.w, a1);
  }
}

// One pillar on one warp.  s.pts holds rows 0..cnt-1; (sx, sy, sz) is the xyz sum over its slots, n the
// reference's num_voxels.  Returns layer-2 channels lane and lane + 32.
__device__ __forceinline__ void pfn_pillar(PfnWarpSmem &s, const float *__restrict__ w2bT, const PfnLane &w,
                                           int lane, int n, int cnt, bool virt, float sx, float sy, float sz,
                                           int cx, int cy, const PfnGeom &g, float &o0, float &o1) {
  const PfnCentre c = pfn_centre(n, sx, sy, sz, cx, cy, g);
  float best = -INFINITY;
  for (int r = 0; r < cnt; ++r) {
    const float y = fmaxf(fmaf(pfn_z1(&s.pts[r][0], c, w.w1), w.s1, w.t1), 0.f);
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
  float b0, b1;
  pfn_w2b_max(w2bT, s.m1, lane, b0, b1);
  float best0 = -INFINITY, best1 = -INFINITY;
  const int rows = cnt + (virt ? 1 : 0);
  for (int r = 0; r < rows; ++r) {
    float a0 = b0, a1 = b1;
    pfn_z2(&s.x1[r][0], w, a0, a1);
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

// packed image from W1 [32, F+5], W2 [64, 64] (nn.Linear layout); the scale / shift entries are copied from
// s1, t1, s2, t2 when those are given, and left alone when they are null (the training passes write them)
static __global__ void pillar_pack_kernel(const float *__restrict__ W1, const float *__restrict__ s1,
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
      if (!s1) continue;
      v = s1[i - kPfnS1];
    } else if (i < kPfnW2a) {
      if (!t1) continue;
      v = t1[i - kPfnT1];
    } else if (i < kPfnW2b) {
      const int o = (i - kPfnW2a) / kPfnC1, k = (i - kPfnW2a) % kPfnC1;
      v = W2[o * kPfnC2 + k];
    } else if (i < kPfnS2) {
      const int k = (i - kPfnW2b) / kPfnC2, o = (i - kPfnW2b) % kPfnC2;
      v = W2[o * kPfnC2 + kPfnC1 + k];
    } else if (i < kPfnT2) {
      if (!s2) continue;
      v = s2[i - kPfnS2];
    } else {
      if (!t2) continue;
      v = t2[i - kPfnT2];
    }
    packed[i] = v;
  }
}

inline bool pfn_native(int F, int P) { return F >= 3 && F <= kPfnMaxF && P >= 1 && P <= kPfnMaxP; }

#ifndef BEVB200_UNSUPPORTED
#define BEVB200_UNSUPPORTED(cond, msg)                                                  \
  do {                                                                                  \
    if (!(cond)) {                                                                      \
      snprintf(::bevb200::g_last_error, sizeof(::bevb200::g_last_error), "%s: %s [%s]", \
               __func__, msg, #cond);                                                   \
      return BEVB200_EUNSUPPORTED;                                                      \
    }                                                                                   \
  } while (0)
#endif

}  // namespace bevb200
