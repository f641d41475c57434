// PointPillars pillar feature net in training mode (mmdet3d/models/backbones/pillar_encoder.py:43-176 with
// BatchNorm1d in train mode): batch statistics over all M * P slots, padded slots included, and the backward
// of the whole net (both linears, both BNs) from the canvas gradient.  DESIGN 4.22.
//
// No per-slot tensor exists.  Every pass re-reads the [R, P, F] rows and recomputes what it needs on one
// warp per pillar with the eval kernel's arithmetic (pillars.cuh).  The P - n padded slots of a pillar have
// a zero input row, so they collapse to two row kinds: slot n (kind A), and P - n - 1 identical rows (kind
// B).  With torch's tie rule (the lowest slot attaining a max takes its gradient), every max gradient that
// lands on padding lands on kind A; kind B rows still count in every BN sum and in dW2.
//
//   forward   pack (live W1, W2) | P1: sum z1, z1^2 | stats 1 | P2: sum z2, z2^2 | stats 2 |
//             P3: the max into the canvas; saves the layer-2 argmax and x^2 there per pillar
//   backward  B1: sum g2, g2 x^2 from the saved values | bn 2 | B2: dz2 on every row, dW2, dy1, g1,
//             sum g1, g1 x^1 | bn 1 | dW2 reduce | B3: dz1, dW1 | dW1 reduce
//
// Sums are double, per chunk of kPtChunk source rows, each chunk's warps added in warp order, and the chunks
// added in chunk order: bit-reproducible, independent of the grid size.  No float atomics.
#include "pillars.cuh"

namespace bevb200 {

constexpr int kPtWarps = kPfnWarps, kPtThreads = kPtWarps * 32;
constexpr int kPtChunk = 128;                   // source rows per partial
constexpr int kPtRounds = kPtChunk / kPtWarps;  // one pillar per warp per round
constexpr int kPtPartA = 2 * kPfnC2;            // per-chunk channel sums (doubles)
constexpr int kPtPartW = kPfnC2 * kPfnC2;       // per-chunk weight-gradient sums (doubles): dW2, or dW1 [13][32]
constexpr uint8_t kPtNoGrad = 0xFF;             // saved layer-2 argmax of a channel whose max is <= 0

enum PtPass { kP1 = 0, kP2, kP3, kB1, kB2, kB3 };

// state: packed image | stat (double) [mean1 32 | invstd1 32 | mean2 64 | invstd2 64] | info [pillars, few rows] |
//        am2 [R][64] uint8 | xh2 [R][64] fp32
struct PtState {
  float *packed;
  double *stat;
  int32_t *info;
  uint8_t *am2;
  float *xh2;
};

static PtState pt_state(void *base, int rows, size_t *bytes) {
  Arena a(base, ~size_t(0));
  PtState s;
  s.packed = a.take<float>(kPfnPacked);
  s.stat = a.take<double>(2 * kPfnC1 + 2 * kPfnC2);
  s.info = a.take<int32_t>(4);
  s.am2 = a.take<uint8_t>((size_t)rows * kPfnC2);
  s.xh2 = a.take<float>((size_t)rows * kPfnC2);
  *bytes = a.off;
  return s;
}

static int pt_chunks(int rows) { return rows > 0 ? (rows + kPtChunk - 1) / kPtChunk : 1; }

// workspace: partA [chunks][128] | partW [chunks][4096] | coef (double) [mg2 64 | mgx2 64 | mg1 32 | mgx1 32]
struct PtWork {
  double *partA, *partW;
  double *coef;
};

static PtWork pt_work(void *base, int rows, size_t *bytes) {
  Arena a(base, ~size_t(0));
  const size_t chunks = pt_chunks(rows);
  PtWork w;
  w.partA = a.take<double>(chunks * kPtPartA);
  w.partW = a.take<double>(chunks * kPtPartW);
  w.coef = a.take<double>(2 * kPfnC2 + 2 * kPfnC1);
  *bytes = a.off;
  return w;
}

struct PtArgs {
  const float *voxels;
  const int32_t *num_points, *coords4, *n_dev;
  int R, cap, P, F;
  PfnGeom g;
  const float *packed;
  const double *stat, *coef;  // BN statistics and backward coefficients stay double: their rounding would shift
                              // every row alike, and that bias adds up over the non-centred input columns
  const int32_t *info;
  uint8_t *am2;
  float *xh2;
  float *canvas;             // P3
  const float *grad_canvas;  // B passes
  int B, nx, ny;
  double *partA, *partW;
};

// the backward's per-warp rows: dz2 of every row (real rows, then kind A, then kind B), their multiplicity,
// and the per-pillar sum of dz2
struct __align__(16) PtWarpB {
  float dz[kPfnMaxP][kPfnC2];
  float dsum[kPfnC2];
  float rw[kPfnMaxP];
  int rows;
};

template <int kPass>
constexpr int pt_acc() {
  return kPass == kP1 || kPass == kB2 ? 2 : kPass == kB3 ? kPfnD : 4;
}

template <int kPass>
constexpr size_t pt_smem_bytes() {
  size_t b = sizeof(PfnWarpSmem) * kPtWarps + sizeof(float) * kPfnC1 * kPfnC2 +
             sizeof(double) * kPtWarps * pt_acc<kPass>() * 32;
  if (kPass == kB2 || kPass == kB3) b += sizeof(PtWarpB) * kPtWarps + 2 * sizeof(float) * kPfnC2 * kPfnC1;
  return b;
}

__device__ __forceinline__ bool pt_valid(const PtArgs &a, int v) {
  if (v >= a.R) return false;
  const int s = v / a.cap;
  const int n = a.n_dev ? min(max(__ldg(a.n_dev + s), 0), a.cap) : a.cap;
  return v - s * a.cap < n;
}

// canvas offset of channel 0 of the pillar's cell, or -1 outside the canvas
__device__ __forceinline__ long long pt_cell(const PtArgs &a, int4 c) {
  if ((unsigned)c.x >= (unsigned)a.B || (unsigned)c.y >= (unsigned)a.nx || (unsigned)c.z >= (unsigned)a.ny) return -1;
  return (long long)c.x * kPfnC2 * a.nx * a.ny + (long long)c.y * a.ny + c.z;
}

template <int kPass>
__global__ void __launch_bounds__(kPtThreads) pillar_train_kernel(PtArgs a) {
  constexpr int kAcc = pt_acc<kPass>();
  constexpr bool kBwd = kPass == kB2 || kPass == kB3;
  extern __shared__ __align__(16) unsigned char pt_smem[];
  PfnWarpSmem *sm = reinterpret_cast<PfnWarpSmem *>(pt_smem);
  float *w2bT = reinterpret_cast<float *>(sm + kPtWarps);
  double *red = reinterpret_cast<double *>(w2bT + kPfnC1 * kPfnC2);
  PtWarpB *smb = reinterpret_cast<PtWarpB *>(red + kPtWarps * kAcc * 32);
  float *w2a_s = reinterpret_cast<float *>(smb + kPtWarps);  // [64][32]: W2[o][k]
  float *w2b_s = w2a_s + kPfnC2 * kPfnC1;                     // [64][32]: W2[o][32 + k]
  if (kPass != kP1 && a.info[1]) return;                      // too few rows: nothing to compute
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  PfnLane w;
  pfn_block_setup(a.packed, w2bT, w);
  if constexpr (kBwd) {
    for (int i = threadIdx.x; i < kPfnC2 * kPfnC1; i += blockDim.x) {
      const int o = i / kPfnC1, k = i % kPfnC1;
      w2a_s[i] = a.packed[kPfnW2a + i];
      w2b_s[i] = a.packed[kPfnW2b + k * kPfnC2 + o];
    }
    __syncthreads();
  }
  const double *st = a.stat;
  const double mean1 = st[lane], inv1 = st[kPfnC1 + lane];
  const float mean20 = (float)st[2 * kPfnC1 + lane], mean21 = (float)st[2 * kPfnC1 + 32 + lane];
  const float inv20 = (float)st[2 * kPfnC1 + kPfnC2 + lane], inv21 = (float)st[2 * kPfnC1 + kPfnC2 + 32 + lane];
  double mg20 = 0.0, mg21 = 0.0, mgx20 = 0.0, mgx21 = 0.0, mg1 = 0.0, mgx1 = 0.0;
  if constexpr (kBwd) {
    mg20 = a.coef[lane]; mg21 = a.coef[32 + lane];
    mgx20 = a.coef[kPfnC2 + lane]; mgx21 = a.coef[kPfnC2 + 32 + lane];
    mg1 = a.coef[2 * kPfnC2 + lane]; mgx1 = a.coef[2 * kPfnC2 + kPfnC1 + lane];
  }
  PfnWarpSmem &s = sm[warp];
  PtWarpB &sb = smb[warp];
  const int chunks = (a.R + kPtChunk - 1) / kPtChunk;
  for (int chunk = blockIdx.x; chunk < chunks; chunk += gridDim.x) {
    double acc[kAcc];
#pragma unroll
    for (int j = 0; j < kAcc; ++j) acc[j] = 0.0;
    // B2: thread t owns dW2[o][k] and dW2[o][32 + k] for k = t % 32, o = t / 32 + 4 i
    double wacc[kPass == kB2 ? 32 : 1];
#pragma unroll
    for (int j = 0; j < (kPass == kB2 ? 32 : 1); ++j) wacc[j] = 0.0;
    for (int round = 0; round < kPtRounds; ++round) {
      const int v = chunk * kPtChunk + round * kPtWarps + warp;
      const bool valid = pt_valid(a, v);
      int nrows = 0;
      if constexpr (kPass == kB1) {
        if (!valid) continue;
        const long long cell = pt_cell(a, reinterpret_cast<const int4 *>(a.coords4)[v]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int ch = lane + 32 * h;
          if (cell >= 0 && a.am2[(long long)v * kPfnC2 + ch] != kPtNoGrad) {
            const double G = a.grad_canvas[cell + (long long)ch * a.nx * a.ny];
            acc[h] += G;
            acc[2 + h] += G * (double)a.xh2[(long long)v * kPfnC2 + ch];
          }
        }
      } else if (valid) {
        const int n = a.num_points[v];
        float3 p = make_float3(0.f, 0.f, 0.f);
        if (lane < a.P) p = pfn_stage_row(s, lane, a.voxels + ((long long)v * a.P + lane) * a.F, a.F);
        const float sx = warp_sum(p.x), sy = warp_sum(p.y), sz = warp_sum(p.z);
        __syncwarp();
        const int cnt = min(max(n, 0), a.P), pad = a.P - cnt;
        const int4 c4 = reinterpret_cast<const int4 *>(a.coords4)[v];
        const PfnCentre c = pfn_centre(n, sx, sy, sz, c4.y, c4.z, a.g);
        if constexpr (kPass == kP1) {
          for (int r = 0; r < cnt; ++r) {
            const float z = pfn_z1(&s.pts[r][0], c, w.w1);
            acc[0] += z;
            acc[1] += (double)z * z;
          }
        } else {
          // layer 1: rows, kind A / B rows (relu(t1)), the max and its lowest argmax
          float best = -INFINITY;
          int am1 = 0;
          for (int r = 0; r < cnt; ++r) {
            const float y = fmaxf(fmaf(pfn_z1(&s.pts[r][0], c, w.w1), w.s1, w.t1), 0.f);
            s.x1[r][lane] = y;
            if (y > best) { best = y; am1 = r; }
          }
          if (pad > 0) {
            const float y = fmaxf(w.t1, 0.f);
            s.x1[cnt][lane] = y;
            if (pad > 1) s.x1[cnt + 1][lane] = y;
            if (y > best) { best = y; am1 = cnt; }
          }
          s.m1[lane] = best;
          __syncwarp();
          float b0, b1;
          pfn_w2b_max(w2bT, s.m1, lane, b0, b1);
          const int rf = cnt + (pad > 0 ? 1 : 0);  // kind B has kind A's layer-2 row
          nrows = cnt + min(pad, 2);
          if constexpr (kPass == kP2) {
            for (int r = 0; r < rf; ++r) {
              float a0 = b0, a1 = b1;
              pfn_z2(&s.x1[r][0], w, a0, a1);
              const double m = r < cnt ? 1.0 : (double)pad;
              acc[0] += m * a0;
              acc[1] += m * a1;
              acc[2] += m * ((double)a0 * a0);
              acc[3] += m * ((double)a1 * a1);
            }
          } else if constexpr (kPass == kP3) {
            float best0 = -INFINITY, best1 = -INFINITY, z0 = 0.f, z1 = 0.f;
            int arg0 = 0, arg1 = 0;
            for (int r = 0; r < rf; ++r) {
              float a0 = b0, a1 = b1;
              pfn_z2(&s.x1[r][0], w, a0, a1);
              const float y0 = fmaf(a0, w.s20, w.t20), y1 = fmaf(a1, w.s21, w.t21);
              if (y0 > best0) { best0 = y0; arg0 = r; z0 = a0; }
              if (y1 > best1) { best1 = y1; arg1 = r; z1 = a1; }
            }
            const long long cell = pt_cell(a, c4), plane = (long long)a.nx * a.ny;
            if (cell >= 0) {
              a.canvas[cell + lane * plane] = fmaxf(best0, 0.f);
              a.canvas[cell + (lane + 32) * plane] = fmaxf(best1, 0.f);
            }
            const long long o = (long long)v * kPfnC2;
            a.am2[o + lane] = best0 > 0.f ? (uint8_t)arg0 : kPtNoGrad;
            a.am2[o + lane + 32] = best1 > 0.f ? (uint8_t)arg1 : kPtNoGrad;
            a.xh2[o + lane] = (z0 - mean20) * inv20;
            a.xh2[o + lane + 32] = (z1 - mean21) * inv21;
          } else {
            // layer 2 backward: dz2 = s2 (g2 - mean g2 - x^2 mean g2 x^2) on every row
            const long long cell = pt_cell(a, c4), plane = (long long)a.nx * a.ny;
            const long long o = (long long)v * kPfnC2;
            const int am20 = a.am2[o + lane], am21 = a.am2[o + lane + 32];
            const float G0 = cell >= 0 && am20 != kPtNoGrad ? a.grad_canvas[cell + lane * plane] : 0.f;
            const float G1 = cell >= 0 && am21 != kPtNoGrad ? a.grad_canvas[cell + (lane + 32) * plane] : 0.f;
            float D0 = 0.f, D1 = 0.f;
            for (int r = 0; r < rf; ++r) {
              float a0 = b0, a1 = b1;
              pfn_z2(&s.x1[r][0], w, a0, a1);
              const double xh0 = ((double)a0 - st[2 * kPfnC1 + lane]) * st[2 * kPfnC1 + kPfnC2 + lane];
              const double xh1 = ((double)a1 - st[2 * kPfnC1 + 32 + lane]) * st[2 * kPfnC1 + kPfnC2 + 32 + lane];
              const float base0 = (float)(-mg20 - xh0 * mgx20), base1 = (float)(-mg21 - xh1 * mgx21);
              const float dz0 = (float)((double)w.s20 * ((r == am20 ? G0 : 0.0) - mg20 - xh0 * mgx20));
              const float dz1 = (float)((double)w.s21 * ((r == am21 ? G1 : 0.0) - mg21 - xh1 * mgx21));
              sb.dz[r][lane] = dz0;
              sb.dz[r][lane + 32] = dz1;
              D0 += dz0;
              D1 += dz1;
              if (r == cnt && pad > 1) {  // kind B: no max gradient
                sb.dz[cnt + 1][lane] = w.s20 * base0;
                sb.dz[cnt + 1][lane + 32] = w.s21 * base1;
                D0 = fmaf((float)(pad - 1), w.s20 * base0, D0);
                D1 = fmaf((float)(pad - 1), w.s21 * base1, D1);
              }
            }
            sb.dsum[lane] = D0;
            sb.dsum[lane + 32] = D1;
            if (lane < nrows) sb.rw[lane] = lane == cnt + 1 ? (float)(pad - 1) : 1.f;
            __syncwarp();
            // layer 1 backward (lane = layer-1 channel): dy1 = W2a^T dz2 per row, the max gradient W2b^T sum dz2
            // to the argmax row, ReLU mask, then BN 1
            float dmax = 0.f;
            for (int q = 0; q < kPfnC2; ++q) dmax = fmaf(w2b_s[q * kPfnC1 + lane], sb.dsum[q], dmax);
            const int rl = kPass == kB2 ? nrows : cnt;
            for (int r = 0; r < rl; ++r) {
              float dy = 0.f;
#pragma unroll 8
              for (int q = 0; q < kPfnC2; ++q) dy = fmaf(w2a_s[q * kPfnC1 + lane], sb.dz[r][q], dy);
              if (r == am1) dy += dmax;
              const float g1 = s.x1[r][lane] > 0.f ? dy : 0.f;
              const float z = r < cnt ? pfn_z1(&s.pts[r][0], c, w.w1) : 0.f;
              const double xh = ((double)z - mean1) * inv1;
              if constexpr (kPass == kB2) {
                const double m = r == cnt + 1 ? (double)(pad - 1) : 1.0;
                acc[0] += m * g1;
                acc[1] += m * (g1 * xh);
              } else {
                const double dz1 = (double)w.s1 * ((double)g1 - mg1 - xh * mgx1);
                float d[kPfnD];
                pfn_decorate(&s.pts[r][0], c, d);
#pragma unroll
                for (int j = 0; j < kPfnD; ++j) acc[j] += dz1 * d[j];
              }
            }
          }
        }
      }
      if constexpr (kPass == kB2) {
        if (lane == 0) sb.rows = nrows;
        __syncthreads();
        const int k = threadIdx.x & 31, o0 = threadIdx.x >> 5;
        for (int q = 0; q < kPtWarps; ++q) {  // the warps' pillars in warp order
          const int rows = smb[q].rows;
          if (rows == 0) continue;
          float t[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) t[i] = 0.f;
          for (int r = 0; r < rows; ++r) {
            const float x = smb[q].rw[r] * sm[q].x1[r][k];
#pragma unroll
            for (int i = 0; i < 16; ++i) t[i] = fmaf(smb[q].dz[r][o0 + 4 * i], x, t[i]);
          }
          const float m = sm[q].m1[k];
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            wacc[2 * i] += t[i];
            wacc[2 * i + 1] += smb[q].dsum[o0 + 4 * i] * m;
          }
        }
        __syncthreads();
      }
      __syncwarp();
    }
    // chunk end: the warps' accumulators in warp order
#pragma unroll
    for (int j = 0; j < kAcc; ++j) red[(warp * kAcc + j) * 32 + lane] = acc[j];
    __syncthreads();
    double *part = kPass == kB3 ? a.partW + (long long)chunk * kPtPartW : a.partA + (long long)chunk * kPtPartA;
    for (int e = threadIdx.x; e < kAcc * 32; e += blockDim.x) {
      double t = red[e];
      for (int q = 1; q < kPtWarps; ++q) t += red[q * kAcc * 32 + e];
      part[e] = t;
    }
    if constexpr (kPass == kB2) {
      const int k = threadIdx.x & 31, o0 = threadIdx.x >> 5;
      double *pw = a.partW + (long long)chunk * kPtPartW;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        pw[(o0 + 4 * i) * kPfnC2 + k] = wacc[2 * i];
        pw[(o0 + 4 * i) * kPfnC2 + kPfnC1 + k] = wacc[2 * i + 1];
      }
    }
    __syncthreads();
  }
}

__device__ __forceinline__ double pt_chunk_sum(const double *__restrict__ part, int stride, int chunks, int e) {
  double t = 0.0;
  for (int k = 0; k < chunks; ++k) t += part[(long long)k * stride + e];
  return t;
}

// number of slots the BN statistics run over: P * (valid pillars of every segment)
__device__ __forceinline__ double pt_slots(const int32_t *n_dev, int segments, int cap, int P) {
  long long m = 0;
  for (int s = 0; s < segments; ++s) m += n_dev ? min(max(__ldg(n_dev + s), 0), cap) : cap;
  return (double)m * P;
}

// batch statistics of one layer (C channels): mean / invstd, the scale / shift into the packed image, the
// running statistics (torch's BatchNorm1d in train mode); layer 1 also decides the few-rows flag
__global__ void pt_stats_kernel(const double *__restrict__ part, int chunks, int C, const int32_t *__restrict__ n_dev,
                                int segments, int cap, int P, bevb200_encoder_bn_t bn, double *__restrict__ stat_mean,
                                double *__restrict__ stat_inv, float *__restrict__ scale, float *__restrict__ shift,
                                int32_t *__restrict__ info, int32_t *__restrict__ status, int first) {
  const double N = pt_slots(n_dev, segments, cap, P);
  const int ch = threadIdx.x;
  if (first && ch == 0) {
    info[0] = (int32_t)(N / P);
    info[1] = N < 2.0;
    *status = N < 2.0 ? BEVB200_PILLAR_FEW_ROWS : 0;
  }
  if (N < 2.0 || ch >= C) return;
  const double s = pt_chunk_sum(part, kPtPartA, chunks, ch), ss = pt_chunk_sum(part, kPtPartA, chunks, C + ch);
  const double mean = s / N;
  const double var = fmax(ss / N - mean * mean, 0.0);  // biased: the normalisation's
  const double invstd = 1.0 / sqrt(var + (double)bn.eps);
  const double sc = (double)bn.weight[ch] * invstd;
  stat_mean[ch] = mean;
  stat_inv[ch] = invstd;
  scale[ch] = (float)sc;
  shift[ch] = (float)((double)bn.bias[ch] - mean * sc);
  const double m = bn.momentum;
  bn.running_mean[ch] = (float)((1.0 - m) * bn.running_mean[ch] + m * mean);
  bn.running_var[ch] = (float)((1.0 - m) * bn.running_var[ch] + m * var * N / (N - 1.0));
  if (ch == 0 && bn.num_batches_tracked) *bn.num_batches_tracked += 1;
}

// BN backward sums of one layer: dbeta = sum g, dgamma = sum g x^, coef = [sum g / N | sum g x^ / N]
__global__ void pt_bn_bwd_kernel(const double *__restrict__ part, int chunks, int C, const int32_t *__restrict__ n_dev,
                                 int segments, int cap, int P, const int32_t *__restrict__ info,
                                 float *__restrict__ dgamma, float *__restrict__ dbeta, double *__restrict__ coef) {
  const int ch = threadIdx.x;
  if (ch >= C) return;
  if (info[1]) {
    dgamma[ch] = 0.f;
    dbeta[ch] = 0.f;
    return;
  }
  const double N = pt_slots(n_dev, segments, cap, P);
  const double s = pt_chunk_sum(part, kPtPartA, chunks, ch), sx = pt_chunk_sum(part, kPtPartA, chunks, C + ch);
  dbeta[ch] = (float)s;
  dgamma[ch] = (float)sx;
  coef[ch] = s / N;
  coef[C + ch] = sx / N;
}

// dW2 [64, 64] from partials [o][k]; dW1 [32, F + 5] from partials [packed column][channel]
__global__ void pt_wgrad_kernel(const double *__restrict__ part, int chunks, int layer, int F,
                                const int32_t *__restrict__ info, float *__restrict__ out) {
  const int total = layer == 2 ? kPfnC2 * kPfnC2 : kPfnC1 * (F + 5);
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    int src = e;
    if (layer == 1) {
      const int c = e / (F + 5), col = e % (F + 5);
      src = (col < F ? col : kPfnMaxF + col - F) * kPfnC1 + c;
    }
    out[e] = info[1] ? 0.f : (float)pt_chunk_sum(part, kPtPartW, chunks, src);
  }
}

template <int kPass>
static int pt_launch(const PtArgs &a, cudaStream_t st) {
  constexpr size_t smem = pt_smem_bytes<kPass>();
  BEVB200_CUDA(cudaFuncSetAttribute(pillar_train_kernel<kPass>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)smem));
  const int grid = min(pt_chunks(a.R), kNumSMs * (kPass == kB2 || kPass == kB3 ? 2 : 4));
  BEVB200_LAUNCH(pillar_train_kernel<kPass>, grid, kPtThreads, smem, st, a);
  return BEVB200_OK;
}

#define PT_TRY(expr)      \
  do {                    \
    const int rc__ = (expr); \
    if (rc__) return rc__; \
  } while (0)

// argument checks shared by both calls; fills a's row source
static int pt_rows(const char *fn, const float *voxels, const int32_t *num_points, const int32_t *coords4, int rows,
                   int segments, const int32_t *n_dev, int P, int F, float vx, float vy, float x_off, float y_off,
                   int batch, int nx, int ny, PtArgs &a) {
  if (!pfn_native(F, P)) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: native pillar net: F 3..8, P 1..32", fn);
    return BEVB200_EUNSUPPORTED;
  }
  if (rows < 0 || segments < 1 || rows % segments != 0 || batch < 1 || nx < 1 || ny < 1) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: bad sizes", fn);
    return BEVB200_EINVAL;
  }
  if (rows > 0 && !(voxels && num_points && coords4)) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: null argument", fn);
    return BEVB200_EINVAL;
  }
  a = PtArgs{};
  a.voxels = voxels;
  a.num_points = num_points;
  a.coords4 = coords4;
  a.n_dev = n_dev;
  a.R = rows;
  a.cap = rows > 0 ? rows / segments : 1;
  a.P = P;
  a.F = F;
  a.g = PfnGeom{vx, vy, x_off, y_off};
  a.B = batch;
  a.nx = nx;
  a.ny = ny;
  return BEVB200_OK;
}

}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_pillar_train_state_bytes(int rows, int max_points) {
  if (rows < 0 || max_points < 1 || max_points > kPfnMaxP) return 0;
  size_t b;
  pt_state(nullptr, rows, &b);
  return b;
}

size_t bevb200_pillar_train_workspace_bytes(int rows, int max_points) {
  if (rows < 0 || max_points < 1 || max_points > kPfnMaxP) return 0;
  size_t b;
  pt_work(nullptr, rows, &b);
  return b;
}

int bevb200_pillar_forward_train(const float *voxels, const int32_t *num_points, const int32_t *coords4, int rows,
                                 int segments, const int32_t *n_dev, int max_points, int num_features, float vx,
                                 float vy, float x_off, float y_off, const float *w1, const float *w2,
                                 const bevb200_encoder_bn_t *bn, float *canvas, int batch, int nx, int ny,
                                 int32_t *status_dev, void *state, size_t state_bytes, void *workspace,
                                 size_t workspace_bytes, void *stream) {
  PtArgs a;
  PT_TRY(pt_rows(__func__, voxels, num_points, coords4, rows, segments, n_dev, max_points, num_features, vx, vy,
                 x_off, y_off, batch, nx, ny, a));
  BEVB200_REQUIRE(w1 && w2 && bn && canvas && status_dev && state && workspace, "null argument");
  for (int l = 0; l < 2; ++l)
    BEVB200_REQUIRE(bn[l].weight && bn[l].bias && bn[l].running_mean && bn[l].running_var, "null BN pointer");
  size_t need_s, need_w;
  const PtState S = pt_state(state, rows, &need_s);
  const PtWork W = pt_work(workspace, rows, &need_w);
  if (state_bytes < need_s || workspace_bytes < need_w) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: state %zu < %zu or workspace %zu < %zu bytes", __func__,
             state_bytes, need_s, workspace_bytes, need_w);
    return BEVB200_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  a.packed = S.packed;
  a.stat = S.stat;
  a.info = S.info;
  a.am2 = S.am2;
  a.xh2 = S.xh2;
  a.canvas = canvas;
  a.partA = W.partA;
  a.partW = W.partW;
  const int chunks = pt_chunks(rows);
  double *mean1 = S.stat, *inv1 = S.stat + kPfnC1, *mean2 = S.stat + 2 * kPfnC1, *inv2 = mean2 + kPfnC2;
  BEVB200_LAUNCH(pillar_pack_kernel, grid_for(kPfnPacked, 256), 256, 0, st, w1, nullptr, nullptr, w2, nullptr,
                 nullptr, num_features, S.packed);
  PT_TRY(pt_launch<kP1>(a, st));
  BEVB200_LAUNCH(pt_stats_kernel, 1, kPfnC2, 0, st, W.partA, chunks, kPfnC1, n_dev, segments, a.cap, max_points, bn[0],
                 mean1, inv1, S.packed + kPfnS1, S.packed + kPfnT1, S.info, status_dev, 1);
  PT_TRY(pt_launch<kP2>(a, st));
  BEVB200_LAUNCH(pt_stats_kernel, 1, kPfnC2, 0, st, W.partA, chunks, kPfnC2, n_dev, segments, a.cap, max_points, bn[1],
                 mean2, inv2, S.packed + kPfnS2, S.packed + kPfnT2, S.info, status_dev, 0);
  PT_TRY(pt_launch<kP3>(a, st));
  return BEVB200_OK;
}

int bevb200_pillar_backward_train(const float *voxels, const int32_t *num_points, const int32_t *coords4, int rows,
                                  int segments, const int32_t *n_dev, int max_points, int num_features, float vx,
                                  float vy, float x_off, float y_off, const float *grad_canvas, int batch, int nx,
                                  int ny, const void *state, size_t state_bytes, float *grad_w1, float *grad_w2,
                                  float *grad_gamma1, float *grad_beta1, float *grad_gamma2, float *grad_beta2,
                                  void *workspace, size_t workspace_bytes, void *stream) {
  PtArgs a;
  PT_TRY(pt_rows(__func__, voxels, num_points, coords4, rows, segments, n_dev, max_points, num_features, vx, vy,
                 x_off, y_off, batch, nx, ny, a));
  BEVB200_REQUIRE(grad_canvas && state && grad_w1 && grad_w2 && grad_gamma1 && grad_beta1 && grad_gamma2 &&
                      grad_beta2 && workspace,
                  "null argument");
  size_t need_s, need_w;
  const PtState S = pt_state(const_cast<void *>(state), rows, &need_s);
  const PtWork W = pt_work(workspace, rows, &need_w);
  if (state_bytes < need_s || workspace_bytes < need_w) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: state %zu < %zu or workspace %zu < %zu bytes", __func__,
             state_bytes, need_s, workspace_bytes, need_w);
    return BEVB200_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  a.packed = S.packed;
  a.stat = S.stat;
  a.info = S.info;
  a.am2 = S.am2;
  a.xh2 = S.xh2;
  a.grad_canvas = grad_canvas;
  a.coef = W.coef;
  a.partA = W.partA;
  a.partW = W.partW;
  const int chunks = pt_chunks(rows);
  PT_TRY(pt_launch<kB1>(a, st));
  BEVB200_LAUNCH(pt_bn_bwd_kernel, 1, kPfnC2, 0, st, W.partA, chunks, kPfnC2, n_dev, segments, a.cap, max_points,
                 S.info, grad_gamma2, grad_beta2, W.coef);
  PT_TRY(pt_launch<kB2>(a, st));
  BEVB200_LAUNCH(pt_bn_bwd_kernel, 1, kPfnC2, 0, st, W.partA, chunks, kPfnC1, n_dev, segments, a.cap, max_points,
                 S.info, grad_gamma1, grad_beta1, W.coef + 2 * kPfnC2);
  BEVB200_LAUNCH(pt_wgrad_kernel, grid_for(kPfnC2 * kPfnC2, 256), 256, 0, st, W.partW, chunks, 2, num_features, S.info,
                 grad_w2);
  PT_TRY(pt_launch<kB3>(a, st));
  BEVB200_LAUNCH(pt_wgrad_kernel, grid_for(kPfnC1 * (kPfnMaxF + 5), 256), 256, 0, st, W.partW, chunks, 1,
                 num_features, S.info, grad_w1);
  return BEVB200_OK;
}

}  // extern "C"
