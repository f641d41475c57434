// CenterHead and TransFusion training losses and their gradients on the device: CenterHead.loss
// (models/heads/bbox/centerpoint.py:584-634) and TransFusionHead.loss (models/heads/bbox/transfusion.py:587-713) with
// the loss functions of mmdet 2.20 (GaussianFocalLoss, FocalLoss(use_sigmoid=True) through mmcv 1.4's
// sigmoid_focal_loss CUDA op, L1Loss), with no host synchronisation and no allocation.
//
// Forward, two launches per head:
//   *_forward_kernel   every CTA covers one tile of one term -- 1024 elements of a dense focal map (float4 loads when
//                      the map allows them), 1024 (class or box channel, proposal) elements of one decoder layer, or
//                      the max_objs x code gathered slots of one (task, sample) -- and writes its double partial sum,
//                      its count (positives or mask sum) and its status bits to its own workspace slot.
//   *_reduce_kernel    one warp per term adds the term's slots in a fixed order (lane strides, shuffle tree), forms the avg factor on the device
//                      (max(count, 1), fp32(num + 1e-4), max(sum num_pos, 1)) and writes the fp32 loss and the avg
//                      factor.  No atomics and no memset: every slot is written each call, so the sums are
//                      reproducible bit for bit.
// Backward, the elementwise gradients recomputed from the same inputs, each gradient element written once:
//   CenterHead   chl_backward_kernel: the heatmap gradients and a zero fill of the regression gradient maps;
//                chl_slots_kernel: one CTA per (task, sample) compacts the masked-in slots in slot order (a
//                masked-out slot's contribution is 0 * sgn = 0); the thread of a slot that is the first with its cell
//                adds the contributions of every slot with that cell in slot order and stores the sums (duplicate
//                cells add deterministically).
//   TransFusion  tfl_backward_kernel, one launch: the dense heatmap gradient and the dense [B, c, N] cls and box
//                gradients (columns of untrained layers 0).
//
// The sigmoid is torch's on CUDA, 1 / (1 + expf(-x)) in fp32 with IEEE division (the library is built without
// fast-math), so clip_sigmoid's clamp decision -- and with it the set of zero gradients -- is the reference's.  The
// elementwise losses and gradients are then evaluated in double from that fp32 value.
#include <float.h>
#include <math.h>

#include "common.cuh"

namespace bevb200 {
namespace {

constexpr int kThreads = 256;
constexpr int kTile = 1024;                 // elements per CTA of a dense term: 4 per thread
constexpr int kSlotThreads = 512;
constexpr int kMaxTasks = BEVB200_LOSS_MAX_TASKS;
constexpr int kMaxLayers = BEVB200_LOSS_MAX_LAYERS;
constexpr int kMaxObjs = BEVB200_LOSS_MAX_OBJS;
constexpr int kMaps = 5;                    // reg / center, height, dim, rot, vel
__constant__ int kMapCh[kMaps] = {2, 1, 3, 2, 2};
__constant__ int kMapOf[10] = {0, 0, 1, 2, 2, 2, 3, 3, 4, 4};
__constant__ int kMapC0[kMaps] = {0, 2, 3, 6, 8};

struct Part {
  double sum, cnt;
  int flags, pad;
};

struct Focal {
  double alpha, gamma;
};

// ---- elementwise terms -------------------------------------------------------------------------------
// x^e: repeated products for the integral exponents of the configs (alpha 2, gamma 2 or 4), exp(e log x) otherwise
// (pow's values for x >= 0; NaN for a negative base).
__device__ __forceinline__ double powe(double x, double e) {
  if (e == 1.0) return x;
  if (e == 2.0) return x * x;
  if (e == 4.0) return (x * x) * (x * x);
  if (x > 0.0) return exp(e * log(x));
  return x == 0.0 ? (e > 0.0 ? 0.0 : (e == 0.0 ? 1.0 : INFINITY)) : NAN;
}

__device__ __forceinline__ float sigmoid_f(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

// gaussian_focal_loss of clip_sigmoid(x) against t; *dldx = d loss / d x (0 where the clamp is active).
__device__ __forceinline__ double gaussian_focal(float x, float t, Focal f, double *dldx) {
  const float lo = 1e-4f, hi = 1.f - 1e-4f;
  const float y = sigmoid_f(x);
  const bool pass = y >= lo && y <= hi;
  const float pc = y < lo ? lo : (y > hi ? hi : y);
  const double p = pc, q = 1.0 - p, eps = 1e-12;
  const double lp = log(p + eps), lq = log(q + eps), nw = powe(1.0 - (double)t, f.gamma);
  const bool pos = t == 1.f;
  double loss = -lq * powe(p, f.alpha) * nw;
  double d = nw * (powe(p, f.alpha) / (q + eps) - f.alpha * powe(p, f.alpha - 1.0) * lq);
  if (pos) {
    loss += -lp * powe(q, f.alpha);
    d += -powe(q, f.alpha) / (p + eps) + f.alpha * powe(q, f.alpha - 1.0) * lp;
  }
  if (dldx) *dldx = pass ? d * ((double)y * (1.0 - (double)y)) : 0.0;
  return loss;
}

// mmcv's sigmoid_focal_loss forward and backward (d / dx) of one element, flag = (label == class).
__device__ __forceinline__ double sigmoid_focal(float x, bool flag, Focal f, double *dldx) {
  const double p = sigmoid_f(x);
  const double lp = log(fmax(p, (double)FLT_MIN)), lq = log(fmax(1.0 - p, (double)FLT_MIN));
  if (flag) {
    const double w = f.alpha * powe(1.0 - p, f.gamma);
    if (dldx) *dldx = -w * (1.0 - p - f.gamma * p * lp);
    return -w * lp;
  }
  const double w = (1.0 - f.alpha) * powe(p, f.gamma);
  if (dldx) *dldx = -w * (f.gamma * (1.0 - p) * lq - p);
  return -w * lq;
}

__device__ __forceinline__ double sgn(double d) { return (double)((0.0 < d) - (d < 0.0)); }   // torch: sgn(NaN) = 0

__device__ __forceinline__ float4 ldg4(const float *p) { return __ldg((const float4 *)p); }

// Block sum of (sum, cnt, flags) in a fixed tree; thread 0 writes the slot.
__device__ void store_part(double s, double c, int f, Part *slot) {
  __shared__ double ss[kThreads / 32], sc[kThreads / 32];
  __shared__ int sf[kThreads / 32];
  for (int o = 16; o; o >>= 1) {
    s += __shfl_down_sync(0xffffffffu, s, o);
    c += __shfl_down_sync(0xffffffffu, c, o);
    f |= __shfl_down_sync(0xffffffffu, f, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    ss[warp] = s;
    sc[warp] = c;
    sf[warp] = f;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    Part r = {0.0, 0.0, 0, 0};
    for (int w = 0; w < kThreads / 32; ++w) {
      r.sum += ss[w];
      r.cnt += sc[w];
      r.flags |= sf[w];
    }
    *slot = r;
  }
}

// Focal loss sum and positive count of elements [e0, e0 + kTile) of a dense map of n elements.
__device__ void dense_focal_tile(const float *x, const float *t, long long n, long long e0, bool vec, Focal f,
                                 double &s, double &c) {
  if (vec) {
#pragma unroll
    for (int r = 0; r < kTile / 4 / kThreads; ++r) {
      const long long e = e0 + 4LL * (r * kThreads + threadIdx.x);
      if (e < n) {
        const float4 xv = ldg4(x + e), tv = ldg4(t + e);
        s += gaussian_focal(xv.x, tv.x, f, nullptr) + gaussian_focal(xv.y, tv.y, f, nullptr) +
             gaussian_focal(xv.z, tv.z, f, nullptr) + gaussian_focal(xv.w, tv.w, f, nullptr);
        c += (tv.x == 1.f) + (tv.y == 1.f) + (tv.z == 1.f) + (tv.w == 1.f);
      }
    }
  } else {
    for (int r = 0; r < kTile / kThreads; ++r) {
      const long long e = e0 + r * kThreads + threadIdx.x;
      if (e < n) {
        const float tv = __ldg(t + e);
        s += gaussian_focal(__ldg(x + e), tv, f, nullptr);
        c += tv == 1.f;
      }
    }
  }
}

// Gradient of the same tile scaled by G.
__device__ void dense_focal_grad_tile(const float *x, const float *t, float *g, long long n, long long e0, bool vec,
                                      Focal f, double G) {
  double d;
  if (vec) {
#pragma unroll
    for (int r = 0; r < kTile / 4 / kThreads; ++r) {
      const long long e = e0 + 4LL * (r * kThreads + threadIdx.x);
      if (e < n) {
        const float4 xv = ldg4(x + e), tv = ldg4(t + e);
        float4 o;
        gaussian_focal(xv.x, tv.x, f, &d);
        o.x = (float)(G * d);
        gaussian_focal(xv.y, tv.y, f, &d);
        o.y = (float)(G * d);
        gaussian_focal(xv.z, tv.z, f, &d);
        o.z = (float)(G * d);
        gaussian_focal(xv.w, tv.w, f, &d);
        o.w = (float)(G * d);
        *(float4 *)(g + e) = o;
      }
    }
  } else {
    for (int r = 0; r < kTile / kThreads; ++r) {
      const long long e = e0 + r * kThreads + threadIdx.x;
      if (e < n) {
        gaussian_focal(__ldg(x + e), __ldg(t + e), f, &d);
        g[e] = (float)(G * d);
      }
    }
  }
}

// ---- CenterHead ------------------------------------------------------------------------------------------
struct CHTask {
  const float *heat, *tgt, *map[kMaps], *anno;   // heatmap logits / targets [B, cat, H, W]; anno [B, M, code]
  const int64_t *ind;                            // [B, M]
  const uint8_t *mask;                           // [B, M]
  float *gheat, *gmap[kMaps];                    // gradients (backward only)
  long long n;                                   // B * cat * H * W
  int tile0, ztile0, vec;                        // first heat tile, first zero-fill tile (backward), float4 path
};

struct CHParams {
  CHTask task[kMaxTasks];
  int T, B, HW, M, code, heat_tiles, zero_tiles, zvec;
  float cw[10];
  Focal cls;
  double lw_cls, lw_bbox;
};

__device__ __forceinline__ int find_task(const CHParams &p, int tile, bool zero) {
  int t = 0;
  while (t + 1 < p.T && tile >= (zero ? p.task[t + 1].ztile0 : p.task[t + 1].tile0)) ++t;
  return t;
}

// Slot (b, m), channel c of task t: the L1 term and its weight; false when the slot is skipped (a bad cell).
__device__ __forceinline__ bool ch_slot(const CHParams &p, const CHTask &tk, int b, int m, int c, long long *cell,
                                        double *d, double *w, float *mask_v, int *flags) {
  const long long bm = (long long)b * p.M + m;
  const long long ind = __ldg(tk.ind + bm);
  *mask_v = (float)__ldg(tk.mask + bm);
  if (ind < 0 || ind >= p.HW) {
    if (*mask_v != 0.f) *flags |= BEVB200_LOSS_BAD_IND;
    return false;
  }
  const int k = kMapOf[c], lc = c - kMapC0[k];
  const float pred = __ldg(tk.map[k] + ((long long)b * kMapCh[k] + lc) * p.HW + ind);
  const float tv = __ldg(tk.anno + bm * p.code + c);
  *cell = ind;
  *d = (double)pred - (double)tv;
  *w = __fmul_rn(__fmul_rn(*mask_v, isnan(tv) ? 0.f : 1.f), p.cw[c]);
  return true;
}

__global__ void __launch_bounds__(kThreads) chl_forward_kernel(const __grid_constant__ CHParams p, Part *parts) {
  double s = 0.0, c = 0.0;
  int flags = 0;
  if ((int)blockIdx.x < p.heat_tiles) {
    const CHTask &tk = p.task[find_task(p, blockIdx.x, false)];
    dense_focal_tile(tk.heat, tk.tgt, tk.n, (long long)(blockIdx.x - tk.tile0) * kTile, tk.vec, p.cls, s, c);
  } else {
    const int tb = blockIdx.x - p.heat_tiles, t = tb / p.B, b = tb % p.B;
    const CHTask &tk = p.task[t];
    for (int i = threadIdx.x; i < p.M * p.code; i += kThreads) {
      const int m = i / p.code, ch = i - m * p.code;
      long long cell;
      double d, w;
      float mv;
      if (ch_slot(p, tk, b, m, ch, &cell, &d, &w, &mv, &flags)) s += fabs(d) * w;
      if (ch == 0) c += mv;
    }
  }
  store_part(s, c, flags, parts + blockIdx.x);
}

// Sum of slots [first, last) by one warp: lane l takes slots first + l, first + l + 32, ..., then a fixed shuffle tree.
__device__ __forceinline__ Part warp_sum(const Part *__restrict__ parts, int first, int last) {
  const int lane = threadIdx.x & 31;
  double s = 0.0, c = 0.0;
  int f = 0;
#pragma unroll 8
  for (int i = first + lane; i < last; i += 32) {
    s += parts[i].sum;
    c += parts[i].cnt;
    f |= parts[i].flags;
  }
  for (int o = 16; o; o >>= 1) {
    s += __shfl_down_sync(0xffffffffu, s, o);
    c += __shfl_down_sync(0xffffffffu, c, o);
    f |= __shfl_down_sync(0xffffffffu, f, o);
  }
  return Part{s, c, f, 0};
}

// OR of every warp's lane-0 flags into *status by thread 0.
__device__ __forceinline__ void store_status(int flags, int32_t *status) {
  __shared__ int wf[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) wf[warp] = flags;
  __syncthreads();
  if (threadIdx.x == 0) {
    int f = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) f |= wf[w];
    *status = f;
  }
}

// One warp per term.  losses / avg [2T]: heatmap of task t at 2t, bbox at 2t + 1.
__global__ void chl_reduce_kernel(const __grid_constant__ CHParams p, const Part *__restrict__ parts,
                                  float *__restrict__ losses, float *__restrict__ avg, int32_t *__restrict__ status) {
  const int j = threadIdx.x >> 5, t = j >> 1;
  int first, last;
  if ((j & 1) == 0) {
    first = p.task[t].tile0;
    last = t + 1 < p.T ? p.task[t + 1].tile0 : p.heat_tiles;
  } else {
    first = p.heat_tiles + t * p.B;
    last = first + p.B;
  }
  const Part r = warp_sum(parts, first, last);
  if ((threadIdx.x & 31) == 0) {
    const float a = (j & 1) == 0 ? (float)fmax(r.cnt, 1.0) : __fadd_rn((float)r.cnt, 1e-4f);
    losses[j] = (float)(((j & 1) == 0 ? p.lw_cls : p.lw_bbox) * (r.sum / (double)a));
    avg[j] = a;
  }
  store_status(r.flags, status);
}

__global__ void __launch_bounds__(kThreads) chl_backward_kernel(const __grid_constant__ CHParams p,
                                                                const float *__restrict__ gout,
                                                                const float *__restrict__ avg) {
  if ((int)blockIdx.x < p.heat_tiles) {
    const int t = find_task(p, blockIdx.x, false);
    const CHTask &tk = p.task[t];
    const double G = (double)gout[2 * t] * p.lw_cls / (double)avg[2 * t];
    dense_focal_grad_tile(tk.heat, tk.tgt, tk.gheat, tk.n, (long long)(blockIdx.x - tk.tile0) * kTile, tk.vec, p.cls,
                          G);
    return;
  }
  // zero fill of task t's regression gradient maps, viewed as B * code * HW elements (b, c, cell)
  const int zt = blockIdx.x - p.heat_tiles, t = find_task(p, zt, true);
  const CHTask &tk = p.task[t];
  const long long n = (long long)p.B * p.code * p.HW, e0 = (long long)(zt - tk.ztile0) * kTile;
  const int step = p.zvec ? 4 : 1;
  for (int r = 0; r < kTile / step / kThreads; ++r) {
    const long long e = e0 + (long long)step * (r * kThreads + threadIdx.x);
    if (e >= n) break;
    const long long bc = e / p.HW, cell = e - bc * p.HW;
    const int b = (int)(bc / p.code), c = (int)(bc - (long long)b * p.code);
    const int k = kMapOf[c], lc = c - kMapC0[k];
    float *dst = tk.gmap[k] + ((long long)b * kMapCh[k] + lc) * p.HW + cell;
    if (p.zvec)
      *(float4 *)dst = make_float4(0.f, 0.f, 0.f, 0.f);
    else
      *dst = 0.f;
  }
}

__global__ void __launch_bounds__(kSlotThreads) chl_slots_kernel(const __grid_constant__ CHParams p,
                                                                 const float *__restrict__ gout,
                                                                 const float *__restrict__ avg) {
  __shared__ int cell_s[kMaxObjs], slot_s[kMaxObjs];   // the masked-in slots with a valid cell, in slot order
  __shared__ int warp_n[kSlotThreads / 32];
  __shared__ int n_live;
  const int t = blockIdx.x / p.B, b = blockIdx.x % p.B, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const CHTask &tk = p.task[t];
  const double G = (double)gout[2 * t + 1] * p.lw_bbox / (double)avg[2 * t + 1];
  if (threadIdx.x == 0) n_live = 0;
  __syncthreads();
  for (int m0 = 0; m0 < p.M; m0 += kSlotThreads) {
    const int m = m0 + threadIdx.x;
    int cell = -1;
    if (m < p.M && __ldg(tk.mask + (long long)b * p.M + m) != 0) {   // a masked-out slot adds 0 * sgn(d) = 0
      const long long ind = __ldg(tk.ind + (long long)b * p.M + m);
      cell = ind < 0 || ind >= p.HW ? -1 : (int)ind;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, cell >= 0);
    if (lane == 0) warp_n[warp] = __popc(bal);
    __syncthreads();
    int before = n_live;
    for (int w = 0; w < warp; ++w) before += warp_n[w];
    if (cell >= 0) {
      const int pos = before + __popc(bal & ((1u << lane) - 1u));
      cell_s[pos] = cell;
      slot_s[pos] = m;
    }
    __syncthreads();
    if (threadIdx.x == 0)
      for (int w = 0; w < kSlotThreads / 32; ++w) n_live += warp_n[w];
    __syncthreads();
  }
  const int n = n_live;
  for (int i = threadIdx.x; i < n; i += kSlotThreads) {
    const int cell = cell_s[i];
    bool head = true;
    for (int j = 0; head && j < i; ++j) head = cell_s[j] != cell;
    if (!head) continue;
    // acc sums w * sgn(d) and is scaled by G once.  The sum is exact in double (fp32 weights, at most kMaxObjs
    // terms), so a cell whose duplicate slots cancel gets exactly 0 whatever their order.  Adding G * w * sgn per
    // slot rounded from the third duplicate on: at max_objs 4096 on a 40 x 36 map, cells with three +w and three -w
    // slots spread over several kSlotThreads passes were left with a residue of ~1e-21 instead of 0.
    double acc[10];
#pragma unroll
    for (int c = 0; c < 10; ++c) acc[c] = 0.0;
    for (int j = i; j < n; ++j) {
      if (cell_s[j] != cell) continue;
#pragma unroll
      for (int c = 0; c < 10; ++c) {
        if (c >= p.code) break;
        long long cl;
        double d, w;
        float mv;
        int fl = 0;
        if (ch_slot(p, tk, b, slot_s[j], c, &cl, &d, &w, &mv, &fl)) acc[c] += w * sgn(d);
      }
    }
#pragma unroll
    for (int c = 0; c < 10; ++c) {
      if (c >= p.code) break;
      const int k = kMapOf[c], lc = c - kMapC0[k];
      tk.gmap[k][((long long)b * kMapCh[k] + lc) * p.HW + cell] = (float)(G * acc[c]);
    }
  }
}

// ---- TransFusion -----------------------------------------------------------------------------------------
struct TFParams {
  const float *dense, *dense_tgt, *heat, *map[kMaps], *bt, *bw, *mean_iou;
  const int64_t *labels, *label_w;
  const int32_t *num_pos;
  float *gdense, *gheat, *gmap[kMaps];
  long long n_dense;
  int B, K, N, P, Lt, code, n_num_pos, n_iou, dense_vec, dense_tiles, layer_tiles_cls, layer_tiles_box, col_tiles;
  float cw[10];
  Focal heat_f, cls_f;
  double lw_heat, lw_cls, lw_bbox;
};

// term of a forward tile: 0 heatmap, 1 + 2l cls of layer l, 2 + 2l bbox of layer l; *e0 its first element
__device__ __forceinline__ int tf_term(const TFParams &p, int tile, long long *e0) {
  if (tile < p.dense_tiles) {
    *e0 = (long long)tile * kTile;
    return 0;
  }
  tile -= p.dense_tiles;
  const int per = p.layer_tiles_cls + p.layer_tiles_box, l = tile / per, r = tile - l * per;
  if (r < p.layer_tiles_cls) {
    *e0 = (long long)r * kTile;
    return 1 + 2 * l;
  }
  *e0 = (long long)(r - p.layer_tiles_cls) * kTile;
  return 2 + 2 * l;
}

// Column element (b, ch, n) of the [B, K + code, N] cls / box space in layer l: the loss term and d / dx.
__device__ __forceinline__ double tf_column(const TFParams &p, int b, int ch, int n, double *dldx, int *flags) {
  const long long bn = (long long)b * p.N + n;
  if (ch < p.K) {
    const long long label = __ldg(p.labels + bn);
    if (label < 0 || label > p.K) {
      *flags |= BEVB200_LOSS_BAD_LABEL;
      if (dldx) *dldx = 0.0;
      return 0.0;
    }
    const double w = (double)__ldg(p.label_w + bn);
    const double l = sigmoid_focal(__ldg(p.heat + ((long long)b * p.K + ch) * p.N + n), label == ch, p.cls_f, dldx);
    if (dldx) *dldx *= w;
    return l * w;
  }
  const int c = ch - p.K, k = kMapOf[c], lc = c - kMapC0[k];
  const float pred = __ldg(p.map[k] + ((long long)b * kMapCh[k] + lc) * p.N + n);
  const float tv = __ldg(p.bt + bn * p.code + c);
  const double w = __fmul_rn(__ldg(p.bw + bn * p.code + c), p.cw[c]);
  const double d = (double)pred - (double)tv;
  if (dldx) *dldx = w * sgn(d);
  return fabs(d) * w;
}

__global__ void __launch_bounds__(kThreads) tfl_forward_kernel(const __grid_constant__ TFParams p, Part *parts) {
  double s = 0.0, c = 0.0;
  int flags = 0;
  long long e0;
  const int term = tf_term(p, blockIdx.x, &e0);
  if (term == 0) {
    dense_focal_tile(p.dense, p.dense_tgt, p.n_dense, e0, p.dense_vec, p.heat_f, s, c);
  } else {
    // layer elements (b, ch, pp) flattened as (b * C + ch) * P + pp, C the term's channel count
    const int l = (term - 1) >> 1, is_box = (term & 1) == 0, C = is_box ? p.code : p.K;
    const long long n = (long long)p.B * C * p.P;
    for (int r = 0; r < kTile / kThreads; ++r) {
      const long long e = e0 + r * kThreads + threadIdx.x;
      if (e >= n) break;
      const long long bc = e / p.P;
      const int pp = (int)(e - bc * p.P), b = (int)(bc / C), ch = (int)(bc - (long long)b * C);
      s += tf_column(p, b, is_box ? p.K + ch : ch, l * p.P + pp, nullptr, &flags);
    }
  }
  store_part(s, c, flags, parts + blockIdx.x);
}

// One warp per term.  losses: [0] heatmap, [1 + 2l] cls and [2 + 2l] bbox of layer l, [1 + 2 Lt] matched_ious
// (the last warp); avg: [0] heatmap, [1] the cls / bbox avg factor max(sum num_pos, 1).
__global__ void tfl_reduce_kernel(const __grid_constant__ TFParams p, const Part *__restrict__ parts,
                                  float *__restrict__ losses, float *__restrict__ avg, int32_t *__restrict__ status) {
  const int j = threadIdx.x >> 5, lane = threadIdx.x & 31, nterm = 1 + 2 * p.Lt;
  int flags = 0;
  if (j < nterm) {
    long long np = 0;
    for (int i = 0; i < p.n_num_pos; ++i) np += p.num_pos[i];
    const double a_layer = (double)(np > 1 ? np : 1);
    const int per = p.layer_tiles_cls + p.layer_tiles_box;
    int first, last;
    if (j == 0) {
      first = 0;
      last = p.dense_tiles;
    } else {
      const int l = (j - 1) >> 1;
      first = p.dense_tiles + l * per + ((j & 1) ? 0 : p.layer_tiles_cls);
      last = first + ((j & 1) ? p.layer_tiles_cls : p.layer_tiles_box);
    }
    const Part r = warp_sum(parts, first, last);
    flags = r.flags;
    if (lane == 0) {
      const double a = j == 0 ? fmax(r.cnt, 1.0) : a_layer;
      const double lw = j == 0 ? p.lw_heat : ((j & 1) ? p.lw_cls : p.lw_bbox);
      losses[j] = (float)(lw * (r.sum / a));
      if (j < 2) avg[j] = (float)(j == 0 ? a : a_layer);
    }
  } else if (lane == 0) {
    double s = 0.0;
    for (int i = 0; i < p.n_iou; ++i) s += p.mean_iou[i];
    losses[j] = (float)(s / p.n_iou);
  }
  store_status(flags, status);
}

__global__ void __launch_bounds__(kThreads) tfl_backward_kernel(const __grid_constant__ TFParams p,
                                                                const float *__restrict__ gout,
                                                                const float *__restrict__ avg) {
  if ((int)blockIdx.x < p.dense_tiles) {
    const double G = (double)gout[0] * p.lw_heat / (double)avg[0];
    dense_focal_grad_tile(p.dense, p.dense_tgt, p.gdense, p.n_dense, (long long)blockIdx.x * kTile, p.dense_vec,
                          p.heat_f, G);
    return;
  }
  // every element (b, ch, n) of the [B, K + code, N] cls / box gradient space
  const int C = p.K + p.code;
  const long long n_all = (long long)p.B * C * p.N, e0 = (long long)(blockIdx.x - p.dense_tiles) * kTile;
  for (int r = 0; r < kTile / kThreads; ++r) {
    const long long e = e0 + r * kThreads + threadIdx.x;
    if (e >= n_all) break;
    const long long bc = e / p.N;
    const int n = (int)(e - bc * p.N), b = (int)(bc / C), ch = (int)(bc - (long long)b * C), l = n / p.P;
    double g = 0.0;
    if (l < p.Lt) {
      double d;
      int fl = 0;
      tf_column(p, b, ch, n, &d, &fl);
      g = (double)gout[ch < p.K ? 1 + 2 * l : 2 + 2 * l] * (ch < p.K ? p.lw_cls : p.lw_bbox) / (double)avg[1] * d;
    }
    if (ch < p.K) {
      p.gheat[((long long)b * p.K + ch) * p.N + n] = (float)g;
    } else {
      const int c = ch - p.K, k = kMapOf[c], lc = c - kMapC0[k];
      p.gmap[k][((long long)b * kMapCh[k] + lc) * p.N + n] = (float)g;
    }
  }
}

// ---- host side -------------------------------------------------------------------------------------------
inline int tiles_of(long long n) { return (int)((n + kTile - 1) / kTile); }
inline bool aligned16(const void *q) { return ((uintptr_t)q & 15) == 0; }

// 0 ok, 1 invalid, 2 unsupported
int ch_check(int T, int B, const int *cat, int H, int W, int M, int code) {
  if (T < 1 || B < 1 || H < 1 || W < 1 || M < 1 || !cat || (code != 8 && code != 10)) return 1;
  for (int t = 0; t < T; ++t)
    if (cat[t] < 1) return 1;
  if (T > kMaxTasks || M > kMaxObjs || (long long)H * W >= (1LL << 31)) return 2;
  long long tiles = (long long)T * B;
  for (int t = 0; t < T; ++t) tiles += tiles_of((long long)B * cat[t] * H * W) + tiles_of((long long)B * code * H * W);
  return tiles > (1LL << 30) ? 2 : 0;
}

size_t ch_ws(int T, int B, const int *cat, int H, int W) {
  long long parts = (long long)T * B;
  for (int t = 0; t < T; ++t) parts += tiles_of((long long)B * cat[t] * H * W);
  return align_up((size_t)parts * sizeof(Part));
}

int tf_check(int B, int K, int H, int W, int N, int P, int Lt, int code) {
  if (B < 1 || K < 1 || H < 1 || W < 1 || P < 1 || N < P || N % P || Lt < 1 || Lt > N / P || (code != 8 && code != 10))
    return 1;
  if (Lt > kMaxLayers || (long long)B * (K + code) * N >= (1LL << 34) || (long long)B * K * H * W >= (1LL << 40))
    return 2;
  return 0;
}

void tf_tiles(TFParams &p) {
  p.dense_tiles = tiles_of(p.n_dense);
  p.layer_tiles_cls = tiles_of((long long)p.B * p.K * p.P);
  p.layer_tiles_box = tiles_of((long long)p.B * p.code * p.P);
  p.col_tiles = tiles_of((long long)p.B * (p.K + p.code) * p.N);
}

size_t tf_ws(TFParams &p) {
  tf_tiles(p);
  return align_up((size_t)(p.dense_tiles + p.Lt * (p.layer_tiles_cls + p.layer_tiles_box)) * sizeof(Part));
}

int fill_focal(Focal &f, const double *ab) {
  f.alpha = ab[0];
  f.gamma = ab[1];
  return 0;
}

}  // namespace
}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_centerhead_loss_workspace_bytes(int T, int B, const int *cat, int H, int W, int M, int code) {
  if (ch_check(T, B, cat, H, W, M, code) != 0) return 0;
  return ch_ws(T, B, cat, H, W);
}

static int centerhead_setup(CHParams &p, const float *const *heatmap, const float *const *reg,
                            const float *const *height, const float *const *dim, const float *const *rot,
                            const float *const *vel, const float *const *heat_target, const float *const *anno_box,
                            const int64_t *const *ind, const uint8_t *const *mask, const int *cat, int T, int B,
                            int H, int W, int M, int code, const float *code_weights_host, double cls_alpha,
                            double cls_gamma, double cls_weight, double bbox_weight, float *const *g_heat,
                            float *const *g_maps[kMaps], const char *fn) {
  const int sizes = ch_check(T, B, cat, H, W, M, code);
  if (sizes == 1) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: T, B, H, W, M and every class count must be at least 1, cat "
             "not null, code 8 or 10", fn);
    return BEVB200_EINVAL;
  }
  if (sizes == 2) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: at most %d tasks and %d objects per sample (got T %d, M %d, "
             "%d x %d)", fn, kMaxTasks, kMaxObjs, T, M, H, W);
    return BEVB200_EUNSUPPORTED;
  }
  if (!heatmap || !reg || !height || !dim || !rot || (code == 10 && !vel) || !heat_target || !anno_box || !ind ||
      !mask || !code_weights_host) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: null pointer", fn);
    return BEVB200_EINVAL;
  }
  memset(&p, 0, sizeof(p));
  p.T = T;
  p.B = B;
  p.HW = H * W;
  p.M = M;
  p.code = code;
  p.cls.alpha = cls_alpha;
  p.cls.gamma = cls_gamma;
  p.lw_cls = cls_weight;
  p.lw_bbox = bbox_weight;
  for (int c = 0; c < code; ++c) p.cw[c] = code_weights_host[c];
  p.zvec = p.HW % 4 == 0;
  int tiles = 0, ztiles = 0;
  for (int t = 0; t < T; ++t) {
    CHTask &tk = p.task[t];
    const float *const maps[kMaps] = {reg[t], height[t], dim[t], rot[t], code == 10 ? vel[t] : nullptr};
    if (!heatmap[t] || !heat_target[t] || !anno_box[t] || !ind[t] || !mask[t]) {
      snprintf(g_last_error, sizeof(g_last_error), "%s: null pointer of task %d", fn, t);
      return BEVB200_EINVAL;
    }
    for (int k = 0; k < kMaps; ++k) {
      if (k == 4 && code == 8) break;
      if (!maps[k] || (g_maps && !g_maps[k][t])) {
        snprintf(g_last_error, sizeof(g_last_error), "%s: null regression map %d of task %d", fn, k, t);
        return BEVB200_EINVAL;
      }
      tk.map[k] = maps[k];
      if (g_maps) {
        tk.gmap[k] = g_maps[k][t];
        p.zvec = p.zvec && aligned16(tk.gmap[k]);
      }
    }
    tk.heat = heatmap[t];
    tk.tgt = heat_target[t];
    tk.anno = anno_box[t];
    tk.ind = ind[t];
    tk.mask = mask[t];
    tk.n = (long long)B * cat[t] * p.HW;
    tk.vec = tk.n % 4 == 0 && aligned16(tk.heat) && aligned16(tk.tgt);
    if (g_heat) {
      if (!g_heat[t]) {
        snprintf(g_last_error, sizeof(g_last_error), "%s: null heatmap gradient of task %d", fn, t);
        return BEVB200_EINVAL;
      }
      tk.gheat = g_heat[t];
      tk.vec = tk.vec && aligned16(tk.gheat);
    }
    tk.tile0 = tiles;
    tk.ztile0 = ztiles;
    tiles += tiles_of(tk.n);
    ztiles += tiles_of((long long)B * code * p.HW);
  }
  p.heat_tiles = tiles;
  p.zero_tiles = ztiles;
  return BEVB200_OK;
}

int bevb200_centerhead_loss(const float *const *heatmap, const float *const *reg, const float *const *height,
                            const float *const *dim, const float *const *rot, const float *const *vel,
                            const float *const *heat_target, const float *const *anno_box, const int64_t *const *ind,
                            const uint8_t *const *mask, const int *cat, int T, int B, int H, int W, int M, int code,
                            const float *code_weights_host, double cls_alpha, double cls_gamma, double cls_weight,
                            double bbox_weight, float *losses, float *avg_factors, int32_t *status, void *workspace,
                            size_t workspace_bytes, void *stream) {
  CHParams p;
  const int rc = centerhead_setup(p, heatmap, reg, height, dim, rot, vel, heat_target, anno_box, ind, mask, cat, T, B,
                                  H, W, M, code, code_weights_host, cls_alpha, cls_gamma, cls_weight, bbox_weight,
                                  nullptr, nullptr, __func__);
  if (rc != BEVB200_OK) return rc;
  BEVB200_REQUIRE(losses && avg_factors && status, "null pointer");
  const size_t need = ch_ws(T, B, cat, H, W);
  if (workspace_bytes < need || !workspace) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace %zu < %zu bytes", __func__, workspace_bytes, need);
    return BEVB200_EWORKSPACE;
  }
  Part *parts = (Part *)workspace;
  cudaStream_t st = (cudaStream_t)stream;
  BEVB200_LAUNCH(chl_forward_kernel, p.heat_tiles + T * B, kThreads, 0, st, p, parts);
  BEVB200_LAUNCH(chl_reduce_kernel, 1, 64 * T, 0, st, p, parts, losses, avg_factors, status);
  return BEVB200_OK;
}

int bevb200_centerhead_loss_backward(
    const float *const *heatmap, const float *const *reg, const float *const *height, const float *const *dim,
    const float *const *rot, const float *const *vel, const float *const *heat_target, const float *const *anno_box,
    const int64_t *const *ind, const uint8_t *const *mask, const int *cat, int T, int B, int H, int W, int M, int code,
    const float *code_weights_host, double cls_alpha, double cls_gamma, double cls_weight, double bbox_weight,
    const float *grad_losses, const float *avg_factors, float *const *g_heatmap, float *const *g_reg,
    float *const *g_height, float *const *g_dim, float *const *g_rot, float *const *g_vel, void *stream) {
  BEVB200_REQUIRE(grad_losses && avg_factors && g_heatmap && g_reg && g_height && g_dim && g_rot &&
                      (code != 10 || g_vel),
                  "null pointer");
  float *const *g_maps[kMaps] = {g_reg, g_height, g_dim, g_rot, g_vel};
  CHParams p;
  const int rc = centerhead_setup(p, heatmap, reg, height, dim, rot, vel, heat_target, anno_box, ind, mask, cat, T, B,
                                  H, W, M, code, code_weights_host, cls_alpha, cls_gamma, cls_weight, bbox_weight,
                                  g_heatmap, g_maps, __func__);
  if (rc != BEVB200_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  BEVB200_LAUNCH(chl_backward_kernel, p.heat_tiles + p.zero_tiles, kThreads, 0, st, p, grad_losses, avg_factors);
  BEVB200_LAUNCH(chl_slots_kernel, T * B, kSlotThreads, 0, st, p, grad_losses, avg_factors);
  return BEVB200_OK;
}

static int transfusion_setup(TFParams &p, const float *dense_heatmap, const float *dense_target,
                             const float *heatmap, const float *center, const float *height, const float *dim,
                             const float *rot, const float *vel, const int64_t *labels, const int64_t *label_weights,
                             const float *bbox_targets, const float *bbox_weights, const int32_t *num_pos,
                             int n_num_pos, const float *mean_iou, int n_iou, int B, int K, int H, int W, int N, int P,
                             int Lt, int code, const float *code_weights_host, const double *focal_host,
                             const double *loss_weights_host, const char *fn) {
  const int sizes = tf_check(B, K, H, W, N, P, Lt, code);
  if (sizes == 1) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: B, K, H, W, P and the trained layers Lt must be at least 1, N a "
             "multiple of P with Lt <= N / P, code 8 or 10 (got B %d, K %d, %d x %d, N %d, P %d, Lt %d, code %d)", fn,
             B, K, H, W, N, P, Lt, code);
    return BEVB200_EINVAL;
  }
  if (sizes == 2) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: at most %d trained layers (got %d) or sizes too large", fn,
             kMaxLayers, Lt);
    return BEVB200_EUNSUPPORTED;
  }
  if (!dense_heatmap || !dense_target || !heatmap || !center || !height || !dim || !rot || (code == 10 && !vel) ||
      !labels || !label_weights || !bbox_targets || !bbox_weights || !num_pos || n_num_pos < 1 || !mean_iou ||
      n_iou < 1 || !code_weights_host || !focal_host || !loss_weights_host) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: null pointer or empty num_pos / mean_iou", fn);
    return BEVB200_EINVAL;
  }
  memset(&p, 0, sizeof(p));
  p.dense = dense_heatmap;
  p.dense_tgt = dense_target;
  p.heat = heatmap;
  const float *const maps[kMaps] = {center, height, dim, rot, code == 10 ? vel : nullptr};
  for (int k = 0; k < kMaps; ++k) p.map[k] = maps[k];
  p.bt = bbox_targets;
  p.bw = bbox_weights;
  p.mean_iou = mean_iou;
  p.labels = labels;
  p.label_w = label_weights;
  p.num_pos = num_pos;
  p.n_num_pos = n_num_pos;
  p.n_iou = n_iou;
  p.n_dense = (long long)B * K * H * W;
  p.B = B;
  p.K = K;
  p.N = N;
  p.P = P;
  p.Lt = Lt;
  p.code = code;
  p.dense_vec = p.n_dense % 4 == 0 && aligned16(dense_heatmap) && aligned16(dense_target);
  for (int c = 0; c < code; ++c) p.cw[c] = code_weights_host[c];
  fill_focal(p.heat_f, focal_host);
  fill_focal(p.cls_f, focal_host + 2);
  p.lw_heat = loss_weights_host[0];
  p.lw_cls = loss_weights_host[1];
  p.lw_bbox = loss_weights_host[2];
  tf_tiles(p);
  return BEVB200_OK;
}

size_t bevb200_transfusion_loss_workspace_bytes(int B, int K, int H, int W, int N, int P, int Lt, int code) {
  if (tf_check(B, K, H, W, N, P, Lt, code) != 0) return 0;
  TFParams p;
  memset(&p, 0, sizeof(p));
  p.n_dense = (long long)B * K * H * W;
  p.B = B;
  p.K = K;
  p.N = N;
  p.P = P;
  p.Lt = Lt;
  p.code = code;
  return tf_ws(p);
}

int bevb200_transfusion_loss(const float *dense_heatmap, const float *dense_target, const float *heatmap,
                             const float *center, const float *height, const float *dim, const float *rot,
                             const float *vel, const int64_t *labels, const int64_t *label_weights,
                             const float *bbox_targets, const float *bbox_weights, const int32_t *num_pos,
                             int n_num_pos, const float *mean_iou, int n_iou, int B, int K, int H, int W, int N, int P,
                             int Lt, int code, const float *code_weights_host, const double *focal_host,
                             const double *loss_weights_host, float *losses, float *avg_factors, int32_t *status,
                             void *workspace, size_t workspace_bytes, void *stream) {
  TFParams p;
  const int rc = transfusion_setup(p, dense_heatmap, dense_target, heatmap, center, height, dim, rot, vel, labels,
                                   label_weights, bbox_targets, bbox_weights, num_pos, n_num_pos, mean_iou, n_iou, B, K,
                                   H, W, N, P, Lt, code, code_weights_host, focal_host, loss_weights_host, __func__);
  if (rc != BEVB200_OK) return rc;
  BEVB200_REQUIRE(losses && avg_factors && status, "null pointer");
  const size_t need = tf_ws(p);
  if (workspace_bytes < need || !workspace) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace %zu < %zu bytes", __func__, workspace_bytes, need);
    return BEVB200_EWORKSPACE;
  }
  Part *parts = (Part *)workspace;
  cudaStream_t st = (cudaStream_t)stream;
  BEVB200_LAUNCH(tfl_forward_kernel, p.dense_tiles + Lt * (p.layer_tiles_cls + p.layer_tiles_box), kThreads, 0, st, p,
                 parts);
  BEVB200_LAUNCH(tfl_reduce_kernel, 1, 32 * (2 + 2 * Lt), 0, st, p, parts, losses, avg_factors, status);
  return BEVB200_OK;
}

int bevb200_transfusion_loss_backward(
    const float *dense_heatmap, const float *dense_target, const float *heatmap, const float *center,
    const float *height, const float *dim, const float *rot, const float *vel, const int64_t *labels,
    const int64_t *label_weights, const float *bbox_targets, const float *bbox_weights, int B, int K, int H, int W,
    int N, int P, int Lt, int code, const float *code_weights_host, const double *focal_host,
    const double *loss_weights_host, const float *grad_losses, const float *avg_factors, float *g_dense,
    float *g_heatmap, float *g_center, float *g_height, float *g_dim, float *g_rot, float *g_vel, void *stream) {
  TFParams p;
  const float one = 1.f;
  const int32_t one_pos = 1;
  // num_pos and mean_iou are not read by the backward; any non-null host address passes the checks
  const int rc = transfusion_setup(p, dense_heatmap, dense_target, heatmap, center, height, dim, rot, vel, labels,
                                   label_weights, bbox_targets, bbox_weights, &one_pos, 1, &one, 1, B, K, H, W, N, P,
                                   Lt, code, code_weights_host, focal_host, loss_weights_host, __func__);
  if (rc != BEVB200_OK) return rc;
  BEVB200_REQUIRE(grad_losses && avg_factors && g_dense && g_heatmap && g_center && g_height && g_dim && g_rot &&
                      (code != 10 || g_vel),
                  "null pointer");
  p.num_pos = nullptr;
  p.mean_iou = nullptr;
  p.gdense = g_dense;
  p.gheat = g_heatmap;
  float *const gm[kMaps] = {g_center, g_height, g_dim, g_rot, code == 10 ? g_vel : nullptr};
  for (int k = 0; k < kMaps; ++k) p.gmap[k] = gm[k];
  p.dense_vec = p.dense_vec && aligned16(g_dense);
  cudaStream_t st = (cudaStream_t)stream;
  BEVB200_LAUNCH(tfl_backward_kernel, p.dense_tiles + p.col_tiles, kThreads, 0, st, p, grad_losses, avg_factors);
  return BEVB200_OK;
}

}  // extern "C"
