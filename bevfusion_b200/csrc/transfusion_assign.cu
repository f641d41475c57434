// TransFusion training-target assignment on the device: the semantics of TransFusionHead.get_targets_single
// (models/heads/bbox/transfusion.py:408-525), HungarianAssigner3D.assign (core/bbox/assigners/
// hungarian_assigner.py:82-142) and scipy.optimize.linear_sum_assignment, for a whole batch, with no host
// synchronisation and no allocation.
//
// Three launches per call:
//   tf_cost_kernel     decode + matching cost of every (proposal, gt) pair of every segment (sample, decoder layer),
//                      written in the solver's orientation (rows = the shorter side) into the workspace
//   lsap_kernel        one CTA per segment: scipy's shortest-augmenting-path solver (rectangular_lsap.cpp, Crouse
//                      2016) restated in double, with the same tie breaks, so the assignment is scipy's bit for bit
//   tf_targets_kernel  one CTA per sample: labels, weights, encoded box targets, ious, num_pos and mean iou
// bevb200_lsap runs the solver alone on caller matrices.
//
// The fp32 arithmetic uses explicit round-to-nearest intrinsics: no FMA contraction, one rounding per op in the
// reference's order.  The BEV overlap is rot_overlap of box_nms.cu.
#include <math.h>

#include "common.cuh"
#include "rot_overlap.cuh"

namespace bevb200 {
namespace {

constexpr int kMaxAssign = BEVB200_ASSIGN_MAX;
constexpr int kCostThreads = 256;
constexpr int kTargetThreads = 256;
constexpr int kWideColumns = 1024;   // above this many solver columns a segment gets 8 warps, else one

// ---------------------------------------------------------------------------------------------------------
// Decode, cost, encode
// ---------------------------------------------------------------------------------------------------------
struct AssignParams {
  int B, L, P, K, nmax, box_dim, code_size;
  // prediction strides: heatmap [B, K, N], center [B, 2, N], height [B, 1, N], dim [B, 3, N], rot [B, 2, N]
  int N;
  float dec_osf, dec_vs_x, dec_vs_y, dec_pc_x, dec_pc_y;   // TransFusionBBoxCoder.decode
  float enc_pc_x, enc_pc_y, enc_inv_x, enc_inv_y;          // encode: (x - pc) * fp32(1 / fp32(osf * vs))
  float l1_start_x, l1_start_y, l1_range_x, l1_range_y;    // BBoxBEVL1Cost normalisation
  float alpha, one_minus_alpha, gamma, cls_w, reg_w, iou_w;
  int gamma_two;
  long long pos_weight;                                    // label weight of positives (train_cfg.pos_weight > 0)
};

struct Box7 {
  float x, y, z, dx, dy, dz, yaw;
};

__device__ __forceinline__ int clamp_count(const int32_t *counts, int idx, int cap) {
  const int n = counts ? counts[idx] : cap;
  return n < 0 ? 0 : (n > cap ? cap : n);
}

// TransFusionBBoxCoder.decode (transfusion_bbox_coder.py:39-74) of proposal column n of sample b; `decoded`
// (rows [B, N, box_dim]) replaces the raw predictions when the caller already holds decoded boxes.
__device__ __forceinline__ Box7 proposal_box(const float *__restrict__ center, const float *__restrict__ height,
                                             const float *__restrict__ dim, const float *__restrict__ rot,
                                             const float *__restrict__ decoded, const AssignParams &p, int b,
                                             int n) {
  Box7 r;
  if (decoded) {
    const float *d = decoded + ((long long)b * p.N + n) * p.box_dim;
    r.x = d[0];
    r.y = d[1];
    r.z = d[2];
    r.dx = d[3];
    r.dy = d[4];
    r.dz = d[5];
    r.yaw = d[6];
    return r;
  }
  const long long N = p.N;
  const float *c = center + (long long)b * 2 * N + n;
  r.x = __fadd_rn(__fmul_rn(__fmul_rn(c[0], p.dec_osf), p.dec_vs_x), p.dec_pc_x);
  r.y = __fadd_rn(__fmul_rn(__fmul_rn(c[N], p.dec_osf), p.dec_vs_y), p.dec_pc_y);
  const float *dm = dim + (long long)b * 3 * N + n;
  r.dx = expf(dm[0]);
  r.dy = expf(dm[N]);
  r.dz = expf(dm[2 * N]);
  r.z = __fsub_rn(height[(long long)b * N + n], __fmul_rn(r.dz, 0.5f));
  const float *ro = rot + (long long)b * 2 * N + n;
  r.yaw = atan2f(ro[0], ro[N]);
  return r;
}

__device__ __forceinline__ Box7 gt_box(const float *__restrict__ gt, const AssignParams &p, int b, int g) {
  const float *d = gt + ((long long)b * p.nmax + g) * p.box_dim;
  Box7 r;
  r.x = d[0];
  r.y = d[1];
  r.z = d[2];
  r.dx = d[3];
  r.dy = d[4];
  r.dz = d[5];
  r.yaw = d[6];
  return r;
}

// torch.max / torch.min: NaN propagates
__device__ __forceinline__ float tmax(float a, float b) { return (isnan(a) || isnan(b)) ? __fadd_rn(a, b) : fmaxf(a, b); }
__device__ __forceinline__ float tmin(float a, float b) { return (isnan(a) || isnan(b)) ? __fadd_rn(a, b) : fminf(a, b); }

// BaseInstance3DBoxes.overlaps(a, b) (base_box3d.py:356-445), mode iou, z the bottom: BEV overlap of the
// xywhr2xyxyr boxes times the height overlap, over clamp(va + vb - overlap, 1e-8).
__device__ __forceinline__ float iou3d(const Box7 &a, const Box7 &b) {
  const float ha = __fmul_rn(a.dx, 0.5f), hb = __fmul_rn(b.dx, 0.5f);   // w / 2
  const float ka = __fmul_rn(a.dy, 0.5f), kb = __fmul_rn(b.dy, 0.5f);
  const float xa[5] = {__fsub_rn(a.x, ha), __fsub_rn(a.y, ka), __fadd_rn(a.x, ha), __fadd_rn(a.y, ka), a.yaw};
  const float xb[5] = {__fsub_rn(b.x, hb), __fsub_rn(b.y, kb), __fadd_rn(b.x, hb), __fadd_rn(b.y, kb), b.yaw};
  const float bev = rot_overlap(load_rot(xa), load_rot(xb));
  const float top = tmin(__fadd_rn(a.z, a.dz), __fadd_rn(b.z, b.dz));
  const float bottom = tmax(a.z, b.z);
  float h = __fsub_rn(top, bottom);
  h = h < 0.f ? 0.f : h;   // clamp(min=0); NaN stays
  const float ov = __fmul_rn(bev, h);
  const float va = __fmul_rn(__fmul_rn(a.dx, a.dy), a.dz), vb = __fmul_rn(__fmul_rn(b.dx, b.dy), b.dz);
  float u = __fsub_rn(__fadd_rn(va, vb), ov);
  u = u < 1e-8f ? 1e-8f : u;
  return __fdiv_rn(ov, u);
}

// FocalLossCost (mmdet 2.20 match_cost.py) of one logit for one gt label, BBoxBEVL1Cost and IoU3DCost
// (hungarian_assigner.py:13-35), summed as cls + reg + iou.
__device__ __forceinline__ float pair_cost(float logit, const Box7 &pb, const Box7 &gb, const AssignParams &p) {
  const float sp = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-logit)));                      // sigmoid
  const float q = __fsub_rn(1.f, sp);
  const float pg = p.gamma_two ? __fmul_rn(sp, sp) : powf(sp, p.gamma);
  const float qg = p.gamma_two ? __fmul_rn(q, q) : powf(q, p.gamma);
  const float neg = __fmul_rn(__fmul_rn(-logf(__fadd_rn(q, 1e-12f)), p.one_minus_alpha), pg);
  const float pos = __fmul_rn(__fmul_rn(-logf(__fadd_rn(sp, 1e-12f)), p.alpha), qg);
  const float cls = __fmul_rn(__fsub_rn(pos, neg), p.cls_w);
  const float px = __fdiv_rn(__fsub_rn(pb.x, p.l1_start_x), p.l1_range_x);
  const float py = __fdiv_rn(__fsub_rn(pb.y, p.l1_start_y), p.l1_range_y);
  const float gx = __fdiv_rn(__fsub_rn(gb.x, p.l1_start_x), p.l1_range_x);
  const float gy = __fdiv_rn(__fsub_rn(gb.y, p.l1_start_y), p.l1_range_y);
  const float reg = __fmul_rn(__fadd_rn(fabsf(__fsub_rn(px, gx)), fabsf(__fsub_rn(py, gy))), p.reg_w);
  const float iouc = __fmul_rn(-iou3d(pb, gb), p.iou_w);
  return __fadd_rn(__fadd_rn(cls, reg), iouc);
}

// One thread per (proposal, gt) pair of segment s = b * L + l (blockIdx.y).  The segment's matrix goes to
// ws_cost + s * P * nmax in the solver's orientation: [G, P] when G < P (scipy transposes), else [P, G].
// cost_out (nullable): [S, P, nmax] proposal-major, for tests.
__global__ void __launch_bounds__(kCostThreads)
    tf_cost_kernel(const float *__restrict__ heatmap, const float *__restrict__ center,
                   const float *__restrict__ height, const float *__restrict__ dim, const float *__restrict__ rot,
                   const float *__restrict__ decoded, const float *__restrict__ gt, const int32_t *__restrict__ labels,
                   const int32_t *__restrict__ counts, const __grid_constant__ AssignParams p,
                   float *__restrict__ ws_cost, float *__restrict__ cost_out) {
  const int s = blockIdx.y, b = s / p.L, l = s % p.L;
  const int G = clamp_count(counts, b, p.nmax);
  const long long t = (long long)blockIdx.x * kCostThreads + threadIdx.x;
  if (G == 0 || t >= (long long)p.P * G) return;
  const bool tr = G < p.P;
  int pi, g;
  if (tr) {
    g = (int)(t / p.P);
    pi = (int)(t % p.P);
  } else {
    pi = (int)(t / G);
    g = (int)(t % G);
  }
  const int n = l * p.P + pi;
  const Box7 pb = proposal_box(center, height, dim, rot, decoded, p, b, n);
  const Box7 gb = gt_box(gt, p, b, g);
  const int lab = labels[(long long)b * p.nmax + g];
  float c;
  if (lab < 0 || lab >= p.K) {
    c = __int_as_float(0x7fc00000);   // the reference raises on the label; a NaN column fails the segment
  } else {
    c = pair_cost(heatmap[((long long)b * p.K + lab) * p.N + n], pb, gb, p);
  }
  ws_cost[(long long)s * p.P * p.nmax + t] = c;
  if (cost_out) cost_out[((long long)s * p.P + pi) * p.nmax + g] = c;
}

// ---------------------------------------------------------------------------------------------------------
// The solver
// ---------------------------------------------------------------------------------------------------------
// A segment's matrix, in the caller's orientation: element (r, c) of orig rows R x cols C at base + r*rs + c*cs.
// compact: the pipeline's workspace layout (written in the solver's orientation, rows of the shorter side,
// densely packed); otherwise [S, R, C] row-major with the given pads.
struct LsapArgs {
  const float *cost;
  const int32_t *row_counts, *col_counts;
  int S, R, C, counts_div, compact, cap;   // cap = max(R, C): shared-memory sizing
  long long seg_stride;
  int32_t *col4row, *row4col, *status, *steps;
};

struct Key {
  double v;
  int tie;   // unassigned: -it, else it + 2^30: the smaller key wins
};

__device__ __forceinline__ bool key_less(const Key &a, const Key &b) {
  return a.v < b.v || (a.v == b.v && a.tie < b.tie);
}

__device__ __forceinline__ Key warp_min(Key k) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Key q;
    q.v = __shfl_xor_sync(0xffffffffu, k.v, o);
    q.tie = __shfl_xor_sync(0xffffffffu, k.tie, o);
    if (key_less(q, k)) k = q;
  }
  return k;
}

// scipy's rectangular_lsap.cpp: for each row cur, a Dijkstra search of shortest augmenting paths over the
// remaining columns, reduced costs r = ((minVal + cost[i][j]) - u[i]) - v[j] in double.  The column selected at
// each step is scipy's: among the columns of least path cost, the last unassigned one in `remaining` order, else
// the first one.  `remaining` is kept as the same permutation (reversed start, swap-with-last removal), so the
// parallel argmin over the key (spc, unassigned ? -it : it + 2^30) picks the same column.
__global__ void lsap_kernel(const LsapArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int cap = a.cap;
  double *v = (double *)smem;
  double *spc = v + cap;
  double *u = spc + cap;
  int *path = (int *)(u + cap);
  int *row4col = path + cap;
  int *col4row = row4col + cap;
  int *remaining = col4row + cap;
  unsigned char *SR = (unsigned char *)(remaining + cap);
  unsigned char *SC = SR + cap;
  __shared__ Key red[8];
  __shared__ int sh_flag, sh_sink, sh_i;
  __shared__ double sh_min;

  const int s = blockIdx.x, tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31, warp = tid >> 5;
  const int cidx = s / a.counts_div;
  const int R0 = clamp_count(a.row_counts, cidx, a.R), C0 = clamp_count(a.col_counts, cidx, a.C);
  const bool tr = C0 < R0;
  const int nr = tr ? C0 : R0, nc = tr ? R0 : C0;
  const float *base = a.cost + (long long)s * a.seg_stride;
  long long rs, cs;   // strides of the caller's orientation
  if (a.compact) {
    rs = tr ? 1 : C0;
    cs = tr ? R0 : 1;
  } else {
    rs = a.C;
    cs = 1;
  }
  const long long si = tr ? cs : rs, sj = tr ? rs : cs;   // strides of the solver's orientation

  // scipy refuses NaN and -inf entries before it solves
  if (tid == 0) sh_flag = 0;
  __syncthreads();
  for (long long e = tid; e < (long long)nr * nc; e += nthr) {
    const float c = base[(e / nc) * si + (e % nc) * sj];
    if (isnan(c) || c == -INFINITY) sh_flag = BEVB200_ASSIGN_INVALID_COST;
  }
  for (int j = tid; j < nc; j += nthr) {
    v[j] = 0.0;
    row4col[j] = -1;
    path[j] = -1;
  }
  for (int i = tid; i < nr; i += nthr) {
    u[i] = 0.0;
    col4row[i] = -1;
  }
  __syncthreads();
  int flag = sh_flag;
  long long nsteps = 0;

  for (int cur = 0; cur < nr && !flag; ++cur) {
    for (int j = tid; j < nc; j += nthr) {
      spc[j] = INFINITY;
      SC[j] = 0;
      remaining[j] = nc - 1 - j;
    }
    for (int i = tid; i < nr; i += nthr) SR[i] = 0;
    int num_remaining = nc, i = cur, sink = -1;
    double minVal = 0.0;
    __syncthreads();
    while (sink == -1) {
      ++nsteps;
      if (tid == 0) SR[i] = 1;
      const float *row = base + (long long)i * si;
      const double ui = u[i];
      Key best;
      best.v = INFINITY;
      best.tie = 0x7fffffff;
      for (int it = tid; it < num_remaining; it += nthr) {
        const int j = remaining[it];
        const double r = __dsub_rn(__dsub_rn(__dadd_rn(minVal, (double)row[(long long)j * sj]), ui), v[j]);
        double sj_cost = spc[j];
        if (r < sj_cost) {
          path[j] = i;
          spc[j] = r;
          sj_cost = r;
        }
        Key k;
        k.v = sj_cost;
        k.tie = row4col[j] == -1 ? -it : it + (1 << 30);
        if (key_less(k, best)) best = k;
      }
      best = warp_min(best);
      if (nthr > 32) {
        if (lane == 0) red[warp] = best;
        __syncthreads();
        if (warp == 0) {
          best = lane < (nthr >> 5) ? red[lane] : Key{INFINITY, 0x7fffffff};
          best = warp_min(best);
        }
      }
      if (tid == 0) {
        if (best.v == INFINITY) {   // infeasible: scipy raises
          sh_flag = BEVB200_ASSIGN_INFEASIBLE;
        } else {
          const int it = best.tie < 0 ? -best.tie : (best.tie >= (1 << 30) ? best.tie - (1 << 30) : 0);
          const int j = remaining[it];
          if (row4col[j] == -1) {
            sh_sink = j;
          } else {
            sh_sink = -1;
            sh_i = row4col[j];
          }
          SC[j] = 1;
          remaining[it] = remaining[num_remaining - 1];
          sh_min = best.v;
        }
      }
      __syncthreads();
      flag = sh_flag;
      if (flag) break;
      minVal = sh_min;
      sink = sh_sink;
      if (sink == -1) i = sh_i;
      --num_remaining;
    }
    if (flag) break;
    // duals: u[cur] += minVal; u[i] += minVal - spc[col4row[i]] for the other rows of SR; v[j] -= minVal - spc[j]
    for (int r = tid; r < nr; r += nthr) {
      if (r == cur) {
        u[r] = __dadd_rn(u[r], minVal);
      } else if (SR[r]) {
        u[r] = __dadd_rn(u[r], __dsub_rn(minVal, spc[col4row[r]]));
      }
    }
    for (int j = tid; j < nc; j += nthr)
      if (SC[j]) v[j] = __dsub_rn(v[j], __dsub_rn(minVal, spc[j]));
    __syncthreads();
    if (tid == 0) {   // augment back to cur
      int j = sink;
      while (true) {
        const int r = path[j];
        row4col[j] = r;
        const int t = col4row[r];
        col4row[r] = j;
        j = t;
        if (r == cur) break;
      }
    }
    __syncthreads();
  }
  // outputs in the caller's orientation; a failed segment has no matches
  int32_t *c4r = a.col4row + (long long)s * a.R, *r4c = a.row4col ? a.row4col + (long long)s * a.C : nullptr;
  for (int r = tid; r < a.R; r += nthr) {
    int m = -1;
    if (!flag && r < R0) m = tr ? row4col[r] : col4row[r];
    c4r[r] = m;
  }
  if (r4c) {
    for (int c = tid; c < a.C; c += nthr) {
      int m = -1;
      if (!flag && c < C0) m = tr ? col4row[c] : row4col[c];
      r4c[c] = m;
    }
  }
  if (tid == 0) {
    if (a.status) a.status[s] = flag;
    if (a.steps) a.steps[s] = (int32_t)(nsteps > 0x7fffffffll ? 0x7fffffffll : nsteps);
  }
}

size_t lsap_smem_bytes(int cap) { return (size_t)cap * (3 * sizeof(double) + 4 * sizeof(int) + 2); }

int lsap_threads(int cap) { return cap > kWideColumns ? 256 : 32; }

int launch_lsap(const LsapArgs &a, cudaStream_t st) {
  if (a.S == 0) return BEVB200_OK;
  const size_t smem = lsap_smem_bytes(a.cap);
  if (smem > 48 * 1024)   // the shipped sizes stay below the default limit
    BEVB200_CUDA(cudaFuncSetAttribute(lsap_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  BEVB200_LAUNCH(lsap_kernel, a.S, lsap_threads(a.cap), smem, st, a);
  return BEVB200_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Targets
// ---------------------------------------------------------------------------------------------------------
// One CTA per sample over its N = L * P proposals: match[s * P + p] is the gt of proposal p of segment s or -1.
__global__ void __launch_bounds__(kTargetThreads)
    tf_targets_kernel(const float *__restrict__ center, const float *__restrict__ height,
                      const float *__restrict__ dim, const float *__restrict__ rot, const float *__restrict__ decoded,
                      const float *__restrict__ gt, const int32_t *__restrict__ labels,
                      const int32_t *__restrict__ counts, const __grid_constant__ AssignParams p,
                      const int32_t *__restrict__ match, const int32_t *__restrict__ seg_status,
                      int64_t *__restrict__ out_labels, int64_t *__restrict__ out_label_w,
                      float *__restrict__ bbox_targets, float *__restrict__ bbox_weights, float *__restrict__ ious,
                      int32_t *__restrict__ num_pos, float *__restrict__ mean_iou, int32_t *__restrict__ status,
                      int64_t *__restrict__ gt_inds, float *__restrict__ max_overlaps) {
  __shared__ double red_sum[kTargetThreads];
  __shared__ int red_n[kTargetThreads];
  __shared__ int sh_status;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int G = clamp_count(counts, b, p.nmax);
  if (tid == 0) {
    int st = 0;
    for (int l = 0; l < p.L; ++l) st |= seg_status[b * p.L + l];
    sh_status = st;
  }
  __syncthreads();
  for (int g = tid; g < G; g += kTargetThreads) {
    const int lab = labels[(long long)b * p.nmax + g];
    if (lab < 0 || lab >= p.K) atomicOr(&sh_status, BEVB200_ASSIGN_BAD_LABEL);
  }
  double sum = 0.0;
  int npos = 0;
  for (int n = tid; n < p.N; n += kTargetThreads) {
    const int l = n / p.P, pi = n % p.P;
    const int g = match[((long long)b * p.L + l) * p.P + pi];
    const long long o = (long long)b * p.N + n;
    float *bt = bbox_targets + o * p.code_size, *bw = bbox_weights + o * p.code_size;
    if (g < 0) {
      out_labels[o] = p.K;
      out_label_w[o] = 1;
      for (int d = 0; d < p.code_size; ++d) {
        bt[d] = 0.f;
        bw[d] = 0.f;
      }
      ious[o] = 0.f;
      if (gt_inds) gt_inds[o] = 0;
      if (max_overlaps) max_overlaps[o] = 0.f;
      continue;
    }
    const Box7 gb = gt_box(gt, p, b, g);
    const float iou = iou3d(proposal_box(center, height, dim, rot, decoded, p, b, n), gb);
    out_labels[o] = labels[(long long)b * p.nmax + g];
    out_label_w[o] = p.pos_weight;
    // TransFusionBBoxCoder.encode (transfusion_bbox_coder.py:24-37)
    bt[0] = __fmul_rn(__fsub_rn(gb.x, p.enc_pc_x), p.enc_inv_x);
    bt[1] = __fmul_rn(__fsub_rn(gb.y, p.enc_pc_y), p.enc_inv_y);
    bt[2] = __fadd_rn(gb.z, __fmul_rn(gb.dz, 0.5f));
    bt[3] = logf(gb.dx);
    bt[4] = logf(gb.dy);
    bt[5] = logf(gb.dz);
    bt[6] = sinf(gb.yaw);
    bt[7] = cosf(gb.yaw);
    if (p.code_size == 10) {
      const float *row = gt + ((long long)b * p.nmax + g) * p.box_dim;
      bt[8] = row[7];
      bt[9] = row[8];
    }
    for (int d = 0; d < p.code_size; ++d) bw[d] = 1.f;
    const float c = iou < 0.f ? 0.f : (iou > 1.f ? 1.f : iou);   // clamp(0, 1); NaN stays
    ious[o] = c;
    if (gt_inds) gt_inds[o] = g + 1;
    if (max_overlaps) max_overlaps[o] = iou;
    sum += (double)c;
    ++npos;
  }
  red_sum[tid] = sum;
  red_n[tid] = npos;
  __syncthreads();
  for (int w = kTargetThreads / 2; w > 0; w >>= 1) {   // fixed tree: the result is reproducible
    if (tid < w) {
      red_sum[tid] += red_sum[tid + w];
      red_n[tid] += red_n[tid + w];
    }
    __syncthreads();
  }
  if (tid == 0) {
    const int np = red_n[0];
    num_pos[b] = np;
    // ious[pos].sum() / max(num_pos, 1): torch divides by the Python int as a multiply by its fp32 reciprocal
    mean_iou[b] = __fmul_rn((float)red_sum[0], __fdiv_rn(1.f, (float)(np > 1 ? np : 1)));
    status[b] = sh_status;
  }
}

size_t assign_ws_bytes(int B, int L, int P, int nmax) {
  const size_t S = (size_t)B * L;
  return align_up(S * P * nmax * sizeof(float)) + align_up(S * P * sizeof(int32_t)) +
         align_up(S * sizeof(int32_t));
}

bool assign_sizes_ok(int B, int L, int P, int nmax) {
  return B >= 0 && L >= 1 && P >= 0 && nmax >= 0 && P <= kMaxAssign && nmax <= kMaxAssign &&
         (long long)B * L <= BEVB200_ASSIGN_MAX_SEGMENTS && (long long)L * P <= 0x7fffffffll;
}

}  // namespace
}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_lsap_workspace_bytes(int S, int R, int C) {
  (void)S;
  (void)R;
  (void)C;
  return 0;
}

int bevb200_lsap(const float *cost, const int32_t *row_counts, const int32_t *col_counts, int S, int R, int C,
                 int32_t *col4row, int32_t *row4col, int32_t *status, int32_t *steps, void *workspace,
                 size_t workspace_bytes, void *stream) {
  (void)workspace;
  (void)workspace_bytes;
  BEVB200_REQUIRE(S >= 0 && R >= 0 && C >= 0, "negative size");
  if (R > kMaxAssign || C > kMaxAssign || S > BEVB200_ASSIGN_MAX_SEGMENTS) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: at most %d rows and columns and %d segments (got %d, %d, %d)",
             __func__, kMaxAssign, BEVB200_ASSIGN_MAX_SEGMENTS, R, C, S);
    return BEVB200_EUNSUPPORTED;
  }
  if (S == 0) return BEVB200_OK;
  BEVB200_REQUIRE(col4row || R == 0, "null col4row");
  BEVB200_REQUIRE(cost || (long long)R * C == 0, "null cost");
  LsapArgs a;
  a.cost = cost;
  a.row_counts = row_counts;
  a.col_counts = col_counts;
  a.S = S;
  a.R = R;
  a.C = C;
  a.counts_div = 1;
  a.compact = 0;
  a.cap = max(max(R, C), 1);
  a.seg_stride = (long long)R * C;
  a.col4row = col4row;
  a.row4col = row4col;
  a.status = status;
  a.steps = steps;
  return launch_lsap(a, (cudaStream_t)stream);
}

size_t bevb200_transfusion_assign_workspace_bytes(int B, int L, int P, int nmax) {
  if (!assign_sizes_ok(B, L, P, nmax)) return 0;
  return assign_ws_bytes(B, L, P, nmax);
}

int bevb200_transfusion_assign(const float *heatmap, const float *center, const float *height, const float *dim,
                               const float *rot, const float *decoded, int B, int L, int P, int K,
                               const float *gt_boxes, const int32_t *gt_labels, const int32_t *gt_counts, int nmax,
                               int box_dim, double coder_pc_x, double coder_pc_y, double coder_vs_x,
                               double coder_vs_y, int coder_out_size_factor, int code_size, double pc_x0,
                               double pc_y0, double pc_x1, double pc_y1, double cls_weight, double alpha,
                               double gamma, double reg_weight, double iou_weight, double pos_weight,
                               int64_t *labels, int64_t *label_weights, float *bbox_targets, float *bbox_weights,
                               float *ious, int32_t *num_pos, float *mean_iou, int32_t *status, int64_t *gt_inds,
                               float *max_overlaps, float *cost_out, int32_t *steps, void *workspace,
                               size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(B >= 0 && L >= 1 && P >= 0 && nmax >= 0, "bad size");
  if (!assign_sizes_ok(B, L, P, nmax)) {
    snprintf(g_last_error, sizeof(g_last_error),
             "%s: at most %d proposals and gts per segment and %d segments (got P %d, nmax %d, S %lld)", __func__,
             kMaxAssign, BEVB200_ASSIGN_MAX_SEGMENTS, P, nmax, (long long)B * L);
    return BEVB200_EUNSUPPORTED;
  }
  BEVB200_REQUIRE(K >= 1 && K <= BEVB200_ASSIGN_MAX_CLASSES, "num_classes out of range");
  BEVB200_REQUIRE(box_dim == 7 || box_dim == 9, "box_dim must be 7 or 9");
  BEVB200_REQUIRE(code_size == 8 || (code_size == 10 && box_dim == 9), "code_size must be 8, or 10 with box_dim 9");
  BEVB200_REQUIRE(coder_out_size_factor >= 1, "bad out_size_factor");
  if (B == 0 || P == 0) return BEVB200_OK;
  BEVB200_REQUIRE(heatmap && (decoded || (center && height && dim && rot)), "null predictions");
  BEVB200_REQUIRE((gt_boxes && gt_labels) || nmax == 0, "null ground truth");
  BEVB200_REQUIRE(labels && label_weights && bbox_targets && bbox_weights && ious && num_pos && mean_iou && status,
                  "null output");
  const size_t need = assign_ws_bytes(B, L, P, nmax);
  if (workspace_bytes < need || !workspace) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace %zu < %zu bytes", __func__, workspace_bytes, need);
    return BEVB200_EWORKSPACE;
  }
  AssignParams p;
  memset(&p, 0, sizeof(p));
  p.B = B;
  p.L = L;
  p.P = P;
  p.K = K;
  p.nmax = nmax;
  p.box_dim = box_dim;
  p.code_size = code_size;
  p.N = L * P;
  p.dec_osf = (float)coder_out_size_factor;
  p.dec_vs_x = (float)coder_vs_x;
  p.dec_vs_y = (float)coder_vs_y;
  p.dec_pc_x = (float)coder_pc_x;
  p.dec_pc_y = (float)coder_pc_y;
  p.enc_pc_x = (float)coder_pc_x;
  p.enc_pc_y = (float)coder_pc_y;
  // (x - pc) / (osf * vs): the Python-float divisor becomes an fp32 scalar whose fp32 reciprocal multiplies
  p.enc_inv_x = 1.f / (float)(coder_out_size_factor * coder_vs_x);
  p.enc_inv_y = 1.f / (float)(coder_out_size_factor * coder_vs_y);
  p.l1_start_x = (float)pc_x0;
  p.l1_start_y = (float)pc_y0;
  p.l1_range_x = (float)pc_x1 - (float)pc_x0;
  p.l1_range_y = (float)pc_y1 - (float)pc_y0;
  p.alpha = (float)alpha;
  p.one_minus_alpha = (float)(1.0 - alpha);
  p.gamma = (float)gamma;
  p.gamma_two = gamma == 2.0;
  p.cls_w = (float)cls_weight;
  p.reg_w = (float)reg_weight;
  p.iou_w = (float)iou_weight;
  p.pos_weight = pos_weight > 0 ? (long long)pos_weight : 1;   // a float stored into the int64 tensor truncates
  Arena ar(workspace, workspace_bytes);
  const int S = B * L;
  float *ws_cost = ar.take<float>((size_t)S * P * nmax);
  int32_t *match = ar.take<int32_t>((size_t)S * P);
  int32_t *seg_status = ar.take<int32_t>((size_t)S);
  cudaStream_t st = (cudaStream_t)stream;
  if (nmax > 0) {
    const dim3 grid((unsigned)(((long long)P * nmax + kCostThreads - 1) / kCostThreads), S);
    BEVB200_LAUNCH(tf_cost_kernel, grid, kCostThreads, 0, st, heatmap, center, height, dim, rot, decoded, gt_boxes,
                   gt_labels, gt_counts, p, ws_cost, cost_out);
  }
  LsapArgs a;
  a.cost = ws_cost;
  a.row_counts = nullptr;
  a.col_counts = nmax > 0 ? gt_counts : nullptr;
  a.S = S;
  a.R = P;
  a.C = nmax;
  a.counts_div = L;
  a.compact = 1;
  a.cap = max(max(P, nmax), 1);
  a.seg_stride = (long long)P * nmax;
  a.col4row = match;
  a.row4col = nullptr;
  a.status = seg_status;
  a.steps = steps;
  const int rc = launch_lsap(a, st);
  if (rc != BEVB200_OK) return rc;
  BEVB200_LAUNCH(tf_targets_kernel, B, kTargetThreads, 0, st, center, height, dim, rot, decoded, gt_boxes, gt_labels,
                 gt_counts, p, match, seg_status, labels, label_weights, bbox_targets, bbox_weights, ious, num_pos,
                 mean_iou, status, gt_inds, max_overlaps);
  return BEVB200_OK;
}

}  // extern "C"
