// Fused LSS lift + pool, column formulation (round 2; SURVEY.md section 8(f)1).
//
//   out[cell, :] = sum over kept frustum points p = (cam, d, h, w) in the cell of depth[p] * ctx[cam, h, w, :]
//   (mmdet3d/models/vtransforms/lss.py:68-73 / depth_lss.py:92-97 followed by base.py:141-176, bev_pool.py:84-98)
//
// The round-1 kernel (bevpool.cu, MODE 2) walks the sorted point list and gathers the 320-byte context row of
// EVERY point from L2: 1.84 M x 320 B = 588 MB of L2 -> SM traffic for 13.4 MB of inputs, the same 164 us as pooling
// the materialised volume.  But the BEV grid collapses z: the fH pixels of one image column (cam, w) at one depth bin
// almost always fall into the same cell (exactly, for a level camera), i.e. the sum over a cell is a sum over
// (column, depth bin) SEGMENTS, and a segment's value is a tiny matrix-vector product of data that lives in one
// image column:
//     T[seg, :] = sum_{h in mask(seg)} depth[cam, d, h, w] * ctx[cam, h, w, :]
// Nothing is assumed about the camera: a segment is "the pixels of column (cam, w) at depth bin d that fall into
// cell c", described by a bit mask over h, so tilted cameras / the z-range filter just produce more segments.
//   per calibration (bevb200_bev_pool_lift_prepare): key (column, d, interval) of every kept point -> radix sort ->
//     run-length encode into segments (mask = OR of 1 << h) -> slot of every segment in interval-major order;
//   per frame, kernel 1 (one CTA per image column): the column's context rows (fH x C) and depth values (D x fH)
//     are staged in shared memory ONCE and all of the column's segments are evaluated from there; T rows go to
//     their slots (n_seg x C floats, ~20 MB at C2);
//   per frame, kernel 2 (one warp per interval): adds the interval's T rows in slot order (fixed order: the result
//     is reproducible), writes the cell, zero-fills the empty cells in between.
// HBM / L2 traffic per frame: depth + ctx once (13.4 MB), T written and read once (~2 x 20 MB), the BEV grid once.
// The backward (gradients of depth and ctx, section "backward" below) runs over the same segment tables.
#include <cub/cub.cuh>

#include "bevpool.cuh"

namespace bevb200 {

struct LiftGeom {
  int depth_bins, fh, fw, ncols;   // ncols = B * N * fw image columns
};

// sorted position s -> interval index (intervals tile [0, n_kept)); one thread per interval
__global__ void lift_interval_ids_kernel(const int32_t *__restrict__ starts, int n_intervals, int n_kept,
                                         int32_t *__restrict__ ival_of, const int32_t *__restrict__ counts) {
  device_counts(counts, n_kept, n_intervals);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_intervals; i += gridDim.x * blockDim.x) {
    const int s0 = starts[i], s1 = i + 1 < n_intervals ? starts[i + 1] : n_kept;
    for (int s = s0; s < s1; ++s) ival_of[s] = i;
  }
}

// key = ((column * D + d) << 32) | interval, value = h.  With device counts the keys cover the capacity n_items, and
// the rows at or past n_kept get the key (ncols * D) << 32, which sorts after every real one.
__global__ void lift_keys_kernel(const int32_t *__restrict__ perm, const int32_t *__restrict__ ival_of, int n_kept,
                                 LiftGeom g, unsigned long long *__restrict__ keys, uint32_t *__restrict__ vals,
                                 const int32_t *__restrict__ counts, int n_items) {
  if (counts) n_kept = __ldg(counts); else n_items = n_kept;
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n_items; s += gridDim.x * blockDim.x) {
    if (s >= n_kept) {
      keys[s] = ((unsigned long long)g.ncols * g.depth_bins) << 32;
      vals[s] = 0u;
      continue;
    }
    long long p = perm[s];                         // ((cam * D + d) * fh + h) * fw + w,  cam = b * N + n
    const int w = (int)(p % g.fw); p /= g.fw;
    const int h = (int)(p % g.fh); p /= g.fh;
    const int d = (int)(p % g.depth_bins);
    const int cam = (int)(p / g.depth_bins);
    const unsigned long long cd = (unsigned long long)(cam * g.fw + w) * g.depth_bins + d;
    keys[s] = (cd << 32) | (uint32_t)ival_of[s];
    vals[s] = (uint32_t)h;
  }
}

// n_items flags; a run heads a segment only below the device n_kept (when `counts` is given)
__global__ void lift_heads_kernel(const unsigned long long *__restrict__ keys, int n_items, uint32_t *__restrict__ flags,
                                  const int32_t *__restrict__ counts) {
  const int n = counts ? __ldg(counts) : n_items;
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n_items; s += gridDim.x * blockDim.x)
    flags[s] = s < n && (s == 0 || keys[s] != keys[s - 1]) ? 1u : 0u;
}

// sync-free prepare: n_segments = the scan total; lift_form = BEVB200_LIFT_ROWS when it exceeds the cap of the column
// tables
__global__ void lift_form_kernel(const uint32_t *__restrict__ total, int max_segments, int32_t *__restrict__ n_segments,
                                 int32_t *__restrict__ lift_form) {
  const uint32_t n_seg = *total;
  *n_segments = (int32_t)n_seg;
  *lift_form = n_seg > (uint32_t)max_segments ? BEVB200_LIFT_ROWS : BEVB200_LIFT_COLUMNS;
}

// one thread per sorted element that heads a run: segment record
__global__ void lift_segments_kernel(const unsigned long long *__restrict__ keys, const uint32_t *__restrict__ hs,
                                     const uint32_t *__restrict__ flags, const uint32_t *__restrict__ pos, int n,
                                     unsigned long long *__restrict__ seg_key, unsigned long long *__restrict__ seg_mask,
                                     const int32_t *__restrict__ counts, uint32_t seg_cap) {
  if (counts) n = __ldg(counts);
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
    if (!flags[s] || pos[s] >= seg_cap) continue;   // past the cap the column tables are not used
    const unsigned long long k = keys[s];
    unsigned long long m = 0;
    for (int e = s; e < n && keys[e] == k; ++e) m |= 1ull << hs[e];
    seg_key[pos[s]] = k;
    seg_mask[pos[s]] = m;
  }
}

// with a device segment count (n_seg_dev) the n_items entries past it get the key `beyond`, which sorts last
__global__ void lift_seg_ival_kernel(const unsigned long long *__restrict__ seg_key, int n_items,
                                     uint32_t *__restrict__ ival, uint32_t *__restrict__ idx,
                                     const int32_t *__restrict__ n_seg_dev, uint32_t beyond) {
  const int n_seg = n_seg_dev ? min(__ldg(n_seg_dev), n_items) : n_items;
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n_items; s += gridDim.x * blockDim.x) {
    ival[s] = s < n_seg ? (uint32_t)(seg_key[s] & 0xffffffffull) : beyond;
    idx[s] = (uint32_t)s;
  }
}

// after the stable sort of the segments by interval: slot[seg] = its position; first slot of every interval;
// first segment of every column (segments are in (column, d, interval) order)
__global__ void lift_slots_kernel(const uint32_t *__restrict__ ival_sorted, const uint32_t *__restrict__ seg_sorted,
                                  int n_seg, int n_intervals, int32_t *__restrict__ slot,
                                  int32_t *__restrict__ ival_slot_begin, const int32_t *__restrict__ counts,
                                  const int32_t *__restrict__ n_seg_dev, const int32_t *__restrict__ lift_form) {
  if (form_off(lift_form, BEVB200_LIFT_COLUMNS)) return;
  if (counts) {
    n_intervals = __ldg(counts + 1);
    n_seg = __ldg(n_seg_dev);
    if (n_seg == 0)   // no kept point: an empty slot table, as the host-count prepare writes it
      for (int j = blockIdx.x * blockDim.x + threadIdx.x; j <= n_intervals; j += gridDim.x * blockDim.x)
        ival_slot_begin[j] = 0;
  }
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n_seg; s += gridDim.x * blockDim.x) {
    slot[seg_sorted[s]] = s;
    const uint32_t i = ival_sorted[s];
    if (s == 0 || ival_sorted[s - 1] != i) {
      const uint32_t lo = s == 0 ? 0u : ival_sorted[s - 1] + 1u;
      for (uint32_t j = lo; j <= i; ++j) ival_slot_begin[j] = s;    // intervals without a segment cannot occur, but stay safe
    }
    if (s == n_seg - 1)
      for (uint32_t j = i + 1; j <= (uint32_t)n_intervals; ++j) ival_slot_begin[j] = n_seg;
  }
}

__global__ void lift_col_begin_kernel(const unsigned long long *__restrict__ seg_key, int n_seg, LiftGeom g,
                                      int32_t *__restrict__ col_begin, const int32_t *__restrict__ n_seg_dev,
                                      const int32_t *__restrict__ lift_form) {
  if (form_off(lift_form, BEVB200_LIFT_COLUMNS)) return;
  if (n_seg_dev) n_seg = __ldg(n_seg_dev);
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c <= g.ncols; c += gridDim.x * blockDim.x) {
    const unsigned long long want = ((unsigned long long)c * g.depth_bins) << 32;   // first key of column c
    int lo = 0, hi = n_seg;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (seg_key[mid] < want) lo = mid + 1; else hi = mid;
    }
    col_begin[c] = lo;
  }
}

// ---- per frame ---------------------------------------------------------------------------------
// kernel 1: one CTA per image column.  Shared memory: ctx column [fh][c] and depth column [D][fh].
// A group of c/4 threads evaluates one segment (one float4 of channels per thread).
template <int Q>
__global__ void __launch_bounds__(256)
    lift_columns_kernel(const float *__restrict__ depth, const float4 *__restrict__ ctx, LiftGeom g,
                        const int32_t *__restrict__ col_begin, const unsigned long long *__restrict__ seg_key,
                        const unsigned long long *__restrict__ seg_mask, const int32_t *__restrict__ slot,
                        float4 *__restrict__ partial, const int32_t *__restrict__ lift_form) {
  extern __shared__ __align__(16) uint8_t lift_smem[];
  if (form_off(lift_form, BEVB200_LIFT_COLUMNS)) return;
  float4 *ctx_s = reinterpret_cast<float4 *>(lift_smem);                    // [fh][Q]
  float *dep_s = reinterpret_cast<float *>(lift_smem + (size_t)g.fh * Q * 16);   // [D][fh]
  const int col = blockIdx.x, cam = col / g.fw, w = col % g.fw;
  const int s0 = col_begin[col], s1 = col_begin[col + 1];
  if (s0 == s1) return;
  for (int e = threadIdx.x; e < g.fh * Q; e += blockDim.x) {
    const int h = e / Q, q = e - h * Q;
    ctx_s[e] = __ldg(ctx + ((long long)(cam * g.fh + h) * g.fw + w) * Q + q);
  }
  for (int e = threadIdx.x; e < g.depth_bins * g.fh; e += blockDim.x) {
    const int d = e / g.fh, h = e - d * g.fh;
    dep_s[e] = __ldg(depth + ((long long)(cam * g.depth_bins + d) * g.fh + h) * g.fw + w);
  }
  int *full_slot = reinterpret_cast<int *>(dep_s + g.depth_bins * g.fh);   // [D]: slot of the bin's all-pixels segment
  for (int d = threadIdx.x; d < g.depth_bins; d += blockDim.x) full_slot[d] = -1;
  __syncthreads();
  const unsigned long long full_mask = g.fh >= 64 ? ~0ull : ((1ull << g.fh) - 1ull);
  for (int s = s0 + threadIdx.x; s < s1; s += blockDim.x)
    if (seg_mask[s] == full_mask) full_slot[(int)((seg_key[s] >> 32) % (unsigned long long)g.depth_bins)] = slot[s];
  __syncthreads();
  // Dense path (the common case: every pixel of the column at a depth bin falls into ONE cell): the column is a
  // [D x fh] . [fh x C] product.  A thread owns 4 depth bins x one float4 of channels and walks h once: 5 shared-
  // memory loads per 16 multiply-adds instead of 2 per 4 plus the mask arithmetic of the general path below (the
  // first version of this kernel ran every segment through that path: 121 us, issue bound).
  const int n_dt = (g.depth_bins + 3) / 4;
  for (int task = threadIdx.x; task < n_dt * Q; task += blockDim.x) {
    const int q = task % Q, d0 = (task / Q) * 4;
    int sl[4];
    bool any = false;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      sl[j] = d0 + j < g.depth_bins ? full_slot[d0 + j] : -1;
      any |= sl[j] >= 0;
    }
    if (!any) continue;
    float4 acc[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    const float *dv = dep_s + d0 * g.fh;
    const int dstep = g.fh;
    for (int h = 0; h < g.fh; ++h) {
      const float4 c4 = ctx_s[h * Q + q];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float wgt = d0 + j < g.depth_bins ? dv[j * dstep + h] : 0.f;
        // same arithmetic as lifting first: the product is rounded to fp32, then added
        acc[j].x += __fmul_rn(wgt, c4.x); acc[j].y += __fmul_rn(wgt, c4.y);
        acc[j].z += __fmul_rn(wgt, c4.z); acc[j].w += __fmul_rn(wgt, c4.w);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (sl[j] >= 0) partial[(long long)sl[j] * Q + q] = acc[j];
  }
  // General path: segments that cover only some pixels of the column (tilted cameras, the z filter, a column that
  // straddles a cell boundary)
  constexpr int kGroup = Q <= 4 ? 4 : (Q <= 8 ? 8 : (Q <= 16 ? 16 : (Q <= 32 ? 32 : 64)));   // threads per segment
  const int grp = threadIdx.x / kGroup, q = threadIdx.x % kGroup, ngrp = blockDim.x / kGroup;
  if (q >= Q) return;
  for (int s = s0 + grp; s < s1; s += ngrp) {
    unsigned long long m = seg_mask[s];
    if (m == full_mask) continue;
    const int d = (int)((seg_key[s] >> 32) % (unsigned long long)g.depth_bins);
    const float *dv = dep_s + d * g.fh;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    while (m) {
      const int h = __ffsll((long long)m) - 1;
      m &= m - 1;
      const float wgt = dv[h];
      const float4 c4 = ctx_s[h * Q + q];
      acc.x += __fmul_rn(wgt, c4.x); acc.y += __fmul_rn(wgt, c4.y); acc.z += __fmul_rn(wgt, c4.z); acc.w += __fmul_rn(wgt, c4.w);
    }
    partial[(long long)slot[s] * Q + q] = acc;
  }
}

// kernel 2: one warp per interval; lane handles float4 columns lane, lane + 32, ...
// DEV: sync-free tables (counts / lift_form); a separate instantiation keeps the host-count one as lean as before
template <int Q, bool DEV>
__global__ void __launch_bounds__(256)
    lift_cells_kernel(const float4 *__restrict__ partial, const int32_t *__restrict__ ival_slot_begin,
                      const int32_t *__restrict__ cells, int n_intervals, int zfill, int total_cells,
                      float4 *__restrict__ out, const int32_t *__restrict__ counts,
                      const int32_t *__restrict__ lift_form) {
  constexpr int QPL = (Q + 31) / 32;
  const int lane = lane_id(), warps = (gridDim.x * blockDim.x) >> 5;
  if constexpr (DEV) {
    if (form_off(lift_form, BEVB200_LIFT_COLUMNS)) return;
    n_intervals = __ldg(counts) > 0 ? __ldg(counts + 1) : 0;   // an empty grid is zeroed by zero_fill
  }
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_intervals; i += warps) {
    const int b0 = ival_slot_begin[i], b1 = ival_slot_begin[i + 1];
    const int cell = cells[i];
    float4 acc[QPL];
#pragma unroll
    for (int u = 0; u < QPL; ++u) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = b0; s < b1; ++s) {
#pragma unroll
      for (int u = 0; u < QPL; ++u) {
        const int q = lane + 32 * u;
        if (q < Q) {
          const float4 v = partial[(long long)s * Q + q];
          acc[u].x += v.x; acc[u].y += v.y; acc[u].z += v.z; acc[u].w += v.w;
        }
      }
    }
    if (cell >= 0) {
#pragma unroll
      for (int u = 0; u < QPL; ++u) {
        const int q = lane + 32 * u;
        if (q < Q) out[(long long)cell * Q + q] = acc[u];
      }
    }
    if (zfill) {   // cells ascend with the interval index: this warp also zeroes the gap below its cell
      const int prev = i > 0 ? cells[i - 1] : -1;
      const int hi = i == n_intervals - 1 ? total_cells : cell + 1;
      for (long long e = (long long)(prev + 1) * Q + lane; e < (long long)cell * Q; e += 32) out[e] = make_float4(0.f, 0.f, 0.f, 0.f);
      for (long long e = (long long)(cell + 1) * Q + lane; e < (long long)hi * Q; e += 32) out[e] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// ---- backward ------------------------------------------------------------------------------------
// With G = dL/dout and cell(p) the BEV cell of the kept frustum point p = (cam, d, h, w):
//     ddepth[cam, d, h, w] = ctx[cam, h, w, :] . G[cell(p), :]        (0 for a filtered point)
//     dctx[cam, h, w, :]   = sum over kept d of depth[cam, d, h, w] * G[cell(p), :]
// Every (d, h) of a column lies in at most one segment, so one CTA per image column writes every output element of
// the column exactly once: no memset, no float atomics, and a fixed summation order.

// cell of every segment (through its interval); -1 would mean "outside the grid" (cannot occur for prepared tables)
__global__ void lift_seg_cells_kernel(const unsigned long long *__restrict__ seg_key, int n_seg,
                                      const int32_t *__restrict__ geom_feats, const int32_t *__restrict__ starts, int n,
                                      PoolDims dm, int32_t *__restrict__ seg_cell, const int32_t *__restrict__ counts,
                                      const int32_t *__restrict__ n_seg_dev, const int32_t *__restrict__ lift_form) {
  if (form_off(lift_form, BEVB200_LIFT_COLUMNS)) return;
  if (counts) {
    n = __ldg(counts);
    n_seg = __ldg(n_seg_dev);
  }
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n_seg; s += gridDim.x * blockDim.x)
    seg_cell[s] = interval_cell(geom_feats, starts[(uint32_t)(seg_key[s] & 0xffffffffull)], n, dm);
}

// Shared memory of the column backward: fixed part + per staged segment.  Rows of ctx_s and g_s are padded to Q + 1
// float4 so that the threads of a warp, which walk h (ctx_s) or the segment (g_s), hit distinct banks.
struct LiftBwdSmem {
  size_t fixed, per_seg;
};
static LiftBwdSmem lift_bwd_smem(int q, int fh, int depth_bins) {
  LiftBwdSmem s;
  s.fixed = (size_t)fh * (q + 1) * 16 + (size_t)fh * q * 16 + (size_t)depth_bins * 8;   // ctx_s, acc_s, cov_s
  s.per_seg = (size_t)(q + 1) * 16 + (size_t)fh * 4 + 8 + 4;                             // g_s, dep_s, mask_s, d_s
  return s;
}

// One CTA per image column.  The column's segments are processed in chunks of at most `smax` (the G rows of a
// column need not fit in shared memory: C = 256, many depth bins, or up to D * fh segments of jittered geometry).
// Per chunk: stage the segments' G rows and their depth values; ddepth of every (segment, h in mask) is a C-long dot
// product written straight to global memory; dctx accumulates in shared memory, one (h, float4) per task, over the
// segments in order.  At the end the (d, h) no segment covers get ddepth = 0 and dctx is written once.
template <int Q>
__global__ void __launch_bounds__(256)
    lift_columns_bwd_kernel(const float4 *__restrict__ out_grad, const float *__restrict__ depth,
                            const float4 *__restrict__ ctx, LiftGeom g, const int32_t *__restrict__ col_begin,
                            const unsigned long long *__restrict__ seg_key,
                            const unsigned long long *__restrict__ seg_mask, const int32_t *__restrict__ seg_cell,
                            int smax, float *__restrict__ ddepth, float4 *__restrict__ dctx,
                            const int32_t *__restrict__ lift_form) {
  constexpr int QP = Q + 1;
  extern __shared__ __align__(16) uint8_t lift_bwd_smem_raw[];
  if (form_off(lift_form, BEVB200_LIFT_COLUMNS)) return;
  float4 *ctx_s = reinterpret_cast<float4 *>(lift_bwd_smem_raw);                  // [fh][QP]
  float4 *acc_s = ctx_s + g.fh * QP;                                               // [fh][Q]
  float4 *g_s = acc_s + g.fh * Q;                                                  // [smax][QP]
  unsigned long long *cov_s = reinterpret_cast<unsigned long long *>(g_s + smax * QP);   // [D]
  unsigned long long *mask_s = cov_s + g.depth_bins;                               // [smax]
  float *dep_s = reinterpret_cast<float *>(mask_s + smax);                         // [smax][fh]
  int *d_s = reinterpret_cast<int *>(dep_s + smax * g.fh);                         // [smax]
  const int col = blockIdx.x, cam = col / g.fw, w = col % g.fw;
  const int s0 = col_begin[col], s1 = col_begin[col + 1];
  const bool want_dd = ddepth != nullptr, want_dc = dctx != nullptr;
  const long long dstride = g.fw;                                                  // ddepth / depth: h -> h + 1
  const long long dbase = (long long)cam * g.depth_bins * g.fh * g.fw + w;        // (cam, d = 0, h = 0, w)
  if (want_dd) {
    for (int e = threadIdx.x; e < g.fh * Q; e += blockDim.x) {
      const int h = e / Q, q = e - h * Q;
      ctx_s[h * QP + q] = __ldg(ctx + ((long long)(cam * g.fh + h) * g.fw + w) * Q + q);
    }
    for (int d = threadIdx.x; d < g.depth_bins; d += blockDim.x) cov_s[d] = 0ull;
  }
  if (want_dc)
    for (int e = threadIdx.x; e < g.fh * Q; e += blockDim.x) acc_s[e] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  for (int sa = s0; sa < s1; sa += smax) {
    const int n = min(smax, s1 - sa);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const unsigned long long m = seg_mask[sa + i];
      const int d = (int)((seg_key[sa + i] >> 32) % (unsigned long long)g.depth_bins);
      mask_s[i] = m;
      d_s[i] = d;
      if (want_dd) atomicOr(&cov_s[d], m);   // integer OR: order-independent
    }
    for (int e = threadIdx.x; e < n * Q; e += blockDim.x) {
      const int i = e / Q, q = e - i * Q;
      const int cell = seg_cell[sa + i];
      g_s[i * QP + q] = cell >= 0 ? __ldg(out_grad + (long long)cell * Q + q) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    if (want_dc)
      for (int e = threadIdx.x; e < n * g.fh; e += blockDim.x) {
        const int i = e / g.fh, h = e - i * g.fh;
        dep_s[e] = (mask_s[i] >> h) & 1ull ? __ldg(depth + dbase + ((long long)d_s[i] * g.fh + h) * dstride) : 0.f;
      }
    if (want_dd)
      for (int e = threadIdx.x; e < n * g.fh; e += blockDim.x) {
        const int i = e / g.fh, h = e - i * g.fh;
        if (!((mask_s[i] >> h) & 1ull)) continue;
        const float4 *cr = ctx_s + h * QP, *gr = g_s + i * QP;
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
        for (int q = 0; q < Q; ++q) {
          const float4 c4 = cr[q], g4 = gr[q];
          a.x = fmaf(c4.x, g4.x, a.x); a.y = fmaf(c4.y, g4.y, a.y);
          a.z = fmaf(c4.z, g4.z, a.z); a.w = fmaf(c4.w, g4.w, a.w);
        }
        ddepth[dbase + ((long long)d_s[i] * g.fh + h) * dstride] = (a.x + a.y) + (a.z + a.w);
      }
    __syncthreads();   // dep_s complete
    if (want_dc)
      for (int e = threadIdx.x; e < g.fh * Q; e += blockDim.x) {
        const int h = e / Q, q = e - h * Q;
        float4 a = acc_s[e];
        for (int i = 0; i < n; ++i) {   // segments in order: fixed summation order
          const float wgt = dep_s[i * g.fh + h];
          const float4 g4 = g_s[i * QP + q];
          a.x = fmaf(wgt, g4.x, a.x); a.y = fmaf(wgt, g4.y, a.y);
          a.z = fmaf(wgt, g4.z, a.z); a.w = fmaf(wgt, g4.w, a.w);
        }
        acc_s[e] = a;
      }
    __syncthreads();   // g_s / dep_s / mask_s are overwritten by the next chunk
  }
  if (want_dd)
    for (int e = threadIdx.x; e < g.depth_bins * g.fh; e += blockDim.x) {
      const int d = e / g.fh, h = e - d * g.fh;
      if (!((cov_s[d] >> h) & 1ull)) ddepth[dbase + ((long long)d * g.fh + h) * dstride] = 0.f;
    }
  if (want_dc)
    for (int e = threadIdx.x; e < g.fh * Q; e += blockDim.x) {
      const int h = e / Q, q = e - h * Q;
      dctx[((long long)(cam * g.fh + h) * g.fw + w) * Q + q] = acc_s[e];
    }
}

// Pixel backward (any feature height: the form of the row forward).  First the cell of every frustum point in
// ORIGINAL order (-1 for the filtered ones, which perm lists after the kept ones) ...
__global__ void lift_point_cells_kernel(const int32_t *__restrict__ perm, const int32_t *__restrict__ geom_feats,
                                        const int32_t *__restrict__ starts, const int32_t *__restrict__ lengths,
                                        int n, int n_total, int n_intervals, PoolDims dm,
                                        int32_t *__restrict__ point_cell, const int32_t *__restrict__ counts,
                                        const int32_t *__restrict__ lift_form) {
  const int lane = lane_id(), warps = (gridDim.x * blockDim.x) >> 5;
  if (form_off(lift_form, BEVB200_LIFT_ROWS)) return;
  device_counts(counts, n, n_intervals);
  if (n_intervals == 0) n = 0;   // no interval pools anything: every point is filtered (no cell left unset)
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_intervals; i += warps) {   // warp per interval
    const int s0 = starts[i], len = lengths[i];
    const int32_t c = interval_cell(geom_feats, s0, n, dm);
    for (int s = s0 + lane; s < s0 + len && s < n; s += 32) point_cell[perm[s]] = c;
  }
  for (int s = n + blockIdx.x * blockDim.x + threadIdx.x; s < n_total; s += gridDim.x * blockDim.x)
    point_cell[perm[s]] = -1;
}

// ... then one warp per pixel walks the depth bins in ascending order: ddepth is a warp-reduced dot of the pixel's
// context row (held in registers) with the cell's G row, dctx accumulates in registers.
template <int Q>
__global__ void __launch_bounds__(256)
    lift_pixels_bwd_kernel(const float4 *__restrict__ out_grad, const float *__restrict__ depth,
                           const float4 *__restrict__ ctx, const int32_t *__restrict__ point_cell, int n_pixels,
                           int depth_bins, int ppc, float *__restrict__ ddepth, float4 *__restrict__ dctx,
                           const int32_t *__restrict__ lift_form) {
  constexpr int QPL = (Q + 31) / 32;
  const int lane = lane_id(), warps = (gridDim.x * blockDim.x) >> 5;
  if (form_off(lift_form, BEVB200_LIFT_ROWS)) return;
  const bool want_dd = ddepth != nullptr, want_dc = dctx != nullptr;
  for (int px = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; px < n_pixels; px += warps) {
    const int cam = px / ppc, pix = px - cam * ppc;
    float4 cr[QPL], acc[QPL];
#pragma unroll
    for (int u = 0; u < QPL; ++u) {
      const int q = lane + 32 * u;
      cr[u] = want_dd && q < Q ? __ldg(ctx + (long long)px * Q + q) : make_float4(0.f, 0.f, 0.f, 0.f);
      acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int d = 0; d < depth_bins; ++d) {
      const long long p = ((long long)cam * depth_bins + d) * ppc + pix;
      const int cell = point_cell[p];
      if (cell < 0) {
        if (want_dd && lane == 0) ddepth[p] = 0.f;
        continue;
      }
      float4 g4[QPL];
#pragma unroll
      for (int u = 0; u < QPL; ++u) {
        const int q = lane + 32 * u;
        g4[u] = q < Q ? __ldg(out_grad + (long long)cell * Q + q) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      if (want_dd) {
        float a = 0.f;
#pragma unroll
        for (int u = 0; u < QPL; ++u)
          a += (cr[u].x * g4[u].x + cr[u].y * g4[u].y) + (cr[u].z * g4[u].z + cr[u].w * g4[u].w);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) ddepth[p] = a;
      }
      if (want_dc) {
        const float wgt = __ldg(depth + p);
#pragma unroll
        for (int u = 0; u < QPL; ++u) {
          acc[u].x = fmaf(wgt, g4[u].x, acc[u].x); acc[u].y = fmaf(wgt, g4[u].y, acc[u].y);
          acc[u].z = fmaf(wgt, g4[u].z, acc[u].z); acc[u].w = fmaf(wgt, g4[u].w, acc[u].w);
        }
      }
    }
    if (want_dc)
#pragma unroll
      for (int u = 0; u < QPL; ++u) {
        const int q = lane + 32 * u;
        if (q < Q) dctx[(long long)px * Q + q] = acc[u];
      }
  }
}

struct LiftWs {
  int32_t *ival_of;
  unsigned long long *keys_a, *keys_b;
  uint32_t *vals_a, *vals_b, *flags, *pos, *tiles, *total;
  uint32_t *ival_a, *ival_b, *idx_a, *idx_b;
  char *cub_tmp;
  size_t cub_bytes;
};

static size_t lift_prepare_layout(int n, void *ws, size_t ws_bytes, LiftWs *out) {
  Arena a(ws, ws_bytes);
  LiftWs w;
  const size_t m = n > 0 ? n : 1;
  w.ival_of = a.take<int32_t>(m);
  w.keys_a = a.take<unsigned long long>(m);
  w.keys_b = a.take<unsigned long long>(m);
  w.vals_a = a.take<uint32_t>(m);
  w.vals_b = a.take<uint32_t>(m);
  w.flags = a.take<uint32_t>(m);
  w.pos = a.take<uint32_t>(m);
  w.tiles = a.take<uint32_t>(scan_scratch_elems(m));
  w.total = a.take<uint32_t>(64);
  w.ival_a = a.take<uint32_t>(m);
  w.ival_b = a.take<uint32_t>(m);
  w.idx_a = a.take<uint32_t>(m);
  w.idx_b = a.take<uint32_t>(m);
  size_t c1 = 0, c2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, c1, (const unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                  (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)m, 0, 64, (cudaStream_t)0);
  cub::DeviceRadixSort::SortPairs(nullptr, c2, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const uint32_t *)nullptr,
                                  (uint32_t *)nullptr, (int)m, 0, 32, (cudaStream_t)0);
  w.cub_bytes = c1 > c2 ? c1 : c2;
  w.cub_tmp = a.take<char>(w.cub_bytes);
  if (out) *out = w;
  return a.off;
}

// Workspace of the column forward: one partial row per segment, then the cell of every interval
struct LiftColumnsWs {
  float *partial;
  int32_t *cells;
};
static size_t lift_columns_layout(int n_segments, int n_intervals, int c, void *ws, LiftColumnsWs *out) {
  Arena a(ws, 0);
  LiftColumnsWs w;
  w.partial = a.take<float>((size_t)n_segments * c);
  w.cells = a.take<int32_t>((size_t)n_intervals);
  if (out) *out = w;
  return a.off;
}

// Workspace of both lift backwards: the cell of every segment (column form) or of every frustum point (pixel form),
// room for at least one
static size_t lift_bwd_layout(int items, void *ws, int32_t **cells) {
  Arena a(ws, 0);
  int32_t *p = a.take<int32_t>(items > 0 ? items : 1);
  if (cells) *cells = p;
  return a.off;
}

// the workspace queries of the column forward and both backwards report this much more than the calls require
constexpr size_t kLiftQuerySlack = 256;

// ---- host side ---------------------------------------------------------------------------------------------------
// Each host-count entry and its *_dev twin share one body.  A twin passes `counts` = {n_kept, n_intervals} in device
// memory (the host n_kept / n / n_intervals are then the capacity the tables were sized for), the device segment count
// `n_seg_dev` and the status word `lift_form`; the host sizes every grid from the capacities and the kernels stop at the
// device counts.  Every check comes before the first launch.

static int lift_prepare(const int32_t *perm, const int32_t *interval_starts, int n_kept, int n_intervals, int cameras,
                        int depth_bins, int feature_h, int feature_w, int32_t *col_begin, uint64_t *seg_key,
                        uint64_t *seg_mask, int32_t *seg_slot, int32_t *interval_slot_begin, int32_t *n_segments,
                        void *workspace, size_t workspace_bytes, cudaStream_t st, const int32_t *counts,
                        int max_segments, int32_t *lift_form) {
  const bool dev = counts != nullptr;
  BEVB200_REQUIRE(n_kept >= 0 && n_intervals >= 0 && cameras > 0 && depth_bins > 0 && feature_h > 0 && feature_w > 0,
                  "bad sizes");
  BEVB200_REQUIRE(feature_h <= 64, "feature height > 64: the per-segment pixel mask is 64 bits");
  BEVB200_REQUIRE((long long)cameras * feature_w * depth_bins < (1ll << 31), "too many (column, depth) pairs");
  BEVB200_REQUIRE(col_begin && seg_key && seg_mask && seg_slot && interval_slot_begin && n_segments, "null output");
  if (dev) {
    BEVB200_REQUIRE(n_kept > 0, "capacity must be positive");
    BEVB200_REQUIRE(max_segments > 0 && max_segments <= n_kept, "max_segments must lie in [1, capacity]");
    BEVB200_REQUIRE(lift_form != nullptr, "null lift_form");
  }
  LiftGeom g{depth_bins, feature_h, feature_w, cameras * feature_w};
  if (!dev && (n_kept == 0 || n_intervals == 0)) {
    BEVB200_CUDA(cudaMemsetAsync(n_segments, 0, sizeof(int32_t), st));
    BEVB200_CUDA(cudaMemsetAsync(col_begin, 0, (size_t)(g.ncols + 1) * sizeof(int32_t), st));
    BEVB200_CUDA(cudaMemsetAsync(interval_slot_begin, 0, (size_t)(n_intervals + 1) * sizeof(int32_t), st));
    return BEVB200_OK;
  }
  BEVB200_REQUIRE(perm && interval_starts, "null input");
  LiftWs w;
  if (const int rc = workspace_check("bev_pool_lift_prepare", workspace, workspace_bytes,
                                     lift_prepare_layout(n_kept, workspace, workspace_bytes, &w)))
    return rc;
  BEVB200_LAUNCH(lift_interval_ids_kernel, grid_for(n_intervals, 128), 128, 0, st, interval_starts, n_intervals, n_kept,
                 w.ival_of, counts);
  BEVB200_LAUNCH(lift_keys_kernel, grid_for(n_kept, 256), 256, 0, st, perm, w.ival_of, n_kept, g, w.keys_a, w.vals_a,
                 counts, n_kept);
  // cub takes a host item count: the sync-free prepare sorts all n_kept (capacity) keys, the rows past the device
  // n_kept carrying the key (ncols * D) << 32, which the bit range must then hold.  A stable sort over more bits gives
  // the same order.
  const long long n_cd = (long long)g.ncols * depth_bins;
  int cd_bits = 1;
  while ((1ll << cd_bits) < n_cd + (dev ? 1 : 0)) ++cd_bits;
  size_t cub_bytes = w.cub_bytes;
  BEVB200_CUDA(cub::DeviceRadixSort::SortPairs(w.cub_tmp, cub_bytes, (const unsigned long long *)w.keys_a, w.keys_b,
                                               (const uint32_t *)w.vals_a, w.vals_b, n_kept, 0, 32 + cd_bits, st));
  g_launch_count += (32 + cd_bits + 7) / 8 + 2;
  BEVB200_LAUNCH(lift_heads_kernel, grid_for(n_kept, 256), 256, 0, st, w.keys_b, n_kept, w.flags, counts);
  int rc = exclusive_scan_u32(w.flags, w.pos, n_kept, w.tiles, w.total, false, st);
  if (rc) return rc;
  // the segment records: all of them (host count), or the first max_segments (sync-free)
  const uint32_t seg_cap = dev ? (uint32_t)max_segments : 0xffffffffu;
  if (dev) {
    BEVB200_LAUNCH(lift_form_kernel, 1, 1, 0, st, w.total, max_segments, n_segments, lift_form);
  } else {
    BEVB200_CUDA(cudaMemcpyAsync(n_segments, w.total, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  }
  BEVB200_LAUNCH(lift_segments_kernel, grid_for(n_kept, 256), 256, 0, st, w.keys_b, w.vals_b, w.flags, w.pos, n_kept,
                 (unsigned long long *)seg_key, (unsigned long long *)seg_mask, counts, seg_cap);
  // The slot pass sorts the segments by interval.  The host-count prepare reads the segment count back once (this is
  // a per-calibration call) and sorts exactly that many; the sync-free one sorts max_segments entries, those past the
  // device count keyed after every interval, and its slot and column passes do nothing when the count is over the cap.
  int n_items;
  if (dev) {
    n_items = max_segments;
  } else {
    int32_t n_seg = 0;
    BEVB200_CUDA(cudaMemcpyAsync(&n_seg, w.total, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    BEVB200_CUDA(cudaStreamSynchronize(st));
    n_items = n_seg;
  }
  const int32_t *n_seg_dev = dev ? n_segments : nullptr;
  BEVB200_LAUNCH(lift_seg_ival_kernel, grid_for(n_items, 256), 256, 0, st, (const unsigned long long *)seg_key, n_items,
                 w.ival_a, w.idx_a, n_seg_dev, (uint32_t)n_kept);
  // interval ids are below n_intervals; the sync-free key past the count is n_kept (capacity) and must fit as well
  const long long iv_bound = dev ? (long long)n_kept + 1 : (long long)n_intervals;
  int iv_bits = 1;
  while ((1ll << iv_bits) < iv_bound) ++iv_bits;
  cub_bytes = w.cub_bytes;
  BEVB200_CUDA(cub::DeviceRadixSort::SortPairs(w.cub_tmp, cub_bytes, (const uint32_t *)w.ival_a, w.ival_b,
                                               (const uint32_t *)w.idx_a, w.idx_b, n_items, 0, iv_bits, st));
  g_launch_count += (iv_bits + 7) / 8 + 2;
  BEVB200_LAUNCH(lift_slots_kernel, grid_for(n_items, 256), 256, 0, st, w.ival_b, w.idx_b, n_items, n_intervals,
                 seg_slot, interval_slot_begin, counts, n_seg_dev, lift_form);
  BEVB200_LAUNCH(lift_col_begin_kernel, grid_for(g.ncols + 1, 256), 256, 0, st, (const unsigned long long *)seg_key,
                 n_items, g, col_begin, n_seg_dev, lift_form);
  return BEVB200_OK;
}

static int lift_columns(int b, int d, int h, int w, int n, int c, int n_intervals, const float *depth, const float *ctx,
                        int cameras, int depth_bins, int feature_h, int feature_w, const int32_t *geom_feats,
                        const int32_t *interval_starts, const int32_t *col_begin, const uint64_t *seg_key,
                        const uint64_t *seg_mask, const int32_t *seg_slot, const int32_t *interval_slot_begin,
                        int n_segments, float *out, void *workspace, size_t workspace_bytes, cudaStream_t st,
                        const int32_t *counts, const int32_t *lift_form) {
  BEVB200_REQUIRE(b > 0 && d > 0 && h > 0 && w > 0 && c > 0 && n >= 0 && n_intervals >= 0 && n_segments >= 0, "bad sizes");
  BEVB200_REQUIRE(out != nullptr, "null out");
  BEVB200_REQUIRE(c % 4 == 0 && c <= 256, "channel count must be a multiple of 4, <= 256");
  BEVB200_REQUIRE((long long)b * d * h * w < (1ll << 31), "grid has too many cells");
  // with no segment the cells kernel does not run, so nothing would zero-fill the grid
  const bool work = n > 0 && n_intervals > 0 && n_segments > 0;
  const size_t smem = (size_t)feature_h * c * sizeof(float) + (size_t)depth_bins * feature_h * sizeof(float) +
                      (size_t)depth_bins * sizeof(int);
  // every argument is checked before `out` is written: a refused call leaves it untouched
  LiftColumnsWs ws;
  if (work) {
    BEVB200_REQUIRE(depth && ctx && geom_feats && interval_starts && col_begin && seg_key && seg_mask && seg_slot &&
                        interval_slot_begin, "null input");
    BEVB200_REQUIRE(((uintptr_t)ctx % 16 == 0) && ((uintptr_t)out % 16 == 0), "ctx / out must be 16-byte aligned");
    if (const int rc = workspace_check("bev_pool_lift_columns", workspace, workspace_bytes,
                                       lift_columns_layout(n_segments, n_intervals, c, workspace, &ws)))
      return rc;
    BEVB200_REQUIRE(smem <= 200 * 1024, "image column does not fit in shared memory");
    BEVB200_REQUIRE(TunedWidths::has(c), "no tuned kernel for this channel count");
  }
  const int zfill = (b * d == 1 && work) ? 1 : 0;
  // with zfill the cells kernel zeroes the empty cells; a grid with no kept point (known on the device only) is
  // zeroed by zero_fill, which then does nothing unless the tables are empty
  if (!zfill || counts)
    if (const int rc = zero_fill(out, (size_t)b * d * h * w * c, lift_form, BEVB200_LIFT_COLUMNS, st,
                                 zfill ? counts : nullptr))
      return rc;
  if (!work) return BEVB200_OK;
  PoolDims dm{b, d, h, w};
  LiftGeom g{depth_bins, feature_h, feature_w, cameras * feature_w};
  BEVB200_LAUNCH(pool_interval_cells_kernel, grid_for(n_intervals, 256), 256, 0, st, geom_feats, interval_starts, n,
                 n_intervals, dm, ws.cells, counts);
  const int total_cells = b * d * h * w;
  return TunedWidths::dispatch(c, [&](auto q) {
    constexpr int Q = decltype(q)::value;
    BEVB200_CUDA(cudaFuncSetAttribute(lift_columns_kernel<Q>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    BEVB200_LAUNCH(lift_columns_kernel<Q>, g.ncols, 256, smem, st, depth, (const float4 *)ctx, g, col_begin,
                   (const unsigned long long *)seg_key, (const unsigned long long *)seg_mask, seg_slot,
                   (float4 *)ws.partial, lift_form);
    const auto cells = counts ? &lift_cells_kernel<Q, true> : &lift_cells_kernel<Q, false>;
    BEVB200_LAUNCH(cells, grid_for((long long)n_intervals * 32, 256, kNumSMs * 8), 256, 0, st,
                   (const float4 *)ws.partial, interval_slot_begin, ws.cells, n_intervals, zfill, total_cells,
                   (float4 *)out, counts, lift_form);
    return BEVB200_OK;
  });
}

static int lift_columns_backward(int b, int d, int h, int w, int n, int c, int n_intervals, const float *out_grad,
                                 const float *depth, const float *ctx, int cameras, int depth_bins, int feature_h,
                                 int feature_w, const int32_t *geom_feats, const int32_t *interval_starts,
                                 const int32_t *col_begin, const uint64_t *seg_key, const uint64_t *seg_mask,
                                 int n_segments, float *ddepth, float *dctx, void *workspace, size_t workspace_bytes,
                                 cudaStream_t st, const int32_t *counts, const int32_t *n_seg_dev,
                                 const int32_t *lift_form) {
  BEVB200_REQUIRE(b > 0 && d > 0 && h > 0 && w > 0 && n >= 0 && n_intervals >= 0 && n_segments >= 0, "bad sizes");
  BEVB200_REQUIRE(cameras > 0 && depth_bins > 0 && feature_h > 0 && feature_w > 0, "bad lift dims");
  BEVB200_REQUIRE(feature_h <= 64, "feature height > 64: use bevb200_bev_pool_lift_backward");
  BEVB200_REQUIRE(TunedWidths::has(c), "no tuned kernel for this channel count");
  BEVB200_REQUIRE((long long)b * d * h * w < (1ll << 31), "grid has too many cells");
  BEVB200_REQUIRE((long long)cameras * feature_w * depth_bins < (1ll << 31), "too many (column, depth) pairs");
  if (ddepth == nullptr && dctx == nullptr) return BEVB200_OK;
  BEVB200_REQUIRE(out_grad && col_begin && seg_key && seg_mask, "null input");
  // the interval tables are read through the segments only: with no kept point (empty tables) they may be NULL
  BEVB200_REQUIRE(n_segments == 0 || (geom_feats && interval_starts), "null interval tables");
  BEVB200_REQUIRE(ctx || !ddepth, "ddepth needs ctx");
  BEVB200_REQUIRE(depth || !dctx, "dctx needs depth");
  BEVB200_REQUIRE(((uintptr_t)ctx % 16 == 0) && ((uintptr_t)dctx % 16 == 0) && ((uintptr_t)out_grad % 16 == 0),
                  "ctx / dctx / out_grad must be 16-byte aligned");
  int32_t *seg_cell;
  if (const int rc = workspace_check("bev_pool_lift_columns_backward", workspace, workspace_bytes,
                                     lift_bwd_layout(n_segments, workspace, &seg_cell)))
    return rc;
  const int q = c / 4;
  const LiftBwdSmem sm = lift_bwd_smem(q, feature_h, depth_bins);
  // chunk size: all of a column's segments at once when that stays within ~100 KB (two CTAs per SM), else as many
  // as the 227 KB of one CTA allow
  constexpr size_t kTwoPerSM = 100 * 1024, kMaxSmem = 220 * 1024;
  long long smax = sm.fixed < kTwoPerSM ? (long long)((kTwoPerSM - sm.fixed) / sm.per_seg) : 0;
  if (smax < 32 && sm.fixed < kMaxSmem) smax = (long long)((kMaxSmem - sm.fixed) / sm.per_seg);
  if (smax > 256) smax = 256;
  BEVB200_REQUIRE(smax >= 1, "image column does not fit in shared memory");
  const size_t smem = sm.fixed + (size_t)smax * sm.per_seg;
  LiftGeom g{depth_bins, feature_h, feature_w, cameras * feature_w};
  if (n_segments > 0) {
    PoolDims dm{b, d, h, w};
    BEVB200_LAUNCH(lift_seg_cells_kernel, grid_for(n_segments, 256), 256, 0, st, (const unsigned long long *)seg_key,
                   n_segments, geom_feats, interval_starts, n, dm, seg_cell, counts, n_seg_dev, lift_form);
  }
  return TunedWidths::dispatch(c, [&](auto q) {
    constexpr int Q = decltype(q)::value;
    BEVB200_CUDA(cudaFuncSetAttribute(lift_columns_bwd_kernel<Q>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    BEVB200_LAUNCH(lift_columns_bwd_kernel<Q>, g.ncols, 256, smem, st, (const float4 *)out_grad, depth,
                   (const float4 *)ctx, g, col_begin, (const unsigned long long *)seg_key,
                   (const unsigned long long *)seg_mask, seg_cell, (int)smax, ddepth, (float4 *)dctx, lift_form);
    return BEVB200_OK;
  });
}

static int lift_rows_backward(int b, int d, int h, int w, int n, int n_total, int c, int n_intervals,
                              const float *out_grad, const float *depth, const float *ctx, int depth_bins,
                              int pixels_per_camera, const int32_t *perm, const int32_t *geom_feats,
                              const int32_t *interval_starts, const int32_t *interval_lengths, float *ddepth,
                              float *dctx, void *workspace, size_t workspace_bytes, cudaStream_t st,
                              const int32_t *counts, const int32_t *lift_form) {
  BEVB200_REQUIRE(b > 0 && d > 0 && h > 0 && w > 0 && n >= 0 && n_total >= n && n_intervals >= 0, "bad sizes");
  BEVB200_REQUIRE(depth_bins > 0 && pixels_per_camera > 0 && n_total % ((long long)depth_bins * pixels_per_camera) == 0,
                  "bad lift dims");
  BEVB200_REQUIRE(TunedWidths::has(c), "no tuned kernel for this channel count");
  BEVB200_REQUIRE((long long)b * d * h * w < (1ll << 31), "grid has too many cells");
  if (ddepth == nullptr && dctx == nullptr) return BEVB200_OK;
  BEVB200_REQUIRE(out_grad && perm && geom_feats && interval_starts && interval_lengths, "null input");
  BEVB200_REQUIRE(ctx || !ddepth, "ddepth needs ctx");
  BEVB200_REQUIRE(depth || !dctx, "dctx needs depth");
  BEVB200_REQUIRE(((uintptr_t)ctx % 16 == 0) && ((uintptr_t)dctx % 16 == 0) && ((uintptr_t)out_grad % 16 == 0),
                  "ctx / dctx / out_grad must be 16-byte aligned");
  int32_t *point_cell;
  if (const int rc = workspace_check("bev_pool_lift_backward", workspace, workspace_bytes,
                                     lift_bwd_layout(n_total, workspace, &point_cell)))
    return rc;
  if (n_total == 0) return BEVB200_OK;
  PoolDims dm{b, d, h, w};
  BEVB200_LAUNCH(lift_point_cells_kernel, grid_for((long long)n_total, 256), 256, 0, st, perm, geom_feats,
                 interval_starts, interval_lengths, n, n_total, n_intervals, dm, point_cell, counts, lift_form);
  const int n_pixels = (int)(n_total / depth_bins);
  const int grid = grid_for((long long)n_pixels * 32, 256, kNumSMs * 16);
  return TunedWidths::dispatch(c, [&](auto q) {
    BEVB200_LAUNCH(lift_pixels_bwd_kernel<decltype(q)::value>, grid, 256, 0, st, (const float4 *)out_grad, depth,
                   (const float4 *)ctx, point_cell, n_pixels, depth_bins, pixels_per_camera, ddepth, (float4 *)dctx,
                   lift_form);
    return BEVB200_OK;
  });
}

}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_bev_pool_lift_prepare_workspace_bytes(int n_kept) {
  if (n_kept < 0) return 0;
  return lift_prepare_layout(n_kept, nullptr, 0, nullptr);
}

int bevb200_bev_pool_lift_prepare(const int32_t *perm, const int32_t *interval_starts, int n_kept, int n_intervals,
                                  int cameras, int depth_bins, int feature_h, int feature_w, int32_t *col_begin,
                                  uint64_t *seg_key, uint64_t *seg_mask, int32_t *seg_slot, int32_t *interval_slot_begin,
                                  int32_t *n_segments, void *workspace, size_t workspace_bytes, void *stream) {
  return lift_prepare(perm, interval_starts, n_kept, n_intervals, cameras, depth_bins, feature_h, feature_w, col_begin,
                      seg_key, seg_mask, seg_slot, interval_slot_begin, n_segments, workspace, workspace_bytes,
                      (cudaStream_t)stream, nullptr, 0, nullptr);
}

int bevb200_bev_pool_lift_columns(int b, int d, int h, int w, int n, int c, int n_intervals, const float *depth,
                                  const float *ctx, int cameras, int depth_bins, int feature_h, int feature_w,
                                  const int32_t *geom_feats, const int32_t *interval_starts, const int32_t *col_begin,
                                  const uint64_t *seg_key, const uint64_t *seg_mask, const int32_t *seg_slot,
                                  const int32_t *interval_slot_begin, int n_segments, float *out, void *workspace,
                                  size_t workspace_bytes, void *stream) {
  return lift_columns(b, d, h, w, n, c, n_intervals, depth, ctx, cameras, depth_bins, feature_h, feature_w, geom_feats,
                      interval_starts, col_begin, seg_key, seg_mask, seg_slot, interval_slot_begin, n_segments, out,
                      workspace, workspace_bytes, (cudaStream_t)stream, nullptr, nullptr);
}

size_t bevb200_bev_pool_lift_columns_workspace_bytes(int n_segments, int n_intervals, int c) {
  if (n_segments < 0 || n_intervals < 0 || c <= 0) return 0;
  return lift_columns_layout(n_segments, n_intervals, c, nullptr, nullptr) + kLiftQuerySlack;
}

size_t bevb200_bev_pool_lift_columns_backward_workspace_bytes(int n_segments, int n_intervals, int c) {
  if (n_segments < 0 || n_intervals < 0 || !TunedWidths::has(c)) return 0;
  return lift_bwd_layout(n_segments, nullptr, nullptr) + kLiftQuerySlack;
}

int bevb200_bev_pool_lift_columns_backward(int b, int d, int h, int w, int n, int c, int n_intervals,
                                           const float *out_grad, const float *depth, const float *ctx, int cameras,
                                           int depth_bins, int feature_h, int feature_w, const int32_t *geom_feats,
                                           const int32_t *interval_starts, const int32_t *col_begin,
                                           const uint64_t *seg_key, const uint64_t *seg_mask, int n_segments,
                                           float *ddepth, float *dctx, void *workspace, size_t workspace_bytes,
                                           void *stream) {
  return lift_columns_backward(b, d, h, w, n, c, n_intervals, out_grad, depth, ctx, cameras, depth_bins, feature_h,
                               feature_w, geom_feats, interval_starts, col_begin, seg_key, seg_mask, n_segments, ddepth,
                               dctx, workspace, workspace_bytes, (cudaStream_t)stream, nullptr, nullptr, nullptr);
}

size_t bevb200_bev_pool_lift_backward_workspace_bytes(int n_total, int c) {
  if (n_total < 0 || !TunedWidths::has(c)) return 0;
  return lift_bwd_layout(n_total, nullptr, nullptr) + kLiftQuerySlack;
}

int bevb200_bev_pool_lift_backward(int b, int d, int h, int w, int n, int n_total, int c, int n_intervals,
                                   const float *out_grad, const float *depth, const float *ctx, int depth_bins,
                                   int pixels_per_camera, const int32_t *perm, const int32_t *geom_feats,
                                   const int32_t *interval_starts, const int32_t *interval_lengths, float *ddepth,
                                   float *dctx, void *workspace, size_t workspace_bytes, void *stream) {
  return lift_rows_backward(b, d, h, w, n, n_total, c, n_intervals, out_grad, depth, ctx, depth_bins,
                            pixels_per_camera, perm, geom_feats, interval_starts, interval_lengths, ddepth, dctx,
                            workspace, workspace_bytes, (cudaStream_t)stream, nullptr, nullptr);
}

// ---- sync-free twins ------------------------------------------------------------------------------------------------

size_t bevb200_bev_pool_lift_prepare_dev_workspace_bytes(int n_capacity, int max_segments) {
  if (n_capacity <= 0 || max_segments <= 0 || max_segments > n_capacity) return 0;
  return lift_prepare_layout(n_capacity, nullptr, 0, nullptr);
}

int bevb200_bev_pool_lift_prepare_dev(const int32_t *perm, const int32_t *interval_starts, const int32_t *counts_dev,
                                      int n_capacity, int max_segments, int cameras, int depth_bins, int feature_h,
                                      int feature_w, int32_t *col_begin, uint64_t *seg_key, uint64_t *seg_mask,
                                      int32_t *seg_slot, int32_t *interval_slot_begin, int32_t *n_segments,
                                      int32_t *lift_form, void *workspace, size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(counts_dev != nullptr, "null counts");
  return lift_prepare(perm, interval_starts, n_capacity, n_capacity, cameras, depth_bins, feature_h, feature_w,
                      col_begin, seg_key, seg_mask, seg_slot, interval_slot_begin, n_segments, workspace,
                      workspace_bytes, (cudaStream_t)stream, counts_dev, max_segments, lift_form);
}

size_t bevb200_bev_pool_lift_columns_dev_workspace_bytes(int max_segments, int n_capacity, int c) {
  if (max_segments <= 0 || n_capacity <= 0 || c <= 0) return 0;
  return lift_columns_layout(max_segments, n_capacity, c, nullptr, nullptr) + kLiftQuerySlack;
}

int bevb200_bev_pool_lift_columns_dev(int b, int d, int h, int w, int n_capacity, int c, const float *depth,
                                      const float *ctx, int cameras, int depth_bins, int feature_h, int feature_w,
                                      const int32_t *geom_feats, const int32_t *interval_starts,
                                      const int32_t *col_begin, const uint64_t *seg_key, const uint64_t *seg_mask,
                                      const int32_t *seg_slot, const int32_t *interval_slot_begin, int max_segments,
                                      const int32_t *counts_dev, const int32_t *lift_form, float *out,
                                      void *workspace, size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(n_capacity > 0 && max_segments > 0, "capacities must be positive");
  BEVB200_REQUIRE(max_segments <= n_capacity, "max_segments must lie in [1, capacity]");
  BEVB200_REQUIRE(counts_dev && lift_form, "null counts / lift_form");
  return lift_columns(b, d, h, w, n_capacity, c, n_capacity, depth, ctx, cameras, depth_bins, feature_h, feature_w,
                      geom_feats, interval_starts, col_begin, seg_key, seg_mask, seg_slot, interval_slot_begin,
                      max_segments, out, workspace, workspace_bytes, (cudaStream_t)stream, counts_dev, lift_form);
}

size_t bevb200_bev_pool_lift_columns_backward_dev_workspace_bytes(int max_segments, int c) {
  if (max_segments <= 0 || !TunedWidths::has(c)) return 0;
  return lift_bwd_layout(max_segments, nullptr, nullptr) + kLiftQuerySlack;
}

int bevb200_bev_pool_lift_columns_backward_dev(int b, int d, int h, int w, int n_capacity, int c,
                                               const float *out_grad, const float *depth, const float *ctx,
                                               int cameras, int depth_bins, int feature_h, int feature_w,
                                               const int32_t *geom_feats, const int32_t *interval_starts,
                                               const int32_t *col_begin, const uint64_t *seg_key,
                                               const uint64_t *seg_mask, int max_segments, const int32_t *counts_dev,
                                               const int32_t *n_segments_dev, const int32_t *lift_form, float *ddepth,
                                               float *dctx, void *workspace, size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(n_capacity > 0 && max_segments > 0, "capacities must be positive");
  BEVB200_REQUIRE(max_segments <= n_capacity, "max_segments must lie in [1, capacity]");
  BEVB200_REQUIRE(counts_dev && n_segments_dev && lift_form, "null counts / n_segments / lift_form");
  return lift_columns_backward(b, d, h, w, n_capacity, c, n_capacity, out_grad, depth, ctx, cameras, depth_bins,
                               feature_h, feature_w, geom_feats, interval_starts, col_begin, seg_key, seg_mask,
                               max_segments, ddepth, dctx, workspace, workspace_bytes, (cudaStream_t)stream,
                               counts_dev, n_segments_dev, lift_form);
}

size_t bevb200_bev_pool_lift_backward_dev_workspace_bytes(int n_total, int c) {
  if (n_total <= 0 || !TunedWidths::has(c)) return 0;
  return lift_bwd_layout(n_total, nullptr, nullptr) + kLiftQuerySlack;
}

int bevb200_bev_pool_lift_backward_dev(int b, int d, int h, int w, int n_total, int c, const float *out_grad,
                                       const float *depth, const float *ctx, int depth_bins, int pixels_per_camera,
                                       const int32_t *perm, const int32_t *geom_feats, const int32_t *interval_starts,
                                       const int32_t *interval_lengths, const int32_t *counts_dev,
                                       const int32_t *lift_form, float *ddepth, float *dctx, void *workspace,
                                       size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(n_total > 0, "capacity must be positive");
  BEVB200_REQUIRE(counts_dev != nullptr, "null counts");
  return lift_rows_backward(b, d, h, w, n_total, n_total, c, n_total, out_grad, depth, ctx, depth_bins,
                            pixels_per_camera, perm, geom_feats, interval_starts, interval_lengths, ddepth, dctx,
                            workspace, workspace_bytes, (cudaStream_t)stream, counts_dev, lift_form);
}

}  // extern "C"
