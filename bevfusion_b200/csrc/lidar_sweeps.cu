// LoadPointsFromMultiSweeps + PointsRangeFilter of the LiDAR pipeline (loading.py:87-235, transforms_3d.py:585-614,
// base_points.py:208-232) on the device, bit-exact to the reference's numpy / torch lines.
//
// The raw sweeps live in a store of [slots, slot_cap, load_dim] fp32 rows with a device row count per slot; a frame
// names, per sample, its ordered entries (the key, then the chosen sweeps, or pad copies of the key) by slot, with
// each sweep's float64 pose and time lag.  Every frame parameter is read from device memory, so the three launches
// can be replayed as a CUDA graph with new entries:
//   1. sweeps_count_kernel  one CTA per (1024-row tile, entry, sample): rows kept after remove_close, the transform
//                           and the range filter.  Tiles past the slot's device row count write 0 and exit.
//   2. sweeps_scan_kernel   one CTA per sample: exclusive scan of its tile counts in (entry, tile) order, which is
//                           the reference's concatenation order; the sample's count is min(total, cap).
//   3. sweeps_write_kernel  the grid of 1: each kept row is recomputed and written at its tile offset plus its rank
//                           in the tile (ballot ranks, no atomics), if that is below cap.
// With a per-sample augmentation record (GlobalRotScaleTrans + RandomFlip3D, lidar_aug.cuh), eval_row applies it to
// the row's x, y, z before the range test, in both the count and the write kernel, so counts and rows agree.
// With a paste block (ObjectPaste), the grid gains max_paste entries in front of each sample's sweep entries, one per
// kept object: they come first in the scan order, as the reference concatenates [pasted rows, surviving rows].  A
// pasted row is its object's stored row, column-mapped and translated, then augmented and range-tested.  The sweep
// entries stage the sample's face planes in shared memory and drop every row inside a kept box (eval_row).
// The double expressions are written with _rn intrinsics, so nvcc cannot contract them differently from the FMA chain
// numpy's dgemm evaluates (see DESIGN.md section 4.27).
#include <math.h>

#include "lidar_aug.cuh"
#include "sweeps_scan.cuh"

static_assert(sizeof(bevb200_sweep_entry_t) == BEVB200_SWEEP_ENTRY_BYTES, "entry layout");
static_assert(sizeof(bevb200_sweep_params_t) == BEVB200_SWEEP_PARAMS_BYTES, "params layout");
static_assert(sizeof(bevb200_paste_sample_t) == BEVB200_PASTE_SAMPLE_BYTES, "paste sample layout");
static_assert(sizeof(bevb200_paste_object_t) == BEVB200_PASTE_OBJECT_BYTES, "paste object layout");

namespace bevb200 {
namespace {

constexpr int kThreads = 256;
constexpr int kRounds = 4;
constexpr int kTile = kThreads * kRounds;     // rows per CTA
constexpr int kMaxLoadDim = 64;

struct Frame {
  const float *store;
  const int32_t *slot_rows;
  const bevb200_sweep_params_t *params;
  const bevb200_sweep_entry_t *entries;
  const bevb200_lidar_aug_t *aug;   // [batch] or NULL
  int slots, slot_cap, load_dim, max_entries, out_dim, tiles;
};

// the object store and the frame's paste block (unused by the instances without one)
struct Paste {
  const float *rows;                       // [max_rows, obj_dim]
  const int32_t *table;                    // [num_objects, 2]: first row, rows
  const bevb200_paste_sample_t *samples;   // [batch]
  const bevb200_paste_object_t *objects;   // [batch, max_paste]
  int max_rows, obj_dim, num_objects, object_cap, max_paste;
};

__device__ __forceinline__ bool params_ok(const bevb200_sweep_params_t &p, int load_dim, int out_dim) {
  bool ok = true;
#pragma unroll
  for (int c = 0; c < 8; ++c)
    ok = ok && (c >= out_dim || (p.key_cols[c] >= 0 && p.key_cols[c] < load_dim && p.sweep_cols[c] >= 0 &&
                                 p.sweep_cols[c] < load_dim));
  return ok;
}

// rows of the entry (0 for NONE or a malformed entry); *bad is set for a malformed one
__device__ __forceinline__ int entry_rows(const Frame &f, const bevb200_sweep_entry_t &e, bool *bad) {
  *bad = false;
  if (e.kind == BEVB200_SWEEP_NONE) return 0;
  if ((e.kind != BEVB200_SWEEP_KEY && e.kind != BEVB200_SWEEP_SWEEP && e.kind != BEVB200_SWEEP_PAD) || e.slot < 0 ||
      e.slot >= f.slots) {
    *bad = true;
    return 0;
  }
  return min(max(f.slot_rows[e.slot], 0), f.slot_cap);
}

// in_range_3d: strict fp32 comparisons, NaN fails them all
__device__ __forceinline__ bool in_range(const bevb200_sweep_params_t &p, const float v[8]) {
  return v[0] > p.range[0] && v[1] > p.range[1] && v[2] > p.range[2] && v[0] < p.range[3] && v[1] < p.range[4] &&
         v[2] < p.range[5];
}

// points_in_rbbox on one point: inside a box unless one face gives ((x n0 + y n1) + z n2) + d >= 0 in fp32 with no
// contraction, so a point on a face is outside and a NaN coordinate is inside every box.  planes: [S][6] (n, d).
__device__ __forceinline__ bool in_any_box(const float4 *planes, int S, float x, float y, float z) {
  for (int k = 0; k < S; ++k) {
    bool inside = true;
#pragma unroll
    for (int q = 0; q < 6 && inside; ++q) {
      const float4 pl = planes[6 * k + q];
      inside = !(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, pl.x), __fmul_rn(y, pl.y)), __fmul_rn(z, pl.z)), pl.w) >=
                 0.0f);
    }
    if (inside) return true;
  }
  return false;
}

// One row of an entry: its output columns and whether it survives remove_close, ObjectPaste's removal (kPaste: the
// S boxes' planes), the augmentation and the range filter
template <bool kPaste>
__device__ __forceinline__ bool eval_row(const float *__restrict__ src, const bevb200_sweep_entry_t &e,
                                         const bevb200_sweep_params_t &p, const bevb200_lidar_aug_t &a, int out_dim,
                                         float v[8], const float4 *planes = nullptr, int S = 0) {
  const bool sweep = e.kind == BEVB200_SWEEP_SWEEP;
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = c < out_dim ? __ldg(src + (sweep ? p.sweep_cols[c] : p.key_cols[c])) : 0.f;
  if (p.remove_close && e.kind != BEVB200_SWEEP_KEY) {
    // loading.py:167-169 on the raw sweep row (before use_dim), or on the key's selected columns for a pad copy
    const float x = sweep ? __ldg(src + 0) : v[0], y = sweep ? __ldg(src + 1) : v[1];
    if (fabsf(x) < p.radius && fabsf(y) < p.radius) return false;
  }
  if (sweep) {
    // points_sweep[:, :3] @ R.T (fp32 x fp64 -> dgemm), the fp32 store, then += t in float64 and the fp32 store.
    // The dgemm's accumulator starts at +0.0, so a zero dot product is +0.0 even when every term is -0.0.
    const double p0 = v[0], p1 = v[1], p2 = v[2];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double r = __fma_rn(p2, e.rotation[3 * j + 2], __fma_rn(p1, e.rotation[3 * j + 1],
                                                                    __fma_rn(p0, e.rotation[3 * j + 0], 0.0)));
      v[j] = __double2float_rn(__dadd_rn((double)__double2float_rn(r), e.translation[j]));
    }
    v[4] = __double2float_rn(e.lag);
  } else {
    v[4] = 0.0f;
  }
  if (kPaste && in_any_box(planes, S, v[0], v[1], v[2])) return false;
  aug_point<false>(a, v);
  if (p.has_range) return in_range(p, v);
  return true;
}

// Pasted row i of kept object j of sample b: the object's row through the column map, xyz += fl32(box[:3]) in fp32,
// then the augmentation and the range filter
__device__ __forceinline__ bool eval_paste_row(const float *__restrict__ src, const bevb200_paste_sample_t &s,
                                               const bevb200_paste_object_t &o, const bevb200_sweep_params_t &p,
                                               const bevb200_lidar_aug_t &a, int out_dim, float v[8]) {
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = c < out_dim ? __ldg(src + s.cols[c]) : 0.f;
#pragma unroll
  for (int j = 0; j < 3; ++j) v[j] = __fadd_rn(v[j], o.translation[j]);
  aug_point<false>(a, v);
  if (p.has_range) return in_range(p, v);
  return true;
}

// Whether store object idx exists and its table entry (first row, rows) lies inside the store
__device__ __forceinline__ bool object_ok(const Paste &pz, int idx) {
  if (idx < 0 || idx >= pz.num_objects) return false;
  const int first = pz.table[2 * idx], n = pz.table[2 * idx + 1];
  return first >= 0 && n >= 0 && n <= pz.object_cap && (long long)first + n <= pz.max_rows;
}

// Kept object j of sample b: its first stored row (*src) and its rows; 0 past the sample's count or for a bad object
// (paste_block_ok then rejects the whole block)
__device__ __forceinline__ int paste_object_rows(const Paste &pz, int b, int j, const float **src) {
  const int S = pz.samples[b].count;
  if (j >= S || S > pz.max_paste) return 0;
  const int idx = pz.objects[(size_t)b * pz.max_paste + j].index;
  if (!object_ok(pz, idx)) return 0;
  *src = pz.rows + (size_t)pz.table[2 * idx] * pz.obj_dim;
  return pz.table[2 * idx + 1];
}

// Whether sample b's paste block is well formed: count in [0, max_paste], the column map inside [0, obj_dim) and every
// kept object valid.  Called by every thread of the CTA.
__device__ __forceinline__ bool paste_block_ok(const Paste &pz, int b, int out_dim) {
  const bevb200_paste_sample_t &s = pz.samples[b];
  const int S = s.count;
  bool ok = S >= 0 && S <= pz.max_paste;
#pragma unroll
  for (int c = 0; c < 8; ++c) ok = ok && (c >= out_dim || (s.cols[c] >= 0 && s.cols[c] < pz.obj_dim));
  int bad = 0;
  if (ok)
    for (int j = threadIdx.x; j < S; j += kThreads) bad |= !object_ok(pz, pz.objects[(size_t)b * pz.max_paste + j].index);
  return __syncthreads_or(bad) == 0 && ok;
}

// Stages sample b's face planes (S x 6 float4) in shared memory; returns S, or 0 for a malformed block
__device__ __forceinline__ int paste_stage(const Paste &pz, int b, int out_dim, float4 *planes) {
  const int S = paste_block_ok(pz, b, out_dim) ? pz.samples[b].count : 0;
  for (int i = threadIdx.x; i < 6 * S; i += kThreads) {
    const float *q = pz.objects[(size_t)b * pz.max_paste + i / 6].planes[i % 6];
    planes[i] = make_float4(q[0], q[1], q[2], q[3]);
  }
  __syncthreads();
  return S;
}

template <bool kAug, bool kPaste>
__global__ void __launch_bounds__(kThreads)
sweeps_count_kernel(Frame f, Paste pz, int32_t *__restrict__ tile_counts, int32_t *__restrict__ status) {
  extern __shared__ float4 planes[];   // kPaste: the sample's face planes
  const int t = blockIdx.x, np = kPaste ? pz.max_paste : 0;
  const bevb200_sweep_params_t p = *f.params;
  const bevb200_lidar_aug_t a = aug_record(kAug ? f.aug : nullptr, blockIdx.z);
  const int row0 = t * kTile;
  if (kPaste && (int)blockIdx.y < np) {   // kept object blockIdx.y of the sample
    const float *src = nullptr;
    int n = params_ok(p, f.load_dim, f.out_dim) ? paste_object_rows(pz, blockIdx.z, blockIdx.y, &src) : 0;
    int kept = 0;
    if (row0 < n || (t == 0 && blockIdx.y == 0)) {   // uniform over the CTA
      const bool ok = paste_block_ok(pz, blockIdx.z, f.out_dim);
      if (t == 0 && blockIdx.y == 0 && threadIdx.x == 0 && !ok) atomicOr(status, BEVB200_SWEEPS_BAD_PASTE);
      if (!ok) n = 0;
      const bevb200_paste_sample_t &ps = pz.samples[blockIdx.z];
      const bevb200_paste_object_t &o = pz.objects[(size_t)blockIdx.z * np + blockIdx.y];
      for (int r = 0; r < kRounds && row0 < n; ++r) {
        const int i = row0 + r * kThreads + threadIdx.x;
        float v[8];
        kept += __syncthreads_count(i < n && eval_paste_row(src + (size_t)i * pz.obj_dim, ps, o, p, a, f.out_dim, v));
      }
    }
    if (threadIdx.x == 0) tile_counts[((size_t)blockIdx.z * (np + f.max_entries) + blockIdx.y) * f.tiles + t] = kept;
    return;
  }
  const int ei = blockIdx.z * f.max_entries + (blockIdx.y - np);
  const bevb200_sweep_entry_t e = f.entries[ei];
  bool bad;
  int n = entry_rows(f, e, &bad);
  const bool pbad = !params_ok(p, f.load_dim, f.out_dim);
  if (t == 0 && threadIdx.x == 0 && (bad || pbad))
    atomicOr(status, (bad ? BEVB200_SWEEPS_BAD_ENTRY : 0) | (pbad ? BEVB200_SWEEPS_BAD_PARAMS : 0));
  if (pbad) n = 0;
  int kept = 0;
  if (row0 < n) {
    const int S = kPaste ? paste_stage(pz, blockIdx.z, f.out_dim, planes) : 0;
    const float *base = f.store + (size_t)e.slot * f.slot_cap * f.load_dim;
    for (int r = 0; r < kRounds; ++r) {
      const int i = row0 + r * kThreads + threadIdx.x;
      float v[8];
      kept += __syncthreads_count(i < n && eval_row<kPaste>(base + (size_t)i * f.load_dim, e, p, a, f.out_dim, v,
                                                            planes, S));
    }
  }
  if (threadIdx.x == 0)
    tile_counts[kPaste ? ((size_t)blockIdx.z * (np + f.max_entries) + blockIdx.y) * f.tiles + t
                       : (size_t)ei * f.tiles + t] = kept;
}

__global__ void __launch_bounds__(kThreads)
sweeps_scan_kernel(int32_t *__restrict__ tile_counts, int len, int cap, int32_t *__restrict__ counts,
                   int32_t *__restrict__ status) {
  __shared__ int warp_sum[kThreads / 32];
  int32_t *c = tile_counts + (size_t)blockIdx.x * len;
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  int carry = 0;
  for (int base = 0; base < len; base += kThreads) {
    const int i = base + threadIdx.x;
    const int v = i < len ? c[i] : 0;
    int incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += u;
    }
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
      before += w < warp ? warp_sum[w] : 0;
      total += warp_sum[w];
    }
    if (i < len) c[i] = carry + before + incl - v;
    carry += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    counts[blockIdx.x] = min(carry, cap);
    if (carry > cap) atomicOr(status, BEVB200_SWEEPS_OVERFLOW);
  }
}

// Writes the kept rows of one tile at its scanned offset plus their ballot ranks, below cap
template <typename Eval>
__device__ __forceinline__ void write_tile(int row0, int n, int off, int cap, int out_dim, float *__restrict__ dst,
                                           int *warp_sum, Eval eval) {
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  for (int r = 0; r < kRounds; ++r) {
    const int i = row0 + r * kThreads + threadIdx.x;
    float v[8];
    const bool keep = i < n && eval(i, v);
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_sum[warp] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
      before += w < warp ? warp_sum[w] : 0;
      total += warp_sum[w];
    }
    const int pos = off + before + __popc(m & ((1u << lane) - 1));
    if (keep && pos < cap) {
      float *o = dst + (size_t)pos * out_dim;
#pragma unroll
      for (int c = 0; c < 8; ++c)
        if (c < out_dim) o[c] = v[c];
    }
    off += total;
    __syncthreads();
  }
}

template <bool kAug, bool kPaste>
__global__ void __launch_bounds__(kThreads)
sweeps_write_kernel(Frame f, Paste pz, const int32_t *__restrict__ tile_offsets, int cap, float *__restrict__ out) {
  __shared__ int warp_sum[kThreads / 32];
  extern __shared__ float4 planes[];   // kPaste: the sample's face planes
  const int t = blockIdx.x, np = kPaste ? pz.max_paste : 0;
  if (kPaste && (int)blockIdx.y < np) {   // kept object blockIdx.y of the sample
    const bevb200_sweep_params_t p = *f.params;
    const bevb200_lidar_aug_t a = aug_record(kAug ? f.aug : nullptr, blockIdx.z);
    const int row0 = t * kTile;
    float *dst = out + (size_t)blockIdx.z * cap * f.out_dim;
    const float *src = nullptr;
    const int n = params_ok(p, f.load_dim, f.out_dim) ? paste_object_rows(pz, blockIdx.z, blockIdx.y, &src) : 0;
    const int off = tile_offsets[((size_t)blockIdx.z * (np + f.max_entries) + blockIdx.y) * f.tiles + t];
    if (row0 >= n || off >= cap || !paste_block_ok(pz, blockIdx.z, f.out_dim)) return;   // uniform over the CTA
    const bevb200_paste_sample_t &ps = pz.samples[blockIdx.z];
    const bevb200_paste_object_t &o = pz.objects[(size_t)blockIdx.z * np + blockIdx.y];
    write_tile(row0, n, off, cap, f.out_dim, dst, warp_sum, [&](int i, float v[8]) {
      return eval_paste_row(src + (size_t)i * pz.obj_dim, ps, o, p, a, f.out_dim, v);
    });
    return;
  }
  const int ei = blockIdx.z * f.max_entries + (blockIdx.y - np);
  const bevb200_sweep_entry_t e = f.entries[ei];
  const bevb200_sweep_params_t p = *f.params;
  const bevb200_lidar_aug_t a = aug_record(kAug ? f.aug : nullptr, blockIdx.z);
  bool bad;
  const int n = params_ok(p, f.load_dim, f.out_dim) ? entry_rows(f, e, &bad) : 0;
  const int row0 = t * kTile;
  int off = tile_offsets[kPaste ? ((size_t)blockIdx.z * (np + f.max_entries) + blockIdx.y) * f.tiles + t
                                : (size_t)ei * f.tiles + t];
  if (row0 >= n || off >= cap) return;   // uniform over the CTA
  const int S = kPaste ? paste_stage(pz, blockIdx.z, f.out_dim, planes) : 0;
  const float *base = f.store + (size_t)e.slot * f.slot_cap * f.load_dim;
  float *dst = out + (size_t)blockIdx.z * cap * f.out_dim;
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  for (int r = 0; r < kRounds; ++r) {
    const int i = row0 + r * kThreads + threadIdx.x;
    float v[8];
    const bool keep = i < n && eval_row<kPaste>(base + (size_t)i * f.load_dim, e, p, a, f.out_dim, v, planes, S);
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_sum[warp] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
      before += w < warp ? warp_sum[w] : 0;
      total += warp_sum[w];
    }
    const int pos = off + before + __popc(m & ((1u << lane) - 1));
    if (keep && pos < cap) {
      float *o = dst + (size_t)pos * f.out_dim;
#pragma unroll
      for (int c = 0; c < 8; ++c)
        if (c < f.out_dim) o[c] = v[c];
    }
    off += total;
    __syncthreads();
  }
}

int tiles_for(int slot_cap) { return (slot_cap + kTile - 1) / kTile; }

bool sizes_ok(int batch, int max_entries, int slot_cap) {
  return batch >= 0 && batch <= 65535 && max_entries >= 1 && max_entries <= 65535 && slot_cap >= 1 &&
         (long long)max_entries * slot_cap <= 0x7fffffffLL;
}

}  // namespace

int sweeps_scan(int32_t *tile_counts, int batch, int len, int cap, int32_t *counts, int32_t *status,
                cudaStream_t st) {
  BEVB200_LAUNCH(sweeps_scan_kernel, batch, kThreads, 0, st, tile_counts, len, cap, counts, status);
  return BEVB200_OK;
}

}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_lidar_sweeps_workspace_bytes(int batch, int max_entries, int slot_cap) {
  if (!sizes_ok(batch, max_entries, slot_cap)) return 0;
  return align_up((size_t)batch * max_entries * tiles_for(slot_cap) * sizeof(int32_t));
}

int bevb200_lidar_sweeps_assemble(const float *store, int slots, int slot_cap, int load_dim, const int32_t *slot_rows,
                                  const bevb200_sweep_params_t *params, const bevb200_sweep_entry_t *entries,
                                  int batch, int max_entries, int out_dim, int cap, float *out, int32_t *counts,
                                  int32_t *status, void *workspace, size_t workspace_bytes, void *stream) {
  return bevb200_lidar_sweeps_assemble_aug(store, slots, slot_cap, load_dim, slot_rows, params, entries, nullptr,
                                           batch, max_entries, out_dim, cap, out, counts, status, workspace,
                                           workspace_bytes, stream);
}

size_t bevb200_lidar_sweeps_paste_workspace_bytes(int batch, int max_entries, int slot_cap, int max_paste,
                                                  int object_cap) {
  if (!sizes_ok(batch, max_entries, slot_cap) || max_paste < 0 || max_paste > BEVB200_PASTE_MAX_OBJECTS ||
      max_entries + max_paste > 65535 || object_cap < 1 || (long long)(max_entries + max_paste) * object_cap > 0x7fffffffLL)
    return 0;
  return align_up((size_t)batch * (max_entries + max_paste) * tiles_for(max(slot_cap, object_cap)) * sizeof(int32_t));
}

int bevb200_lidar_sweeps_assemble_aug(const float *store, int slots, int slot_cap, int load_dim,
                                      const int32_t *slot_rows, const bevb200_sweep_params_t *params,
                                      const bevb200_sweep_entry_t *entries, const bevb200_lidar_aug_t *aug, int batch,
                                      int max_entries, int out_dim, int cap, float *out, int32_t *counts,
                                      int32_t *status, void *workspace, size_t workspace_bytes, void *stream) {
  return bevb200_lidar_sweeps_assemble_paste(store, slots, slot_cap, load_dim, slot_rows, params, entries, aug,
                                             nullptr, 0, 0, nullptr, 0, 1, nullptr, nullptr, 0, batch, max_entries,
                                             out_dim, cap, out, counts, status, workspace, workspace_bytes, stream);
}

int bevb200_lidar_sweeps_assemble_paste(const float *store, int slots, int slot_cap, int load_dim,
                                        const int32_t *slot_rows, const bevb200_sweep_params_t *params,
                                        const bevb200_sweep_entry_t *entries, const bevb200_lidar_aug_t *aug,
                                        const float *objects, int max_rows, int obj_dim, const int32_t *object_table,
                                        int num_objects, int object_cap, const bevb200_paste_sample_t *paste,
                                        const bevb200_paste_object_t *paste_objects, int max_paste, int batch,
                                        int max_entries, int out_dim, int cap, float *out, int32_t *counts,
                                        int32_t *status, void *workspace, size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(sizes_ok(batch, max_entries, slot_cap) && slots >= 1,
                  "sizes out of range (0 <= batch <= 65535, 1 <= max_entries <= 65535, slots >= 1, slot_cap >= 1, "
                  "max_entries * slot_cap < 2^31)");
  BEVB200_REQUIRE(load_dim >= 3 && load_dim <= kMaxLoadDim, "load_dim must be in 3..64");
  BEVB200_REQUIRE(out_dim >= 5 && out_dim <= BEVB200_SWEEP_MAX_DIM, "out_dim must be in 5..8");
  BEVB200_REQUIRE(cap >= 1, "cap must be positive");
  BEVB200_REQUIRE(status, "null pointer");
  if (paste) {
    BEVB200_REQUIRE(max_paste >= 1 && max_paste <= BEVB200_PASTE_MAX_OBJECTS, "max_paste must be in 1..256");
    BEVB200_REQUIRE(obj_dim >= 1 && obj_dim <= kMaxLoadDim && max_rows >= 0 && num_objects >= 0 && object_cap >= 1,
                    "object store sizes out of range (1 <= obj_dim <= 64, max_rows >= 0, num_objects >= 0, "
                    "object_cap >= 1)");
  }
  const int np = paste ? max_paste : 0;
  if (batch == 0) {
    BEVB200_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), (cudaStream_t)stream));
    return BEVB200_OK;
  }
  BEVB200_REQUIRE(store && slot_rows && params && entries && out && counts, "null pointer");
  BEVB200_REQUIRE(!paste || (paste_objects && object_table && (objects || max_rows == 0)), "null pointer");
  BEVB200_REQUIRE((uintptr_t)entries % alignof(bevb200_sweep_entry_t) == 0 &&
                      (uintptr_t)params % alignof(bevb200_sweep_params_t) == 0,
                  "misaligned parameter block");
  BEVB200_REQUIRE((uintptr_t)aug % alignof(bevb200_lidar_aug_t) == 0, "misaligned augmentation records");
  BEVB200_REQUIRE((uintptr_t)paste % alignof(bevb200_paste_sample_t) == 0 &&
                      (uintptr_t)paste_objects % alignof(bevb200_paste_object_t) == 0 &&
                      (uintptr_t)object_table % alignof(int32_t) == 0 && (uintptr_t)objects % alignof(float) == 0,
                  "misaligned paste block or object store");
  const size_t need = paste ? bevb200_lidar_sweeps_paste_workspace_bytes(batch, max_entries, slot_cap, max_paste,
                                                                         object_cap)
                            : bevb200_lidar_sweeps_workspace_bytes(batch, max_entries, slot_cap);
  BEVB200_REQUIRE(need > 0, "sizes out of range (max_entries + max_paste <= 65535, "
                            "(max_entries + max_paste) * object_cap < 2^31)");
  if (!workspace || workspace_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace of %zu bytes, need %zu", __func__, workspace_bytes,
             need);
    return BEVB200_EWORKSPACE;
  }
  Frame f{store, slot_rows, params, entries, aug, slots, slot_cap, load_dim, max_entries, out_dim,
          tiles_for(paste ? max(slot_cap, object_cap) : slot_cap)};
  const Paste pz{objects, object_table, paste, paste_objects, max_rows, obj_dim, num_objects, object_cap, np};
  int32_t *tiles = (int32_t *)workspace;
  cudaStream_t st = (cudaStream_t)stream;
  BEVB200_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
  const dim3 grid(f.tiles, np + max_entries, batch);
  // the plain and augmented paths are their own instances, with the registers they had before the paste existed
  const auto count_kernel = paste ? (aug ? sweeps_count_kernel<true, true> : sweeps_count_kernel<false, true>)
                                  : (aug ? sweeps_count_kernel<true, false> : sweeps_count_kernel<false, false>);
  const auto write_kernel = paste ? (aug ? sweeps_write_kernel<true, true> : sweeps_write_kernel<false, true>)
                                  : (aug ? sweeps_write_kernel<true, false> : sweeps_write_kernel<false, false>);
  const size_t smem = (size_t)np * 6 * sizeof(float4);
  BEVB200_LAUNCH(count_kernel, grid, kThreads, smem, st, f, pz, tiles, status);
  const int rc = sweeps_scan(tiles, batch, (np + max_entries) * f.tiles, cap, counts, status, st);
  if (rc) return rc;
  BEVB200_LAUNCH(write_kernel, grid, kThreads, smem, st, f, pz, tiles, cap, out);
  return BEVB200_OK;
}

}  // extern "C"
