// LoadRadarPointsMultiSweeps + the radar face of PointsRangeFilter (loading.py:717-790, transforms_3d.py:607-612,
// radar_points.py:92-107) on the device, bit-exact to the reference's numpy / torch lines.
//
// The raw 18-column radar sweeps live in a store of [slots, slot_cap, 18] fp32 rows with a device row count per slot;
// a frame names, per sample, its sweeps in the reference's concatenation order by slot, with each sweep's float64
// sensor2lidar pose and time lag.  The host composes use_dim into one op code per output column (which derived value
// of the 58-column row it is, and whether it is normalised), so the kernels know the one-hot encodings but not the
// column layout.  Every frame parameter is read from device memory; the three launches can be replayed as a CUDA
// graph with new entries:
//   1. radar_count_kernel  one CTA per (128-row tile, entry, sample): rows kept by the range filter, and the
//                          bad-category check of every row (the reference raises on it before filtering).
//   2. sweeps_scan         (sweeps_scan.cuh) exclusive scan of each sample's tile counts, its count min(total, cap).
//   3. radar_write_kernel  the grid of 1: each kept row's output columns go to shared memory at its ballot rank in
//                          the tile, then the tile's kept rows, consecutive in the output, are stored with
//                          consecutive threads on consecutive floats.
// With a per-sample augmentation record (GlobalRotScaleTrans + RandomFlip3D, lidar_aug.cuh), output columns 0..4 are
// computed first and augmented as RadarPoints does, and the range test reads the augmented x, y; the count and the
// write kernel share aug_head, so counts and rows agree.
// The double expressions are written with _rn intrinsics, so nvcc cannot contract them differently from the FMA
// chain numpy's dgemm evaluates (DESIGN.md sections 4.27, 4.28).
#include <math.h>

#include "lidar_aug.cuh"
#include "sweeps_scan.cuh"

static_assert(sizeof(bevb200_radar_sweep_entry_t) == BEVB200_RADAR_SWEEP_ENTRY_BYTES, "entry layout");
static_assert(sizeof(bevb200_radar_sweep_params_t) == BEVB200_RADAR_SWEEP_PARAMS_BYTES, "params layout");

namespace bevb200 {
namespace {

constexpr int kThreads = 128;
constexpr int kTile = kThreads;                 // rows per CTA
constexpr int kLoadDim = BEVB200_RADAR_LOAD_DIM;
constexpr int kMaxDim = BEVB200_RADAR_SWEEP_MAX_DIM;
constexpr int kPitch = kMaxDim + 1;             // shared row pitch for out_dim 64; an odd pitch is used throughout
static_assert(kThreads >= kMaxDim, "one thread checks each op");

struct Frame {
  const float *store;
  const int32_t *slot_rows;
  const bevb200_radar_sweep_params_t *params;
  const bevb200_radar_sweep_entry_t *entries;
  const bevb200_lidar_aug_t *aug;   // [batch] or NULL; out_dim >= 5 when set
  int slots, slot_cap, max_entries, out_dim, tiles;
};

__device__ __forceinline__ int op_kind(int op) { return op & 0xff; }
__device__ __forceinline__ int op_arg(int op) { return (op >> 8) & 0xff; }
__device__ __forceinline__ int op_block(int op) { return (op >> 16) & 0xff; }

// the one-hot encodings of perform_encodings (loading.py:620-626): source column and width
__device__ __forceinline__ int onehot_width(int block) { return block == 0 ? 8 : block == 1 ? 5 : 18; }

__device__ __forceinline__ bool op_ok(int op) {
  const int kind = op_kind(op), arg = op_arg(op), block = op_block(op);
  if ((op >> 24) & ~1) return false;   // BEVB200_RADAR_OP_NORMALIZE is the only flag
  switch (kind) {
    case BEVB200_RADAR_OP_RAW: return block == 0 && arg < kLoadDim;
    case BEVB200_RADAR_OP_XYZ: return block == 0 && arg < 3;
    case BEVB200_RADAR_OP_VELO:
    case BEVB200_RADAR_OP_VELO_COMP: return block == 0 && arg < 2;
    case BEVB200_RADAR_OP_LAG:
    case BEVB200_RADAR_OP_NUSC: return block == 0 && arg == 0;
    case BEVB200_RADAR_OP_ONE_HOT: return block < 3 && arg < onehot_width(block);
    case BEVB200_RADAR_OP_ORDINAL: return block == 0;
    default: return false;
  }
}

// rows of the entry (0 for NONE or a malformed entry); *bad is set for a malformed one
__device__ __forceinline__ int entry_rows(const Frame &f, const bevb200_radar_sweep_entry_t &e, bool *bad) {
  *bad = false;
  if (e.kind == BEVB200_SWEEP_NONE) return 0;
  if (e.kind != BEVB200_SWEEP_SWEEP || e.slot < 0 || e.slot >= f.slots) {
    *bad = true;
    return 0;
  }
  return min(max(f.slot_rows[e.slot], 0), f.slot_cap);
}

// np.rint(v).astype(int) as a one-hot index of width w (negative indices wrap as numpy's do); -1 where the
// reference raises IndexError (NaN, +-inf and anything outside [-w, w))
__device__ __forceinline__ int onehot_index(float v, int w) {
  const float r = rintf(v);   // exact in fp32: the same value as np.rint on the float64 copy
  if (!(r >= (float)-w && r < (float)w)) return -1;
  const int i = (int)r;
  return i < 0 ? i + w : i;
}

// p @ R[j] as dgemm evaluates it: fma(p2, R[j][2], fma(p1, R[j][1], fma(p0, R[j][0], +0.0)))
__device__ __forceinline__ double chain(double p0, double p1, double p2, const double *R) {
  return __fma_rn(p2, R[2], __fma_rn(p1, R[1], __fma_rn(p0, R[0], 0.0)));
}

// The values of one raw row that are not raw columns (loading.py:744-772, 629-653)
struct Derived {
  float x, y, z;
  double velo0, velo1, comp0, comp1, lag;
  int hot0, hot1, hot2;   // one-hot indices, -1 when the reference raises
  float pdh;              // rint(column 15)
  bool nusc;
};

__device__ __forceinline__ Derived derive(const float *__restrict__ src, const bevb200_radar_sweep_entry_t &e,
                                          bool compensate) {
  Derived d;
  const double p0 = __ldg(src + 0), p1 = __ldg(src + 1), p2 = __ldg(src + 2);
  float xyz[3];
#pragma unroll
  for (int j = 0; j < 3; ++j)   // points_sweep[:, :3] @ R.T stored to fp32, then += t stored to fp32
    xyz[j] = __double2float_rn(__dadd_rn((double)__double2float_rn(chain(p0, p1, p2, e.rotation + 3 * j)),
                                         e.translation[j]));
  const double v6 = __ldg(src + 6), v7 = __ldg(src + 7), v8 = __ldg(src + 8), v9 = __ldg(src + 9);
  // [vx, vy, 0] @ R.T: the +0 column is a real term of the chain (it decides signed zeros)
  d.velo0 = chain(v6, v7, 0.0, e.rotation + 0);
  d.velo1 = chain(v6, v7, 0.0, e.rotation + 3);
  d.comp0 = chain(v8, v9, 0.0, e.rotation + 0);
  d.comp1 = chain(v8, v9, 0.0, e.rotation + 3);
  d.lag = e.time_diff;
  if (compensate) {   // points_sweep[:, :2] += velo_comp * time_diff: the float64 product, the sum, the fp32 store
    xyz[0] = __double2float_rn(__dadd_rn((double)xyz[0], __dmul_rn(d.comp0, d.lag)));
    xyz[1] = __double2float_rn(__dadd_rn((double)xyz[1], __dmul_rn(d.comp1, d.lag)));
  }
  d.x = xyz[0];
  d.y = xyz[1];
  d.z = xyz[2];
  const float c3 = __ldg(src + 3), c11 = __ldg(src + 11), c14 = __ldg(src + 14);
  d.hot0 = onehot_index(c3, 8);
  d.hot1 = onehot_index(c11, 5);
  d.hot2 = onehot_index(c14, 18);
  d.pdh = rintf(__ldg(src + 15));
  d.nusc = c14 == 0.f && c3 < 7.f && c11 == 3.f;
  return d;
}

// output column c: virtual column use_dim[c] in float64, normalised, stored to fp32 as torch.as_tensor does
__device__ __forceinline__ float column(const float *__restrict__ src, const Derived &d,
                                        const bevb200_radar_sweep_params_t *__restrict__ p, int c) {
  const int op = __ldg(p->ops + c), arg = op_arg(op);
  double v;
  switch (op_kind(op)) {
    case BEVB200_RADAR_OP_RAW: v = __ldg(src + arg); break;
    case BEVB200_RADAR_OP_XYZ: v = arg == 0 ? d.x : arg == 1 ? d.y : d.z; break;
    case BEVB200_RADAR_OP_VELO: v = arg == 0 ? d.velo0 : d.velo1; break;
    case BEVB200_RADAR_OP_VELO_COMP: v = arg == 0 ? d.comp0 : d.comp1; break;
    case BEVB200_RADAR_OP_LAG: v = d.lag; break;
    case BEVB200_RADAR_OP_ONE_HOT: {
      const int block = op_block(op);
      v = (block == 0 ? d.hot0 : block == 1 ? d.hot1 : d.hot2) == arg ? 1.0 : 0.0;
      break;
    }
    case BEVB200_RADAR_OP_ORDINAL: v = d.pdh > (float)arg ? 1.0 : 0.0; break;
    default: v = d.nusc ? 1.0 : 0.0; break;
  }
  if (op & BEVB200_RADAR_OP_NORMALIZE)   // normalize_feats: points[:, dim] -= min; points[:, dim] /= (max - min)
    v = __ddiv_rn(__dsub_rn(v, __ldg(p->norm_min + c)), __ldg(p->norm_span + c));
  return __double2float_rn(v);
}

// in_range_bev on output columns 0 and 1: strict fp32 comparisons, NaN fails them
__device__ __forceinline__ bool in_range(const float *__restrict__ src, const Derived &d,
                                         const bevb200_radar_sweep_params_t *__restrict__ p) {
  if (!p->has_range) return true;
  const float x = column(src, d, p, 0), y = column(src, d, p, 1);
  return x > p->range[0] && y > p->range[1] && x < p->range[2] && y < p->range[3];
}

// with an enabled record: output columns 0..4 augmented into v, and in_range_bev on the augmented x, y
__device__ __forceinline__ bool aug_head(const float *__restrict__ src, const Derived &d,
                                         const bevb200_radar_sweep_params_t *__restrict__ p,
                                         const bevb200_lidar_aug_t &a, float v[5]) {
#pragma unroll
  for (int c = 0; c < 5; ++c) v[c] = column(src, d, p, c);
  aug_point<true>(a, v);
  return !p->has_range || (v[0] > p->range[0] && v[1] > p->range[1] && v[0] < p->range[2] && v[1] < p->range[3]);
}

// every thread of the CTA: whether the op codes of the first out_dim columns are malformed
__device__ __forceinline__ bool params_bad(const Frame &f) {
  return __syncthreads_or(threadIdx.x < f.out_dim && !op_ok(__ldg(f.params->ops + threadIdx.x)));
}

template <bool kAug>
__global__ void __launch_bounds__(kThreads)
radar_count_kernel(Frame f, int32_t *__restrict__ tile_counts, int32_t *__restrict__ status) {
  const int t = blockIdx.x, ei = blockIdx.z * f.max_entries + blockIdx.y;
  const bevb200_radar_sweep_entry_t e = f.entries[ei];
  const bevb200_radar_sweep_params_t *p = f.params;
  const bevb200_lidar_aug_t a = aug_record(kAug ? f.aug : nullptr, blockIdx.z);
  bool bad;
  int n = entry_rows(f, e, &bad);
  const bool pbad = params_bad(f);
  if (t == 0 && threadIdx.x == 0 && (bad || pbad))
    atomicOr(status, (bad ? BEVB200_SWEEPS_BAD_ENTRY : 0) | (pbad ? BEVB200_SWEEPS_BAD_PARAMS : 0));
  if (pbad) n = 0;
  const int i = t * kTile + threadIdx.x;
  bool keep = false, bad_category = false;
  if (i < n) {
    const float *src = f.store + ((size_t)e.slot * f.slot_cap + i) * kLoadDim;
    const Derived d = derive(src, e, p->compensate_velocity != 0);
    bad_category = d.hot0 < 0 || d.hot1 < 0 || d.hot2 < 0;
    float v[5];
    keep = a.enabled ? aug_head(src, d, p, a, v) : in_range(src, d, p);
  }
  const int kept = __syncthreads_count(keep);
  if (__syncthreads_or(bad_category) && threadIdx.x == 0) atomicOr(status, BEVB200_RADAR_SWEEPS_BAD_CATEGORY);
  if (threadIdx.x == 0) tile_counts[(size_t)ei * f.tiles + t] = kept;
}

template <bool kAug>
__global__ void __launch_bounds__(kThreads)
radar_write_kernel(Frame f, const int32_t *__restrict__ tile_offsets, int cap, float *__restrict__ out) {
  __shared__ float rows[kTile * kPitch];
  __shared__ int warp_sum[kThreads / 32];
  const int t = blockIdx.x, ei = blockIdx.z * f.max_entries + blockIdx.y;
  const bevb200_radar_sweep_entry_t e = f.entries[ei];
  const bevb200_radar_sweep_params_t *p = f.params;
  const bevb200_lidar_aug_t a = aug_record(kAug ? f.aug : nullptr, blockIdx.z);
  bool bad;
  const int n = params_bad(f) ? 0 : entry_rows(f, e, &bad);
  const int row0 = t * kTile, off = tile_offsets[(size_t)ei * f.tiles + t];
  if (row0 >= n || off >= cap) return;   // uniform over the CTA
  const int i = row0 + threadIdx.x, D = f.out_dim, pitch = D | 1;
  const float *src = f.store + ((size_t)e.slot * f.slot_cap + i) * kLoadDim;
  Derived d;
  float v[5];
  bool keep = false;
  if (i < n) {
    d = derive(src, e, p->compensate_velocity != 0);
    keep = a.enabled ? aug_head(src, d, p, a, v) : in_range(src, d, p);
  }
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) warp_sum[warp] = __popc(m);
  __syncthreads();
  int before = 0, total = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    before += w < warp ? warp_sum[w] : 0;
    total += warp_sum[w];
  }
  const int rank = before + __popc(m & ((1u << lane) - 1));
  if (keep && off + rank < cap) {
    float *r = rows + rank * pitch;
    int c0 = 0;
    if (a.enabled) {
#pragma unroll
      for (int c = 0; c < 5; ++c) r[c] = v[c];
      c0 = 5;
    }
#pragma unroll 1
    for (int c = c0; c < D; ++c) r[c] = column(src, d, p, c);
  }
  __syncthreads();
  // the tile's kept rows are consecutive in the output: one coalesced copy of min(total, cap - off) rows
  const int nk = min(total, cap - off);
  float *dst = out + ((size_t)blockIdx.z * cap + off) * D;
  for (int k = threadIdx.x; k < nk * D; k += kThreads) {
    const int r = k / D;
    dst[k] = rows[r * pitch + (k - r * D)];
  }
}

int tiles_for(int slot_cap) { return (slot_cap + kTile - 1) / kTile; }

bool sizes_ok(int batch, int max_entries, int slot_cap) {
  return batch >= 0 && batch <= 65535 && max_entries >= 1 && max_entries <= 65535 && slot_cap >= 1 &&
         (long long)max_entries * slot_cap <= 0x7fffffffLL;
}

}  // namespace
}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_radar_sweeps_workspace_bytes(int batch, int max_entries, int slot_cap) {
  if (!sizes_ok(batch, max_entries, slot_cap)) return 0;
  return align_up((size_t)batch * max_entries * tiles_for(slot_cap) * sizeof(int32_t));
}

int bevb200_radar_sweeps_assemble(const float *store, int slots, int slot_cap, const int32_t *slot_rows,
                                  const bevb200_radar_sweep_params_t *params,
                                  const bevb200_radar_sweep_entry_t *entries, int batch, int max_entries,
                                  int out_dim, int cap, float *out, int32_t *counts, int32_t *status,
                                  void *workspace, size_t workspace_bytes, void *stream) {
  return bevb200_radar_sweeps_assemble_aug(store, slots, slot_cap, slot_rows, params, entries, nullptr, batch,
                                           max_entries, out_dim, cap, out, counts, status, workspace,
                                           workspace_bytes, stream);
}

int bevb200_radar_sweeps_assemble_aug(const float *store, int slots, int slot_cap, const int32_t *slot_rows,
                                      const bevb200_radar_sweep_params_t *params,
                                      const bevb200_radar_sweep_entry_t *entries, const bevb200_lidar_aug_t *aug,
                                      int batch, int max_entries, int out_dim, int cap, float *out, int32_t *counts,
                                      int32_t *status, void *workspace, size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(sizes_ok(batch, max_entries, slot_cap) && slots >= 1,
                  "sizes out of range (0 <= batch <= 65535, 1 <= max_entries <= 65535, slots >= 1, slot_cap >= 1, "
                  "max_entries * slot_cap < 2^31)");
  BEVB200_REQUIRE(out_dim >= 3 && out_dim <= kMaxDim, "out_dim must be in 3..64");
  BEVB200_REQUIRE(!aug || out_dim >= 5, "the augmentation reads output columns 3 and 4: out_dim must be >= 5");
  BEVB200_REQUIRE(cap >= 1 && (long long)cap * out_dim <= 0x7fffffffLL, "cap must be positive, cap * out_dim < 2^31");
  BEVB200_REQUIRE(status, "null pointer");
  if (batch == 0) {
    BEVB200_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), (cudaStream_t)stream));
    return BEVB200_OK;
  }
  BEVB200_REQUIRE(store && slot_rows && params && entries && out && counts, "null pointer");
  BEVB200_REQUIRE((uintptr_t)entries % alignof(bevb200_radar_sweep_entry_t) == 0 &&
                      (uintptr_t)params % alignof(bevb200_radar_sweep_params_t) == 0,
                  "misaligned parameter block");
  BEVB200_REQUIRE((uintptr_t)aug % alignof(bevb200_lidar_aug_t) == 0, "misaligned augmentation records");
  const size_t need = bevb200_radar_sweeps_workspace_bytes(batch, max_entries, slot_cap);
  if (!workspace || workspace_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace of %zu bytes, need %zu", __func__, workspace_bytes,
             need);
    return BEVB200_EWORKSPACE;
  }
  Frame f{store, slot_rows, params, entries, aug, slots, slot_cap, max_entries, out_dim, tiles_for(slot_cap)};
  int32_t *tiles = (int32_t *)workspace;
  cudaStream_t st = (cudaStream_t)stream;
  BEVB200_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
  const dim3 grid(f.tiles, max_entries, batch);
  // the plain path is its own instance, with the registers it had before the augmentation existed
  const auto count_kernel = aug ? radar_count_kernel<true> : radar_count_kernel<false>;
  const auto write_kernel = aug ? radar_write_kernel<true> : radar_write_kernel<false>;
  BEVB200_LAUNCH(count_kernel, grid, kThreads, 0, st, f, tiles, status);
  const int rc = sweeps_scan(tiles, batch, max_entries * f.tiles, cap, counts, status, st);
  if (rc) return rc;
  BEVB200_LAUNCH(write_kernel, grid, kThreads, 0, st, f, tiles, cap, out);
  return BEVB200_OK;
}

}  // extern "C"
