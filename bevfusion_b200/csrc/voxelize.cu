// Deterministic hard voxelization for sm_90a.
//
// Semantics restated from mmdet3d/ops/voxel/src/voxelization_cuda.cu:231-373 (GPU) and
// voxelization_cpu.cpp:45-101 (CPU): voxel ids in first-appearance order of the point index,
// slot inside a voxel = number of earlier points of that voxel, caps max_points / max_voxels.
// The reference gets there with an O(N^2) scan (:105-147) and a <<<1,1>>> serial kernel
// (:149-180); here it is five O(N) kernels, no device sync:
//
//   K1 vox_insert   coords (fp32 floor-div, IEEE) -> 64-bit cell key -> open-addressing hash
//                   insert (atomicCAS on the key); the CAS winner takes a provisional voxel id
//                   with a warp-aggregated atomicAdd.  Points remember their hash slot.
//   K2 vox_rank     per point: insert its index into the voxel's "P smallest point indices"
//                   list with a chain of atomicMin (a[s] = min(a[s], v); carry max on).  The
//                   final list is the sorted P smallest indices whatever the arrival order, so
//                   the result is deterministic.  A monotone early-out skips the atomics for
//                   points that are already beaten by a full list.
//   K3 vox_flags    point i is the first point of its voxel iff list[0] == i -> ballot words
//   K4 (scan)       exclusive popcount scan over the ballot words = first-appearance order
//   K5 vox_scatter  voxel id = rank of its first point; slot = position in the list; copy the
//                   point row, write coors / num_points (only voxel id < max_voxels).
#include "voxelize.cuh"

namespace bevb200 {

constexpr unsigned long long kEmptyKey = 0xffffffffffffffffull;
constexpr int kListEmpty = 0x7f7f7f7f;  // memset(0x7f) pattern, larger than any point index

// rows the kernels work on: n, or the device count clamped to [0, n] when there is one
__device__ __forceinline__ int live_rows(int n, const int32_t *__restrict__ n_dev) {
  return n_dev ? min(max(*n_dev, 0), n) : n;
}

__device__ __forceinline__ uint32_t hash64(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return (uint32_t)k;
}

__global__ void __launch_bounds__(256)
    vox_insert_kernel(const float *__restrict__ points, int n, const int32_t *__restrict__ n_dev, int nf,
                      VoxParams vp, unsigned long long *__restrict__ keys, int32_t *__restrict__ slot_pvid,
                      uint32_t table_mask, int32_t *__restrict__ point_slot,
                      int32_t *__restrict__ pvid_counter) {
  n = live_rows(n, n_dev);
  const int lane = lane_id();
  for (int base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31; base < n;
       base += gridDim.x * blockDim.x) {
    int i = base + lane;
    int c[3];
    bool valid = i < n && point_coords(points + (long long)i * nf, vp, c);
    int slot = -1;
    bool winner = false;
    if (valid) {
      unsigned long long key =
          ((unsigned long long)c[0] * vp.grid[1] + c[1]) * (unsigned long long)vp.grid[2] + c[2];
      uint32_t h = hash64(key) & table_mask;
      while (true) {
        unsigned long long prev = keys[h];
        if (prev == kEmptyKey) prev = atomicCAS(keys + h, kEmptyKey, key);
        if (prev == kEmptyKey) { winner = true; break; }
        if (prev == key) break;
        h = (h + 1) & table_mask;
      }
      slot = (int)h;
    }
    // warp-aggregated provisional voxel ids for the CAS winners
    unsigned wm = __ballot_sync(0xffffffffu, winner);
    if (wm) {
      int leader = __ffs(wm) - 1;
      int basev = 0;
      if (lane == leader) basev = atomicAdd(pvid_counter, __popc(wm));
      basev = __shfl_sync(0xffffffffu, basev, leader);
      if (winner) slot_pvid[slot] = basev + __popc(wm & ((1u << lane) - 1));
    }
    if (i < n) point_slot[i] = slot;
  }
}

__global__ void __launch_bounds__(256)
    vox_rank_kernel(int n, const int32_t *__restrict__ n_dev, int P, const int32_t *__restrict__ point_slot,
                    const int32_t *__restrict__ slot_pvid, int32_t *__restrict__ point_pvid,
                    int32_t *__restrict__ lists, int32_t *__restrict__ counts) {
  n = live_rows(n, n_dev);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int slot = point_slot[i];
    int pv = slot >= 0 ? slot_pvid[slot] : -1;
    point_pvid[i] = pv;
    if (pv < 0) continue;
    atomicAdd(counts + pv, 1);
    int32_t *a = lists + (long long)pv * P;
    // monotone early-out: the last list entry only ever decreases
    if (*(volatile int32_t *)(a + P - 1) < i) continue;
    int v = i;
    for (int s = 0; s < P; ++s) {
      int old = atomicMin(a + s, v);
      if (old == kListEmpty) break;  // took an empty slot, nothing displaced
      v = max(old, v);               // the larger index moves down the list
    }
  }
}

__global__ void __launch_bounds__(256)
    vox_flags_kernel(int n, const int32_t *__restrict__ n_dev, int P, const int32_t *__restrict__ point_pvid,
                     const int32_t *__restrict__ lists, uint32_t *__restrict__ first_bits) {
  // one ballot word per 32 points (n rounded up to a multiple of 32 by the launch loop); every word up to n is
  // written, so the scan's total counts only the live rows' voxels
  const int live = live_rows(n, n_dev);
  for (int base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31; base < n;
       base += gridDim.x * blockDim.x) {
    int i = base + lane_id();
    bool first = false;
    if (i < live) {
      int pv = point_pvid[i];
      first = pv >= 0 && lists[(long long)pv * P] == i;
    }
    unsigned m = __ballot_sync(0xffffffffu, first);
    if (lane_id() == 0) first_bits[base >> 5] = m;
  }
}

__global__ void __launch_bounds__(256)
    vox_scatter_kernel(const float *__restrict__ points, int n, int nf, VoxParams vp, int P,
                       int max_voxels, const int32_t *__restrict__ point_pvid,
                       const int32_t *__restrict__ lists, const int32_t *__restrict__ counts,
                       const uint32_t *__restrict__ first_bits,
                       const uint32_t *__restrict__ word_prefix,
                       const uint32_t *__restrict__ total_voxels, float *__restrict__ voxels,
                       int32_t *__restrict__ coors, int32_t *__restrict__ num_points,
                       int32_t *__restrict__ voxel_num) {
  if (blockIdx.x == 0 && threadIdx.x == 0)
    *voxel_num = (int32_t)min(*total_voxels, (uint32_t)max_voxels);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int pv = point_pvid[i];
    if (pv < 0) continue;
    const int32_t *a = lists + (long long)pv * P;
    int first = a[0];
    int vid = (int)(word_prefix[first >> 5] + __popc(first_bits[first >> 5] & ((1u << (first & 31)) - 1)));
    if (vid >= max_voxels) continue;
    int slot = -1;
    for (int s = 0; s < P; ++s)
      if (a[s] == i) { slot = s; break; }
    if (slot < 0) continue;  // more than max_points earlier points in this voxel
    const float *src = points + (long long)i * nf;
    float *dst = voxels + ((long long)vid * P + slot) * nf;
    for (int k = 0; k < nf; ++k) dst[k] = src[k];
    if (slot == 0) {
      int c[3];
      point_coords(src, vp, c);
      coors[3ll * vid + 0] = c[0];
      coors[3ll * vid + 1] = c[1];
      coors[3ll * vid + 2] = c[2];
      num_points[vid] = min(counts[pv], P);
    }
  }
}

// K5' (fused): the voxel's first point sums the rows named by the list (slot order), divides by
// the count and writes the mean row + (batch, x, y, z): voxelize + `feats.sum(dim=1) / sizes` +
// `F.pad(coords, (1, 0), value=k)` (bevfusion.py:178-195) without the [M, P, F] intermediate.
__global__ void __launch_bounds__(256)
    vox_mean_kernel(const float *__restrict__ points, int n, const int32_t *__restrict__ n_dev, int nf,
                    VoxParams vp, int P, int max_voxels, int batch_idx, const int32_t *__restrict__ point_pvid,
                    const int32_t *__restrict__ lists, const int32_t *__restrict__ counts,
                    const uint32_t *__restrict__ first_bits,
                    const uint32_t *__restrict__ word_prefix,
                    const uint32_t *__restrict__ total_voxels, float *__restrict__ feats,
                    int32_t *__restrict__ coords4, int32_t *__restrict__ num_points,
                    int32_t *__restrict__ voxel_num) {
  n = live_rows(n, n_dev);
  if (blockIdx.x == 0 && threadIdx.x == 0)
    *voxel_num = (int32_t)min(*total_voxels, (uint32_t)max_voxels);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int pv = point_pvid[i];
    if (pv < 0) continue;
    const int32_t *a = lists + (long long)pv * P;
    if (a[0] != i) continue;  // only the voxel's first point works
    int vid = (int)(word_prefix[i >> 5] + __popc(first_bits[i >> 5] & ((1u << (i & 31)) - 1)));
    if (vid >= max_voxels) continue;
    const int cnt = min(counts[pv], P);
    float acc[8];
    const int nfc = min(nf, 8);
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int s = 0; s < cnt; ++s) {
      const float *src = points + (long long)a[s] * nf;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (k < nfc) acc[k] = __fadd_rn(acc[k], src[k]);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (k < nfc) feats[(long long)vid * nf + k] = __fdiv_rn(acc[k], (float)cnt);
    int c[3];
    point_coords(points + (long long)i * nf, vp, c);
    *reinterpret_cast<int4 *>(coords4 + 4ll * vid) = make_int4(batch_idx, c[0], c[1], c[2]);
    if (num_points) num_points[vid] = cnt;
  }
}

__global__ void dynamic_voxelize_kernel(const float *__restrict__ points, int n, int nf,
                                        VoxParams vp, int32_t *__restrict__ coors) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int c[3];
    bool ok = point_coords(points + (long long)i * nf, vp, c);
    coors[3ll * i + 0] = ok ? c[0] : -1;
    coors[3ll * i + 1] = ok ? c[1] : -1;
    coors[3ll * i + 2] = ok ? c[2] : -1;
  }
}

__global__ void voxel_mean_kernel(const float *__restrict__ voxels,
                                  const int32_t *__restrict__ coors,
                                  const int32_t *__restrict__ num_points, int m, int P, int nf,
                                  int batch_idx, float *__restrict__ feats,
                                  int32_t *__restrict__ coords4) {
  long long total = (long long)m * nf;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    int v = (int)(idx / nf), k = (int)(idx % nf);
    // bevfusion.py:191-195: feats.sum(dim=1) / sizes  (all P slots, unused ones are zero)
    float s = 0.f;
    for (int p = 0; p < P; ++p) s += voxels[((long long)v * P + p) * nf + k];
    feats[idx] = __fdiv_rn(s, (float)num_points[v]);
    if (k == 0) {
      coords4[4ll * v + 0] = batch_idx;  // F.pad(c, (1, 0), value=k), bevfusion.py:183
      coords4[4ll * v + 1] = coors[3ll * v + 0];
      coords4[4ll * v + 2] = coors[3ll * v + 1];
      coords4[4ll * v + 3] = coors[3ll * v + 2];
    }
  }
}

int make_params(const float *vs, const float *range, VoxParams *vp) {
  for (int k = 0; k < 3; ++k) {
    vp->vs[k] = vs[k];
    vp->lo[k] = range[k];
    // voxelization_cuda.cu:256-258: grid = round((max - min) / voxel) in fp32
    vp->grid[k] = (int)roundf((range[3 + k] - range[k]) / vs[k]);
    if (!(vs[k] > 0.f) || vp->grid[k] <= 0) return -1;
  }
  return 0;
}

static size_t vox_layout(int n, int P, void *ws, size_t ws_bytes, VoxWs *out) {
  Arena a(ws, ws_bytes);
  VoxWs w;
  uint32_t ts = 1024;
  while (ts < 2u * (uint32_t)(n > 0 ? n : 1)) ts <<= 1;
  w.table_size = ts;
  w.nwords = ((size_t)n + 31) / 32;
  w.keys = a.take<unsigned long long>(ts);
  w.lists = a.take<int32_t>((size_t)n * P);
  w.counts = a.take<int32_t>(n);
  w.pvid_counter = a.take<int32_t>(64);
  w.total = (uint32_t *)(w.pvid_counter + 1);
  w.slot_pvid = a.take<int32_t>(ts);
  w.point_slot = a.take<int32_t>(n);
  w.point_pvid = a.take<int32_t>(n);
  w.first_bits = a.take<uint32_t>(w.nwords);
  w.word_prefix = a.take<uint32_t>(w.nwords);
  w.tiles = a.take<uint32_t>(scan_scratch_elems(w.nwords));
  if (out) *out = w;
  return a.off;
}

// K1-K4, shared by the plain, the mean-fused and the pillar-fused entry points
int vox_front(const char *who, const float *points, int n, const int32_t *n_dev, int num_features,
              const VoxParams &vp, int max_points, void *workspace, size_t workspace_bytes, cudaStream_t st,
              VoxWs *wout) {
  VoxWs w;
  size_t need = vox_layout(n, max_points, workspace, workspace_bytes, &w);
  if (workspace == nullptr || workspace_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace too small (%zu < %zu)", who,
             workspace_bytes, need);
    return BEVB200_EWORKSPACE;
  }
  // keys = empty (0xff..), lists = 0x7f7f7f7f, counts / counters = 0: the three regions are
  // laid out back to back in that order (see vox_layout)
  BEVB200_CUDA(cudaMemsetAsync(w.keys, 0xff, (size_t)w.table_size * sizeof(unsigned long long), st));
  BEVB200_CUDA(cudaMemsetAsync(w.lists, 0x7f, (size_t)n * max_points * sizeof(int32_t), st));
  BEVB200_CUDA(cudaMemsetAsync(w.counts, 0, (char *)w.slot_pvid - (char *)w.counts, st));
  const int grid = grid_for(n, 256);
  BEVB200_LAUNCH(vox_insert_kernel, grid, 256, 0, st, points, n, n_dev, num_features, vp, w.keys,
                 w.slot_pvid, w.table_size - 1, w.point_slot, w.pvid_counter);
  BEVB200_LAUNCH(vox_rank_kernel, grid, 256, 0, st, n, n_dev, max_points, w.point_slot, w.slot_pvid,
                 w.point_pvid, w.lists, w.counts);
  BEVB200_LAUNCH(vox_flags_kernel, grid, 256, 0, st, n, n_dev, max_points, w.point_pvid, w.lists,
                 w.first_bits);
  int rc = exclusive_scan_u32(w.first_bits, w.word_prefix, w.nwords, w.tiles, w.total, true, st);
  if (rc) return rc;
  *wout = w;
  return BEVB200_OK;
}

}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_hard_voxelize_workspace_bytes(int num_points, int max_points) {
  if (num_points < 0 || max_points <= 0) return 0;
  return vox_layout(num_points, max_points, nullptr, 0, nullptr);
}

int bevb200_hard_voxelize(const float *points, int num_points, int num_features,
                          const float *voxel_size_host, const float *coors_range_host,
                          int max_points, int max_voxels, float *voxels, int32_t *coors,
                          int32_t *num_points_per_voxel, int32_t *voxel_num, void *workspace,
                          size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(num_points >= 0 && num_features >= 3, "bad point tensor shape");
  BEVB200_REQUIRE(max_points > 0 && max_voxels > 0, "max_points / max_voxels must be positive");
  BEVB200_REQUIRE(voxel_size_host && coors_range_host && voxel_num, "null argument");
  VoxParams vp;
  BEVB200_REQUIRE(make_params(voxel_size_host, coors_range_host, &vp) == 0, "bad voxel grid");
  cudaStream_t st = (cudaStream_t)stream;
  const int n = num_points;
  if (n == 0) {
    BEVB200_CUDA(cudaMemsetAsync(voxel_num, 0, sizeof(int32_t), st));
    return BEVB200_OK;
  }
  BEVB200_REQUIRE(points && voxels && coors && num_points_per_voxel, "null argument");
  VoxWs w;
  int rc = vox_front("hard_voxelize", points, n, nullptr, num_features, vp, max_points, workspace,
                     workspace_bytes, st, &w);
  if (rc) return rc;
  BEVB200_LAUNCH(vox_scatter_kernel, grid_for(n, 256), 256, 0, st, points, n, num_features, vp,
                 max_points, max_voxels, w.point_pvid, w.lists, w.counts, w.first_bits, w.word_prefix,
                 w.total, voxels, coors, num_points_per_voxel, voxel_num);
  return BEVB200_OK;
}

int bevb200_hard_voxelize_mean(const float *points, int num_points, int num_features,
                               const float *voxel_size_host, const float *coors_range_host,
                               int max_points, int max_voxels, int batch_idx, float *feats,
                               int32_t *coords4, int32_t *num_points_per_voxel, int32_t *voxel_num,
                               void *workspace, size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(num_points >= 0 && num_features >= 3 && num_features <= 8, "bad point tensor shape");
  BEVB200_REQUIRE(max_points > 0 && max_voxels > 0, "max_points / max_voxels must be positive");
  BEVB200_REQUIRE(voxel_size_host && coors_range_host && voxel_num, "null argument");
  VoxParams vp;
  BEVB200_REQUIRE(make_params(voxel_size_host, coors_range_host, &vp) == 0, "bad voxel grid");
  cudaStream_t st = (cudaStream_t)stream;
  const int n = num_points;
  if (n == 0) {
    BEVB200_CUDA(cudaMemsetAsync(voxel_num, 0, sizeof(int32_t), st));
    return BEVB200_OK;
  }
  BEVB200_REQUIRE(points && feats && coords4, "null argument");
  BEVB200_REQUIRE((uintptr_t)coords4 % 16 == 0, "coords must be 16-byte aligned");
  VoxWs w;
  int rc = vox_front("hard_voxelize_mean", points, n, nullptr, num_features, vp, max_points, workspace,
                     workspace_bytes, st, &w);
  if (rc) return rc;
  BEVB200_LAUNCH(vox_mean_kernel, grid_for(n, 256), 256, 0, st, points, n, nullptr, num_features, vp,
                 max_points, max_voxels, batch_idx, w.point_pvid, w.lists, w.counts, w.first_bits,
                 w.word_prefix, w.total, feats, coords4, num_points_per_voxel, voxel_num);
  return BEVB200_OK;
}

int bevb200_hard_voxelize_mean_dev(const float *points, const int32_t *num_points_dev, int max_rows,
                                   int num_features, const float *voxel_size_host,
                                   const float *coors_range_host, int max_points, int max_voxels,
                                   int batch_idx, float *feats, int32_t *coords4,
                                   int32_t *num_points_per_voxel, int32_t *voxel_num, void *workspace,
                                   size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(max_rows >= 0 && num_features >= 3 && num_features <= 8, "bad point tensor shape");
  BEVB200_REQUIRE(max_points > 0 && max_voxels > 0, "max_points / max_voxels must be positive");
  BEVB200_REQUIRE(voxel_size_host && coors_range_host && voxel_num, "null argument");
  VoxParams vp;
  BEVB200_REQUIRE(make_params(voxel_size_host, coors_range_host, &vp) == 0, "bad voxel grid");
  cudaStream_t st = (cudaStream_t)stream;
  const int n = max_rows;
  if (n == 0) {
    BEVB200_CUDA(cudaMemsetAsync(voxel_num, 0, sizeof(int32_t), st));
    return BEVB200_OK;
  }
  BEVB200_REQUIRE(points && num_points_dev && feats && coords4, "null argument");
  BEVB200_REQUIRE((uintptr_t)coords4 % 16 == 0, "coords must be 16-byte aligned");
  VoxWs w;
  int rc = vox_front("hard_voxelize_mean_dev", points, n, num_points_dev, num_features, vp, max_points,
                     workspace, workspace_bytes, st, &w);
  if (rc) return rc;
  BEVB200_LAUNCH(vox_mean_kernel, grid_for(n, 256), 256, 0, st, points, n, num_points_dev, num_features, vp,
                 max_points, max_voxels, batch_idx, w.point_pvid, w.lists, w.counts, w.first_bits,
                 w.word_prefix, w.total, feats, coords4, num_points_per_voxel, voxel_num);
  return BEVB200_OK;
}

int bevb200_dynamic_voxelize(const float *points, int num_points, int num_features,
                             const float *voxel_size_host, const float *coors_range_host,
                             int32_t *coors, void *stream) {
  BEVB200_REQUIRE(num_points >= 0 && num_features >= 3, "bad point tensor shape");
  BEVB200_REQUIRE(voxel_size_host && coors_range_host, "null argument");
  VoxParams vp;
  BEVB200_REQUIRE(make_params(voxel_size_host, coors_range_host, &vp) == 0, "bad voxel grid");
  if (num_points == 0) return BEVB200_OK;
  BEVB200_REQUIRE(points && coors, "null argument");
  BEVB200_LAUNCH(dynamic_voxelize_kernel, grid_for(num_points, 256), 256, 0, (cudaStream_t)stream,
                 points, num_points, num_features, vp, coors);
  return BEVB200_OK;
}

int bevb200_voxel_mean(const float *voxels, const int32_t *coors, const int32_t *num_points,
                       int num_voxels, int max_points, int num_features, int batch_idx,
                       float *feats, int32_t *coords4, void *stream) {
  BEVB200_REQUIRE(num_voxels >= 0 && max_points > 0 && num_features > 0, "bad sizes");
  if (num_voxels == 0) return BEVB200_OK;
  BEVB200_REQUIRE(voxels && coors && num_points && feats && coords4, "null argument");
  BEVB200_LAUNCH(voxel_mean_kernel, grid_for((long long)num_voxels * num_features, 256), 256, 0,
                 (cudaStream_t)stream, voxels, coors, num_points, num_voxels, max_points,
                 num_features, batch_idx, feats, coords4);
  return BEVB200_OK;
}

}  // extern "C"
