// CenterHead box decode on the device: the first half of CenterHead.get_bboxes (models/heads/bbox/centerpoint.py
// :669-698) and CenterPointBBoxCoder.decode (core/bbox/coders/centerpoint_bbox_coders.py:62-225) for all T tasks and
// B samples of a frame -- sigmoid, the two-stage top-K, the regression gathers, the box decode, the score and centre
// range masks and the compaction -- with no host synchronisation and no allocation.  Segment s = t * B + b.
//
// Two launches per call:
//   chd_candidates_kernel  one CTA per tile of 1024 consecutive flat cells (c * H * W + row * W + col) of a segment:
//                          the score s of every cell and its order-preserving 64-bit key, written in index order to
//                          the tile's slice of the workspace with the tile's count.  With a score threshold only the
//                          cells with s > threshold, or NaN, are candidates: a NaN takes one of the K places in the
//                          reference and is masked afterwards, so it must count towards K; every other cell at or
//                          below the threshold would be masked had it been selected.
//   chd_decode_kernel      one CTA per segment: topk_select.cuh's exact select and sort of the K largest keys (value
//                          descending, NaN first, ties by ascending flat index), then per winner the gathers from the
//                          NCHW maps at its cell, the decode, the masks, and a block scan that compacts the survivors
//                          to the front of the segment in their order.  Rows at and after the count are zero.
//
// The reference's two top-k stages (per class, then over cat * K) select the K largest of the cat * H * W values;
// with stable sorts its order on equal values is class, then cell: the flat index.  Its "xs" is the row: trunc(float(ind)
// / float(W)), which equals ind / W in integers for ind < 2^24 (the quotient's rounding error, at most 2^-24 relative,
// is below the 1 / W that separates a non-integer quotient from the next integer), and "ys" the column.  Every
// arithmetic step is one fp32 rounding, in the reference's order, with no contraction; expf and atan2f are the
// accurate ones: the library is built without fast-math.
#include <math.h>

#include "topk_select.cuh"

namespace bevb200 {
namespace {

using namespace topk;

constexpr int kCandThreads = 256;
constexpr int kCellsPerThread = kTile / kCandThreads;
constexpr int kMaxTasks = BEVB200_DECODE_MAX_TASKS;

struct DecodeTask {
  const float *heat, *reg, *height, *dim, *rot, *vel;   // reg and vel null when absent
  int cat, chw;                                          // classes, cat * H * W
};

struct DecodeParams {
  DecodeTask task[kMaxTasks];
  int B, H, W, K, hw, tiles, code;      // tiles = ceil(max chw / kTile): every segment has that many slices
  int heat_is_logit, dim_is_log, use_thr;
  float thr, out_size_factor, voxel_x, voxel_y, pc_x, pc_y;
  float lo[3], hi[3];                   // post_center_range
};

__device__ __forceinline__ float score_of(const DecodeParams &p, float v) {
  return p.heat_is_logit ? sigmoid_as<float>(v) : v;
}

__global__ void __launch_bounds__(kCandThreads, 1)
    chd_candidates_kernel(const __grid_constant__ DecodeParams p, uint64_t *__restrict__ cand,
                          int32_t *__restrict__ tile_count) {
  const int seg = blockIdx.y, tile = blockIdx.x, tid = threadIdx.x;
  const DecodeTask &tk = p.task[seg / p.B];
  const float *heat = tk.heat + (long long)(seg % p.B) * tk.chw;
  uint64_t key[kCellsPerThread];
  unsigned bal[kCellsPerThread];
#pragma unroll
  for (int r = 0; r < kCellsPerThread; ++r) {
    const int flat = tile * kTile + r * kCandThreads + tid;
    bool keep = false;
    key[r] = 0;
    if (flat < tk.chw) {
      const float s = score_of(p, __ldg(heat + flat));
      keep = !p.use_thr || s > p.thr || isnan(s);
      key[r] = full_key(s, flat);
    }
    bal[r] = __ballot_sync(0xffffffffu, keep);
  }
  const long long slot = (long long)seg * p.tiles + tile;
  write_tile_keys<kCandThreads>(key, bal, cand + slot * kTile, tile_count + slot);
}

__global__ void __launch_bounds__(kSelectThreads, 1)
    chd_decode_kernel(const __grid_constant__ DecodeParams p, const uint64_t *__restrict__ cand_all,
                      const int32_t *__restrict__ count_all, int sort_n, float *__restrict__ boxes,
                      float *__restrict__ scores, float *__restrict__ labels, int32_t *__restrict__ index,
                      int32_t *__restrict__ counts) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint64_t *sel = (uint64_t *)smem;               // [sort_n]
  uint64_t *buf = sel + sort_n;                   // [kBufCap]
  __shared__ int warp_kept[kSelectWarps];
  const int seg = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int K = p.K, code = p.code;
  const DecodeTask &tk = p.task[seg / p.B];
  const int b = seg % p.B;
  const int nsel = select_top_keys(cand_all + (long long)seg * p.tiles * kTile, count_all + (long long)seg * p.tiles,
                                   p.tiles, K, sort_n, sel, buf);

  float *obox = boxes + (long long)seg * K * code;
  float *oscore = scores + (long long)seg * K, *olabel = labels + (long long)seg * K;
  int32_t *oindex = index ? index + (long long)seg * K : nullptr;
  const long long plane = (long long)b * p.hw;    // a one-channel map's offset of this sample
  int kept = 0;
  for (int j0 = 0; j0 < nsel; j0 += kSelectThreads) {
    const int j = j0 + tid;
    bool keep = false;
    float row[9], s = 0.f;
    int label = 0, ind = 0;
    if (j < nsel) {
      const int flat = (int)key_flat(sel[j]);
      label = flat / p.hw;
      ind = flat - label * p.hw;
      s = score_of(p, __ldg(tk.heat + (long long)b * tk.chw + flat));
      float x = (float)(ind / p.W), y = (float)(ind % p.W);        // the reference's xs is the row, ys the column
      if (tk.reg) {
        x = __fadd_rn(x, __ldg(tk.reg + 2 * plane + ind));
        y = __fadd_rn(y, __ldg(tk.reg + 2 * plane + p.hw + ind));
      } else {
        x = __fadd_rn(x, 0.5f);
        y = __fadd_rn(y, 0.5f);
      }
      row[0] = __fadd_rn(__fmul_rn(__fmul_rn(x, p.out_size_factor), p.voxel_x), p.pc_x);
      row[1] = __fadd_rn(__fmul_rn(__fmul_rn(y, p.out_size_factor), p.voxel_y), p.pc_y);
      row[2] = __ldg(tk.height + plane + ind);
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        const float v = __ldg(tk.dim + 3 * plane + d * p.hw + ind);
        row[3 + d] = p.dim_is_log ? expf(v) : v;
      }
      row[6] = atan2f(__ldg(tk.rot + 2 * plane + ind), __ldg(tk.rot + 2 * plane + p.hw + ind));
      row[7] = row[8] = 0.f;
      if (tk.vel) {
        row[7] = __ldg(tk.vel + 2 * plane + ind);
        row[8] = __ldg(tk.vel + 2 * plane + p.hw + ind);
      }
      keep = !p.use_thr || s > p.thr;
#pragma unroll
      for (int d = 0; d < 3; ++d) keep = keep && row[d] >= p.lo[d] && row[d] <= p.hi[d];
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_kept[warp] = __popc(bal);
    __syncthreads();
    const int mine = warp_kept[lane];             // every warp scans the 32 warp counts
    int incl = mine;
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    const int before = __shfl_sync(0xffffffffu, incl - mine, warp), total = __shfl_sync(0xffffffffu, incl, 31);
    if (keep) {
      const int pos = kept + before + __popc(bal & ((1u << lane) - 1u));
#pragma unroll
      for (int d = 0; d < 9; ++d)
        if (d < code) obox[(long long)pos * code + d] = row[d];
      oscore[pos] = s;
      olabel[pos] = (float)label;
      if (oindex) oindex[pos] = ind;
    }
    kept += total;
    __syncthreads();
  }
  if (tid == 0) counts[seg] = kept;
  for (int i = kept * code + tid; i < K * code; i += kSelectThreads) obox[i] = 0.f;
  for (int i = kept + tid; i < K; i += kSelectThreads) {
    oscore[i] = 0.f;
    olabel[i] = 0.f;
    if (oindex) oindex[i] = 0;
  }
}

size_t select_smem_bytes(int K) { return (size_t)(sort_size(K) + kBufCap) * sizeof(uint64_t); }

// 0 ok, 1 invalid, 2 unsupported
int check_sizes(int T, int B, const int *cat, int H, int W) {
  if (T < 1 || B < 1 || H < 1 || W < 1 || !cat) return 1;
  if (T > kMaxTasks || (long long)T * B > BEVB200_DECODE_MAX_SEGMENTS) return 2;
  for (int t = 0; t < T; ++t)
    if (cat[t] < 1) return 1;
  for (int t = 0; t < T; ++t)
    if (cat[t] > BEVB200_DECODE_MAX_CLASSES || (long long)cat[t] * H * W > BEVB200_DECODE_MAX_CELLS) return 2;
  return 0;
}

int max_tiles(int T, const int *cat, int H, int W) {
  int m = 0;
  for (int t = 0; t < T; ++t) m = max(m, (cat[t] * H * W + kTile - 1) / kTile);
  return m;
}

size_t ws_bytes(int T, int B, int tiles) {
  const size_t slices = (size_t)T * B * tiles;
  return align_up(slices * kTile * sizeof(uint64_t)) + align_up(slices * sizeof(int32_t));
}

}  // namespace
}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_centerhead_decode_workspace_bytes(int T, int B, const int *cat, int H, int W) {
  if (check_sizes(T, B, cat, H, W) != 0) return 0;
  return ws_bytes(T, B, max_tiles(T, cat, H, W));
}

int bevb200_centerhead_decode(const float *const *heatmap, const float *const *reg, const float *const *height,
                              const float *const *dim, const float *const *rot, const float *const *vel,
                              const int *cat, int T, int B, int H, int W, int max_num, int heat_is_logit,
                              int dim_is_log, double out_size_factor, double voxel_x, double voxel_y, double pc_x,
                              double pc_y, const double *post_center_range, int use_score_threshold,
                              double score_threshold, float *boxes, float *scores, float *labels, int32_t *index,
                              int32_t *counts, void *workspace, size_t workspace_bytes, void *stream) {
  const int sizes = check_sizes(T, B, cat, H, W);
  BEVB200_REQUIRE(sizes != 1, "T, B, H, W and every class count must be at least 1, cat not null");
  if (sizes == 2 || max_num > BEVB200_DECODE_MAX_K) {
    snprintf(g_last_error, sizeof(g_last_error),
             "%s: at most %d tasks, %d task-samples, %d classes and %d cells per task and sample, max_num %d (got T "
             "%d, B %d, H %d, W %d, max_num %d)",
             __func__, kMaxTasks, BEVB200_DECODE_MAX_SEGMENTS, BEVB200_DECODE_MAX_CLASSES, BEVB200_DECODE_MAX_CELLS,
             BEVB200_DECODE_MAX_K, T, B, H, W, max_num);
    return BEVB200_EUNSUPPORTED;
  }
  BEVB200_REQUIRE(max_num >= 1 && (long long)max_num <= (long long)H * W, "max_num must be in 1..H * W");
  BEVB200_REQUIRE(heatmap && height && dim && rot && post_center_range && boxes && scores && labels && counts,
                  "null pointer");
  DecodeParams p;
  memset(&p, 0, sizeof(p));
  for (int t = 0; t < T; ++t) {
    BEVB200_REQUIRE(heatmap[t] && height[t] && dim[t] && rot[t] && (!reg || reg[t]) && (!vel || vel[t]),
                    "null map pointer");
    DecodeTask &tk = p.task[t];
    tk.heat = heatmap[t];
    tk.reg = reg ? reg[t] : nullptr;
    tk.height = height[t];
    tk.dim = dim[t];
    tk.rot = rot[t];
    tk.vel = vel ? vel[t] : nullptr;
    tk.cat = cat[t];
    tk.chw = cat[t] * H * W;
  }
  p.B = B;
  p.H = H;
  p.W = W;
  p.K = max_num;
  p.hw = H * W;
  p.tiles = max_tiles(T, cat, H, W);
  p.code = vel ? 9 : 7;
  p.heat_is_logit = heat_is_logit != 0;
  p.dim_is_log = dim_is_log != 0;
  p.use_thr = use_score_threshold != 0;
  p.thr = (float)score_threshold;
  p.out_size_factor = (float)out_size_factor;
  p.voxel_x = (float)voxel_x;
  p.voxel_y = (float)voxel_y;
  p.pc_x = (float)pc_x;
  p.pc_y = (float)pc_y;
  for (int d = 0; d < 3; ++d) {
    p.lo[d] = (float)post_center_range[d];
    p.hi[d] = (float)post_center_range[3 + d];
  }
  const size_t need = ws_bytes(T, B, p.tiles);
  if (workspace_bytes < need || !workspace) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace %zu < %zu bytes", __func__, workspace_bytes, need);
    return BEVB200_EWORKSPACE;
  }
  const int S = T * B;
  Arena ar(workspace, workspace_bytes);
  uint64_t *cand = ar.take<uint64_t>((size_t)S * p.tiles * kTile);
  int32_t *tile_count = ar.take<int32_t>((size_t)S * p.tiles);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)p.tiles, (unsigned)S);
  BEVB200_LAUNCH(chd_candidates_kernel, grid, kCandThreads, 0, st, p, cand, tile_count);
  const size_t smem = select_smem_bytes(p.K);
  if (smem > 44 * 1024)
    BEVB200_CUDA(cudaFuncSetAttribute(chd_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  BEVB200_LAUNCH(chd_decode_kernel, S, kSelectThreads, smem, st, p, cand, tile_count, sort_size(p.K), boxes, scores,
                 labels, index, counts);
  return BEVB200_OK;
}

}  // extern "C"
