// Sparse convolution filter gradient on the tensor cores (BF16x3-class precision, no atomics).
//
//   dW[k][ci][co] = sum over output rows o of  features[nbr[k][o]][ci] * out_grad[o][co]      (spconv_ops.h:363-456,
//   the `torch::mm_out(filterGradSub, inputBuffer.t(), outputBuffer)` per kernel offset of indiceConvBackward)
//
// The reduction runs over ROWS, so both operands are "MN-major" for the tensor core: a row of an operand tile is one
// reduction index and holds the M (or N) elements contiguously -- which is how the split images of spconv_v6.cu store
// a row (per 16 channels: 16 bf16 hi | 16 bf16 lo); ldmatrix.trans turns such rows into mma.sync fragments.  The
// kernel
//   * gives every CTA work items (row chunk, kernel offset k): the accumulator dW[k] (Cin x Cout fp32, in the
//     registers of 8 warps: warp w owns channel rows (w & 1) * Cin / 2 .. and columns (w >> 1) * Cout / 4 ..) lives
//     for the whole item and is written once as a partial dW; a second kernel adds the partials of the chunks in a
//     fixed order (bit-reproducible, like the SIMT path it replaces);
//   * per stage of 32 rows gathers the feature rows (through nbr, missing rows as zeros) and the contiguous out-grad
//     rows with 16-byte cp.async into XOR-swizzled tiles (chunk c of row r at c ^ (r & 7): conflict-free ldmatrix),
//     in a ring of cp.async stages;
//   * multiplies hi.hi + hi.lo + lo.hi per 16-row k step (the lo.lo term is below the fp32 rounding of the sum).
#include <stdlib.h>

#include "spconv.cuh"
#include "tc_ptx.cuh"

namespace bevb200 {

constexpr int kWgtThreads = 256;
constexpr int kWgtRows = 32;           // reduction rows per stage
constexpr int kWgtStages = 3;

struct WgtParams {
  const uint8_t *fsplit;       // [n_in][ci_eff * 4 B]
  const uint8_t *gsplit;       // [n_out][co_eff * 4 B]
  const int32_t *nbr;          // [kvol][n_out]
  float *partial;              // [n_chunks][kvol][c_in][c_out]
  int n_in, n_out, c_in, c_out, kvol;
  int n_chunks, tiles_per_chunk, n_tiles;   // tiles of kWgtRows rows
};

template <int CI, int CO>
struct WgtShape {
  static constexpr int kFRow = CI * 4, kGRow = CO * 4;           // bytes per operand row
  static constexpr int kStage = kWgtRows * (kFRow + kGRow);
  static constexpr int kSmem = kWgtStages * kStage;
};

// byte offset of logical 16-byte chunk c of row r in a tile of `row_bytes` rows (XOR swizzle inside 128-byte lines)
__device__ __forceinline__ uint32_t wgt_off(int r, int c, int row_bytes) {
  return (uint32_t)(r * row_bytes + ((c ^ (r & 7)) << 4));
}

template <int CI, int CO>
__global__ void __launch_bounds__(kWgtThreads, 1) spconv_wgrad_tc_kernel(const WgtParams p) {
  using Sh = WgtShape<CI, CO>;
  constexpr int FR = Sh::kFRow, GR = Sh::kGRow;
  constexpr int MT = CI / 32;          // m16 tiles per warp (two warps along Cin)
  constexpr int NT = CO / 32;          // n8 tiles per warp (four warps along Cout)
  constexpr int FCH = FR / 16, GCH = GR / 16;   // 16-byte chunks per row
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const uint32_t smem = smem_u32(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = (warp & 1) * (CI / 2), wn = (warp >> 1) * (CO / 4);
  const unsigned long long fbase = reinterpret_cast<unsigned long long>(p.fsplit);
  const unsigned long long gbase = reinterpret_cast<unsigned long long>(p.gsplit);
  const int n_items = p.n_chunks * p.kvol;

  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int chunk = item / p.kvol, k = item - chunk * p.kvol;
    const int t_begin = chunk * p.tiles_per_chunk, t_end = min(p.n_tiles, t_begin + p.tiles_per_chunk);
    const int nt_items = t_end - t_begin;
    const int32_t *nbr_k = p.nbr + (long long)k * p.n_out;
    auto load_stage = [&](int i) {
      const uint32_t f = smem + (uint32_t)(i % kWgtStages) * Sh::kStage, g = f + kWgtRows * FR;
      const int o0 = (t_begin + i) * kWgtRows;
      for (int u = tid; u < kWgtRows * FCH; u += kWgtThreads) {
        const int r = u / FCH, c = u - r * FCH;
        int src = o0 + r < p.n_out ? __ldg(nbr_k + o0 + r) : -1;
        if (src >= p.n_in) src = -1;
        cp_async16_row(f + wgt_off(r, c, FR), fbase + (unsigned long long)(uint32_t)max(src, 0) * FR + c * 16, src);
      }
      for (int u = tid; u < kWgtRows * GCH; u += kWgtThreads) {
        const int r = u / GCH, c = u - r * GCH;
        const int o = o0 + r < p.n_out ? o0 + r : -1;
        cp_async16_row(g + wgt_off(r, c, GR), gbase + (unsigned long long)(uint32_t)max(o, 0) * GR + c * 16, o);
      }
    };
    float acc[MT][NT][4];
#pragma unroll
    for (int a = 0; a < MT; ++a)
#pragma unroll
      for (int b = 0; b < NT; ++b)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[a][b][e] = 0.f;
#pragma unroll
    for (int s = 0; s < kWgtStages - 1; ++s) {
      if (s < nt_items) load_stage(s);
      cp_async_commit();
    }
    for (int i = 0; i < nt_items; ++i) {
      cp_async_wait<kWgtStages - 2>();
      __syncthreads();
      if (i + kWgtStages - 1 < nt_items) load_stage(i + kWgtStages - 1);
      cp_async_commit();
      const uint32_t f = smem + (uint32_t)(i % kWgtStages) * Sh::kStage, g = f + kWgtRows * FR;
#pragma unroll
      for (int ks = 0; ks < kWgtRows / 16; ++ks) {
        // A = F^T: m = input channel, k = row.  Matrix q of ldmatrix.x4.trans: rows k0 + 8 (q >> 1) .., channels
        // m0 + 8 (q & 1) ..; the channel group m0 / 16 keeps hi at chunk 4 (m0 / 16) + 0 / 1, lo at + 2 / 3.
        uint32_t ahi[MT][4], alo[MT][4];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          const int m0 = wm + 16 * mt, q = lane >> 3;
          const int r = ks * 16 + 8 * (q >> 1) + (lane & 7);
          const int c = 4 * (m0 >> 4) + (q & 1);
          ldsm_x4_t(f + wgt_off(r, c, FR), ahi[mt]);
          ldsm_x4_t(f + wgt_off(r, c + 2, FR), alo[mt]);
        }
        // B = G: k = row, n = output channel.  x4.trans: matrices (rows k0 .. / k0 + 8 ..) x (n0 .. / n0 + 8 ..)
#pragma unroll
        for (int nt = 0; nt < NT; nt += 2) {
          const int n0 = wn + 8 * nt, q = lane >> 3;
          uint32_t bh[4], bl[4];
          if constexpr (NT == 1) {
            const int r = ks * 16 + 8 * (q & 1) + (lane & 7);
            const int c = 4 * (n0 >> 4) + ((n0 >> 3) & 1);
            uint32_t t2[2];
            ldsm_x2_t(g + wgt_off(r, c, GR), t2);
            bh[0] = t2[0]; bh[1] = t2[1];
            ldsm_x2_t(g + wgt_off(r, c + 2, GR), t2);
            bl[0] = t2[0]; bl[1] = t2[1];
          } else {
            const int r = ks * 16 + 8 * (q & 1) + (lane & 7);
            const int n = n0 + 8 * (q >> 1);
            const int c = 4 * (n >> 4) + ((n >> 3) & 1);
            ldsm_x4_t(g + wgt_off(r, c, GR), bh);
            ldsm_x4_t(g + wgt_off(r, c + 2, GR), bl);
          }
#pragma unroll
          for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int h = 0; h < (NT == 1 ? 1 : 2); ++h) {
              mma_bf16_16816(acc[mt][nt + h], alo[mt], bh[2 * h], bh[2 * h + 1]);
              mma_bf16_16816(acc[mt][nt + h], ahi[mt], bl[2 * h], bl[2 * h + 1]);
              mma_bf16_16816(acc[mt][nt + h], ahi[mt], bh[2 * h], bh[2 * h + 1]);
            }
        }
      }
    }
    cp_async_wait<0>();
    __syncthreads();                   // the ring is free for the next item
    float *dst_k = p.partial + ((long long)chunk * p.kvol + k) * p.c_in * p.c_out;
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const int ci = wm + 16 * mt + (lane >> 2), co = wn + 8 * nt + 2 * (lane & 3);
        if (co < p.c_out) {
          if (ci < p.c_in)
            *reinterpret_cast<float2 *>(dst_k + (long long)ci * p.c_out + co) = make_float2(acc[mt][nt][0], acc[mt][nt][1]);
          if (ci + 8 < p.c_in)
            *reinterpret_cast<float2 *>(dst_k + (long long)(ci + 8) * p.c_out + co) = make_float2(acc[mt][nt][2], acc[mt][nt][3]);
        }
      }
  }
}

bool spconv_wgrad_tc_ok(int c_in, int c_out, int kvol) {
  static const bool enabled = [] {
    const char *e = getenv("BEVB200_WGRAD_TC");
    return e == nullptr || atoi(e) != 0;
  }();
  return enabled && c_in >= 1 && c_in <= 128 && (c_out == 16 || c_out == 32 || c_out == 64 || c_out == 128) &&
         kvol >= 1 && kvol <= 27;
}

// channel count of an operand image: 128-byte slabs of 32 channels, 1 / 2 / 4 of them (zero padded)
static int wgt_eff(int c) { return c <= 32 ? 32 : (c <= 64 ? 64 : 128); }

// The shape of a launch: row tiles and row chunks (~3 work items per SM, every chunk non-empty).
struct WgtPlan {
  int ci_eff, co_eff;
  int n_tiles, n_chunks, tiles_per_chunk;
};
static WgtPlan wgt_plan(int n_out, int c_in, int c_out, int kvol) {
  WgtPlan w;
  w.ci_eff = wgt_eff(c_in);
  w.co_eff = wgt_eff(c_out);
  w.n_tiles = (n_out + kWgtRows - 1) / kWgtRows;
  int n_chunks = (3 * kNumSMs) / kvol;
  if (n_chunks < 1) n_chunks = 1;
  if (n_chunks > w.n_tiles) n_chunks = w.n_tiles > 0 ? w.n_tiles : 1;
  w.tiles_per_chunk = w.n_tiles > 0 ? (w.n_tiles + n_chunks - 1) / n_chunks : 1;
  w.n_chunks = w.n_tiles > 0 ? (w.n_tiles + w.tiles_per_chunk - 1) / w.tiles_per_chunk : 1;
  return w;
}

// where spconv_wgrad_tc() leaves the split image of out_grad inside its workspace; for c_out = 32 / 64 / 128 it is the
// row image of out_grad the forward kernel takes, which the input gradient can gather from instead of splitting again
const void *spconv_wgrad_tc_grad_image(const void *workspace, int n_in, int c_in) {
  return (const uint8_t *)workspace + align_up((size_t)n_in * wgt_eff(c_in) * 4);
}

size_t spconv_wgrad_tc_workspace_bytes(int n_in, int n_out, int c_in, int c_out, int kvol) {
  if (!spconv_wgrad_tc_ok(c_in, c_out, kvol) || n_in <= 0 || n_out <= 0) return 0;
  const WgtPlan w = wgt_plan(n_out, c_in, c_out, kvol);
  return align_up((size_t)n_in * w.ci_eff * 4) + align_up((size_t)n_out * w.co_eff * 4) +
         align_up((size_t)w.n_chunks * kvol * c_in * c_out * sizeof(float));
}

template <int CI, int CO>
static int wgt_launch(const WgtParams &p, cudaStream_t st) {
  constexpr int smem = WgtShape<CI, CO>::kSmem;
  const int n_items = p.n_chunks * p.kvol;
  const int grid = n_items < kNumSMs ? n_items : kNumSMs;
  BEVB200_CUDA(cudaFuncSetAttribute(spconv_wgrad_tc_kernel<CI, CO>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  BEVB200_LAUNCH((spconv_wgrad_tc_kernel<CI, CO>), grid, kWgtThreads, smem, st, p);
  return BEVB200_OK;
}
template <int CI>
static int wgt_launch_co(const WgtParams &p, int co_eff, cudaStream_t st) {
  if (co_eff == 32) return wgt_launch<CI, 32>(p, st);
  if (co_eff == 64) return wgt_launch<CI, 64>(p, st);
  return wgt_launch<CI, 128>(p, st);
}

int spconv_wgrad_tc(const float *features, const float *out_grad, const int32_t *nbr, int n_in, int n_out,
                    int c_in, int c_out, int kvol, float *weight_grad, void *workspace, cudaStream_t st) {
  BEVB200_REQUIRE(spconv_wgrad_tc_ok(c_in, c_out, kvol), "shape has no tensor-core filter gradient");
  const WgtPlan w = wgt_plan(n_out, c_in, c_out, kvol);
  const int ci_eff = w.ci_eff, co_eff = w.co_eff;
  uint8_t *fsplit = (uint8_t *)workspace;
  uint8_t *gsplit = fsplit + align_up((size_t)n_in * ci_eff * 4);
  float *partial = (float *)(gsplit + align_up((size_t)n_out * co_eff * 4));
  int rc = spconv_v6_split_rows(features, n_in, nullptr, c_in, ci_eff, fsplit, st);
  if (!rc) rc = spconv_v6_split_rows(out_grad, n_out, nullptr, c_out, co_eff, gsplit, st);
  if (rc) return rc;
  WgtParams p;
  memset(&p, 0, sizeof(p));
  p.fsplit = fsplit;
  p.gsplit = gsplit;
  p.nbr = nbr;
  p.partial = partial;
  p.n_in = n_in; p.n_out = n_out; p.c_in = c_in; p.c_out = c_out; p.kvol = kvol;
  p.n_tiles = w.n_tiles; p.n_chunks = w.n_chunks; p.tiles_per_chunk = w.tiles_per_chunk;
  if (ci_eff == 32) rc = wgt_launch_co<32>(p, co_eff, st);
  else if (ci_eff == 64) rc = wgt_launch_co<64>(p, co_eff, st);
  else rc = wgt_launch_co<128>(p, co_eff, st);
  if (rc) return rc;
  return spconv_wgrad_reduce(partial, (long long)kvol * c_in * c_out, p.n_chunks, weight_grad, st);
}

}  // namespace bevb200
