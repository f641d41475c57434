// Sparse convolution forward, exact-fp32 SIMT path (BEVB200_PREC_FP32) + dense() for sm_90a.
//
// Replaces spconv::indiceConv<float> (spconv_ops.h:260-361): the reference runs, per kernel
// offset, gather (reordering.cu.h:22-98) -> torch::mm_out (cuBLAS SGEMM) -> scatter-add
// (reordering.cu.h:100-157), i.e. ~80 launches per conv and every pair row crossing HBM three
// times.  Here one output-stationary implicit-GEMM kernel walks the 27 offsets for a tile of
// output rows: A rows are gathered straight from the feature matrix through the neighbour
// table, accumulators stay in registers across all offsets, and the BN / residual / ReLU
// epilogue (SparseSequential + SparseBasicBlock, modules.py:127-139, sparse_block.py:94-110)
// is applied before the single store of each output row.
//
// This file is the fp32-FFMA variant (bit-for-bit fp32 products, fp32 accumulation); the
// tensor-core variants live in spconv_v6.cu, and spconv_fwd.cu picks between them.
#include "spconv.cuh"

namespace bevb200 {

constexpr int kSimtThreads = 256;
constexpr int kSimtBK = 16;

template <int BN, int TN>
__global__ void __launch_bounds__(kSimtThreads)
    spconv_simt_kernel(const float *__restrict__ features, const float *__restrict__ weight,
                       const int32_t *__restrict__ nbr, int n_in, int n_out, int c_in, int c_out,
                       int kvol, const float *__restrict__ scale, const float *__restrict__ shift,
                       const float *__restrict__ residual, int relu, float *__restrict__ out) {
  constexpr int TM = 4, TX = BN / TN, TY = kSimtThreads / TX, BM = TY * TM, BK = kSimtBK;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN];
  __shared__ int nb[BM];
  const int tid = threadIdx.x, tx = tid % TX, ty = tid / TX;
  const int row0 = blockIdx.x * BM;
  const bool vec_a = (c_in % 4 == 0) && ((uintptr_t)features % 16 == 0);
  const bool vec_b = (c_out % 4 == 0) && ((uintptr_t)weight % 16 == 0);

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int k = 0; k < kvol; ++k) {
    int any = 0;
    for (int r = tid; r < BM; r += kSimtThreads) {
      int o = row0 + r;
      int j = o < n_out ? __ldg(nbr + (long long)k * n_out + o) : -1;
      if (j >= n_in) j = -1;
      nb[r] = j;
      any |= (j >= 0);
    }
    if (!__syncthreads_or(any)) continue;  // no row of this tile has a neighbour at offset k
    const float *wk = weight + (long long)k * c_in * c_out;
    for (int c0 = 0; c0 < c_in; c0 += BK) {
      // A tile: gathered feature rows, stored transposed (k-major) for conflict-free reads
      for (int e = tid; e < BM * (BK / 4); e += kSimtThreads) {
        int r = e / (BK / 4), cq = e % (BK / 4);
        int src = nb[r];
        int c = c0 + 4 * cq;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (src >= 0 && c < c_in) {
          const float *p = features + (long long)src * c_in + c;
          if (vec_a && c + 3 < c_in) {
            v = __ldg(reinterpret_cast<const float4 *>(p));
          } else {
            v.x = __ldg(p);
            if (c + 1 < c_in) v.y = __ldg(p + 1);
            if (c + 2 < c_in) v.z = __ldg(p + 2);
            if (c + 3 < c_in) v.w = __ldg(p + 3);
          }
        }
        As[4 * cq + 0][r] = v.x;
        As[4 * cq + 1][r] = v.y;
        As[4 * cq + 2][r] = v.z;
        As[4 * cq + 3][r] = v.w;
      }
      // B tile: W[k][c0 .. c0+BK) x [0 .. BN)
      for (int e = tid; e < BK * (BN / 4); e += kSimtThreads) {
        int kk = e / (BN / 4), nq = e % (BN / 4);
        int c = c0 + kk, n = 4 * nq;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c < c_in && n < c_out) {
          const float *p = wk + (long long)c * c_out + n;
          if (vec_b && n + 3 < c_out) {
            v = __ldg(reinterpret_cast<const float4 *>(p));
          } else {
            v.x = __ldg(p);
            if (n + 1 < c_out) v.y = __ldg(p + 1);
            if (n + 2 < c_out) v.z = __ldg(p + 2);
            if (n + 3 < c_out) v.w = __ldg(p + 3);
          }
        }
        *reinterpret_cast<float4 *>(&Bs[kk][n]) = v;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        float4 a4 = *reinterpret_cast<const float4 *>(&As[kk][ty * TM]);
        float a[TM] = {a4.x, a4.y, a4.z, a4.w};
        float b[TN];
#pragma unroll
        for (int j4 = 0; j4 < TN / 4; ++j4) {
          float4 b4 = *reinterpret_cast<const float4 *>(&Bs[kk][tx * TN + 4 * j4]);
          b[4 * j4 + 0] = b4.x; b[4 * j4 + 1] = b4.y; b[4 * j4 + 2] = b4.z; b[4 * j4 + 3] = b4.w;
        }
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }

  // epilogue: folded BN (scale, shift) -> + residual -> ReLU -> store
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int o = row0 + ty * TM + i;
    if (o >= n_out) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int c = tx * TN + j;
      if (c >= c_out) continue;
      float y = acc[i][j];
      if (scale) y = y * __ldg(scale + c);
      if (shift) y = y + __ldg(shift + c);
      if (residual) y += __ldg(residual + (long long)o * c_out + c);
      if (relu) y = fmaxf(y, 0.f);
      out[(long long)o * c_out + c] = y;
    }
  }
}

template <int BN, int TN>
static int launch_simt(const float *features, const float *weight, const int32_t *nbr, int n_in,
                       int n_out, int c_in, int c_out, int kvol, const float *scale,
                       const float *shift, const float *residual, int relu, float *out,
                       cudaStream_t st) {
  constexpr int BM = (kSimtThreads / (BN / TN)) * 4;
  int grid = (n_out + BM - 1) / BM;
  BEVB200_LAUNCH((spconv_simt_kernel<BN, TN>), grid, kSimtThreads, 0, st, features, weight, nbr,
                 n_in, n_out, c_in, c_out, kvol, scale, shift, residual, relu, out);
  return BEVB200_OK;
}

int spconv_forward_simt(const float *features, const float *weight, const int32_t *nbr, int n_in,
                        int n_out, int c_in, int c_out, int kvol, const float *scale,
                        const float *shift, const float *residual, int relu, float *out,
                        cudaStream_t st) {
  if (c_out <= 16)
    return launch_simt<16, 4>(features, weight, nbr, n_in, n_out, c_in, c_out, kvol, scale, shift,
                              residual, relu, out, st);
  if (c_out <= 32)
    return launch_simt<32, 4>(features, weight, nbr, n_in, n_out, c_in, c_out, kvol, scale, shift,
                              residual, relu, out, st);
  if (c_out <= 64)
    return launch_simt<64, 4>(features, weight, nbr, n_in, n_out, c_in, c_out, kvol, scale, shift,
                              residual, relu, out, st);
  if (c_out <= 128)
    return launch_simt<128, 8>(features, weight, nbr, n_in, n_out, c_in, c_out, kvol, scale, shift,
                               residual, relu, out, st);
  snprintf(g_last_error, sizeof(g_last_error), "spconv_forward: c_out %d > 128 unsupported", c_out);
  return BEVB200_EUNSUPPORTED;
}

}  // namespace bevb200
