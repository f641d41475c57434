// Sparse convolution backward (fp32) for sm_90a.
//
// Replaces spconv::indiceConvBackward<float> (spconv_ops.h:363-456): per kernel offset the
// reference gathers features and out-grad rows, runs two cuBLAS GEMMs (filtersGrad[k] = in^T dout,
// inBuf = dout W[k]^T) and scatter-adds inBuf into inputGrad.  Here:
//   * input gradient  = ONE implicit-GEMM launch of the forward kernel on the transposed
//     neighbour table (nbrT[k, j] = output row fed by input row j through offset k) with the
//     per-offset transposed weights:  dIn[j] = sum_k dOut[nbrT[k, j]] @ W[k]^T
//   * weight gradient = two kernels, NO atomics: CTA (offset k, fixed chunk of 2048 output rows)
//     accumulates the Cin x Cout outer-product sum of its chunk in registers and stores it as a
//     partial; a second kernel adds the partials of every element in ascending chunk order.  The
//     result is bit-reproducible run to run (the reference's cuBLAS GEMM per offset is too; the
//     round-1 version with fp32 atomicAdd was not).
#include "spconv.cuh"

namespace bevb200 {

__global__ void nbr_transpose_kernel(const int32_t *__restrict__ nbr, int kvol, int n_out, int n_in,
                                     int32_t *__restrict__ nbr_t) {
  const long long total = (long long)kvol * n_out;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(t / n_out), o = (int)(t % n_out);
    const int j = nbr[t];
    if (j >= 0 && j < n_in) nbr_t[(long long)k * n_in + j] = o;   // unique writer per (k, j)
  }
}

__global__ void weight_transpose_kernel(const float *__restrict__ w, int kvol, int c_in, int c_out,
                                        float *__restrict__ wt) {
  const long long total = (long long)kvol * c_in * c_out;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(t % c_out), ci = (int)((t / c_out) % c_in), k = (int)(t / ((long long)c_out * c_in));
    wt[((long long)k * c_out + co) * c_in + ci] = w[t];
  }
}

// dW[k][ci][co] += sum over output rows o of the chunk with j = nbr[k, o] >= 0 of f[j][ci] * g[o][co]
constexpr int kWgChunk = 2048;   // output rows per CTA
constexpr int kWgStep = 16;      // rows staged per step
template <int TCI, int TCO>     // per-thread micro-tile; 256 threads cover (16*TCI) x (16*TCO)
__global__ void __launch_bounds__(256)
    spconv_wgrad_kernel(const float *__restrict__ features, const float *__restrict__ out_grad,
                        const int32_t *__restrict__ nbr, int n_in, int n_out, int c_in, int c_out,
                        float *__restrict__ partial) {   // [chunk][k][c_in][c_out]
  constexpr int BCI = 16 * TCI, BCO = 16 * TCO;
  __shared__ float fs[kWgStep][BCI + 1];
  __shared__ float gs[kWgStep][BCO + 1];
  __shared__ int js[kWgStep];
  const int k = blockIdx.y;
  const int o_begin = blockIdx.x * kWgChunk, o_end = min(n_out, o_begin + kWgChunk);
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  for (int ci0 = 0; ci0 < c_in; ci0 += BCI) {
    for (int co0 = 0; co0 < c_out; co0 += BCO) {
      float acc[TCI][TCO];
#pragma unroll
      for (int a = 0; a < TCI; ++a)
#pragma unroll
        for (int b = 0; b < TCO; ++b) acc[a][b] = 0.f;
      for (int o0 = o_begin; o0 < o_end; o0 += kWgStep) {
        if (tid < kWgStep) {
          const int o = o0 + tid;
          int j = o < o_end ? __ldg(nbr + (long long)k * n_out + o) : -1;
          js[tid] = (j >= 0 && j < n_in) ? j : -1;
        }
        __syncthreads();
        for (int e = tid; e < kWgStep * BCI; e += 256) {
          const int r = e / BCI, c = e % BCI, j = js[r];
          fs[r][c] = (j >= 0 && ci0 + c < c_in) ? __ldg(features + (long long)j * c_in + ci0 + c) : 0.f;
        }
        for (int e = tid; e < kWgStep * BCO; e += 256) {
          const int r = e / BCO, c = e % BCO, o = o0 + r;
          gs[r][c] = (js[r] >= 0 && co0 + c < c_out) ? __ldg(out_grad + (long long)o * c_out + co0 + c) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < kWgStep; ++r) {
          float fa[TCI], gb[TCO];
#pragma unroll
          for (int a = 0; a < TCI; ++a) fa[a] = fs[r][ty * TCI + a];
#pragma unroll
          for (int b = 0; b < TCO; ++b) gb[b] = gs[r][tx * TCO + b];
#pragma unroll
          for (int a = 0; a < TCI; ++a)
#pragma unroll
            for (int b = 0; b < TCO; ++b) acc[a][b] = fmaf(fa[a], gb[b], acc[a][b]);
        }
        __syncthreads();
      }
#pragma unroll
      for (int a = 0; a < TCI; ++a)
#pragma unroll
        for (int b = 0; b < TCO; ++b) {
          const int ci = ci0 + ty * TCI + a, co = co0 + tx * TCO + b;
          if (ci < c_in && co < c_out)
            partial[(((long long)blockIdx.x * gridDim.y + k) * c_in + ci) * c_out + co] = acc[a][b];
        }
    }
  }
}

// Round-2 filter-gradient kernel for the encoder's channel counts (16 / 32 / 64 / 128 on both sides): ONE pass over
// the chunk's rows for the whole Cin x Cout tile (the generic kernel above re-reads the rows once per 64 x 64 block and
// synchronises every 16 rows).  256 threads as a 16 x 16 grid, thread tile TCI x TCO = (Cin/16) x (Cout/16); 32 rows
// of features (gathered through nbr) and of out-grad are staged per step; rows without a neighbour are staged as zeros.
constexpr int kWg2Step = 32;
template <int TCI, int TCO>
__global__ void __launch_bounds__(256)
    spconv_wgrad2_kernel(const float *__restrict__ features, const float *__restrict__ out_grad,
                         const int32_t *__restrict__ nbr, int n_in, int n_out, float *__restrict__ partial) {
  constexpr int CI = 16 * TCI, CO = 16 * TCO;
  __shared__ __align__(16) float fs[kWg2Step][CI];
  __shared__ __align__(16) float gs[kWg2Step][CO];
  __shared__ int js[kWg2Step];
  const int k = blockIdx.y;
  const int o_begin = blockIdx.x * kWgChunk, o_end = min(n_out, o_begin + kWgChunk);
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  float acc[TCI][TCO];
#pragma unroll
  for (int a = 0; a < TCI; ++a)
#pragma unroll
    for (int b = 0; b < TCO; ++b) acc[a][b] = 0.f;
  for (int o0 = o_begin; o0 < o_end; o0 += kWg2Step) {
    if (tid < kWg2Step) {
      const int o = o0 + tid;
      const int j = o < o_end ? __ldg(nbr + (long long)k * n_out + o) : -1;
      js[tid] = (j >= 0 && j < n_in) ? j : -1;
    }
    __syncthreads();
    for (int e = tid; e < kWg2Step * (CI / 4); e += 256) {
      const int r = e / (CI / 4), c4 = e % (CI / 4), j = js[r];
      const float4 v = j >= 0 ? __ldg(reinterpret_cast<const float4 *>(features + (long long)j * CI) + c4)
                              : make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4 *>(&fs[r][4 * c4]) = v;
    }
    for (int e = tid; e < kWg2Step * (CO / 4); e += 256) {
      const int r = e / (CO / 4), c4 = e % (CO / 4);
      const float4 v = js[r] >= 0 ? __ldg(reinterpret_cast<const float4 *>(out_grad + (long long)(o0 + r) * CO) + c4)
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4 *>(&gs[r][4 * c4]) = v;
    }
    __syncthreads();
#pragma unroll 4
    for (int r = 0; r < kWg2Step; ++r) {
      float fa[TCI], gb[TCO];
#pragma unroll
      for (int a = 0; a < TCI; ++a) fa[a] = fs[r][ty * TCI + a];
#pragma unroll
      for (int b = 0; b < TCO; ++b) gb[b] = gs[r][tx * TCO + b];
#pragma unroll
      for (int a = 0; a < TCI; ++a)
#pragma unroll
        for (int b = 0; b < TCO; ++b) acc[a][b] = fmaf(fa[a], gb[b], acc[a][b]);
    }
    __syncthreads();
  }
  float *dst = partial + ((long long)blockIdx.x * gridDim.y + k) * CI * CO;
#pragma unroll
  for (int a = 0; a < TCI; ++a)
#pragma unroll
    for (int b = 0; b < TCO; ++b) dst[(ty * TCI + a) * CO + tx * TCO + b] = acc[a][b];
}

// dW[e] = sum over chunks (ascending) of partial[chunk][e]
__global__ void spconv_wgrad_reduce_kernel(const float *__restrict__ partial, long long elems, int n_chunks,
                                           float *__restrict__ w_grad) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < elems; e += (long long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int ch = 0; ch < n_chunks; ++ch) s += partial[(long long)ch * elems + e];
    w_grad[e] = s;
  }
}

int spconv_wgrad_reduce(const float *partial, long long elems, int n_chunks, float *weight_grad, cudaStream_t st) {
  BEVB200_LAUNCH(spconv_wgrad_reduce_kernel, grid_for(elems, 256), 256, 0, st, partial, elems, n_chunks, weight_grad);
  return BEVB200_OK;
}

}  // namespace bevb200

using namespace bevb200;

extern "C" {

int bevb200_rulebook_transpose(const int32_t *nbr, int kernel_volume, int n_out, int n_in,
                               int32_t *nbr_t, void *stream) {
  BEVB200_REQUIRE(kernel_volume > 0 && n_out >= 0 && n_in >= 0, "bad sizes");
  if (n_in == 0) return BEVB200_OK;
  BEVB200_REQUIRE(nbr_t != nullptr, "null nbr_t");
  cudaStream_t st = (cudaStream_t)stream;
  BEVB200_CUDA(cudaMemsetAsync(nbr_t, 0xff, (size_t)kernel_volume * n_in * sizeof(int32_t), st));
  if (n_out == 0) return BEVB200_OK;
  BEVB200_REQUIRE(nbr != nullptr, "null nbr");
  BEVB200_LAUNCH(nbr_transpose_kernel, grid_for((long long)kernel_volume * n_out, 256), 256, 0, st, nbr,
                 kernel_volume, n_out, n_in, nbr_t);
  return BEVB200_OK;
}

size_t bevb200_spconv_backward_workspace_bytes(int n_in, int n_out, int c_in, int c_out, int kernel_volume) {
  if (n_in < 0 || n_out < 0 || c_in <= 0 || c_out <= 0 || kernel_volume <= 0) return 0;
  const size_t w = align_up((size_t)kernel_volume * c_in * c_out * sizeof(float));
  const size_t chunks = ((size_t)n_out + kWgChunk - 1) / kWgChunk;
  const size_t simt = w * (chunks ? chunks : 1);          // one partial dW per chunk of output rows
  const size_t tc = spconv_wgrad_tc_workspace_bytes(n_in, n_out, c_in, c_out, kernel_volume);   // split images + partials
  const size_t pk = align_up(spconv_v6_packed_bytes(c_out, c_in, kernel_volume));   // W^T image of the input gradient
  return w + (simt > tc ? simt : tc) + pk;                // transposed weights + the larger of the two + that image
}

int bevb200_spconv_backward(const float *features, const float *weight, const float *out_grad,
                            const int32_t *nbr, const int32_t *nbr_t, int n_in, int n_out, int c_in,
                            int c_out, int kernel_volume, int precision, float *input_grad,
                            float *weight_grad, void *workspace, size_t workspace_bytes,
                            void *stream) {
  BEVB200_REQUIRE(n_in >= 0 && n_out >= 0 && c_in > 0 && c_out > 0 && kernel_volume > 0, "bad sizes");
  BEVB200_REQUIRE(weight && weight_grad, "null weight");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t wbytes = (size_t)kernel_volume * c_in * c_out * sizeof(float);
  BEVB200_CUDA(cudaMemsetAsync(weight_grad, 0, wbytes, st));
  if (n_in == 0) return BEVB200_OK;
  BEVB200_REQUIRE(input_grad != nullptr, "null input_grad");
  if (n_out == 0) {
    BEVB200_CUDA(cudaMemsetAsync(input_grad, 0, (size_t)n_in * c_in * sizeof(float), st));
    return BEVB200_OK;
  }
  BEVB200_REQUIRE(features && out_grad && nbr && nbr_t, "null argument");
  if (workspace == nullptr ||
      workspace_bytes < bevb200_spconv_backward_workspace_bytes(n_in, n_out, c_in, c_out, kernel_volume)) {
    snprintf(g_last_error, sizeof(g_last_error), "spconv_backward: workspace too small");
    return BEVB200_EWORKSPACE;
  }
  // dIn = sparse_conv(dOut, W^T, nbrT)
  float *wt = (float *)workspace;
  BEVB200_LAUNCH(weight_transpose_kernel, grid_for((long long)kernel_volume * c_in * c_out, 256), 256, 0,
                 st, weight, kernel_volume, c_in, c_out, wt);
  int rc;
  const bool tc_wgrad = (precision == BEVB200_PREC_BF16X3 || precision == BEVB200_PREC_TF32) &&
                        spconv_wgrad_tc_ok(c_in, c_out, kernel_volume) && (uintptr_t)features % 16 == 0 &&
                        (uintptr_t)out_grad % 16 == 0;
  char *tc_ws = (char *)workspace + align_up(wbytes);
  // One split of out_grad serves both gradients when the filter gradient's out-grad image is the generation-6 row
  // image (c_out = 32 / 64 / 128) and the input gradient runs on split images: dW first, then dIn gathers from it.
  if (tc_wgrad && (c_out == 32 || c_out == 64 || c_out == 128) &&
      spconv_forward_path(precision, c_out, c_in, kernel_volume, false, out_grad, input_grad, nullptr) ==
          FwdPath::kSplit) {
    rc = spconv_wgrad_tc(features, out_grad, nbr, n_in, n_out, c_in, c_out, kernel_volume, weight_grad, tc_ws, st);
    if (rc) return rc;
    void *packed = tc_ws + spconv_wgrad_tc_workspace_bytes(n_in, n_out, c_in, c_out, kernel_volume);
    rc = spconv_v6_pack_weights(wt, c_out, c_in, kernel_volume, packed, st);
    if (rc) return rc;
    return spconv_v6_forward(spconv_wgrad_tc_grad_image(tc_ws, n_in, c_in), packed, nbr_t, n_in, n_out, n_in, nullptr, c_out,
                             c_in, kernel_volume, nullptr, nullptr, nullptr, nullptr, 0, input_grad, nullptr, st);
  }
  rc = spconv_forward(out_grad, wt, nullptr, nbr_t, n_out, n_in, c_out, c_in, kernel_volume, nullptr, nullptr, nullptr,
                      0, precision, input_grad, st);
  if (rc) return rc;
  // dW on the tensor cores (spconv_wgrad_tc.cu) for the tensor-core precisions and channel counts 32 / 64 / 128 ...
  if (tc_wgrad)
    return spconv_wgrad_tc(features, out_grad, nbr, n_in, n_out, c_in, c_out, kernel_volume, weight_grad, tc_ws, st);
  // ... else SIMT: per-chunk partials, then an ordered reduction (no atomics)
  const int n_chunks = (n_out + kWgChunk - 1) / kWgChunk;
  float *partial = (float *)((char *)workspace + align_up(wbytes));
  dim3 grid(n_chunks, kernel_volume);
  auto pow16 = [](int c) { return c == 16 || c == 32 || c == 64 || c == 128; };
  const bool aligned = (uintptr_t)features % 16 == 0 && (uintptr_t)out_grad % 16 == 0;
#define WG2(TI, TO)                                                                                            \
  BEVB200_LAUNCH((spconv_wgrad2_kernel<TI, TO>), grid, 256, 0, st, features, out_grad, nbr, n_in, n_out, partial)
  if (pow16(c_in) && pow16(c_out) && aligned) {
    const int key = (c_in / 16) * 16 + c_out / 16;
    switch (key) {
      case 1 * 16 + 1: WG2(1, 1); break;
      case 1 * 16 + 2: WG2(1, 2); break;
      case 2 * 16 + 1: WG2(2, 1); break;
      case 2 * 16 + 2: WG2(2, 2); break;
      case 2 * 16 + 4: WG2(2, 4); break;
      case 4 * 16 + 2: WG2(4, 2); break;
      case 4 * 16 + 4: WG2(4, 4); break;
      case 4 * 16 + 8: WG2(4, 8); break;
      case 8 * 16 + 4: WG2(8, 4); break;
      case 8 * 16 + 8: WG2(8, 8); break;
      default:
        BEVB200_LAUNCH((spconv_wgrad_kernel<2, 2>), grid, 256, 0, st, features, out_grad, nbr, n_in, n_out, c_in,
                       c_out, partial);
    }
  } else if (c_in >= 64 && c_out >= 64) {
    BEVB200_LAUNCH((spconv_wgrad_kernel<4, 4>), grid, 256, 0, st, features, out_grad, nbr, n_in, n_out,
                   c_in, c_out, partial);
  } else if (c_in >= 32 && c_out >= 32) {
    BEVB200_LAUNCH((spconv_wgrad_kernel<2, 2>), grid, 256, 0, st, features, out_grad, nbr, n_in, n_out,
                   c_in, c_out, partial);
  } else {
    BEVB200_LAUNCH((spconv_wgrad_kernel<1, 1>), grid, 256, 0, st, features, out_grad, nbr, n_in, n_out,
                   c_in, c_out, partial);
  }
#undef WG2
  return spconv_wgrad_reduce(partial, (long long)kernel_volume * c_in * c_out, n_chunks, weight_grad, st);
}

}  // extern "C"
