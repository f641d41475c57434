// Sparse convolution: every function one spconv translation unit (or encoder.cu) calls in another.  Internal header.
//
//   spconv_fwd.cu       forward C ABI, the path decision, the TF32 weight image
//   spconv_simt.cu      exact-fp32 SIMT forward kernel
//   spconv_v6.cu        tensor-core forward kernels (mma.sync, wgmma) and the BF16x3 operand images
//   spconv_bwd.cu       backward C ABI, SIMT filter-gradient kernels, the ordered partial reduction
//   spconv_wgrad_tc.cu  tensor-core filter gradient
#pragma once
#include "common.cuh"

namespace bevb200 {

// ---- spconv_fwd.cu ---------------------------------------------------------------------------
// The kernels one forward call runs on.
enum class FwdPath {
  kSimt,    // exact-fp32 SIMT kernel: BEVB200_PREC_FP32 and every shape / alignment the tensor cores cannot take
  kSplit,   // BF16X3 on split images of the rows and weights, built in stream-ordered temporaries
  kTf32,    // TF32 / 3xTF32 on fp32 rows, zero-padded into a temporary when c_in is not a power of two >= 8
  kNone,    // the weights come packed, but only the SIMT kernel (which takes unpacked weights) can run the call
};
FwdPath spconv_forward_path(int precision, int c_in, int c_out, int kvol, bool packed, const float *features,
                            const float *out, const float *residual);
// One forward on the path above; exactly one of weight ([kvol][c_in][c_out]) and packed (the image of
// bevb200_spconv_pack_weights) is given.
int spconv_forward(const float *features, const float *weight, const float *packed, const int32_t *nbr, int n_in,
                   int n_out, int c_in, int c_out, int kvol, const float *scale, const float *shift,
                   const float *residual, int relu, int precision, float *out, cudaStream_t st);

// ---- spconv_simt.cu --------------------------------------------------------------------------
// any c_in, c_out <= 128 (BEVB200_EUNSUPPORTED above)
int spconv_forward_simt(const float *features, const float *weight, const int32_t *nbr, int n_in, int n_out,
                        int c_in, int c_out, int kvol, const float *scale, const float *shift, const float *residual,
                        int relu, float *out, cudaStream_t st);

// ---- spconv_v6.cu ----------------------------------------------------------------------------
// channels of a split-image row: c_in rounded up to 16 / 32 / 64 / 128; 0 above 128
int spconv_v6_cin_eff(int c_in);
// c_out in {16, 32, 64, 128}, 1 <= c_in <= 128, 1 <= kvol <= 27
bool spconv_v6_shape_ok(int c_in, int c_out, int kvol);
size_t spconv_v6_packed_bytes(int c_in, int c_out, int kvol);
int spconv_v6_pack_weights(const float *weight, int c_in, int c_out, int kvol, void *packed, cudaStream_t st);
// fp32 rows [n, c_in] -> split image [n, c_eff * 4 B] (c_eff a multiple of 16, >= c_in; zero padded), where
// n = min(n_cap, *n_dev), or n_cap when n_dev is null
int spconv_v6_split_rows(const float *features, int n_cap, const int32_t *n_dev, int c_in, int c_eff, void *split,
                         cudaStream_t st);
// BF16X3 forward on a split image with c_in (a multiple of 16, <= 128) channels per row.  The residual comes as fp32
// rows or as a split image (residual_split), at most one of the two; out and / or out_split receive the result.
int spconv_v6_forward(const void *features_split, const void *packed, const int32_t *nbr, long long nbr_stride,
                      int n_in, int n_out, const int32_t *n_out_dev, int c_in, int c_out, int kvol, const float *scale,
                      const float *shift, const float *residual, const void *residual_split, int relu, float *out,
                      void *out_split, cudaStream_t st);
// TF32 (tf32x3 = false) / 3xTF32 forward on fp32 rows [n_in][c_in], c_in a power of two 8 .. 128
int spconv_v6_forward_tf32(const float *rows, const void *packed, const int32_t *nbr, int n_in, int n_out, int c_in,
                           int c_out, int kvol, bool tf32x3, const float *scale, const float *shift,
                           const float *residual, int relu, float *out, cudaStream_t st);

// ---- spconv_wgrad_tc.cu ----------------------------------------------------------------------
// the shapes the tensor-core filter gradient takes (and BEVB200_WGRAD_TC is not 0)
bool spconv_wgrad_tc_ok(int c_in, int c_out, int kvol);
size_t spconv_wgrad_tc_workspace_bytes(int n_in, int n_out, int c_in, int c_out, int kvol);
int spconv_wgrad_tc(const float *features, const float *out_grad, const int32_t *nbr, int n_in, int n_out, int c_in,
                    int c_out, int kvol, float *weight_grad, void *workspace, cudaStream_t st);
// the split image of out_grad that spconv_wgrad_tc() leaves in its workspace
const void *spconv_wgrad_tc_grad_image(const void *workspace, int n_in, int c_in);

// ---- spconv_bwd.cu ---------------------------------------------------------------------------
// weight_grad[e] = sum over the chunks, in ascending order, of partial[chunk][e]: bit-reproducible
int spconv_wgrad_reduce(const float *partial, long long elems, int n_chunks, float *weight_grad, cudaStream_t st);

}  // namespace bevb200
