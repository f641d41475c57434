// Sparse convolution forward: the C ABI, the choice of kernels for a call, and the TF32 weight image.
//
//   out[o, :] = epilogue( sum_k features[nbr[k, o], :] @ W[k] )          (spconv_ops.h:260-361)
//
// spconv_forward_path() picks the kernels of every forward call, and of the input gradient of
// bevb200_spconv_backward, from the precision, the shape, the pointer alignments and whether the weights come packed:
//   * BEVB200_PREC_FP32, and whatever the tensor cores cannot take: the exact-fp32 SIMT kernel (spconv_simt.cu);
//   * BEVB200_PREC_BF16X3 (default; ~5e-6 .. 1e-5 of max|out| vs the float64 oracle): the mma.sync / wgmma kernels of
//     spconv_v6.cu on the bf16 hi|lo images of the rows and weights, built here in stream-ordered temporaries;
//   * BEVB200_PREC_TF32X3 (1e-6 .. 1e-5) and BEVB200_PREC_TF32 (single pass, ~8e-4: below the 1e-4 parity bar,
//     measurement only): the mma.sync kernel of spconv_v6.cu on zero-padded fp32 rows and the tf32 weight image
//     packed here; it splits the rows into tf32 hi / lo in registers.
#include "spconv.cuh"

namespace bevb200 {

constexpr int kKBlock = 32;                       // channels per K block = one 128-byte row line

// weight [K][Cin][Cout] fp32 -> packed [nkb][nsplit][Cout][32] in the swizzled smem image.  The K
// axis is the concatenation over kernel offsets of the Cin channels (kk = k*Cin + ci), cut into
// blocks of 32; element (n, c) of block kb sits at float index n*32 + (((c/4) ^ (n&7)) * 4) + (c%4).
// c_in_eff >= c_in is the (zero-padded) channel count the kernel runs with.
__global__ void spconv_pack_weights_kernel(const float *__restrict__ w, int kvol, int c_in, int c_in_eff,
                                           int c_out, int nkb, int nsplit, float *__restrict__ packed) {
  const long long total = (long long)nkb * c_out * 32;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(t % 32);
    const int n = (int)((t / 32) % c_out);
    const int kb = (int)(t / (32ll * c_out));
    const int kk = kb * 32 + c;
    const int k = kk / c_in_eff, ci = kk % c_in_eff;
    const float v = (k < kvol && ci < c_in) ? w[((long long)k * c_in + ci) * c_out + n] : 0.f;
    const float hi = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
    const long long blk = (long long)kb * nsplit;
    const int pos = n * 32 + ((((c >> 2) ^ (n & 7)) << 2) | (c & 3));
    packed[(blk + 0) * c_out * 32 + pos] = hi;
    if (nsplit == 2) packed[(blk + 1) * c_out * 32 + pos] = v - hi;
  }
}

// [n, c_in] -> [n, c_eff] rows, zero padded (c_eff a multiple of 4: 16-byte aligned rows)
__global__ void spconv_pad_rows_kernel(const float *__restrict__ in, int n, int c_in, int c_eff,
                                       float *__restrict__ out) {
  const long long total = (long long)n * (c_eff / 4);
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int g4 = (int)(t % (c_eff / 4));
    const long long r = t / (c_eff / 4);
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = 4 * g4 + e < c_in ? in[r * c_in + 4 * g4 + e] : 0.f;
    *reinterpret_cast<float4 *>(out + r * c_eff + 4 * g4) = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// Input channels the TF32 modes run with: zero-padded to the next power of two, 8 .. 128 (conv_input: Cin = 5 -> 8).
// 0 = no tensor-core form.
static int tc_cin_eff(int c_in) {
  for (int e = 8; e <= 128; e <<= 1)
    if (c_in <= e) return e;
  return 0;
}

static int tc_nkb(int c_in_eff, int kvol) { return (kvol * c_in_eff + kKBlock - 1) / kKBlock; }

// The weight image of a (shape, precision) that bevb200_spconv_packed_weight_bytes() gives a size.
static int pack_weights(const float *weight, int c_in, int c_out, int kvol, int precision, void *packed,
                        cudaStream_t st) {
  if (precision == BEVB200_PREC_BF16X3) return spconv_v6_pack_weights(weight, c_in, c_out, kvol, packed, st);
  const int nsplit = precision == BEVB200_PREC_TF32X3 ? 2 : 1;
  const int ce = tc_cin_eff(c_in);
  const int nkb = tc_nkb(ce, kvol);
  BEVB200_LAUNCH(spconv_pack_weights_kernel, grid_for((long long)nkb * c_out * 32, 256), 256, 0, st,
                 weight, kvol, c_in, ce, c_out, nkb, nsplit, (float *)packed);
  return BEVB200_OK;
}

FwdPath spconv_forward_path(int precision, int c_in, int c_out, int kvol, bool packed, const float *features,
                            const float *out, const float *residual) {
  const bool aligned = (uintptr_t)out % 16 == 0 && (residual == nullptr || (uintptr_t)residual % 16 == 0);
  if (aligned && spconv_v6_shape_ok(c_in, c_out, kvol)) {
    // the split pass and the pad kernel read rows at any alignment; the TF32 kernel gathers unpadded rows directly
    if (precision == BEVB200_PREC_BF16X3) return FwdPath::kSplit;
    if ((precision == BEVB200_PREC_TF32X3 || precision == BEVB200_PREC_TF32) &&
        (tc_cin_eff(c_in) != c_in || (uintptr_t)features % 16 == 0))
      return FwdPath::kTf32;
  }
  return packed ? FwdPath::kNone : FwdPath::kSimt;
}

int spconv_forward(const float *features, const float *weight, const float *packed, const int32_t *nbr, int n_in,
                   int n_out, int c_in, int c_out, int kvol, const float *scale, const float *shift,
                   const float *residual, int relu, int precision, float *out, cudaStream_t st) {
  const FwdPath path = spconv_forward_path(precision, c_in, c_out, kvol, packed != nullptr, features, out, residual);
  if (path == FwdPath::kSimt)
    return spconv_forward_simt(features, weight, nbr, n_in, n_out, c_in, c_out, kvol, scale, shift, residual, relu,
                               out, st);
  if (path == FwdPath::kNone) {
    snprintf(g_last_error, sizeof(g_last_error), "spconv_forward: shape needs the unpacked weights");
    return BEVB200_EINVAL;
  }
  // stream-ordered temporaries, released on every exit path
  struct Temps {
    cudaStream_t st;
    void *rows = nullptr, *weights = nullptr;
    ~Temps() {
      if (weights) cudaFreeAsync(weights, st);
      if (rows) cudaFreeAsync(rows, st);
    }
  } tmp;
  tmp.st = st;
  // The operand rows: BF16X3 consumes their split image (SparseEncoder's fused path never comes here: its convs hand
  // the image to each other, bevb200_encoder_forward); the TF32 modes take fp32 rows, zero-padded when c_in is not a
  // power of two (e.g. conv_input: Cin = 5 -> 8).
  const bool split = path == FwdPath::kSplit;
  const int c_eff = split ? spconv_v6_cin_eff(c_in) : tc_cin_eff(c_in);
  if (split || c_eff != c_in) {
    BEVB200_CUDA(cudaMallocAsync(&tmp.rows, (size_t)(n_in > 0 ? n_in : 1) * c_eff * 4, st));
    if (split) {
      const int rc = spconv_v6_split_rows(features, n_in, nullptr, c_in, c_eff, tmp.rows, st);
      if (rc) return rc;
    } else if (n_in > 0) {
      BEVB200_LAUNCH(spconv_pad_rows_kernel, grid_for((long long)n_in * (c_eff / 4), 256), 256, 0, st, features,
                     n_in, c_in, c_eff, (float *)tmp.rows);
    }
  }
  if (packed == nullptr) {
    BEVB200_CUDA(cudaMallocAsync(&tmp.weights, bevb200_spconv_packed_weight_bytes(c_in, c_out, kvol, precision), st));
    const int rc = pack_weights(weight, c_in, c_out, kvol, precision, tmp.weights, st);
    if (rc) return rc;
  }
  const void *rows = tmp.rows ? tmp.rows : features;
  const void *wimage = packed ? packed : tmp.weights;
  if (split)
    return spconv_v6_forward(rows, wimage, nbr, n_out, n_in, n_out, nullptr, c_eff, c_out, kvol, scale, shift,
                             residual, nullptr, relu, out, nullptr, st);
  return spconv_v6_forward_tf32((const float *)rows, wimage, nbr, n_in, n_out, c_eff, c_out, kvol,
                                precision == BEVB200_PREC_TF32X3, scale, shift, residual, relu, out, st);
}

}  // namespace bevb200

using namespace bevb200;

extern "C" {

int bevb200_spconv_forward(const float *features, const float *weight, const int32_t *nbr,
                           int n_in, int n_out, int c_in, int c_out, int kernel_volume,
                           const float *scale, const float *shift, const float *residual,
                           int relu, int precision, float *out, void *stream) {
  BEVB200_REQUIRE(n_in >= 0 && n_out >= 0 && c_in > 0 && c_out > 0 && kernel_volume > 0,
                  "bad sizes");
  if (n_out == 0) return BEVB200_OK;
  BEVB200_REQUIRE(weight && nbr && out, "null argument");
  BEVB200_REQUIRE(features != nullptr || n_in == 0, "null features");
  BEVB200_REQUIRE(precision == BEVB200_PREC_FP32 || precision == BEVB200_PREC_TF32X3 ||
                      precision == BEVB200_PREC_TF32 || precision == BEVB200_PREC_BF16X3,
                  "unknown precision mode");
  return spconv_forward(features, weight, nullptr, nbr, n_in, n_out, c_in, c_out, kernel_volume, scale, shift,
                        residual, relu, precision, out, (cudaStream_t)stream);
}

int bevb200_spconv_padded_channels(int c_in, int precision) {
  // BF16X3: the split pass pads
  if (precision == BEVB200_PREC_FP32 || precision == BEVB200_PREC_BF16X3 || c_in < 1) return c_in;
  const int e = tc_cin_eff(c_in);
  return e ? e : c_in;
}

size_t bevb200_spconv_packed_weight_bytes(int c_in, int c_out, int kernel_volume, int precision) {
  if (!spconv_v6_shape_ok(c_in, c_out, kernel_volume)) return 0;
  if (precision == BEVB200_PREC_BF16X3) return spconv_v6_packed_bytes(c_in, c_out, kernel_volume);
  if (precision != BEVB200_PREC_TF32X3 && precision != BEVB200_PREC_TF32) return 0;
  const int nsplit = precision == BEVB200_PREC_TF32X3 ? 2 : 1;
  return (size_t)tc_nkb(tc_cin_eff(c_in), kernel_volume) * nsplit * c_out * 32 * sizeof(float);
}

int bevb200_spconv_pack_weights(const float *weight, int c_in, int c_out, int kernel_volume,
                                int precision, float *packed, void *stream) {
  BEVB200_REQUIRE(weight && packed, "null argument");
  BEVB200_REQUIRE(bevb200_spconv_packed_weight_bytes(c_in, c_out, kernel_volume, precision) > 0,
                  "shape / precision has no packed form");
  return pack_weights(weight, c_in, c_out, kernel_volume, precision, packed, (cudaStream_t)stream);
}

int bevb200_spconv_forward_packed(const float *features, const float *packed_weight,
                                  const int32_t *nbr, int n_in, int n_out, int c_in, int c_out,
                                  int kernel_volume, const float *scale, const float *shift,
                                  const float *residual, int relu, int precision, float *out,
                                  void *stream) {
  BEVB200_REQUIRE(n_in >= 0 && n_out >= 0 && c_in > 0 && c_out > 0 && kernel_volume > 0,
                  "bad sizes");
  if (n_out == 0) return BEVB200_OK;
  BEVB200_REQUIRE(packed_weight && nbr && out, "null argument");
  BEVB200_REQUIRE(bevb200_spconv_packed_weight_bytes(c_in, c_out, kernel_volume, precision) > 0,
                  "shape / precision has no packed form");
  return spconv_forward(features, nullptr, packed_weight, nbr, n_in, n_out, c_in, c_out, kernel_volume, scale,
                        shift, residual, relu, precision, out, (cudaStream_t)stream);
}

}  // extern "C"
