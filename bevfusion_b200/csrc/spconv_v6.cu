// Sparse convolution forward on the Hopper tensor cores, BF16x3, FP16 and TF32 precisions: a warp-specialised wgmma
// kernel (spconv_wg_kernel, BF16x3 / FP16 at Cout >= 64, described above it) and the mma.sync kernel below.
//
//   out[o, :] = epilogue( sum_k features[nbr[k, o], :] @ W[k] )          (spconv_ops.h:260-361)
//
// The GEMM K axis is the concatenation over the kernel offsets of the Cin channels, cut into blocks of 32 channels;
// every operand row stores 4 bytes per channel, so one K block of one row is one 128-byte line:
//   * BF16x3 (mode 0, the default): PRE-SPLIT FEATURES.  A row is stored as the bf16 image the tensor core
//     consumes: per group of 16 channels 32 B of bf16 "hi" followed by 32 B of bf16 "lo" (hi = rn(x),
//     lo = rn(x - hi)).  The producing conv writes that image from its epilogue (and fp32 rows only where dense()
//     needs them; a residual is read from a split image too), so the split is done once per row instead of once
//     per (row, kernel offset) visit.  Per 16-channel step: lo*W_hi + hi*W_lo + hi*W_hi, fp32 accumulate.
//   * TF32 (mode 1) and 3xTF32 (mode 2): zero-padded fp32 rows, split into tf32 hi / lo in registers.
//   * FP16 (mode 3, the encoder plan's BEVB200_PREC_FP16): a row is c_eff fp16 channels, 2 B each.  The kernels see it
//     as c_eff / 2 four-byte units, so a K block is 64 channels, the gather and the swizzle are those of the other
//     modes, and a 16-channel step is one fp16 MMA (the products are exact in the fp32 accumulator).  The epilogue
//     rounds once to fp16 (round to nearest, overflow to inf) and writes the fp16 image; a residual is read from one.
//   * INT8 (modes 4 and 5, the encoder plan's BEVB200_PREC_INT8): a row is c_eff u8 channels, c_eff / 4 four-byte
//     units, so a K block is 128 channels and a k32 step of 8-bit values is the 32 B a k16 step of fp16 reads: the
//     fragments, the ldmatrix loads (no .trans: the weight image is K-major) and the wgmma descriptors are those of
//     FP16.  Mode 4 multiplies u8 rows by s8 weights into exact int32 accumulators; mode 5 is the FP16 MMA on fp16
//     rows (the chain's first conv).  Both end in the quantising epilogue of v6_store_chunk_q8.
// A CTA (8 warps, two CTAs per SM) owns 128-row output tiles, persistent over the tiles; per K block all 256
// threads gather the 128 neighbour rows with 16-byte cp.async (zero fill for missing neighbours) into an XOR-
// swizzled tile (16-byte chunk c of row r at (c ^ (r & 7)): conflict-free ldmatrix) and copy the weight block
// beside it, in a ring of cp.async stages; the neighbour indices of a stage are loaded one stage ahead.  Warp w
// multiplies rows 32 (w & 3) .. + 31 by columns (w >> 2) * Cout / 2 .. + Cout / 2 - 1 with ldmatrix + mma.sync,
// the accumulators stay in registers across all K blocks, and the tile's epilogue (folded BN, residual, ReLU, fp32
// rows and / or the split image) runs once through a shared-memory transpose.  The number of output rows may be
// read from device memory (n_out_dev), so a strided conv needs no host round trip and the whole encoder can be
// captured in a CUDA graph.
#include <type_traits>

#include "spconv.cuh"
#include "tc_ptx.cuh"

namespace bevb200 {

constexpr int kV6Threads = 256;
constexpr int kV6TileM = 128;
constexpr int kV6AStageBytes = kV6TileM * 128;   // 128 rows x 128 B

struct V6Params {
  const uint8_t *rows;          // operand rows, c_in * 4 bytes each: split image (mode 0) or fp32 (modes 1, 2)
  const uint8_t *wpacked;
  const int32_t *nbr;           // [kvol][nbr_stride]
  long long nbr_stride;
  const int32_t *n_out_dev;     // optional device-side row count (<= n_out)
  const float *scale, *shift, *residual;
  const uint8_t *residual_split; // residual rows as a split image (x = hi + lo, exact to 2^-17 |x|): lets a producer
                                 // skip its fp32 copy; may alias out_split (a thread reads its chunk before writing it)
  float *out;                   // optional fp32 rows [n_out, c_out]
  uint8_t *out_split;           // optional split image [n_out, c_out * 4 B]
  int n_in, n_out;
  int c_in, c_out, kvol, relu;
  int nkb, cin_shift;
};
// The INT8 instances' parameters (a separate type: the other instances' parameter block, and so their code, is unchanged)
struct V6ParamsQ8 : V6Params {
  const float *qparams;         // [r_out, s_res] on the device
  int out_half;                 // out_split is an fp16 image (the chain's last conv), not u8
};

// MMA mode of an instance: 0 BF16x3, 1 TF32, 2 3xTF32, 3 FP16, 4 u8 x s8 (INT8), 5 FP16 with the INT8 epilogue
template <int MODE>
using v6_acc_t = typename std::conditional<MODE == 4, int, float>::type;
template <int MODE>
using v6_params_t = typename std::conditional<MODE >= 4, V6ParamsQ8, V6Params>::type;

// INT8 epilogue of 16 channels [c0, c0 + 16) of one row; fl() is one fp32 round-to-nearest op (no contraction):
//   v = fl(fl(acc * a[c]) + shift[c]);  v = fl(v + fl(float(res_u8) * s_res));  v = max(v, 0)
//   u8 image: q = clamp(rint(fl(v * r_out)), 0, 255) (NaN -> 0, +inf -> 255);  fp16 image: half(v)
// The residual image may be this launch's own out_split (a lane reads its 16 bytes before it writes them).
__device__ __forceinline__ void v6_store_chunk_q8(const V6ParamsQ8 &p, const float (&acc)[16], int orow, int c0) {
  const int c_out = p.c_out;
  float y[16];
#pragma unroll
  for (int e = 0; e < 16; ++e) y[e] = __fadd_rn(__fmul_rn(acc[e], __ldg(p.scale + c0 + e)), __ldg(p.shift + c0 + e));
  if (p.residual_split) {
    const float s_res = __ldg(p.qparams + 1);
    const uint4 h = *reinterpret_cast<const uint4 *>(p.residual_split + (long long)orow * c_out + c0);
    const uint32_t hw[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
    for (int e = 0; e < 16; ++e)
      y[e] = __fadd_rn(y[e], __fmul_rn((float)((hw[e >> 2] >> (8 * (e & 3))) & 0xffu), s_res));
  }
  if (p.relu) {
#pragma unroll
    for (int e = 0; e < 16; ++e) y[e] = fmaxf(y[e], 0.f);
  }
  if (p.out_half) {
    uint32_t h[8];
#pragma unroll
    for (int e = 0; e < 16; e += 2) {
      const __half2 v = __floats2half2_rn(y[e], y[e + 1]);
      h[e / 2] = *reinterpret_cast<const uint32_t *>(&v);
    }
    uint4 *row = reinterpret_cast<uint4 *>(p.out_split + ((long long)orow * c_out + c0) * 2);
    row[0] = make_uint4(h[0], h[1], h[2], h[3]);
    row[1] = make_uint4(h[4], h[5], h[6], h[7]);
  } else {
    const float r_out = __ldg(p.qparams);
    uint32_t q[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int e = 0; e < 16; ++e) {
      // fmaxf first: NaN -> 0; the clamp to [0, 255] commutes with rint at these integer bounds
      const float t = fminf(fmaxf(__fmul_rn(y[e], r_out), 0.f), 255.f);
      q[e >> 2] |= (uint32_t)__float2int_rn(t) << (8 * (e & 3));
    }
    *reinterpret_cast<uint4 *>(p.out_split + (long long)orow * c_out + c0) = make_uint4(q[0], q[1], q[2], q[3]);
  }
}

// one 16-bit k16 / 8-bit k32 MMA of the FP16 (3, 5) and INT8 (4) modes
template <int MODE>
__device__ __forceinline__ void v6_mma_k32b(v6_acc_t<MODE> (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (MODE == 4) mma_u8s8_16832(d, a, b0, b1);
  else mma_f16_16816(d, a, b0, b1);
}

// Epilogue of NC (8 or 16) consecutive channels [c0, c0 + NC) of one row: folded BN, residual, ReLU,
// then the fp32 row and / or its split image.  NC channels = NC/8 16-byte chunks of hi and of lo.
// F16: residual_split and out_split are fp16 images [n, c_out] instead of split images.
template <int NC, bool F16>
__device__ __forceinline__ void v6_store_chunk(const V6Params &p, float (&acc)[NC], int orow, int c0) {
  const int c_out = p.c_out;
  float y[NC];
#pragma unroll
  for (int e = 0; e < NC; ++e) {
    float t = acc[e];
    if (p.scale) t *= __ldg(p.scale + c0 + e);
    if (p.shift) t += __ldg(p.shift + c0 + e);
    y[e] = t;
  }
  if (p.residual) {
    const float4 *res = reinterpret_cast<const float4 *>(p.residual + (long long)orow * c_out + c0);
#pragma unroll
    for (int j = 0; j < NC / 4; ++j) {
      const float4 rv = __ldg(res + j);
      y[4 * j] += rv.x; y[4 * j + 1] += rv.y; y[4 * j + 2] += rv.z; y[4 * j + 3] += rv.w;
    }
  } else if (F16 && p.residual_split) {
    // plain loads (the image may be this launch's own out_split, rewritten below by the same lane)
    const uint4 *row = reinterpret_cast<const uint4 *>(p.residual_split + ((long long)orow * c_out + c0) * 2);
#pragma unroll
    for (int j = 0; j < NC / 8; ++j) {
      const uint4 h = row[j];
      const uint32_t hw[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&hw[e]));
        y[8 * j + 2 * e] += f.x;
        y[8 * j + 2 * e + 1] += f.y;
      }
    }
  } else if (p.residual_split) {
    // plain loads (the image may be this launch's own out_split, rewritten below by the same lane)
    const uint8_t *row = p.residual_split + (long long)orow * (c_out * 4) + (c0 >> 4) * 64 + (c0 & 15) * 2;
#pragma unroll
    for (int j = 0; j < NC / 8; ++j) {
      const uint4 h = *reinterpret_cast<const uint4 *>(row + 16 * j);
      const uint4 l = *reinterpret_cast<const uint4 *>(row + 32 + 16 * j);
      const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        y[8 * j + 2 * e] += __uint_as_float(hw[e] << 16) + __uint_as_float(lw[e] << 16);
        y[8 * j + 2 * e + 1] += __uint_as_float(hw[e] & 0xffff0000u) + __uint_as_float(lw[e] & 0xffff0000u);
      }
    }
  }
  if (p.relu) {
#pragma unroll
    for (int e = 0; e < NC; ++e) y[e] = fmaxf(y[e], 0.f);
  }
  if (p.out) {
    float4 *dst = reinterpret_cast<float4 *>(p.out + (long long)orow * c_out + c0);
#pragma unroll
    for (int j = 0; j < NC / 4; ++j) dst[j] = make_float4(y[4 * j], y[4 * j + 1], y[4 * j + 2], y[4 * j + 3]);
  }
  if (F16 && p.out_split) {
    uint32_t h[NC / 2];
#pragma unroll
    for (int e = 0; e < NC; e += 2) {
      const __half2 v = __floats2half2_rn(y[e], y[e + 1]);
      h[e / 2] = *reinterpret_cast<const uint32_t *>(&v);
    }
    uint4 *row = reinterpret_cast<uint4 *>(p.out_split + ((long long)orow * c_out + c0) * 2);
#pragma unroll
    for (int j = 0; j < NC / 8; ++j) row[j] = make_uint4(h[4 * j], h[4 * j + 1], h[4 * j + 2], h[4 * j + 3]);
  } else if (p.out_split) {
    uint32_t hi[NC / 2], lo[NC / 2];
#pragma unroll
    for (int e = 0; e < NC; e += 2) split_pair(y[e], y[e + 1], hi[e / 2], lo[e / 2]);
    // group g = c0 / 16 starts at g * 64 B: [hi 32 B | lo 32 B]; c0 % 16 is 0 or 8
    uint8_t *row = p.out_split + (long long)orow * (c_out * 4) + (c0 >> 4) * 64 + (c0 & 15) * 2;
#pragma unroll
    for (int j = 0; j < NC / 8; ++j) {
      *reinterpret_cast<uint4 *>(row + 16 * j) = make_uint4(hi[4 * j], hi[4 * j + 1], hi[4 * j + 2], hi[4 * j + 3]);
      *reinterpret_cast<uint4 *>(row + 32 + 16 * j) = make_uint4(lo[4 * j], lo[4 * j + 1], lo[4 * j + 2], lo[4 * j + 3]);
    }
  }
}

// weight bytes per K block and ring depth of a (mode, Cout) instance: as many stages (<= 4) as fit two CTAs per SM
template <int MODE, int COUT>
struct V6Shape {
  static constexpr int kB = (MODE == 2 ? 2 : 1) * COUT * 128;
  static constexpr int kStage = kV6AStageBytes + kB;
  static constexpr int kStages = (110 * 1024) / kStage > 4 ? 4 : (110 * 1024) / kStage;
  static constexpr int kLd = COUT + 4;                         // fp32 row pitch of the epilogue transpose
  static constexpr int kEpi = kV6TileM * kLd * 4;
  static constexpr int kSmem = kStages * kStage > kEpi ? kStages * kStage : kEpi;
  static_assert(kStages >= 2, "no room for two stages");
};

template <int MODE, int COUT>
__global__ void __launch_bounds__(kV6Threads, 2) spconv_v6_kernel(const v6_params_t<MODE> p) {
  using Sh = V6Shape<MODE, COUT>;
  constexpr int S = Sh::kStages, kB = Sh::kB, kStage = Sh::kStage;
  constexpr int NT = COUT / 16;                   // n8 tiles per warp (the two warp halves split the columns)
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const uint32_t smem = smem_u32(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nkb = p.nkb;

  // Programmatic dependent launch: the previous kernel of the stream may still be draining until here; its
  // results (feature image, row count) are only touched below.  Without the launch attribute both are no-ops.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  int n_out = p.n_out;
  if (p.n_out_dev) n_out = min(n_out, __ldg(p.n_out_dev));
  const int n_tiles = (n_out + kV6TileM - 1) / kV6TileM;

  // copy role: rows cr + 32 j (j < 4), logical 16-byte chunk cc of the K block = channels kb * 32 + 4 cc .. + 3 of the
  // concatenation over kernel offsets (c_in < 32: one K block spans 32 / c_in offsets)
  const int cr = tid >> 3, cc = tid & 7;
  const unsigned long long fbase = reinterpret_cast<unsigned long long>(p.rows);
  const uint32_t row_bytes = (uint32_t)p.c_in * 4u;
  const int cin_mask = p.c_in - 1;
  // mma role
  const int wm = (warp & 3) * 32, wn = (warp >> 2) * (COUT / 2);

  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int row0 = tile * kV6TileM;
    auto load_idx = [&](int kb, int (&idx)[4]) {
      const int k = (kb * 32 + 4 * cc) >> p.cin_shift;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int row = row0 + cr + 32 * j;
        idx[j] = -1;
        if (kb < nkb && k < p.kvol && row < n_out) idx[j] = __ldg(p.nbr + (long long)k * p.nbr_stride + row);
      }
    };
    auto load_stage = [&](int kb, const int (&idx)[4]) {
      const uint32_t a = smem + (uint32_t)(kb % S) * kStage, b = a + kV6AStageBytes;
      const unsigned coff = (unsigned)(((kb * 32 + 4 * cc) & cin_mask) << 2);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int r = cr + 32 * j;
        const int src = idx[j] >= p.n_in ? -1 : idx[j];
        cp_async16_row(a + (uint32_t)(r * 128 + ((cc ^ (r & 7)) << 4)),
                       fbase + (unsigned long long)(uint32_t)max(src, 0) * row_bytes + coff, src);
      }
      const uint8_t *src = p.wpacked + (size_t)kb * kB;
      for (int i = tid; i < kB / 16; i += kV6Threads) cp_async16(b + (uint32_t)i * 16u, src + (size_t)i * 16);
    };

    v6_acc_t<MODE> acc[2][NT][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0;

    int nidx[4];
#pragma unroll
    for (int s = 0; s < S - 1; ++s) {
      int idx[4];
      load_idx(s, idx);
      if (s < nkb) load_stage(s, idx);
      cp_async_commit();
    }
    load_idx(S - 1, nidx);

    for (int kb = 0; kb < nkb; ++kb) {
      cp_async_wait<S - 2>();
      __syncthreads();                       // stage kb has landed; stage kb - 1 is free again
      {
        const int kn = kb + S - 1;
        if (kn < nkb) load_stage(kn, nidx);
        cp_async_commit();
        load_idx(kn + 1, nidx);              // consumed one iteration later: the load overlaps the MMAs
      }
      const uint32_t a = smem + (uint32_t)(kb % S) * kStage, b = a + kV6AStageBytes;
      if constexpr (MODE == 0) {
#pragma unroll
        for (int g = 0; g < 2; ++g) {        // the two 16-channel groups of the K block
          uint32_t ahi[2][4], alo[2][4];
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            const int r = wm + 16 * mt + (lane & 15), lc = 4 * g + (lane >> 4);
            ldsm_x4(a + (uint32_t)(r * 128 + ((lc ^ (r & 7)) << 4)), ahi[mt]);
            ldsm_x4(a + (uint32_t)(r * 128 + (((lc + 2) ^ (r & 7)) << 4)), alo[mt]);
          }
          if constexpr (NT == 1) {
            const int n = wn + (lane & 7), lc = 2 * g + ((lane >> 3) & 1);
            uint32_t bh[2], bl[2];
            ldsm_x2(b + (uint32_t)(n * 128 + ((lc ^ (n & 7)) << 4)), bh);
            ldsm_x2(b + (uint32_t)(n * 128 + (((lc + 4) ^ (n & 7)) << 4)), bl);
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
              mma_bf16_16816(acc[mt][0], alo[mt], bh[0], bh[1]);
              mma_bf16_16816(acc[mt][0], ahi[mt], bl[0], bl[1]);
              mma_bf16_16816(acc[mt][0], ahi[mt], bh[0], bh[1]);
            }
          } else {
#pragma unroll
            for (int nt = 0; nt < NT; nt += 2) {
              const int n = wn + nt * 8 + (lane & 7) + ((lane >> 4) << 3), lc = 2 * g + ((lane >> 3) & 1);
              uint32_t bh[4], bl[4];
              ldsm_x4(b + (uint32_t)(n * 128 + ((lc ^ (n & 7)) << 4)), bh);
              ldsm_x4(b + (uint32_t)(n * 128 + (((lc + 4) ^ (n & 7)) << 4)), bl);
#pragma unroll
              for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  mma_bf16_16816(acc[mt][nt + h], alo[mt], bh[2 * h], bh[2 * h + 1]);
                  mma_bf16_16816(acc[mt][nt + h], ahi[mt], bl[2 * h], bl[2 * h + 1]);
                  mma_bf16_16816(acc[mt][nt + h], ahi[mt], bh[2 * h], bh[2 * h + 1]);
                }
            }
          }
        }
      } else if constexpr (MODE >= 3) {
        // four k16 steps of 16 fp16 channels (INT8: k32 steps of 32 u8 channels): chunks 2 ks, 2 ks + 1 (not
        // unrolled at Cout 128: it would spill)
#pragma unroll(COUT == 128 ? 1 : 4)
        for (int ks = 0; ks < 4; ++ks) {
          uint32_t af[2][4];
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            const int r = wm + 16 * mt + (lane & 15), lc = 2 * ks + (lane >> 4);
            ldsm_x4(a + (uint32_t)(r * 128 + ((lc ^ (r & 7)) << 4)), af[mt]);
          }
          const int lc = 2 * ks + ((lane >> 3) & 1);
          if constexpr (NT == 1) {
            const int n = wn + (lane & 7);
            uint32_t bf[2];
            ldsm_x2(b + (uint32_t)(n * 128 + ((lc ^ (n & 7)) << 4)), bf);
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) v6_mma_k32b<MODE>(acc[mt][0], af[mt], bf[0], bf[1]);
          } else {
#pragma unroll
            for (int nt = 0; nt < NT; nt += 2) {
              const int n = wn + nt * 8 + (lane & 7) + ((lane >> 4) << 3);
              uint32_t bf[4];
              ldsm_x4(b + (uint32_t)(n * 128 + ((lc ^ (n & 7)) << 4)), bf);
#pragma unroll
              for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int h = 0; h < 2; ++h) v6_mma_k32b<MODE>(acc[mt][nt + h], af[mt], bf[2 * h], bf[2 * h + 1]);
            }
          }
        }
      } else {
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {     // four k8 steps of 8 fp32 channels
          uint32_t ahi[2][4], alo[2][4];
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            const int r = wm + 16 * mt + (lane & 15), lc = 2 * ks + (lane >> 4);
            uint32_t raw[4];
            ldsm_x4(a + (uint32_t)(r * 128 + ((lc ^ (r & 7)) << 4)), raw);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float x = __uint_as_float(raw[e]);
              ahi[mt][e] = cvt_tf32(x);
              alo[mt][e] = MODE == 2 ? cvt_tf32(x - __uint_as_float(ahi[mt][e])) : 0u;
            }
          }
#pragma unroll
          for (int nt = 0; nt < NT; nt += 2) {
            const int lc = 2 * ks + ((lane >> 3) & 1);
            uint32_t bh[4], bl[4] = {0u, 0u, 0u, 0u};
            if constexpr (NT == 1) {
              const int n = wn + (lane & 7);
              uint32_t t2[2];
              ldsm_x2(b + (uint32_t)(n * 128 + ((lc ^ (n & 7)) << 4)), t2);
              bh[0] = t2[0]; bh[1] = t2[1]; bh[2] = bh[3] = 0u;
              if constexpr (MODE == 2) {
                ldsm_x2(b + (uint32_t)((COUT + n) * 128 + ((lc ^ (n & 7)) << 4)), t2);
                bl[0] = t2[0]; bl[1] = t2[1];
              }
            } else {
              const int n = wn + nt * 8 + (lane & 7) + ((lane >> 4) << 3);
              ldsm_x4(b + (uint32_t)(n * 128 + ((lc ^ (n & 7)) << 4)), bh);
              if constexpr (MODE == 2) ldsm_x4(b + (uint32_t)((COUT + n) * 128 + ((lc ^ (n & 7)) << 4)), bl);
            }
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
              for (int h = 0; h < (NT == 1 ? 1 : 2); ++h) {
                if constexpr (MODE == 2) {
                  mma_tf32_1688(acc[mt][nt + h], alo[mt], bh[2 * h], bh[2 * h + 1]);
                  mma_tf32_1688(acc[mt][nt + h], ahi[mt], bl[2 * h], bl[2 * h + 1]);
                }
                mma_tf32_1688(acc[mt][nt + h], ahi[mt], bh[2 * h], bh[2 * h + 1]);
              }
          }
        }
      }
    }
    cp_async_wait<0>();
    __syncthreads();                         // every warp is done with the ring: reuse it for the transpose

    // ------------------------------- epilogue of the tile ----------------------------------------
    float *cs = reinterpret_cast<float *>(smem_raw);
    constexpr int LD = Sh::kLd;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        // INT8: float(acc), rounded to nearest (exact below 2^24)
        const int r = wm + 16 * mt + (lane >> 2), c = wn + nt * 8 + 2 * (lane & 3);
        *reinterpret_cast<float2 *>(cs + r * LD + c) = make_float2((float)acc[mt][nt][0], (float)acc[mt][nt][1]);
        *reinterpret_cast<float2 *>(cs + (r + 8) * LD + c) = make_float2((float)acc[mt][nt][2], (float)acc[mt][nt][3]);
      }
    __syncthreads();
    constexpr int kChunks = COUT / 16;
    for (int it = tid; it < kV6TileM * kChunks; it += kV6Threads) {
      const int r = it / kChunks, j = it - r * kChunks;
      const int orow = row0 + r;
      if (orow < n_out) {
        float v[16];
#pragma unroll
        for (int e = 0; e < 16; e += 4) {
          const float4 q = *reinterpret_cast<const float4 *>(cs + r * LD + 16 * j + e);
          v[e] = q.x; v[e + 1] = q.y; v[e + 2] = q.z; v[e + 3] = q.w;
        }
        if constexpr (MODE >= 4) v6_store_chunk_q8(p, v, orow, 16 * j);
        else v6_store_chunk<16, MODE == 3>(p, v, orow, 16 * j);
      }
    }
    __syncthreads();                         // the transpose area is the next tile's ring
  }
}

// ---- BF16x3 forward on warpgroup MMAs (mode 0) -----------------------------------------------
// Warp-specialised and persistent: warpgroup 0 is the producer, warpgroups 1 and 2 the consumers.  A tile is
// kTileM output rows; each consumer warpgroup owns kMT m64 blocks of it and keeps their accumulators (Cout / 2
// fp32 per thread and block) in registers across all K blocks.  Per K block one ring stage holds
//   * A: the tile's gathered rows, 128 B each, laid out as before (16-byte chunk c of row r at c ^ (r & 7)), which
//     is the K-major SWIZZLE_128B layout wgmma reads: the four k16 slices of a row (hi / lo of the two 16-channel
//     groups) are the same descriptor moved 0 / 32 / 64 / 96 B along the row;
//   * B: the K block's packed weight rows (Cout x 128 B, same swizzle), one bulk copy.
// The producer gathers the rows with 16-byte cp.async (zero fill for missing neighbours), each thread arriving on
// the stage's "full" barrier when its copies land (cp.async.mbarrier.arrive.noinc); one thread adds the weight
// copy's bytes to the same barrier.  Consumers wait on "full", issue the 3 x 2 x kMT wgmmas of the block (FP16, mode 3:
// 4 x kMT, one per 16 channels of the 64-channel block), keep one
// block in flight (wait_group 1) and then release the previous stage on its "empty" barrier.  The tile's epilogue
// goes through a small per-warp transpose buffer, so the producer keeps filling the ring meanwhile.
constexpr int kWgThreads = 384;
constexpr int kWgMinKBlocks = 16;               // fewer K blocks per tile: spconv_v6_kernel
constexpr int kWgSmemMax = 227 * 1024;        // opt-in dynamic shared memory per block on sm_90

template <int COUT>
struct WgShape {
  static_assert(COUT == 64 || COUT == 128, "Cout <= 32 runs on spconv_v6_kernel");
  static constexpr int kMT = 2;                                // m64 blocks per consumer warpgroup
  static constexpr int kTileM = 2 * 64 * kMT;                  // 256 rows share one weight stage
  static constexpr int kA = kTileM * 128;
  static constexpr int kB = COUT * 128;
  static constexpr int kStage = kA + kB;                       // multiple of 1024: every stage stays atom-aligned
  static constexpr int kSlice = 32;                            // columns per epilogue transpose step
  static constexpr int kLd = kSlice + 4;
  static constexpr int kEpi = 8 * 16 * kLd * 4;                // one 16-row buffer per consumer warp
  static constexpr int kFixed = 1024 + kEpi + 2 * 8 * 8;       // alignment slack, transpose buffers, barriers
  static constexpr int kStages = (kWgSmemMax - kFixed) / kStage > 8 ? 8 : (kWgSmemMax - kFixed) / kStage;
  static constexpr int kSmem = kFixed + kStages * kStage;
  static_assert(kStage % 1024 == 0 && kStages >= 2, "ring does not fit");
};

template <bool F16, int COUT>
__device__ __forceinline__ void wgmma_nc(float (&d)[COUT / 2], uint64_t da, uint64_t db, int accumulate) {
  if constexpr (COUT == 64) wgmma_n64<F16>(d, da, db, accumulate);
  else wgmma_n128<F16>(d, da, db, accumulate);
}

// MODE 0 (BF16x3), 3 (FP16), 4 (INT8) or 5 (FP16 with the INT8 epilogue)
template <int MODE, int COUT>
__global__ void __launch_bounds__(kWgThreads, 1) spconv_wg_kernel(const v6_params_t<MODE> p) {
  using Sh = WgShape<COUT>;
  constexpr int S = Sh::kStages, MT = Sh::kMT, TM = Sh::kTileM;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bars = smem + S * Sh::kStage;                 // full[S], then empty[S]
  float *epi = reinterpret_cast<float *>(smem_raw + (bars - smem_u32(smem_raw)) + 2 * 8 * 8);
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
  const int nkb = p.nkb;

  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(bars + 8 * s, 128 + 1);                        // 128 producer threads + the weight copy
      mbar_init(bars + 8 * (S + s), 8);                        // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // Programmatic dependent launch: the previous kernel of the stream may still be draining until here; its
  // results (feature image, row count) are only touched below.  Without the launch attribute both are no-ops.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  int n_out = p.n_out;
  if (p.n_out_dev) n_out = min(n_out, __ldg(p.n_out_dev));
  const int n_tiles = (n_out + TM - 1) / TM;

  if (wg == 0) {
    // ------------------------------------ producer ------------------------------------------------
    setmaxnreg_dec<40>();
    // rows pr + 16 j of the tile, logical 16-byte chunk cc of the K block = channels kb * 32 + 4 cc .. + 3 of the
    // concatenation over kernel offsets (c_in < 32: one K block spans 32 / c_in offsets)
    constexpr int J = TM / 16;
    const int cc = tid & 7, pr = tid >> 3;
    const unsigned long long fbase = reinterpret_cast<unsigned long long>(p.rows);
    const uint32_t row_bytes = (uint32_t)p.c_in * 4u;
    const int cin_mask = p.c_in - 1;
    auto load_idx = [&](int tile, int kb, int (&idx)[J]) {
      const int k = (kb * 32 + 4 * cc) >> p.cin_shift;
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int row = tile * TM + pr + 16 * j;
        idx[j] = -1;
        if (k < p.kvol && row < n_out) idx[j] = __ldg(p.nbr + (long long)k * p.nbr_stride + row);
      }
    };
    int idx[J];
    int tile = blockIdx.x, kb = 0;
    if (tile < n_tiles) load_idx(tile, 0, idx);
    for (uint32_t it = 0; tile < n_tiles; ++it) {
      const uint32_t s = it % S, full = bars + 8 * s;
      mbar_wait(bars + 8 * (S + s), ((it / S) & 1) ^ 1);     // the consumers are done with the stage
      const uint32_t a = smem + s * Sh::kStage;
      if (tid == 0) {
        mbar_arrive_expect_tx(full, Sh::kB);
        bulk_copy_g2s(a + Sh::kA, p.wpacked + (size_t)kb * Sh::kB, Sh::kB, full);
      }
      const unsigned coff = (unsigned)(((kb * 32 + 4 * cc) & cin_mask) << 2);
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int r = pr + 16 * j;
        const int src = idx[j] >= p.n_in ? -1 : idx[j];
        cp_async16_row(a + (uint32_t)(r * 128 + ((cc ^ (r & 7)) << 4)),
                       fbase + (unsigned long long)(uint32_t)max(src, 0) * row_bytes + coff, src);
      }
      cp_async_mbar_arrive_noinc(full);
      if (++kb == nkb) { kb = 0; tile += gridDim.x; }
      if (tile < n_tiles) load_idx(tile, kb, idx);           // next stage's indices: the load overlaps the wait
    }
  } else {
    // ------------------------------------ consumers -----------------------------------------------
    setmaxnreg_inc<232>();
    const int cw = wg - 1, warp = (tid >> 5) & 3;
    v6_acc_t<MODE> acc[MT][COUT / 2];
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        const uint32_t s = it % S;
        mbar_wait(bars + 8 * s, (it / S) & 1);
        // the rows arrived through cp.async (generic proxy) and are read by wgmma (async proxy)
        fence_proxy_async_smem();
        wgmma_fence();
        const uint32_t a = smem + s * Sh::kStage + cw * (MT * 64 * 128), b = smem + s * Sh::kStage + Sh::kA;
        if constexpr (MODE >= 3) {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {  // the four k16 (INT8: k32) slices of the K block, A and W alike
            const uint64_t bd = wgmma_desc_sw128(b + 32 * ks);
#pragma unroll
            for (int m = 0; m < MT; ++m) {
              const uint64_t ad = wgmma_desc_sw128(a + m * (64 * 128) + 32 * ks);
              if constexpr (MODE != 4) wgmma_nc<true, COUT>(acc[m], ad, bd, kb > 0 || ks > 0);
              else if constexpr (COUT == 64) wgmma_n64_i8(acc[m], ad, bd, kb > 0 || ks > 0);
              else wgmma_n128_i8(acc[m], ad, bd, kb > 0 || ks > 0);
            }
          }
        } else {
#pragma unroll
          for (int g = 0; g < 2; ++g) {     // the two 16-channel groups of the K block: A [hi | lo], W [hi, hi | lo, lo]
            const uint64_t bh = wgmma_desc_sw128(b + 32 * g), bl = wgmma_desc_sw128(b + 64 + 32 * g);
#pragma unroll
            for (int m = 0; m < MT; ++m) {
              const uint64_t ah = wgmma_desc_sw128(a + m * (64 * 128) + 64 * g), al = wgmma_desc_sw128(a + m * (64 * 128) + 64 * g + 32);
              wgmma_nc<false, COUT>(acc[m], al, bh, kb > 0 || g > 0);
              wgmma_nc<false, COUT>(acc[m], ah, bl, 1);
              wgmma_nc<false, COUT>(acc[m], ah, bh, 1);
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (kb > 0 && lane == 0) mbar_arrive(bars + 8 * (S + (it - 1) % S));
      }
      wgmma_wait<0>();
#pragma unroll
      for (int m = 0; m < MT; ++m) wgmma_pin(acc[m]);
      if (lane == 0) mbar_arrive(bars + 8 * (S + (it - 1) % S));

      // ------------------------------- epilogue of the tile ----------------------------------------
      // fragment of block m: rows 16 warp + lane / 4 (+ 8), columns 8 i + 2 (lane % 4) (+ 1)
      constexpr int SW = Sh::kSlice, LD = Sh::kLd, CH = SW / 16;
      float *buf = epi + (cw * 4 + warp) * 16 * LD;
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        const int rbase = tile * TM + cw * (MT * 64) + 64 * m + 16 * warp;
#pragma unroll
        for (int c0 = 0; c0 < COUT; c0 += SW) {
#pragma unroll
          for (int i = 0; i < SW / 8; ++i) {
            const int r = lane >> 2, c = 8 * i + 2 * (lane & 3), q = 4 * (c0 / 8 + i);
            *reinterpret_cast<float2 *>(buf + r * LD + c) = make_float2((float)acc[m][q], (float)acc[m][q + 1]);
            *reinterpret_cast<float2 *>(buf + (r + 8) * LD + c) = make_float2((float)acc[m][q + 2], (float)acc[m][q + 3]);
          }
          __syncwarp();
          const int r = lane / CH, j = lane % CH;
          if (lane < 16 * CH && rbase + r < n_out) {
            float v[16];
#pragma unroll
            for (int e = 0; e < 16; e += 4) {
              const float4 q = *reinterpret_cast<const float4 *>(buf + r * LD + 16 * j + e);
              v[e] = q.x; v[e + 1] = q.y; v[e + 2] = q.z; v[e + 3] = q.w;
            }
            if constexpr (MODE >= 4) v6_store_chunk_q8(p, v, rbase + r, c0 + 16 * j);
            else v6_store_chunk<16, MODE == 3>(p, v, rbase + r, c0 + 16 * j);
          }
          __syncwarp();
        }
      }
    }
  }
}

// ---- operand images --------------------------------------------------------------------------
// fp32 rows [n, c_in] -> split image [n, c_eff * 4 B], c_eff = c_in rounded up to 16 (zero padded).
// One thread per (row, 8 channels): 16 B of hi and 16 B of lo.
__global__ void spconv_v6_split_rows_kernel(const float *__restrict__ in, int n_cap,
                                            const int32_t *__restrict__ n_dev, int c_in, int c_eff,
                                            uint8_t *__restrict__ out) {
  int n = n_cap;
  if (n_dev) n = min(n, __ldg(n_dev));
  const int per_row = c_eff >> 3;
  const long long total = (long long)n * per_row;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(t % per_row);
    const long long r = t / per_row;
    float x[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] = 8 * j + e < c_in ? in[r * c_in + 8 * j + e] : 0.f;
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int e = 0; e < 8; e += 2) split_pair(x[e], x[e + 1], hi[e / 2], lo[e / 2]);
    uint8_t *dst = out + r * ((long long)c_eff * 4) + (j >> 1) * 64 + (j & 1) * 16;
    *reinterpret_cast<uint4 *>(dst) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4 *>(dst + 32) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  }
}

// Weight image of the three-product form: one stage (Cout rows of 128 B, contiguous) per 32-wide K block, row n =
// [W_hi kk 0-15 | W_hi kk 16-31 | W_lo kk 0-15 | W_lo kk 16-31] (32 B each), SWIZZLE_128B.
__global__ void spconv_v6_pack_rows_kernel(const float *__restrict__ w, int kvol, int c_in, int c_in_eff,
                                           int c_out, int nkb, uint16_t *__restrict__ packed) {
  const long long total = (long long)nkb * c_out * 32;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int cc = (int)(t % 32);
    const int n = (int)((t / 32) % c_out);
    const int kb = (int)(t / (32ll * c_out));
    const int kk = kb * 32 + cc;
    const int k = kk / c_in_eff, ci = kk % c_in_eff;
    const float v = (k < kvol && ci < c_in) ? w[((long long)k * c_in + ci) * c_out + n] : 0.f;
    uint32_t u = __float_as_uint(v);
    u += 0x7fffu + ((u >> 16) & 1u);
    const uint32_t hb = u >> 16;
    const float lo = v - __uint_as_float(hb << 16);
    uint32_t ul = __float_as_uint(lo);
    ul += 0x7fffu + ((ul >> 16) & 1u);
    // logical 16-byte chunk: hi -> cc / 8 (0..3), lo -> 4 + cc / 8; physical chunk = logical ^ (n & 7)
    uint16_t *row = packed + ((long long)kb * c_out + n) * 64;
    row[(((cc >> 3) ^ (n & 7)) << 3) | (cc & 7)] = (uint16_t)hb;
    row[((((cc >> 3) + 4) ^ (n & 7)) << 3) | (cc & 7)] = (uint16_t)(ul >> 16);
  }
}

// fp16 rows [n, c_in] -> fp16 image [n, c_eff] (zero padded, exact); one thread per (row, 8 channels)
__global__ void spconv_v6_f16_rows_kernel(const __half *__restrict__ in, int n_cap, const int32_t *__restrict__ n_dev,
                                          int c_in, int c_eff, uint8_t *__restrict__ out) {
  int n = n_cap;
  if (n_dev) n = min(n, max(__ldg(n_dev), 0));
  const int per_row = c_eff >> 3;
  const long long total = (long long)n * per_row;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(t % per_row);
    const long long r = t / per_row;
    uint32_t h[4];
#pragma unroll
    for (int e = 0; e < 8; e += 2) {
      const int c = 8 * j + e;
      const __half2 v = __halves2half2(c < c_in ? in[r * c_in + c] : __ushort_as_half(0),
                                       c + 1 < c_in ? in[r * c_in + c + 1] : __ushort_as_half(0));
      h[e / 2] = *reinterpret_cast<const uint32_t *>(&v);
    }
    *reinterpret_cast<uint4 *>(out + (r * c_eff + 8 * j) * 2) = make_uint4(h[0], h[1], h[2], h[3]);
  }
}

// Weight image of the fp16 form: one stage (Cout rows of 128 B) per 64-wide K block, row n = fp16(W) of kk 0-63,
// SWIZZLE_128B (16-byte chunk kk / 8 at (kk / 8) ^ (n & 7)).
__global__ void spconv_v6_pack_f16_kernel(const float *__restrict__ w, int kvol, int c_in, int c_in_eff, int c_out,
                                          int nkb, __half *__restrict__ packed) {
  const long long total = (long long)nkb * c_out * 64;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int cc = (int)(t % 64);
    const int n = (int)((t / 64) % c_out);
    const int kb = (int)(t / (64ll * c_out));
    const int kk = kb * 64 + cc;
    const int k = kk / c_in_eff, ci = kk % c_in_eff;
    const float v = (k < kvol && ci < c_in) ? w[((long long)k * c_in + ci) * c_out + n] : 0.f;
    packed[((long long)kb * c_out + n) * 64 + ((((cc >> 3) ^ (n & 7)) << 3) | (cc & 7))] = __float2half_rn(v);
  }
}

// Per-output-channel weight scale of the INT8 form: s_w[n] = fl(max |W[.., .., n]| / 127), or 1 when that max is 0
__global__ void spconv_v6_i8_scales_kernel(const float *__restrict__ w, int kvol, int c_in, int c_out,
                                           float *__restrict__ s_w) {
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < c_out; n += gridDim.x * blockDim.x) {
    float m = 0.f;
    for (long long t = 0; t < (long long)kvol * c_in; ++t) m = fmaxf(m, fabsf(w[t * c_out + n]));
    s_w[n] = m > 0.f ? __fdiv_rn(m, 127.f) : 1.f;
  }
}

// Weight image of the INT8 form: one stage (Cout rows of 128 B) per 128-wide K block, row n = q_w of kk 0-127 with
// q_w = clamp(rint(fl(W / s_w[n])), -127, 127) (ties to even), SWIZZLE_128B (16-byte chunk kk / 16 at (kk / 16) ^ (n & 7)).
__global__ void spconv_v6_pack_i8_kernel(const float *__restrict__ w, const float *__restrict__ s_w, int kvol,
                                         int c_in, int c_in_eff, int c_out, int nkb, int8_t *__restrict__ packed) {
  const long long total = (long long)nkb * c_out * 128;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int cc = (int)(t % 128);
    const int n = (int)((t / 128) % c_out);
    const int kb = (int)(t / (128ll * c_out));
    const int kk = kb * 128 + cc;
    const int k = kk / c_in_eff, ci = kk % c_in_eff;
    const float v = (k < kvol && ci < c_in) ? w[((long long)k * c_in + ci) * c_out + n] : 0.f;
    const float x = fminf(fmaxf(__fdiv_rn(v, __ldg(s_w + n)), -127.f), 127.f);
    packed[((long long)kb * c_out + n) * 128 + ((((cc >> 4) ^ (n & 7)) << 4) | (cc & 15))] = (int8_t)__float2int_rn(x);
  }
}

int spconv_v6_cin_eff(int c_in) {
  for (int e = 16; e <= 128; e <<= 1)
    if (c_in <= e) return e;
  return 0;
}
bool spconv_v6_shape_ok(int c_in, int c_out, int kvol) {
  return (c_out == 16 || c_out == 32 || c_out == 64 || c_out == 128) && c_in >= 1 &&
         spconv_v6_cin_eff(c_in) != 0 && kvol >= 1 && kvol <= 27;
}
static int v6_nkb(int c_eff, int kvol) { return (kvol * c_eff + 31) / 32; }

size_t spconv_v6_packed_bytes(int c_in, int c_out, int kvol) {
  if (!spconv_v6_shape_ok(c_in, c_out, kvol)) return 0;
  return (size_t)v6_nkb(spconv_v6_cin_eff(c_in), kvol) * c_out * 128;
}
// K blocks of 64 fp16 channels = 32 four-byte units
static int v6_nkb_f16(int c_eff, int kvol) { return v6_nkb(c_eff / 2, kvol); }

size_t spconv_v6_packed_bytes_f16(int c_in, int c_out, int kvol) {
  if (!spconv_v6_shape_ok(c_in, c_out, kvol)) return 0;
  return (size_t)v6_nkb_f16(spconv_v6_cin_eff(c_in), kvol) * c_out * 128;
}

// K blocks of 128 u8 channels = 32 four-byte units
static int v6_nkb_i8(int c_eff, int kvol) { return v6_nkb(c_eff / 4, kvol); }

size_t spconv_v6_packed_bytes_i8(int c_in, int c_out, int kvol) {
  if (!spconv_v6_shape_ok(c_in, c_out, kvol)) return 0;
  return (size_t)v6_nkb_i8(spconv_v6_cin_eff(c_in), kvol) * c_out * 128;
}

int spconv_v6_pack_weights_i8(const float *weight, int c_in, int c_out, int kvol, float *s_w, void *packed,
                              cudaStream_t st) {
  const int ce = spconv_v6_cin_eff(c_in);
  const int nkb = v6_nkb_i8(ce, kvol);
  BEVB200_LAUNCH(spconv_v6_i8_scales_kernel, (c_out + 127) / 128, 128, 0, st, weight, kvol, c_in, c_out, s_w);
  BEVB200_LAUNCH(spconv_v6_pack_i8_kernel, grid_for((long long)nkb * c_out * 128, 256), 256, 0, st, weight, s_w, kvol,
                 c_in, ce, c_out, nkb, (int8_t *)packed);
  return BEVB200_OK;
}

int spconv_v6_pack_weights_f16(const float *weight, int c_in, int c_out, int kvol, void *packed, cudaStream_t st) {
  const int ce = spconv_v6_cin_eff(c_in);
  const int nkb = v6_nkb_f16(ce, kvol);
  BEVB200_LAUNCH(spconv_v6_pack_f16_kernel, grid_for((long long)nkb * c_out * 64, 256), 256, 0, st, weight, kvol,
                 c_in, ce, c_out, nkb, (__half *)packed);
  return BEVB200_OK;
}

int spconv_v6_f16_rows(const __half *rows, int n_cap, const int32_t *n_dev, int c_in, int c_eff, void *image,
                       cudaStream_t st) {
  BEVB200_REQUIRE(c_eff >= c_in && c_eff % 16 == 0 && c_in >= 1, "bad padded channel count");
  if (n_cap <= 0) return BEVB200_OK;
  BEVB200_LAUNCH(spconv_v6_f16_rows_kernel, grid_for((long long)n_cap * (c_eff / 8), 256), 256, 0, st, rows, n_cap,
                 n_dev, c_in, c_eff, (uint8_t *)image);
  return BEVB200_OK;
}

int spconv_v6_pack_weights(const float *weight, int c_in, int c_out, int kvol, void *packed, cudaStream_t st) {
  const int ce = spconv_v6_cin_eff(c_in);
  const int nkb = v6_nkb(ce, kvol);
  BEVB200_LAUNCH(spconv_v6_pack_rows_kernel, grid_for((long long)nkb * c_out * 32, 256), 256, 0, st, weight, kvol,
                 c_in, ce, c_out, nkb, (uint16_t *)packed);
  return BEVB200_OK;
}

// c_eff: 16 .. 128 for the forward kernels; the filter-gradient kernel wants whole 128-byte slabs (spconv_wgrad_tc.cu)
int spconv_v6_split_rows(const float *features, int n_cap, const int32_t *n_dev, int c_in, int c_eff, void *split,
                         cudaStream_t st) {
  BEVB200_REQUIRE(c_eff >= c_in && c_eff % 16 == 0 && c_in >= 1, "bad padded channel count");
  if (n_cap <= 0) return BEVB200_OK;
  BEVB200_LAUNCH(spconv_v6_split_rows_kernel, grid_for((long long)n_cap * (c_eff / 8), 256), 256, 0, st, features,
                 n_cap, n_dev, c_in, c_eff, (uint8_t *)split);
  return BEVB200_OK;
}

// Both forward kernels launch with programmatic stream serialisation: the launch overlaps the tail of the previous
// kernel in the stream (21 back-to-back convs per frame), and the kernel waits for its results (griddepcontrol.wait).
template <typename P>
static int v6_launch_kernel(void (*kernel)(P), int grid, int threads, int smem, const P &p, cudaStream_t st) {
  BEVB200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3((unsigned)threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  BEVB200_CUDA(cudaLaunchKernelEx(&cfg, kernel, p));
  ++g_launch_count;
  return BEVB200_OK;
}

template <int MODE, int COUT>
static int v6_launch_one(const v6_params_t<MODE> &p, cudaStream_t st) {
  const int n_tiles = (p.n_out + kV6TileM - 1) / kV6TileM;
  return v6_launch_kernel(spconv_v6_kernel<MODE, COUT>, n_tiles < 2 * kNumSMs ? n_tiles : 2 * kNumSMs, kV6Threads,
                          V6Shape<MODE, COUT>::kSmem, p, st);
}

template <int MODE>
static int v6_launch(const v6_params_t<MODE> &p, cudaStream_t st) {
  switch (p.c_out) {
    case 16: return v6_launch_one<MODE, 16>(p, st);
    case 32: return v6_launch_one<MODE, 32>(p, st);
    case 64: return v6_launch_one<MODE, 64>(p, st);
    case 128: return v6_launch_one<MODE, 128>(p, st);
  }
  BEVB200_REQUIRE(false, "output channel count has no tensor-core form");
}

template <int MODE, int COUT>
static int wg_launch_one(const v6_params_t<MODE> &p, cudaStream_t st) {
  using Sh = WgShape<COUT>;
  const int n_tiles = (p.n_out + Sh::kTileM - 1) / Sh::kTileM;
  return v6_launch_kernel(spconv_wg_kernel<MODE, COUT>, n_tiles < kNumSMs ? n_tiles : kNumSMs, kWgThreads, Sh::kSmem,
                          p, st);
}

template <int MODE>
static int wg_launch(const v6_params_t<MODE> &p, cudaStream_t st) {
  switch (p.c_out) {
    case 64: return wg_launch_one<MODE, 64>(p, st);
    case 128: return wg_launch_one<MODE, 128>(p, st);
  }
  BEVB200_REQUIRE(false, "output channel count has no tensor-core form");
}

static void v6_common(V6Params &p, const void *rows, const void *packed, const int32_t *nbr, long long nbr_stride,
                      int n_in, int n_out, const int32_t *n_out_dev, int c_in, int c_out, int kvol, const float *scale,
                      const float *shift, const float *residual, int relu, float *out) {
  memset(&p, 0, sizeof(p));
  p.rows = (const uint8_t *)rows;
  p.wpacked = (const uint8_t *)packed;
  p.nbr = nbr;
  p.nbr_stride = nbr_stride;
  p.n_out_dev = n_out_dev;
  p.scale = scale; p.shift = shift; p.residual = residual;
  p.out = out;
  p.n_in = n_in; p.n_out = n_out; p.c_in = c_in; p.c_out = c_out; p.kvol = kvol; p.relu = relu;
  p.nkb = v6_nkb(c_in, kvol);
  p.cin_shift = 0;
  while ((1 << p.cin_shift) < c_in) ++p.cin_shift;
}

int spconv_v6_forward(const void *features_split, const void *packed, const int32_t *nbr, long long nbr_stride,
                      int n_in, int n_out, const int32_t *n_out_dev, int c_in, int c_out, int kvol, const float *scale,
                      const float *shift, const float *residual, const void *residual_split, int relu, float *out,
                      void *out_split, cudaStream_t st) {
  BEVB200_REQUIRE(!(residual && residual_split), "residual given twice");
  BEVB200_REQUIRE(residual_split == nullptr || (uintptr_t)residual_split % 16 == 0, "residual image must be 16-byte aligned");
  BEVB200_REQUIRE(c_in == spconv_v6_cin_eff(c_in) && spconv_v6_shape_ok(c_in, c_out, kvol), "shape has no tensor-core form");
  BEVB200_REQUIRE(features_split && packed && nbr, "null argument");
  BEVB200_REQUIRE((uintptr_t)features_split % 16 == 0 && (out == nullptr || (uintptr_t)out % 16 == 0) &&
                      (out_split == nullptr || (uintptr_t)out_split % 16 == 0) &&
                      (residual == nullptr || (uintptr_t)residual % 16 == 0) && (uintptr_t)packed % 16 == 0,
                  "operands must be 16-byte aligned");
  if (n_out <= 0) return BEVB200_OK;
  V6Params p;
  v6_common(p, features_split, packed, nbr, nbr_stride, n_in, n_out, n_out_dev, c_in, c_out, kvol, scale, shift,
            residual, relu, out);
  p.residual_split = (const uint8_t *)residual_split;
  p.out_split = (uint8_t *)out_split;
  // The warpgroup-MMA kernel wins where the tensor work per gathered row is large (Cout >= 64) and a tile has K
  // blocks enough to amortise its pipeline fill and epilogue.  At Cout <= 32 the row gather bounds both kernels
  // and two mma.sync CTAs per SM keep more of it in flight; the k(1,1,3) conv_out (12 K blocks) is faster there too.
  return p.c_out >= 64 && p.nkb >= kWgMinKBlocks ? wg_launch<0>(p, st) : v6_launch<0>(p, st);
}

int spconv_v6_forward_f16(const void *rows, const void *packed, const int32_t *nbr, long long nbr_stride, int n_in,
                          int n_out, const int32_t *n_out_dev, int c_in, int c_out, int kvol, const float *scale,
                          const float *shift, const float *residual, const void *residual_f16, int relu, float *out,
                          void *out_f16, cudaStream_t st) {
  BEVB200_REQUIRE(!(residual && residual_f16), "residual given twice");
  BEVB200_REQUIRE(c_in == spconv_v6_cin_eff(c_in) && spconv_v6_shape_ok(c_in, c_out, kvol), "shape has no tensor-core form");
  BEVB200_REQUIRE(rows && packed && nbr, "null argument");
  BEVB200_REQUIRE((uintptr_t)rows % 16 == 0 && (out == nullptr || (uintptr_t)out % 16 == 0) &&
                      (out_f16 == nullptr || (uintptr_t)out_f16 % 16 == 0) &&
                      (residual == nullptr || (uintptr_t)residual % 16 == 0) &&
                      (residual_f16 == nullptr || (uintptr_t)residual_f16 % 16 == 0) && (uintptr_t)packed % 16 == 0,
                  "operands must be 16-byte aligned");
  if (n_out <= 0) return BEVB200_OK;
  V6Params p;
  // the kernels address a row in four-byte units: c_in fp16 channels are c_in / 2 of them
  v6_common(p, rows, packed, nbr, nbr_stride, n_in, n_out, n_out_dev, c_in / 2, c_out, kvol, scale, shift, residual,
            relu, out);
  p.residual_split = (const uint8_t *)residual_f16;
  p.out_split = (uint8_t *)out_f16;
  // the same layers as BF16x3 take the wgmma kernel: >= kWgMinKBlocks K blocks of 32 channels (half as many fp16 blocks)
  return p.c_out >= 64 && v6_nkb(c_in, kvol) >= kWgMinKBlocks ? wg_launch<3>(p, st) : v6_launch<3>(p, st);
}

int spconv_v6_forward_i8(const void *rows, bool f16_rows, const void *packed, const int32_t *nbr, long long nbr_stride,
                         int n_in, int n_out, const int32_t *n_out_dev, int c_in, int c_out, int kvol, const float *a,
                         const float *shift, const float *qparams, const void *residual_u8, int relu, bool out_half,
                         void *out_image, cudaStream_t st) {
  BEVB200_REQUIRE(c_in == spconv_v6_cin_eff(c_in) && spconv_v6_shape_ok(c_in, c_out, kvol), "shape has no tensor-core form");
  BEVB200_REQUIRE(rows && packed && nbr && a && shift && qparams && out_image, "null argument");
  BEVB200_REQUIRE((uintptr_t)rows % 16 == 0 && (uintptr_t)out_image % 16 == 0 && (uintptr_t)packed % 16 == 0 &&
                      (residual_u8 == nullptr || (uintptr_t)residual_u8 % 16 == 0),
                  "operands must be 16-byte aligned");
  if (n_out <= 0) return BEVB200_OK;
  V6ParamsQ8 p;
  // four-byte units of a row: c_in / 2 fp16 channels (the first conv), c_in / 4 u8 channels
  v6_common(p, rows, packed, nbr, nbr_stride, n_in, n_out, n_out_dev, f16_rows ? c_in / 2 : c_in / 4, c_out, kvol, a,
            shift, nullptr, relu, nullptr);
  p.residual_split = (const uint8_t *)residual_u8;
  p.out_split = (uint8_t *)out_image;
  p.qparams = qparams;
  p.out_half = out_half;
  // the same layers as BF16x3 take the wgmma kernel: >= kWgMinKBlocks K blocks of 32 channels
  if (p.c_out >= 64 && v6_nkb(c_in, kvol) >= kWgMinKBlocks) return f16_rows ? wg_launch<5>(p, st) : wg_launch<4>(p, st);
  return f16_rows ? v6_launch<5>(p, st) : v6_launch<4>(p, st);
}

// TF32 (tf32x3 = false) / 3xTF32 forward on zero-padded fp32 rows [n_in][c_in] (c_in a power of two, 8 .. 128) and
// the tf32 weight image of spconv_fwd.cu ([K block][hi (| lo)][Cout][32 fp32], chunk-swizzled like the bf16 images)
int spconv_v6_forward_tf32(const float *rows, const void *packed, const int32_t *nbr, int n_in, int n_out, int c_in,
                           int c_out, int kvol, bool tf32x3, const float *scale, const float *shift,
                           const float *residual, int relu, float *out, cudaStream_t st) {
  BEVB200_REQUIRE(c_in >= 8 && (c_in & (c_in - 1)) == 0 && spconv_v6_shape_ok(c_in, c_out, kvol),
                  "shape has no tensor-core form");
  if (n_out <= 0) return BEVB200_OK;
  V6Params p;
  v6_common(p, rows, packed, nbr, n_out, n_in, n_out, nullptr, c_in, c_out, kvol, scale, shift, residual, relu, out);
  return tf32x3 ? v6_launch<2>(p, st) : v6_launch<1>(p, st);
}

}  // namespace bevb200

using namespace bevb200;

extern "C" {

int bevb200_spconv_split_channels(int c_in) { return spconv_v6_cin_eff(c_in); }

int bevb200_spconv_split_rows(const float *features, int n, const int32_t *n_dev, int c_in, void *split,
                              void *stream) {
  BEVB200_REQUIRE(n >= 0 && c_in >= 1 && spconv_v6_cin_eff(c_in) != 0, "bad sizes");
  if (n == 0) return BEVB200_OK;
  BEVB200_REQUIRE(features && split && (uintptr_t)split % 16 == 0, "null / unaligned argument");
  return spconv_v6_split_rows(features, n, n_dev, c_in, spconv_v6_cin_eff(c_in), split, (cudaStream_t)stream);
}

size_t bevb200_spconv_split_weight_bytes(int c_in, int c_out, int kernel_volume) {
  return spconv_v6_packed_bytes(c_in, c_out, kernel_volume);
}

int bevb200_spconv_pack_split_weights(const float *weight, int c_in, int c_out, int kernel_volume, void *packed,
                                      void *stream) {
  BEVB200_REQUIRE(spconv_v6_shape_ok(c_in, c_out, kernel_volume), "shape has no tensor-core form");
  BEVB200_REQUIRE(weight && packed, "null argument");
  return spconv_v6_pack_weights(weight, c_in, c_out, kernel_volume, packed, (cudaStream_t)stream);
}

int bevb200_spconv_forward_split(const void *features_split, const void *packed_weight, const int32_t *nbr,
                                 long long nbr_stride, int n_in, int n_out, const int32_t *n_out_dev, int c_in,
                                 int c_out, int kernel_volume, const float *scale, const float *shift,
                                 const float *residual, int relu, float *out, void *out_split, void *stream) {
  BEVB200_REQUIRE(n_in >= 0 && n_out >= 0 && nbr_stride >= n_out, "bad sizes");
  BEVB200_REQUIRE(out != nullptr || out_split != nullptr, "no output requested");
  return spconv_v6_forward(features_split, packed_weight, nbr, nbr_stride, n_in, n_out, n_out_dev, c_in, c_out,
                           kernel_volume, scale, shift, residual, nullptr, relu, out, out_split, (cudaStream_t)stream);
}

}  // extern "C"
