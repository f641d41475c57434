// Radar feature net for sm_90a: decoration + 1..4 RFN layers (linear, BN, ReLU) + the slot max of
// mmdet3d/models/backbones/radar_encoder.py:47-184, on BF16x3 mma.sync tiles of 16 point rows.
//
// Semantics kept from the reference (DESIGN 4.12):
//   - row = [x, y, z normalised to the point-cloud range, the other F - 3 features, x - (cx*vx + x_off),
//     y - (cy*vy + y_off)] (the centre offsets from the raw x, y), then nan_to_num (NaN -> 0, +-inf -> +-FLT_MAX)
//   - every layer runs on all P slots; slots >= n are the same zero row, so a pillar with n < P takes the
//     max with one "virtual" row, a constant of the weights computed by the pack step; n == P takes none
//   - BN is folded per channel (eval statistics) and applied per row before the max
//
// Rows of all pillars are packed into one table (pillar order does not matter: each row's products do
// not depend on its tile neighbours, and the max below is exact in any order).  One warp per 16-row tile:
// the activations stay in shared memory as a bf16 hi | lo split image that the next layer's ldmatrix
// reads; the weights are pre-arranged in mma fragment order and read straight through L1.  The last
// layer's rows (>= 0 after ReLU) go into the zeroed output by atomicMax on their int bits: pillars may
// cross tile boundaries and the result is still bit-reproducible.
//
// Two row sources build the table: the [M, P, F] voxel tensor (RadarFeatureNet contract, rows out) and
// the hard voxelizer's per-voxel slot lists (K1-K4 of voxelize.cu), which never writes [M, P, F] and
// stores straight into the channels-first BEV canvas.
#include <cfloat>

#include "tc_ptx.cuh"
#include "voxelize.cuh"

namespace bevb200 {

constexpr int kRfnMaxLayers = 4, kRfnMaxC = 128, kRfnMaxP = 32, kRfnWarps = 4;
constexpr int kRfnPitch = (kRfnMaxC + 8) * 2;      // bytes per split-image row (272: ldmatrix conflict-free)
constexpr int kRfnPlane = 16 * kRfnPitch;         // hi plane, then lo plane
constexpr int kRfnYPitch = kRfnMaxC + 4;          // fp32 pitch of the last layer's rows (fits in both planes)
static_assert(16 * kRfnYPitch * 4 <= 2 * kRfnPlane, "last-layer rows do not fit the split image");

// packed image: per layer l the weight fragments (K_l/16 k-steps x N_l/8 n-tiles x 32 lanes of uint4
// {W_hi b0, W_hi b1, W_lo b0, W_lo b1}), then per layer scale [N_l] | shift [N_l], then the virtual row
struct RfnNet {
  int layers, f;           // layer count, point features F (layer-0 input is F + 2 columns)
  int k[kRfnMaxLayers];    // input columns, padded to 16
  int n[kRfnMaxLayers];    // output channels
  int frag[kRfnMaxLayers]; // offset of the layer's fragments, uint4 units
  int ss[kRfnMaxLayers];   // offset of scale (then shift), float units
  int vrow;                // offset of the virtual row, float units
  size_t bytes;
};

struct RfnGeom {
  float vx, vy, x_off, y_off;  // pillar centre = idx * v + off (radar_encoder.py:135-138)
  float lo[3], range[3];       // xyz normalisation (radar_encoder.py:162-164)
};

static bool rfn_layout(int in_channels, int n_layers, const int *widths, RfnNet *net) {
  if (in_channels < 3 || in_channels + 2 > kRfnMaxC || n_layers < 1 || n_layers > kRfnMaxLayers || !widths)
    return false;
  RfnNet t{};
  t.layers = n_layers;
  t.f = in_channels;
  size_t frag = 0;
  int k = (in_channels + 2 + 15) / 16 * 16;
  for (int l = 0; l < n_layers; ++l) {
    const int n = widths[l];
    if (n < 16 || n > kRfnMaxC || n % 16) return false;
    t.k[l] = k;
    t.n[l] = n;
    t.frag[l] = (int)frag;
    frag += (size_t)(k / 16) * (n / 8) * 32;
    k = n;
  }
  size_t fl = frag * 4;  // in floats
  for (int l = 0; l < n_layers; ++l) {
    t.ss[l] = (int)fl;
    fl += 2 * t.n[l];
  }
  t.vrow = (int)fl;
  fl += t.n[n_layers - 1];
  t.bytes = fl * sizeof(float);
  if (net) *net = t;
  return true;
}

// x = hi + lo with hi = rn_bf16(x) (truncated instead where rounding would overflow to inf, so +-FLT_MAX
// stays finite) and lo = rn_bf16(x - hi); bf16 bits in the low halves
__device__ __forceinline__ void split_bf16(float x, uint32_t &hi, uint32_t &lo) {
  uint32_t h = cvt_bf16x2(0.f, x) & 0xffffu;
  if ((h & 0x7f80u) == 0x7f80u && fabsf(x) <= FLT_MAX) h = __float_as_uint(x) >> 16;
  lo = cvt_bf16x2(0.f, x - __uint_as_float(h << 16)) & 0xffffu;
  hi = h;
}
__device__ __forceinline__ void split_pair_bf16(float x0, float x1, uint32_t &hi, uint32_t &lo) {
  uint32_t h0, l0, h1, l1;
  split_bf16(x0, h0, l0);
  split_bf16(x1, h1, l1);
  hi = h0 | (h1 << 16);
  lo = l0 | (l1 << 16);
}

__device__ __forceinline__ float nan_to_num(float v) {
  return v != v ? 0.f : fminf(fmaxf(v, -FLT_MAX), FLT_MAX);
}

struct __align__(16) RfnWarpSmem {
  uint8_t act[2 * kRfnPlane];  // split image [hi | lo][16 rows][kRfnPitch B]; the last layer's fp32 rows
  int row[16], out[16];
  int2 cxy[16];
};

// One layer on the warp's 16 rows: D[16, N] = A[16, K] W^T in BF16x3 (lo*W_hi + hi*W_lo + hi*W_hi, fp32
// accumulate), then folded BN and ReLU.  The result replaces A in place (split image), or for the last
// layer lands as fp32 rows of pitch kRfnYPitch.
template <int N, bool LAST>
__device__ __forceinline__ void rfn_layer(RfnWarpSmem &s, int ksteps, const uint4 *__restrict__ frag,
                                          const float *__restrict__ scale, const float *__restrict__ shift,
                                          int lane) {
  constexpr int NT = N / 8;
  float acc[NT][4];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
  const uint32_t a0 = smem_u32(s.act) + (uint32_t)((lane & 15) * kRfnPitch + (lane >> 4) * 16);
  for (int ks = 0; ks < ksteps; ++ks) {
    uint32_t ahi[4], alo[4];
    ldsm_x4(a0 + ks * 32, ahi);
    ldsm_x4(a0 + kRfnPlane + ks * 32, alo);
    const uint4 *f = frag + (size_t)ks * NT * 32 + lane;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const uint4 w = __ldg(f + nt * 32);
      mma_bf16_16816(acc[nt], alo, w.x, w.y);
      mma_bf16_16816(acc[nt], ahi, w.z, w.w);
      mma_bf16_16816(acc[nt], ahi, w.x, w.y);
    }
  }
  __syncwarp();  // every lane's ldmatrix of A is done before A is overwritten
  const int g = lane >> 2, c0 = 2 * (lane & 3);
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    const int c = nt * 8 + c0;
    const float2 sc = __ldg(reinterpret_cast<const float2 *>(scale + c));
    const float2 sh = __ldg(reinterpret_cast<const float2 *>(shift + c));
    const float y00 = fmaxf(fmaf(acc[nt][0], sc.x, sh.x), 0.f), y01 = fmaxf(fmaf(acc[nt][1], sc.y, sh.y), 0.f);
    const float y10 = fmaxf(fmaf(acc[nt][2], sc.x, sh.x), 0.f), y11 = fmaxf(fmaf(acc[nt][3], sc.y, sh.y), 0.f);
    if constexpr (LAST) {
      float *y = reinterpret_cast<float *>(s.act);
      *reinterpret_cast<float2 *>(y + g * kRfnYPitch + c) = make_float2(y00, y01);
      *reinterpret_cast<float2 *>(y + (g + 8) * kRfnYPitch + c) = make_float2(y10, y11);
    } else {
      uint32_t h, l;
      split_pair_bf16(y00, y01, h, l);
      *reinterpret_cast<uint32_t *>(s.act + g * kRfnPitch + c * 2) = h;
      *reinterpret_cast<uint32_t *>(s.act + kRfnPlane + g * kRfnPitch + c * 2) = l;
      split_pair_bf16(y10, y11, h, l);
      *reinterpret_cast<uint32_t *>(s.act + (g + 8) * kRfnPitch + c * 2) = h;
      *reinterpret_cast<uint32_t *>(s.act + kRfnPlane + (g + 8) * kRfnPitch + c * 2) = l;
    }
  }
  __syncwarp();
}

template <bool LAST>
__device__ __forceinline__ void rfn_layer_n(int n, RfnWarpSmem &s, int ksteps, const uint4 *frag, const float *scale,
                                            const float *shift, int lane) {
  switch (n) {
#define RFN_CASE(N) \
  case N: rfn_layer<N, LAST>(s, ksteps, frag, scale, shift, lane); break;
    RFN_CASE(16) RFN_CASE(32) RFN_CASE(48) RFN_CASE(64) RFN_CASE(80) RFN_CASE(96) RFN_CASE(112) RFN_CASE(128)
#undef RFN_CASE
    default: break;
  }
}

// Row table entry: {row index into `rows` (F floats each), output pillar index, cx, cy}.
// out[pillar * ps + c * cs] (rows form: [M, C], ps = C, cs = 1; canvas: ps = 1, cs = nx * ny).  The shape and
// geometry stay in parameter space (__grid_constant__): indexing them by layer needs no local copy.
__global__ void __launch_bounds__(kRfnWarps * 32)
    radar_tiles_kernel(const float *__restrict__ rows, const __grid_constant__ RfnGeom g,
                       const __grid_constant__ RfnNet net, const uint8_t *__restrict__ packed,
                       const int4 *__restrict__ table, const uint32_t *__restrict__ total_rows, int max_rows,
                       float *__restrict__ out, long long ps, long long cs) {
  __shared__ RfnWarpSmem sm[kRfnWarps];
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  RfnWarpSmem &s = sm[warp];
  const int total = (int)min(*total_rows, (uint32_t)max_rows);
  const int tiles = (total + 15) / 16, F = net.f, k0 = net.k[0];
  const uint4 *frag = reinterpret_cast<const uint4 *>(packed);
  const float *pf = reinterpret_cast<const float *>(packed);
  const int L = net.layers;
  int C = 0;
#pragma unroll
  for (int l = 0; l < kRfnMaxLayers; ++l) C = l == L - 1 ? net.n[l] : C;
  for (int tile = blockIdx.x * kRfnWarps + warp; tile < tiles; tile += gridDim.x * kRfnWarps) {
    if (lane < 16) {
      const int j = tile * 16 + lane;
      const int4 e = j < total ? table[j] : make_int4(0, -1, 0, 0);
      s.row[lane] = e.x;
      s.out[lane] = e.y;
      s.cxy[lane] = make_int2(e.z, e.w);
    }
    __syncwarp();
    // decorate the 16 rows into the split image; lane = column (point rows are 4 * F bytes, not 16-byte
    // aligned: each row is read as consecutive floats across the warp)
#pragma unroll 2
    for (int r = 0; r < 16; ++r) {
      const bool ok = s.out[r] >= 0;
      const float *p = rows + (long long)s.row[r] * F;
      const int2 cxy = s.cxy[r];
      for (int k = lane; k < k0; k += 32) {
        float v = 0.f;
        if (ok) {
          if (k < F) {
            v = p[k];
            if (k < 3) {
              const float lo = k == 0 ? g.lo[0] : k == 1 ? g.lo[1] : g.lo[2];
              const float span = k == 0 ? g.range[0] : k == 1 ? g.range[1] : g.range[2];
              v = __fdiv_rn(__fsub_rn(v, lo), span);
            }
          } else if (k < F + 2) {
            // coors * v + offset, two roundings as in the reference (no contraction into an FMA)
            const float c = (float)(k == F ? cxy.x : cxy.y);
            const float ctr = __fadd_rn(__fmul_rn(c, k == F ? g.vx : g.vy), k == F ? g.x_off : g.y_off);
            v = __fsub_rn(p[k - F], ctr);
          }
          v = nan_to_num(v);
        }
        uint32_t h, l;
        split_bf16(v, h, l);
        *reinterpret_cast<uint16_t *>(s.act + r * kRfnPitch + k * 2) = (uint16_t)h;
        *reinterpret_cast<uint16_t *>(s.act + kRfnPlane + r * kRfnPitch + k * 2) = (uint16_t)l;
      }
    }
    __syncwarp();
#pragma unroll
    for (int l = 0; l < kRfnMaxLayers; ++l) {  // one pass per layer slot; the last real one takes the max
      if (l < L - 1)
        rfn_layer_n<false>(net.n[l], s, net.k[l] / 16, frag + net.frag[l], pf + net.ss[l], pf + net.ss[l] + net.n[l],
                           lane);
      else if (l == L - 1)
        rfn_layer_n<true>(C, s, net.k[l] / 16, frag + net.frag[l], pf + net.ss[l], pf + net.ss[l] + C, lane);
    }
    // segmented max over the tile's rows (a pillar's rows are consecutive), then atomicMax: values are >= 0,
    // so their int bits order like the floats and the zeroed output is the identity
    const float *y = reinterpret_cast<const float *>(s.act);
    for (int c = lane; c < C; c += 32) {
      int cur = -1, best = 0;
      for (int r = 0; r < 16; ++r) {
        const int o = s.out[r];
        if (o < 0) break;
        if (o != cur) {
          if (cur >= 0 && best > 0) atomicMax(reinterpret_cast<int *>(out + cur * ps + c * cs), best);
          cur = o;
          best = 0;
        }
        best = max(best, __float_as_int(y[r * kRfnYPitch + c]));
      }
      if (cur >= 0 && best > 0) atomicMax(reinterpret_cast<int *>(out + cur * ps + c * cs), best);
    }
    __syncwarp();  // the next tile overwrites s
  }
}

// Warp-cooperative table fill for up to 32 pillars, one per lane: the warp reserves sum(cnt) rows with one
// atomic, every pillar's rows land consecutively, and pillars with n < P fold the virtual row into out.
// `row0` is the pillar's first row index (rows form) or, with `lists`, the slot-list base (fused form).
__device__ __forceinline__ void rfn_fill_table(int lane, int cnt, bool virt, int row0, const int32_t *lists,
                                               int out_idx, int cx, int cy, int4 *__restrict__ table,
                                               uint32_t *__restrict__ total_rows, const float *__restrict__ vrow,
                                               int C, float *__restrict__ out, long long ps, long long cs) {
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  const int sum = __shfl_sync(0xffffffffu, incl, 31);
  if (sum == 0 && !__any_sync(0xffffffffu, virt)) return;
  uint32_t base = 0;
  if (lane == 0 && sum > 0) base = atomicAdd(total_rows, (uint32_t)sum);
  base = __shfl_sync(0xffffffffu, base, 0);
  const int first = (int)base + incl - cnt;
  for (int p = 0; p < 32; ++p) {
    const int pc = __shfl_sync(0xffffffffu, cnt, p), pf = __shfl_sync(0xffffffffu, first, p);
    const int pr = __shfl_sync(0xffffffffu, row0, p), po = __shfl_sync(0xffffffffu, out_idx, p);
    const int px = __shfl_sync(0xffffffffu, cx, p), py = __shfl_sync(0xffffffffu, cy, p);
    const bool pv = __shfl_sync(0xffffffffu, (int)virt, p) != 0;
    if (lane < pc) table[pf + lane] = make_int4(lists ? lists[pr + lane] : pr + lane, po, px, py);
    if (pv)
      for (int c = lane; c < C; c += 32) {
        const int b = __float_as_int(vrow[c]);
        if (b > 0) atomicMax(reinterpret_cast<int *>(out + po * ps + c * cs), b);
      }
  }
}

// rows source: pillar v's rows are voxels[v, 0 .. min(n, P) - 1]
__global__ void radar_rows_table_kernel(const int32_t *__restrict__ num_points, const int32_t *__restrict__ coords4,
                                        int cap, const int32_t *__restrict__ n_dev, int P,
                                        const float *__restrict__ vrow, int C, int4 *__restrict__ table,
                                        uint32_t *__restrict__ total_rows, float *__restrict__ out) {
  const int lane = lane_id();
  const int m = n_dev ? min(*n_dev, cap) : cap;
  const int stride = gridDim.x * blockDim.x;
  for (int v0 = blockIdx.x * blockDim.x + (threadIdx.x & ~31); v0 < m; v0 += stride) {
    const int v = v0 + lane;
    int cnt = 0, cx = 0, cy = 0;
    bool virt = false;
    if (v < m) {
      const int n = num_points[v];
      cnt = min(max(n, 0), P);
      virt = n < P;
      cx = coords4[4ll * v + 1];
      cy = coords4[4ll * v + 2];
    }
    rfn_fill_table(lane, cnt, virt, v * P, nullptr, v, cx, cy, table, total_rows, vrow, C, out, C, 1);
  }
}

// fused source: the voxelizer's slot lists after K1-K4; one warp per 32-point word of first-point flags,
// lane l is the voxel whose first point is point 32 * word + l (if any)
__global__ void radar_points_table_kernel(const float *__restrict__ points, int F, int n_points, VoxParams vp, int P,
                                          int max_voxels, const int32_t *__restrict__ point_pvid,
                                          const int32_t *__restrict__ counts, const uint32_t *__restrict__ first_bits,
                                          const uint32_t *__restrict__ word_prefix,
                                          const uint32_t *__restrict__ total_voxels, long long nwords,
                                          const int32_t *__restrict__ lists, const float *__restrict__ vrow, int C,
                                          int4 *__restrict__ table, uint32_t *__restrict__ total_rows,
                                          float *__restrict__ canvas, int32_t *__restrict__ voxel_num) {
  if (blockIdx.x == 0 && threadIdx.x == 0) *voxel_num = (int32_t)min(*total_voxels, (uint32_t)max_voxels);
  const int lane = lane_id();
  const long long plane = (long long)vp.grid[0] * vp.grid[1];
  const long long wpb = blockDim.x >> 5;
  for (long long wd = blockIdx.x * wpb + (threadIdx.x >> 5); wd < nwords; wd += (long long)gridDim.x * wpb) {
    const uint32_t bits = first_bits[wd];
    const uint32_t vid = word_prefix[wd] + __popc(bits & ((1u << lane) - 1u));
    const long long i = wd * 32 + lane;
    int cnt = 0, c[3] = {0, 0, 0}, row0 = 0, cell = 0;
    if (((bits >> lane) & 1u) && vid < (uint32_t)max_voxels && i < n_points) {
      const int pv = point_pvid[i];
      cnt = min(counts[pv], P);
      point_coords(points + i * F, vp, c);
      cell = c[0] * vp.grid[1] + c[1];
      row0 = pv * P;
    }
    rfn_fill_table(lane, cnt, cnt > 0 && cnt < P, row0, lists, cell, c[0], c[1], table, total_rows, vrow, C, canvas,
                   1, plane);
  }
}

struct RfnPackArgs {
  const float *w[kRfnMaxLayers], *scale[kRfnMaxLayers], *shift[kRfnMaxLayers];
};

// weight fragments: for lane (g, t) of n-tile nt at k-step ks, b0 = W[n][k0, k0 + 1], b1 = W[n][k0 + 8, k0 + 9]
// with n = 8 nt + g, k0 = 16 ks + 2 t (the m16n8k16 B fragment; nn.Linear layout is already column-major B)
__global__ void radar_pack_frag_kernel(RfnPackArgs a, RfnNet net, uint4 *__restrict__ frag) {
  const int total = net.ss[0] / 4;  // the fragments end where the folded BN starts
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int l = net.layers - 1;
    while (l > 0 && i < net.frag[l]) --l;
    const int nt_count = net.n[l] / 8;
    const int j = i - net.frag[l], lane = j & 31, nt = (j >> 5) % nt_count, ks = (j >> 5) / nt_count;
    const int kin = l == 0 ? net.f + 2 : net.n[l - 1];
    const int n = nt * 8 + (lane >> 2), k0 = ks * 16 + 2 * (lane & 3);
    uint32_t hi[2], lo[2];
    for (int b = 0; b < 2; ++b) {
      const int k = k0 + 8 * b;
      const float x0 = k < kin ? a.w[l][n * kin + k] : 0.f, x1 = k + 1 < kin ? a.w[l][n * kin + k + 1] : 0.f;
      split_pair_bf16(x0, x1, hi[b], lo[b]);
    }
    frag[i] = make_uint4(hi[0], hi[1], lo[0], lo[1]);
  }
}

// folded BN per layer and the virtual row: the zero input row through every layer (fp32 FMA), one block
__global__ void __launch_bounds__(kRfnMaxC) radar_pack_vrow_kernel(RfnPackArgs a, RfnNet net, float *__restrict__ pf) {
  __shared__ float v[kRfnMaxC];
  const int c = threadIdx.x;
  v[c] = 0.f;
  __syncthreads();
  for (int l = 0; l < net.layers; ++l) {
    const int kin = l == 0 ? net.f + 2 : net.n[l - 1], n = net.n[l];
    float y = 0.f;
    if (c < n) {
      const float sc = a.scale[l][c], sh = a.shift[l][c];
      pf[net.ss[l] + c] = sc;
      pf[net.ss[l] + n + c] = sh;
      float acc = 0.f;
      for (int k = 0; k < kin; ++k) acc = fmaf(a.w[l][c * kin + k], v[k], acc);
      y = fmaxf(fmaf(acc, sc, sh), 0.f);
    }
    __syncthreads();
    v[c] = y;
    __syncthreads();
  }
  if (c < net.n[net.layers - 1]) pf[net.vrow + c] = v[c];
}

#define BEVB200_RADAR_UNSUPPORTED(cond, msg)                                            \
  do {                                                                                  \
    if (!(cond)) {                                                                      \
      snprintf(::bevb200::g_last_error, sizeof(::bevb200::g_last_error), "%s: %s [%s]", \
               __func__, msg, #cond);                                                   \
      return BEVB200_EUNSUPPORTED;                                                      \
    }                                                                                   \
  } while (0)

static const char *kRfnShapeMsg = "native radar net: 1..4 layers of widths 16..128 (multiples of 16), 3 <= F <= 126, "
                                  "1 <= P <= 32";

static size_t rfn_table_bytes(long long rows) { return align_up((size_t)rows * sizeof(int4)) + 256; }

static RfnGeom rfn_geom(float vx, float vy, float x_off, float y_off, const float *pc_min, const float *pc_span) {
  return RfnGeom{vx, vy, x_off, y_off, {pc_min[0], pc_min[1], pc_min[2]}, {pc_span[0], pc_span[1], pc_span[2]}};
}

static int rfn_tiles_grid(long long max_rows) { return grid_for((max_rows + 15) / 16, kRfnWarps, kNumSMs * 8); }

}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_radar_packed_bytes(int in_channels, int n_layers, const int *widths) {
  RfnNet net;
  return rfn_layout(in_channels, n_layers, widths, &net) ? net.bytes : 0;
}

int bevb200_radar_pack_weights(const float *const *weights, const float *const *scales, const float *const *shifts,
                               int in_channels, int n_layers, const int *widths, void *packed, void *stream) {
  RfnNet net;
  BEVB200_RADAR_UNSUPPORTED(rfn_layout(in_channels, n_layers, widths, &net), kRfnShapeMsg);
  BEVB200_REQUIRE(weights && scales && shifts && packed, "null argument");
  RfnPackArgs a{};
  for (int l = 0; l < n_layers; ++l) {
    BEVB200_REQUIRE(weights[l] && scales[l] && shifts[l], "null layer argument");
    a.w[l] = weights[l];
    a.scale[l] = scales[l];
    a.shift[l] = shifts[l];
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int nfrag = net.ss[0] / 4;
  BEVB200_LAUNCH(radar_pack_frag_kernel, grid_for(nfrag, 256), 256, 0, st, a, net, (uint4 *)packed);
  BEVB200_LAUNCH(radar_pack_vrow_kernel, 1, kRfnMaxC, 0, st, a, net, (float *)packed);
  return BEVB200_OK;
}

size_t bevb200_radar_features_workspace_bytes(int cap, int max_points) {
  if (cap < 0 || max_points < 1 || max_points > kRfnMaxP) return 0;
  return rfn_table_bytes((long long)cap * max_points);
}

int bevb200_radar_features(const float *voxels, const int32_t *num_points, const int32_t *coords4, int cap,
                           const int32_t *n_dev, int max_points, int num_features, int n_layers, const int *widths,
                           float vx, float vy, float x_off, float y_off, const float *pc_min, const float *pc_span,
                           const void *packed, float *out_rows, void *workspace, size_t workspace_bytes,
                           void *stream) {
  RfnNet net;
  BEVB200_RADAR_UNSUPPORTED(rfn_layout(num_features, n_layers, widths, &net), kRfnShapeMsg);
  BEVB200_RADAR_UNSUPPORTED(max_points >= 1 && max_points <= kRfnMaxP, kRfnShapeMsg);
  BEVB200_REQUIRE(cap >= 0 && (long long)cap * max_points < (1ll << 31), "bad sizes");
  BEVB200_REQUIRE(pc_min && pc_span, "null argument");
  if (cap == 0) return BEVB200_OK;
  BEVB200_REQUIRE(voxels && num_points && coords4 && packed && out_rows && workspace, "null argument");
  const long long max_rows = (long long)cap * max_points;
  BEVB200_REQUIRE(workspace_bytes >= rfn_table_bytes(max_rows), "workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int C = net.n[n_layers - 1];
  int4 *table = (int4 *)workspace;
  uint32_t *total = (uint32_t *)((uint8_t *)workspace + align_up((size_t)max_rows * sizeof(int4)));
  BEVB200_CUDA(cudaMemsetAsync(total, 0, sizeof(uint32_t), st));
  BEVB200_CUDA(cudaMemsetAsync(out_rows, 0, (size_t)cap * C * sizeof(float), st));
  const float *vrow = (const float *)packed + net.vrow;
  BEVB200_LAUNCH(radar_rows_table_kernel, grid_for(cap, 256), 256, 0, st, num_points, coords4, cap, n_dev,
                 max_points, vrow, C, table, total, out_rows);
  BEVB200_LAUNCH(radar_tiles_kernel, rfn_tiles_grid(max_rows), kRfnWarps * 32, 0, st, voxels,
                 rfn_geom(vx, vy, x_off, y_off, pc_min, pc_span), net, (const uint8_t *)packed, table, total,
                 (int)max_rows, out_rows, (long long)C, 1ll);
  return BEVB200_OK;
}

size_t bevb200_hard_voxelize_radar_workspace_bytes(int num_points, int max_points) {
  if (num_points < 0 || max_points < 1 || max_points > kRfnMaxP) return 0;
  return align_up(bevb200_hard_voxelize_workspace_bytes(num_points, max_points)) + rfn_table_bytes(num_points);
}

// the host-count and device-count fused entries: n rows (the host count, or the row cap with n_dev)
static int hard_voxelize_radar(const char *who, const float *points, int n, const int32_t *n_dev, int num_features,
                               const float *voxel_size_host, const float *coors_range_host, int max_points,
                               int max_voxels, int n_layers, const int *widths, float vx, float vy, float x_off,
                               float y_off, const float *pc_min, const float *pc_span, const void *packed,
                               float *canvas, int nx, int ny, int32_t *voxel_num, void *workspace,
                               size_t workspace_bytes, cudaStream_t st) {
  RfnNet net;
  BEVB200_RADAR_UNSUPPORTED(rfn_layout(num_features, n_layers, widths, &net), kRfnShapeMsg);
  BEVB200_RADAR_UNSUPPORTED(max_points >= 1 && max_points <= kRfnMaxP, kRfnShapeMsg);
  BEVB200_REQUIRE(n >= 0 && max_voxels > 0, "bad sizes");
  BEVB200_REQUIRE(voxel_size_host && coors_range_host && voxel_num && pc_min && pc_span, "null argument");
  VoxParams vp;
  BEVB200_REQUIRE(make_params(voxel_size_host, coors_range_host, &vp) == 0, "bad voxel grid");
  BEVB200_RADAR_UNSUPPORTED(vp.grid[2] == 1, "radar pillars need a voxel grid one cell high");
  BEVB200_REQUIRE(vp.grid[0] == nx && vp.grid[1] == ny, "canvas shape differs from the voxel grid");
  if (n == 0) {
    BEVB200_CUDA(cudaMemsetAsync(voxel_num, 0, sizeof(int32_t), st));
    return BEVB200_OK;
  }
  BEVB200_REQUIRE(points && packed && canvas && workspace, "null argument");
  BEVB200_REQUIRE(workspace_bytes >= bevb200_hard_voxelize_radar_workspace_bytes(n, max_points),
                  "workspace too small");
  const size_t vox_bytes = align_up(bevb200_hard_voxelize_workspace_bytes(n, max_points));
  int4 *table = (int4 *)((uint8_t *)workspace + vox_bytes);
  uint32_t *total = (uint32_t *)((uint8_t *)table + align_up((size_t)n * sizeof(int4)));
  BEVB200_CUDA(cudaMemsetAsync(total, 0, sizeof(uint32_t), st));
  VoxWs w;
  // with a device count of 0 no point is a voxel's first: the table stays empty, voxel_num becomes 0 and the
  // tiles kernel finds no rows, so the host early-out above needs no device twin
  int rc = vox_front(who, points, n, n_dev, num_features, vp, max_points, workspace, vox_bytes, st, &w);
  if (rc) return rc;
  const int C = net.n[n_layers - 1];
  const float *vrow = (const float *)packed + net.vrow;
  BEVB200_LAUNCH(radar_points_table_kernel, grid_for((long long)w.nwords, 8), 256, 0, st, points, num_features, n, vp,
                 max_points, max_voxels, w.point_pvid, w.counts, w.first_bits, w.word_prefix, w.total,
                 (long long)w.nwords, w.lists, vrow, C, table, total, canvas, voxel_num);
  BEVB200_LAUNCH(radar_tiles_kernel, rfn_tiles_grid(n), kRfnWarps * 32, 0, st, points,
                 rfn_geom(vx, vy, x_off, y_off, pc_min, pc_span), net, (const uint8_t *)packed, table, total, n,
                 canvas, 1ll, (long long)nx * ny);
  return BEVB200_OK;
}

int bevb200_hard_voxelize_radar(const float *points, int num_points, int num_features, const float *voxel_size_host,
                                const float *coors_range_host, int max_points, int max_voxels, int n_layers,
                                const int *widths, float vx, float vy, float x_off, float y_off, const float *pc_min,
                                const float *pc_span, const void *packed, float *canvas, int nx, int ny,
                                int32_t *voxel_num, void *workspace, size_t workspace_bytes, void *stream) {
  return hard_voxelize_radar("hard_voxelize_radar", points, num_points, nullptr, num_features, voxel_size_host,
                             coors_range_host, max_points, max_voxels, n_layers, widths, vx, vy, x_off, y_off, pc_min,
                             pc_span, packed, canvas, nx, ny, voxel_num, workspace, workspace_bytes,
                             (cudaStream_t)stream);
}

int bevb200_hard_voxelize_radar_dev(const float *points, const int32_t *num_points_dev, int max_rows,
                                    int num_features, const float *voxel_size_host, const float *coors_range_host,
                                    int max_points, int max_voxels, int n_layers, const int *widths, float vx,
                                    float vy, float x_off, float y_off, const float *pc_min, const float *pc_span,
                                    const void *packed, float *canvas, int nx, int ny, int32_t *voxel_num,
                                    void *workspace, size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(max_rows == 0 || num_points_dev, "null argument");
  return hard_voxelize_radar("hard_voxelize_radar_dev", points, max_rows, num_points_dev, num_features,
                             voxel_size_host, coors_range_host, max_points, max_voxels, n_layers, widths, vx, vy,
                             x_off, y_off, pc_min, pc_span, packed, canvas, nx, ny, voxel_num, workspace,
                             workspace_bytes, (cudaStream_t)stream);
}

}  // extern "C"
