// Sparse-conv rulebook for sm_90a (replaces spconv::getIndicePair<3>, spconv_ops.h:27-141,
// kernels indice.cu.h:22-203, geometry.h:24-85 `getValidOutPos`), and dense().
//
// The reference fills a dense int32 grid of the whole output volume (85 M ints = 340 MB at
// 1440x1440x41, re-allocated for every conv) and, for strided convs, sorts candidate outputs
// with torch::_unique.  Here the active sites live in a BITMAP of the dense grid (1 bit per site:
// 10.6 MB at 1440x1440x41, L2 resident) with a popcount prefix per word, interleaved in one uint2
// cell per 32 sites so that a lookup is one 8-byte load:
//     rank(site) = cell.y + popc(cell.x & below(bit))
// which IS the ascending-flat-index order the reference's GPU path produces for strided convs
// (no sort), and a membership test + rank lookup for SubM (through rank2row, because SubM
// keeps the input row order).  The prefix comes from a single-pass decoupled-look-back scan.
//
// Output: offset-major neighbour table nbr[k, o] (input row or -1); converters to / from the
// reference's indicePairs[K,2,N] + indiceNum[K] layout are provided for the drop-in API.
//
// The kernels serve both the per-conv C API below and the encoder plan (encoder.cu), which reaches
// them through the launchers declared in rulebook.cuh.
#include "rulebook.cuh"

namespace bevb200 {

__device__ __forceinline__ int row_count(const int32_t *n_dev, int cap) {
  const int n = n_dev ? __ldg(n_dev) : cap;
  return min(max(n, 0), cap);
}
__device__ __forceinline__ long long flat_site(int b, int x, int y, int z, const int shape[3]) {
  return (((long long)b * shape[0] + x) * shape[1] + y) * shape[2] + z;   // tensorview.h:453-464
}
__device__ __forceinline__ int site_rank(const uint2 cell, uint32_t bit) {
  if (!(cell.x & bit)) return -1;
  return (int)(cell.y + __popc(cell.x & (bit - 1)));
}

// active sites <- rows
__global__ void rb_mark_rows_kernel(const int32_t *__restrict__ idx, int cap, const int32_t *__restrict__ n_dev,
                                    ConvGeom g, uint2 *__restrict__ cells) {
  const int n = row_count(n_dev, cap);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int4 c = *reinterpret_cast<const int4 *>(idx + 4ll * i);   // (b, x, y, z)
    if ((unsigned)c.x >= (unsigned)g.batch || (unsigned)c.y >= (unsigned)g.in_shape[0] ||
        (unsigned)c.z >= (unsigned)g.in_shape[1] || (unsigned)c.w >= (unsigned)g.in_shape[2])
      continue;
    const long long s = flat_site(c.x, c.y, c.z, c.w, g.in_shape);
    atomicOr(&cells[s >> 5].x, 1u << (s & 31));
  }
}

// Input-side walk of a strided conv: the output site reached from input site q through kernel offset k is
// p = (q + pad - k*dil) / stride (exists iff divisible and inside the output grid) -- the set getValidOutPos
// enumerates.  One thread per input row; per dimension only the offsets with (q + pad - k*dil) % stride == 0
// reach an output site, so the thread walks the <= prod(ceil(K/s)) valid (kx, ky, kz) combinations (8 of 27
// for k3 s2).  MARK sets the output sites; FILL writes nbr[k][rank] = row into a table pre-filled with -1.
// FILL is the reference's scatter: a row just outside the input grid still feeds the border outputs it
// reaches, which the output-side gather (rb_gather_kernel) would not find.
template <bool FILL>
__global__ void rb_walk_kernel(const int32_t *__restrict__ idx, int cap, const int32_t *__restrict__ n_dev,
                               ConvGeom g, uint2 *__restrict__ cells_out, int n_out, int32_t *__restrict__ nbr) {
  const int n = row_count(n_dev, cap);
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const int4 c = *reinterpret_cast<const int4 *>(idx + 4ll * j);
    if ((unsigned)c.x >= (unsigned)g.batch) continue;
    const int q[3] = {c.y, c.z, c.w};
    for (int kx = 0; kx < g.ksize[0]; ++kx) {
      int vx = q[0] + g.pad[0] - kx * g.dil[0];
      if (vx < 0 || vx % g.stride[0]) continue;
      vx /= g.stride[0];
      if (vx >= g.out_shape[0]) continue;
      for (int ky = 0; ky < g.ksize[1]; ++ky) {
        int vy = q[1] + g.pad[1] - ky * g.dil[1];
        if (vy < 0 || vy % g.stride[1]) continue;
        vy /= g.stride[1];
        if (vy >= g.out_shape[1]) continue;
        for (int kz = 0; kz < g.ksize[2]; ++kz) {
          int vz = q[2] + g.pad[2] - kz * g.dil[2];
          if (vz < 0 || vz % g.stride[2]) continue;
          vz /= g.stride[2];
          if (vz >= g.out_shape[2]) continue;
          const long long s = flat_site(c.x, vx, vy, vz, g.out_shape);
          const uint32_t bit = 1u << (s & 31);
          if (FILL) {
            const int o = site_rank(__ldg(cells_out + (s >> 5)), bit);
            const int k = (kx * g.ksize[1] + ky) * g.ksize[2] + kz;
            if (o >= 0 && o < n_out) nbr[(long long)k * n_out + o] = j;
          } else if (!(cells_out[s >> 5].x & bit)) {
            atomicOr(&cells_out[s >> 5].x, bit);
          }
        }
      }
    }
  }
}

// ---- single-pass scan (decoupled look-back): cells[w].y = sum_{v < w} popc(cells[v].x) ----------
constexpr unsigned long long kFlagAgg = 1ull << 32, kFlagIncl = 2ull << 32;

__global__ void __launch_bounds__(kSiteScanThreads)
    rb_scan_kernel(uint2 *__restrict__ cells, size_t nwords, unsigned long long *status, uint32_t *ticket,
                   uint32_t *total) {
  __shared__ uint32_t s_warp[kSiteScanThreads / 32];
  __shared__ uint32_t s_tile, s_excl;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_tile = atomicAdd(ticket, 1u);     // tiles are taken in launch order: forward progress
  __syncthreads();
  const uint32_t tile = s_tile;
  const size_t base = (size_t)tile * kSiteScanTile + (size_t)tid * kSiteScanPer;
  uint32_t v[kSiteScanPer], sum = 0;
#pragma unroll
  for (int j = 0; j < kSiteScanPer; ++j) {
    v[j] = base + j < nwords ? (uint32_t)__popc(cells[base + j].x) : 0u;
    sum += v[j];
  }
  uint32_t incl = sum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  uint32_t woff = 0, tile_total = 0;
#pragma unroll
  for (int w = 0; w < kSiteScanThreads / 32; ++w) {
    const uint32_t x = s_warp[w];
    if (w < warp) woff += x;
    tile_total += x;
  }
  if (tid == 0) {
    uint32_t excl = 0;
    if (tile == 0) {
      atomicExch(status + 0, kFlagIncl | tile_total);
    } else {
      atomicExch(status + tile, kFlagAgg | tile_total);
      for (int j = (int)tile - 1; j >= 0; --j) {
        unsigned long long st;
        do {
          st = *reinterpret_cast<volatile unsigned long long *>(status + j);
        } while ((st >> 32) == 0);
        excl += (uint32_t)st;
        if ((st >> 32) == 2) break;
      }
      atomicExch(status + tile, kFlagIncl | (unsigned long long)(excl + tile_total));
    }
    s_excl = excl;
    if ((size_t)(tile + 1) * kSiteScanTile >= nwords) *total = excl + tile_total;
  }
  __syncthreads();
  uint32_t run = s_excl + woff + (incl - sum);
#pragma unroll
  for (int j = 0; j < kSiteScanPer; ++j) {
    if (base + j < nwords) cells[base + j].y = run;
    run += v[j];
  }
}

// rows that keep their own order (SubM, the encoder's level 0): rank (ascending site) -> row
__global__ void rb_rank2row_kernel(const int32_t *__restrict__ idx, int cap, const int32_t *__restrict__ n_dev,
                                   ConvGeom g, const uint2 *__restrict__ cells, int32_t *__restrict__ rank2row) {
  const int n = row_count(n_dev, cap);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int4 c = *reinterpret_cast<const int4 *>(idx + 4ll * i);
    if ((unsigned)c.x >= (unsigned)g.batch || (unsigned)c.y >= (unsigned)g.in_shape[0] ||
        (unsigned)c.z >= (unsigned)g.in_shape[1] || (unsigned)c.w >= (unsigned)g.in_shape[2])
      continue;
    const long long s = flat_site(c.x, c.y, c.z, c.w, g.in_shape);
    const int r = site_rank(__ldg(cells + (s >> 5)), 1u << (s & 31));
    if (r >= 0 && r < cap) rank2row[r] = i;   // duplicate coordinates: any one row wins (reference: last)
  }
}

__global__ void rb_count_kernel(const uint32_t *total, int cap, int32_t *n_out, int32_t *overflow) {
  const uint32_t t = *total;
  *n_out = t > (uint32_t)cap ? cap : (int)t;
  if (t > (uint32_t)cap && overflow) atomicOr(overflow, 1);
}

// rows built from a bitmap: ascending flat index = the reference's GPU order after torch::_unique
// (spconv_ops.h:130-136, indice.cu.h:112-127)
__global__ void rb_out_indices_kernel(const uint2 *__restrict__ cells, size_t nwords, int X, int Y, int Z, int cap,
                                      int32_t *__restrict__ out_idx) {
  for (size_t w = blockIdx.x * (size_t)blockDim.x + threadIdx.x; w < nwords; w += (size_t)gridDim.x * blockDim.x) {
    const uint2 cell = cells[w];
    uint32_t m = cell.x;
    if (!m) continue;
    int r = (int)cell.y;
    while (m) {
      const int bit = __ffs(m) - 1;
      m &= m - 1;
      long long s = ((long long)w << 5) + bit;
      const int z = (int)(s % Z); s /= Z;
      const int y = (int)(s % Y); s /= Y;
      const int x = (int)(s % X); s /= X;
      if (r < cap) *reinterpret_cast<int4 *>(out_idx + 4ll * r) = make_int4((int)s, x, y, z);
      ++r;
    }
  }
}

// nbr[k][o] = row of the input site (o * stride - pad + k * dil), or -1.  grid (row tiles, kx * ky): a
// thread walks the kz column of one (kx, ky); consecutive z are consecutive bits, so the column usually
// costs ONE 8-byte cell load.  Writes every entry: no -1 fill pass, coalesced stores.
__global__ void __launch_bounds__(256)
    rb_gather_kernel(const int32_t *__restrict__ qidx, int qcap, const int32_t *__restrict__ nq_dev, ConvGeom g,
                  const uint2 *__restrict__ cells_in, const int32_t *__restrict__ rank2row, int in_cap,
                  int32_t *__restrict__ nbr, long long nbr_stride) {
  const int n = row_count(nq_dev, qcap);
  const int kxy = blockIdx.y, ky = kxy % g.ksize[1], kx = kxy / g.ksize[1];
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < n; o += gridDim.x * blockDim.x) {
    const int4 c = *reinterpret_cast<const int4 *>(qidx + 4ll * o);
    const int x = c.y * g.stride[0] - g.pad[0] + kx * g.dil[0];
    const int y = c.z * g.stride[1] - g.pad[1] + ky * g.dil[1];
    const bool ok_xy = (unsigned)c.x < (unsigned)g.batch && (unsigned)x < (unsigned)g.in_shape[0] &&
                       (unsigned)y < (unsigned)g.in_shape[1];
    const long long col = ok_xy ? flat_site(c.x, x, y, 0, g.in_shape) : 0;
    long long cur_w = -1;
    uint2 cell = make_uint2(0u, 0u);
    for (int kz = 0; kz < g.ksize[2]; ++kz) {
      const int z = c.w * g.stride[2] - g.pad[2] + kz * g.dil[2];
      int row = -1;
      if (ok_xy && (unsigned)z < (unsigned)g.in_shape[2]) {
        const long long s = col + z;
        if ((s >> 5) != cur_w) {
          cur_w = s >> 5;
          cell = __ldg(cells_in + cur_w);
        }
        const int r = site_rank(cell, 1u << (s & 31));
        if (r >= 0 && r < in_cap) row = rank2row ? __ldg(rank2row + r) : r;
      }
      nbr[(long long)(kxy * g.ksize[2] + kz) * nbr_stride + o] = row;
    }
  }
}

// dense() + permute(0,1,4,2,3) + view(N, C*D, H, W) (structure.py:49-59, sparse_encoder.py:126-130)
__global__ void __launch_bounds__(256)
    sparse_to_dense_kernel(const float *__restrict__ features, const int32_t *__restrict__ idx, int cap,
                           const int32_t *__restrict__ n_dev, int c, int batch, int X, int Y, int Z, int z_major,
                           long long out_batch_stride, float *__restrict__ out) {
  // grid (row tiles, channel groups): a thread handles one site and the channels ch0, ch0+gridDim.y, ..
  // (site fastest across the warp: neighbouring sites -> nearby stores; no per-element division)
  const int n = row_count(n_dev, cap);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int4 p = *reinterpret_cast<const int4 *>(idx + 4ll * i);   // (b, x, y, z)
    if ((unsigned)p.x >= (unsigned)batch || (unsigned)p.y >= (unsigned)X || (unsigned)p.z >= (unsigned)Y ||
        (unsigned)p.w >= (unsigned)Z)
      continue;
    const long long site = z_major ? ((long long)p.w * X + p.y) * Y + p.z : ((long long)p.y * Y + p.z) * Z + p.w;
    const long long plane = (long long)X * Y * Z;
    float *o = out + p.x * out_batch_stride + site;
    for (int ch = blockIdx.y; ch < c; ch += gridDim.y) o[ch * plane] = features[(long long)i * c + ch];
  }
}

// ---- layout converters ----------------------------------------------------------------
// one CTA per kernel offset: ordered compaction of the valid (in, out) pairs
__global__ void __launch_bounds__(1024)
    rb_to_pairs_kernel(const int32_t *__restrict__ nbr, int n_out, int n_in,
                       int32_t *__restrict__ pairs, int32_t *__restrict__ num) {
  __shared__ int warp_cnt[32];
  __shared__ int carry_s;
  const int k = blockIdx.x, lane = lane_id(), warp = threadIdx.x >> 5;
  int32_t *pin = pairs + (2ll * k) * n_in, *pout = pairs + (2ll * k + 1) * n_in;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < n_out; base += blockDim.x) {
    int o = base + threadIdx.x;
    int j = o < n_out ? nbr[(long long)k * n_out + o] : -1;
    bool v = j >= 0;
    unsigned m = __ballot_sync(0xffffffffu, v);
    if (lane == 0) warp_cnt[warp] = __popc(m);
    __syncthreads();
    int off = carry_s;
    for (int w = 0; w < warp; ++w) off += warp_cnt[w];
    int pos = off + __popc(m & ((1u << lane) - 1));
    if (v && pos < n_in) { pin[pos] = j; pout[pos] = o; }
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += warp_cnt[w];
      carry_s += tot;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) num[k] = min(carry_s, n_in);
}

__global__ void rb_pairs_to_nbr_kernel(const int32_t *__restrict__ pairs,
                                       const int32_t *__restrict__ num, int kvol, int pairs_dim,
                                       int n_out, int inverse, int32_t *__restrict__ nbr) {
  const long long total = (long long)kvol * pairs_dim;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    int k = (int)(t / pairs_dim), p = (int)(t % pairs_dim);
    if (p >= num[k]) continue;
    int a = pairs[(2ll * k) * pairs_dim + p], b = pairs[(2ll * k + 1) * pairs_dim + p];
    int in = inverse ? b : a, out = inverse ? a : b;
    if (in >= 0 && out >= 0 && out < n_out) nbr[(long long)k * n_out + out] = in;
  }
}

// ---- launchers (rulebook.cuh) ------------------------------------------------------------
int rb_mark_rows(const int32_t *idx, int cap, const int32_t *n_dev, const ConvGeom &g, uint2 *cells, cudaStream_t st) {
  BEVB200_LAUNCH(rb_mark_rows_kernel, grid_for(cap, 256), 256, 0, st, idx, cap, n_dev, g, cells);
  return BEVB200_OK;
}

int rb_mark_outputs(const int32_t *idx, int cap, const int32_t *n_dev, const ConvGeom &g, uint2 *cells_out,
                    cudaStream_t st) {
  BEVB200_LAUNCH(rb_walk_kernel<false>, grid_for(cap, 128), 128, 0, st, idx, cap, n_dev, g, cells_out, 0,
                 (int32_t *)nullptr);
  return BEVB200_OK;
}

int rb_fill_outputs(const int32_t *idx, int cap, const int32_t *n_dev, const ConvGeom &g, const uint2 *cells_out,
                    int n_out, int32_t *nbr, cudaStream_t st) {
  // the FILL form only reads the cells
  BEVB200_LAUNCH(rb_walk_kernel<true>, grid_for(cap, 128), 128, 0, st, idx, cap, n_dev, g,
                 const_cast<uint2 *>(cells_out), n_out, nbr);
  return BEVB200_OK;
}

int rb_scan(const SiteBitmap &m, cudaStream_t st) {
  BEVB200_LAUNCH(rb_scan_kernel, (unsigned)((m.nwords + kSiteScanTile - 1) / kSiteScanTile), kSiteScanThreads, 0, st,
                 m.cells, m.nwords, m.status, m.ticket, m.total);
  return BEVB200_OK;
}

int rb_rank2row(const int32_t *idx, int cap, const int32_t *n_dev, const ConvGeom &g, const uint2 *cells,
                int32_t *rank2row, cudaStream_t st) {
  BEVB200_LAUNCH(rb_rank2row_kernel, grid_for(cap, 256), 256, 0, st, idx, cap, n_dev, g, cells, rank2row);
  return BEVB200_OK;
}

int rb_count(const uint32_t *total, int cap, int32_t *n_out, int32_t *overflow, cudaStream_t st) {
  BEVB200_LAUNCH(rb_count_kernel, 1, 1, 0, st, total, cap, n_out, overflow);
  return BEVB200_OK;
}

int rb_out_indices(const SiteBitmap &m, const int shape[3], int cap, int32_t *out_idx, cudaStream_t st) {
  BEVB200_LAUNCH(rb_out_indices_kernel, grid_for((long long)m.nwords, 256), 256, 0, st, m.cells, m.nwords, shape[0],
                 shape[1], shape[2], cap, out_idx);
  return BEVB200_OK;
}

int rb_gather(const int32_t *qidx, int qcap, const int32_t *nq_dev, const ConvGeom &g, const uint2 *cells_in,
              const int32_t *rank2row, int in_cap, int32_t *nbr, long long nbr_stride, cudaStream_t st) {
  BEVB200_LAUNCH(rb_gather_kernel, dim3(grid_for(qcap, 256, kNumSMs * 4), g.ksize[0] * g.ksize[1]), 256, 0, st, qidx,
                 qcap, nq_dev, g, cells_in, rank2row, in_cap, nbr, nbr_stride);
  return BEVB200_OK;
}

int sparse_to_dense(const float *features, const int32_t *idx, int cap, const int32_t *n_dev, int c, int batch,
                    const int shape[3], int z_major, long long out_batch_stride, float *out, cudaStream_t st) {
  const int X = shape[0], Y = shape[1], Z = shape[2];
  const long long per_batch = (long long)c * X * Y * Z;
  if (out_batch_stride == 0) out_batch_stride = per_batch;
  BEVB200_REQUIRE(out_batch_stride >= per_batch, "output batch stride too small");
  if (out_batch_stride == per_batch) {
    BEVB200_CUDA(cudaMemsetAsync(out, 0, (size_t)batch * per_batch * sizeof(float), st));
  } else {  // channel slice of a wider [B, C_total, ...] buffer (the fuser's concatenated input)
    BEVB200_CUDA(cudaMemset2DAsync(out, (size_t)out_batch_stride * sizeof(float), 0, (size_t)per_batch * sizeof(float),
                                   batch, st));
  }
  if (cap == 0) return BEVB200_OK;
  BEVB200_REQUIRE(features && idx, "null argument");
  BEVB200_LAUNCH(sparse_to_dense_kernel, dim3(grid_for(cap, 256, kNumSMs), c < 32 ? c : 32), 256, 0, st, features, idx,
                 cap, n_dev, c, batch, X, Y, Z, z_major, out_batch_stride, out);
  return BEVB200_OK;
}

// ---- per-conv rulebook: workspace = the bitmap of the output grid + rank2row -------------
static size_t rb_layout(int n_in, int batch, const int32_t *out_shape, void *ws, size_t ws_bytes, SiteBitmap *map,
                        int32_t **rank2row) {
  Arena a(ws, ws_bytes);
  const SiteBitmap m = take_site_bitmap(a, (long long)batch * out_shape[0] * out_shape[1] * out_shape[2]);
  int32_t *r2r = a.take<int32_t>(n_in > 0 ? n_in : 1);
  if (map) *map = m;
  if (rank2row) *rank2row = r2r;
  return a.off;
}

static int make_geom(int batch, const int32_t *in_shape, const int32_t *out_shape,
                     const int32_t *ksize, const int32_t *stride, const int32_t *pad,
                     const int32_t *dil, int subm, ConvGeom *g) {
  g->batch = batch;
  for (int d = 0; d < 3; ++d) {
    g->in_shape[d] = in_shape[d];
    g->out_shape[d] = out_shape[d];
    g->ksize[d] = ksize[d];
    g->dil[d] = dil[d];
    // spconv_ops.h:74-83: SubM forces stride 1 and padding k/2
    g->stride[d] = subm ? 1 : stride[d];
    g->pad[d] = subm ? ksize[d] / 2 : pad[d];
    if (ksize[d] <= 0 || g->stride[d] <= 0 || dil[d] <= 0 || out_shape[d] <= 0 || in_shape[d] <= 0 ||
        g->pad[d] < 0)
      return -1;
  }
  return 0;
}

}  // namespace bevb200

using namespace bevb200;

#define RB_COMMON_CHECKS()                                                                     \
  BEVB200_REQUIRE(n_in >= 0 && batch_size > 0, "bad sizes");                                   \
  BEVB200_REQUIRE(spatial_shape_host && out_shape_host && ksize_host && stride_host &&         \
                      padding_host && dilation_host, "null argument");                         \
  ConvGeom g;                                                                                  \
  BEVB200_REQUIRE(make_geom(batch_size, spatial_shape_host, out_shape_host, ksize_host,        \
                            stride_host, padding_host, dilation_host, subm, &g) == 0,          \
                  "bad convolution geometry");                                                 \
  const int kvol = g.ksize[0] * g.ksize[1] * g.ksize[2];                                       \
  BEVB200_REQUIRE(kvol <= 4096, "kernel volume > 4096 (spconv_ops.h:50)");                     \
  if (subm)                                                                                    \
    for (int d = 0; d < 3; ++d)                                                                \
      BEVB200_REQUIRE(out_shape_host[d] == spatial_shape_host[d], "SubM keeps the spatial shape"); \
  SiteBitmap map;                                                                              \
  int32_t *rank2row;                                                                           \
  size_t need = rb_layout(n_in, batch_size, out_shape_host, workspace, workspace_bytes, &map, &rank2row); \
  if (workspace == nullptr || workspace_bytes < need) {                                        \
    snprintf(g_last_error, sizeof(g_last_error), "rulebook: workspace too small (%zu < %zu)",  \
             workspace_bytes, need);                                                           \
    return BEVB200_EWORKSPACE;                                                                 \
  }                                                                                            \
  cudaStream_t st = (cudaStream_t)stream

extern "C" {

size_t bevb200_rulebook_workspace_bytes(int n_in, int batch_size, const int32_t *out_shape_host) {
  if (n_in < 0 || batch_size <= 0 || !out_shape_host) return 0;
  return rb_layout(n_in, batch_size, out_shape_host, nullptr, 0, nullptr, nullptr);
}

int bevb200_rulebook_prepare(const int32_t *indices, int n_in, int batch_size,
                             const int32_t *spatial_shape_host, const int32_t *out_shape_host,
                             const int32_t *ksize_host, const int32_t *stride_host,
                             const int32_t *padding_host, const int32_t *dilation_host, int subm,
                             int32_t *n_out, void *workspace, size_t workspace_bytes,
                             void *stream) {
  RB_COMMON_CHECKS();
  BEVB200_REQUIRE(n_out != nullptr, "null n_out");
  // the bitmap, its prefixes and the scan state start from zero on every call
  BEVB200_CUDA(cudaMemsetAsync(map.cells, 0, map.bytes, st));
  if (n_in == 0) {
    BEVB200_CUDA(cudaMemsetAsync(n_out, 0, sizeof(int32_t), st));
    return BEVB200_OK;
  }
  BEVB200_REQUIRE(indices != nullptr, "null indices");
  int rc = subm ? rb_mark_rows(indices, n_in, nullptr, g, map.cells, st)
                : rb_mark_outputs(indices, n_in, nullptr, g, map.cells, st);
  if (!rc) rc = rb_scan(map, st);
  if (rc) return rc;
  if (subm) {
    // every rank is written by the row that set its bit
    rc = rb_rank2row(indices, n_in, nullptr, g, map.cells, rank2row, st);
    if (rc) return rc;
    // SubM: outputs are the inputs, in input order (spconv_ops.h:101)
    int32_t n32 = n_in;
    BEVB200_CUDA(cudaMemcpyAsync(n_out, &n32, sizeof(int32_t), cudaMemcpyHostToDevice, st));
    return BEVB200_OK;
  }
  return rb_count(map.total, INT32_MAX, n_out, nullptr, st);
}

int bevb200_rulebook_fill(const int32_t *indices, int n_in, int batch_size,
                          const int32_t *spatial_shape_host, const int32_t *out_shape_host,
                          const int32_t *ksize_host, const int32_t *stride_host,
                          const int32_t *padding_host, const int32_t *dilation_host, int subm,
                          int n_out, int32_t *out_indices, int32_t *nbr, void *workspace,
                          size_t workspace_bytes, void *stream) {
  RB_COMMON_CHECKS();
  BEVB200_REQUIRE(n_out >= 0, "negative n_out");
  if (n_out == 0 || n_in == 0) return BEVB200_OK;
  BEVB200_REQUIRE(indices && nbr, "null argument");
  if (subm) {
    BEVB200_REQUIRE(n_out == n_in, "SubM: n_out must equal n_in");
    if (out_indices && out_indices != indices)
      BEVB200_CUDA(cudaMemcpyAsync(out_indices, indices, (size_t)n_in * 4 * sizeof(int32_t),
                                   cudaMemcpyDeviceToDevice, st));
    return rb_gather(indices, n_in, nullptr, g, map.cells, rank2row, n_in, nbr, n_in, st);
  }
  // strided: filled input-side, so rows just outside the input grid still reach border outputs
  BEVB200_REQUIRE(out_indices != nullptr, "null out_indices");
  BEVB200_CUDA(cudaMemsetAsync(nbr, 0xff, (size_t)kvol * n_out * sizeof(int32_t), st));
  int rc = rb_out_indices(map, g.out_shape, n_out, out_indices, st);
  if (rc) return rc;
  return rb_fill_outputs(indices, n_in, nullptr, g, map.cells, n_out, nbr, st);
}

int bevb200_rulebook_fill_subm_sorted(const int32_t *indices, int n, int batch_size,
                                      const int32_t *spatial_shape_host, const int32_t *ksize_host,
                                      const int32_t *dilation_host, int32_t *nbr, void *workspace,
                                      size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(n >= 0 && batch_size > 0, "bad sizes");
  BEVB200_REQUIRE(spatial_shape_host && ksize_host && dilation_host, "null argument");
  ConvGeom g;
  const int32_t ones[3] = {1, 1, 1}, zeros[3] = {0, 0, 0};
  BEVB200_REQUIRE(make_geom(batch_size, spatial_shape_host, spatial_shape_host, ksize_host, ones, zeros,
                            dilation_host, 1, &g) == 0, "bad convolution geometry");
  SiteBitmap map;
  size_t need = rb_layout(0, batch_size, spatial_shape_host, workspace, workspace_bytes, &map, nullptr);
  if (workspace == nullptr || workspace_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "rulebook: workspace too small (%zu < %zu)", workspace_bytes, need);
    return BEVB200_EWORKSPACE;
  }
  if (n == 0) return BEVB200_OK;
  BEVB200_REQUIRE(indices && nbr, "null argument");
  // the rows are the strided conv's outputs in rank order: the rank is the row
  return rb_gather(indices, n, nullptr, g, map.cells, nullptr, n, nbr, n, (cudaStream_t)stream);
}

int bevb200_rulebook_to_pairs(const int32_t *nbr, int kernel_volume, int n_out, int n_in,
                              int32_t *indice_pairs, int32_t *indice_num, void *stream) {
  BEVB200_REQUIRE(kernel_volume > 0 && n_out >= 0 && n_in >= 0, "bad sizes");
  BEVB200_REQUIRE(indice_num != nullptr, "null indice_num");
  cudaStream_t st = (cudaStream_t)stream;
  BEVB200_CUDA(cudaMemsetAsync(indice_num, 0, (size_t)kernel_volume * sizeof(int32_t), st));
  if (n_in == 0) return BEVB200_OK;
  BEVB200_REQUIRE(indice_pairs != nullptr, "null indice_pairs");
  BEVB200_CUDA(cudaMemsetAsync(indice_pairs, 0xff, (size_t)kernel_volume * 2 * n_in * sizeof(int32_t), st));
  if (n_out == 0) return BEVB200_OK;
  BEVB200_REQUIRE(nbr != nullptr, "null nbr");
  BEVB200_LAUNCH(rb_to_pairs_kernel, kernel_volume, 1024, 0, st, nbr, n_out, n_in, indice_pairs,
                 indice_num);
  return BEVB200_OK;
}

int bevb200_pairs_to_nbr(const int32_t *indice_pairs, const int32_t *indice_num,
                         int kernel_volume, int pairs_dim, int n_out, int inverse, int32_t *nbr,
                         void *stream) {
  BEVB200_REQUIRE(kernel_volume > 0 && pairs_dim >= 0 && n_out >= 0, "bad sizes");
  if (n_out == 0) return BEVB200_OK;
  BEVB200_REQUIRE(nbr != nullptr, "null nbr");
  cudaStream_t st = (cudaStream_t)stream;
  BEVB200_CUDA(cudaMemsetAsync(nbr, 0xff, (size_t)kernel_volume * n_out * sizeof(int32_t), st));
  if (pairs_dim == 0) return BEVB200_OK;
  BEVB200_REQUIRE(indice_pairs && indice_num, "null argument");
  BEVB200_LAUNCH(rb_pairs_to_nbr_kernel, grid_for((long long)kernel_volume * pairs_dim, 256), 256, 0,
                 st, indice_pairs, indice_num, kernel_volume, pairs_dim, n_out, inverse, nbr);
  return BEVB200_OK;
}

int bevb200_sparse_to_dense(const float *features, const int32_t *indices, int n, int c,
                            int batch_size, const int32_t *spatial_shape_host, int z_major,
                            long long out_batch_stride, float *out, void *stream) {
  BEVB200_REQUIRE(n >= 0 && c > 0 && batch_size > 0 && spatial_shape_host && out, "bad argument");
  const int shape[3] = {spatial_shape_host[0], spatial_shape_host[1], spatial_shape_host[2]};
  BEVB200_REQUIRE(shape[0] > 0 && shape[1] > 0 && shape[2] > 0, "bad spatial shape");
  return sparse_to_dense(features, indices, n, nullptr, c, batch_size, shape, z_major, out_batch_stride, out,
                         (cudaStream_t)stream);
}

}  // extern "C"
