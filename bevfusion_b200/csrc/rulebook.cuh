// Site-bitmap rulebook and dense() kernels (rulebook.cu).  Internal header: the per-conv C API and the
// encoder plan (encoder.cu) launch the same kernels through these host launchers.
//
// Kernels that walk rows take a host-side cap and a nullable device-side count n_dev: they use
// min(max(*n_dev, 0), cap) rows, or cap rows when n_dev is null.
#pragma once
#include "common.cuh"

namespace bevb200 {

// One conv from the grid of its input rows (in_shape) to the grid of its outputs (out_shape).
struct ConvGeom {
  int in_shape[3], out_shape[3], ksize[3], stride[3], pad[3], dil[3];
  int batch;
};

// Site bitmap of a dense grid of B*X*Y*Z sites, one uint2 cell per 32 sites: .x = the bits, .y = the number of set
// bits in all earlier words (written by rb_scan), so rank(site) = cell.y + popc(cell.x & below(bit)) -- ascending flat
// index order.  `status` / `ticket` are the state of the single-pass scan.  The first `bytes` bytes from `cells`
// (cells, status, ticket, total) must be zero before a bitmap is marked.
constexpr int kSiteScanThreads = 256, kSiteScanPer = 16, kSiteScanTile = kSiteScanThreads * kSiteScanPer;
struct SiteBitmap {
  uint2 *cells;
  unsigned long long *status;
  uint32_t *ticket, *total;
  size_t nwords, bytes;
};
inline SiteBitmap take_site_bitmap(Arena &a, long long sites) {
  SiteBitmap m;
  const size_t off = a.off;
  m.nwords = (size_t)((sites + 31) / 32);
  m.cells = a.take<uint2>(m.nwords);
  m.status = a.take<unsigned long long>((m.nwords + kSiteScanTile - 1) / kSiteScanTile + 1);
  m.ticket = a.take<uint32_t>(4);
  m.total = a.take<uint32_t>(4);
  m.bytes = a.off - off;
  return m;
}

// set the sites of rows inside g.in_shape
int rb_mark_rows(const int32_t *idx, int cap, const int32_t *n_dev, const ConvGeom &g, uint2 *cells, cudaStream_t st);
// input-side walk of a strided conv: set the output sites the input rows reach ...
int rb_mark_outputs(const int32_t *idx, int cap, const int32_t *n_dev, const ConvGeom &g, uint2 *cells_out,
                    cudaStream_t st);
// ... or, once ranked, write nbr[k][rank] = input row (nbr pre-filled with -1 by the caller)
int rb_fill_outputs(const int32_t *idx, int cap, const int32_t *n_dev, const ConvGeom &g, const uint2 *cells_out,
                    int n_out, int32_t *nbr, cudaStream_t st);
// cells[w].y = sum of popc(cells[v].x) over v < w, *total = the sum over all words; one launch
int rb_scan(const SiteBitmap &m, cudaStream_t st);
// rank2row[rank of a row's site] = the row
int rb_rank2row(const int32_t *idx, int cap, const int32_t *n_dev, const ConvGeom &g, const uint2 *cells,
                int32_t *rank2row, cudaStream_t st);
// *n_out = min(*total, cap); *overflow (nullable) |= 1 when the cap truncates
int rb_count(const uint32_t *total, int cap, int32_t *n_out, int32_t *overflow, cudaStream_t st);
// out_idx[rank] = (b, x, y, z) of every set site with rank < cap
int rb_out_indices(const SiteBitmap &m, const int shape[3], int cap, int32_t *out_idx, cudaStream_t st);
// output-side gather: nbr[k * nbr_stride + o] = row of the input site o * stride - pad + k * dil, or -1
// (the rank itself when rank2row is null)
int rb_gather(const int32_t *qidx, int qcap, const int32_t *nq_dev, const ConvGeom &g, const uint2 *cells_in,
              const int32_t *rank2row, int in_cap, int32_t *nbr, long long nbr_stride, cudaStream_t st);
// dense(): zero `out`, then scatter the rows (layout: bevb200_sparse_to_dense in the public header)
int sparse_to_dense(const float *features, const int32_t *idx, int cap, const int32_t *n_dev, int c, int batch,
                    const int shape[3], int z_major, long long out_batch_stride, float *out, cudaStream_t st);

}  // namespace bevb200
