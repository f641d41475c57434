/*
 * bevfusion_b200.h -- C ABI of libbevfusion_b200.so (sm_90a / NVIDIA H100).
 *
 * Drop-in boundary for the BEVFusion view-transform / LiDAR-voxel hot path of
 * mit-han-lab/bevfusion (reference tree mounted at /root/reference in the build
 * container; citations are file:line in that tree).  Every entry point takes plain
 * device pointers, sizes and a CUDA stream; no torch types cross this boundary.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _host
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream)
 *   - return value: 0 on success, negative BEVB200_E* on failure; the failing
 *     call's message is available from bevb200_last_error() (thread-local)
 *   - calls are asynchronous on `stream`; none of them synchronises the device
 *   - no global mutable state: re-entrant across host threads / streams as long
 *     as the caller gives each in-flight call its own workspace
 *   - workspaces: query the *_workspace_bytes() function, allocate that many bytes
 *     (256-B aligned) and pass them in; contents are scratch
 *   - there is NO CPU fallback anywhere in this library
 */
#ifndef BEVFUSION_B200_H_
#define BEVFUSION_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define BEVB200_API __attribute__((visibility("default")))
#else
#define BEVB200_API
#endif

#define BEVB200_OK 0
#define BEVB200_EINVAL (-1)    /* bad argument (null pointer, bad size, unsupported shape) */
#define BEVB200_ECUDA (-2)     /* CUDA runtime / launch error */
#define BEVB200_EWORKSPACE (-3) /* workspace too small */
#define BEVB200_EUNSUPPORTED (-4)

BEVB200_API int bevb200_version(void);
BEVB200_API const char *bevb200_last_error(void);
/* number of kernels launched by this library on the calling thread since the last
 * reset (bench.py's "gpu_launches" figure comes from here) */
BEVB200_API long long bevb200_launch_count(void);
BEVB200_API void bevb200_reset_launch_count(void);

/* ------------------------------------------------------------------------------------
 * bev_pool  (reference: mmdet3d/ops/bev_pool/src/bev_pool_cuda.cu, bev_pool_cpu.cpp)
 * ---------------------------------------------------------------------------------- */

/* Replaces `void bev_pool(int b,int d,int h,int w,int n,int c,int n_intervals,
 *                         const float* x,const int* geom_feats,const int* interval_starts,
 *                         const int* interval_lengths,float* out)`
 * (bev_pool_cuda.cu:86-90, called from bev_pool_forward bev_pool_cpu.cpp:22-47).
 *   x               [n, c] fp32, rows sorted by rank (the op's contract)
 *   geom_feats      [n, 4] int32 (x, y, z, b) of each sorted row
 *   interval_starts [n_intervals], interval_lengths [n_intervals] int32; interval i is
 *                   rows [starts[i], starts[i] + lengths[i]) of x, and the cell of its
 *                   first row receives their sum.  Intervals ascend and do not overlap,
 *                   but need not tile [0, n): rows outside every interval contribute
 *                   nothing.  A row whose geom_feats lies outside the grid heads no cell.
 *   out             [b, d, h, w, c] fp32; EVERY element is written (cells without an
 *                   interval get 0), so the caller need not pre-zero it
 * Differences from the reference launcher: runs on `stream` (the reference uses the
 * legacy default stream, bev_pool_cuda.cu:88); sums each interval with a fixed
 * chunked order (deterministic run to run).
 * workspace: bevb200_bev_pool_workspace_bytes(n, c); a smaller one gives
 * BEVB200_EWORKSPACE.  A call refused with BEVB200_EINVAL or BEVB200_EWORKSPACE leaves
 * `out` untouched. */
BEVB200_API size_t bevb200_bev_pool_workspace_bytes(int n, int c);
BEVB200_API int bevb200_bev_pool(int b, int d, int h, int w, int n, int c, int n_intervals,
                     const float *x, const int32_t *geom_feats,
                     const int32_t *interval_starts, const int32_t *interval_lengths,
                     float *out, void *workspace, size_t workspace_bytes, void *stream);

/* Replaces `void bev_pool_grad(...)` (bev_pool_cuda.cu:92-96, called from
 * bev_pool_backward bev_pool_cpu.cpp:60-87).
 *   out_grad [b, d, h, w, c] fp32 contiguous -> x_grad [n, c] fp32 (sorted-row order).
 * Every row of x_grad that belongs to an interval is written; rows not covered by any
 * interval (none, for intervals produced by the reference's QuickCumsumCuda) are zeroed. */
BEVB200_API int bevb200_bev_pool_grad(int b, int d, int h, int w, int n, int c, int n_intervals,
                          const float *out_grad, const int32_t *geom_feats,
                          const int32_t *interval_starts, const int32_t *interval_lengths,
                          float *x_grad, void *stream);

/* native variants of the two calls above: rows are read (written) through `perm`,
 * the sorted->original row map produced by bevb200_bev_pool_prepare_*, so that the
 * caller never materialises x[kept][argsort] (base.py:168, bev_pool.py:94).
 *   x / x_grad  [n_total, c] in ORIGINAL (unsorted, unfiltered) order
 *   perm        [n_total] int32: perm[i] for i < n = original row of sorted row i; the tail
 *               perm[n .. n_total) lists the filtered-out rows (only bev_pool_grad_perm reads it)
 * These calls REQUIRE tables produced by bevb200_bev_pool_prepare_* (intervals tile [0, n) in
 * ascending rank order); bev_pool_perm relies on that to zero-fill the empty cells in the same
 * pass.  bev_pool_grad_perm zero-fills the rows of x_grad that were filtered out. */
BEVB200_API int bevb200_bev_pool_perm(int b, int d, int h, int w, int n, int c, int n_intervals,
                          const float *x, const int32_t *perm, const int32_t *geom_feats,
                          const int32_t *interval_starts, const int32_t *interval_lengths,
                          float *out, void *workspace, size_t workspace_bytes, void *stream);
BEVB200_API int bevb200_bev_pool_grad_perm(int b, int d, int h, int w, int n, int n_total, int c,
                               int n_intervals, const float *out_grad, const int32_t *perm,
                               const int32_t *geom_feats, const int32_t *interval_starts,
                               const int32_t *interval_lengths, float *x_grad, void *stream);

/* Op layout [B, Z, X, Y, C] -> module layout [B, Z*C, X, Y] in one tiled transpose: replaces
 * `x.permute(0, 4, 1, 2, 3).contiguous()` (bev_pool.py:97) + `torch.cat(x.unbind(dim=2), 1)`
 * (base.py:174).  rows = X*Y.  out_batch_stride (floats; 0 = nz*rows*c) lets `out` be a channel
 * slice of a wider [B, C_total, X, Y] buffer, i.e. the camera half of the fuser's concatenated
 * input (fusers/conv.py:16 `torch.cat(inputs, dim=1)`) written in place. */
BEVB200_API int bevb200_bev_channels_first(const float *in, float *out, int batch, int nz, int rows, int c,
                                           long long out_batch_stride, void *stream);

/* Fused LSS lift + pool ("next" row (f)1 of SURVEY.md section 8; BEVPoolv2-style): the lifted volume
 * x[p, :] = depth[p] * ctx[pixel(p), :] of LSSTransform / DepthLSSTransform.get_cam_feats
 * (mmdet3d/models/vtransforms/lss.py:68-73, depth_lss.py:92-97) is never materialised; the pooling
 * kernel gathers the (L2-resident) context row and the depth weight of every kept frustum point:
 *     out[cell] = sum_{p in cell} fp32(depth[p] * ctx[pixel(p), :])
 *   depth  [n_total] fp32 = softmax depth volume flattened as [B*N, D, fH*fW]
 *   ctx    [B*N*fH*fW, c] fp32, channels-last context features
 *   original point index i -> pixel row (i / (depth_bins*pixels_per_camera)) * pixels_per_camera
 *                                       + i % pixels_per_camera
 * Tables as for bevb200_bev_pool_perm (from bevb200_bev_pool_prepare_geom).  Backward:
 * bevb200_bev_pool_lift_backward (any feature height) and bevb200_bev_pool_lift_columns_backward below.
 * workspace: bevb200_bev_pool_workspace_bytes(n, c).  A call refused with BEVB200_EINVAL or BEVB200_EWORKSPACE
 * leaves `out` untouched. */
BEVB200_API int bevb200_bev_pool_lift(int b, int d, int h, int w, int n, int c, int n_intervals,
                          const float *depth, const float *ctx, int depth_bins,
                          int pixels_per_camera, const int32_t *perm, const int32_t *geom_feats,
                          const int32_t *interval_starts, const int32_t *interval_lengths,
                          float *out, void *workspace, size_t workspace_bytes, void *stream);

/* Column formulation of the fused lift + pool (round 2).  The BEV grid collapses z, so the fH pixels of one image
 * column (cam, w) at one depth bin (almost) always fall into one cell: the kept points are grouped into SEGMENTS
 * (column, depth bin, cell) with a bit mask over the pixel row h (feature_h <= 64), a segment's value
 *     T[seg, :] = sum_{h in mask} fp32(depth[cam, d, h, w] * ctx[cam, h, w, :])
 * is evaluated from ONE shared-memory copy of the column's context rows and depth values, and a cell is the sum of
 * its segments in a fixed order.  Nothing is assumed about the cameras (tilt or the z filter only add segments).
 * Reads depth + ctx once (13.4 MB at C2) instead of one 320-byte context row per kept point (588 MB through L2).
 *   bevb200_bev_pool_lift_prepare   per calibration, from the tables of bevb200_bev_pool_prepare_*: perm [n_kept]
 *       (sorted -> original index over [cameras, depth_bins, feature_h, feature_w], cameras = B*N) and
 *       interval_starts.  Outputs (device): col_begin int32[cameras*feature_w + 1], seg_key / seg_mask
 *       uint64[n_kept] (first n_segments entries valid; key = ((column*depth_bins + d) << 32) | interval),
 *       seg_slot int32[n_kept], interval_slot_begin int32[n_intervals + 1], n_segments int32[1].
 *       Synchronises the stream once (it needs the segment count).
 *   bevb200_bev_pool_lift_columns   per frame: depth [cameras, depth_bins, feature_h, feature_w] fp32,
 *       ctx [cameras, feature_h, feature_w, c] fp32 -> out [b, d, h, w, c] (fully written).  n_segments as read
 *       back from the prepare call; workspace: bevb200_bev_pool_lift_columns_workspace_bytes().  A call refused
 *       with BEVB200_EINVAL or BEVB200_EWORKSPACE leaves `out` untouched. */
BEVB200_API size_t bevb200_bev_pool_lift_prepare_workspace_bytes(int n_kept);
BEVB200_API int bevb200_bev_pool_lift_prepare(const int32_t *perm, const int32_t *interval_starts, int n_kept,
                                  int n_intervals, int cameras, int depth_bins, int feature_h, int feature_w,
                                  int32_t *col_begin, uint64_t *seg_key, uint64_t *seg_mask, int32_t *seg_slot,
                                  int32_t *interval_slot_begin, int32_t *n_segments, void *workspace,
                                  size_t workspace_bytes, void *stream);
BEVB200_API size_t bevb200_bev_pool_lift_columns_workspace_bytes(int n_segments, int n_intervals, int c);
BEVB200_API int bevb200_bev_pool_lift_columns(int b, int d, int h, int w, int n, int c, int n_intervals,
                                  const float *depth, const float *ctx, int cameras, int depth_bins,
                                  int feature_h, int feature_w, const int32_t *geom_feats,
                                  const int32_t *interval_starts, const int32_t *col_begin,
                                  const uint64_t *seg_key, const uint64_t *seg_mask, const int32_t *seg_slot,
                                  const int32_t *interval_slot_begin, int n_segments, float *out,
                                  void *workspace, size_t workspace_bytes, void *stream);

/* Backward of the fused lift + pool.  With G = out_grad [b, d, h, w, c] fp32 (the gradient of the raw pooled output)
 * and cell(p) the cell of the kept frustum point p = (cam, d, h, w):
 *     ddepth[cam, d, h, w] = sum_c ctx[cam, h, w, c] * G[cell(p), c]     (0 where p is filtered)
 *     dctx[cam, h, w, :]   = sum over the kept d of depth[cam, d, h, w] * G[cell(p), :]
 * without the lifted volume or its gradient.  ddepth [cameras, depth_bins, feature_h, feature_w] and
 * dctx [cameras, feature_h, feature_w, c] fp32 are fully written (no pre-zeroing); either may be NULL, and that
 * gradient is skipped.  c in {16, 32, 64, 80, 96, 128, 160, 256}; ctx, dctx and out_grad 16-byte aligned.  No float
 * atomics: the result is bit-reproducible run to run.  No host synchronisation (graph-capturable).
 *   bevb200_bev_pool_lift_columns_backward   feature_h <= 64, over the segment tables of bevb200_bev_pool_lift_prepare
 *       (seg_slot / interval_slot_begin are not needed).  One CTA per image column; the column's G rows are staged in
 *       shared memory in chunks, so any number of depth bins / segments per column works.
 *       workspace: bevb200_bev_pool_lift_columns_backward_workspace_bytes() (one int per segment).
 *   bevb200_bev_pool_lift_backward           any feature_h, over the plain tables of bevb200_bev_pool_prepare_*
 *       (perm [n_total] including the filtered tail, as for bevb200_bev_pool_grad_perm); depth / ctx laid out as for
 *       bevb200_bev_pool_lift.  One warp per pixel walks the depth bins in order.
 *       workspace: bevb200_bev_pool_lift_backward_workspace_bytes() (one int per frustum point).
 * The workspace queries return 0 for bad sizes or an unsupported channel count. */
BEVB200_API size_t bevb200_bev_pool_lift_columns_backward_workspace_bytes(int n_segments, int n_intervals, int c);
BEVB200_API int bevb200_bev_pool_lift_columns_backward(int b, int d, int h, int w, int n, int c, int n_intervals,
                                  const float *out_grad, const float *depth, const float *ctx, int cameras,
                                  int depth_bins, int feature_h, int feature_w, const int32_t *geom_feats,
                                  const int32_t *interval_starts, const int32_t *col_begin, const uint64_t *seg_key,
                                  const uint64_t *seg_mask, int n_segments, float *ddepth, float *dctx,
                                  void *workspace, size_t workspace_bytes, void *stream);
BEVB200_API size_t bevb200_bev_pool_lift_backward_workspace_bytes(int n_total, int c);
BEVB200_API int bevb200_bev_pool_lift_backward(int b, int d, int h, int w, int n, int n_total, int c,
                                  int n_intervals, const float *out_grad, const float *depth, const float *ctx,
                                  int depth_bins, int pixels_per_camera, const int32_t *perm,
                                  const int32_t *geom_feats, const int32_t *interval_starts,
                                  const int32_t *interval_lengths, float *ddepth, float *dctx, void *workspace,
                                  size_t workspace_bytes, void *stream);

/* Sync-free twins (*_dev) of the pooling, lift and lift-prepare calls above, for tables rebuilt every step without a
 * host round trip (augmented training, per-sample calibration) and for CUDA-graph capture of that rebuild.  Each twin
 * runs the same kernels as its host-count call, but reads the sizes from device memory:
 *   counts_dev   int32[2] = {n_kept, n_intervals} as bevb200_bev_pool_prepare_* writes them
 *   n_capacity   the size every table was allocated for (n_total, the frustum points of the plan): grids are sized from
 *                it and the kernels stop at the device counts, so n_kept and n_intervals never reach the host
 *   max_segments the capacity of the column tables (seg_key / seg_mask / seg_slot); 1 <= max_segments <= n_capacity
 *   lift_form    int32[1] status word written by bevb200_bev_pool_lift_prepare_dev: BEVB200_LIFT_COLUMNS when the
 *                device segment count fits under max_segments, BEVB200_LIFT_ROWS when it does not.  A lift call of a
 *                form the word does not name launches its kernels, which exit at once: a caller launches both forms
 *                (columns, then rows) and exactly one writes the output.  The column twins require it; the row twins
 *                take NULL for "always run".
 * Results are bit-identical to the host-count call on the same tables, including the zero-filled cells and rows for
 * n_kept == 0 or n_intervals == 0.  Every argument is checked before the first write; a capacity <= 0 is refused.  The
 * workspace queries take capacities and return 0 for a capacity <= 0 (or an unsupported channel count where the
 * host-count query does).  None of these calls synchronises the host.
 *   bevb200_bev_pool_perm_dev / _grad_perm_dev            bevb200_bev_pool_perm / _grad_perm; tables [n_capacity]
 *   bevb200_bev_pool_lift_dev / _lift_backward_dev        the row lift (any feature_h) and its backward
 *   bevb200_bev_pool_lift_prepare_dev                     column tables from device n_kept / n_intervals: sorts all
 *       n_capacity keys (rows past n_kept sort last), writes n_segments[1] and lift_form[1]; interval_slot_begin
 *       int32[n_capacity + 1], seg_* [max_segments].  Past the cap the column tables are not filled.
 *   bevb200_bev_pool_lift_columns_dev / _columns_backward_dev   the column lift and its backward (feature_h <= 64) */
#define BEVB200_LIFT_COLUMNS 0
#define BEVB200_LIFT_ROWS 1
BEVB200_API size_t bevb200_bev_pool_dev_workspace_bytes(int n_capacity, int c);
BEVB200_API int bevb200_bev_pool_perm_dev(int b, int d, int h, int w, int n_capacity, int c, const float *x,
                                  const int32_t *perm, const int32_t *geom_feats, const int32_t *interval_starts,
                                  const int32_t *interval_lengths, const int32_t *counts_dev, float *out,
                                  void *workspace, size_t workspace_bytes, void *stream);
BEVB200_API int bevb200_bev_pool_grad_perm_dev(int b, int d, int h, int w, int n_total, int c, const float *out_grad,
                                  const int32_t *perm, const int32_t *geom_feats, const int32_t *interval_starts,
                                  const int32_t *interval_lengths, const int32_t *counts_dev, float *x_grad,
                                  void *stream);
BEVB200_API int bevb200_bev_pool_lift_dev(int b, int d, int h, int w, int n_capacity, int c, const float *depth,
                                  const float *ctx, int depth_bins, int pixels_per_camera, const int32_t *perm,
                                  const int32_t *geom_feats, const int32_t *interval_starts,
                                  const int32_t *interval_lengths, const int32_t *counts_dev,
                                  const int32_t *lift_form, float *out, void *workspace, size_t workspace_bytes,
                                  void *stream);
BEVB200_API size_t bevb200_bev_pool_lift_prepare_dev_workspace_bytes(int n_capacity, int max_segments);
BEVB200_API int bevb200_bev_pool_lift_prepare_dev(const int32_t *perm, const int32_t *interval_starts,
                                  const int32_t *counts_dev, int n_capacity, int max_segments, int cameras,
                                  int depth_bins, int feature_h, int feature_w, int32_t *col_begin, uint64_t *seg_key,
                                  uint64_t *seg_mask, int32_t *seg_slot, int32_t *interval_slot_begin,
                                  int32_t *n_segments, int32_t *lift_form, void *workspace, size_t workspace_bytes,
                                  void *stream);
BEVB200_API size_t bevb200_bev_pool_lift_columns_dev_workspace_bytes(int max_segments, int n_capacity, int c);
BEVB200_API int bevb200_bev_pool_lift_columns_dev(int b, int d, int h, int w, int n_capacity, int c,
                                  const float *depth, const float *ctx, int cameras, int depth_bins, int feature_h,
                                  int feature_w, const int32_t *geom_feats, const int32_t *interval_starts,
                                  const int32_t *col_begin, const uint64_t *seg_key, const uint64_t *seg_mask,
                                  const int32_t *seg_slot, const int32_t *interval_slot_begin, int max_segments,
                                  const int32_t *counts_dev, const int32_t *lift_form, float *out, void *workspace,
                                  size_t workspace_bytes, void *stream);
BEVB200_API size_t bevb200_bev_pool_lift_columns_backward_dev_workspace_bytes(int max_segments, int c);
BEVB200_API int bevb200_bev_pool_lift_columns_backward_dev(int b, int d, int h, int w, int n_capacity, int c,
                                  const float *out_grad, const float *depth, const float *ctx, int cameras,
                                  int depth_bins, int feature_h, int feature_w, const int32_t *geom_feats,
                                  const int32_t *interval_starts, const int32_t *col_begin, const uint64_t *seg_key,
                                  const uint64_t *seg_mask, int max_segments, const int32_t *counts_dev,
                                  const int32_t *n_segments_dev, const int32_t *lift_form, float *ddepth, float *dctx,
                                  void *workspace, size_t workspace_bytes, void *stream);
BEVB200_API size_t bevb200_bev_pool_lift_backward_dev_workspace_bytes(int n_total, int c);
BEVB200_API int bevb200_bev_pool_lift_backward_dev(int b, int d, int h, int w, int n_total, int c,
                                  const float *out_grad, const float *depth, const float *ctx, int depth_bins,
                                  int pixels_per_camera, const int32_t *perm, const int32_t *geom_feats,
                                  const int32_t *interval_starts, const int32_t *interval_lengths,
                                  const int32_t *counts_dev, const int32_t *lift_form, float *ddepth, float *dctx,
                                  void *workspace, size_t workspace_bytes, void *stream);


/* bev_pool precompute.  Replaces, on device and in one call, the index glue of
 * BaseTransform.bev_pool (mmdet3d/models/vtransforms/base.py:149-169: quantise, batch
 * index, bounds mask), bev_pool() (ops/bev_pool/bev_pool.py:87-94: rank, argsort,
 * gathers) and QuickCumsumCuda.forward (bev_pool.py:41-46: interval table).
 *
 *   geom_xyz   [n_total, 3] fp32 lidar-frame frustum points (get_geometry output)
 *   n_per_batch  n_total / B (batch index of point i is i / n_per_batch, base.py:151-157)
 *   lower_host[3] = (bx - dx/2) evaluated in fp32 exactly as base.py:149 does,
 *   dx_host[3], nx_host[3] = grid cells along x, y, z (base.py:15-21)
 *   idx = trunc_toward_zero((g - lower) / dx) in fp32; kept iff 0 <= idx_k < nx_k
 *   rank = x*(W*D*B) + y*(D*B) + z*B + b with (B, D, H, W) = (B, nz, nx, ny)
 * Outputs (all sized for the worst case n_total):
 *   ranks_sorted [n_total] int32, perm [n_total] int32 (ascending original index
 *   inside equal ranks -- a stable sort; the reference's argsort is unstable so any
 *   order is within its contract), geom_sorted [n_total, 4] int32 (x, y, z, b),
 *   interval_starts / interval_lengths [n_total] int32,
 *   counts [2] int32 = {n_kept, n_intervals}  (device memory; read it back once)
 */
BEVB200_API size_t bevb200_bev_pool_prepare_workspace_bytes(int n_total);
BEVB200_API int bevb200_bev_pool_prepare_geom(const float *geom_xyz, int n_total, int n_per_batch,
                                  const float *lower_host, const float *dx_host,
                                  const int32_t *nx_host, int B, int32_t *ranks_sorted,
                                  int32_t *perm, int32_t *geom_sorted,
                                  int32_t *interval_starts, int32_t *interval_lengths,
                                  int32_t *counts, void *workspace, size_t workspace_bytes,
                                  void *stream);
/* Same, starting from already quantised int64 coords [n, 4] = (x, y, z, b) as handed to
 * bev_pool() (bev_pool.py:84).  Rows outside [0,H)x[0,W)x[0,D)x[0,B) are dropped
 * (the reference would write out of bounds for them). */
/* bevb200_bev_pool_prepare_geom with BaseTransform.get_geometry (mmdet3d/models/vtransforms/base.py:92-135) fused in:
 * the lidar-frame frustum points are computed inside the rank pass and the 96 MB [B, N, D, fH, fW, 3] tensor is never
 * written (geom_out, nullable, receives it for checks).  Explicit fp32 arithmetic, products summed left to right:
 *   p = frustum - post_trans;  q = inv(post_rot) p;  u = (q.x q.z, q.y q.z, q.z);  v = (R inv(K)) u + t;
 *   optionally v = extra_R v + extra_t (the lidar augmentation, per batch item).
 * frustum [n_frustum, 3] = (u, v, d) of create_frustum (base.py:66-89); cam_params [cameras, 24] =
 * {inv(post_rot) 9, post_trans 3, camera2lidar_rot . inv(intrinsics) 9, camera2lidar_trans 3} -- the 3x3 inverses and
 * the product are the caller's (torch, as the reference computes them); extra_params [B, 12] or NULL; cameras = B *
 * cams_per_batch.  Not bit-identical to torch's batched matmul (whose summation order is unspecified): a frustum point
 * within an ulp of a cell boundary can land in the neighbouring cell. */
BEVB200_API int bevb200_bev_pool_prepare_cameras(const float *frustum, int n_frustum, int cameras, int cams_per_batch,
                                     const float *cam_params, const float *extra_params,
                                     const float *lower_host, const float *dx_host, const int32_t *nx_host, int B,
                                     float *geom_out, int32_t *ranks_sorted, int32_t *perm, int32_t *geom_sorted,
                                     int32_t *interval_starts, int32_t *interval_lengths, int32_t *counts,
                                     void *workspace, size_t workspace_bytes, void *stream);
BEVB200_API int bevb200_bev_pool_prepare_coords(const int64_t *coords, int n, int B, int D, int H, int W,
                                    int32_t *ranks_sorted, int32_t *perm,
                                    int32_t *geom_sorted, int32_t *interval_starts,
                                    int32_t *interval_lengths, int32_t *counts,
                                    void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------
 * voxelization (reference: mmdet3d/ops/voxel/src/voxelization.h, voxelization_cuda.cu)
 * ---------------------------------------------------------------------------------- */

/* Replaces voxelization::hard_voxelize_gpu (voxelization_cuda.cu:231-373; bound as
 * voxel_layer.hard_voxelize, voxelization.h:58-81), deterministic=True semantics:
 *   - c_k = (int)floor((p_k - min_k) / vs_k) in fp32, valid iff 0 <= c_k < grid_k,
 *     grid_k = round((max_k - min_k) / vs_k)                 (:37-58, :256-258)
 *   - voxel ids in order of first appearance by point index; only the first
 *     max_voxels distinct voxels are kept                     (:149-180)
 *   - a point's slot = number of earlier points in its voxel; kept iff < max_points
 *   - voxels[v, slot, :] = points[i, :], coors[v] = (cx, cy, cz) (x,y,z order in this
 *     fork), num_points_per_voxel[v] = min(count, max_points)
 * The caller pre-zeroes voxels / coors / num_points_per_voxel at cap size
 * (voxelize.py:52-54); only used slots are written.  The number of voxels is written to
 * voxel_num (DEVICE int32[1]) -- the reference returns it as a host int after a device
 * sync (:369-370); the host wrapper does that read.
 * No O(N^2) scan, no <<<1,1>>> kernel, no device synchronisation. */
BEVB200_API size_t bevb200_hard_voxelize_workspace_bytes(int num_points, int max_points);
BEVB200_API int bevb200_hard_voxelize(const float *points, int num_points, int num_features,
                          const float *voxel_size_host, const float *coors_range_host,
                          int max_points, int max_voxels, float *voxels, int32_t *coors,
                          int32_t *num_points_per_voxel, int32_t *voxel_num,
                          void *workspace, size_t workspace_bytes, void *stream);

/* Fused voxelize + mean-reduce + batch pad: what BEVFusion.voxelize does around the op when
 * voxelize_reduce is on (mmdet3d/models/fusion_models/bevfusion.py:169-197 -- hard_voxelize, then
 * `feats.sum(dim=1) / sizes` and `F.pad(coords, (1, 0), value=k)`), without materialising the
 * [M, max_points, F] voxel tensor.  Same voxel order / caps as bevb200_hard_voxelize.
 *   feats  [max_voxels, F] mean point row per voxel (slot-order fp32 sum, IEEE divide)
 *   coords4 [max_voxels, 4] int32 (batch_idx, x, y, z), 16-byte aligned
 *   num_points_per_voxel [max_voxels] (nullable), voxel_num device int32
 * Rows >= voxel_num are left untouched.  F <= 8.  Workspace as bevb200_hard_voxelize. */
BEVB200_API int bevb200_hard_voxelize_mean(const float *points, int num_points, int num_features,
                               const float *voxel_size_host, const float *coors_range_host,
                               int max_points, int max_voxels, int batch_idx, float *feats,
                               int32_t *coords4, int32_t *num_points_per_voxel, int32_t *voxel_num,
                               void *workspace, size_t workspace_bytes, void *stream);

/* bevb200_hard_voxelize_mean on the first *num_points_dev (DEVICE int32[1], clamped to [0, max_rows]) rows of
 * points [max_rows, F]: the same outputs, bit for bit, as bevb200_hard_voxelize_mean with that host count, without
 * reading the count on the host.  Workspace as bevb200_hard_voxelize_workspace_bytes(max_rows, max_points). */
BEVB200_API int bevb200_hard_voxelize_mean_dev(const float *points, const int32_t *num_points_dev, int max_rows,
                                               int num_features, const float *voxel_size_host,
                                               const float *coors_range_host, int max_points, int max_voxels,
                                               int batch_idx, float *feats, int32_t *coords4,
                                               int32_t *num_points_per_voxel, int32_t *voxel_num, void *workspace,
                                               size_t workspace_bytes, void *stream);

/* Replaces voxelization::dynamic_voxelize_gpu (voxelization_cuda.cu:485-528):
 * coors[i] = (cx, cy, cz) or (-1,-1,-1) when the point is out of range.  (The reference
 * kernel only guarantees coors[i][0] == -1 for such points, :38-47.) */
BEVB200_API int bevb200_dynamic_voxelize(const float *points, int num_points, int num_features,
                             const float *voxel_size_host, const float *coors_range_host,
                             int32_t *coors, void *stream);

/* Fused BEVFusion.voxelize glue (mmdet3d/models/fusion_models/bevfusion.py:183,191-195):
 * feats[v, :] = sum_slot voxels[v, slot, :] / num[v]  and coords[v] = (batch_idx, x, y, z). */
BEVB200_API int bevb200_voxel_mean(const float *voxels, const int32_t *coors, const int32_t *num_points,
                       int num_voxels, int max_points, int num_features, int batch_idx,
                       float *feats, int32_t *coords4, void *stream);

/* ---- PointPillars pillar feature net (mmdet3d/models/backbones/pillar_encoder.py:20-258) -----------
 * The shipped PillarFeatureNet: in_channels F, feat_channels [64, 64], with_distance False, eval-mode
 * BN folded into per-channel scale / shift.  Per pillar v with n = num_points[v] and P slots:
 *   rows = [raw F, xyz - sum_slots(xyz) / n, x - (cx*vx + x_off), y - (cy*vy + y_off)], slots >= n zero
 *   x1 = relu(s1 * (rows W1^T) + t1)            [P, 32]   (a zero row gives relu(t1))
 *   out = max_slots relu(s2 * ([x1, max_slots x1] W2^T) + t2)   [64]
 * Padded slots take part in both maxes (a pillar with n < P has one extra row, n == P none).  Exact fp32,
 * bit-reproducible (no atomics).
 *
 * bevb200_pillar_packed_bytes() is 0 unless 3 <= in_channels <= 8, c1 == 32 (layer-1 units) and c2 == 64;
 * bevb200_pillar_pack_weights() builds the packed image from device fp32 w1 [32, F+5], w2 [64, 64]
 * (nn.Linear layout) and the folded BN scale / shift of each layer, BEVB200_EUNSUPPORTED otherwise. */
BEVB200_API size_t bevb200_pillar_packed_bytes(int in_channels, int c1, int c2);
BEVB200_API int bevb200_pillar_pack_weights(const float *w1, const float *scale1, const float *shift1,
                                const float *w2, const float *scale2, const float *shift2, int in_channels,
                                int c1, int c2, float *packed, void *stream);

/* PillarFeatureNet.forward (:141-176): voxels [cap, P, F] fp32, num_points [cap] int32 (>= 1),
 * coords4 [cap, 4] int32 (b, x, y, z); out_rows [cap, 64] fp32.  Pillars v < min(*n_dev, cap) are
 * computed (n_dev nullable: cap), other rows are left untouched.  1 <= P <= 32 and 3 <= F <= 8, else
 * BEVB200_EUNSUPPORTED. */
BEVB200_API int bevb200_pillar_features(const float *voxels, const int32_t *num_points, const int32_t *coords4,
                            int cap, const int32_t *n_dev, int max_points, int num_features, float vx,
                            float vy, float x_off, float y_off, const float *packed, float *out_rows,
                            void *stream);

/* Hard voxelization + pillar feature net + PointPillarsScatter for one sample: the pillars of
 * bevb200_hard_voxelize (same order and caps) go through the net above straight from the point rows,
 * without the [M, P, F] voxel tensor, and land in canvas [64, nx, ny] fp32 at (x, y).  The caller
 * zeroes the canvas.  The voxel grid must be (nx, ny, 1), else BEVB200_EINVAL / BEVB200_EUNSUPPORTED.
 * voxel_num is the device pillar count; no host synchronisation.  Workspace as bevb200_hard_voxelize. */
BEVB200_API int bevb200_hard_voxelize_pillars(const float *points, int num_points, int num_features,
                                  const float *voxel_size_host, const float *coors_range_host,
                                  int max_points, int max_voxels, float vx, float vy, float x_off,
                                  float y_off, const float *packed, float *canvas, int nx, int ny,
                                  int32_t *voxel_num, void *workspace, size_t workspace_bytes,
                                  void *stream);

/* ---- Radar feature net (mmdet3d/models/backbones/radar_encoder.py:47-220) ---------------------------
 * RadarFeatureNet with in_channels F and feat_channels [C_0 .. C_{L-1}], eval-mode BN folded into
 * per-channel scale / shift.  Per pillar v with n = num_points[v], coords (b, cx, cy, z) and P slots:
 *   row = [(xyz - pc_min) / pc_span, features 3..F-1, x - (cx*vx + x_off), y - (cy*vy + y_off)]
 *         (the centre offsets from the raw x, y), nan_to_num (NaN -> 0, +-inf -> +-FLT_MAX)
 *   x_{l+1} = relu(s_l * (x_l W_l^T) + t_l) for every row;   out = max over the rows   [C_{L-1}]
 * Padded slots are zero rows: a pillar with n < P also takes the max with the "virtual" row (the zero
 * row through every layer, computed once by the pack step), one with n == P does not.  The linears run
 * as BF16x3 mma.sync (lo*W_hi + hi*W_lo + hi*W_hi, fp32 accumulate); the result is bit-reproducible and
 * identical between the two forms below.  pc_min / pc_span are HOST float[3] (pc_span = pc_max - pc_min,
 * computed in double and rounded once).
 *
 * bevb200_radar_packed_bytes() is 0 unless 1 <= n_layers <= 4, every width (host int[n_layers]) is a
 * multiple of 16 in 16..128 and 3 <= in_channels <= 126; bevb200_radar_pack_weights() builds the packed
 * image from host arrays of n_layers device pointers: weights[l] fp32 [C_l, C_{l-1}] (nn.Linear layout,
 * C_{-1} = F + 2), scales[l] / shifts[l] fp32 [C_l].  Unsupported shapes give BEVB200_EUNSUPPORTED. */
BEVB200_API size_t bevb200_radar_packed_bytes(int in_channels, int n_layers, const int *widths);
BEVB200_API int bevb200_radar_pack_weights(const float *const *weights, const float *const *scales,
                                           const float *const *shifts, int in_channels, int n_layers,
                                           const int *widths, void *packed, void *stream);

/* RadarFeatureNet.forward (:141-184): voxels [cap, P, F] fp32, num_points [cap] int32, coords4 [cap, 4]
 * int32 (b, x, y, z); out_rows [cap, C_{L-1}] fp32 is zeroed, then pillars v < min(*n_dev, cap) are
 * computed (n_dev nullable: cap).  Slots >= n of voxels are never read.  1 <= P <= 32, else
 * BEVB200_EUNSUPPORTED.  Workspace: bevb200_radar_features_workspace_bytes(cap, P) device bytes. */
BEVB200_API size_t bevb200_radar_features_workspace_bytes(int cap, int max_points);
BEVB200_API int bevb200_radar_features(const float *voxels, const int32_t *num_points, const int32_t *coords4,
                                       int cap, const int32_t *n_dev, int max_points, int num_features,
                                       int n_layers, const int *widths, float vx, float vy, float x_off,
                                       float y_off, const float *pc_min, const float *pc_span, const void *packed,
                                       float *out_rows, void *workspace, size_t workspace_bytes, void *stream);

/* Hard voxelization + radar feature net + PointPillarsScatter for one sample: the pillars of
 * bevb200_hard_voxelize (same order and caps) go through the net above straight from the point rows,
 * without the [M, P, F] voxel tensor, and land in canvas [C_{L-1}, nx, ny] fp32 at (x, y).  The caller
 * zeroes the canvas.  The voxel grid must be (nx, ny, 1).  voxel_num is the device pillar count; no host
 * synchronisation.  Workspace: bevb200_hard_voxelize_radar_workspace_bytes(num_points, P) device bytes. */
BEVB200_API size_t bevb200_hard_voxelize_radar_workspace_bytes(int num_points, int max_points);
BEVB200_API int bevb200_hard_voxelize_radar(const float *points, int num_points, int num_features,
                                            const float *voxel_size_host, const float *coors_range_host,
                                            int max_points, int max_voxels, int n_layers, const int *widths,
                                            float vx, float vy, float x_off, float y_off, const float *pc_min,
                                            const float *pc_span, const void *packed, float *canvas, int nx,
                                            int ny, int32_t *voxel_num, void *workspace, size_t workspace_bytes,
                                            void *stream);

/* bevb200_hard_voxelize_radar on the first *num_points_dev (DEVICE int32[1], clamped to [0, max_rows]) rows of
 * points [max_rows, F]: the same canvas and voxel_num, bit for bit, as bevb200_hard_voxelize_radar with that host
 * count, without reading the count on the host (a device count of 0 leaves the canvas as it is and sets voxel_num
 * to 0).  Workspace: bevb200_hard_voxelize_radar_workspace_bytes(max_rows, P) device bytes. */
BEVB200_API int bevb200_hard_voxelize_radar_dev(const float *points, const int32_t *num_points_dev, int max_rows,
                                                int num_features, const float *voxel_size_host,
                                                const float *coors_range_host, int max_points, int max_voxels,
                                                int n_layers, const int *widths, float vx, float vy, float x_off,
                                                float y_off, const float *pc_min, const float *pc_span,
                                                const void *packed, float *canvas, int nx, int ny, int32_t *voxel_num,
                                                void *workspace, size_t workspace_bytes, void *stream);

/* ---- Rotated BEV IoU and NMS (mmdet3d/ops/iou3d/src/{iou3d.cpp,iou3d_kernel.cu},
 *      core/post_processing/box3d_nms.py:180-219 circle_nms) ----------------------------------------
 * Boxes are [x1, y1, x2, y2, ry] fp32 (xywhr2xyxyr form): the axis-aligned extent turned by ry about its
 * centre, x' = (x-cx) cos r + (y-cy) sin r + cx, y' = -(x-cx) sin r + (y-cy) cos r + cy
 * (iou3d_kernel.cu:116-124).  overlap = area of box a clipped by box b in b's own frame (Sutherland-Hodgman);
 * iou = overlap / max(sa + sb - overlap, 1e-8) with sa, sb the
 * unrotated extents' areas (:249-256).  A box with a NaN coordinate overlaps nothing (IoU 0).  fp32: the
 * value differs from the reference's own fp32 arithmetic in the last bits (DESIGN.md section 4.13). */

/* boxes_overlap_bev_gpu / boxes_iou_bev_gpu (iou3d.cpp:48-94): a [na, 5], b [nb, 5] fp32 ->
 * out [na, nb] fp32 row-major, every element written.  na <= 1,048,560, else BEVB200_EINVAL. */
BEVB200_API int bevb200_boxes_iou_bev(const float *a, int na, const float *b, int nb, float *out, void *stream);
BEVB200_API int bevb200_boxes_overlap_bev(const float *a, int na, const float *b, int nb, float *out,
                                          void *stream);

/* Greedy NMS over S independent segments (one (task, sample) box list each), replacing nms_gpu /
 * nms_normal_gpu (iou3d.cpp:96-210, host loop :132-145) and circle_nms, in two launches and without
 * host synchronisation or allocation:
 *   boxes      [S, nmax, D] fp32, each segment sorted by descending score; D = 5 ([x1, y1, x2, y2, ry])
 *              for ROTATE and NORMAL, D = 2 (centre x, y) for CIRCLE
 *   counts     [S] int32 device, boxes of segment s are rows [0, counts[s]) (clamped to [0, nmax]);
 *              nullable: every segment holds nmax
 *   mode       ROTATE: pair (i, j) suppressed when rotated iou > (float)thresh (iou3d_kernel.cu:300);
 *              NORMAL: the axis-aligned iou of :335-343 (ry ignored) > (float)thresh;
 *              CIRCLE: fp32 dx*dx + dy*dy <= thresh compared in double (box3d_nms.py:213-216; thresh is
 *              the config's min_radius, compared with the squared distance as the reference does)
 *   order      [S, nmax] int64 device, nullable: keep holds order[s, i] instead of the sorted position i
 *   keep       [S, post_max] int64 device: kept boxes in score order, the first keep_count[s] entries of
 *              the greedy keep list, the rest -1.  keep_count [S] int32 device = min(kept, post_max).
 * The result equals the reference's host loop bit for bit for the same suppression mask.  An empty
 * segment gives keep_count 0.  nmax <= BEVB200_NMS_MAX_BOXES (the suppression bitmap lives in shared
 * memory) and S <= BEVB200_NMS_MAX_SEGMENTS, else BEVB200_EUNSUPPORTED.  Workspace (the pair mask,
 * S * nmax * ceil(nmax / 64) * 8 bytes): bevb200_nms_workspace_bytes(S, nmax), 0 for unsupported sizes;
 * a smaller one gives BEVB200_EWORKSPACE. */
#define BEVB200_NMS_ROTATE 0
#define BEVB200_NMS_NORMAL 1
#define BEVB200_NMS_CIRCLE 2
#define BEVB200_NMS_MAX_BOXES 65536
#define BEVB200_NMS_MAX_SEGMENTS 65535
BEVB200_API size_t bevb200_nms_workspace_bytes(int S, int nmax);
BEVB200_API int bevb200_nms(const float *boxes, const int32_t *counts, int S, int nmax, int mode, double thresh,
                            int post_max, const int64_t *order, int64_t *keep, int32_t *keep_count,
                            void *workspace, size_t workspace_bytes, void *stream);

/* ---- Heatmap training targets of CenterHead and TransFusionHead (centerpoint.py:432-582
 *      get_targets_single, the heatmap block of transfusion.py:526-573, core/utils/gaussian.py) ------------
 * Three launches (zero, assign, draw), no host synchronisation, no allocation; CUDA-graph capturable.
 *   boxes       [B, nmax, box_dim] fp32 device, LiDARInstance3DBoxes.tensor rows (x, y, z_bottom, dx, dy, dz, yaw
 *               [, vx, vy]); box_dim 7 or 9
 *   labels      [B, nmax] int32 device; counts [B] int32 device (sample b is rows [0, counts[b]), clamped to
 *               [0, nmax]; nullable: every sample holds nmax)
 *   label_table_host  [num_labels, 2] int32 host: (task, channel within the task) of each label, task -1 for a
 *               label of no task; task_classes_host [num_tasks] int32 host: classes per task (ncls_t)
 *   pc_x, pc_y, vs_x, vs_y  point_cloud_range[0:2] and voxel_size[0:2] as fp32; fmap_x = grid_size[0] // osf,
 *               fmap_y = grid_size[1] // osf
 * Per object, in fp32 with one rounding per op: width = dx / vs_x / osf, length = dy / vs_y / osf; drawn only if
 * width > 0 and length > 0; r = gaussian_radius((length, width), gaussian_overlap) op for op (gaussian.py:55-84),
 * radius = max(min_radius, int(r)); coor = (x - pc) / vs / osf, (cx, cy) = coor truncated toward zero.  The
 * gaussian exp(-(dx^2 + dy^2) / (2 sigma^2)), sigma = (2 radius + 1) / 6, is evaluated in double, set to 0 below
 * DBL_EPSILON and rounded to fp32, over the window rows cx +- radius, columns cy +- radius of a [fmap_y, fmap_x]
 * plane, clipped to the plane (the reference draws center_int[[1, 0]]), and maxed into the heatmap.
 * mode CENTERHEAD: objects are assigned to their task's slots by class in task order, then by index
 *               (centerpoint.py:463-486); slots >= max_objs are dropped and not drawn; a centre with cx outside
 *               [0, fmap_x) or cy outside [0, fmap_y) is skipped.  Labels of no task are dropped, as the reference's
 *               task masks drop them.  Outputs, task-major: heatmap [T][B, ncls_t, fmap_y, fmap_x],
 *               anno_box [T][B, max_objs, box_dim == 9 ? 10 : 8] fp32 ((coor - c)[2], z + dz / 2, log(dims) if
 *               norm_bbox else dims, sin(yaw), cos(yaw)[, vx, vy]), ind int64 [T][B, max_objs] = cx * fmap_y + cy,
 *               mask uint8 [T][B, max_objs]; every slot is written (zeros for empty slots).
 * mode TRANSFUSION: num_tasks 1, no max_objs cap, no range test (a centre up to radius cells off the map draws its
 *               in-map part); heatmap [B, ncls, fmap_y, fmap_x]; anno_box, ind, mask unused (nullable).
 * status [1] int32 device: objects with width, length > 0 skipped because int(r) is undefined (r not finite or
 * >= 2^30, where the reference raises) or, in TRANSFUSION mode, because the label is of no task (the reference
 * would wrap a negative label or raise).  An object whose centre is not finite is skipped without a count.
 * nmax <= BEVB200_HEAD_TARGETS_MAX_BOXES, else BEVB200_EUNSUPPORTED; num_tasks <= BEVB200_HEAD_TARGETS_MAX_TASKS,
 * num_labels <= BEVB200_HEAD_TARGETS_MAX_LABELS.  Workspace (one draw record per object, 16 * B * nmax bytes):
 * bevb200_head_targets_workspace_bytes(B, nmax), 0 for unsupported sizes; a smaller one gives
 * BEVB200_EWORKSPACE. */
#define BEVB200_HEAD_TARGETS_CENTERHEAD 0
#define BEVB200_HEAD_TARGETS_TRANSFUSION 1
#define BEVB200_HEAD_TARGETS_MAX_BOXES 4096
#define BEVB200_HEAD_TARGETS_MAX_TASKS 32
#define BEVB200_HEAD_TARGETS_MAX_LABELS 256
BEVB200_API size_t bevb200_head_targets_workspace_bytes(int B, int nmax);
BEVB200_API int bevb200_head_targets(const float *boxes, const int32_t *labels, const int32_t *counts, int B,
                                     int nmax, int box_dim, const int32_t *label_table_host, int num_labels,
                                     const int32_t *task_classes_host, int num_tasks, float pc_x, float pc_y,
                                     float vs_x, float vs_y, int out_size_factor, int fmap_x, int fmap_y,
                                     double gaussian_overlap, int min_radius, int mode, int max_objs, int norm_bbox,
                                     float *heatmap, float *anno_box, int64_t *ind, uint8_t *mask, int32_t *status,
                                     void *workspace, size_t workspace_bytes, void *stream);
/* draw_heatmap_gaussian(heatmap, (x, y), radius, k) (gaussian.py:24-52) on one [height, width] fp32 plane, through
 * the draw kernel of bevb200_head_targets with one record: column x, row y.  Every cell of the window clipped to the
 * plane becomes torch.max(cell, k * gaussian) (any k; zeros of the gaussian included; NaN propagates).
 * 0 <= radius < 2^30, else BEVB200_EINVAL. */
BEVB200_API int bevb200_draw_heatmap_gaussian(float *heatmap, int height, int width, int x, int y, int radius,
                                              float k, void *stream);

/* ---- Exact linear sum assignment and the TransFusion training-target assignment (transfusion.py:408-525
 *      get_targets_single, core/bbox/assigners/hungarian_assigner.py, scipy.optimize.linear_sum_assignment) ----
 * The solver is scipy's rectangular_lsap.cpp (shortest augmenting paths, Crouse 2016) restated in double with
 * the same column selection and tie breaks: for the same fp32 matrix it returns scipy's assignment bit for bit,
 * ties included.  A segment is one independent matrix; it is transposed when it has fewer columns than rows, as
 * scipy does.  One CTA per segment; no host synchronisation, no allocation, CUDA-graph capturable.
 * Per-segment status bits (nonzero: the segment has no matches; scipy / the reference would raise):
 *   BEVB200_ASSIGN_INVALID_COST  a cost entry is NaN or -inf
 *   BEVB200_ASSIGN_BAD_LABEL     (transfusion_assign) a gt label outside [0, K); its cost column is NaN
 *   BEVB200_ASSIGN_INFEASIBLE    +inf entries leave no complete assignment
 * Limits: at most BEVB200_ASSIGN_MAX rows and columns per segment, BEVB200_ASSIGN_MAX_SEGMENTS segments and
 * BEVB200_ASSIGN_MAX_CLASSES classes, else BEVB200_EUNSUPPORTED. */
#define BEVB200_ASSIGN_MAX 4096
#define BEVB200_ASSIGN_MAX_SEGMENTS 65535
#define BEVB200_ASSIGN_MAX_CLASSES 256
#define BEVB200_ASSIGN_INVALID_COST 1
#define BEVB200_ASSIGN_BAD_LABEL 2
#define BEVB200_ASSIGN_INFEASIBLE 4

/* linear_sum_assignment of S matrices at once:
 *   cost        [S, R, C] fp32 device; segment s is its top-left row_counts[s] x col_counts[s] block (counts int32
 *               device, clamped to [0, R] / [0, C]; nullable: R / C)
 *   col4row     [S, R] int32 device: the column matched to each row, -1 for none (padding rows included)
 *   row4col     [S, C] int32 device, nullable: the row matched to each column, -1 for none
 *   status      [S] int32 device, nullable: the status bits above
 *   steps       [S] int32 device, nullable: the solver's Dijkstra steps (columns settled) per segment
 * The solver keeps its state in shared memory: the workspace query returns 0, and workspace may be null. */
BEVB200_API size_t bevb200_lsap_workspace_bytes(int S, int R, int C);
BEVB200_API int bevb200_lsap(const float *cost, const int32_t *row_counts, const int32_t *col_counts, int S, int R,
                             int C, int32_t *col4row, int32_t *row4col, int32_t *status, int32_t *steps,
                             void *workspace, size_t workspace_bytes, void *stream);

/* TransFusionHead.get_targets (everything but the heatmap) for B samples and L decoder layers of P proposals
 * (N = L * P) in three launches (cost, solver, targets).  Segment s = b * L + l is layer l of sample b.
 *   heatmap     [B, K, N] fp32 logits; center [B, 2, N] (feature cells), height [B, 1, N] (gravity-centre z),
 *               dim [B, 3, N] (log sizes), rot [B, 2, N] (sin, cos): the head's raw predictions, decoded as
 *               TransFusionBBoxCoder.decode does (cx = center * osf * vs + pc, dims = exp, z = height - dz / 2,
 *               yaw = atan2).  decoded [B, N, box_dim] fp32, nullable: boxes already decoded (center, height,
 *               dim, rot are then unused)
 *   gt_boxes    [B, nmax, box_dim] fp32 (x, y, z_bottom, dx, dy, dz, yaw[, vx, vy]); gt_labels [B, nmax] int32;
 *               gt_counts [B] int32 device (clamped to [0, nmax]; nullable: nmax)
 *   coder_*     TransFusionBBoxCoder pc_range[0:2], voxel_size[0:2] and out_size_factor; code_size 8 or 10 (10
 *               needs box_dim 9); pc_x0, pc_y0, pc_x1, pc_y1: train_cfg.point_cloud_range[0, 1, 3, 4]
 *   cls_weight, alpha, gamma, reg_weight, iou_weight: FocalLossCost, BBoxBEVL1Cost, IoU3DCost; pos_weight:
 *               train_cfg.pos_weight
 * Cost per (proposal, gt), fp32 with one rounding per op in the reference's order: focal class cost of the gt's
 * label (p = sigmoid, (pos - neg) * w) + L1 of the xy normalised by the range, times reg_weight + (-iou3d) *
 * iou_weight, iou3d = rotated BEV overlap (as bevb200_boxes_overlap_bev) * height overlap / clamp(va + vb - ov,
 * 1e-8).  The assignment is scipy's on that matrix.  Outputs, all written:
 *   labels        [B, N] int64: the matched gt's label, K when unmatched
 *   label_weights [B, N] int64: 1; positives (int64)pos_weight when pos_weight > 0
 *   bbox_targets  [B, N, code_size] fp32: TransFusionBBoxCoder.encode of the matched gt ((x - pc) * the fp32
 *                 reciprocal of (float)(osf * vs), z + dz / 2, log dims, sin, cos[, vx, vy]), 0 when unmatched
 *   bbox_weights  [B, N, code_size] fp32: 1 on matched rows; ious [B, N] fp32: clamp(iou3d, 0, 1) on matches
 *   num_pos [B] int32, mean_iou [B] fp32 = sum(ious of the positives) / max(num_pos, 1); status [B] int32: the
 *                 status bits of the sample's segments ORed
 *   gt_inds [B, N] int64, nullable: matched gt + 1, 0 when unmatched; max_overlaps [B, N] fp32, nullable: the
 *                 unclamped iou3d of matches, 0 elsewhere (HungarianAssigner3D's AssignResult)
 *   cost_out      [B * L, P, nmax] fp32, nullable: the cost matrix, proposal-major; entries of absent gts are
 *                 not written
 *   steps         [B * L] int32, nullable: the solver's steps per segment
 * A sample with no gt gets all-negative targets (the reference raises).  Workspace:
 * bevb200_transfusion_assign_workspace_bytes(B, L, P, nmax) (4 * B * L * (P * nmax + P + 1) bytes, aligned), 0
 * for unsupported sizes; a smaller one gives BEVB200_EWORKSPACE. */
BEVB200_API size_t bevb200_transfusion_assign_workspace_bytes(int B, int L, int P, int nmax);
BEVB200_API int bevb200_transfusion_assign(
    const float *heatmap, const float *center, const float *height, const float *dim, const float *rot,
    const float *decoded, int B, int L, int P, int K, const float *gt_boxes, const int32_t *gt_labels,
    const int32_t *gt_counts, int nmax, int box_dim, double coder_pc_x, double coder_pc_y, double coder_vs_x,
    double coder_vs_y, int coder_out_size_factor, int code_size, double pc_x0, double pc_y0, double pc_x1,
    double pc_y1, double cls_weight, double alpha, double gamma, double reg_weight, double iou_weight,
    double pos_weight, int64_t *labels, int64_t *label_weights, float *bbox_targets, float *bbox_weights,
    float *ious, int32_t *num_pos, float *mean_iou, int32_t *status, int64_t *gt_inds, float *max_overlaps,
    float *cost_out, int32_t *steps, void *workspace, size_t workspace_bytes, void *stream);

/* ---- TransFusion query proposals (TransFusionHead.forward_single, transfusion.py:237-281 and :322-325) ----------
 * The query initialisation of the head for B samples in two launches (peak, select), no host synchronisation, no
 * allocation; CUDA-graph capturable and the same bit for bit on every run.
 *   heatmap     [B, C, H, W] device, the dense heatmap logits; dtype BEVB200_PROPOSALS_F32 or _F16
 *   kernel_size k, the nms_kernel_size: odd, 3 <= k <= BEVB200_PROPOSALS_MAX_KERNEL, k <= H and k <= W; p = k / 2
 *   exempt0, exempt1  classes whose peak test is against themselves (nuScenes 8, 9; Waymo 1, 2), -1 for none
 * With s = sigmoid(x) as torch computes it on CUDA (1 / (1 + expf(-x)) in fp32, IEEE division, rounded to fp16 for
 * fp16 input), local_max = the k x k window maximum (NaN propagates, as max_pool2d) on cells at least p from every
 * edge and 0 in the border band, or s itself for an exempt class, the masked plane is m = s * (s == local_max): a
 * border cell is 0, a NaN stays NaN.  Over the C * H * W values of m per sample, flat index c * H * W + h * W + w,
 * the first K = num_proposals in descending value (NaN above everything) with ties by ascending flat index, i.e.
 * argsort(descending=True, stable=True)[:K], give:
 *   labels               [B, K] int64 device: flat / (H * W)  (the reference's query_labels)
 *   index                [B, K] int64 device: flat % (H * W)
 *   query_heatmap_score  [B, C, K] device in the heatmap's dtype: m[b, :, index], every class at each selected cell
 * Every output element is written.  BEVB200_EINVAL: a size < 1, an even k or k = 1, H or W < k, an exempt class
 * outside [-1, C), K < 1 or K > C * H * W, a null pointer.  BEVB200_EUNSUPPORTED: another dtype, or B, C, C * H * W,
 * K or k above the limits below.  Workspace (each tile of 1024 cells gets 1024 8-byte key slots and a count):
 * bevb200_transfusion_proposals_workspace_bytes(B, C, H, W) = align256(8 * B * T * 1024) + align256(4 * B * T),
 * T = ceil(C * H * W / 1024); 0 for unsupported sizes; a smaller one gives BEVB200_EWORKSPACE. */
#define BEVB200_PROPOSALS_F32 0
#define BEVB200_PROPOSALS_F16 1
#define BEVB200_PROPOSALS_MAX_BATCH 65535
#define BEVB200_PROPOSALS_MAX_CLASSES 64
#define BEVB200_PROPOSALS_MAX_CELLS (1 << 24)   /* C * H * W per sample */
#define BEVB200_PROPOSALS_MAX_K 4096
#define BEVB200_PROPOSALS_MAX_KERNEL 15
BEVB200_API size_t bevb200_transfusion_proposals_workspace_bytes(int B, int C, int H, int W);
BEVB200_API int bevb200_transfusion_proposals(const void *heatmap, int dtype, int B, int C, int H, int W,
                                              int num_proposals, int kernel_size, int exempt0, int exempt1,
                                              int64_t *labels, int64_t *index, void *query_heatmap_score,
                                              void *workspace, size_t workspace_bytes, void *stream);

/* ---- CenterHead box decode (CenterHead.get_bboxes, centerpoint.py:669-698, and CenterPointBBoxCoder.decode,
 * core/bbox/coders/centerpoint_bbox_coders.py:62-225) -----------------------------------------------------------
 * The decode of all T tasks x B samples of a frame in two launches (candidates, select + decode), no host
 * synchronisation, no allocation; CUDA-graph capturable and the same bit for bit on every run.  Segment
 * s = t * B + b.  Host arrays of T entries give each task's device maps, fp32 contiguous NCHW:
 *   heatmap[t] [B, cat[t], H, W]   reg[t] [B, 2, H, W]   height[t] [B, 1, H, W]   dim[t] [B, 3, H, W]
 *   rot[t] [B, 2, H, W] (sine, cosine)   vel[t] [B, 2, H, W]
 * reg may be NULL (no task has it: the centre is the cell's middle, + 0.5) and so may vel (box code size 7 instead
 * of 9); otherwise every entry is a map.  heat_is_logit != 0: the score is sigmoid(heatmap) as torch computes it on
 * CUDA (1 / (1 + expf(-x)), IEEE division), else the heatmap itself; dim_is_log != 0: dim is expf(dim) (the head's
 * norm_bbox), else dim itself.
 * Per segment, over the task's cat * H * W scores with flat index c * H * W + row * W + col, the first
 * K = max_num in descending score (NaN above everything) with ties by ascending flat index are taken: the
 * reference's per-class top-k followed by its top-k over cat * K, with stable sorts.  label = flat / (H * W),
 * ind = flat % (H * W).  The reference names the map [B, N, W, H]: its xs = trunc(float(ind) / float(W)) is the ROW
 * (equal to ind / W for ind < 2^24) and its ys = ind % W the column.  Each step is one fp32 rounding, in this order:
 *   x = ((row + reg[0]) * out_size_factor) * voxel_x + pc_x      y = ((col + reg[1]) * out_size_factor) * voxel_y + pc_y
 * (+ 0.5 without reg; the double arguments are rounded to fp32 first), and the box row is
 *   [x, y, height, dim0, dim1, dim2, atan2f(rot[0], rot[1]), vel0, vel1]    all maps read at ind.
 * A selected row survives when (use_score_threshold == 0 or score > score_threshold, strict, in fp32; a NaN score
 * took one of the K places and fails this test) and post_center_range[0..2] <= (x, y, height) <=
 * post_center_range[3..5] (6 host doubles, rounded to fp32; inclusive).  Survivors are compacted to the front of the
 * segment in their descending-score order:
 *   boxes  [T * B, K, code] fp32   scores [T * B, K] fp32   labels [T * B, K] fp32 (the reference's clses.float())
 *   index  [T * B, K] int32, nullable: ind of each row      counts [T * B] int32
 * Rows at and after counts[s] are zero in every output.  A refused call writes nothing.
 * BEVB200_EINVAL: T, B, H, W or a class count < 1, max_num < 1 or > H * W (the reference's per-class topk raises), a
 * null required pointer.  BEVB200_EUNSUPPORTED: T, T * B, a class count, cat * H * W or max_num above the limits
 * below.  Workspace: bevb200_centerhead_decode_workspace_bytes(T, B, cat, H, W) = align256(8 * T * B * Tl * 1024) +
 * align256(4 * T * B * Tl), Tl = ceil(max cat * H * W / 1024); 0 for unsupported sizes; a smaller one gives
 * BEVB200_EWORKSPACE. */
#define BEVB200_DECODE_MAX_TASKS 16
#define BEVB200_DECODE_MAX_SEGMENTS 65535      /* T * B */
#define BEVB200_DECODE_MAX_CLASSES 64          /* per task */
#define BEVB200_DECODE_MAX_CELLS (1 << 24)     /* cat * H * W per task and sample */
#define BEVB200_DECODE_MAX_K 4096
BEVB200_API size_t bevb200_centerhead_decode_workspace_bytes(int T, int B, const int *cat, int H, int W);
BEVB200_API int bevb200_centerhead_decode(
    const float *const *heatmap, const float *const *reg, const float *const *height, const float *const *dim,
    const float *const *rot, const float *const *vel, const int *cat, int T, int B, int H, int W, int max_num,
    int heat_is_logit, int dim_is_log, double out_size_factor, double voxel_x, double voxel_y, double pc_x,
    double pc_y, const double *post_center_range, int use_score_threshold, double score_threshold, float *boxes,
    float *scores, float *labels, int32_t *index, int32_t *counts, void *workspace, size_t workspace_bytes,
    void *stream);

/* ---- TransFusion box decode (TransFusionHead.get_bboxes, models/heads/bbox/transfusion.py:715-851, and
 * TransFusionBBoxCoder.decode, core/bbox/coders/transfusion_bbox_coder.py:39-124) -------------------------------
 * The inference tail of the head for B samples of P proposals: one launch without NMS, four with NMS tasks (decode
 * and segments, the two of bevb200_nms, merge); no host synchronisation, no allocation; CUDA-graph capturable and
 * the same bit for bit on every run.  Device maps, contiguous, all of one dtype BEVB200_TFDECODE_F32 or _F16:
 *   heatmap [B, C, N] logits   center [B, 2, N]   height [B, 1, N]   dim [B, 3, N] log sizes   rot [B, 2, N] (sin,
 *   cos)   vel [B, 2, N] or NULL (box code 7 instead of 9); N >= P, and the last P columns are read (the reference's
 *   [..., -num_proposals:]: N = layers * P when the decoder layers are concatenated)
 *   query_heatmap_score [B, C, P] in the maps' dtype   query_labels [B, P] int64 (transfusion_proposals' labels);
 *   both NULL: the heatmap holds the scores themselves (TransFusionBBoxCoder.decode's input), score_c = heatmap_c
 * Per proposal n, each product rounded once in the maps' dtype (fp16: computed in fp32, rounded to half):
 *   score_c = (sigmoid(heatmap_c) * query_heatmap_score_c) * (c == query_labels[n])   (a label outside [0, C)
 *   matches no class); label and score = max over c: the first NaN if any, else the first maximum.
 *   box = [x, y, z, dx, dy, dz, yaw(, vx, vy)]: x = ((center0 * osf) * voxel_x) + pc_x (y alike), dims = exp(dim),
 *   z = height - dz * 0.5, yaw = atan2(sin, cos); the double arguments are rounded to fp32 first.
 * A row survives when (use_score_threshold == 0 or score > score_threshold, strict; for fp16 the threshold is
 * rounded to half, as torch's scalar comparison does) and, unless post_center_range (6 host doubles) is NULL,
 * (x, y, z) lies within it, limits included, compared in fp32 against the fp32-rounded limits.
 * NMS (nms_mode BEVB200_NMS_CIRCLE or BEVB200_NMS_ROTATE; BEVB200_TFDECODE_NMS_NONE for none): task_of_class[C]
 * (host) maps each class to a task in [0, num_tasks) or -1; task_nms[num_tasks] (host) flags the tasks with NMS.
 * Rows of a class in no task are dropped; rows of a task without NMS are kept; the rows of each NMS task of each
 * sample are sorted by descending score (stable: ties in row order, NaN first) and suppressed by bevb200_nms:
 *   CIRCLE  fp32 squared centre distance <= nms_thresh, at most post_max kept (circle_nms' default is 83);
 *   ROTATE  rotated BEV IoU of xywhr2xyxyr(x, y, dx, dy, yaw) in fp32 > (float)nms_thresh, the first pre_max rows of
 *           the sorted list, at most post_max kept.
 * Kept rows stay in proposal order.  Outputs (rows at and after counts[b] are zero):
 *   boxes [B, P, code] and scores [B, P] in the maps' dtype   labels [B, P] int32   index [B, P] int32: the
 *   proposal of each row   counts [B] int32
 * A refused call writes nothing.  BEVB200_EINVAL: B, C or P < 1, N < P, a null pointer, another nms_mode, with NMS
 * pre_max or post_max < 1, a null table or a task_of_class entry outside [-1, num_tasks).  BEVB200_EUNSUPPORTED:
 * another dtype, B, P, C or num_tasks above the limits below, or (with NMS) NMS tasks x B above
 * BEVB200_NMS_MAX_SEGMENTS.  Workspace: bevb200_transfusion_get_bboxes_workspace_bytes(B, P, code_size, dtype,
 * nms_mode, num_nms_tasks, post_max) = 0 without NMS tasks, else, R = B * P, S = num_nms_tasks * B, e = 4 (fp32)
 * or 2 (fp16), D = 2 (CIRCLE) or 5 (ROTATE), every term rounded up to 256 bytes: e R code + e R + 4 R + 4 R + 4 B +
 * 4 S P D + 8 S P + 4 S + 8 S post_max + 4 S + bevb200_nms_workspace_bytes(S, P); 0 for unsupported sizes; a
 * smaller one gives BEVB200_EWORKSPACE. */
#define BEVB200_TFDECODE_F32 0
#define BEVB200_TFDECODE_F16 1
#define BEVB200_TFDECODE_NMS_NONE (-1)
#define BEVB200_TFDECODE_MAX_BATCH 65535
#define BEVB200_TFDECODE_MAX_PROPOSALS 4096
#define BEVB200_TFDECODE_MAX_CLASSES 64           /* classes, and tasks */
BEVB200_API size_t bevb200_transfusion_get_bboxes_workspace_bytes(int B, int P, int code_size, int dtype,
                                                                  int nms_mode, int num_nms_tasks, int post_max);
BEVB200_API int bevb200_transfusion_get_bboxes(
    const void *heatmap, const void *query_heatmap_score, const int64_t *query_labels, const void *center,
    const void *height, const void *dim, const void *rot, const void *vel, int dtype, int B, int C, int N, int P,
    double out_size_factor, double voxel_x, double voxel_y, double pc_x, double pc_y,
    const double *post_center_range, int use_score_threshold, double score_threshold, int nms_mode,
    const int *task_of_class, const int *task_nms, int num_tasks, double nms_thresh, int pre_max, int post_max,
    void *boxes, void *scores, int32_t *labels, int32_t *index, int32_t *counts, void *workspace,
    size_t workspace_bytes, void *stream);

/* ---- CenterHead and TransFusion training losses ----------------------------------------------------------------
 * CenterHead.loss (models/heads/bbox/centerpoint.py:584-634) and TransFusionHead.loss (transfusion.py:587-713) with
 * mmdet 2.20's GaussianFocalLoss, FocalLoss(use_sigmoid=True) (mmcv 1.4's sigmoid_focal_loss CUDA op) and L1Loss,
 * all reduction "mean".  Forward: two launches; backward: two (CenterHead) or one (TransFusion).  No allocation, no
 * host synchronisation, stream-ordered, CUDA-graph capturable; every output element is written and the sums are
 * taken in double in a fixed order, so results are reproducible bit for bit.
 *   clip_sigmoid(x) = clamp(1 / (1 + expf(-x)), fp32(1e-4), fp32(1 - 1e-4)), its gradient 0 outside those bounds
 *     (bounds included in the passing range).  Inputs are never modified (the reference's sigmoid_ is in place).
 *   gaussian focal (alpha, gamma = focal_host pair): per element, p = clip_sigmoid(x), eps = 1e-12,
 *     -log(p + eps) (1 - p)^alpha [t == 1] - log(1 - p + eps) p^alpha (1 - t)^gamma;  sum / max(count(t == 1), 1)
 *   sigmoid focal (alpha, gamma), logits [R, K], int64 labels [R] with K the background:
 *     -[l == c] alpha (1 - p)^gamma log(max(p, FLT_MIN)) - [l != c] (1 - alpha) p^gamma log(max(1 - p, FLT_MIN)),
 *     times the row's int64 label weight, sum / avg; a label outside [0, K] skips its row and sets
 *     BEVB200_LOSS_BAD_LABEL
 *   L1: sum |pred - target| w / avg; a NaN target gives a NaN loss even at w = 0, its gradient is 0 (sgn(NaN) = 0)
 *   each loss is multiplied by its loss_weight.
 * CenterHead, per task t (maps [B, ch, H, W] fp32; vel only with code 10):
 *   heatmap[t] [B, cat[t], H, W] logits vs heat_target[t];  pred = cat(reg, height, dim, rot[, vel]) gathered at
 *   ind[t] [B, M] int64 (cell row * W + col) against anno_box[t] [B, M, code] with weights
 *   fp32(mask[t] (uint8 [B, M]) * isnotnan(target)) * fp32(code_weights[c]) and avg fp32(sum mask[t] + 1e-4).
 *   An ind outside [0, H * W) skips its slot; on a slot with mask != 0 it sets BEVB200_LOSS_BAD_IND.
 *   losses / avg_factors [2T] fp32: heatmap of task t at 2t, bbox at 2t + 1; status [1] int32.
 *   Backward: grad_losses [2T] (device); gradients of every map (same shapes), each element written once; slots that
 *   share a cell add their contributions in slot order.
 * TransFusion (the cls and box terms of trained layer l use columns l * P .. (l + 1) * P of N):
 *   dense_heatmap [B, K, H, W] logits vs dense_target;  heatmap [B, K, N] logits, labels / label_weights [B, N]
 *   int64;  center [B, 2, N], height [B, 1, N], dim [B, 3, N], rot [B, 2, N], vel [B, 2, N] against
 *   bbox_targets [B, N, code] with weights fp32(bbox_weights * code_weights[c]);  avg max(sum num_pos, 1) with
 *   num_pos int32 [n_num_pos].  losses: [0] heatmap, [1 + 2l] cls, [2 + 2l] bbox of layer l < Lt,
 *   [1 + 2 Lt] matched_ious = mean of mean_iou fp32 [n_iou];  avg_factors [2]: heatmap, layers.  Backward:
 *   grad_losses [1 + 2 Lt]; the cls and box gradients are dense over [B, c, N], 0 in columns of untrained layers.
 * focal_host: 4 doubles (heatmap alpha, gamma, cls alpha, gamma; CenterHead: 2); loss_weights_host (TransFusion):
 * heatmap, cls, bbox.  BEVB200_EINVAL: a size < 1, code not 8 or 10, N not a multiple of P, Lt > N / P, a null
 * pointer.  BEVB200_EUNSUPPORTED: more than BEVB200_LOSS_MAX_TASKS tasks, BEVB200_LOSS_MAX_OBJS slots or
 * BEVB200_LOSS_MAX_LAYERS trained layers.  A smaller workspace than the query gives BEVB200_EWORKSPACE. */
#define BEVB200_LOSS_MAX_TASKS 16
#define BEVB200_LOSS_MAX_OBJS 4096
#define BEVB200_LOSS_MAX_LAYERS 15
#define BEVB200_LOSS_BAD_IND 1
#define BEVB200_LOSS_BAD_LABEL 2
BEVB200_API size_t bevb200_centerhead_loss_workspace_bytes(int T, int B, const int *cat, int H, int W, int M,
                                                           int code);
BEVB200_API int bevb200_centerhead_loss(
    const float *const *heatmap, const float *const *reg, const float *const *height, const float *const *dim,
    const float *const *rot, const float *const *vel, const float *const *heat_target, const float *const *anno_box,
    const int64_t *const *ind, const uint8_t *const *mask, const int *cat, int T, int B, int H, int W, int M, int code,
    const float *code_weights_host, double cls_alpha, double cls_gamma, double cls_weight, double bbox_weight,
    float *losses, float *avg_factors, int32_t *status, void *workspace, size_t workspace_bytes, void *stream);
BEVB200_API int bevb200_centerhead_loss_backward(
    const float *const *heatmap, const float *const *reg, const float *const *height, const float *const *dim,
    const float *const *rot, const float *const *vel, const float *const *heat_target, const float *const *anno_box,
    const int64_t *const *ind, const uint8_t *const *mask, const int *cat, int T, int B, int H, int W, int M, int code,
    const float *code_weights_host, double cls_alpha, double cls_gamma, double cls_weight, double bbox_weight,
    const float *grad_losses, const float *avg_factors, float *const *g_heatmap, float *const *g_reg,
    float *const *g_height, float *const *g_dim, float *const *g_rot, float *const *g_vel, void *stream);
BEVB200_API size_t bevb200_transfusion_loss_workspace_bytes(int B, int K, int H, int W, int N, int P, int Lt,
                                                            int code);
BEVB200_API int bevb200_transfusion_loss(
    const float *dense_heatmap, const float *dense_target, const float *heatmap, const float *center,
    const float *height, const float *dim, const float *rot, const float *vel, const int64_t *labels,
    const int64_t *label_weights, const float *bbox_targets, const float *bbox_weights, const int32_t *num_pos,
    int n_num_pos, const float *mean_iou, int n_iou, int B, int K, int H, int W, int N, int P, int Lt, int code,
    const float *code_weights_host, const double *focal_host, const double *loss_weights_host, float *losses,
    float *avg_factors, int32_t *status, void *workspace, size_t workspace_bytes, void *stream);
BEVB200_API int bevb200_transfusion_loss_backward(
    const float *dense_heatmap, const float *dense_target, const float *heatmap, const float *center,
    const float *height, const float *dim, const float *rot, const float *vel, const int64_t *labels,
    const int64_t *label_weights, const float *bbox_targets, const float *bbox_weights, int B, int K, int H, int W,
    int N, int P, int Lt, int code, const float *code_weights_host, const double *focal_host,
    const double *loss_weights_host, const float *grad_losses, const float *avg_factors, float *g_dense,
    float *g_heatmap, float *g_center, float *g_height, float *g_dim, float *g_rot, float *g_vel, void *stream);

/* ---- BEV map segmentation (BEVSegmentationHead, models/heads/segm/vanilla.py; evaluate_map) ----------------------
 * Grid transform: dst[p][i][j] = sum_{(r, wy) in rows[i]} wy * sum_{(c, wx) in cols[j]} wx * src[p][r][c] for every
 * plane p (sample x channel) of NCHW maps, fp32 accumulation, fp32 (half == 0) or fp16 I/O.  rows / cols are CSR
 * tables (ptr [dst_h + 1] / [dst_w + 1], int32 index, fp32 weight, entries in ascending index order); block b covers
 * destination rows [b * rows_per_block, ...) and reads source rows [block_lo[b], block_lo[b] + block_rows[b]), which
 * must hold every row its taps name, block_rows[b] <= max_block_rows.  BEVGridTransform's forward passes the
 * composite prescale + grid_sample taps (<= 4 per output index; taps outside the input are absent: zeros padding);
 * its backward passes the transposed tables to map grad_output to grad_input.  One launch; every destination element
 * is written once (an empty sum is 0), no atomics: reproducible bit for bit.  The tables are built by
 * bevfusion_b200/map_seg.py.  Shared memory is bevb200_map_grid_smem_bytes(); above 48 KiB gives
 * BEVB200_EUNSUPPORTED.
 * Losses, per class k of logits [B, K, H, W] (fp32, or fp16 with logits_half) against target [B, K, H, W]
 * (target_type BEVB200_MAP_TARGET_*: fp32, uint8 / bool, int64; widened to fp32), evaluated in double:
 *   ce = (1 - t) x + log(1 + exp(-x))          d ce / dx = (1 - t) p - t (1 - p),  p = sigmoid(x)
 *   focal (sigmoid_focal_loss, alpha = -1, gamma = 2): m = t (1 - p) + (1 - t) p,  loss = ce m^2,
 *     d / dx = (d ce / dx) m^2 + 2 ce m (1 - 2t) p (1 - p)
 *   losses[k] = fp32(sum over B * H * W / (B * H * W)).  Forward: two launches (double partials per workspace slot,
 *   fixed-order reduce); backward: one launch, grad_logits (logits' dtype) = grad_losses[k] / (B H W) * d / dx.
 * Counts: for each class k and threshold t, with label = gt != 0 (NaN is a positive label) and pred >= thresholds[t]
 *   in fp32 (a NaN pred is negative), ADDS tp, fp, fn into int64 counts [3, K, T] (tp at [0], fp [1], fn [2]).
 *   pred fp32 or fp16 (pred_half), gt as target_type.  One launch; shared-memory counters and one integer atomic
 *   per counter per CTA: exact and order-independent.  T <= BEVB200_MAP_MAX_THRESHOLDS. */
#define BEVB200_MAP_TARGET_F32 0
#define BEVB200_MAP_TARGET_U8 1
#define BEVB200_MAP_TARGET_I64 2
#define BEVB200_MAP_MAX_THRESHOLDS 16
BEVB200_API size_t bevb200_map_grid_smem_bytes(int src_w, int dst_w, int col_nnz, int max_block_rows);
BEVB200_API int bevb200_map_grid_transform(
    const void *src, void *dst, int half, long long planes, int src_h, int src_w, int dst_h, int dst_w,
    const int32_t *row_ptr, const int32_t *row_idx, const float *row_w, const int32_t *col_ptr, const int32_t *col_idx,
    const float *col_w, int col_nnz, const int32_t *block_lo, const int32_t *block_rows, int rows_per_block,
    int max_block_rows, void *stream);
BEVB200_API size_t bevb200_map_seg_loss_workspace_bytes(int B, int K, int H, int W);
BEVB200_API int bevb200_map_seg_loss(const void *logits, int logits_half, const void *target, int target_type, int B,
                                     int K, int H, int W, int focal, float *losses, void *workspace,
                                     size_t workspace_bytes, void *stream);
BEVB200_API int bevb200_map_seg_loss_backward(const void *logits, int logits_half, const void *target,
                                              int target_type, int B, int K, int H, int W, int focal,
                                              const float *grad_losses, void *grad_logits, void *stream);
BEVB200_API int bevb200_map_seg_counts(const void *pred, int pred_half, const void *gt, int gt_type, int B, int K,
                                       int H, int W, const float *thresholds_host, int T, int64_t *counts,
                                       void *stream);

/* ---- LiDAR depth images for the depth-aware camera lift ------------------------------------
 * BaseDepthTransform.forward's per-sample loop (mmdet3d/models/vtransforms/base.py:279-329):
 * undo the lidar augmentation, project every point into every camera with lidar2image, clamp z to
 * [1e-5, 1e5], perspective divide, apply the image augmentation, keep points on the image and
 * write their distance at (row, col).  Colliding points: the one with the LARGEST index wins (the
 * sequential meaning of the reference's index_put; its CUDA result is arbitrary).
 *   points [N, F] device fp32 (xyz first); lidar_aug_matrix [4,4], lidar2image [ncam,4,4],
 *   img_aug_matrix [ncam,4,4]: device fp32 row-major, one sample.
 *   one_hot == 0: channel 0 = distance ("scalar", :318-319); one_hot != 0: depth_bins channels,
 *   1.0 at bin (long)min(dist, depth_bins-1) (:320-325).  add_features != 0 appends F channels
 *   holding the winner's point row with xyz minus the lidar-aug translation (:327-329; the
 *   reference has shifted them in place at :290 -- the caller's points are NOT modified here).
 *   depth [ncam, channels, H, W] is fully written.  ncam <= 16. */
BEVB200_API size_t bevb200_depth_rasterize_workspace_bytes(int ncam, int height, int width);
BEVB200_API int bevb200_depth_rasterize(const float *points, int num_points, int num_features,
                            const float *lidar_aug_matrix, const float *lidar2image,
                            const float *img_aug_matrix, int ncam, int height, int width, int one_hot,
                            int depth_bins, int add_features, float *depth, void *workspace,
                            size_t workspace_bytes, void *stream);

/* ---- DynamicScatter (mmdet3d/ops/voxel/src/scatter_points_cuda.cu:187-315; pybind
 * `dynamic_point_to_voxel_forward / _backward`, voxelization.cpp:10-11) -----------------------
 * reduce_type: 0 sum, 1 mean, 2 max (scatter_points_cuda.cu:7).
 * Forward: rows of `coors` [N, ndim] (ndim 1..4; a row with a negative entry is dropped) name
 * voxels; output voxels are the unique rows in lexicographic order (= at::unique_dim, :208).
 *   reduced_feats [>=M, C], out_coors [>=M, ndim], coors_map [N] (voxel row or -1),
 *   reduce_count [>=M], reduce_from [>=M, C] (nullable; arg-max point per (voxel, channel) for
 *   the max backward), meta[2] device int32 = {M, number of rows with an entry too large for the
 *   key (>= 2^20 for ndim <= 3, >= 2^15 for ndim 4; such rows are dropped and the caller should
 *   raise)}.  Size the outputs for M = N.  Sums run in ascending point order: reproducible,
 *   unlike the reference's float atomics. */
BEVB200_API size_t bevb200_dynamic_scatter_workspace_bytes(int num_points);
BEVB200_API int bevb200_dynamic_scatter(const float *feats, const int32_t *coors, int num_points,
                            int num_features, int ndim, int reduce_type, float *reduced_feats,
                            int32_t *out_coors, int32_t *coors_map, int32_t *reduce_count,
                            int32_t *reduce_from, int32_t *meta, void *workspace,
                            size_t workspace_bytes, void *stream);
/* Backward (:243-315): grad_feats [N, C] is fully written.  For max, `reduce_from` [M, C] is
 * used as given when reduce_from_valid != 0, else rebuilt by traceback from feats /
 * reduced_feats (smallest point index attaining the maximum, :145-160). */
BEVB200_API int bevb200_dynamic_scatter_backward(const float *grad_reduced_feats, const float *feats,
                                     const float *reduced_feats, const int32_t *coors_map,
                                     const int32_t *reduce_count, int32_t *reduce_from,
                                     int reduce_from_valid, int num_points, int num_reduced,
                                     int num_features, int reduce_type, float *grad_feats,
                                     void *stream);

/* ------------------------------------------------------------------------------------
 * sparse convolution (reference: mmdet3d/ops/spconv/include/spconv/spconv_ops.h,
 * indice.cu.h, geometry.h, reordering.cu.h)
 * ---------------------------------------------------------------------------------- */

/* Rulebook.  Replaces spconv::getIndicePair<3> (spconv_ops.h:27-141; bound as
 * sparse_conv_ext.get_indice_pairs_3d, all.cc:22-27) for transpose == 0.
 *
 * The rulebook is produced in offset-major neighbour-table form
 *     nbr[k * n_out + o] = input row feeding output row o through kernel offset k, or -1
 * (k = (off_x*K_y + off_y)*K_z + off_z as geometry.h:57-73), which is what the
 * implicit-GEMM kernel consumes; bevb200_rulebook_to_pairs() converts it to the
 * reference's indicePairs[K,2,N] / indiceNum[K] layout.
 *
 * Two calls because the number of outputs of a strided conv is data dependent:
 *   1. bevb200_rulebook_prepare: marks the active output sites in a bitmap over the
 *      dense output grid, ranks them with a single-pass scan (bits and popcount prefix
 *      interleaved per 32 sites), and writes n_out (device int32[1]).  SubM:
 *      n_out = n_in and the output sites are the input sites in input order
 *      (spconv_ops.h:76-101).  Strided: output rows are ordered by ascending flat index
 *      ((b*X + x)*Y + y)*Z + z -- the order of the reference's GPU path after
 *      torch::_unique (spconv_ops.h:130-136, indice.cu.h:112-127).
 *   2. bevb200_rulebook_fill: writes out_indices [n_out, 4] (b, x, y, z) and
 *      nbr [K, n_out] using the state left in `workspace` by step 1.  SubM gathers each
 *      output's neighbours from the bitmap.  Strided scatters from the inputs, as the
 *      reference does, so an input row just outside the input grid still feeds the
 *      border outputs it reaches.
 * The encoder plan (bevb200_encoder_forward) builds its rulebooks with the same kernels.
 */
BEVB200_API size_t bevb200_rulebook_workspace_bytes(int n_in, int batch_size, const int32_t *out_shape_host);
BEVB200_API int bevb200_rulebook_prepare(const int32_t *indices, int n_in, int batch_size,
                             const int32_t *spatial_shape_host, const int32_t *out_shape_host,
                             const int32_t *ksize_host, const int32_t *stride_host,
                             const int32_t *padding_host, const int32_t *dilation_host,
                             int subm, int32_t *n_out, void *workspace,
                             size_t workspace_bytes, void *stream);
BEVB200_API int bevb200_rulebook_fill(const int32_t *indices, int n_in, int batch_size,
                          const int32_t *spatial_shape_host, const int32_t *out_shape_host,
                          const int32_t *ksize_host, const int32_t *stride_host,
                          const int32_t *padding_host, const int32_t *dilation_host,
                          int subm, int n_out, int32_t *out_indices, int32_t *nbr,
                          void *workspace, size_t workspace_bytes, void *stream);

/* SubM rulebook of a tensor whose rows ARE the outputs of the strided conv whose
 * bevb200_rulebook_prepare() left its state in `workspace` (same batch size and output grid =
 * this tensor's spatial shape): the site bitmap and its ranks are reused as they are (the rows
 * are already in rank order), so no marking / scan / rank table pass is needed. */
BEVB200_API int bevb200_rulebook_fill_subm_sorted(const int32_t *indices, int n, int batch_size,
                                      const int32_t *spatial_shape_host, const int32_t *ksize_host,
                                      const int32_t *dilation_host, int32_t *nbr, void *workspace,
                                      size_t workspace_bytes, void *stream);

/* nbr[K, n_out] -> indicePairs[K, 2, n_in] (-1 padded) + indiceNum[K]
 * (layout of spconv_ops.h:53-57).  Pairs of one offset are emitted in ascending output
 * row (the reference's GPU order is atomic-arrival order, i.e. unspecified). */
BEVB200_API int bevb200_rulebook_to_pairs(const int32_t *nbr, int kernel_volume, int n_out, int n_in,
                              int32_t *indice_pairs, int32_t *indice_num, void *stream);
/* indicePairs[K, 2, n_pairs_dim] + indiceNum[K] -> nbr[K, n_out].  inverse != 0 swaps the
 * roles of the two pair columns (spconv_ops.h:316,345). */
BEVB200_API int bevb200_pairs_to_nbr(const int32_t *indice_pairs, const int32_t *indice_num,
                         int kernel_volume, int pairs_dim, int n_out, int inverse,
                         int32_t *nbr, void *stream);

/* Sparse convolution forward.  Replaces spconv::indiceConv<float> (spconv_ops.h:260-361;
 * bound as sparse_conv_ext.indice_conv_fp32) -- the per-offset gather -> mm_out ->
 * scatter-add loop -- with ONE output-stationary implicit-GEMM kernel:
 *     out[o, :] = epilogue( sum_k features[nbr[k, o], :] @ weight[k] )
 *   features [n_in, c_in] fp32, weight [K, c_in, c_out] fp32 (conv.py:100 layout
 *   [kx,ky,kz,Cin,Cout] flattened), nbr [K, n_out], out [n_out, c_out] fp32.
 * Optional fused epilogue (all may be NULL / 0), applied in this order:
 *     y = acc * scale[c] + shift[c]      (folded eval-mode BatchNorm1d / bias)
 *     y += residual[o, c]                (SparseBasicBlock identity, sparse_block.py:105)
 *     y = max(y, 0) if relu
 * precision: BEVB200_PREC_FP32  exact fp32 FFMA accumulation (SIMT)
 *            BEVB200_PREC_TF32X3 mma.sync tensor cores, 3xTF32 split (fp32-class accuracy)
 *            BEVB200_PREC_TF32   mma.sync single-pass TF32 (fast mode, ~1e-3 rel)
 *            BEVB200_PREC_BF16X3 bf16 hi/lo split on mma.sync (wgmma for c_out 64 / 128 with >= 16 K blocks of 32):
 *                                half the MMAs and operand bytes of TF32X3, per-product error ~2^-17
 *                                (measured ~1e-5 relative per layer)
 */
#define BEVB200_PREC_FP32 0
#define BEVB200_PREC_TF32X3 1
#define BEVB200_PREC_TF32 2
#define BEVB200_PREC_BF16X3 3 /* bf16 MMAs: a = bf16 hi + bf16 lo, hi*hi + hi*lo + lo*hi (3 MMAs per 16 K) */
#define BEVB200_PREC_FP16 4   /* fp16 operands, fp32 accumulation (1 MMA per 16 K): the encoder plan only
                                 (bevb200_encoder_set_precision); the per-conv calls refuse it */
/* 5 is not a precision: every plan refuses it */
#define BEVB200_PREC_INT8 6   /* u8 activations x s8 weights, exact int32 accumulation: the encoder plan's eval forward
                                 only (bevb200_encoder_set_precision); the per-conv calls refuse it */
BEVB200_API int bevb200_spconv_forward(const float *features, const float *weight, const int32_t *nbr,
                           int n_in, int n_out, int c_in, int c_out, int kernel_volume,
                           const float *scale, const float *shift, const float *residual,
                           int relu, int precision, float *out, void *stream);

/* Tensor-core path with pre-packed weights.  The tensor-core kernel consumes the weights as a
 * pre-swizzled shared-memory image (K blocks of 32 over the concatenated (offset, channel)
 * axis, tf32 hi / lo parts); bevb200_spconv_forward() builds it into a stream-ordered temporary
 * on every call, these entry points let a caller with static weights (eval mode) do it once.
 * bevb200_spconv_packed_weight_bytes() returns 0 when (c_in, c_out, kernel_volume, precision)
 * has no tensor-core form (c_out in {16,32,64,128}, c_in <= 128, kernel_volume <= 27, precision
 * TF32X3, TF32 or BF16X3); such shapes go through bevb200_spconv_forward(), which falls back to
 * the fp32 SIMT kernel on the GPU.
 * Input channels are zero-padded to bevb200_spconv_padded_channels(c_in, precision) = 8, 16, 32,
 * 64 or 128 (SparseEncoder.conv_input: 5 -> 8): the packed image already contains the padding,
 * so the image packed for c_in is also the image for the padded count.  A caller that passes
 * features with fewer channels than that gets them copied into a stream-ordered padded temporary
 * on every call; passing rows that are already padded (and the padded count as c_in) avoids it. */
BEVB200_API int bevb200_spconv_padded_channels(int c_in, int precision);
BEVB200_API size_t bevb200_spconv_packed_weight_bytes(int c_in, int c_out, int kernel_volume, int precision);
BEVB200_API int bevb200_spconv_pack_weights(const float *weight, int c_in, int c_out, int kernel_volume,
                                int precision, float *packed, void *stream);
BEVB200_API int bevb200_spconv_forward_packed(const float *features, const float *packed_weight,
                                  const int32_t *nbr, int n_in, int n_out, int c_in, int c_out,
                                  int kernel_volume, const float *scale, const float *shift,
                                  const float *residual, int relu, int precision, float *out,
                                  void *stream);

/* Generation-6 tensor-core path (BEVB200_PREC_BF16X3), split operand images.
 * The tensor-core kernel consumes a feature row as the bf16 image of its hi/lo split: per group of 16
 * channels 32 B of bf16 hi (= rn(x)) then 32 B of bf16 lo (= rn(x - hi)); c * 4 bytes per row, c a
 * multiple of 16.  A conv writes that image of ITS output from the epilogue (out_split), so a chain of
 * convs (SparseEncoder) splits each row once instead of once per (row, kernel offset) visit, and
 * bevb200_spconv_forward() -- the fp32-in / fp32-out drop-in for indice_conv_fp32 -- is
 * split_rows + forward_split.
 *   bevb200_spconv_split_channels(c)   channel count of the image (c rounded up to 16, <= 128; 0: none)
 *   bevb200_spconv_split_rows          fp32 rows [n, c_in] -> image [n, split_channels(c_in) * 4 B],
 *                                      zero padded; n_dev (nullable, device int32) caps n on the device
 *   bevb200_spconv_pack_split_weights  weight [K, c_in, c_out] fp32 -> the kernel's shared-memory image
 *                                      (bevb200_spconv_split_weight_bytes bytes; c_in is the REAL count)
 *   bevb200_spconv_forward_split       features_split [n_in, c_in * 4 B] (c_in = the padded count),
 *                                      nbr [K][nbr_stride] (rows >= n_out unused), n_out_dev (nullable):
 *                                      device-side row count <= n_out, read by the persistent kernel --
 *                                      no host round trip for the output count of a strided conv;
 *                                      out (fp32 rows) and / or out_split (image) are written, epilogue
 *                                      as bevb200_spconv_forward. */
BEVB200_API int bevb200_spconv_split_channels(int c_in);
BEVB200_API int bevb200_spconv_split_rows(const float *features, int n, const int32_t *n_dev, int c_in,
                              void *split, void *stream);
BEVB200_API size_t bevb200_spconv_split_weight_bytes(int c_in, int c_out, int kernel_volume);
BEVB200_API int bevb200_spconv_pack_split_weights(const float *weight, int c_in, int c_out, int kernel_volume,
                                      void *packed, void *stream);
BEVB200_API int bevb200_spconv_forward_split(const void *features_split, const void *packed_weight,
                                 const int32_t *nbr, long long nbr_stride, int n_in, int n_out,
                                 const int32_t *n_out_dev, int c_in, int c_out, int kernel_volume,
                                 const float *scale, const float *shift, const float *residual, int relu,
                                 float *out, void *out_split, void *stream);

/* Sparse convolution backward.  Replaces spconv::indiceConvBackward<float> (spconv_ops.h:363-456;
 * bound as sparse_conv_ext.indice_conv_backward_fp32):
 *     input_grad[j, :]  = sum_k out_grad[nbr_t[k, j], :] @ weight[k]^T     [n_in, c_in]
 *     weight_grad[k]    = sum_o features[nbr[k, o], :]^T (x) out_grad[o, :] [K, c_in, c_out]
 * nbr_t [K, n_in] is the transposed neighbour table from bevb200_rulebook_transpose()
 * (nbr_t[k, j] = the output row that input row j feeds through offset k, or -1).
 * Precondition: each input row feeds at most one output per offset (nbr[k, :] holds no valid row twice), as in
 * every rulebook of a sparse conv; the transpose keeps one writer per (k, j) and is undefined otherwise.
 * Entries of nbr outside [0, n_in) are missing neighbours.  input_grad and weight_grad are overwritten, not
 * accumulated into; an input row that feeds no output gets 0 and an offset without pairs gets dW[k] = 0.
 * The input gradient runs the forward implicit-GEMM kernel on (out_grad, W^T, nbr_t) in the
 * requested precision.  The weight gradient sums chunks of rows into per-chunk partials and adds those in
 * ascending chunk order: no atomics, bit-reproducible run to run.  It runs on the tensor cores
 * (spconv_wgrad_tc.cu: mma.sync on ldmatrix.trans fragments of the bf16 hi/lo images of the gathered feature rows
 * and the out-grad rows) when precision is BEVB200_PREC_BF16X3 or BEVB200_PREC_TF32, 1 <= c_in <= 128,
 * c_out in {16, 32, 64, 128}, kernel_volume <= 27 and features and out_grad are 16-byte aligned; everything else,
 * and BEVB200_WGRAD_TC=0, takes the exact-fp32 SIMT kernels.  So BEVB200_PREC_TF32 computes dW at BF16x3-class
 * accuracy (~1e-5 relative); only its input gradient is single-pass TF32.
 * workspace: bevb200_spconv_backward_workspace_bytes() (the transposed weights, the operand images, the partials);
 * a smaller workspace returns BEVB200_EWORKSPACE. */
BEVB200_API int bevb200_rulebook_transpose(const int32_t *nbr, int kernel_volume, int n_out, int n_in,
                               int32_t *nbr_t, void *stream);
BEVB200_API size_t bevb200_spconv_backward_workspace_bytes(int n_in, int n_out, int c_in, int c_out, int kernel_volume);
BEVB200_API int bevb200_spconv_backward(const float *features, const float *weight, const float *out_grad,
                            const int32_t *nbr, const int32_t *nbr_t, int n_in, int n_out, int c_in,
                            int c_out, int kernel_volume, int precision, float *input_grad,
                            float *weight_grad, void *workspace, size_t workspace_bytes,
                            void *stream);

/* SparseConvTensor.dense() (structure.py:49-59) fused with SparseEncoder's
 * permute(0,1,4,2,3).view(N, C*D, H, W) (sparse_encoder.py:126-130):
 *   out[b, c*Z + z, x, y] = features[i, c] for indices[i] = (b, x, y, z); zero elsewhere.
 * With z_major == 0 the plain channels-first dense layout out[b, c, x, y, z] is written.
 * out must hold B*C*X*Y*Z floats; it is fully written (zero filled) by the call.
 * out_batch_stride (floats; 0 = C*X*Y*Z) lets `out` be a channel slice of a wider
 * [B, C_total, X, Y] buffer: the LiDAR half of the fuser input (fusers/conv.py:16) in place. */
BEVB200_API int bevb200_sparse_to_dense(const float *features, const int32_t *indices, int n, int c,
                            int batch_size, const int32_t *spatial_shape_host, int z_major,
                            long long out_batch_stride, float *out, void *stream);

/* ------------------------------------------------------------------------------------
 * SparseEncoder as one native, sync-free call (reference: the python loop of
 * mmdet3d/models/backbones/sparse_encoder.py:99-132 over spconv/conv.py:114-223, with the
 * BatchNorm1d / ReLU / residual modules of spconv/modules.py:127-139 and ops/sparse_block.py:94-110).
 *
 * A plan is a chain of convs (conv i reads the output of conv i-1): SubMConv3d or strided
 * SparseConv3d, each followed by y = acc * scale + shift (folded eval-mode BN / bias), an optional
 * residual add of the OUTPUT of one of the two previous convs (SparseBasicBlock identity) and an
 * optional ReLU.
 * No row count ever returns to the host: buffers are sized by caps (level 0 = max_voxels; a strided
 * conv makes at most prod(ceil(k/s)) outputs per input row and one per output site; level_caps_host,
 * nullable, may tighten the caps of the levels >= 1), kernels read their counts from device memory,
 * so bevb200_encoder_forward() is a fixed sequence of ~45 launches that may be captured in a CUDA graph.
 * BEVB200_PREC_BF16X3 arithmetic (spconv generation 6).  Channel counts: 16 / 32 / 64 / 128 (the first
 * conv's c_in: anything <= 128).
 *   create            host-only object; destroy() frees it (and the CUDA events it may own)
 *   param_bytes       device bytes of the parameter buffer (packed weights, scales, shifts)
 *   set_conv          packs weight [K, c_in, c_out] fp32 and copies scale / shift [c_out] (nullable)
 *                     into the parameter buffer (device pointers, stream ordered)
 *   workspace_bytes   device scratch for (max_voxels, batch_size, caps)
 *   forward           voxel_features [max_voxels, in_channels] fp32, coors [max_voxels, 4] int32
 *                     (b, x, y, z), n_voxels_dev (nullable device int32: valid rows <= max_voxels);
 *                     dense_out [B, C*Z, X, Y] (out_batch_stride floats, 0 = dense) is fully written;
 *                     status_dev int32[1 + levels]: [0] != 0 when a cap truncated a level,
 *                     [1 + l] = rows of level l.  rulebook_stream (nullable): a second stream the
 *                     rulebooks are built on, forked from / joined to `stream` with events. */
typedef struct {
  int32_t c_in, c_out;
  int32_t ksize[3], stride[3], padding[3], dilation[3];
  int32_t subm;          /* 1: SubMConv3d (stride 1, padding k/2 forced, spconv_ops.h:74-83) */
  int32_t relu;
  int32_t residual_from; /* -1, or j = i - 1 or i - 2 (on the same level): add the output of conv j
                            before the ReLU.  Earlier convs are refused: each level keeps two
                            split images, and conv j + 2 overwrites conv j's. */
} bevb200_encoder_conv_t;
typedef struct bevb200_encoder bevb200_encoder_t;
BEVB200_API int bevb200_encoder_create(int in_channels, const int32_t *sparse_shape_host,
                           const bevb200_encoder_conv_t *convs, int n_convs, bevb200_encoder_t **out);
BEVB200_API void bevb200_encoder_destroy(bevb200_encoder_t *enc);
/* FP16 plans.  bevb200_encoder_set_precision(enc, BEVB200_PREC_FP16) makes a plan fp16 (BEVB200_PREC_BF16X3, the
 * default, makes it BF16x3 again); call it before the size queries and set_conv, which then report and pack the fp16
 * layout.  An fp16 plan runs only the _f16 calls below, a BF16x3 plan only the others: the wrong one returns
 * BEVB200_EINVAL before it writes anything.  In the _f16 calls the row data is half (voxel_features, dense_out,
 * grad_dense, grad_voxel_features); weights, BN parameters and weight / BN gradients stay fp32.
 * Numerical contract (fp32 accumulation throughout; every conversion to fp16 rounds to nearest, overflows to +-inf
 * and keeps NaN, so a loss scaler sees an overflow):
 *   inputs     voxel features are rounded once to fp16 (half features pass exactly); the weights are rounded to fp16
 *              when packed (set_conv; forward_train_f16 packs the live weights on every call)
 *   eval       y16 = fp16(relu(acc * scale + shift [+ y16 of residual_from])), one rounding per conv
 *   training   z16 = fp16(acc) is saved; the batch mean / variance are those of z16 (double partials over fixed
 *              2048-row chunks, bit-reproducible); running statistics fp32, updated as in forward_train (and
 *              BEVB200_ENCODER_FEW_ROWS likewise); y16 = fp16(relu(gamma (z16 - mean) invstd + beta [+ y16 res]))
 *   output     dense_out [B, C*Z, X, Y] half holds the last conv's y16 exactly
 *   backward   grad_dense half; the BN backward runs in fp32 on z16; dz is rounded once to an fp16 image that is the
 *              MMA operand of the input gradient (forward kernel on W^T) and of the filter gradient; dW in fp32
 *              with the ordered chunk reduce; grad_voxel_features rounded once to fp16; BN gradients fp32
 * train_saved on an fp16 plan gives the offsets of z16 ([cap, c_out] half) and of the fp16 image y16 ([cap, c_out]
 * half).  bevb200_encoder_precision returns the plan's precision. */
/* INT8 plans (eval only).  bevb200_encoder_set_precision(enc, BEVB200_PREC_INT8) makes a plan INT8; it returns
 * BEVB200_EINVAL, and leaves the plan as it was, when a conv of the chain has no ReLU (every stored activation must be
 * >= 0).  Call it before the size queries, which then report the INT8 layout exactly.  An INT8 plan packs conv i
 * with bevb200_encoder_set_conv_int8 (bevb200_encoder_set_conv refuses it) and runs bevb200_encoder_forward_f16
 * (half voxel_features in, half dense_out out); every training call, and the training size queries (which return 0),
 * refuse it before they read any other argument.
 * Numerical contract.  fl(.) is one fp32 round-to-nearest op, with no FMA contraction.
 *   weights    per output channel c, on the raw conv weight (before any BN fold), when set_conv_int8 packs it:
 *              s_w[c] = fl(max |W[.., .., c]| / 127) (1 when that max is 0), q_w = clamp(rint(fl(W / s_w[c])), -127,
 *              127), rint rounding half to even
 *   scales     conv i has one per-tensor output scale s_i > 0 (calibrated by the caller); r_i = fl(1 / s_i).  Conv i
 *              reads with s_in = s_{i-1}, its residual with s_res = s_{residual_from}
 *   conv 0     the fp16 plan's first conv: features rounded once to fp16, fp16 weights, fp32 accumulation acc;
 *              a[c] = bn_scale[c]
 *   convs 1..  u8 rows x q_w, exact int32 accumulation acc; a[c] = fl(fl(s_in * s_w[c]) * bn_scale[c])
 *   epilogue   v = fl(fl(float(acc) * a[c]) + shift[c]) (bn_scale 1 and shift 0 when absent);
 *              with a residual v = fl(v + fl(float(res_u8) * s_res)); then v = max(v, 0)
 *   output     q = clamp(rint(fl(v * r_i)), 0, 255) as u8 (+inf saturates to 255, NaN becomes 0); the last conv
 *              writes half(v) instead, which dense_out holds exactly
 * set_conv_int8 takes weight [K, c_in, c_out], scale / shift [c_out] (nullable) as set_conv does, and the host
 * scales s_in (ignored for conv 0), s_out and s_res (ignored without a residual); a scale that is not finite and > 0
 * returns BEVB200_EINVAL. */
BEVB200_API int bevb200_encoder_set_precision(bevb200_encoder_t *enc, int precision);
BEVB200_API int bevb200_encoder_precision(const bevb200_encoder_t *enc);
BEVB200_API size_t bevb200_encoder_param_bytes(const bevb200_encoder_t *enc);
BEVB200_API int bevb200_encoder_num_levels(const bevb200_encoder_t *enc);
BEVB200_API int bevb200_encoder_output_shape(const bevb200_encoder_t *enc, int32_t *shape_out, int32_t *channels_out);
BEVB200_API int bevb200_encoder_set_conv(bevb200_encoder_t *enc, int conv, const float *weight, const float *scale,
                             const float *shift, void *params, size_t params_bytes, void *stream);
BEVB200_API int bevb200_encoder_set_conv_int8(bevb200_encoder_t *enc, int conv, const float *weight, const float *scale,
                                  const float *shift, float s_in, float s_out, float s_res, void *params,
                                  size_t params_bytes, void *stream);
BEVB200_API int bevb200_encoder_level_caps(const bevb200_encoder_t *enc, int max_voxels, int batch_size,
                               const int32_t *level_caps_host, int32_t *caps_out);
BEVB200_API size_t bevb200_encoder_workspace_bytes(const bevb200_encoder_t *enc, int max_voxels, int batch_size,
                                       const int32_t *level_caps_host);
BEVB200_API int bevb200_encoder_forward(bevb200_encoder_t *enc, const void *params, const float *voxel_features,
                            const int32_t *coors, int max_voxels, const int32_t *n_voxels_dev,
                            int batch_size, const int32_t *level_caps_host, float *dense_out,
                            long long out_batch_stride, int32_t *status_dev, void *workspace,
                            size_t workspace_bytes, void *stream, void *rulebook_stream);
BEVB200_API int bevb200_encoder_forward_f16(bevb200_encoder_t *enc, const void *params, const void *voxel_features,
                                const int32_t *coors, int max_voxels, const int32_t *n_voxels_dev,
                                int batch_size, const int32_t *level_caps_host, void *dense_out,
                                long long out_batch_stride, int32_t *status_dev, void *workspace,
                                size_t workspace_bytes, void *stream, void *rulebook_stream);

/* status_dev[0] bits of the encoder calls */
#define BEVB200_ENCODER_TRUNCATED 1  /* a level cap truncated a level's rows */
#define BEVB200_ENCODER_FEW_ROWS 2   /* training: a level had fewer than 2 valid rows (torch's BatchNorm1d raises);
                                        its BN used what rows it had, and the running statistics were left alone */

/* Training mode of the same plan: torch's BatchNorm1d in train mode in place of the folded BN, with a
 * whole-encoder backward on the forward's rulebooks.  Both calls are sync-free and may be captured in a CUDA graph.
 *   train_state_bytes  device bytes that live from forward_train to backward (rulebooks, the packed weights, and per
 *                      conv its fp32 pre-BN rows, its output's split image and its batch statistics), sized by the
 *                      caps of (max_voxels, batch_size, level_caps_host)
 *   forward_train      weights[i]: conv i's live fp32 weight [K, c_in, c_out] (packed on every call); bn[i]: its
 *                      BatchNorm1d.  Per conv: the conv without epilogue into fp32 rows z; per-channel batch mean and
 *                      biased variance over the level's valid rows (double partials over fixed 2048-row chunks, added
 *                      in a fixed order: bit-reproducible); running_mean / running_var updated in place with
 *                      `momentum` (unbiased variance) and *num_batches_tracked += 1 (nullable) when the level has
 *                      >= 2 rows, else BEVB200_ENCODER_FEW_ROWS is set; then y = relu(gamma (z - mean) invstd + beta
 *                      [+ y of residual_from]).  The other arguments are those of bevb200_encoder_forward.
 *   train_saved        byte offsets inside the state of conv i's pre-BN rows z ([cap, c_out] fp32) and of its
 *                      output's split image ([cap, c_out * 4 B]: per 16 channels 16 bf16 hi, then 16 bf16 lo;
 *                      y = hi + lo); only the level's first status_dev[1 + l] rows are defined
 *   backward           grad_dense [B, C*Z, X, Y] (out_batch_stride floats, 0 = dense) -> grad_voxel_features
 *                      [max_voxels, in_channels] (nullable: skipped; rows past the valid count are 0),
 *                      grad_weights[i] [K, c_in, c_out], grad_bn_weight[i] / grad_bn_bias[i] [c_out].  Every output
 *                      is overwritten, never accumulated.  weights are the ones forward_train read; state is only
 *                      read, so one state may be differentiated more than once. */
typedef struct {
  const float *weight, *bias;         /* gamma, beta [c_out] */
  float *running_mean, *running_var;  /* [c_out], updated in place */
  int64_t *num_batches_tracked;       /* [1], nullable */
  float eps, momentum;
} bevb200_encoder_bn_t;
BEVB200_API size_t bevb200_encoder_train_state_bytes(const bevb200_encoder_t *enc, int max_voxels, int batch_size,
                                         const int32_t *level_caps_host);
BEVB200_API int bevb200_encoder_train_saved(const bevb200_encoder_t *enc, int max_voxels, int batch_size,
                                const int32_t *level_caps_host, int conv, size_t *pre_bn_offset,
                                size_t *out_image_offset);
BEVB200_API int bevb200_encoder_forward_train(bevb200_encoder_t *enc, const float *const *weights,
                                  const bevb200_encoder_bn_t *bn, const float *voxel_features,
                                  const int32_t *coors, int max_voxels, const int32_t *n_voxels_dev,
                                  int batch_size, const int32_t *level_caps_host, float *dense_out,
                                  long long out_batch_stride, int32_t *status_dev, void *state,
                                  size_t state_bytes, void *stream, void *rulebook_stream);
BEVB200_API int bevb200_encoder_forward_train_f16(bevb200_encoder_t *enc, const float *const *weights,
                                      const bevb200_encoder_bn_t *bn, const void *voxel_features,
                                      const int32_t *coors, int max_voxels, const int32_t *n_voxels_dev,
                                      int batch_size, const int32_t *level_caps_host, void *dense_out,
                                      long long out_batch_stride, int32_t *status_dev, void *state,
                                      size_t state_bytes, void *stream, void *rulebook_stream);
BEVB200_API size_t bevb200_encoder_backward_workspace_bytes(const bevb200_encoder_t *enc, int max_voxels,
                                                int batch_size, const int32_t *level_caps_host);
BEVB200_API int bevb200_encoder_backward(const bevb200_encoder_t *enc, const float *const *weights,
                             const void *state, size_t state_bytes, int max_voxels, int batch_size,
                             const int32_t *level_caps_host, const float *grad_dense,
                             long long out_batch_stride, float *grad_voxel_features,
                             float *const *grad_weights, float *const *grad_bn_weight,
                             float *const *grad_bn_bias, void *workspace, size_t workspace_bytes,
                             void *stream);
BEVB200_API int bevb200_encoder_backward_f16(const bevb200_encoder_t *enc, const float *const *weights,
                                 const void *state, size_t state_bytes, int max_voxels, int batch_size,
                                 const int32_t *level_caps_host, const void *grad_dense,
                                 long long out_batch_stride, void *grad_voxel_features,
                                 float *const *grad_weights, float *const *grad_bn_weight,
                                 float *const *grad_bn_bias, void *workspace, size_t workspace_bytes,
                                 void *stream);

/* ---- PointPillars pillar feature net, training mode (pillar_encoder.py:43-176, BatchNorm1d in train mode) ----
 * The net of bevb200_pillar_features (F 3..8, P 1..32, feat_channels [64, 64], no distance feature; anything else
 * gives BEVB200_EUNSUPPORTED) with batch statistics over all M * P slots, padded slots included (n = P * valid
 * pillars, biased variance for the normalisation), and the backward of both linears and both BNs.
 * Row source: voxels [rows, P, F] fp32, num_points [rows] int32, coords4 [rows, 4] int32 (b, x, y, z).  The rows
 * form `segments` segments of cap = rows / segments rows; rows [s cap, s cap + min(n_dev[s], cap)) are valid
 * (n_dev: DEVICE int32 [segments], nullable: every row), everything else is never read.
 *   forward_train   w1 [32, F+5], w2 [64, 64] fp32 (nn.Linear layout, read on every call); bn: HOST array of the two
 *                   layers' BatchNorm1d (bevb200_encoder_bn_t).  running_mean / running_var are updated in place with
 *                   `momentum` (unbiased variance) and *num_batches_tracked += 1 (nullable).  The pillar maxes land in
 *                   the caller-zeroed canvas [batch, 64, nx, ny] at (b, x, y).  status_dev[0] is set to 0 or
 *                   BEVB200_PILLAR_FEW_ROWS (n < 2): then the running statistics and the canvas are left alone and
 *                   the backward writes zero gradients.
 *   backward_train  grad_canvas [batch, 64, nx, ny] -> grad_w1 [32, F+5], grad_w2 [64, 64], grad_gamma / grad_beta
 *                   of each layer; every output is overwritten.  The row source must be the forward's; state is only
 *                   read, so one state may be differentiated more than once.
 * Sums are double over fixed 128-row chunks added in a fixed order: bit-reproducible, no float atomics, independent of
 * the grid.  No per-slot buffer, no host synchronisation, no allocation.  state (forward -> backward) and workspace
 * (both calls) come from the queries (0 for an unsupported P); a smaller one gives BEVB200_EWORKSPACE before any
 * write. */
#define BEVB200_PILLAR_FEW_ROWS 2
BEVB200_API size_t bevb200_pillar_train_state_bytes(int rows, int max_points);
BEVB200_API size_t bevb200_pillar_train_workspace_bytes(int rows, int max_points);
BEVB200_API int bevb200_pillar_forward_train(const float *voxels, const int32_t *num_points, const int32_t *coords4,
                                             int rows, int segments, const int32_t *n_dev, int max_points,
                                             int num_features, float vx, float vy, float x_off, float y_off,
                                             const float *w1, const float *w2, const bevb200_encoder_bn_t *bn,
                                             float *canvas, int batch, int nx, int ny, int32_t *status_dev,
                                             void *state, size_t state_bytes, void *workspace,
                                             size_t workspace_bytes, void *stream);
BEVB200_API int bevb200_pillar_backward_train(const float *voxels, const int32_t *num_points, const int32_t *coords4,
                                              int rows, int segments, const int32_t *n_dev, int max_points,
                                              int num_features, float vx, float vy, float x_off, float y_off,
                                              const float *grad_canvas, int batch, int nx, int ny, const void *state,
                                              size_t state_bytes, float *grad_w1, float *grad_w2,
                                              float *grad_gamma1, float *grad_beta1, float *grad_gamma2,
                                              float *grad_beta2, void *workspace, size_t workspace_bytes,
                                              void *stream);

/* ---- ImageAug3D + ImageNormalize of the camera pipeline (transforms_3d.py:98-192, 992-1006) ----------------------
 * For each of `cams` uint8 RGB images [in_h, in_w, 3] (images [cams, in_h, in_w, 3], HWC as Pillow holds them) and
 * its draw (draws: DEVICE double [cams, BEVB200_IMAGE_AUG_DRAW_FIELDS] = resize, resize_w, resize_h, crop_x, crop_y,
 * flip (0 / 1), rotate in degrees), out [cams, 3, out_h, out_w] fp32 equals bit for bit
 *     TF.normalize(TF.to_tensor(img.resize((resize_w, resize_h)).crop((crop_x, crop_y, crop_x + out_w,
 *                  crop_y + out_h))[.transpose(FLIP_LEFT_RIGHT)].rotate(rotate)), mean, std)
 * with Pillow's default BICUBIC resample, its crop fill 0, Image.rotate's NEAREST / fill 0 / no-expand rule, and
 * u8 / 255 then (x - mean) / std in fp32.  aug_matrix [cams, 4, 4] fp32 is ImageAug3D's img_aug_matrix from the same
 * draw (resize is the float scale the matrix uses; resize_w / resize_h are the resized image's sides).
 * Only the crop window's columns and rows (with the vertical filter's support) are resampled.  Three launches, no host
 * synchronisation, no allocation: CUDA-graph capturable.  status [1] int32 (device) is zeroed, then gets
 *   BEVB200_IMAGE_AUG_BAD_DRAW        a field is not finite, a size / crop / flip is not an integer in range
 *                                     (1 <= resize_* < 2^19, |crop| <= 2^30, flip 0 or 1)
 *   BEVB200_IMAGE_AUG_OVER_CAPACITY   the draw's filter is wider than the workspace was sized for (resize_w below
 *                                     min_resize_w or resize_h below min_resize_h)
 * and that camera's outputs and matrix are NaN.  Sizes: 1 <= out_h, out_w <= 16384, 1 <= in_h, in_w < 2^19,
 * cams <= 65535.  Workspace: bevb200_image_aug_workspace_bytes(cams, in_h, in_w, out_h, out_w, min_resize_w,
 * min_resize_h) (0 for unsupported sizes): per camera its parameters, coefficient tables for the crop window and
 * in_h x out_w RGBx staging rows, in disjoint regions; a smaller one gives BEVB200_EWORKSPACE before any launch. */
#define BEVB200_IMAGE_AUG_DRAW_FIELDS 7
#define BEVB200_IMAGE_AUG_BAD_DRAW 1
#define BEVB200_IMAGE_AUG_OVER_CAPACITY 2
BEVB200_API size_t bevb200_image_aug_workspace_bytes(int cams, int in_h, int in_w, int out_h, int out_w,
                                                     int min_resize_w, int min_resize_h);
BEVB200_API int bevb200_image_aug(const uint8_t *images, int cams, int in_h, int in_w, const double *draws, int out_h,
                                  int out_w, int min_resize_w, int min_resize_h, float mean0, float mean1,
                                  float mean2, float std0, float std1, float std2, float *out, float *aug_matrix,
                                  int32_t *status, void *workspace, size_t workspace_bytes, void *stream);

/* ---- LoadPointsFromMultiSweeps + PointsRangeFilter of the LiDAR pipeline (loading.py:87-235,
 *      transforms_3d.py:585-614, base_points.py:208-232) ------------------------------------------------------------
 * store [slots, slot_cap, load_dim] fp32 holds raw point rows (DEVICE), slot_rows [slots] int32 (DEVICE) the rows of
 * each slot.  For each of `batch` samples, entries [batch, max_entries] (DEVICE) lists its entries in the reference's
 * concatenation order: the key, then the chosen sweeps in the order of `choices`, or pad copies of the key; unused
 * entries are BEVB200_SWEEP_NONE.  params (DEVICE) holds the column maps, remove_close and the range.  Per row:
 *   KEY    out[c] = raw[key_cols[c]], out[4] = +0
 *   SWEEP  dropped iff remove_close and |raw[0]| < radius and |raw[1]| < radius; out[c] = raw[sweep_cols[c]]; then
 *          out[j] = fl32(fl32(fma(p2, R[j][2], fma(p1, R[j][1], fma(p0, R[j][0], +0.0)))) + t[j]) in float64 for
 *          j < 3 (p = out[0..2]) and out[4] = fl32(lag)
 *   PAD    a KEY row, dropped iff remove_close and |out[0]| < radius and |out[1]| < radius
 * and with has_range a row is kept iff range[0] < x < range[3], range[1] < y < range[4], range[2] < z < range[5] in
 * fp32 (NaN is dropped).  out [batch, cap, out_dim] receives each sample's kept rows in order, counts [batch] int32
 * (DEVICE) min(kept, cap); rows past counts[b] are left untouched and nothing is written past cap.  status [1] int32
 * (DEVICE) is zeroed, then gets
 *   BEVB200_SWEEPS_OVERFLOW    a sample kept more than cap rows (its first cap rows are written)
 *   BEVB200_SWEEPS_BAD_ENTRY   an entry has an unknown kind or a slot outside [0, slots) (it contributes no rows)
 *   BEVB200_SWEEPS_BAD_PARAMS  a column map names a column outside [0, load_dim) (no sample gets rows)
 * Three launches sized by (batch, max_entries, slot_cap), no atomics on the output order, no host synchronisation:
 * CUDA-graph capturable with the store, params and entries refreshed between replays.  Sizes: 3 <= load_dim <= 64,
 * 5 <= out_dim <= 8, cap >= 1, batch <= 65535, max_entries <= 65535, max_entries * slot_cap < 2^31.  Workspace:
 * bevb200_lidar_sweeps_workspace_bytes(batch, max_entries, slot_cap) (0 for unsupported sizes): one int32 per
 * 1024-row tile; a smaller one gives BEVB200_EWORKSPACE before any write. */
#define BEVB200_SWEEP_NONE 0
#define BEVB200_SWEEP_KEY 1
#define BEVB200_SWEEP_SWEEP 2
#define BEVB200_SWEEP_PAD 3
#define BEVB200_SWEEP_MAX_DIM 8
#define BEVB200_SWEEPS_OVERFLOW 1
#define BEVB200_SWEEPS_BAD_ENTRY 2
#define BEVB200_SWEEPS_BAD_PARAMS 4
#define BEVB200_SWEEP_ENTRY_BYTES 112
#define BEVB200_SWEEP_PARAMS_BYTES 100
typedef struct {
  int32_t kind;              /* BEVB200_SWEEP_* */
  int32_t slot;
  double rotation[9];        /* sensor2lidar_rotation, row-major (SWEEP) */
  double translation[3];     /* sensor2lidar_translation (SWEEP) */
  double lag;                /* timestamp / 1e6 - sweep timestamp / 1e6 (SWEEP) */
} bevb200_sweep_entry_t;
typedef struct {
  int32_t key_cols[BEVB200_SWEEP_MAX_DIM];     /* LoadPointsFromFile's use_dim composed with the sweep loader's */
  int32_t sweep_cols[BEVB200_SWEEP_MAX_DIM];   /* the sweep loader's use_dim */
  int32_t remove_close;
  int32_t has_range;
  float radius;                                /* fl32(radius) */
  float range[6];                              /* fl32(point_cloud_range) */
} bevb200_sweep_params_t;
BEVB200_API size_t bevb200_lidar_sweeps_workspace_bytes(int batch, int max_entries, int slot_cap);
BEVB200_API int bevb200_lidar_sweeps_assemble(const float *store, int slots, int slot_cap, int load_dim,
                                              const int32_t *slot_rows, const bevb200_sweep_params_t *params,
                                              const bevb200_sweep_entry_t *entries, int batch, int max_entries,
                                              int out_dim, int cap, float *out, int32_t *counts, int32_t *status,
                                              void *workspace, size_t workspace_bytes, void *stream);

/* ---- LoadRadarPointsMultiSweeps + the radar face of PointsRangeFilter (loading.py:717-790,
 *      transforms_3d.py:607-612, radar_points.py:92-107) -----------------------------------------------------------
 * store [slots, slot_cap, 18] fp32 holds raw radar rows (DEVICE), slot_rows [slots] int32 (DEVICE) the rows of each
 * slot.  For each of `batch` samples, entries [batch, max_entries] (DEVICE) lists its sweeps in the reference's
 * concatenation order (radars in the order of results['radar'], within each its first min(len, sweeps_num) sweeps);
 * kind is BEVB200_SWEEP_SWEEP, or BEVB200_SWEEP_NONE for unused entries.  Per raw row r, with R, t and td the entry's
 * rotation, translation and time_diff and chain_j(p) = fma(p2, R[j][2], fma(p1, R[j][1], fma(p0, R[j][0], +0.0)))
 * in float64, the reference's 58-column float64 row is
 *   0-2    x_j = fl32(fl32(chain_j(r0, r1, r2)) + t[j]); with compensate_velocity x_j = fl32(x_j + vc_j * td), j < 2
 *   3-5, 10-17  the raw values          6-7  velo_j = chain_j(r6, r7, +0)      8-9  vc_j = chain_j(r8, r9, +0)
 *   18     td                            19-26, 27-31, 32-49  one-hot of rint(r3) (8), rint(r11) (5), rint(r14) (18)
 *   50-56  rint(r15) > i, i = 0..6       57   r14 == 0 && r3 < 7 && r11 == 3
 * (rint rounds half to even; one-hot indices in [-w, -1] wrap as numpy's do).  params (DEVICE) gives, per output
 * column c < out_dim, an op code naming one of these values (kind | arg << 8 | block << 16, plus
 * BEVB200_RADAR_OP_NORMALIZE for (v - norm_min[c]) / norm_span[c] in float64), then fl32; with has_range a row is
 * kept iff range[0] < out[0] < range[2] and range[1] < out[1] < range[3] in fp32 (NaN is dropped).  out [batch, cap,
 * out_dim] receives each sample's kept rows in order, counts [batch] int32 (DEVICE) min(kept, cap); rows past
 * counts[b] are left untouched and nothing is written past cap.  status [1] int32 (DEVICE) is zeroed, then gets
 *   BEVB200_SWEEPS_OVERFLOW              a sample kept more than cap rows (its first cap rows are written)
 *   BEVB200_SWEEPS_BAD_ENTRY             an entry has an unknown kind or a slot outside [0, slots) (no rows)
 *   BEVB200_SWEEPS_BAD_PARAMS            an op code of the first out_dim columns is malformed (no sample gets rows)
 *   BEVB200_RADAR_SWEEPS_BAD_CATEGORY    a row's one-hot source is NaN or rounds outside [-w, w), where the
 *                                        reference raises IndexError; that block of the row stays zero
 * Three launches sized by (batch, max_entries, slot_cap), no atomics on the output order, no host synchronisation:
 * CUDA-graph capturable with the store, params and entries refreshed between replays.  Sizes: 3 <= out_dim <= 64,
 * cap >= 1, cap * out_dim < 2^31, batch <= 65535, max_entries <= 65535, max_entries * slot_cap < 2^31.  Workspace:
 * bevb200_radar_sweeps_workspace_bytes(batch, max_entries, slot_cap) (0 for unsupported sizes): one int32 per
 * 128-row tile; a smaller one gives BEVB200_EWORKSPACE before any write. */
#define BEVB200_RADAR_LOAD_DIM 18
#define BEVB200_RADAR_SWEEP_MAX_DIM 64
#define BEVB200_RADAR_OP_RAW 0          /* arg: raw column */
#define BEVB200_RADAR_OP_XYZ 1          /* arg: j in 0..2 */
#define BEVB200_RADAR_OP_VELO 2         /* arg: j in 0..1 */
#define BEVB200_RADAR_OP_VELO_COMP 3    /* arg: j in 0..1 */
#define BEVB200_RADAR_OP_LAG 4
#define BEVB200_RADAR_OP_ONE_HOT 5      /* block: 0 (r3, 8), 1 (r11, 5), 2 (r14, 18); arg: the value */
#define BEVB200_RADAR_OP_ORDINAL 6      /* arg: the threshold i */
#define BEVB200_RADAR_OP_NUSC 7
#define BEVB200_RADAR_OP_NORMALIZE (1 << 24)
#define BEVB200_RADAR_SWEEPS_BAD_CATEGORY 8
#define BEVB200_RADAR_SWEEP_ENTRY_BYTES 112
#define BEVB200_RADAR_SWEEP_PARAMS_BYTES 1304
typedef struct {
  int32_t kind;              /* BEVB200_SWEEP_SWEEP or BEVB200_SWEEP_NONE */
  int32_t slot;
  double rotation[9];        /* sensor2lidar_rotation, row-major */
  double translation[3];     /* sensor2lidar_translation */
  double time_diff;          /* sweeps[0]['timestamp'] * 1e-6 - sweep['timestamp'] * 1e-6 */
} bevb200_radar_sweep_entry_t;
typedef struct {
  double norm_min[BEVB200_RADAR_SWEEP_MAX_DIM];    /* normalize_dims min, as float64 */
  double norm_span[BEVB200_RADAR_SWEEP_MAX_DIM];   /* max - min, computed as Python does */
  int32_t ops[BEVB200_RADAR_SWEEP_MAX_DIM];        /* per output column: the op code above */
  int32_t compensate_velocity;
  int32_t has_range;
  float range[4];                                  /* fl32(x_min, y_min, x_max, y_max) */
} bevb200_radar_sweep_params_t;
BEVB200_API size_t bevb200_radar_sweeps_workspace_bytes(int batch, int max_entries, int slot_cap);
BEVB200_API int bevb200_radar_sweeps_assemble(const float *store, int slots, int slot_cap, const int32_t *slot_rows,
                                              const bevb200_radar_sweep_params_t *params,
                                              const bevb200_radar_sweep_entry_t *entries, int batch, int max_entries,
                                              int out_dim, int cap, float *out, int32_t *counts, int32_t *status,
                                              void *workspace, size_t workspace_bytes, void *stream);

/* ---- GlobalRotScaleTrans + RandomFlip3D on the LiDAR and radar clouds and the GT boxes, ObjectRangeFilter and
 *      ObjectNameFilter (transforms_3d.py:195-232, 323-353, 534-636; base_points.py:137-272, lidar_points.py:29-34,
 *      radar_points.py:27-90, base_box3d.py:148-232, lidar_box3d.py:140-205, utils.py:6-19) ------------------------
 * One record per sample (DEVICE).  Every scalar is computed on the host with the reference's torch CPU calls: the
 * device evaluates no sine or cosine.  With enabled = 0 the sample is left exactly as it is (no identity matrix is
 * applied: it would change signed zeros and infinities).  Otherwise, in fp32 with one rounding per operation and
 * chain_j(p, R) = fma(p2, R[2][j], fma(p1, R[1][j], fma(p0, R[0][j], +0))) (every term evaluated, the zero entries
 * included; a 2-term chain for 2-vectors):
 *   rot_scale_trans  xyz = chain(xyz, point_rot); xyz += translation; xyz *= scale
 *                    radar also: c34 = chain(c34, point_rot[:2, :2]); c34 *= scale (output columns 3 and 4)
 *                    boxes: xyz = chain(xyz, box_rot); yaw += yaw_inc; vel = chain(vel, box_rot[:2, :2]) (9 columns);
 *                    xyz += translation; columns :6 and 7: *= scale
 *   flip_horizontal  y = -y (radar: and column 4; boxes: columns 1::7, then yaw = -yaw + fl32(pi))
 *   flip_vertical    x = -x (radar: and column 3; boxes: columns 0::7, then yaw = -yaw)
 * The sweep entry points below apply the record to each assembled row before the range test, so the range filter
 * sees the augmented row, as PointsRangeFilter does after RandomFlip3D.  A NULL aug pointer is the plain path. */
#define BEVB200_LIDAR_AUG_BYTES 108
typedef struct {
  int32_t enabled;           /* 0: leave the sample untouched */
  int32_t rot_scale_trans;   /* GlobalRotScaleTrans drew (is_train) */
  int32_t flip_horizontal;
  int32_t flip_vertical;
  float translation[3];      /* fl32(translation) */
  float scale;               /* fl32(scale) */
  float yaw_inc;             /* fl32(theta) */
  float point_rot[9];        /* rot_mat_T of BasePoints.rotate(fl32(-theta)), row-major */
  float box_rot[9];          /* rot_mat_T of LiDARInstance3DBoxes.rotate(fl32(theta)), row-major */
} bevb200_lidar_aug_t;

/* bevb200_lidar_sweeps_assemble with the sweep rows augmented by aug [batch] (DEVICE, or NULL for none) between the
 * transform and the range test.  Everything else is as bevb200_lidar_sweeps_assemble, which is this call with NULL. */
BEVB200_API int bevb200_lidar_sweeps_assemble_aug(const float *store, int slots, int slot_cap, int load_dim,
                                                  const int32_t *slot_rows, const bevb200_sweep_params_t *params,
                                                  const bevb200_sweep_entry_t *entries,
                                                  const bevb200_lidar_aug_t *aug, int batch, int max_entries,
                                                  int out_dim, int cap, float *out, int32_t *counts,
                                                  int32_t *status, void *workspace, size_t workspace_bytes,
                                                  void *stream);
/* bevb200_radar_sweeps_assemble with output columns 0..4 augmented by aug [batch] (DEVICE, or NULL for none) after
 * normalisation and before the range test; with aug, out_dim must be >= 5 (RadarPoints reads columns 3 and 4).
 * bevb200_radar_sweeps_assemble is this call with NULL. */
BEVB200_API int bevb200_radar_sweeps_assemble_aug(const float *store, int slots, int slot_cap,
                                                  const int32_t *slot_rows, const bevb200_radar_sweep_params_t *params,
                                                  const bevb200_radar_sweep_entry_t *entries,
                                                  const bevb200_lidar_aug_t *aug, int batch, int max_entries,
                                                  int out_dim, int cap, float *out, int32_t *counts,
                                                  int32_t *status, void *workspace, size_t workspace_bytes,
                                                  void *stream);

/* GT boxes: boxes [batch, nmax, box_dim] fp32, labels [batch, nmax] int32, counts [batch] int32 (DEVICE; the padded
 * layout of head_targets.pad_gt), box_dim 7 or 9, 0 <= nmax <= BEVB200_HEAD_TARGETS_MAX_BOXES.  Per box in order:
 * the record's transforms (above), then ObjectRangeFilter (kept iff range[0] < x < range[2] and range[1] < y <
 * range[3] in fp32; NaN is dropped) with limit_yaw(0.5, 2 pi): yaw - floor(yaw / fl32(2 pi) + 0.5) * fl32(2 pi), then
 * ObjectNameFilter (kept iff 0 <= label < num_classes).  The survivors go in order to out_boxes [batch, nmax,
 * box_dim] / out_labels [batch, nmax], out_counts [batch] their number; the rest of each sample's rows are zeroed.
 * aug may be NULL (no augmentation).  One CTA per sample, ballot ranks, no atomics on the output order, no host
 * synchronisation.  status [1] int32 (DEVICE) is zeroed, then gets
 *   BEVB200_BOX_AUG_BAD_COUNT  a count outside [0, nmax] (read as clamped to it)
 * In and out must not overlap. */
#define BEVB200_BOX_AUG_BAD_COUNT 1
BEVB200_API int bevb200_box_aug(const float *boxes, const int32_t *labels, const int32_t *counts, int batch, int nmax,
                                int box_dim, const bevb200_lidar_aug_t *aug, float range_x_min, float range_y_min,
                                float range_x_max, float range_y_max, int num_classes, float *out_boxes,
                                int32_t *out_labels, int32_t *out_counts, int32_t *status, void *stream);

/* ---- ObjectPaste (GT-database sampling) on the assembled LiDAR cloud (transforms_3d.py:357-449, dbsampler.py,
 *      box_np_ops.py:430-451, 692-775) -------------------------------------------------------------------------------
 * The draw and the collision test run on the host (bevfusion_b200/object_paste.py); the device receives the kept
 * objects.  objects [max_rows, obj_dim] fp32 (DEVICE) holds raw object rows as the database files store them;
 * object_table [num_objects, 2] int32 (DEVICE) gives each object's first row and row count (an object is valid iff
 * first >= 0, 0 <= rows <= object_cap and first + rows <= max_rows).  paste [batch] (DEVICE) gives per sample the
 * count S of kept objects and the column map of points_loader.use_dim; paste_objects [batch, max_paste] (DEVICE) the
 * kept objects in the reference's order, each with its store index, fl32(box[:3]) and its 6 face planes (n, d) from
 * points_in_rbbox(origin (0.5, 0.5, 0), z axis), computed on the host with the reference's numpy calls.
 * Per sample, with S >= 1:
 *   KEY, SWEEP and PAD rows, after the pose transform and before the augmentation, are dropped iff they lie in any
 *   kept box: a row is in a box unless one face gives ((x * n0 + y * n1) + z * n2) + d >= 0, each operation one fp32
 *   rounding with no contraction.  So a row exactly on a face is kept, and a row with a NaN coordinate is dropped.
 *   Pasted rows come first, object by object in order: out[c] = row[cols[c]], out[j] += translation[j] (j < 3, fp32),
 *   then the augmentation and the range test as for every other row (no remove_close, no pose transform).
 * A sample with S = 0 is assembled exactly as bevb200_lidar_sweeps_assemble_aug assembles it.  status also gets
 *   BEVB200_SWEEPS_BAD_PASTE   a sample's count is outside [0, max_paste], a column of its map outside [0, obj_dim),
 *                              or a kept object's index or table entry invalid: that block pastes and removes nothing
 * Everything else is as bevb200_lidar_sweeps_assemble_aug, which is this call with a NULL paste block (the object
 * arguments are then ignored).  The grid gains max_paste entries per sample, tiled as the sweep entries are, over
 * 1024-row tiles of max(slot_cap, object_cap) rows.  Sizes: 1 <= max_paste <= BEVB200_PASTE_MAX_OBJECTS,
 * 1 <= obj_dim <= 64, object_cap >= 1, max_entries + max_paste <= 65535, (max_entries + max_paste) * object_cap
 * < 2^31.  Workspace: bevb200_lidar_sweeps_paste_workspace_bytes(batch, max_entries, slot_cap, max_paste,
 * object_cap) (0 for unsupported sizes). */
#define BEVB200_SWEEPS_BAD_PASTE 8
#define BEVB200_PASTE_MAX_OBJECTS 256
#define BEVB200_PASTE_SAMPLE_BYTES 48
#define BEVB200_PASTE_OBJECT_BYTES 112
typedef struct {
  int32_t count;                           /* kept objects, 0..max_paste */
  int32_t cols[BEVB200_SWEEP_MAX_DIM];     /* points_loader.use_dim: output column c = object row[cols[c]] */
  int32_t reserved[3];
} bevb200_paste_sample_t;
typedef struct {
  int32_t index;                           /* the object in object_table */
  float translation[3];                    /* fl32(box[:3]) */
  float planes[6][4];                      /* per face: normal[3], d (surface_equ_3d's normal and -einsum) */
} bevb200_paste_object_t;
BEVB200_API size_t bevb200_lidar_sweeps_paste_workspace_bytes(int batch, int max_entries, int slot_cap, int max_paste,
                                                              int object_cap);
BEVB200_API int bevb200_lidar_sweeps_assemble_paste(const float *store, int slots, int slot_cap, int load_dim,
                                                    const int32_t *slot_rows, const bevb200_sweep_params_t *params,
                                                    const bevb200_sweep_entry_t *entries,
                                                    const bevb200_lidar_aug_t *aug, const float *objects,
                                                    int max_rows, int obj_dim, const int32_t *object_table,
                                                    int num_objects, int object_cap,
                                                    const bevb200_paste_sample_t *paste,
                                                    const bevb200_paste_object_t *paste_objects, int max_paste,
                                                    int batch, int max_entries, int out_dim, int cap, float *out,
                                                    int32_t *counts, int32_t *status, void *workspace,
                                                    size_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* BEVFUSION_B200_H_ */
