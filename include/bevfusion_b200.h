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
BEVB200_API size_t bevb200_encoder_param_bytes(const bevb200_encoder_t *enc);
BEVB200_API int bevb200_encoder_num_levels(const bevb200_encoder_t *enc);
BEVB200_API int bevb200_encoder_output_shape(const bevb200_encoder_t *enc, int32_t *shape_out, int32_t *channels_out);
BEVB200_API int bevb200_encoder_set_conv(bevb200_encoder_t *enc, int conv, const float *weight, const float *scale,
                             const float *shift, void *params, size_t params_bytes, void *stream);
BEVB200_API int bevb200_encoder_level_caps(const bevb200_encoder_t *enc, int max_voxels, int batch_size,
                               const int32_t *level_caps_host, int32_t *caps_out);
BEVB200_API size_t bevb200_encoder_workspace_bytes(const bevb200_encoder_t *enc, int max_voxels, int batch_size,
                                       const int32_t *level_caps_host);
BEVB200_API int bevb200_encoder_forward(bevb200_encoder_t *enc, const void *params, const float *voxel_features,
                            const int32_t *coors, int max_voxels, const int32_t *n_voxels_dev,
                            int batch_size, const int32_t *level_caps_host, float *dense_out,
                            long long out_batch_stride, int32_t *status_dev, void *workspace,
                            size_t workspace_bytes, void *stream, void *rulebook_stream);

#ifdef __cplusplus
}
#endif
#endif /* BEVFUSION_B200_H_ */
