"""bev_pool -- host-side mirror of mmdet3d/ops/bev_pool (bev_pool.py:1-98, bev_pool_cpu.cpp).

Same names, argument order and return layouts as the reference op:

    bev_pool_ext.bev_pool_forward(x, geom_feats, interval_lengths, interval_starts, b, d, h, w)
    bev_pool_ext.bev_pool_backward(out_grad, geom_feats, interval_lengths, interval_starts, b, d, h, w)
    QuickCumsumCuda.apply(x, geom_feats, ranks, B, D, H, W)
    bev_pool(feats, coords, B, D, H, W) -> [B, C, D, H, W]

plus the native plan API (BEVPoolPlan) that precomputes rank / sort / interval tables once
per calibration on the device and then pools straight from the un-sorted, un-filtered feature
volume.  All compute happens in libbevfusion_b200.so; CPU tensors are rejected.
"""
import ctypes
import os

import torch
from torch.autograd.function import once_differentiable

from . import _C

__all__ = ["bev_pool", "bev_pool_ext", "QuickCumsumCuda", "BEVPoolPlan", "gen_dx_bx"]

# status word of a sync-free plan's fused lift (tables.lift_form; BEVB200_LIFT_* in include/bevfusion_b200.h)
_LIFT_COLUMNS, _LIFT_ROWS = 0, 1
# default column-table cap of a sync-free plan, per (camera, image column, depth bin): see DESIGN.md section 4.24
_SEGMENTS_PER_COLUMN_BIN = 5


def _ws(nbytes, device):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)


class _BevPoolExt:
    """Stand-in for the reference pybind module `bev_pool_ext` (bev_pool_cpu.cpp:89-94)."""

    @staticmethod
    def bev_pool_forward(x, geom_feats, interval_lengths, interval_starts, b, d, h, w):
        _C.require_cuda(x, "x", torch.float32)
        _C.require_cuda(geom_feats, "geom_feats", torch.int32)
        _C.require_cuda(interval_lengths, "interval_lengths", torch.int32)
        _C.require_cuda(interval_starts, "interval_starts", torch.int32)
        n, c = x.shape
        b, d, h, w = int(b), int(d), int(h), int(w)
        n_int = interval_lengths.shape[0]
        with torch.cuda.device(x.device):
            out = torch.empty((b, d, h, w, c), dtype=x.dtype, device=x.device)
            nbytes = _C.lib().bevb200_bev_pool_workspace_bytes(n, c)
            ws = _ws(nbytes, x.device)
            rc = _C.lib().bevb200_bev_pool(b, d, h, w, n, c, n_int, _C.ptr(x), _C.ptr(geom_feats),
                                           _C.ptr(interval_starts), _C.ptr(interval_lengths),
                                           _C.ptr(out), _C.ptr(ws), ws.numel(),
                                           _C.current_stream(x.device))
        _C.check(rc, "bev_pool_forward")
        return out

    @staticmethod
    def bev_pool_backward(out_grad, geom_feats, interval_lengths, interval_starts, b, d, h, w):
        _C.require_cuda(out_grad, "out_grad", torch.float32)
        _C.require_cuda(geom_feats, "geom_feats", torch.int32)
        _C.require_cuda(interval_lengths, "interval_lengths", torch.int32)
        _C.require_cuda(interval_starts, "interval_starts", torch.int32)
        n = geom_feats.shape[0]
        c = out_grad.shape[4]
        b, d, h, w = int(b), int(d), int(h), int(w)
        with torch.cuda.device(out_grad.device):
            x_grad = torch.empty((n, c), dtype=out_grad.dtype, device=out_grad.device)
            rc = _C.lib().bevb200_bev_pool_grad(b, d, h, w, n, c, interval_lengths.shape[0],
                                                _C.ptr(out_grad), _C.ptr(geom_feats),
                                                _C.ptr(interval_starts), _C.ptr(interval_lengths),
                                                _C.ptr(x_grad), _C.current_stream(out_grad.device))
        _C.check(rc, "bev_pool_backward")
        return x_grad


bev_pool_ext = _BevPoolExt()


class QuickCumsumCuda(torch.autograd.Function):
    """Same contract as the reference class (bev_pool.py:38-81): x / geom_feats / ranks are
    already sorted by rank; interval table from rank changes; grad w.r.t. the sorted rows."""

    @staticmethod
    def forward(ctx, x, geom_feats, ranks, B, D, H, W):
        kept = torch.ones(x.shape[0], device=x.device, dtype=torch.bool)
        kept[1:] = ranks[1:] != ranks[:-1]
        interval_starts = torch.where(kept)[0].int()
        interval_lengths = torch.zeros_like(interval_starts)
        interval_lengths[:-1] = interval_starts[1:] - interval_starts[:-1]
        interval_lengths[-1] = x.shape[0] - interval_starts[-1]
        geom_feats = geom_feats.int().contiguous()
        out = bev_pool_ext.bev_pool_forward(x.contiguous(), geom_feats, interval_lengths,
                                            interval_starts, B, D, H, W)
        ctx.save_for_backward(interval_starts, interval_lengths, geom_feats)
        ctx.saved_shapes = B, D, H, W
        return out

    @staticmethod
    def backward(ctx, out_grad):
        interval_starts, interval_lengths, geom_feats = ctx.saved_tensors
        B, D, H, W = ctx.saved_shapes
        out_grad = out_grad.contiguous()
        x_grad = bev_pool_ext.bev_pool_backward(out_grad, geom_feats, interval_lengths,
                                                interval_starts, B, D, H, W)
        return x_grad, None, None, None, None, None, None


class _PoolTables:
    """Device-resident rank / perm / interval tables of one (geometry, grid) pair.

    Tables of a sync-free plan (BEVPoolPlan.from_cameras(..., sync=False)) are sized for all n_total points and carry
    `counts`, int32 [4] on the device = {n_kept, n_intervals, n_segments, lift form}; n_kept, n_intervals, n_segments
    and lift_form are then 0-d views of it, and only the leading n_kept / n_intervals entries of the tables are valid."""

    def __init__(self, ranks, perm, geom, starts, lengths, n_kept, n_intervals, n_total, dims, counts=None):
        self.ranks, self.perm, self.geom = ranks, perm, geom
        self.starts, self.lengths = starts, lengths
        self.n_kept, self.n_intervals, self.n_total = n_kept, n_intervals, n_total
        self.dims = dims  # (B, D, H, W)
        self.counts = counts
        if counts is not None:
            self.n_segments, self.lift_form = counts[2], counts[3]
        self._ws_cache = {}

    def counts_ptr(self, k):
        """device address of counts[k]"""
        return _C.ptr(self.counts) + 4 * k

    def workspace(self, key, nbytes, device):
        """A workspace kept with the tables (sync-free plans allocate once per channel count).  One asked for during a
        CUDA-graph capture comes from the graph's pool and is not kept."""
        if torch.cuda.is_current_stream_capturing():
            return _ws(nbytes, device)
        ws = self._ws_cache.get(key)
        if ws is None or ws.numel() < nbytes:
            ws = self._ws_cache[key] = _ws(nbytes, device)
        return ws


def _finish_tables(n_total, device, dims, call):
    i32 = dict(dtype=torch.int32, device=device)
    ranks = torch.empty(n_total, **i32)
    perm = torch.empty(n_total, **i32)
    geom = torch.empty((n_total, 4), **i32)
    starts = torch.empty(n_total, **i32)
    lengths = torch.empty(n_total, **i32)
    counts = torch.zeros(2, **i32)
    ws = _ws(_C.lib().bevb200_bev_pool_prepare_workspace_bytes(n_total), device)
    rc = call(ranks, perm, geom, starts, lengths, counts, ws)
    _C.check(rc, "bev_pool_prepare")
    n_kept, n_int = (int(v) for v in counts.tolist())  # one D2H read per calibration
    return _PoolTables(ranks, perm, geom[:n_kept], starts[:n_int], lengths[:n_int], n_kept, n_int,
                       n_total, dims)


def prepare_from_coords(coords, B, D, H, W):
    """rank + stable sort + interval table of already-quantised (x, y, z, b) coords
    (what bev_pool() does at bev_pool.py:87-94 and QuickCumsumCuda at :41-46)."""
    _C.require_cuda(coords, "coords")
    coords = coords.long().contiguous()
    n = coords.shape[0]
    B, D, H, W = int(B), int(D), int(H), int(W)
    with torch.cuda.device(coords.device):
        return _finish_tables(n, coords.device, (B, D, H, W), lambda r, p, g, s, l, c, ws:
                              _C.lib().bevb200_bev_pool_prepare_coords(
                                  _C.ptr(coords), n, B, D, H, W, _C.ptr(r), _C.ptr(p), _C.ptr(g),
                                  _C.ptr(s), _C.ptr(l), _C.ptr(c), _C.ptr(ws), ws.numel(),
                                  _C.current_stream(coords.device)))


def gen_dx_bx(xbound, ybound, zbound):
    """Same arithmetic as mmdet3d/models/vtransforms/base.py:15-21."""
    dx = torch.Tensor([row[2] for row in [xbound, ybound, zbound]])
    bx = torch.Tensor([row[0] + row[2] / 2.0 for row in [xbound, ybound, zbound]])
    nx = torch.LongTensor([(row[1] - row[0]) / row[2] for row in [xbound, ybound, zbound]])
    return dx, bx, nx


def _grid_host(dx, bx, nx, B):
    """Host arrays of the quantisation grid -- fp32 lower = bx - dx/2 (base.py:149, evaluated in fp32), fp32 dx,
    int32 nx -- and the pooled dims (B, nz, nx, ny)."""
    lower = bx.float().cpu() - dx.float().cpu() / 2.0
    lower_h = _C.host_array(ctypes.c_float, [float(v) for v in lower])
    dx_h = _C.host_array(ctypes.c_float, [float(v) for v in dx.float().cpu()])
    nx_h = _C.host_array(ctypes.c_int32, [int(v) for v in nx])
    return lower_h, dx_h, nx_h, (int(B), int(nx[2]), int(nx[0]), int(nx[1]))


def prepare_from_geometry(geom_xyz, dx, bx, nx, B):
    """quantise + filter + rank + sort + intervals of lidar-frame frustum points
    (base.py:149-169 then bev_pool.py:87-94, :41-46), all on the device."""
    _C.require_cuda(geom_xyz, "geom_xyz", torch.float32)
    g = geom_xyz.reshape(-1, 3)
    n_total = g.shape[0]
    assert n_total % B == 0
    lower_h, dx_h, nx_h, dims = _grid_host(dx, bx, nx, B)
    with torch.cuda.device(g.device):
        return _finish_tables(n_total, g.device, dims, lambda r, p, gm, s, l, c, ws:
                              _C.lib().bevb200_bev_pool_prepare_geom(
                                  _C.ptr(g), n_total, n_total // B,
                                  ctypes.cast(lower_h, ctypes.c_void_p),
                                  ctypes.cast(dx_h, ctypes.c_void_p),
                                  ctypes.cast(nx_h, ctypes.c_void_p), int(B), _C.ptr(r), _C.ptr(p),
                                  _C.ptr(gm), _C.ptr(s), _C.ptr(l), _C.ptr(c), _C.ptr(ws),
                                  ws.numel(), _C.current_stream(g.device)))


def _camera_params(dev, B, N, camera2lidar_rots, camera2lidar_trans, intrins, post_rots, post_trans, extra_rots,
                   extra_trans, inverse):
    """cam_params [B*N, 24] and extra_params [B, 12] (or None) of bevb200_bev_pool_prepare_cameras; `inverse` computes
    the batched 3x3 inverses"""
    f32 = dict(dtype=torch.float32, device=dev)
    inv_post = inverse(post_rots.to(**f32))
    combine = camera2lidar_rots.to(**f32).matmul(inverse(intrins.to(**f32)))
    cam = torch.cat([inv_post.reshape(B * N, 9), post_trans.to(**f32).reshape(B * N, 3), combine.reshape(B * N, 9),
                     camera2lidar_trans.to(**f32).reshape(B * N, 3)], 1).contiguous()
    extra = None
    if extra_rots is not None or extra_trans is not None:
        er = extra_rots.to(**f32) if extra_rots is not None else torch.eye(3, **f32).repeat(B, 1, 1)
        et = extra_trans.to(**f32) if extra_trans is not None else torch.zeros(B, 3, **f32)
        extra = torch.cat([er.reshape(B, 9), et.reshape(B, 3)], 1).contiguous()
    return cam, extra


def prepare_from_cameras(frustum, camera2lidar_rots, camera2lidar_trans, intrins, post_rots, post_trans, dx, bx, nx,
                         extra_rots=None, extra_trans=None, return_geometry=False):
    """get_geometry (base.py:92-135) + quantise / filter / rank / sort / intervals in one library call: the
    [B, N, D, fH, fW, 3] geometry tensor is not materialised.  frustum [D, fH, fW, 3] from create_frustum; the
    calibration tensors are the reference's ([B, N, 3, 3] / [B, N, 3]; extra_* [B, 3, 3] / [B, 3]), on the GPU.
    The 3x3 inverses and the rots @ inv(intrins) product are computed with torch exactly as the reference does."""
    _C.require_cuda(frustum, "frustum", torch.float32)
    dev = frustum.device
    B, N = camera2lidar_trans.shape[:2]
    f32 = dict(dtype=torch.float32, device=dev)
    cam, extra = _camera_params(dev, B, N, camera2lidar_rots, camera2lidar_trans, intrins, post_rots, post_trans,
                                extra_rots, extra_trans, torch.inverse)
    fr = frustum.reshape(-1, 3).contiguous()
    n_fr = fr.shape[0]
    n_total = n_fr * B * N
    lower_h, dx_h, nx_h, dims = _grid_host(dx, bx, nx, B)
    with torch.cuda.device(dev):
        geom = torch.empty((n_total, 3), **f32) if return_geometry else None
        tables = _finish_tables(n_total, dev, dims, lambda r, p, gm, s, l, c, ws:
                                _C.lib().bevb200_bev_pool_prepare_cameras(
                                    _C.ptr(fr), n_fr, B * N, N, _C.ptr(cam), _C.ptr(extra),
                                    ctypes.cast(lower_h, ctypes.c_void_p), ctypes.cast(dx_h, ctypes.c_void_p),
                                    ctypes.cast(nx_h, ctypes.c_void_p), int(B), _C.ptr(geom), _C.ptr(r), _C.ptr(p),
                                    _C.ptr(gm), _C.ptr(s), _C.ptr(l), _C.ptr(c), _C.ptr(ws), ws.numel(),
                                    _C.current_stream(dev)))
    return (tables, geom) if return_geometry else tables


class _PoolPerm(torch.autograd.Function):
    """out[b, d, h, w, :] = sum of the rows of x (ORIGINAL order) that fall into the cell."""

    @staticmethod
    def forward(ctx, x, tables):
        _C.require_cuda(x, "x", torch.float32)
        assert x.shape[0] == tables.n_total
        B, D, H, W = tables.dims
        c = x.shape[1]
        with torch.cuda.device(x.device):
            out = torch.empty((B, D, H, W, c), dtype=x.dtype, device=x.device)
            if tables.counts is not None:       # sync-free tables: sizes from the device
                L = _C.lib()
                ws = tables.workspace(("pool", c), L.bevb200_bev_pool_dev_workspace_bytes(tables.n_total, c), x.device)
                rc = L.bevb200_bev_pool_perm_dev(
                    B, D, H, W, tables.n_total, c, _C.ptr(x), _C.ptr(tables.perm), _C.ptr(tables.geom),
                    _C.ptr(tables.starts), _C.ptr(tables.lengths), _C.ptr(tables.counts), _C.ptr(out), _C.ptr(ws),
                    ws.numel(), _C.current_stream(x.device))
                _C.check(rc, "bev_pool_perm_dev")
                ctx.tables, ctx.c = tables, c
                return out
            ws = _ws(_C.lib().bevb200_bev_pool_workspace_bytes(tables.n_kept, c), x.device)
            rc = _C.lib().bevb200_bev_pool_perm(
                B, D, H, W, tables.n_kept, c, tables.n_intervals, _C.ptr(x), _C.ptr(tables.perm),
                _C.ptr(tables.geom), _C.ptr(tables.starts), _C.ptr(tables.lengths), _C.ptr(out),
                _C.ptr(ws), ws.numel(), _C.current_stream(x.device))
        _C.check(rc, "bev_pool_perm")
        ctx.tables = tables
        ctx.c = c
        return out

    @staticmethod
    def backward(ctx, out_grad):
        t = ctx.tables
        B, D, H, W = t.dims
        out_grad = out_grad.contiguous()
        with torch.cuda.device(out_grad.device):
            x_grad = torch.empty((t.n_total, ctx.c), dtype=out_grad.dtype, device=out_grad.device)
            if t.counts is not None:
                rc = _C.lib().bevb200_bev_pool_grad_perm_dev(
                    B, D, H, W, t.n_total, ctx.c, _C.ptr(out_grad), _C.ptr(t.perm), _C.ptr(t.geom), _C.ptr(t.starts),
                    _C.ptr(t.lengths), _C.ptr(t.counts), _C.ptr(x_grad), _C.current_stream(out_grad.device))
                _C.check(rc, "bev_pool_grad_perm_dev")
                return x_grad, None
            rc = _C.lib().bevb200_bev_pool_grad_perm(
                B, D, H, W, t.n_kept, t.n_total, ctx.c, t.n_intervals, _C.ptr(out_grad),
                _C.ptr(t.perm), _C.ptr(t.geom), _C.ptr(t.starts), _C.ptr(t.lengths),
                _C.ptr(x_grad), _C.current_stream(out_grad.device))
        _C.check(rc, "bev_pool_grad_perm")
        return x_grad, None


def bev_pool(feats, coords, B, D, H, W):
    """Drop-in for mmdet3d.ops.bev_pool.bev_pool (bev_pool.py:84-98).

    feats [N, C] fp32, coords [N, 4] integer (x, y, z, b).  Returns [B, C, D, H, W].
    Rank, (stable) sort and interval table are computed by one library call; the features are
    never gathered into sorted order -- the pooling kernel reads them through the permutation,
    and the backward pass writes gradients straight back in the caller's row order."""
    assert feats.shape[0] == coords.shape[0]
    tables = prepare_from_coords(coords, B, D, H, W)
    x = _PoolPerm.apply(feats.contiguous(), tables)
    x = x.permute(0, 4, 1, 2, 3).contiguous()
    return x


class _LiftPool(torch.autograd.Function):
    """out = BEVPoolPlan.lift_pool(depth, ctx) with gradients for depth and ctx.  Saves depth and ctx, never the
    lifted volume; the forward is the inference forward, bit for bit."""

    @staticmethod
    def forward(fctx, plan, depth, ctx):
        out = plan._lift_pool_forward(depth, ctx)
        fctx.plan = plan
        fctx.save_for_backward(depth, ctx)
        return out

    @staticmethod
    @once_differentiable
    def backward(fctx, out_grad):
        depth, ctx = fctx.saved_tensors
        _, want_depth, want_ctx = fctx.needs_input_grad
        ddepth, dctx = fctx.plan._lift_pool_backward(out_grad.contiguous(), depth, ctx, want_depth, want_ctx)
        return None, ddepth, dctx


class BEVPoolPlan:
    """Precomputed pooling plan for a fixed camera geometry (native API).

    plan = BEVPoolPlan(geom, xbound, ybound, zbound)       # once per calibration / augmentation
    bev  = plan(x)    # x [B, N, D, H, W, C] -> [B, C*nz, nx, ny]  == BaseTransform.bev_pool(geom, x)
    """

    def __init__(self, geom, xbound, ybound, zbound):
        self.dx, self.bx, self.nx = gen_dx_bx(xbound, ybound, zbound)
        self.B = geom.shape[0]
        self.tables = prepare_from_geometry(geom.contiguous(), self.dx, self.bx, self.nx, self.B)

    @classmethod
    def from_cameras(cls, frustum, camera2lidar_rots, camera2lidar_trans, intrins, post_rots, post_trans,
                     xbound, ybound, zbound, extra_rots=None, extra_trans=None, sync=True, max_segments=None):
        """Plan straight from the calibration: get_geometry (base.py:92-135) runs inside the plan build, the
        96 MB geometry tensor is never written (what a per-sample camera2lidar needs every frame).

        sync=False builds a sync-free plan for calibration that changes every step (training augmentation,
        per-sample camera2lidar): every table, count and workspace is allocated once, at capacity for
        (B, N, D, fH, fW); rebuild_() refills them from new calibration without a host round trip, and pool, lift,
        lift_pool and their backward read the point, interval and segment counts from the device.  A step of
        rebuild_ -> lift_pool -> backward can then be captured in a CUDA graph.  max_segments caps the column
        tables of the fused lift (default: _SEGMENTS_PER_COLUMN_BIN per (camera, image column, depth bin)); a
        calibration with more segments runs the row kernels instead, chosen on the device (tables.lift_form)."""
        self = cls.__new__(cls)
        self.dx, self.bx, self.nx = gen_dx_bx(xbound, ybound, zbound)
        self.B = int(camera2lidar_trans.shape[0])
        if not sync:
            self._init_sync_free(frustum, int(camera2lidar_trans.shape[1]), max_segments)
            self.rebuild_(camera2lidar_rots, camera2lidar_trans, intrins, post_rots, post_trans, extra_rots, extra_trans)
            return self
        self.tables = prepare_from_cameras(frustum, camera2lidar_rots, camera2lidar_trans, intrins, post_rots,
                                           post_trans, self.dx, self.bx, self.nx, extra_rots, extra_trans)
        return self

    def _init_sync_free(self, frustum, N, max_segments):
        _C.require_cuda(frustum, "frustum", torch.float32)
        if frustum.dim() != 4 or frustum.shape[3] != 3:
            raise ValueError("frustum must be [D, fH, fW, 3], got %s" % (tuple(frustum.shape),))
        D, fH, fW = (int(v) for v in frustum.shape[:3])
        B, dev = self.B, frustum.device
        self._frustum = frustum.reshape(-1, 3).contiguous()
        n_total = self._frustum.shape[0] * B * N
        self._grid = _grid_host(self.dx, self.bx, self.nx, B)
        self._cams = (B, N, D, fH, fW)
        L = _C.lib()
        i32 = dict(dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            counts = torch.zeros(4, **i32)
            self.tables = _PoolTables(torch.empty(n_total, **i32), torch.empty(n_total, **i32),
                                      torch.empty((n_total, 4), **i32), torch.empty(n_total, **i32),
                                      torch.empty(n_total, **i32), counts[0], counts[1], n_total, self._grid[3],
                                      counts=counts)
            self._prepare_ws = _ws(L.bevb200_bev_pool_prepare_workspace_bytes(n_total), dev)
            self._columns = fH <= 64
            if not self._columns:
                # the segment mask holds 64 pixel rows: taller features always run the row kernels
                counts[3] = _LIFT_ROWS
                self.max_segments = 0
                return
            if max_segments is None:
                max_segments = _SEGMENTS_PER_COLUMN_BIN * B * N * fW * D
            self.max_segments = min(int(max_segments), n_total)
            if self.max_segments <= 0:
                raise ValueError("max_segments must be positive, got %d" % self.max_segments)
            cap = self.max_segments
            self._seg = dict(col_begin=torch.empty(B * N * fW + 1, **i32),
                             seg_key=torch.empty(cap, dtype=torch.int64, device=dev),
                             seg_mask=torch.empty(cap, dtype=torch.int64, device=dev),
                             seg_slot=torch.empty(cap, **i32), ival_begin=torch.empty(n_total + 1, **i32),
                             ws=_ws(L.bevb200_bev_pool_lift_prepare_dev_workspace_bytes(n_total, cap), dev))

    def rebuild_(self, camera2lidar_rots, camera2lidar_trans, intrins, post_rots, post_trans, extra_rots=None,
                 extra_trans=None):
        """Refill a sync-free plan's tables (and the fused lift's column tables) from new calibration, in place and
        without synchronising the host: [B, N, 3, 3] / [B, N, 3] fp32 tensors on the plan's device as for
        from_cameras, extra_* [B, 3, 3] / [B, 3] or None.  Raises ValueError, before any launch and with the tables
        untouched, on a wrong shape, dtype or device."""
        if getattr(self, "_cams", None) is None:
            raise ValueError("rebuild_ needs a plan built with BEVPoolPlan.from_cameras(..., sync=False)")
        B, N, D, fH, fW = self._cams
        t = self.tables
        dev = t.perm.device
        args = [("camera2lidar_rots", camera2lidar_rots, (B, N, 3, 3)),
                ("camera2lidar_trans", camera2lidar_trans, (B, N, 3)), ("intrins", intrins, (B, N, 3, 3)),
                ("post_rots", post_rots, (B, N, 3, 3)), ("post_trans", post_trans, (B, N, 3)),
                ("extra_rots", extra_rots, (B, 3, 3)), ("extra_trans", extra_trans, (B, 3))]
        for name, v, shape in args:
            if v is None and name.startswith("extra"):
                continue
            if not isinstance(v, torch.Tensor):
                raise ValueError("%s must be a tensor" % name)
            if tuple(v.shape) != shape:
                raise ValueError("%s has shape %s, the plan needs %s" % (name, tuple(v.shape), shape))
            if v.dtype != torch.float32:
                raise ValueError("%s must be float32, got %s" % (name, v.dtype))
            if v.device != dev:
                raise ValueError("%s is on %s, the plan on %s" % (name, v.device, dev))
        # torch.linalg.inv_ex runs the factorisation of torch.inverse without reading its error flag back to the
        # host: the same inverses, bit for bit, and capturable in a CUDA graph
        cam, extra = _camera_params(dev, B, N, camera2lidar_rots, camera2lidar_trans, intrins, post_rots, post_trans,
                                    extra_rots, extra_trans, lambda m: torch.linalg.inv_ex(m)[0])
        lower_h, dx_h, nx_h, _ = self._grid
        fr = self._frustum
        L = _C.lib()
        with torch.cuda.device(dev):
            stream = _C.current_stream(dev)
            rc = L.bevb200_bev_pool_prepare_cameras(
                _C.ptr(fr), fr.shape[0], B * N, N, _C.ptr(cam), _C.ptr(extra), ctypes.cast(lower_h, ctypes.c_void_p),
                ctypes.cast(dx_h, ctypes.c_void_p), ctypes.cast(nx_h, ctypes.c_void_p), B, None, _C.ptr(t.ranks),
                _C.ptr(t.perm), _C.ptr(t.geom), _C.ptr(t.starts), _C.ptr(t.lengths), _C.ptr(t.counts),
                _C.ptr(self._prepare_ws), self._prepare_ws.numel(), stream)
            _C.check(rc, "bev_pool_prepare_cameras")
            if self._columns:
                sg = self._seg
                rc = L.bevb200_bev_pool_lift_prepare_dev(
                    _C.ptr(t.perm), _C.ptr(t.starts), _C.ptr(t.counts), t.n_total, self.max_segments, B * N, D, fH, fW,
                    _C.ptr(sg["col_begin"]), _C.ptr(sg["seg_key"]), _C.ptr(sg["seg_mask"]), _C.ptr(sg["seg_slot"]),
                    _C.ptr(sg["ival_begin"]), t.counts_ptr(2), t.counts_ptr(3), _C.ptr(sg["ws"]), sg["ws"].numel(),
                    stream)
                _C.check(rc, "bev_pool_lift_prepare_dev")
        return self

    def pool(self, x):
        """[B, N, D, H, W, C] (or [N', C]) -> raw op output [B, nz, nx, ny, C]."""
        c = x.shape[-1]
        return _PoolPerm.apply(x.reshape(-1, c).contiguous(), self.tables)

    def _lift_tables(self, cameras, D, fH, fW):
        """(column, depth bin, cell) segment tables of the column lift, built once per plan on first use."""
        key = (cameras, D, fH, fW)
        cached = getattr(self, "_lift_cache", None)
        if cached is not None and cached[0] == key:
            if torch.cuda.is_current_stream_capturing():
                self._lift_captured = True
            return cached[1]
        if cached is not None and getattr(self, "_lift_captured", False):
            # a graph captured earlier still reads these tables at every replay: dropping them would let the
            # allocator reuse the memory under it, so tables a capture used stay alive with the plan
            self.__dict__.setdefault("_lift_graph_held", []).append(cached[1])
        self._lift_captured = False
        t = self.tables
        dev = t.perm.device
        L = _C.lib()
        with torch.cuda.device(dev):
            i32 = dict(dtype=torch.int32, device=dev)
            col_begin = torch.empty(cameras * fW + 1, **i32)
            seg_key = torch.empty(max(t.n_kept, 1), dtype=torch.int64, device=dev)
            seg_mask = torch.empty(max(t.n_kept, 1), dtype=torch.int64, device=dev)
            seg_slot = torch.empty(max(t.n_kept, 1), **i32)
            ival_begin = torch.empty(t.n_intervals + 1, **i32)
            n_seg = torch.zeros(1, **i32)
            ws = _ws(L.bevb200_bev_pool_lift_prepare_workspace_bytes(t.n_kept), dev)
            rc = L.bevb200_bev_pool_lift_prepare(_C.ptr(t.perm), _C.ptr(t.starts), t.n_kept, t.n_intervals, cameras, D,
                                                 fH, fW, _C.ptr(col_begin), _C.ptr(seg_key), _C.ptr(seg_mask),
                                                 _C.ptr(seg_slot), _C.ptr(ival_begin), _C.ptr(n_seg), _C.ptr(ws),
                                                 ws.numel(), _C.current_stream(dev))
            _C.check(rc, "bev_pool_lift_prepare")
            n = int(n_seg.item())
            tables = (col_begin, seg_key[:max(n, 1)].clone(), seg_mask[:max(n, 1)].clone(), seg_slot[:max(n, 1)].clone(),
                      ival_begin, n)
        self._lift_cache = (key, tables)
        return tables

    def lift_pool(self, depth, ctx):
        """Fused LSS lift + pool: `depth` [B, N, D, fH, fW] softmax volume and `ctx` [B, N, fH, fW, C]
        channels-last context features -> raw op output [B, nz, nx, ny, C], equal to
        pool(depth.unsqueeze(-1) * ctx.unsqueeze(2)) without materialising that volume
        (lss.py:68-73 / depth_lss.py:92-97 followed by base.py:141-176).

        Differentiable in `depth` and `ctx` (training): when grad is enabled and either requires grad, the
        backward computes their gradients straight from the output gradient, again without the volume or
        its gradient (saved for backward: depth, ctx and this plan)."""
        if torch.is_grad_enabled() and (depth.requires_grad or ctx.requires_grad):
            return _LiftPool.apply(self, depth, ctx)
        return self._lift_pool_forward(depth, ctx)

    def _lift_pool_forward(self, depth, ctx):
        _C.require_cuda(depth, "depth", torch.float32)
        _C.require_cuda(ctx, "ctx", torch.float32)
        B, N, D, fH, fW = depth.shape
        c = ctx.shape[-1]
        assert tuple(ctx.shape) == (B, N, fH, fW, c)
        t = self.tables
        assert depth.numel() == t.n_total
        Bq, Dq, Hq, Wq = t.dims
        if t.counts is not None:
            return self._lift_pool_forward_dev(depth, ctx)
        if fH <= 64 and os.environ.get("BEVB200_LIFT_VARIANT", "columns") != "rows":
            # column formulation: context rows and depth values of an image column are staged once in shared
            # memory and every (column, depth bin, cell) segment is evaluated from there
            col_begin, seg_key, seg_mask, seg_slot, ival_begin, n_seg = self._lift_tables(B * N, D, fH, fW)
            L = _C.lib()
            with torch.cuda.device(depth.device):
                out = torch.empty((Bq, Dq, Hq, Wq, c), dtype=torch.float32, device=depth.device)
                ws = _ws(L.bevb200_bev_pool_lift_columns_workspace_bytes(n_seg, t.n_intervals, c), depth.device)
                rc = L.bevb200_bev_pool_lift_columns(
                    Bq, Dq, Hq, Wq, t.n_kept, c, t.n_intervals, _C.ptr(depth), _C.ptr(ctx), B * N, D, fH, fW,
                    _C.ptr(t.geom), _C.ptr(t.starts), _C.ptr(col_begin), _C.ptr(seg_key), _C.ptr(seg_mask),
                    _C.ptr(seg_slot), _C.ptr(ival_begin), n_seg, _C.ptr(out), _C.ptr(ws), ws.numel(),
                    _C.current_stream(depth.device))
            _C.check(rc, "bev_pool_lift_columns")
            return out
        with torch.cuda.device(depth.device):
            out = torch.empty((Bq, Dq, Hq, Wq, c), dtype=torch.float32, device=depth.device)
            ws = _ws(_C.lib().bevb200_bev_pool_workspace_bytes(t.n_kept, c), depth.device)
            rc = _C.lib().bevb200_bev_pool_lift(
                Bq, Dq, Hq, Wq, t.n_kept, c, t.n_intervals, _C.ptr(depth), _C.ptr(ctx), D, fH * fW,
                _C.ptr(t.perm), _C.ptr(t.geom), _C.ptr(t.starts), _C.ptr(t.lengths), _C.ptr(out),
                _C.ptr(ws), ws.numel(), _C.current_stream(depth.device))
        _C.check(rc, "bev_pool_lift")
        return out

    def _lift_pool_forward_dev(self, depth, ctx):
        """sync-free plan: the column and the row form are both launched and the status word of the column-table
        prepare (tables.lift_form) lets exactly one of them write `out`"""
        B, N, D, fH, fW = self._cams
        if tuple(depth.shape) != (B, N, D, fH, fW):
            raise ValueError("depth has shape %s, the plan needs %s" % (tuple(depth.shape), self._cams))
        c = ctx.shape[-1]
        t = self.tables
        Bq, Dq, Hq, Wq = t.dims
        dev = depth.device
        L = _C.lib()
        with torch.cuda.device(dev):
            stream = _C.current_stream(dev)
            out = torch.empty((Bq, Dq, Hq, Wq, c), dtype=torch.float32, device=dev)
            if self._columns:
                sg = self._seg
                ws = t.workspace(("columns", c), L.bevb200_bev_pool_lift_columns_dev_workspace_bytes(
                    self.max_segments, t.n_total, c), dev)
                rc = L.bevb200_bev_pool_lift_columns_dev(
                    Bq, Dq, Hq, Wq, t.n_total, c, _C.ptr(depth), _C.ptr(ctx), B * N, D, fH, fW, _C.ptr(t.geom),
                    _C.ptr(t.starts), _C.ptr(sg["col_begin"]), _C.ptr(sg["seg_key"]), _C.ptr(sg["seg_mask"]),
                    _C.ptr(sg["seg_slot"]), _C.ptr(sg["ival_begin"]), self.max_segments, _C.ptr(t.counts),
                    t.counts_ptr(3), _C.ptr(out), _C.ptr(ws), ws.numel(), stream)
                _C.check(rc, "bev_pool_lift_columns_dev")
            ws = t.workspace(("pool", c), L.bevb200_bev_pool_dev_workspace_bytes(t.n_total, c), dev)
            rc = L.bevb200_bev_pool_lift_dev(
                Bq, Dq, Hq, Wq, t.n_total, c, _C.ptr(depth), _C.ptr(ctx), D, fH * fW, _C.ptr(t.perm), _C.ptr(t.geom),
                _C.ptr(t.starts), _C.ptr(t.lengths), _C.ptr(t.counts), t.counts_ptr(3), _C.ptr(out), _C.ptr(ws),
                ws.numel(), stream)
            _C.check(rc, "bev_pool_lift_dev")
        return out

    def _lift_pool_backward(self, out_grad, depth, ctx, want_depth, want_ctx):
        """(ddepth, dctx) of lift_pool from the gradient of its output; a gradient not wanted is None.
        The column kernel runs wherever the column formulation can (fH <= 64), the pixel kernel otherwise."""
        _C.require_cuda(out_grad, "out_grad", torch.float32)
        B, N, D, fH, fW = depth.shape
        c = ctx.shape[-1]
        t = self.tables
        Bq, Dq, Hq, Wq = t.dims
        assert tuple(out_grad.shape) == (Bq, Dq, Hq, Wq, c)
        dev = depth.device
        L = _C.lib()
        with torch.cuda.device(dev):
            ddepth = torch.empty_like(depth) if want_depth else None
            dctx = torch.empty_like(ctx) if want_ctx else None
            if t.counts is not None:
                # sync-free plan: both backwards are launched, the status word picks the one that writes
                stream = _C.current_stream(dev)
                nbytes = L.bevb200_bev_pool_lift_backward_dev_workspace_bytes(t.n_total, c)
                if self._columns:
                    nbytes = max(nbytes, L.bevb200_bev_pool_lift_columns_backward_dev_workspace_bytes(
                        self.max_segments, c))
                ws = t.workspace("backward", nbytes, dev)
                if self._columns:
                    sg = self._seg
                    rc = L.bevb200_bev_pool_lift_columns_backward_dev(
                        Bq, Dq, Hq, Wq, t.n_total, c, _C.ptr(out_grad), _C.ptr(depth), _C.ptr(ctx), B * N, D, fH, fW,
                        _C.ptr(t.geom), _C.ptr(t.starts), _C.ptr(sg["col_begin"]), _C.ptr(sg["seg_key"]),
                        _C.ptr(sg["seg_mask"]), self.max_segments, _C.ptr(t.counts), t.counts_ptr(2), t.counts_ptr(3),
                        _C.ptr(ddepth), _C.ptr(dctx), _C.ptr(ws), ws.numel(), stream)
                    _C.check(rc, "bev_pool_lift_columns_backward_dev")
                rc = L.bevb200_bev_pool_lift_backward_dev(
                    Bq, Dq, Hq, Wq, t.n_total, c, _C.ptr(out_grad), _C.ptr(depth), _C.ptr(ctx), D, fH * fW,
                    _C.ptr(t.perm), _C.ptr(t.geom), _C.ptr(t.starts), _C.ptr(t.lengths), _C.ptr(t.counts),
                    t.counts_ptr(3), _C.ptr(ddepth), _C.ptr(dctx), _C.ptr(ws), ws.numel(), stream)
                _C.check(rc, "bev_pool_lift_backward_dev")
            elif fH <= 64:
                col_begin, seg_key, seg_mask, _, _, n_seg = self._lift_tables(B * N, D, fH, fW)
                ws = _ws(L.bevb200_bev_pool_lift_columns_backward_workspace_bytes(n_seg, t.n_intervals, c), dev)
                rc = L.bevb200_bev_pool_lift_columns_backward(
                    Bq, Dq, Hq, Wq, t.n_kept, c, t.n_intervals, _C.ptr(out_grad), _C.ptr(depth), _C.ptr(ctx), B * N, D,
                    fH, fW, _C.ptr(t.geom), _C.ptr(t.starts), _C.ptr(col_begin), _C.ptr(seg_key), _C.ptr(seg_mask),
                    n_seg, _C.ptr(ddepth), _C.ptr(dctx), _C.ptr(ws), ws.numel(), _C.current_stream(dev))
                _C.check(rc, "bev_pool_lift_columns_backward")
            else:
                ws = _ws(L.bevb200_bev_pool_lift_backward_workspace_bytes(t.n_total, c), dev)
                rc = L.bevb200_bev_pool_lift_backward(
                    Bq, Dq, Hq, Wq, t.n_kept, t.n_total, c, t.n_intervals, _C.ptr(out_grad), _C.ptr(depth),
                    _C.ptr(ctx), D, fH * fW, _C.ptr(t.perm), _C.ptr(t.geom), _C.ptr(t.starts), _C.ptr(t.lengths),
                    _C.ptr(ddepth), _C.ptr(dctx), _C.ptr(ws), ws.numel(), _C.current_stream(dev))
                _C.check(rc, "bev_pool_lift_backward")
        return ddepth, dctx

    def lift(self, depth, ctx, out=None):
        """lift_pool + the module output layout of __call__: depth [B, N, D, fH, fW], ctx [B, N, fH, fW, C]
        -> [B, C*nz, nx, ny] (optionally written into `out`, e.g. the fuser's camera channels)."""
        return self._channels_first(self.lift_pool(depth, ctx), out)

    def __call__(self, x, out=None):
        """pool + module output layout.  `out` (optional) is a [B, Z*C, X, Y] float32 view that is
        dense inside each batch item -- e.g. the camera channels of the fuser's concatenated
        input (fusers/conv.py:16) -- and is written in place."""
        return self._channels_first(self.pool(x), out)

    @staticmethod
    def _channels_first(pooled, out=None):
        # pooled [B, Z, X, Y, C]; bev_pool.py:97 permute(0,4,1,2,3).contiguous() followed by base.py:174
        # cat(unbind(dim=2), 1) puts channel z*C + c at [b, :, x, y]: one tiled transpose does both
        B, Z, X, Y, C = pooled.shape
        if pooled.requires_grad:
            res = pooled.permute(0, 1, 4, 2, 3).contiguous().view(B, Z * C, X, Y)
            return res if out is None else out.copy_(res)
        from .spconv.ops import _batch_stride_of
        with torch.cuda.device(pooled.device):
            if out is None:
                out = torch.empty((B, Z * C, X, Y), dtype=pooled.dtype, device=pooled.device)
            stride = _batch_stride_of(out, (B, Z * C, X, Y))
            rc = _C.lib().bevb200_bev_channels_first(_C.ptr(pooled), _C.ptr(out), B, Z, X * Y, C, stride,
                                                     _C.current_stream(pooled.device))
        _C.check(rc, "bev_channels_first")
        return out
