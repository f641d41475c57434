"""voxelize -- host-side mirror of mmdet3d/ops/voxel (voxelize.py:1-148, voxelization.h:58-95).

    voxel_layer.hard_voxelize(points, voxels, coors, num_points_per_voxel, voxel_size,
                              coors_range, max_points, max_voxels, NDim=3, deterministic=True) -> int
    voxel_layer.dynamic_voxelize(points, coors, voxel_size, coors_range, NDim=3)
    voxelization(points, voxel_size, coors_range, max_points, max_voxels, deterministic)
    Voxelization(voxel_size, point_cloud_range, max_num_points, max_voxels, deterministic)

GPU only (north star: no CPU fallback): CPU tensors raise."""
import ctypes

import torch
from torch import nn
from torch.autograd import Function
from torch.nn.modules.utils import _pair

from . import _C

__all__ = ["voxel_layer", "voxelization", "Voxelization", "voxelize_mean", "voxelize_mean_fused",
           "voxelize_batch"]


def _floats(vals, n):
    vals = [float(v) for v in vals]
    if len(vals) != n:
        raise ValueError("expected %d values, got %d" % (n, len(vals)))
    return _C.host_array(ctypes.c_float, vals)

_REDUCE = {"sum": 0, "mean": 1, "max": 2}      # voxelization.h:12-22 convert_reduce_type


def _reduce_code(reduce_type):
    if reduce_type not in _REDUCE:
        raise ValueError("do not support reduce type " + str(reduce_type))
    return _REDUCE[reduce_type]


def _dynamic_scatter_forward(feats, coors, reduce_type):
    code = _reduce_code(reduce_type)
    _C.require_cuda(feats, "feats", torch.float32)
    _C.require_cuda(coors, "coors", torch.int32)
    n, c = feats.shape
    ndim = coors.shape[1]
    if coors.shape[0] != n:
        raise ValueError("feats and coors must have the same number of rows")
    dev = feats.device
    if n == 0:                                   # scatter_points_cuda.cu:196-200
        return (feats.clone().detach(), coors.clone().detach(),
                coors.new_empty((0,), dtype=torch.int32), coors.new_empty((0,), dtype=torch.int32), None)
    with torch.cuda.device(dev):
        reduced = torch.empty((n, c), dtype=torch.float32, device=dev)
        out_coors = torch.empty((n, ndim), dtype=torch.int32, device=dev)
        coors_map = torch.empty((n,), dtype=torch.int32, device=dev)
        count = torch.empty((n,), dtype=torch.int32, device=dev)
        reduce_from = torch.empty((n, c), dtype=torch.int32, device=dev) if code == 2 else None
        meta = torch.empty((2,), dtype=torch.int32, device=dev)
        nbytes = _C.lib().bevb200_dynamic_scatter_workspace_bytes(n)
        ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)
        rc = _C.lib().bevb200_dynamic_scatter(
            _C.ptr(feats), _C.ptr(coors), n, c, ndim, code, _C.ptr(reduced), _C.ptr(out_coors),
            _C.ptr(coors_map), _C.ptr(count), _C.ptr(reduce_from), _C.ptr(meta), _C.ptr(ws), ws.numel(),
            _C.current_stream(dev))
    _C.check(rc, "dynamic_scatter")
    m, too_big = (int(v) for v in meta.tolist())
    if too_big:
        raise ValueError("%d coordinate rows exceed the key range (2^20 per column, 2^15 with 4 columns)"
                         % too_big)
    return (reduced[:m], out_coors[:m], coors_map, count[:m],
            reduce_from[:m] if reduce_from is not None else None)


def _dynamic_scatter_backward(grad_feats, grad_reduced, feats, reduced, coors_map, count, reduce_type,
                              reduce_from):
    code = _reduce_code(reduce_type)
    _C.require_cuda(grad_feats, "grad_feats", torch.float32)
    _C.require_cuda(grad_reduced, "grad_reduced_feats", torch.float32)
    n, c = grad_feats.shape
    m = grad_reduced.shape[0]
    dev = grad_feats.device
    with torch.cuda.device(dev):
        valid = reduce_from is not None
        if code == 2 and not valid:
            _C.require_cuda(feats, "feats", torch.float32)
            _C.require_cuda(reduced, "reduced_feats", torch.float32)
            reduce_from = torch.empty((max(m, 1), c), dtype=torch.int32, device=dev)
        rc = _C.lib().bevb200_dynamic_scatter_backward(
            _C.ptr(grad_reduced), _C.ptr(feats), _C.ptr(reduced), _C.ptr(coors_map), _C.ptr(count),
            _C.ptr(reduce_from), int(valid), n, m, c, code, _C.ptr(grad_feats), _C.current_stream(dev))
    _C.check(rc, "dynamic_scatter_backward")


class _VoxelLayer:
    """Stand-in for the reference pybind module `voxel_layer` (voxelization.cpp:7-12)."""

    @staticmethod
    def hard_voxelize(points, voxels, coors, num_points_per_voxel, voxel_size, coors_range,
                      max_points, max_voxels, NDim=3, deterministic=True):
        # `deterministic` is accepted for API parity; this implementation is always
        # deterministic (and does not need the O(N^2) scan that made the flag necessary).
        if NDim != 3:
            raise NotImplementedError("only NDim == 3 is supported")
        _C.require_cuda(points, "points", torch.float32)
        _C.require_cuda(voxels, "voxels", torch.float32)
        _C.require_cuda(coors, "coors", torch.int32)
        _C.require_cuda(num_points_per_voxel, "num_points_per_voxel", torch.int32)
        n, f = points.shape
        if voxels.shape[0] < max_voxels or voxels.shape[1] != max_points or voxels.shape[2] != f:
            raise ValueError("voxels must be [>=max_voxels, max_points, num_features]")
        vs, cr = _floats(voxel_size, 3), _floats(coors_range, 6)
        with torch.cuda.device(points.device):
            voxel_num = torch.zeros(1, dtype=torch.int32, device=points.device)
            nbytes = _C.lib().bevb200_hard_voxelize_workspace_bytes(n, int(max_points))
            ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=points.device)
            rc = _C.lib().bevb200_hard_voxelize(
                _C.ptr(points), n, f, ctypes.cast(vs, ctypes.c_void_p),
                ctypes.cast(cr, ctypes.c_void_p), int(max_points), int(max_voxels),
                _C.ptr(voxels), _C.ptr(coors), _C.ptr(num_points_per_voxel), _C.ptr(voxel_num),
                _C.ptr(ws), ws.numel(), _C.current_stream(points.device))
        _C.check(rc, "hard_voxelize")
        return int(voxel_num.item())  # host int, like voxelization_cuda.cu:369-372

    @staticmethod
    def dynamic_voxelize(points, coors, voxel_size, coors_range, NDim=3):
        if NDim != 3:
            raise NotImplementedError("only NDim == 3 is supported")
        _C.require_cuda(points, "points", torch.float32)
        _C.require_cuda(coors, "coors", torch.int32)
        n, f = points.shape
        vs, cr = _floats(voxel_size, 3), _floats(coors_range, 6)
        with torch.cuda.device(points.device):
            rc = _C.lib().bevb200_dynamic_voxelize(
                _C.ptr(points), n, f, ctypes.cast(vs, ctypes.c_void_p),
                ctypes.cast(cr, ctypes.c_void_p), _C.ptr(coors), _C.current_stream(points.device))
        _C.check(rc, "dynamic_voxelize")

    @staticmethod
    def dynamic_point_to_voxel_forward(feats, coors, reduce_type="max"):
        """voxelization.h:97-109 / scatter_points_cuda.cu:187-241.  Returns
        [reduced_feats [M, C], out_coors [M, ndim], coors_map [N] int32, reduce_count [M] int32];
        voxels are the unique coordinate rows in lexicographic order, rows with a negative
        entry are dropped (coors_map -1).

        NaN features: sum and mean propagate them.  max ignores them, as the reference's fmaxf
        reduction does (:22-30): a voxel's maximum is taken over its non-NaN values, a voxel
        holding only NaN yields -inf, and the backward pass gives a NaN element no gradient
        (NaN never equals the maximum, :162)."""
        out = _dynamic_scatter_forward(feats, coors, reduce_type)
        return [out[0], out[1], out[2], out[3]]

    @staticmethod
    def dynamic_point_to_voxel_backward(grad_feats, grad_reduced_feats, feats, reduced_feats,
                                        coors_map, reduce_count, reduce_type="max"):
        """voxelization.h:111-127 / scatter_points_cuda.cu:243-315: fills grad_feats in place."""
        _dynamic_scatter_backward(grad_feats, grad_reduced_feats, feats, reduced_feats, coors_map,
                                  reduce_count, reduce_type, None)


voxel_layer = _VoxelLayer()
hard_voxelize = voxel_layer.hard_voxelize
dynamic_voxelize = voxel_layer.dynamic_voxelize


class _Voxelization(Function):
    """Same contract as the reference Function (voxelize.py:10-71)."""

    @staticmethod
    def forward(ctx, points, voxel_size, coors_range, max_points=35, max_voxels=20000,
                deterministic=True):
        points = points.contiguous()
        if max_points == -1 or max_voxels == -1:
            coors = points.new_zeros(size=(points.size(0), 3), dtype=torch.int)
            dynamic_voxelize(points, coors, voxel_size, coors_range, 3)
            return coors
        voxels = points.new_zeros(size=(max_voxels, max_points, points.size(1)))
        coors = points.new_zeros(size=(max_voxels, 3), dtype=torch.int)
        num_points_per_voxel = points.new_zeros(size=(max_voxels,), dtype=torch.int)
        voxel_num = hard_voxelize(points, voxels, coors, num_points_per_voxel, voxel_size,
                                  coors_range, max_points, max_voxels, 3, deterministic)
        return voxels[:voxel_num], coors[:voxel_num], num_points_per_voxel[:voxel_num]


voxelization = _Voxelization.apply


class Voxelization(nn.Module):
    """Same constructor and forward as mmdet3d.ops.Voxelization (voxelize.py:77-148)."""

    def __init__(self, voxel_size, point_cloud_range, max_num_points, max_voxels=20000,
                 deterministic=True):
        super().__init__()
        self.voxel_size = voxel_size
        self.point_cloud_range = point_cloud_range
        self.max_num_points = max_num_points
        self.max_voxels = max_voxels if isinstance(max_voxels, tuple) else _pair(max_voxels)
        self.deterministic = deterministic
        pcr = torch.tensor(point_cloud_range, dtype=torch.float32)
        vs = torch.tensor(voxel_size, dtype=torch.float32)
        grid_size = torch.round((pcr[3:] - pcr[:3]) / vs).long()
        self.grid_size = grid_size
        self.pcd_shape = [*grid_size[:2], 1]

    def forward(self, input):
        max_voxels = self.max_voxels[0] if self.training else self.max_voxels[1]
        return voxelization(input, self.voxel_size, self.point_cloud_range, self.max_num_points,
                            max_voxels, self.deterministic)

    def __repr__(self):
        return (self.__class__.__name__ + "(voxel_size=" + str(self.voxel_size)
                + ", point_cloud_range=" + str(self.point_cloud_range) + ", max_num_points="
                + str(self.max_num_points) + ", max_voxels=" + str(self.max_voxels)
                + ", deterministic=" + str(self.deterministic) + ")")


def voxelize_mean(voxels, coors, num_points, batch_idx=0):
    """Fused glue of BEVFusion.voxelize (bevfusion.py:183,191-195): mean over the points of a
    voxel and (batch, x, y, z) coords.  Returns (feats [M, F] fp32, coords [M, 4] int32)."""
    _C.require_cuda(voxels, "voxels", torch.float32)
    _C.require_cuda(coors, "coors", torch.int32)
    _C.require_cuda(num_points, "num_points", torch.int32)
    m, p, f = voxels.shape
    with torch.cuda.device(voxels.device):
        feats = torch.empty((m, f), dtype=torch.float32, device=voxels.device)
        coords4 = torch.empty((m, 4), dtype=torch.int32, device=voxels.device)
        rc = _C.lib().bevb200_voxel_mean(_C.ptr(voxels), _C.ptr(coors), _C.ptr(num_points), m, p, f,
                                         int(batch_idx), _C.ptr(feats), _C.ptr(coords4),
                                         _C.current_stream(voxels.device))
    _C.check(rc, "voxel_mean")
    return feats, coords4


def voxelize_mean_fused(points, voxel_size, coors_range, max_points, max_voxels, batch_idx=0, sync=True):
    """hard voxelization + per-voxel mean + (batch, x, y, z) coords in one pass over the points
    (bevfusion.py:178-195 with voxelize_reduce), never materialising the [M, max_points, F]
    voxel tensor.  Returns (feats [M, F], coords [M, 4] int32, num_points [M] int32).

    sync=False keeps the voxel count on the device (the reference returns it as a host int,
    voxelization_cuda.cu:369-370): the tensors come back at their cap size [max_voxels, ...] together
    with `voxel_num` (device int32[1]); rows >= voxel_num are unspecified.  SparseEncoder takes that
    count as `num_voxels=`, so a whole LiDAR frame needs no host round trip."""
    _C.require_cuda(points, "points", torch.float32)
    n, f = points.shape
    vs, cr = _floats(voxel_size, 3), _floats(coors_range, 6)
    dev = points.device
    with torch.cuda.device(dev):
        feats = torch.empty((max_voxels, f), dtype=torch.float32, device=dev)
        coords4 = torch.empty((max_voxels, 4), dtype=torch.int32, device=dev)
        num = torch.empty((max_voxels,), dtype=torch.int32, device=dev)
        voxel_num = torch.zeros(1, dtype=torch.int32, device=dev)
        nbytes = _C.lib().bevb200_hard_voxelize_workspace_bytes(n, int(max_points))
        ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)
        rc = _C.lib().bevb200_hard_voxelize_mean(
            _C.ptr(points), n, f, ctypes.cast(vs, ctypes.c_void_p), ctypes.cast(cr, ctypes.c_void_p),
            int(max_points), int(max_voxels), int(batch_idx), _C.ptr(feats), _C.ptr(coords4),
            _C.ptr(num), _C.ptr(voxel_num), _C.ptr(ws), ws.numel(), _C.current_stream(dev))
    _C.check(rc, "hard_voxelize_mean")
    if not sync:
        return feats, coords4, num, voxel_num
    m = int(voxel_num.item())
    return feats[:m], coords4[:m], num[:m]


@torch.no_grad()
def voxelize_batch(points, voxelize_module, voxelize_reduce=True):
    """BEVFusion.voxelize (mmdet3d/models/fusion_models/bevfusion.py:169-197): per-sample hard
    voxelization, batch index prepended to the coords (F.pad(c, (1, 0), value=k)), concatenation,
    and -- with voxelize_reduce -- the mean over the points of each voxel.

    points: list of [N_k, F] CUDA tensors.  Returns (feats, coords [M, 4] int32 (b, x, y, z), sizes)."""
    feats, coords, sizes = [], [], []
    hard = isinstance(voxelize_module, Voxelization) and voxelize_module.max_num_points > 0
    for k, res in enumerate(points):
        if hard and voxelize_reduce and res.shape[1] <= 8:   # fused: no [M, P, F] intermediate (kernel: F <= 8;
            # wider rows, e.g. 45-dim radar points, take the generic Voxelization + mean below)
            mv = voxelize_module.max_voxels[0 if voxelize_module.training else 1]
            f, c4, n = voxelize_mean_fused(res.contiguous(), voxelize_module.voxel_size,
                                           voxelize_module.point_cloud_range,
                                           voxelize_module.max_num_points, mv, k)
            feats.append(f); coords.append(c4); sizes.append(n)
            continue
        ret = voxelize_module(res)
        if isinstance(ret, tuple):     # not len(ret) == 3: dynamic coords of a 3-point sample are [3, 3]
            f, c, n = ret
            if voxelize_reduce:
                f, c4 = voxelize_mean(f.contiguous(), c.contiguous(), n.contiguous(), k)
            else:
                c4 = torch.nn.functional.pad(c, (1, 0), mode="constant", value=k)
            sizes.append(n)
        else:                      # dynamic voxelization: coords only
            f, c = res, ret
            c4 = torch.nn.functional.pad(c, (1, 0), mode="constant", value=k)
        feats.append(f)
        coords.append(c4)
    feats = torch.cat(feats, dim=0)
    coords = torch.cat(coords, dim=0)
    sizes = torch.cat(sizes, dim=0) if sizes else sizes
    return feats, coords, sizes
