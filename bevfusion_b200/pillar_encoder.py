"""pillar_encoder -- mirror of mmdet3d/models/backbones/pillar_encoder.py (PointPillars).

    PFNLayer(in_channels, out_channels, norm_cfg=None, last_layer=False)
    PillarFeatureNet(in_channels, feat_channels, with_distance, voxel_size, point_cloud_range, norm_cfg)
    PointPillarsScatter(in_channels, output_shape)
    PointPillarsEncoder(pts_voxel_encoder, pts_middle_encoder)      (config dicts with `type`)

Same constructor arguments, sub-module names and state_dict keys as the reference.  In eval mode
without autograd, fp32, the shipped shape (feat_channels [64, 64], with_distance False, F <= 8,
P <= 32) runs the native pillar kernel (csrc/pillars.cu); training and other shapes run a torch
restatement of the reference forward.  PointPillarsEncoder.forward_points fuses voxelization, the
pillar net and the scatter per sample.  GPU only: CPU tensors raise."""
import ctypes

import torch
from torch import nn
from torch.autograd import Function
from torch.nn import functional as F

from . import _C
from .sparse_block import bn_fold_key, bn_scale_shift, build_norm_layer
from .spconv.ops import sparse_to_dense
from .voxelize import Voxelization, _floats

__all__ = ["PFNLayer", "PillarFeatureNet", "PointPillarsScatter", "PointPillarsEncoder"]


def get_paddings_indicator(actual_num, max_num, axis=0):
    """mask[v, s] = s < actual_num[v]  (pillar_encoder.py:20-40)"""
    actual_num = torch.unsqueeze(actual_num, axis + 1)
    max_num_shape = [1] * len(actual_num.shape)
    max_num_shape[axis + 1] = -1
    max_num = torch.arange(max_num, dtype=torch.int, device=actual_num.device).view(max_num_shape)
    return actual_num.int() > max_num


class PFNLayer(nn.Module):
    """linear (no bias) -> BN1d over all slots -> ReLU -> max over slots, concatenated back onto every
    slot unless last_layer (pillar_encoder.py:43-88)."""

    def __init__(self, in_channels, out_channels, norm_cfg=None, last_layer=False):
        super().__init__()
        self.name = "PFNLayer"
        self.last_vfe = last_layer
        if not self.last_vfe:
            out_channels = out_channels // 2
        self.units = out_channels
        if norm_cfg is None:
            norm_cfg = dict(type="BN1d", eps=1e-3, momentum=0.01)
        self.norm_cfg = norm_cfg
        self.linear = nn.Linear(in_channels, self.units, bias=False)
        self.norm = build_norm_layer(self.norm_cfg, self.units)[1]

    def forward(self, inputs):
        x = self.linear(inputs)
        x = self.norm(x.permute(0, 2, 1).contiguous()).permute(0, 2, 1).contiguous()
        x = F.relu(x)
        x_max = torch.max(x, dim=1, keepdim=True)[0]
        if self.last_vfe:
            return x_max
        return torch.cat([x, x_max.repeat(1, inputs.shape[1], 1)], dim=2)


class PillarFeatureNet(nn.Module):
    """Pillar decoration + PFN layers (pillar_encoder.py:91-176).  forward(features [M, P, F],
    num_voxels [M], coors [M, 4] (b, x, y, z)) -> [M, C]."""

    def __init__(self, in_channels=4, feat_channels=(64,), with_distance=False, voxel_size=(0.2, 0.2, 4),
                 point_cloud_range=(0, -40, -3, 70.4, 40, 1), norm_cfg=None):
        super().__init__()
        self.name = "PillarFeatureNet"
        assert len(feat_channels) > 0
        self.in_channels = in_channels
        in_channels += 5
        if with_distance:
            in_channels += 1
        self._with_distance = with_distance
        feat_channels = [in_channels] + list(feat_channels)
        pfn_layers = []
        for i in range(len(feat_channels) - 1):
            pfn_layers.append(PFNLayer(feat_channels[i], feat_channels[i + 1], norm_cfg=norm_cfg,
                                       last_layer=i >= len(feat_channels) - 2))
        self.pfn_layers = nn.ModuleList(pfn_layers)
        self.vx = voxel_size[0]
        self.vy = voxel_size[1]
        self.x_offset = self.vx / 2 + point_cloud_range[0]
        self.y_offset = self.vy / 2 + point_cloud_range[1]
        self._packed_cache = None

    def native_supported(self, max_points):
        """True when the native kernel computes this net: eval-mode BN1d with running statistics,
        two PFN layers of 32 and 64 units, no distance feature, F <= 8 and P <= 32."""
        layers = list(self.pfn_layers)
        return (len(layers) == 2 and not self._with_distance and 1 <= max_points <= 32
                and _C.lib().bevb200_pillar_packed_bytes(self.in_channels, layers[0].units, layers[1].units) > 0
                and all(isinstance(l.norm, nn.BatchNorm1d) and l.norm.track_running_stats
                        and l.norm.running_mean is not None for l in layers))

    def _use_native(self, features):
        return (not self.training and not torch.is_grad_enabled() and features.dtype == torch.float32
                and features.dim() == 3 and features.shape[2] == self.in_channels
                and self.native_supported(features.shape[1]))

    def packed_weights(self):
        """Native weight image (folded BN), rebuilt only when a parameter or statistic changes."""
        l1, l2 = self.pfn_layers
        key = tuple((w.data_ptr(), w._version) for w in (l1.linear.weight, l2.linear.weight))
        key += bn_fold_key(l1.norm) + bn_fold_key(l2.norm)
        if self._packed_cache is not None and self._packed_cache[0] == key:
            return self._packed_cache[1]
        dev = l1.linear.weight.device
        _C.require_cuda(l1.linear.weight, "pfn_layers.0.linear.weight", torch.float32)
        s1, t1 = bn_scale_shift(l1.norm)
        s2, t2 = bn_scale_shift(l2.norm)
        w1 = l1.linear.weight.detach().contiguous()
        w2 = l2.linear.weight.detach().contiguous()
        with torch.cuda.device(dev):
            nbytes = _C.lib().bevb200_pillar_packed_bytes(self.in_channels, l1.units, l2.units)
            packed = torch.empty(nbytes // 4, dtype=torch.float32, device=dev)
            rc = _C.lib().bevb200_pillar_pack_weights(_C.ptr(w1), _C.ptr(s1), _C.ptr(t1), _C.ptr(w2), _C.ptr(s2),
                                                      _C.ptr(t2), self.in_channels, l1.units, l2.units,
                                                      _C.ptr(packed), _C.current_stream(dev))
        _C.check(rc, "pillar_pack_weights")
        self._packed_cache = (key, packed)
        return packed

    def _geometry(self):
        return float(self.vx), float(self.vy), float(self.x_offset), float(self.y_offset)

    def forward(self, features, num_voxels, coors):
        _C.require_cuda(features, "features", contiguous=False)
        if self._use_native(features):
            return self._forward_native(features, num_voxels, coors)
        return self._forward_torch(features, num_voxels, coors)

    def _forward_native(self, features, num_voxels, coors):
        m, p, f = features.shape
        features = features.contiguous()
        num = _C.require_cuda(num_voxels.to(torch.int32).contiguous(), "num_voxels")
        coors = _C.require_cuda(coors.to(torch.int32).contiguous(), "coors")
        if coors.shape != (m, 4) or num.shape != (m,):
            raise ValueError("expected num_voxels [M] and coors [M, 4] for features [M, P, F]")
        packed = self.packed_weights()
        dev = features.device
        with torch.cuda.device(dev):
            out = torch.empty((m, self.pfn_layers[-1].units), dtype=torch.float32, device=dev)
            rc = _C.lib().bevb200_pillar_features(_C.ptr(features), _C.ptr(num), _C.ptr(coors), m, None, p, f,
                                                  *self._geometry(), _C.ptr(packed), _C.ptr(out),
                                                  _C.current_stream(dev))
        _C.check(rc, "pillar_features")
        return out

    def _forward_torch(self, features, num_voxels, coors):
        dtype = features.dtype
        points_mean = features[:, :, :3].sum(dim=1, keepdim=True) / num_voxels.type_as(features).view(-1, 1, 1)
        f_cluster = features[:, :, :3] - points_mean
        f_center = torch.zeros_like(features[:, :, :2])
        f_center[:, :, 0] = features[:, :, 0] - (coors[:, 1].to(dtype).unsqueeze(1) * self.vx + self.x_offset)
        f_center[:, :, 1] = features[:, :, 1] - (coors[:, 2].to(dtype).unsqueeze(1) * self.vy + self.y_offset)
        features_ls = [features, f_cluster, f_center]
        if self._with_distance:
            features_ls.append(torch.norm(features[:, :, :3], 2, 2, keepdim=True))
        features = torch.cat(features_ls, dim=-1)
        mask = get_paddings_indicator(num_voxels, features.shape[1], axis=0)
        features = features * torch.unsqueeze(mask, -1).type_as(features)
        for pfn in self.pfn_layers:
            features = pfn(features)
        # the reference squeezes every unit dimension; only the slot one is meant
        return features.squeeze(1)


class _Scatter(Function):
    """canvas[b, :, x, y] = feats[v] via the library's dense(); the gradient is the gather back."""

    @staticmethod
    def forward(ctx, feats, coords, batch_size, nx, ny):
        ctx.save_for_backward(coords)
        return sparse_to_dense(feats.contiguous(), coords, batch_size, (nx, ny, 1), z_major=True)

    @staticmethod
    def backward(ctx, grad):
        (coords,) = ctx.saved_tensors
        c = coords.long()
        return grad[c[:, 0], :, c[:, 1], c[:, 2]], None, None, None, None


class PointPillarsScatter(nn.Module):
    """Pillar rows -> channels-first BEV canvas [B, C, nx, ny] (pillar_encoder.py:179-237): indices
    x * ny + y, zeros elsewhere."""

    def __init__(self, in_channels=64, output_shape=(512, 512), **kwargs):
        super().__init__()
        self.in_channels = in_channels
        self.output_shape = output_shape
        self.nx = output_shape[0]
        self.ny = output_shape[1]

    def extra_repr(self):
        return f"in_channels={self.in_channels}, output_shape={tuple(self.output_shape)}"

    def forward(self, voxel_features, coords, batch_size):
        _C.require_cuda(voxel_features, "voxel_features", torch.float32, contiguous=False)
        coords = _C.require_cuda(coords.to(torch.int32).contiguous(), "coords")
        return _Scatter.apply(voxel_features, coords, int(batch_size), int(self.nx), int(self.ny))


_BACKBONES = {"PillarFeatureNet": PillarFeatureNet, "PointPillarsScatter": PointPillarsScatter}


def _build(cfg):
    cfg = dict(cfg)
    kind = cfg.pop("type")
    if kind not in _BACKBONES:
        raise KeyError("unknown pillar backbone type %r" % kind)
    return _BACKBONES[kind](**cfg)


class PointPillarsEncoder(nn.Module):
    """PillarFeatureNet + PointPillarsScatter (pillar_encoder.py:240-258)."""

    def __init__(self, pts_voxel_encoder, pts_middle_encoder, **kwargs):
        super().__init__()
        self.pts_voxel_encoder = _build(pts_voxel_encoder)
        self.pts_middle_encoder = _build(pts_middle_encoder)

    def forward(self, feats, coords, batch_size, sizes):
        x = self.pts_voxel_encoder(feats, sizes, coords)
        return self.pts_middle_encoder(x, coords, batch_size)

    def forward_points(self, points_list, voxelize):
        """Voxelize (hard, `voxelize` = Voxelization) -> pillar net -> scatter for each sample of
        `points_list` ([N_k, F] fp32 CUDA tensors), straight into one zeroed [B, C, nx, ny] canvas.
        Same result as voxelize_batch(voxelize_reduce=False) -> forward(), without the [M, P, F]
        voxel tensor and without a host synchronisation (CUDA-graph capturable).  Eval mode and no
        autograd only; the voxel grid must be (nx, ny, 1)."""
        enc, scat = self.pts_voxel_encoder, self.pts_middle_encoder
        if not isinstance(voxelize, Voxelization) or voxelize.max_num_points <= 0:
            raise ValueError("forward_points needs a hard Voxelization module")
        if self.training or enc.training or voxelize.training or torch.is_grad_enabled():
            raise RuntimeError("forward_points runs in eval mode under torch.no_grad() only")
        grid = [int(g) for g in voxelize.grid_size]
        if grid != [int(scat.nx), int(scat.ny), 1]:
            raise ValueError("voxel grid %s differs from the scatter output shape (%d, %d, 1)"
                             % (grid, scat.nx, scat.ny))
        P = int(voxelize.max_num_points)
        if not enc.native_supported(P):
            raise ValueError("forward_points needs the native pillar net shape (feat_channels [64, 64], "
                             "with_distance False, F <= 8, P <= 32)")
        for k, pts in enumerate(points_list):
            _C.require_cuda(pts, "points[%d]" % k, torch.float32)
            if pts.dim() != 2 or pts.shape[1] != enc.in_channels:
                raise ValueError("points[%d] must be [N, %d]" % (k, enc.in_channels))
        dev = points_list[0].device
        B, C = len(points_list), enc.pfn_layers[-1].units
        packed = enc.packed_weights()
        vs, cr = _floats(voxelize.voxel_size, 3), _floats(voxelize.point_cloud_range, 6)
        mv = int(voxelize.max_voxels[1])
        with torch.cuda.device(dev):
            canvas = torch.zeros((B, C, scat.nx, scat.ny), dtype=torch.float32, device=dev)
            voxel_num = torch.zeros(B, dtype=torch.int32, device=dev)
            nmax = max(int(p.shape[0]) for p in points_list)
            nbytes = _C.lib().bevb200_hard_voxelize_workspace_bytes(nmax, P)
            ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)
            for k, pts in enumerate(points_list):
                rc = _C.lib().bevb200_hard_voxelize_pillars(
                    _C.ptr(pts), int(pts.shape[0]), enc.in_channels, ctypes.cast(vs, ctypes.c_void_p),
                    ctypes.cast(cr, ctypes.c_void_p), P, mv, *enc._geometry(), _C.ptr(packed), _C.ptr(canvas[k]),
                    int(scat.nx), int(scat.ny), _C.ptr(voxel_num[k:k + 1]), _C.ptr(ws), ws.numel(),
                    _C.current_stream(dev))
                _C.check(rc, "hard_voxelize_pillars")
        return canvas
