"""radar_encoder -- mirror of mmdet3d/models/backbones/radar_encoder.py (camera+radar config).

    RFNLayer(in_channels, out_channels, norm_cfg=None, last_layer=False)
    RadarFeatureNet(in_channels, feat_channels, with_distance, voxel_size, point_cloud_range, norm_cfg)
    RadarEncoder(pts_voxel_encoder, pts_middle_encoder, ...)   (config dicts with `type`; the scatter is
                                                                PointPillarsScatter)

Same constructor arguments, sub-module names and state_dict keys as the reference.  In eval mode without
autograd, fp32, a native shape (1..4 layers, widths multiples of 16 up to 128, F + 2 <= 128, P <= 32)
runs the native radar kernel (csrc/radar.cu); training and other shapes run a torch restatement of the
reference forward.  RadarEncoder.forward_points fuses voxelization, the radar net and the scatter per
sample.  GPU only: CPU tensors raise.

Two deliberate differences from the reference, on both paths:
  - the caller's `features` tensor is never modified (the reference normalises its xyz in place);
  - `torch.backends.cudnn.enabled` is never touched (the reference sets it to False and back to True
    around every BN call, which also re-enables cuDNN for a caller that had disabled it).
`with_distance` is stored and, as in the reference, read by nothing."""
import ctypes

import torch
from torch import nn
from torch.nn import functional as F

from . import _C
from .pillar_encoder import PointPillarsScatter, get_paddings_indicator
from .sparse_block import bn_fold_key, bn_scale_shift, build_norm_layer
from .voxelize import Voxelization, _floats

__all__ = ["RFNLayer", "RadarFeatureNet", "RadarEncoder"]


class RFNLayer(nn.Module):
    """linear (no bias) -> BN1d over all slots -> ReLU on every slot; the last layer also takes the
    slot max (radar_encoder.py:47-82)."""

    def __init__(self, in_channels, out_channels, norm_cfg=None, last_layer=False):
        super().__init__()
        self.name = "RFNLayer"
        self.last_vfe = last_layer
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
        if self.last_vfe:
            return torch.max(x, dim=1, keepdim=True)[0]
        return x


class RadarFeatureNet(nn.Module):
    """Radar pillar decoration + RFN layers (radar_encoder.py:85-184).  forward(features [M, P, F],
    num_voxels [M], coors [M, 4] (b, x, y, z)) -> [M, C]."""

    def __init__(self, in_channels=4, feat_channels=(64,), with_distance=False, voxel_size=(0.2, 0.2, 4),
                 point_cloud_range=(0, -40, -3, 70.4, 40, 1), norm_cfg=None):
        super().__init__()
        self.name = "RadarFeatureNet"
        assert len(feat_channels) > 0
        self.in_channels = in_channels
        in_channels += 2
        self._with_distance = with_distance
        self.export_onnx = False
        feat_channels = [in_channels] + list(feat_channels)
        rfn_layers = []
        for i in range(len(feat_channels) - 1):
            rfn_layers.append(RFNLayer(feat_channels[i], feat_channels[i + 1], norm_cfg=norm_cfg,
                                       last_layer=i >= len(feat_channels) - 2))
        self.rfn_layers = nn.ModuleList(rfn_layers)
        self.vx = voxel_size[0]
        self.vy = voxel_size[1]
        self.x_offset = self.vx / 2 + point_cloud_range[0]
        self.y_offset = self.vy / 2 + point_cloud_range[1]
        self.pc_range = point_cloud_range
        self._packed_cache = None

    def _widths(self):
        w = [l.units for l in self.rfn_layers]
        return (ctypes.c_int * len(w))(*w)

    def native_supported(self, max_points):
        """True when the native kernel computes this net: eval-mode BN1d with running statistics,
        1..4 layers of widths that are multiples of 16 up to 128, F + 2 <= 128 and P <= 32."""
        layers = list(self.rfn_layers)
        return (1 <= max_points <= 32
                and _C.lib().bevb200_radar_packed_bytes(self.in_channels, len(layers), self._widths()) > 0
                and all(isinstance(l.norm, nn.BatchNorm1d) and l.norm.track_running_stats
                        and l.norm.running_mean is not None for l in layers))

    def _use_native(self, features):
        return (not self.training and not torch.is_grad_enabled() and features.dtype == torch.float32
                and features.dim() == 3 and features.shape[2] == self.in_channels
                and self.native_supported(features.shape[1]))

    def packed_weights(self):
        """Native weight image (bf16 hi | lo fragments, folded BN, the virtual row), rebuilt only when
        a parameter or statistic changes."""
        key = ()
        for l in self.rfn_layers:
            key += ((l.linear.weight.data_ptr(), l.linear.weight._version),) + bn_fold_key(l.norm)
        if self._packed_cache is not None and self._packed_cache[0] == key:
            return self._packed_cache[1]
        w0 = self.rfn_layers[0].linear.weight
        dev = w0.device
        _C.require_cuda(w0, "rfn_layers.0.linear.weight", torch.float32)
        ws = [l.linear.weight.detach().contiguous() for l in self.rfn_layers]
        folds = [bn_scale_shift(l.norm) for l in self.rfn_layers]
        L = len(ws)
        arr = lambda ts: (ctypes.c_void_p * L)(*[_C.ptr(t) for t in ts])
        with torch.cuda.device(dev):
            nbytes = _C.lib().bevb200_radar_packed_bytes(self.in_channels, L, self._widths())
            packed = torch.empty(nbytes // 4, dtype=torch.float32, device=dev)
            rc = _C.lib().bevb200_radar_pack_weights(
                ctypes.cast(arr(ws), ctypes.c_void_p), ctypes.cast(arr([s for s, _ in folds]), ctypes.c_void_p),
                ctypes.cast(arr([t for _, t in folds]), ctypes.c_void_p), self.in_channels, L, self._widths(),
                _C.ptr(packed), _C.current_stream(dev))
        _C.check(rc, "radar_pack_weights")
        self._packed_cache = (key, packed)
        return packed

    def _geometry(self):
        """(vx, vy, x_off, y_off), then host float[3] pc_min and pc_span (pc_max - pc_min in double)."""
        r = [float(v) for v in self.pc_range]
        lo = _C.host_array(ctypes.c_float, r[:3])
        span = _C.host_array(ctypes.c_float, [r[3] - r[0], r[4] - r[1], r[5] - r[2]])
        return (float(self.vx), float(self.vy), float(self.x_offset), float(self.y_offset),
                ctypes.cast(lo, ctypes.c_void_p), ctypes.cast(span, ctypes.c_void_p)), (lo, span)

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
        geom, _keep = self._geometry()
        dev = features.device
        L = len(self.rfn_layers)
        with torch.cuda.device(dev):
            out = torch.empty((m, self.rfn_layers[-1].units), dtype=torch.float32, device=dev)
            nbytes = _C.lib().bevb200_radar_features_workspace_bytes(m, p)
            ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)
            rc = _C.lib().bevb200_radar_features(_C.ptr(features), _C.ptr(num), _C.ptr(coors), m, None, p, f, L,
                                                 self._widths(), *geom, _C.ptr(packed), _C.ptr(out), _C.ptr(ws),
                                                 ws.numel(), _C.current_stream(dev))
        _C.check(rc, "radar_features")
        return out

    def _forward_torch(self, features, num_voxels, coors):
        dtype = features.dtype
        f_center = torch.zeros_like(features[:, :, :2])
        f_center[:, :, 0] = features[:, :, 0] - (coors[:, 1].to(dtype).unsqueeze(1) * self.vx + self.x_offset)
        f_center[:, :, 1] = features[:, :, 1] - (coors[:, 2].to(dtype).unsqueeze(1) * self.vy + self.y_offset)
        # the reference normalises xyz in the caller's tensor; this works on a copy (its points_mean /
        # f_cluster are never used and are not computed)
        r = self.pc_range
        xyz = torch.cat([(features[:, :, 0:1] - r[0]) / (r[3] - r[0]),
                         (features[:, :, 1:2] - r[1]) / (r[4] - r[1]),
                         (features[:, :, 2:3] - r[2]) / (r[5] - r[2])], dim=-1)
        features = torch.cat([xyz, features[:, :, 3:], f_center], dim=-1)
        mask = get_paddings_indicator(num_voxels, features.shape[1], axis=0)
        features = torch.nan_to_num(features * torch.unsqueeze(mask, -1).type_as(features))
        for rfn in self.rfn_layers:
            features = rfn(features)
        # the reference squeezes every unit dimension; only the slot one is meant
        return features.squeeze(1)


_BACKBONES = {"RadarFeatureNet": RadarFeatureNet, "PointPillarsScatter": PointPillarsScatter}


def _build(cfg):
    cfg = dict(cfg)
    kind = cfg.pop("type")
    if kind not in _BACKBONES:
        raise KeyError("unknown radar backbone type %r" % kind)
    return _BACKBONES[kind](**cfg)


class RadarEncoder(nn.Module):
    """RadarFeatureNet + PointPillarsScatter (radar_encoder.py:187-220).  pts_transformer_encoder,
    post_scatter and pts_bev_encoder are accepted for config compatibility; no shipped config sets them
    and a non-None value raises NotImplementedError."""

    def __init__(self, pts_voxel_encoder, pts_middle_encoder, pts_transformer_encoder=None, pts_bev_encoder=None,
                 post_scatter=None, **kwargs):
        super().__init__()
        for name, cfg in (("pts_transformer_encoder", pts_transformer_encoder),
                          ("pts_bev_encoder", pts_bev_encoder), ("post_scatter", post_scatter)):
            if cfg is not None:
                raise NotImplementedError("RadarEncoder: %s is not implemented" % name)
        self.pts_voxel_encoder = _build(pts_voxel_encoder)
        self.pts_middle_encoder = _build(pts_middle_encoder)
        self.pts_transformer_encoder = None
        self.pts_bev_encoder = None
        self.post_scatter = None

    def forward(self, feats, coords, batch_size, sizes, img_features=None):
        x = self.pts_voxel_encoder(feats, sizes, coords)
        return self.pts_middle_encoder(x, coords, batch_size)

    def forward_points(self, points_list, voxelize, return_voxel_num=False, num_points=None):
        """Voxelize (hard, `voxelize` = Voxelization) -> radar net -> scatter for each sample of
        `points_list` ([N_k, F] fp32 CUDA tensors), straight into one zeroed [B, C, nx, ny] canvas.
        Same result as voxelize_batch(voxelize_reduce=False) -> forward(), bit for bit, without the
        [M, P, F] voxel tensor and without a host synchronisation (CUDA-graph capturable).  Eval mode
        and no autograd only; the voxel grid must be (nx, ny, 1).  return_voxel_num: also return the
        device int32 [B] pillar counts.

        num_points (device int32 [B]): points_list is one padded [B, cap, F] tensor (RadarSweepStore.assemble with
        sync=False) and sample k is its first num_points[k] rows, read on the device only; the result equals the
        call on [points[k, :num_points[k]] for k in range(B)]."""
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
            raise ValueError("forward_points needs a native radar net shape (1..4 layers of widths that are "
                             "multiples of 16 up to 128, F + 2 <= 128, P <= 32)")
        if num_points is not None:
            _C.require_cuda(points_list, "points", torch.float32)
            _C.require_cuda(num_points, "num_points", torch.int32)
            if points_list.dim() != 3 or points_list.shape[2] != enc.in_channels:
                raise ValueError("points must be [B, cap, %d] with num_points" % enc.in_channels)
            if num_points.shape != (points_list.shape[0],) or num_points.device != points_list.device:
                raise ValueError("num_points must be int32 [B] on the points' device")
        else:
            for k, pts in enumerate(points_list):
                _C.require_cuda(pts, "points[%d]" % k, torch.float32)
                if pts.dim() != 2 or pts.shape[1] != enc.in_channels:
                    raise ValueError("points[%d] must be [N, %d]" % (k, enc.in_channels))
        dev = points_list[0].device
        B, C, L = len(points_list), enc.rfn_layers[-1].units, len(enc.rfn_layers)
        packed = enc.packed_weights()
        geom, _keep = enc._geometry()
        vs, cr = _floats(voxelize.voxel_size, 3), _floats(voxelize.point_cloud_range, 6)
        mv = int(voxelize.max_voxels[1])
        with torch.cuda.device(dev):
            canvas = torch.zeros((B, C, scat.nx, scat.ny), dtype=torch.float32, device=dev)
            voxel_num = torch.zeros(B, dtype=torch.int32, device=dev)
            nmax = max(int(p.shape[0]) for p in points_list)
            nbytes = _C.lib().bevb200_hard_voxelize_radar_workspace_bytes(nmax, P)
            ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)
            for k, pts in enumerate(points_list):
                args = (enc.in_channels, ctypes.cast(vs, ctypes.c_void_p), ctypes.cast(cr, ctypes.c_void_p), P, mv, L,
                        enc._widths(), *geom, _C.ptr(packed), _C.ptr(canvas[k]), int(scat.nx), int(scat.ny),
                        _C.ptr(voxel_num[k:k + 1]), _C.ptr(ws), ws.numel(), _C.current_stream(dev))
                if num_points is None:
                    rc = _C.lib().bevb200_hard_voxelize_radar(_C.ptr(pts), int(pts.shape[0]), *args)
                else:
                    rc = _C.lib().bevb200_hard_voxelize_radar_dev(_C.ptr(pts), _C.ptr(num_points[k:k + 1]),
                                                                  int(pts.shape[0]), *args)
                _C.check(rc, "hard_voxelize_radar")
        return (canvas, voxel_num) if return_voxel_num else canvas
