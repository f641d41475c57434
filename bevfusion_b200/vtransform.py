"""View-transform geometry glue -- mirror of the parts of
mmdet3d/models/vtransforms/base.py that feed bev_pool: gen_dx_bx (:15-21), create_frustum
(:66-89), get_geometry (:92-135) and BaseTransform.bev_pool (:141-176).  Plain torch; the
pooling itself goes through bevfusion_b200.bev_pool."""
import torch
from torch import nn

from . import _C
from .bev_pool import BEVPoolPlan, bev_pool, gen_dx_bx

__all__ = ["gen_dx_bx", "create_frustum", "get_geometry", "LSSGeometry", "points_to_depth"]


def points_to_depth(points, lidar2image, img_aug_matrix, lidar_aug_matrix, image_size,
                    depth_input="scalar", depth_bins=None, add_depth_features=False,
                    height_expand=False):
    """The depth-image half of BaseDepthTransform.forward (base.py:266-329).

    points: list of B [N_b, F] CUDA fp32 tensors (NOT modified -- the reference shifts their xyz in
    place at :290); lidar2image / img_aug_matrix [B, ncam, 4, 4]; lidar_aug_matrix [B, 4, 4].
    Returns depth [B, ncam, channels, iH, iW] with channels = (1 | depth_bins) (+ F).  Colliding
    points: the largest point index wins (sequential index_put semantics)."""
    if depth_input not in ("scalar", "one-hot"):
        raise ValueError("depth_input must be 'scalar' or 'one-hot'")
    one_hot = depth_input == "one-hot"
    if one_hot and not depth_bins:
        raise ValueError("one-hot depth needs depth_bins (the frustum's D)")
    iH, iW = (int(v) for v in image_size)
    B = len(points)
    ncam = int(lidar2image.shape[1])
    if height_expand:                                    # base.py:266-270 (radar pillars)
        expanded = []
        for p in points:
            q = p.repeat_interleave(8, dim=0)
            q[:, 2] = torch.arange(0.25, 2.25, 0.25, device=p.device).repeat(p.shape[0])
            expanded.append(q)
        points = expanded
    for b, pts in enumerate(points):                    # no CPU fallback: fail before any allocation
        _C.require_cuda(pts, "points[%d]" % b, torch.float32)
    dev = points[0].device
    F = int(points[0].shape[1])
    if any(p.shape[1] != F for p in points):             # before any sample is rasterised
        raise ValueError("all samples must have the same number of point features")
    channels = (int(depth_bins) if one_hot else 1) + (F if add_depth_features else 0)
    l2i = lidar2image.to(device=dev, dtype=torch.float32).contiguous()
    ia = img_aug_matrix.to(device=dev, dtype=torch.float32).contiguous()
    la = lidar_aug_matrix.to(device=dev, dtype=torch.float32).contiguous()
    with torch.cuda.device(dev):
        depth = torch.empty((B, ncam, channels, iH, iW), dtype=torch.float32, device=dev)
        nbytes = _C.lib().bevb200_depth_rasterize_workspace_bytes(ncam, iH, iW)
        ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)
        for b in range(B):
            p = points[b]
            rc = _C.lib().bevb200_depth_rasterize(
                _C.ptr(p), int(p.shape[0]), F, _C.ptr(la[b]), _C.ptr(l2i[b]), _C.ptr(ia[b]), ncam, iH, iW,
                int(one_hot), int(depth_bins or 0), int(bool(add_depth_features)), _C.ptr(depth[b]),
                _C.ptr(ws), ws.numel(), _C.current_stream(dev))
            _C.check(rc, "depth_rasterize")
    return depth


def create_frustum(image_size, feature_size, dbound):
    """base.py:66-89 -> [D, fH, fW, 3] = (u, v, d)."""
    iH, iW = image_size
    fH, fW = feature_size
    ds = torch.arange(*dbound, dtype=torch.float).view(-1, 1, 1).expand(-1, fH, fW)
    D = ds.shape[0]
    xs = torch.linspace(0, iW - 1, fW, dtype=torch.float).view(1, 1, fW).expand(D, fH, fW)
    ys = torch.linspace(0, iH - 1, fH, dtype=torch.float).view(1, fH, 1).expand(D, fH, fW)
    return torch.stack((xs, ys, ds), -1)


def get_geometry(frustum, camera2lidar_rots, camera2lidar_trans, intrins, post_rots, post_trans,
                 extra_rots=None, extra_trans=None):
    """base.py:92-135 -> [B, N, D, fH, fW, 3] lidar-frame xyz of every frustum point (fp32)."""
    B, N, _ = camera2lidar_trans.shape
    points = frustum - post_trans.view(B, N, 1, 1, 1, 3)
    points = torch.inverse(post_rots).view(B, N, 1, 1, 1, 3, 3).matmul(points.unsqueeze(-1))
    points = torch.cat((points[:, :, :, :, :, :2] * points[:, :, :, :, :, 2:3],
                        points[:, :, :, :, :, 2:3]), 5)
    combine = camera2lidar_rots.matmul(torch.inverse(intrins))
    points = combine.view(B, N, 1, 1, 1, 3, 3).matmul(points).squeeze(-1)
    points = points + camera2lidar_trans.view(B, N, 1, 1, 1, 3)
    if extra_rots is not None:
        points = (extra_rots.view(B, 1, 1, 1, 1, 3, 3).repeat(1, N, 1, 1, 1, 1, 1)
                  .matmul(points.unsqueeze(-1)).squeeze(-1))
    if extra_trans is not None:
        points = points + extra_trans.view(B, 1, 1, 1, 1, 3).repeat(1, N, 1, 1, 1, 1)
    return points


class LSSGeometry(nn.Module):
    """The index side of BaseTransform: owns dx / bx / nx and the frustum, turns calibration
    into a BEVPoolPlan (cached per calibration), pools lifted features into BEV."""

    def __init__(self, image_size, feature_size, xbound, ybound, zbound, dbound):
        super().__init__()
        self.image_size, self.feature_size = image_size, feature_size
        self.xbound, self.ybound, self.zbound, self.dbound = xbound, ybound, zbound, dbound
        dx, bx, nx = gen_dx_bx(xbound, ybound, zbound)
        self.dx = nn.Parameter(dx, requires_grad=False)
        self.bx = nn.Parameter(bx, requires_grad=False)
        self.nx = nn.Parameter(nx, requires_grad=False)
        self.frustum = nn.Parameter(create_frustum(image_size, feature_size, dbound),
                                    requires_grad=False)
        self.D = self.frustum.shape[0]
        self._plan_key, self._plan = None, None

    def geometry(self, camera2lidar_rots, camera2lidar_trans, intrins, post_rots, post_trans, **kw):
        return get_geometry(self.frustum, camera2lidar_rots, camera2lidar_trans, intrins, post_rots,
                            post_trans, kw.get("extra_rots"), kw.get("extra_trans"))

    def plan(self, geom, key=None):
        """BEVPoolPlan for `geom`; re-used while `key` (e.g. a calibration hash) is unchanged."""
        if key is not None and key == self._plan_key and self._plan is not None:
            return self._plan
        self._plan = BEVPoolPlan(geom, self.xbound, self.ybound, self.zbound)
        self._plan_key = key
        return self._plan

    def bev_pool_reference_path(self, geom_feats, x):
        """BaseTransform.bev_pool exactly as base.py:141-176 does it (torch index glue +
        the drop-in bev_pool op); used by the parity tests."""
        B, N, D, H, W, C = x.shape
        Nprime = B * N * D * H * W
        x = x.reshape(Nprime, C)
        geom_feats = ((geom_feats - (self.bx - self.dx / 2.0)) / self.dx).long()
        geom_feats = geom_feats.view(Nprime, 3)
        batch_ix = torch.cat([torch.full([Nprime // B, 1], ix, device=x.device, dtype=torch.long)
                              for ix in range(B)])
        geom_feats = torch.cat((geom_feats, batch_ix), 1)
        kept = ((geom_feats[:, 0] >= 0) & (geom_feats[:, 0] < self.nx[0])
                & (geom_feats[:, 1] >= 0) & (geom_feats[:, 1] < self.nx[1])
                & (geom_feats[:, 2] >= 0) & (geom_feats[:, 2] < self.nx[2]))
        x = x[kept]
        geom_feats = geom_feats[kept]
        x = bev_pool(x, geom_feats, B, int(self.nx[2]), int(self.nx[0]), int(self.nx[1]))
        return torch.cat(x.unbind(dim=2), 1)
