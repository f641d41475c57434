"""SparseConvTensor -- mirror of mmdet3d/ops/spconv/structure.py:21-63."""
import numpy as np
import torch

from . import ops


class _ToDenseFunction(torch.autograd.Function):
    """dense() with a backward: the gradient of a scatter is the gather at the same sites."""

    @staticmethod
    def forward(ctx, features, indices, batch_size, spatial_shape):
        ctx.save_for_backward(indices)
        ctx.in_dtype = features.dtype
        # the scatter kernel takes fp32 rows; like the reference's scatter_nd the result has the features' dtype
        out = ops.sparse_to_dense(features.float().contiguous(), indices, batch_size, spatial_shape, z_major=False)
        return out.to(features.dtype)

    @staticmethod
    def backward(ctx, grad):
        (indices,) = ctx.saved_tensors
        idx = indices.long()
        g = grad[idx[:, 0], :, idx[:, 1], idx[:, 2], idx[:, 3]]          # [N, C]
        return g.to(ctx.in_dtype), None, None, None


class SparseConvTensor:
    def __init__(self, features, indices, spatial_shape, batch_size, grid=None):
        self.features = features
        self.indices = indices
        self.spatial_shape = spatial_shape
        self.batch_size = batch_size
        self.indice_dict = {}
        self.grid = grid

    @property
    def spatial_size(self):
        return np.prod(self.spatial_shape)

    def find_indice_pair(self, key):
        if key is None:
            return None
        return self.indice_dict.get(key, None)

    def dense(self, channels_first=True):
        """[B, C, X, Y, Z] (channels_first) or [B, X, Y, Z, C]; zero outside the active set.
        Differentiable w.r.t. the features like the reference's scatter_nd (structure.py:5-18)."""
        out = _ToDenseFunction.apply(self.features, self.indices.int().contiguous(), int(self.batch_size),
                                     tuple(int(v) for v in self.spatial_shape))
        if channels_first:
            return out
        ndim = len(self.spatial_shape)
        return out.permute(0, *range(2, ndim + 2), 1).contiguous()

    @property
    def sparity(self):
        return self.indices.shape[0] / np.prod(self.spatial_shape) / self.batch_size
