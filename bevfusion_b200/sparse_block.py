"""SparseBasicBlock / make_sparse_convmodule -- mirror of mmdet3d/ops/sparse_block.py:62-176
without mmcv / mmdet (build_conv_layer / build_norm_layer / BasicBlock are restated: same
sub-module names conv1, bn1, conv2, bn2 so reference checkpoints load)."""
import torch
from torch import nn

from . import spconv
from .spconv.conv import CONV_LAYERS


def build_conv_layer(cfg, *args, **kwargs):
    cfg = dict(cfg)
    layer_type = cfg.pop("type")
    if layer_type not in CONV_LAYERS:
        raise KeyError("Unrecognized sparse conv type %s" % layer_type)
    return CONV_LAYERS[layer_type](*args, **kwargs, **cfg)


def build_norm_layer(cfg, num_features, postfix=""):
    cfg = dict(cfg)
    layer_type = cfg.pop("type")
    requires_grad = cfg.pop("requires_grad", True)
    cfg.setdefault("eps", 1e-5)
    if layer_type in ("BN1d", "BN"):
        layer = nn.BatchNorm1d(num_features, **cfg)
    else:
        raise KeyError("Unrecognized norm type %s" % layer_type)
    for p in layer.parameters():
        p.requires_grad = requires_grad
    return "bn" + str(postfix), layer


def bn_fold_key(bn):
    """Cache key of the folded (scale, shift) of a BatchNorm: (data_ptr, _version) of every tensor that
    defines it.  A train-mode forward updates running_mean / running_var in place without bumping their
    version counters (the BN kernels' schemas do not mark them as mutated), but it does increment
    num_batches_tracked, so that counter is part of the key.  In-place writes through `.data` (e.g.
    `bn.running_mean.data.copy_(x)`) bypass the version counter and are not tracked; assigning a new
    tensor, or writing in place under torch.no_grad(), is."""
    tensors = (bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.num_batches_tracked)
    return tuple((t.data_ptr(), t._version) for t in tensors if t is not None)


def bn_scale_shift(bn):
    """Fold an eval-mode BatchNorm1d into per-channel (scale, shift); cached on the module until
    one of its parameters / buffers changes (bn_fold_key)."""
    key = bn_fold_key(bn)
    cached = getattr(bn, "_b200_fold", None)
    if cached is not None and cached[0] == key:
        return cached[1]
    out = _bn_scale_shift(bn)
    bn._b200_fold = (key, out)
    return out


def _bn_scale_shift(bn):
    scale = (bn.weight.detach() if bn.affine else torch.ones_like(bn.running_mean)) \
        * torch.rsqrt(bn.running_var + bn.eps)
    shift = (bn.bias.detach() if bn.affine else torch.zeros_like(bn.running_mean)) \
        - bn.running_mean * scale
    return scale.float().contiguous(), shift.float().contiguous()


class SparseBasicBlock(spconv.SparseModule):
    """conv1 -> bn1 -> relu -> conv2 -> bn2 -> (+identity) -> relu  (sparse_block.py:94-110)."""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None, conv_cfg=None, norm_cfg=None):
        super().__init__()
        norm_cfg = norm_cfg or dict(type="BN1d")
        self.norm1_name, norm1 = build_norm_layer(norm_cfg, planes, postfix=1)
        self.norm2_name, norm2 = build_norm_layer(norm_cfg, planes, postfix=2)
        self.conv1 = build_conv_layer(conv_cfg, inplanes, planes, 3, stride=stride, padding=1,
                                      dilation=1, bias=False)
        self.add_module(self.norm1_name, norm1)
        self.conv2 = build_conv_layer(conv_cfg, planes, planes, 3, padding=1, bias=False)
        self.add_module(self.norm2_name, norm2)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride

    @property
    def norm1(self):
        return getattr(self, self.norm1_name)

    @property
    def norm2(self):
        return getattr(self, self.norm2_name)

    def forward(self, x):
        identity = x.features
        assert x.features.dim() == 2, f"x.features.dim()={x.features.dim()}"
        out = self.conv1(x)
        out.features = self.norm1(out.features)
        out.features = self.relu(out.features)
        out = self.conv2(out)
        out.features = self.norm2(out.features)
        if self.downsample is not None:
            identity = self.downsample(x)
        out.features += identity
        out.features = self.relu(out.features)
        return out

    def forward_fused(self, x, precision=None):
        """Eval-mode forward with BN / residual / ReLU folded into the two conv epilogues."""
        assert self.downsample is None
        s1, t1 = bn_scale_shift(self.norm1)
        s2, t2 = bn_scale_shift(self.norm2)
        out = self.conv1(x, scale=s1, shift=t1, relu=True, precision=precision)
        out = self.conv2(out, scale=s2, shift=t2, residual=x.features.contiguous(), relu=True,
                         precision=precision)
        return out


def make_sparse_convmodule(in_channels, out_channels, kernel_size, indice_key, stride=1, padding=0,
                           conv_type="SubMConv3d", norm_cfg=None, order=("conv", "norm", "act")):
    """sparse_block.py:113-176."""
    assert isinstance(order, tuple) and len(order) <= 3
    assert set(order) | {"conv", "norm", "act"} == {"conv", "norm", "act"}
    conv_cfg = dict(type=conv_type, indice_key=indice_key)
    layers = []
    for layer in order:
        if layer == "conv":
            layers.append(build_conv_layer(conv_cfg, in_channels, out_channels, kernel_size,
                                           stride=stride, padding=padding, bias=False))
        elif layer == "norm":
            layers.append(build_norm_layer(norm_cfg, out_channels)[1])
        elif layer == "act":
            layers.append(nn.ReLU(inplace=True))
    return spconv.SparseSequential(*layers)
