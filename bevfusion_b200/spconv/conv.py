"""Sparse convolution modules -- mirror of mmdet3d/ops/spconv/conv.py:40-455.

Same constructor arguments, parameter names and shapes (`weight [k0,k1,k2,Cin,Cout]`, optional
`bias [Cout]`, conv.py:100-104) so reference state_dicts load unchanged.  The forward pass builds
(or re-uses) a neighbour-table rulebook and runs ONE implicit-GEMM kernel per conv."""
import math

import numpy as np
import torch
from torch.nn import init
from torch.nn.parameter import Parameter

from . import functional as Fsp
from . import ops
from .modules import SparseModule
from .structure import SparseConvTensor

# registry used by make_sparse_convmodule / configs (the reference registers these names in
# mmcv's CONV_LAYERS, conv.py:226-455)
CONV_LAYERS = {}


def register(cls):
    CONV_LAYERS[cls.__name__] = cls
    return cls


def _fan_in(weight):
    """Inputs feeding one output channel of a [k..., Cin, Cout] filter (conv.py:107-112 init)."""
    return weight[..., 0].numel()


class SparseConvolution(SparseModule):
    def __init__(self, ndim, in_channels, out_channels, kernel_size=3, stride=1, padding=0,
                 dilation=1, groups=1, bias=True, subm=False, output_padding=0, transposed=False,
                 inverse=False, indice_key=None, fused_bn=False):
        super().__init__()
        assert groups == 1
        if not isinstance(kernel_size, (list, tuple)):
            kernel_size = [kernel_size] * ndim
        if not isinstance(stride, (list, tuple)):
            stride = [stride] * ndim
        if not isinstance(padding, (list, tuple)):
            padding = [padding] * ndim
        if not isinstance(dilation, (list, tuple)):
            dilation = [dilation] * ndim
        if not isinstance(output_padding, (list, tuple)):
            output_padding = [output_padding] * ndim
        for d, s in zip(dilation, stride):
            assert any([s == 1, d == 1]), "don't support this."
        self.ndim = ndim
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.kernel_size = list(kernel_size)
        self.conv1x1 = np.prod(kernel_size) == 1
        self.stride = list(stride)
        self.padding = list(padding)
        self.dilation = list(dilation)
        self.transposed = transposed
        self.inverse = inverse
        self.output_padding = list(output_padding)
        self.groups = groups
        self.subm = subm
        self.indice_key = indice_key
        self.fused_bn = fused_bn
        self.weight = Parameter(torch.Tensor(*kernel_size, in_channels, out_channels))
        if bias:
            self.bias = Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter("bias", None)
        self._packed_cache = None
        self.reset_parameters()

    def _packed_weight(self, precision):
        """tensor-core image of the weights, rebuilt only when the parameter changes"""
        if precision is None:
            precision = ops.default_precision()
        if precision == ops.PREC_FP32:
            return None
        w = self.weight
        # keyed on the parameter itself, so a half parameter is widened and packed once, not every call
        key = (int(precision), w.data_ptr(), w._version, str(w.device), w.dtype)
        if self._packed_cache is None or self._packed_cache[0] != key:
            self._packed_cache = (key, ops.pack_weights(w.detach().float().contiguous(), precision))
        return self._packed_cache[1]

    def reset_parameters(self):
        init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            bound = 1 / math.sqrt(_fan_in(self.weight))
            init.uniform_(self.bias, -bound, bound)

    # -- rulebook lookup / build (conv.py:152-182) ------------------------------------------
    def _rulebook(self, input):
        """Returns (Rulebook, out_spatial_shape).  Rulebooks are cached in input.indice_dict
        under `indice_key` exactly like the reference, and additionally under a structural
        key when indice_key is None: the rulebook is a pure function of (indices, geometry),
        so SparseBasicBlock convs (which pass no key, sparse_block.py:62-110) share one
        instead of rebuilding it per conv as the reference does."""
        if self.transposed or self.inverse:
            raise NotImplementedError("transposed / inverse sparse conv is outside the hot path")
        indices = input.indices
        skey = ("__auto__", indices.data_ptr(), indices.shape[0], tuple(input.spatial_shape),
                tuple(self.kernel_size), tuple(self.stride), tuple(self.padding),
                tuple(self.dilation), bool(self.subm))
        key = self.indice_key
        datas = input.indice_dict.get(key, None) if key is not None else None
        if datas is None:
            datas = input.indice_dict.get(skey, None)      # same geometry built under another key
            if datas is not None and key is not None:
                input.indice_dict[key] = datas
        if datas is not None:
            return datas[2], datas[5]
        side = input.indice_dict.get("__rulebook_stream__")
        if side is None:
            rb, out_shape = ops.get_rulebook(indices, input.batch_size, input.spatial_shape,
                                             self.kernel_size, self.stride, self.padding,
                                             self.dilation, self.output_padding, self.subm,
                                             self.transposed)
        else:
            # The rulebook depends on the indices only, not on the features: build it on a side
            # stream so its kernels -- and the host wait for the output count of a strided conv --
            # overlap with the convolutions already queued on the main stream (SparseEncoder's
            # fused path sets this up; the convs wait on `rb.ready`).
            main = torch.cuda.current_stream(indices.device)
            with torch.cuda.stream(side):
                rb, out_shape = ops.get_rulebook(indices, input.batch_size, input.spatial_shape,
                                                 self.kernel_size, self.stride, self.padding,
                                                 self.dilation, self.output_padding, self.subm,
                                                 self.transposed)
                rb.ready = torch.cuda.Event()
                rb.ready.record(side)
            for t in (rb.nbr, rb.outids):
                t.record_stream(main)
        # (outids, indices, indice_pairs, indice_pair_num, spatial_shape) as conv.py:176-182,
        # with the Rulebook object in the indice_pairs slot, plus the output shape
        datas = (rb.outids, indices, rb, None, input.spatial_shape, out_shape)
        input.indice_dict[skey] = datas
        if key is not None:
            input.indice_dict[key] = datas
        return rb, out_shape

    def forward(self, input, scale=None, shift=None, residual=None, relu=False, precision=None):
        """conv.py:114-223.  The optional keyword arguments fuse eval-mode BatchNorm
        (scale, shift), a residual add and ReLU into the conv epilogue."""
        assert isinstance(input, SparseConvTensor)
        features = input.features
        fused = scale is not None or shift is not None or residual is not None or relu
        needs_grad = torch.is_grad_enabled() and (features.requires_grad or self.weight.requires_grad)
        if fused and needs_grad:
            # the fused epilogues are an inference path: refusing is better than silently dropping gradients
            raise RuntimeError("fused BN / residual / ReLU epilogues do not record gradients; call the conv "
                               "without them (or under torch.no_grad())")
        if self.conv1x1:
            features = torch.mm(input.features, self.weight.view(self.in_channels, self.out_channels))
            if self.bias is not None:
                features = features + self.bias
            if scale is not None:
                features = features * scale
            if shift is not None:
                features = features + shift
            if residual is not None:
                features = features + residual
            if relu:
                features = torch.relu(features)
            out_tensor = SparseConvTensor(features, input.indices, input.spatial_shape,
                                          input.batch_size)
            out_tensor.indice_dict = input.indice_dict
            out_tensor.grid = input.grid
            return out_tensor
        rb, out_spatial_shape = self._rulebook(input)
        ready = getattr(rb, "ready", None)
        if ready is not None:                       # built on the side stream: order this stream after it
            torch.cuda.current_stream(features.device).wait_event(ready)
            rb.ready = None
        if fused or not needs_grad:
            # half features or weights (mixed-precision training, ops.indice_conv's rule): widened to
            # fp32 once, the same kernel, the output narrowed once after the epilogue
            half = torch.half in (features.dtype, self.weight.dtype)
            if self.bias is not None:
                # bias folds into the epilogue shift: (acc + b) * s + t = acc * s + (b * s + t)
                b = self.bias.detach().float()
                shift = b * scale + shift if scale is not None and shift is not None else (
                    b * scale if scale is not None else (b + shift if shift is not None else b))
            weight = self.weight.detach()
            if half:
                features, weight = features.float(), weight.float()
                residual = None if residual is None else residual.float().contiguous()
            out_features = ops.sparse_conv(features.contiguous(), weight.contiguous(),
                                           rb.nbr, rb.n_out, scale, shift, residual, relu, precision,
                                           packed=self._packed_weight(precision))
            if half:
                out_features = out_features.half()
        else:
            fn = Fsp.indice_subm_conv if self.subm else Fsp.indice_conv
            out_features = fn(features, self.weight, rb, None, rb.n_out)
            if self.bias is not None:
                out_features += self.bias
        out_tensor = SparseConvTensor(out_features, rb.outids, out_spatial_shape, input.batch_size)
        out_tensor.indice_dict = input.indice_dict
        out_tensor.grid = input.grid
        return out_tensor


@register
class SparseConv3d(SparseConvolution):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1,
                 groups=1, bias=True, indice_key=None):
        super().__init__(3, in_channels, out_channels, kernel_size, stride, padding, dilation,
                         groups, bias, indice_key=indice_key)


@register
class SubMConv3d(SparseConvolution):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1,
                 groups=1, bias=True, indice_key=None):
        super().__init__(3, in_channels, out_channels, kernel_size, stride, padding, dilation,
                         groups, bias, True, indice_key=indice_key)
