"""EncoderPlan -- host side of bevb200_encoder_* (csrc/encoder.cu): a SparseEncoder in eval mode as ONE
native call with no host synchronisation (row counts stay on the device), so a frame can be captured in
a CUDA graph.  Replaces the python loop of mmdet3d/models/backbones/sparse_encoder.py:113-130 over
spconv/conv.py:114-223 (one rulebook build + ~80 launches + one device->host count per conv there)."""
import ctypes

import torch

from . import _C
from .sparse_block import SparseBasicBlock, bn_fold_key, bn_scale_shift


class _ConvDesc(ctypes.Structure):
    # mirrors bevb200_encoder_conv_t (include/bevfusion_b200.h)
    _fields_ = [("c_in", ctypes.c_int32), ("c_out", ctypes.c_int32), ("ksize", ctypes.c_int32 * 3),
                ("stride", ctypes.c_int32 * 3), ("padding", ctypes.c_int32 * 3), ("dilation", ctypes.c_int32 * 3),
                ("subm", ctypes.c_int32), ("relu", ctypes.c_int32), ("residual_from", ctypes.c_int32)]


def _chain_of(encoder):
    """[(conv module, bn module or None, relu, residual_from)] in execution order
    (sparse_encoder.py:113-124, sparse_block.py:94-110)."""
    chain = []

    def add_module_seq(seq):
        conv = seq[0]
        bn = seq[1] if len(seq) > 1 and isinstance(seq[1], torch.nn.BatchNorm1d) else None
        relu = any(isinstance(m, torch.nn.ReLU) for m in seq)
        chain.append((conv, bn, relu, -1))

    add_module_seq(encoder.conv_input)
    for stage in encoder.encoder_layers:
        for block in stage:
            if isinstance(block, SparseBasicBlock):
                if block.downsample is not None:
                    raise NotImplementedError("SparseBasicBlock.downsample")
                identity = len(chain) - 1            # the output of the conv before conv1
                chain.append((block.conv1, block.norm1, True, -1))
                chain.append((block.conv2, block.norm2, True, identity))
            else:
                add_module_seq(block)
    add_module_seq(encoder.conv_out)
    return chain


def supported(encoder):
    """The native plan covers the (conv, norm, act) order with 3-D convs whose channel counts have a
    tensor-core form; anything else stays on the modular path."""
    if encoder.order != ("conv", "norm", "act"):
        return False
    try:
        chain = _chain_of(encoder)
    except NotImplementedError:
        return False
    for i, (conv, bn, relu, res) in enumerate(chain):
        if conv.ndim != 3 or conv.transposed or conv.inverse or conv.conv1x1:
            return False
        if conv.out_channels not in (16, 32, 64, 128) or conv.in_channels > 128:
            return False
        if i > 0 and conv.in_channels not in (16, 32, 64, 128):
            return False
    return True


class EncoderPlan:
    def __init__(self, encoder):
        self.encoder = encoder
        self.chain = _chain_of(encoder)
        L = _C.lib()
        descs = (_ConvDesc * len(self.chain))()
        for d, (conv, bn, relu, res) in zip(descs, self.chain):
            d.c_in, d.c_out = conv.in_channels, conv.out_channels
            for k in range(3):
                d.ksize[k], d.stride[k] = conv.kernel_size[k], conv.stride[k]
                d.padding[k], d.dilation[k] = conv.padding[k], conv.dilation[k]
            d.subm, d.relu, d.residual_from = int(conv.subm), int(relu), res
        shape = (ctypes.c_int32 * 3)(*[int(v) for v in encoder.sparse_shape])
        handle = ctypes.c_void_p()
        _C.check(L.bevb200_encoder_create(int(encoder.in_channels), shape, descs, len(self.chain),
                                          ctypes.byref(handle)), "encoder_create")
        self._h = handle
        self.n_levels = L.bevb200_encoder_num_levels(self._h)
        oshape = (ctypes.c_int32 * 3)()
        oc = ctypes.c_int32()
        _C.check(L.bevb200_encoder_output_shape(self._h, oshape, ctypes.byref(oc)), "encoder_output_shape")
        self.out_shape, self.out_channels = [int(v) for v in oshape], int(oc.value)
        self._params = None
        self._param_key = None
        self._ws = None
        self._ws_captured = False    # a CUDA graph recorded a forward that uses self._ws
        self._graph_held = []        # replaced workspaces that a captured graph still writes into
        self._side = None
        self.status = None           # int32[1 + levels] of the last forward (device)

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                _C.lib().bevb200_encoder_destroy(h)
            except Exception:
                pass

    # -- parameters: packed once, re-packed when a weight / BN tensor changes -------------------
    def _sync_params(self, dev):
        key = (str(dev),)
        for conv, bn, _, _ in self.chain:
            key += tuple((t.data_ptr(), t._version) for t in (conv.weight, conv.bias) if t is not None)
            if bn is not None:
                key += bn_fold_key(bn)
        if key == self._param_key:
            return
        L = _C.lib()
        nbytes = L.bevb200_encoder_param_bytes(self._h)
        if self._params is None or self._params.device != dev:
            self._params = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)
        stream = _C.current_stream(dev)
        keep = []
        for i, (conv, bn, _, _) in enumerate(self.chain):
            scale = shift = None
            if bn is not None:
                scale, shift = bn_scale_shift(bn)
            if conv.bias is not None:      # (acc + b) * s + t = acc * s + (b * s + t)
                b = conv.bias.detach().float()
                shift = (b * scale + shift) if scale is not None else b
                shift = shift.contiguous()
            w = conv.weight.detach().float().contiguous()
            keep += [w, scale, shift]
            _C.check(L.bevb200_encoder_set_conv(self._h, i, _C.ptr(w), _C.ptr(scale), _C.ptr(shift),
                                                _C.ptr(self._params), self._params.numel(), stream),
                     "encoder_set_conv")
        self._param_key = key

    def level_caps(self, max_voxels, batch_size, user_caps=None):
        caps = (ctypes.c_int32 * self.n_levels)()
        _C.check(_C.lib().bevb200_encoder_level_caps(self._h, int(max_voxels), int(batch_size),
                                                     self._caps_arg(user_caps), caps), "encoder_level_caps")
        return [int(v) for v in caps]

    def _caps_arg(self, user_caps):
        if user_caps is None:
            return None
        assert len(user_caps) == self.n_levels
        return (ctypes.c_int32 * self.n_levels)(*[int(v) for v in user_caps])

    def forward(self, voxel_features, coors, batch_size, n_voxels_dev=None, out=None, level_caps=None,
                overlap_rulebooks=True):
        """voxel_features [N, C] fp32, coors [N, 4] int32 (b, x, y, z); with n_voxels_dev (device
        int32[1]) only the first n rows are valid -- nothing is read back.  Returns [B, C*D, H, W]."""
        _C.require_cuda(voxel_features, "voxel_features", torch.float32)
        _C.require_cuda(coors, "coors", torch.int32)
        dev = voxel_features.device
        n = voxel_features.shape[0]
        assert coors.shape[0] == n and coors.shape[1] == 4 and voxel_features.shape[1] == self.encoder.in_channels
        B = int(batch_size)
        X, Y, Z = self.out_shape
        shape = (B, self.out_channels * Z, X, Y)
        L = _C.lib()
        with torch.cuda.device(dev):
            if out is None:
                out = torch.empty(shape, dtype=torch.float32, device=dev)
            from .spconv.ops import _batch_stride_of
            stride = _batch_stride_of(out, shape)
            if n == 0:
                out.zero_()
                return out
            self._sync_params(dev)
            caps = self._caps_arg(level_caps)
            need = L.bevb200_encoder_workspace_bytes(self._h, n, B, caps)
            if self._ws is None or self._ws.device != dev or self._ws.numel() < need:
                # a graph captured earlier replays into the old block: once freed, the allocator would hand it
                # to other tensors, so a captured workspace stays alive with the plan
                if self._ws_captured:
                    self._graph_held.append(self._ws)
                self._ws, self._ws_captured = None, False
                self._ws = torch.empty(int(need * 1.25) + 4096, dtype=torch.uint8, device=dev)
            if torch.cuda.is_current_stream_capturing():
                self._ws_captured = True
            if self.status is None or self.status.device != dev:
                self.status = torch.zeros(1 + self.n_levels, dtype=torch.int32, device=dev)
            side = 0
            if overlap_rulebooks:
                if self._side is None or self._side.device != dev:
                    self._side = torch.cuda.Stream(device=dev)
                side = self._side.cuda_stream
            rc = L.bevb200_encoder_forward(self._h, _C.ptr(self._params), _C.ptr(voxel_features), _C.ptr(coors),
                                           n, _C.ptr(n_voxels_dev), B, caps, _C.ptr(out), stride,
                                           _C.ptr(self.status), _C.ptr(self._ws), self._ws.numel(),
                                           _C.current_stream(dev), side)
        _C.check(rc, "encoder_forward")
        return out

    def overflowed(self):
        """True when a level cap truncated the last forward (host sync)."""
        return self.status is not None and int(self.status[0].item()) != 0
