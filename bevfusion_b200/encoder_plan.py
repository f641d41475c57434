"""EncoderPlan -- host side of bevb200_encoder_* (csrc/encoder.cu): a SparseEncoder in eval mode as ONE
native call with no host synchronisation (row counts stay on the device), so a frame can be captured in
a CUDA graph.  Replaces the python loop of mmdet3d/models/backbones/sparse_encoder.py:113-130 over
spconv/conv.py:114-223 (one rulebook build + ~80 launches + one device->host count per conv there).

forward_train() is the same chain in training mode (batch-statistics BatchNorm, running statistics updated
in place) with a native whole-encoder backward, also sync-free and capturable.

A plan runs one precision: BF16x3 (the default, fp32 rows in and out), FP16 (fp16 operands with fp32
accumulation, half rows in and out) or INT8 (eval only: u8 activations x s8 weights with int32 accumulation and the
module's calibrated per-conv scales, half rows in and out); the numerical contracts are in include/bevfusion_b200.h.
Each plan packs its own weight image, so a module keeps one plan per precision."""
import ctypes

import torch

from . import _C
from .sparse_block import SparseBasicBlock, bn_fold_key, bn_scale_shift
from .spconv.ops import PREC_BF16X3, PREC_FP16, PREC_INT8


class _ConvDesc(ctypes.Structure):
    # mirrors bevb200_encoder_conv_t (include/bevfusion_b200.h)
    _fields_ = [("c_in", ctypes.c_int32), ("c_out", ctypes.c_int32), ("ksize", ctypes.c_int32 * 3),
                ("stride", ctypes.c_int32 * 3), ("padding", ctypes.c_int32 * 3), ("dilation", ctypes.c_int32 * 3),
                ("subm", ctypes.c_int32), ("relu", ctypes.c_int32), ("residual_from", ctypes.c_int32)]


class _BNDesc(ctypes.Structure):
    # mirrors bevb200_encoder_bn_t (include/bevfusion_b200.h)
    _fields_ = [("weight", ctypes.c_void_p), ("bias", ctypes.c_void_p), ("running_mean", ctypes.c_void_p),
                ("running_var", ctypes.c_void_p), ("num_batches_tracked", ctypes.c_void_p),
                ("eps", ctypes.c_float), ("momentum", ctypes.c_float)]


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
    def __init__(self, encoder, precision=PREC_BF16X3):
        if precision not in (PREC_BF16X3, PREC_FP16, PREC_INT8):
            raise ValueError("an encoder plan runs the bf16x3, the fp16 or the int8 precision")
        self.encoder = encoder
        self.precision = precision
        self.f16 = precision == PREC_FP16
        self.i8 = precision == PREC_INT8
        self.row_dtype = torch.float16 if self.f16 or self.i8 else torch.float32
        self.chain = _chain_of(encoder)
        if self.i8 and not all(relu for _, _, relu, _ in self.chain):
            raise ValueError("the int8 plan needs a ReLU after every conv (its activations are stored as u8)")
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
        if self.f16 or self.i8:
            _C.check(L.bevb200_encoder_set_precision(self._h, precision), "encoder_set_precision")
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
        scales = None
        if self.i8:
            scales = self.encoder.int8_scales()
            if scales is None:
                raise ValueError("the int8 plan needs calibrated scales: SparseEncoder.calibrate_int8() or "
                                 "set_int8_scales()")
            scales = [float(v) for v in scales]
        key = (str(dev), None if scales is None else tuple(scales))
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
            if self.i8:
                res = self.chain[i][3]
                _C.check(L.bevb200_encoder_set_conv_int8(self._h, i, _C.ptr(w), _C.ptr(scale), _C.ptr(shift),
                                                         scales[i - 1] if i > 0 else 1.0, scales[i],
                                                         scales[res] if res >= 0 else 1.0, _C.ptr(self._params),
                                                         self._params.numel(), stream), "encoder_set_conv_int8")
                continue
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
        """voxel_features [N, C] fp32 (an fp16 or int8 plan: fp16), coors [N, 4] int32 (b, x, y, z); with n_voxels_dev
        (device int32[1]) only the first n rows are valid -- nothing is read back.  Returns [B, C*D, H, W] in the
        rows' dtype."""
        _C.require_cuda(voxel_features, "voxel_features", self.row_dtype)
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
                out = torch.empty(shape, dtype=self.row_dtype, device=dev)
            elif out.dtype != self.row_dtype:
                raise ValueError("out= must have the plan's row dtype %s" % self.row_dtype)
            from .spconv.ops import _batch_stride_of
            stride = _batch_stride_of(out, shape, self.row_dtype)
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
            fwd = L.bevb200_encoder_forward_f16 if self.f16 or self.i8 else L.bevb200_encoder_forward
            rc = fwd(self._h, _C.ptr(self._params), _C.ptr(voxel_features), _C.ptr(coors), n, _C.ptr(n_voxels_dev),
                     B, caps, _C.ptr(out), stride, _C.ptr(self.status), _C.ptr(self._ws), self._ws.numel(),
                     _C.current_stream(dev), side)
        _C.check(rc, "encoder_forward")
        return out

    # -- training ------------------------------------------------------------------------------
    def train_state_bytes(self, max_voxels, batch_size, level_caps=None):
        """Device bytes one training forward keeps for its backward (sized by the level caps)."""
        return int(_C.lib().bevb200_encoder_train_state_bytes(self._h, int(max_voxels), int(batch_size),
                                                              self._caps_arg(level_caps)))

    def backward_workspace_bytes(self, max_voxels, batch_size, level_caps=None):
        return int(_C.lib().bevb200_encoder_backward_workspace_bytes(self._h, int(max_voxels), int(batch_size),
                                                                     self._caps_arg(level_caps)))

    def saved_rows(self, state, max_voxels, batch_size, conv, level_caps=None):
        """(pre-BN rows z, output rows y) of conv `conv` as saved by a training forward into `state`: fp32
        [cap, c_out] each (y decoded from its split image; an fp16 plan: the saved z16 and y16, fp16 [cap, c_out]);
        only the level's first status[1 + l] rows are defined."""
        zo, yo = ctypes.c_size_t(), ctypes.c_size_t()
        _C.check(_C.lib().bevb200_encoder_train_saved(self._h, int(max_voxels), int(batch_size),
                                                      self._caps_arg(level_caps), int(conv), ctypes.byref(zo),
                                                      ctypes.byref(yo)), "encoder_train_saved")
        c = self.chain[conv][0].out_channels
        cap = self.level_caps(max_voxels, batch_size, level_caps)[self.level_of(conv)]
        if self.f16:
            return (state[zo.value:zo.value + cap * c * 2].view(torch.float16).view(cap, c),
                    state[yo.value:yo.value + cap * c * 2].view(torch.float16).view(cap, c))
        z = state[zo.value:zo.value + cap * c * 4].view(torch.float32).view(cap, c)
        img = state[yo.value:yo.value + cap * c * 4].view(torch.bfloat16).view(cap, c // 16, 2, 16).float()
        return z, (img[:, :, 0] + img[:, :, 1]).reshape(cap, c)

    def level_of(self, conv):
        """level of conv `conv`'s output rows (0 = the voxels)."""
        return sum(1 for cv, _, _, _ in self.chain[:conv + 1] if not cv.subm)

    def _bn_descs(self, bn_weights, bn_biases, running):
        descs = (_BNDesc * len(self.chain))()
        for d, (_, bn, _, _), g, b, (rm, rv) in zip(descs, self.chain, bn_weights, bn_biases, running):
            d.weight, d.bias = g.data_ptr(), b.data_ptr()
            d.running_mean, d.running_var = rm.data_ptr(), rv.data_ptr()
            d.num_batches_tracked = _C.ptr(bn.num_batches_tracked)
            d.eps, d.momentum = float(bn.eps), float(bn.momentum)
        return descs

    def _forward_train_native(self, voxel_features, coors, batch_size, n_voxels_dev, level_caps, overlap_rulebooks,
                              weights, bn_weights, bn_biases):
        """One training forward: returns (dense output, state).  Updates the running statistics in place.
        An fp16 plan takes half or fp32 features (rounded once to fp16) and widens half weights and BN tensors
        for the call (the C ABI takes fp32 parameters); half running statistics are updated through fp32 copies."""
        dev = voxel_features.device
        n = voxel_features.shape[0]
        B = int(batch_size)
        X, Y, Z = self.out_shape
        L = _C.lib()
        voxel_features = voxel_features.to(self.row_dtype).contiguous()
        weights = [_f32(w) for w in weights]
        bn_weights, bn_biases = [_f32(g) for g in bn_weights], [_f32(b) for b in bn_biases]
        running = [(_f32(bn.running_mean), _f32(bn.running_var)) for _, bn, _, _ in self.chain]
        with torch.cuda.device(dev):
            out = torch.empty((B, self.out_channels * Z, X, Y), dtype=self.row_dtype, device=dev)
            caps = self._caps_arg(level_caps)
            state = torch.empty(L.bevb200_encoder_train_state_bytes(self._h, n, B, caps), dtype=torch.uint8,
                                device=dev)
            if self.status is None or self.status.device != dev:
                self.status = torch.zeros(1 + self.n_levels, dtype=torch.int32, device=dev)
            side = 0
            if overlap_rulebooks:
                if self._side is None or self._side.device != dev:
                    self._side = torch.cuda.Stream(device=dev)
                side = self._side.cuda_stream
            wp = (ctypes.c_void_p * len(weights))(*[w.data_ptr() for w in weights])
            fwd = L.bevb200_encoder_forward_train_f16 if self.f16 else L.bevb200_encoder_forward_train
            rc = fwd(self._h, wp, self._bn_descs(bn_weights, bn_biases, running), _C.ptr(voxel_features),
                     _C.ptr(coors), n, _C.ptr(n_voxels_dev), B, caps, _C.ptr(out), 0, _C.ptr(self.status),
                     _C.ptr(state), state.numel(), _C.current_stream(dev), side)
        _C.check(rc, "encoder_forward_train")
        for (_, bn, _, _), (rm, rv) in zip(self.chain, running):
            if rm is not bn.running_mean:          # half running statistics: updated through fp32 copies
                bn.running_mean.copy_(rm)
                bn.running_var.copy_(rv)
        # torch's BatchNorm bumps num_batches_tracked's version (add_(1)); the eval plan's fold key reads it
        for _, bn, _, _ in self.chain:
            if bn.num_batches_tracked is not None:
                torch.autograd.graph.increment_version(bn.num_batches_tracked)
        return out, state

    def _backward_native(self, state, n, batch_size, level_caps, grad_out, weights, need_input):
        """Gradients in the native dtypes: features in the plan's row dtype, everything else fp32."""
        dev = grad_out.device
        L = _C.lib()
        grad_out = grad_out.to(self.row_dtype).contiguous()
        weights = [_f32(w) for w in weights]
        with torch.cuda.device(dev):
            caps = self._caps_arg(level_caps)
            ws = torch.empty(L.bevb200_encoder_backward_workspace_bytes(self._h, n, int(batch_size), caps),
                             dtype=torch.uint8, device=dev)
            gfeat = (torch.empty((n, self.encoder.in_channels), dtype=self.row_dtype, device=dev)
                     if need_input else None)
            gw = [torch.empty_like(w) for w in weights]
            gg = [torch.empty(cv.out_channels, dtype=torch.float32, device=dev) for cv, _, _, _ in self.chain]
            gb = [torch.empty_like(g) for g in gg]

            def arr(ts):
                return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])

            bwd = L.bevb200_encoder_backward_f16 if self.f16 else L.bevb200_encoder_backward
            rc = bwd(self._h, arr(weights), _C.ptr(state), state.numel(), n, int(batch_size), caps, _C.ptr(grad_out),
                     0, _C.ptr(gfeat), arr(gw), arr(gg), arr(gb), _C.ptr(ws), ws.numel(), _C.current_stream(dev))
        _C.check(rc, "encoder_backward")
        return gfeat, gw, gg, gb

    def forward_train(self, voxel_features, coors, batch_size, n_voxels_dev=None, level_caps=None,
                      overlap_rulebooks=True):
        """Training-mode forward of the encoder (torch's BatchNorm1d in train mode, ReLU, residuals):
        voxel_features [N, C] fp32, coors [N, 4] int32, n_voxels_dev as in forward().  Differentiable in the
        features, every conv weight and every BN weight / bias; the backward is one native call on this
        forward's rulebooks.  Under torch.no_grad() it still normalises with batch statistics and updates the
        running statistics, and keeps nothing for a backward.
        An fp16 plan also takes half features, half conv weights and half BN modules; its output is half and the
        gradients come back in each tensor's dtype.  An int8 plan has no training form."""
        if self.i8:
            raise ValueError("the int8 plan runs the eval forward only")
        ok = (torch.float32, torch.float16) if self.f16 else (torch.float32,)
        if voxel_features.dtype not in ok:
            raise ValueError("voxel_features must be %s" % " or ".join(str(t) for t in ok))
        _C.require_cuda(voxel_features, "voxel_features", voxel_features.dtype)
        _C.require_cuda(coors, "coors", torch.int32)
        n = voxel_features.shape[0]
        assert coors.shape[0] == n and coors.shape[1] == 4 and voxel_features.shape[1] == self.encoder.in_channels
        if n == 0:
            raise ValueError("a training forward needs at least one voxel (BatchNorm statistics)")
        weights = [conv.weight for conv, _, _, _ in self.chain]
        for w in weights:
            if w.dtype not in ok:
                raise ValueError("conv weights must be %s" % " or ".join(str(t) for t in ok))
            _C.require_cuda(w, "conv weight", w.dtype)
        bn_w = [bn.weight for _, bn, _, _ in self.chain]
        bn_b = [bn.bias for _, bn, _, _ in self.chain]
        params = weights + bn_w + bn_b
        if torch.is_grad_enabled() and (voxel_features.requires_grad or any(p.requires_grad for p in params)):
            return _EncoderTrainFn.apply(self, coors, batch_size, n_voxels_dev, level_caps, overlap_rulebooks,
                                         voxel_features, *params)
        with torch.no_grad():
            out, _ = self._forward_train_native(voxel_features, coors, batch_size, n_voxels_dev, level_caps,
                                                overlap_rulebooks, weights, bn_w, bn_b)
        return out

    def overflowed(self):
        """True when a level cap truncated the last forward (host sync)."""
        return self.status is not None and int(self.status[0].item()) != 0


def _f32(t):
    """t itself when fp32, else an fp32 copy (the C ABI takes fp32 parameters)."""
    return t if t.dtype == torch.float32 else t.detach().float().contiguous()


class _EncoderTrainFn(torch.autograd.Function):
    """EncoderPlan.forward_train with the native backward.  The conv and BN parameters are saved with
    save_for_backward, so an in-place update between forward and backward raises; the state (rulebooks,
    pre-BN rows, output images, batch statistics) is allocated per call and saved alongside them."""

    @staticmethod
    def forward(ctx, plan, coors, batch_size, n_voxels_dev, level_caps, overlap_rulebooks, voxel_features, *params):
        nc = len(plan.chain)
        out, state = plan._forward_train_native(voxel_features, coors, batch_size, n_voxels_dev, level_caps,
                                                overlap_rulebooks, params[:nc], params[nc:2 * nc], params[2 * nc:])
        ctx.save_for_backward(state, *params)     # the state is freed with the graph's saved tensors
        ctx.plan, ctx.n, ctx.batch_size, ctx.level_caps = plan, voxel_features.shape[0], batch_size, level_caps
        ctx.feature_dtype = voxel_features.dtype
        return out

    @staticmethod
    def backward(ctx, grad_out):
        state, *params = ctx.saved_tensors
        plan = ctx.plan
        nc = len(plan.chain)
        gfeat, gw, gg, gb = plan._backward_native(state, ctx.n, ctx.batch_size, ctx.level_caps,
                                                  grad_out.contiguous(), params[:nc], ctx.needs_input_grad[6])
        if gfeat is not None:
            gfeat = gfeat.to(ctx.feature_dtype)
        grads = [g.to(p.dtype) for g, p in zip(gw + gg + gb, params)]     # each in its parameter's dtype
        return (None,) * 6 + (gfeat,) + tuple(grads)
