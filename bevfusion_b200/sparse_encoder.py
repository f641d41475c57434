"""SparseEncoder -- mirror of mmdet3d/models/backbones/sparse_encoder.py:11-217 (the VoxelNet
middle encoder of BEVFusion's LiDAR branch), without mmcv / mmdet.  Same constructor, same
sub-module names (conv_input, encoder_layers.encoder_layer{i}, conv_out) and state_dict."""
import os

import torch
from torch import nn

from . import spconv
from .sparse_block import SparseBasicBlock, bn_scale_shift, make_sparse_convmodule
from .spconv import ops as sp_ops


class SparseEncoder(nn.Module):
    def __init__(self, in_channels, sparse_shape, order=("conv", "norm", "act"),
                 norm_cfg=dict(type="BN1d", eps=1e-3, momentum=0.01), base_channels=16,
                 output_channels=128,
                 encoder_channels=((16,), (32, 32, 32), (64, 64, 64), (64, 64, 64)),
                 encoder_paddings=((1,), (1, 1, 1), (1, 1, 1), ((0, 1, 1), 1, 1)),
                 block_type="conv_module"):
        super().__init__()
        assert block_type in ["conv_module", "basicblock"]
        self.sparse_shape = sparse_shape
        self.in_channels = in_channels
        self.order = tuple(order)
        self.base_channels = base_channels
        self.output_channels = output_channels
        self.encoder_channels = encoder_channels
        self.encoder_paddings = encoder_paddings
        self.stage_num = len(self.encoder_channels)
        self.fp16_enabled = False
        assert isinstance(order, (list, tuple)) and len(order) == 3
        assert set(order) == {"conv", "norm", "act"}
        if self.order[0] != "conv":  # pre activate
            self.conv_input = make_sparse_convmodule(in_channels, self.base_channels, 3,
                                                     norm_cfg=norm_cfg, padding=1,
                                                     indice_key="subm1", conv_type="SubMConv3d",
                                                     order=("conv",))
        else:
            self.conv_input = make_sparse_convmodule(in_channels, self.base_channels, 3,
                                                     norm_cfg=norm_cfg, padding=1,
                                                     indice_key="subm1", conv_type="SubMConv3d")
        encoder_out_channels = self.make_encoder_layers(make_sparse_convmodule, norm_cfg,
                                                        self.base_channels, block_type=block_type)
        self.overlap_rulebooks = os.environ.get("BEVB200_RULEBOOK_STREAM", "1") != "0"
        # eval mode, default precision: the whole encoder is one native, sync-free call (encoder_plan.py);
        # BEVB200_ENCODER_NATIVE=0 keeps the per-conv python loop below (A/B runs, other precisions)
        self.native_plan = os.environ.get("BEVB200_ENCODER_NATIVE", "1") != "0"
        self._plan = None
        self._plan_f16 = None        # the fp16 plan: its own weight image, never shared with the bf16x3 one
        self._plan_int8 = None
        # per-conv output scales of the int8 plan (calibrate_int8 / set_int8_scales): a plain attribute, not a buffer,
        # so the state_dict stays the reference's and its checkpoints load with strict=True
        self._int8_scales = None
        self.rulebook_lookahead = os.environ.get("BEVB200_RULEBOOK_LOOKAHEAD", "1") != "0"
        self.conv_out = make_sparse_convmodule(encoder_out_channels, self.output_channels,
                                               kernel_size=(1, 1, 3), stride=(1, 1, 2),
                                               norm_cfg=norm_cfg, padding=0,
                                               indice_key="spconv_down2", conv_type="SparseConv3d")

    def plan(self, precision=sp_ops.PREC_BF16X3):
        """The native EncoderPlan of this module for `precision` (bf16x3, fp16 or int8, built lazily), or None when
        a layer has no native form."""
        attr = {sp_ops.PREC_FP16: "_plan_f16", sp_ops.PREC_INT8: "_plan_int8"}.get(precision, "_plan")
        if getattr(self, attr) is None:
            from . import encoder_plan
            setattr(self, attr, encoder_plan.EncoderPlan(self, precision) if encoder_plan.supported(self) else False)
        return getattr(self, attr) or None

    def forward(self, voxel_features, coors, batch_size, fused=None, precision=None, out=None,
                num_voxels=None, **kwargs):
        """sparse_encoder.py:99-132.  voxel_features [N, C] fp32 or fp16, coors [N, 4] int32
        (batch, x, y, z).  Returns spatial features [B, C*D, H, W], in half when the features or the
        conv weights are (each conv computes in fp32 and narrows its output once).

        fused=None picks the fused path (BN / ReLU / residual in the conv epilogues, dense()
        written directly in the output layout) whenever the module is in eval mode.  `out`
        (fused path) is an optional [B, C*D, H, W] view to write into, e.g. the LiDAR channels
        of the fuser's concatenated input (fusers/conv.py:16).

        precision=sp_ops.PREC_FP16 runs the native plan in fp16 (fp32 accumulation; the contract is in
        include/bevfusion_b200.h) and returns half: in eval mode under no_grad, and in training mode with
        `num_voxels=`.  Anything else raises a ValueError; there is no fp16 form of the per-conv path.

        precision=sp_ops.PREC_INT8 runs the native plan on u8 activations and s8 weights with the scales of
        calibrate_int8() / set_int8_scales() and returns half: in eval mode under no_grad only."""
        coors = coors.int()
        if fused is None:
            fused = not self.training and self.order == ("conv", "norm", "act")
        if precision is None:
            precision = sp_ops.default_precision()
        if precision == sp_ops.PREC_INT8:
            return self._forward_int8(voxel_features, coors, batch_size, fused, out, num_voxels)
        if precision == sp_ops.PREC_FP16:
            return self._forward_fp16(voxel_features, coors, batch_size, fused, out, num_voxels)
        if (fused and self.native_plan and precision == sp_ops.PREC_BF16X3 and not torch.is_grad_enabled()
                and voxel_features.dtype == torch.float32 and self.conv_input[0].weight.dtype == torch.float32
                and self.plan() is not None):
            # `num_voxels` (device int32[1]): only the first rows are valid -- no host round trip
            return self.plan().forward(voxel_features.contiguous(), coors.contiguous(), batch_size,
                                       n_voxels_dev=num_voxels, out=out, overlap_rulebooks=self.overlap_rulebooks)
        if num_voxels is not None and self.training:
            return self._forward_train_native(voxel_features, coors, batch_size, num_voxels, precision, out)
        if num_voxels is not None:
            raise ValueError("num_voxels= needs the native plan (eval mode, bf16x3, no grad)")
        x = spconv.SparseConvTensor(voxel_features, coors, self.sparse_shape, batch_size)
        if fused:
            return self._forward_fused(x, precision, out)
        if out is not None:
            raise ValueError("out= is only supported on the fused (eval) path")
        x = self.conv_input(x)
        encode_features = []
        for encoder_layer in self.encoder_layers:
            x = encoder_layer(x)
            encode_features.append(x)
        out = self.conv_out(encode_features[-1])
        spatial_features = out.dense()
        N, C, H, W, D = spatial_features.shape
        spatial_features = spatial_features.permute(0, 1, 4, 2, 3).contiguous()
        return spatial_features.view(N, C * D, H, W)

    def _forward_train_native(self, voxel_features, coors, batch_size, num_voxels, precision, out):
        """Training mode with a device-side voxel count: the native training plan (EncoderPlan.forward_train),
        sync-free and capturable.  What it does not cover raises instead of falling back."""
        def refuse(reason):
            raise ValueError("num_voxels= in training mode runs the native training plan, which needs " + reason)
        if precision == sp_ops.PREC_FP16:
            if voxel_features.dtype not in (torch.float32, torch.float16):
                refuse("fp32 or fp16 features")
        elif precision != sp_ops.PREC_BF16X3:
            refuse("the bf16x3 or the fp16 precision")
        elif voxel_features.dtype != torch.float32 or any(p.dtype != torch.float32 for p in self.parameters()):
            refuse("fp32 features and weights (no half)")
        if out is not None:
            refuse("no out= (the output is a fresh tensor)")
        plan = self.plan(precision)
        if plan is None:
            refuse("a chain of (conv, norm, act) modules with tensor-core channel counts")
        for conv, bn, _, _ in plan.chain:
            if conv.bias is not None:
                refuse("convs without bias")
            if bn is None or not bn.affine or not bn.track_running_stats:
                refuse("an affine BatchNorm1d with running statistics after every conv")
            if bn.momentum is None:
                refuse("a BatchNorm momentum (momentum=None, the cumulative average, is not covered)")
        return plan.forward_train(voxel_features.contiguous(), coors.contiguous(), batch_size,
                                  n_voxels_dev=num_voxels, overlap_rulebooks=self.overlap_rulebooks)

    def _forward_fp16(self, voxel_features, coors, batch_size, fused, out, num_voxels):
        """precision=PREC_FP16: the fp16 plan, or a ValueError before anything runs."""
        if self.training:
            if num_voxels is None:
                raise ValueError("fp16 training runs the native training plan: pass num_voxels= (device int32[1])")
            return self._forward_train_native(voxel_features, coors, batch_size, num_voxels, sp_ops.PREC_FP16, out)
        if not fused:
            raise ValueError("the fp16 precision runs on the native plan only (no per-conv path): fused must not be False")
        if torch.is_grad_enabled():
            raise ValueError("fp16 in eval mode runs the native plan under torch.no_grad() only")
        if voxel_features.dtype not in (torch.float32, torch.float16):
            raise ValueError("the fp16 plan takes fp32 or fp16 features")
        plan = self.plan(sp_ops.PREC_FP16)
        if plan is None:
            raise ValueError("the fp16 precision needs a chain of (conv, norm, act) modules with tensor-core channel "
                             "counts")
        if out is not None and out.dtype != torch.float16:
            raise ValueError("out= of an fp16 forward must be half")
        return plan.forward(voxel_features.to(torch.float16).contiguous(), coors.contiguous(), batch_size,
                            n_voxels_dev=num_voxels, out=out, overlap_rulebooks=self.overlap_rulebooks)

    def _forward_int8(self, voxel_features, coors, batch_size, fused, out, num_voxels):
        """precision=PREC_INT8: the int8 plan, or a ValueError before anything runs."""
        if self.training:
            raise ValueError("the int8 precision runs in eval mode only (there is no int8 training)")
        if not fused:
            raise ValueError("the int8 precision runs on the native plan only (no per-conv path): fused must not be False")
        if torch.is_grad_enabled():
            raise ValueError("the int8 precision runs under torch.no_grad() only")
        if voxel_features.dtype not in (torch.float32, torch.float16):
            raise ValueError("the int8 plan takes fp32 or fp16 features")
        plan = self.plan(sp_ops.PREC_INT8) if self.plan() is not None and self._relu_chain() else None
        if plan is None:
            raise ValueError("the int8 precision needs a chain of (conv, norm, act) modules with tensor-core channel "
                             "counts and a ReLU after every conv")
        if self._int8_scales is None:
            raise ValueError("the int8 precision needs calibrated scales: call calibrate_int8() or set_int8_scales()")
        if out is not None and out.dtype != torch.float16:
            raise ValueError("out= of an int8 forward must be half")
        return plan.forward(voxel_features.to(torch.float16).contiguous(), coors.contiguous(), batch_size,
                            n_voxels_dev=num_voxels, out=out, overlap_rulebooks=self.overlap_rulebooks)

    def _relu_chain(self):
        from .encoder_plan import _chain_of
        return all(relu for _, _, relu, _ in _chain_of(self))

    def calibrate_int8(self, batches):
        """Sets the int8 plan's per-conv output scales from an fp32 eval pass of the per-conv path (bf16x3, folded
        BN) over `batches`, an iterable of (voxel_features, coors, batch_size): s_i = fl(amax_i / 255), amax_i the
        largest output of chain conv i (after its residual and ReLU) over all batches, or 1 when that is 0.
        Returns the scales (float32 [n_convs], on the host)."""
        from .encoder_plan import _chain_of, supported
        if not supported(self) or not self._relu_chain():
            raise ValueError("int8 calibration needs a chain the int8 plan runs (ReLU after every conv)")
        chain = _chain_of(self)
        amax = torch.zeros(len(chain), dtype=torch.float64)
        n = 0
        with torch.no_grad():
            for voxel_features, coors, batch_size in batches:
                x = spconv.SparseConvTensor(voxel_features.float().contiguous(), coors.int().contiguous(),
                                            self.sparse_shape, batch_size)
                outs = []
                for conv, bn, relu, res in chain:
                    s, t = bn_scale_shift(bn) if bn is not None else (None, None)
                    x = conv(x, scale=s, shift=t, residual=outs[res].features if res >= 0 else None, relu=relu,
                             precision=sp_ops.PREC_BF16X3)
                    outs.append(x)
                m = torch.stack([o.features.max() if o.features.numel() else o.features.new_zeros(())
                                 for o in outs]).double().cpu()
                amax = torch.maximum(amax, m)
                n += 1
        if n == 0:
            raise ValueError("calibrate_int8 needs at least one batch")
        amax32 = amax.float()
        scales = torch.where(amax32 > 0, amax32 / 255.0, torch.ones_like(amax32))   # fp32 division: fl(amax / 255)
        self.set_int8_scales(scales)
        return self.int8_scales()

    def int8_scales(self):
        """The int8 plan's per-conv output scales (float32 [n_convs], host), or None before calibration."""
        return None if self._int8_scales is None else self._int8_scales.clone()

    def set_int8_scales(self, scales):
        """Restores scales saved from int8_scales(): one finite, positive value per chain conv."""
        from .encoder_plan import _chain_of
        t = torch.as_tensor(scales).detach().to("cpu", torch.float32).flatten().clone()
        if t.numel() != len(_chain_of(self)):
            raise ValueError("int8 scales: %d values for %d convs" % (t.numel(), len(_chain_of(self))))
        if not bool((torch.isfinite(t) & (t > 0)).all()):
            raise ValueError("int8 scales must be finite and > 0")
        self._int8_scales = t

    @staticmethod
    def _convmodule_fused(seq, x, precision):
        conv, bn = seq[0], seq[1]
        s, t = bn_scale_shift(bn)
        return conv(x, scale=s, shift=t, relu=True, precision=precision)

    def _conv_sequence(self):
        """the SparseConvolution modules in execution order (sparse_encoder.py:113-124)"""
        seq = [self.conv_input[0]]
        for stage in self.encoder_layers:
            for block in stage:
                seq += [block.conv1, block.conv2] if isinstance(block, SparseBasicBlock) else [block[0]]
        seq.append(self.conv_out[0])
        return seq

    def _forward_fused(self, x, precision, dense_out=None):
        ahead = None
        seq = self._conv_sequence()
        strided = [i for i, cv in enumerate(seq) if not cv.subm]
        if self.overlap_rulebooks:
            # rulebooks on a side stream (see SparseConvolution._rulebook): their kernels and the
            # host waits for the strided convs' output counts hide behind the queued convolutions
            dev = x.features.device
            streams = self.__dict__.setdefault("_rulebook_streams", {})   # per module, not a package global
            side = streams.get(dev)
            if side is None:
                side = streams[dev] = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))    # the voxel coordinates are ready
            x.indice_dict["__rulebook_stream__"] = side
            if self.rulebook_lookahead:
                # ... and AHEAD of need: a rulebook is a function of the voxel indices alone, so as soon
                # as three convs of a stage are queued, the rulebook of the strided conv that closes the
                # stage is built behind them.  tools/encoder_timeline.py showed the main stream idle for
                # 145 us before the first strided conv and 64 us before the second; with the look-ahead
                # the frame rate moved from 285.2 to 286.8 frames/s on the same box -- the idle time is
                # mostly contention of the rulebook kernels with the running convs, not the host wait.
                cur = {"indices": x.indices, "shape": x.spatial_shape, "next": 0}

                def ahead(upto):
                    while cur["next"] <= min(upto, len(seq) - 1):
                        cv = seq[cur["next"]]
                        stub = spconv.SparseConvTensor(None, cur["indices"], cur["shape"], x.batch_size)
                        stub.indice_dict = x.indice_dict
                        rb, out_shape = cv._rulebook(stub)
                        if not cv.subm:
                            cur["indices"], cur["shape"] = rb.outids, out_shape
                        cur["next"] += 1

        def next_strided(pos):
            return next((i for i in strided if i >= pos), len(seq) - 1)

        pos, queued = 0, 0      # next conv to run; convs queued since the last strided conv
        blocks = [self.conv_input] + [b for stage in self.encoder_layers for b in stage] + [self.conv_out]
        for block in blocks:
            n_convs = 2 if isinstance(block, SparseBasicBlock) else 1
            if ahead:
                ahead(pos + n_convs - 1)                      # what this block needs right now
            if isinstance(block, SparseBasicBlock):
                x = block.forward_fused(x, precision)
            else:
                x = self._convmodule_fused(block, x, precision)
            closes_stage = ahead is not None and pos + n_convs - 1 in strided
            pos += n_convs
            queued = 1 if closes_stage else queued + n_convs
            if ahead and queued >= 3:
                ahead(next_strided(pos))                      # the rest, hidden behind >= 3 queued convs
        out = x
        if out.features.dtype != torch.float32:
            # half features (the native plan takes fp32 only): each conv above widened and narrowed its
            # own rows; the scatter runs on widened rows and the output keeps the features' dtype
            dense = sp_ops.sparse_to_dense(out.features.float(), out.indices, int(out.batch_size),
                                           out.spatial_shape, z_major=True)
            return dense.to(out.features.dtype) if dense_out is None else dense_out.copy_(dense)
        # dense() + permute(0,1,4,2,3) + view(N, C*D, H, W) in one kernel
        return sp_ops.sparse_to_dense(out.features, out.indices, int(out.batch_size),
                                      out.spatial_shape, z_major=True, out=dense_out)

    def make_encoder_layers(self, make_block, norm_cfg, in_channels, block_type="conv_module",
                            conv_cfg=dict(type="SubMConv3d")):
        """sparse_encoder.py:134-217."""
        assert block_type in ["conv_module", "basicblock"]
        self.encoder_layers = spconv.SparseSequential()
        for i, blocks in enumerate(self.encoder_channels):
            blocks_list = []
            for j, out_channels in enumerate(tuple(blocks)):
                padding = tuple(self.encoder_paddings[i])[j]
                if i != 0 and j == 0 and block_type == "conv_module":
                    blocks_list.append(make_block(in_channels, out_channels, 3, norm_cfg=norm_cfg,
                                                  stride=2, padding=padding,
                                                  indice_key=f"spconv{i + 1}",
                                                  conv_type="SparseConv3d"))
                elif block_type == "basicblock":
                    if j == len(blocks) - 1 and i != len(self.encoder_channels) - 1:
                        blocks_list.append(make_block(in_channels, out_channels, 3,
                                                      norm_cfg=norm_cfg, stride=2, padding=padding,
                                                      indice_key=f"spconv{i + 1}",
                                                      conv_type="SparseConv3d"))
                    else:
                        blocks_list.append(SparseBasicBlock(out_channels, out_channels,
                                                            norm_cfg=norm_cfg, conv_cfg=conv_cfg))
                else:
                    blocks_list.append(make_block(in_channels, out_channels, 3, norm_cfg=norm_cfg,
                                                  padding=padding, indice_key=f"subm{i + 1}",
                                                  conv_type="SubMConv3d"))
                in_channels = out_channels
            stage_name = f"encoder_layer{i + 1}"
            self.encoder_layers.add_module(stage_name, spconv.SparseSequential(*blocks_list))
        return out_channels


def voxelnet_0p075_encoder():
    """SparseEncoder as configured by configs/nuscenes/det/transfusion/secfpn/lidar/voxelnet_0p075.yaml."""
    return SparseEncoder(in_channels=5, sparse_shape=[1440, 1440, 41], output_channels=128,
                         order=("conv", "norm", "act"),
                         encoder_channels=((16, 16, 32), (32, 32, 64), (64, 64, 128), (128, 128)),
                         encoder_paddings=((0, 0, 1), (0, 0, 1), (0, 0, (1, 1, 0)), (0, 0)),
                         block_type="basicblock")
