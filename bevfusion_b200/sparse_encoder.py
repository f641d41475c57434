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
        self.rulebook_lookahead = os.environ.get("BEVB200_RULEBOOK_LOOKAHEAD", "1") != "0"
        self.conv_out = make_sparse_convmodule(encoder_out_channels, self.output_channels,
                                               kernel_size=(1, 1, 3), stride=(1, 1, 2),
                                               norm_cfg=norm_cfg, padding=0,
                                               indice_key="spconv_down2", conv_type="SparseConv3d")

    def plan(self):
        """The native EncoderPlan of this module (built lazily), or None when a layer has no native form."""
        if self._plan is None:
            from . import encoder_plan
            self._plan = encoder_plan.EncoderPlan(self) if encoder_plan.supported(self) else False
        return self._plan or None

    def forward(self, voxel_features, coors, batch_size, fused=None, precision=None, out=None,
                num_voxels=None, **kwargs):
        """sparse_encoder.py:99-132.  voxel_features [N, C] fp32 or fp16, coors [N, 4] int32
        (batch, x, y, z).  Returns spatial features [B, C*D, H, W], in half when the features or the
        conv weights are (each conv computes in fp32 and narrows its output once).

        fused=None picks the fused path (BN / ReLU / residual in the conv epilogues, dense()
        written directly in the output layout) whenever the module is in eval mode.  `out`
        (fused path) is an optional [B, C*D, H, W] view to write into, e.g. the LiDAR channels
        of the fuser's concatenated input (fusers/conv.py:16)."""
        coors = coors.int()
        if fused is None:
            fused = not self.training and self.order == ("conv", "norm", "act")
        if precision is None:
            precision = sp_ops.default_precision()
        if (fused and self.native_plan and precision == sp_ops.PREC_BF16X3 and not torch.is_grad_enabled()
                and voxel_features.dtype == torch.float32 and self.conv_input[0].weight.dtype == torch.float32
                and self.plan() is not None):
            # `num_voxels` (device int32[1]): only the first rows are valid -- no host round trip
            return self.plan().forward(voxel_features.contiguous(), coors.contiguous(), batch_size,
                                       n_voxels_dev=num_voxels, out=out, overlap_rulebooks=self.overlap_rulebooks)
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
