"""Generates tests/golden/pillars_train_tiny.npz: one training step of the REFERENCE's own pillar encoder
(mmdet3d/models/backbones/pillar_encoder.py, loaded with the stubs of make_pillars_golden.py), run in float64 on
the CPU under autograd with a seeded canvas gradient.  Writes only pillars_train_tiny.npz.

The input is make_pillars_golden's: batch 2 on a 16 x 12 grid, P 20, every count 1..P and several n == P
pillars, some negative BN scales.  Cases (prefix in the file):
  A     the shipped config, random BN parameters
  beta  a large layer-1 shift, so the padded row wins the layer-1 max for some channels
  zero  a layer-1 channel that is zero after ReLU on every slot (ties at 0)
Each records the state_dict before the step, the canvas, the gradients of both linear weights and both BN
weights / biases, and the running statistics and num_batches_tracked after the step.

Run:  python tests/golden/make_pillars_train_golden.py      (needs the reference tree)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_pillars_golden import load_reference_module, make_pillars, randomize  # noqa: E402


def gen():
    ns = load_reference_module()
    torch.manual_seed(0)
    rng = np.random.default_rng(11)
    P, F, nx, ny, batch = 20, 5, 16, 12, 2
    vs = [0.2, 0.2, 8.0]
    pcr = [-1.6, -1.2, -5.0, 1.6, 1.2, 3.0]
    norm_cfg = dict(type="BN1d", eps=1e-3, momentum=0.01)
    feats, num, coors = make_pillars(rng, P, F, nx, ny, batch, vs, pcr, 96)
    out = dict(features=feats, num_voxels=num, coors=coors, P=P, F=F, nx=nx, ny=ny, batch=batch,
               voxel_size=np.array(vs), point_cloud_range=np.array(pcr))
    gcan = rng.standard_normal((batch, 64, nx, ny))
    out["grad_canvas"] = gcan
    for name in ("A", "beta", "zero"):
        enc = ns["PointPillarsEncoder"](
            dict(type="PillarFeatureNet", in_channels=F, voxel_size=vs, point_cloud_range=pcr, norm_cfg=norm_cfg,
                 feat_channels=[64, 64], with_distance=False),
            dict(type="PointPillarsScatter", in_channels=64, output_shape=[nx, ny])).double()
        net = enc.pts_voxel_encoder
        randomize(net, rng)
        bn1 = net.pfn_layers[0].norm
        if name == "beta":
            bn1.bias.data += 1.5
        if name == "zero":
            bn1.weight.data[3] = 0.5
            bn1.bias.data[3] = -50.0
        sd = {k: v.detach().clone().numpy() for k, v in enc.state_dict().items()}
        for k, v in sd.items():
            out["%s__sd__%s" % (name, k)] = v
        out["%s__sd_keys" % name] = np.array(list(sd))
        enc.train()
        canvas = enc(torch.from_numpy(feats), torch.from_numpy(coors), torch.tensor(batch), torch.from_numpy(num))
        (canvas * torch.from_numpy(gcan)).sum().backward()
        out[name + "__canvas"] = canvas.detach().numpy()
        for i, layer in enumerate(net.pfn_layers):
            out["%s__dW%d" % (name, i + 1)] = layer.linear.weight.grad.numpy()
            out["%s__dg%d" % (name, i + 1)] = layer.norm.weight.grad.numpy()
            out["%s__db%d" % (name, i + 1)] = layer.norm.bias.grad.numpy()
            out["%s__rm%d" % (name, i + 1)] = layer.norm.running_mean.numpy().copy()
            out["%s__rv%d" % (name, i + 1)] = layer.norm.running_var.numpy().copy()
            out["%s__nbt%d" % (name, i + 1)] = int(layer.norm.num_batches_tracked)
    np.savez_compressed(os.path.join(HERE, "pillars_train_tiny.npz"), **out)


if __name__ == "__main__":
    gen()
