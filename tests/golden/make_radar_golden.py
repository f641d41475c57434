"""Generates tests/golden/radar_tiny.npz from the REFERENCE's own radar encoder source
(mmdet3d/models/backbones/radar_encoder.py), executed in float64 on the CPU with stubs for the modules it
imports but the encoder does not use (mmcv.cnn, mmcv.cnn.resnet, mmcv.cnn.bricks.non_local,
mmdet.models.BACKBONES, mmdet3d.models.builder, mmdet3d.ops.feature_decorator, torchvision.utils,
flash_attn.flash_attention).  Writes only radar_tiny.npz.

The [M, P, F] input is built directly: counts cover 1..P including several n == P, padded slots are zero,
each pillar's points lie in its pillar, the other columns look like radar_use_dims (rcs, velocities, time,
one-hot blocks).  BN weights and running statistics are random, with some negative scales.  The reference
normalises xyz in its input tensor, so it gets a clone.

  A  the shipped config: in_channels 45, feat_channels [128, 128, 128, 64], P 20, voxel (0.8, 0.8, 8) on a
     16 x 12 grid, batch 2; eval and train-mode outputs, running statistics after the train step, the scatter
  B  in_channels 18 (the first 18 columns), feat_channels [128, 64]; eval and train-mode outputs

Run:  python tests/golden/make_radar_golden.py      (needs the reference tree)
"""
import os
import sys
import types

import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("BEVFUSION_REFERENCE", "/root/reference")


def load_reference_module():
    def build_norm_layer(cfg, num_features):
        cfg = dict(cfg)
        assert cfg.pop("type") == "BN1d"
        return "bn", nn.BatchNorm1d(num_features, **cfg)

    def unused(*args, **kwargs):
        raise AssertionError("not used by the radar encoder")

    class Registry:
        def __init__(self):
            self.modules = {}

        def register_module(self):
            def deco(cls):
                self.modules[cls.__name__] = cls
                return cls
            return deco

    backbones = Registry()

    def build_backbone(cfg):
        cfg = dict(cfg)
        return backbones.modules[cfg.pop("type")](**cfg)

    stubs = {"mmcv": {}, "mmcv.cnn": {"build_conv_layer": unused, "build_norm_layer": build_norm_layer},
             "mmcv.cnn.resnet": {"make_res_layer": unused, "BasicBlock": object},
             "mmcv.cnn.bricks": {}, "mmcv.cnn.bricks.non_local": {"NonLocal2d": object},
             "mmdet": {}, "mmdet.models": {"BACKBONES": backbones}, "mmdet3d": {}, "mmdet3d.models": {},
             "mmdet3d.models.builder": {"build_backbone": build_backbone},
             "mmdet3d.ops": {"feature_decorator": unused},
             "torchvision": {}, "torchvision.utils": {"save_image": unused},
             "flash_attn": {}, "flash_attn.flash_attention": {"FlashMHA": object}}
    saved = {k: sys.modules.get(k) for k in stubs}
    for name, attrs in stubs.items():
        mod = types.ModuleType(name)
        mod.__dict__.update(attrs)
        sys.modules[name] = mod
    try:
        path = os.path.join(REF, "mmdet3d", "models", "backbones", "radar_encoder.py")
        ns = {"__name__": "reference_radar_encoder"}
        exec(compile(open(path).read(), path, "exec"), ns)
        # the scatter the radar config uses registers from the reference's pillar encoder
        ppath = os.path.join(REF, "mmdet3d", "models", "backbones", "pillar_encoder.py")
        pns = {"__name__": "reference_pillar_encoder"}
        exec(compile(open(ppath).read(), ppath, "exec"), pns)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return ns


def randomize(net, rng):
    for layer in net.rfn_layers:
        w = layer.linear.weight
        w.data = torch.from_numpy(rng.standard_normal(tuple(w.shape)) / np.sqrt(w.shape[1]))
        bn, u = layer.norm, layer.units
        sign = np.where(rng.uniform(size=u) < 0.25, -1.0, 1.0)
        bn.weight.data = torch.from_numpy(sign * rng.uniform(0.5, 1.5, size=u))
        bn.bias.data = torch.from_numpy(rng.uniform(-0.5, 0.5, size=u))
        bn.running_mean.data = torch.from_numpy(rng.uniform(-0.3, 0.3, size=u))
        bn.running_var.data = torch.from_numpy(rng.uniform(0.5, 2.0, size=u))


def make_pillars(rng, P, F, nx, ny, batch, vs, lo, count):
    cells = rng.permutation(batch * nx * ny)[:count]
    coors = np.stack([cells // (nx * ny), (cells // ny) % nx, cells % ny, np.zeros_like(cells)], 1).astype(np.int32)
    num = rng.integers(1, P + 1, size=count).astype(np.int32)
    num[:P] = np.arange(1, P + 1)          # every count 1..P
    num[P:P + 4] = P                       # and several full pillars
    feats = np.zeros((count, P, F))
    for v in range(count):
        k = num[v]
        feats[v, :k, 0] = lo[0] + (coors[v, 1] + rng.uniform(size=k)) * vs[0]
        feats[v, :k, 1] = lo[1] + (coors[v, 2] + rng.uniform(size=k)) * vs[1]
        feats[v, :k, 2] = rng.uniform(lo[2], lo[2] + vs[2], size=k)
        feats[v, :k, 3] = rng.uniform(-10, 40, size=k)                # rcs
        feats[v, :k, 4:6] = rng.normal(0, 3, size=(k, 2))             # compensated velocity
        feats[v, :k, 6] = rng.choice([0.0, 0.05, 0.1, 0.25], size=k)  # time_diff
        feats[v, :k, 7:] = (rng.uniform(size=(k, F - 7)) < 0.2).astype(np.float64)  # one-hot / ordinal blocks
    return feats, num, coors


def gen_radar():
    ns = load_reference_module()
    torch.manual_seed(0)
    rng = np.random.default_rng(11)
    P, F, nx, ny, batch = 20, 45, 16, 12, 2
    vs = [0.8, 0.8, 8.0]
    pcr = [-6.4, -4.8, -5.0, 6.4, 4.8, 3.0]
    norm_cfg = dict(type="BN1d", eps=1e-3, momentum=0.01)
    feats, num, coors = make_pillars(rng, P, F, nx, ny, batch, vs, pcr, 96)
    feats = feats.astype(np.float32)       # what an fp32 caller holds; the reference runs on it in float64
    out = dict(features=feats, num_voxels=num, coors=coors, P=P, F=F, nx=nx, ny=ny, batch=batch,
               voxel_size=np.array(vs), point_cloud_range=np.array(pcr), B__in_channels=18)
    configs = {"A": dict(in_channels=45, feat_channels=[128, 128, 128, 64]),
               "B": dict(in_channels=18, feat_channels=[128, 64])}
    for name, cfg in configs.items():
        enc = ns["RadarEncoder"](
            dict(type="RadarFeatureNet", with_distance=False, voxel_size=vs, point_cloud_range=pcr,
                 norm_cfg=norm_cfg, **cfg),
            dict(type="PointPillarsScatter", in_channels=64, output_shape=[nx, ny])).double()
        randomize(enc.pts_voxel_encoder, rng)
        sd = {k: v.detach().clone().numpy() for k, v in enc.state_dict().items()}
        for k, v in sd.items():
            out["%s__sd__%s" % (name, k)] = v
        out["%s__sd_keys" % name] = np.array(list(sd))
        x = torch.from_numpy(np.ascontiguousarray(feats[:, :, :cfg["in_channels"]], np.float64))
        n, c = torch.from_numpy(num), torch.from_numpy(coors)
        enc.eval()
        with torch.no_grad():
            out[name + "__eval"] = enc.pts_voxel_encoder(x.clone(), n, c).numpy()
            if name == "A":
                out[name + "__canvas"] = enc(x.clone(), c, torch.tensor(batch), n).numpy()
        enc.train()
        with torch.no_grad():
            out[name + "__train"] = enc.pts_voxel_encoder(x.clone(), n, c).numpy()
        for i, layer in enumerate(enc.pts_voxel_encoder.rfn_layers):
            out["%s__train_running_mean%d" % (name, i)] = layer.norm.running_mean.numpy().copy()
            out["%s__train_running_var%d" % (name, i)] = layer.norm.running_var.numpy().copy()
    np.savez_compressed(os.path.join(HERE, "radar_tiny.npz"), **out)


if __name__ == "__main__":
    gen_radar()
