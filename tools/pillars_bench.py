"""PointPillars LiDAR encoder on the shipped config (pointpillars.yaml: voxel 0.2 x 0.2 x 8, range +-51.2 /
-5..3, P 20, feat_channels [64, 64]) and synthetic.lidar_cloud, batch 1:

    python tools/pillars_bench.py OUT_DIR [--window 1.0]

(a) fused:  PointPillarsEncoder.forward_points: voxelizer front + pillar kernel straight into the canvas
(b) native: voxelize_batch (hard voxelization, [M, P, F]) -> native PillarFeatureNet -> PointPillarsScatter
(c) torch:  the same voxelization -> the torch restatement of the reference PillarFeatureNet -> the
            reference's scatter (zeroed canvas, index assignment), as mmdet3d runs it
Reports CUDA-event times over windows of at least --window seconds after a warm-up (three alternating rounds, the
median is reported), the pillar kernel alone on the [M, P, F] tensor, M, R (rows the net evaluates: kept points
plus one padded row per pillar with n < P), algorithmic bytes and FLOPs from shapes, the largest error of (a) and
(b) against (c) and against the float64 oracle, and the card name / power limit read in the same run.  Writes
OUT_DIR/pillars_bench.json.  Needs a CUDA device: there is no CPU path."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200.pillar_encoder import PointPillarsEncoder  # noqa: E402
from bevfusion_b200.voxelize import Voxelization, voxelize_batch  # noqa: E402
from pillars_oracle import layers_from_state_dict, pillar_feature_net, pillars_scatter  # noqa: E402

VS, PCR, P, NX, NY = [0.2, 0.2, 8.0], [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], 20, 512, 512


def card_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (v.strip() for v in q.split(","))
    return {"name": name, "power_limit": power, "clocks_max_sm": clock}


def timed_ms(fn, window_s):
    """mean CUDA-event time of fn() over a window of at least window_s seconds (after the caller's warm-up)."""
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    one = max(start.elapsed_time(stop), 1e-3)
    n = max(10, int(window_s * 1e3 / one) + 1)
    start.record()
    for _ in range(n):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / n


def make_encoder(dev):
    enc = PointPillarsEncoder(
        dict(type="PillarFeatureNet", in_channels=5, feat_channels=[64, 64], with_distance=False, voxel_size=VS,
             point_cloud_range=PCR, norm_cfg=dict(type="BN1d", eps=1e-3, momentum=0.01)),
        dict(type="PointPillarsScatter", in_channels=64, output_shape=[NX, NY]))
    g = torch.Generator().manual_seed(0)
    for layer in enc.pts_voxel_encoder.pfn_layers:
        bn, u = layer.norm, layer.units
        bn.weight.data = torch.where(torch.rand(u, generator=g) < 0.25, -1.0, 1.0) * (0.5 + torch.rand(u, generator=g))
        bn.bias.data = torch.rand(u, generator=g) - 0.5
        bn.running_mean.data = 0.6 * torch.rand(u, generator=g) - 0.3
        bn.running_var.data = 0.5 + 1.5 * torch.rand(u, generator=g)
    return enc.to(dev).eval()


def reference_scatter(voxel_features, coords, batch_size, c):
    """pillar_encoder.py:203-237 as the reference runs it"""
    canvases = []
    for b in range(batch_size):
        canvas = torch.zeros(c, NX * NY, dtype=voxel_features.dtype, device=voxel_features.device)
        m = coords[:, 0] == b
        this = coords[m, :]
        idx = (this[:, 1] * NY + this[:, 2]).long()
        canvas[:, idx] = voxel_features[m, :].t()
        canvases.append(canvas)
    return torch.stack(canvases, 0).view(batch_size, c, NX, NY)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--window", type=float, default=1.0)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = card_info()
    enc = make_encoder(dev)
    net = enc.pts_voxel_encoder
    vox = Voxelization(VS, PCR, P, (30000, 60000)).eval()
    pts = torch.from_numpy(S.lidar_cloud(seed=0)).to(dev)

    def run_a():
        return enc.forward_points([pts], vox)

    def run_b():
        feats, coords, sizes = voxelize_batch([pts], vox, voxelize_reduce=False)
        return enc(feats, coords, 1, sizes)

    def run_c():
        feats, coords, sizes = voxelize_batch([pts], vox, voxelize_reduce=False)
        return reference_scatter(net._forward_torch(feats, sizes, coords), coords, 1, 64)

    with torch.no_grad():
        feats, coords, sizes = voxelize_batch([pts], vox, voxelize_reduce=False)

        def run_kernel():
            return net._forward_native(feats, sizes, coords)

        outs = {k: f() for k, f in (("a", run_a), ("b", run_b), ("c", run_c))}
        for f in (run_a, run_b, run_c, run_kernel):          # warm-up
            for _ in range(3):
                f()
        torch.cuda.synchronize()
        rounds = {k: [] for k in ("a", "b", "c", "kernel")}
        for _ in range(3):
            for k, f in (("a", run_a), ("b", run_b), ("c", run_c), ("kernel", run_kernel)):
                rounds[k].append(timed_ms(f, args.window))
    n = sizes.cpu().numpy()
    M, F_ = int(n.shape[0]), int(pts.shape[1])
    kept = int(np.minimum(n, P).sum())
    R = kept + int((n < P).sum())
    sd = {k: v.detach().double().cpu().numpy() for k, v in net.state_dict().items()}
    rows64, _ = pillar_feature_net(feats.cpu().numpy(), n, coords.cpu().numpy(), layers_from_state_dict(sd, "", 2),
                                   net.vx, net.vy, net.x_offset, net.y_offset)
    gold = pillars_scatter(rows64, coords.cpu().numpy(), 1, NX, NY)
    ref_c = outs["c"].double().cpu().numpy()

    def err(x, g):
        return float(np.abs(x.double().cpu().numpy() - g).max() / np.abs(g).max())

    flops = 2 * R * (F_ + 5) * 32 + 2 * R * 32 * 64 + 2 * M * 32 * 64
    canvas_bytes = 64 * NX * NY * 4
    result = {
        "card": card,
        "config": {"voxel_size": VS, "point_cloud_range": PCR, "max_points": P, "feat_channels": [64, 64],
                   "batch": 1, "cloud": "synthetic.lidar_cloud(seed=0)", "points": int(pts.shape[0])},
        "M": M, "R": R, "kept_points": kept, "pillars_full": int((n == P).sum()),
        "algorithmic": {
            "flops": flops,
            "pillar_kernel_bytes": M * P * F_ * 4 + M * 4 + M * 16 + M * 64 * 4,
            "fused_bytes": kept * (F_ * 4 + 4) + canvas_bytes + M * 64 * 4,
            "canvas_bytes": canvas_bytes,
        },
        "ms": {k: statistics.median(v) for k, v in rounds.items()},
        "ms_rounds": rounds,
        "max_rel_err": {"a_vs_c": err(outs["a"], ref_c), "b_vs_c": err(outs["b"], ref_c),
                        "a_vs_oracle": err(outs["a"], gold), "b_vs_oracle": err(outs["b"], gold),
                        "c_vs_oracle": err(outs["c"], gold)},
        "a_equals_b": bool(torch.equal(outs["a"], outs["b"])),
    }
    k = result["ms"]["kernel"] * 1e-3
    result["pillar_kernel_rate"] = {"gflop_per_s": flops / k / 1e9,
                                    "gbyte_per_s": result["algorithmic"]["pillar_kernel_bytes"] / k / 1e9}
    with open(os.path.join(args.out_dir, "pillars_bench.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({"ms": result["ms"], "M": M, "R": R, "err": result["max_rel_err"], "card": card}))


if __name__ == "__main__":
    main()
