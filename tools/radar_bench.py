"""Radar encoder of the camera+radar config (camera+radar/default.yaml: voxel 0.8 x 0.8 x 8, range +-51.2 / -5..3,
P 20, in_channels 45, feat_channels [128, 128, 128, 64]) on synthetic.radar_cloud, batch 1 and batch 4:

    python tools/radar_bench.py OUT_DIR [--window 1.0]

(a) fused:  RadarEncoder.forward_points: voxelizer front + radar kernel straight into the canvas
(b) native: voxelize_batch (hard voxelization, [M, P, F]) -> native RadarFeatureNet -> PointPillarsScatter
(c) torch:  the same voxelization -> the torch restatement of the reference RadarFeatureNet -> the reference's
            scatter (zeroed canvas, index assignment), as mmdet3d runs it
Reports CUDA-event times over windows of at least --window seconds after a warm-up (three alternating rounds, the
median is reported): eager calls, and (a) and the rows form of the radar net on the [M, P, F] tensor ("kernel":
memsets, table, tiles) also as 20 calls in one CUDA graph, which is their device time; then a torch.profiler pass
gives each kernel's device time per call.  Also M, R (real rows evaluated), FLOPs
from shapes, the largest error of (a) and (b) against (c) and against the float64 oracle, and the card name / power
limit read in the same run.  Writes OUT_DIR/radar_bench.json.  Needs a CUDA device: there is no CPU path."""
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
from bevfusion_b200.radar_encoder import RadarEncoder  # noqa: E402
from bevfusion_b200.voxelize import Voxelization, voxelize_batch  # noqa: E402
from radar_oracle import layers_from_state_dict, radar_feature_net, radar_scatter  # noqa: E402

VS, PCR, P, NX, NY = [0.8, 0.8, 8.0], [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], 20, 128, 128
FEAT = [128, 128, 128, 64]


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


def graph_ms(fn, window_s, reps=20):
    """device time of one fn() call: `reps` calls captured in one CUDA graph, replays timed with timed_ms (the
    eager loop of a call this small measures the host, not the GPU)"""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    return timed_ms(g.replay, window_s) / reps


def kernel_us(fn, calls=20):
    """mean device time per fn() call of each kernel / memset, from torch.profiler in a pass of its own"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            out[e.key[:80]] = t / calls
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def make_encoder(dev):
    enc = RadarEncoder(
        dict(type="RadarFeatureNet", in_channels=45, feat_channels=FEAT, with_distance=False, voxel_size=VS,
             point_cloud_range=PCR, norm_cfg=dict(type="BN1d", eps=1e-3, momentum=0.01)),
        dict(type="PointPillarsScatter", in_channels=64, output_shape=[NX, NY]))
    g = torch.Generator().manual_seed(0)
    for layer in enc.pts_voxel_encoder.rfn_layers:
        bn, u = layer.norm, layer.units
        bn.weight.data = torch.where(torch.rand(u, generator=g) < 0.25, -1.0, 1.0) * (0.5 + torch.rand(u, generator=g))
        bn.bias.data = torch.rand(u, generator=g) - 0.5
        bn.running_mean.data = 0.6 * torch.rand(u, generator=g) - 0.3
        bn.running_var.data = 0.5 + 1.5 * torch.rand(u, generator=g)
    return enc.to(dev).eval()


def reference_scatter(voxel_features, coords, batch_size, c):
    """pillar_encoder.py PointPillarsScatter as the reference runs it"""
    canvases = []
    for b in range(batch_size):
        canvas = torch.zeros(c, NX * NY, dtype=voxel_features.dtype, device=voxel_features.device)
        m = coords[:, 0] == b
        this = coords[m, :]
        idx = (this[:, 1] * NY + this[:, 2]).long()
        canvas[:, idx] = voxel_features[m, :].t()
        canvases.append(canvas)
    return torch.stack(canvases, 0).view(batch_size, c, NX, NY)


def run_batch(enc, vox, clouds, window):
    net = enc.pts_voxel_encoder
    B = len(clouds)

    def run_a():
        return enc.forward_points(clouds, vox)

    def run_b():
        feats, coords, sizes = voxelize_batch(clouds, vox, voxelize_reduce=False)
        return enc(feats, coords, B, sizes)

    def run_c():
        feats, coords, sizes = voxelize_batch(clouds, vox, voxelize_reduce=False)
        return reference_scatter(net._forward_torch(feats, sizes, coords), coords, B, 64)

    with torch.no_grad():
        feats, coords, sizes = voxelize_batch(clouds, vox, voxelize_reduce=False)

        def run_kernel():
            return net._forward_native(feats, sizes, coords)

        outs = {k: f() for k, f in (("a", run_a), ("b", run_b), ("c", run_c))}
        for f in (run_a, run_b, run_c, run_kernel):          # warm-up
            for _ in range(3):
                f()
        torch.cuda.synchronize()
        rounds = {k: [] for k in ("a", "b", "c", "kernel", "a_graph", "kernel_graph")}
        for _ in range(3):
            for k, f in (("a", run_a), ("b", run_b), ("c", run_c), ("kernel", run_kernel)):
                rounds[k].append(timed_ms(f, window))
            rounds["a_graph"].append(graph_ms(run_a, window))
            rounds["kernel_graph"].append(graph_ms(run_kernel, window))
        profile_a, profile_kernel = kernel_us(run_a), kernel_us(run_kernel)
    n = sizes.cpu().numpy()
    M = int(n.shape[0])
    R = int(np.minimum(n, P).sum())
    sd = {k: v.detach().double().cpu().numpy() for k, v in net.state_dict().items()}
    rows64, _ = radar_feature_net(feats.cpu().numpy(), n, coords.cpu().numpy(), layers_from_state_dict(sd, "", 4),
                                  net.vx, net.vy, net.x_offset, net.y_offset, net.pc_range)
    gold = radar_scatter(rows64, coords.cpu().numpy(), B, NX, NY)
    ref_c = outs["c"].double().cpu().numpy()

    def err(x, g):
        return float(np.abs(x.double().cpu().numpy() - g).max() / np.abs(g).max())

    macs = 47 * 128 + 2 * 128 * 128 + 128 * 64
    flops = 2 * R * macs                                      # useful: real rows only (the virtual row is packed)
    issued = 3 * 2 * 16 * ((R + 15) // 16) * (48 * 128 + 2 * 128 * 128 + 128 * 64)  # BF16x3, 16-row tiles
    result = {
        "batch": B, "points": [int(p.shape[0]) for p in clouds],
        "M": M, "R": R, "pillars_full": int((n == P).sum()),
        "flops_useful": flops, "flops_issued_bf16x3": issued,
        "ms": {k: statistics.median(v) for k, v in rounds.items()},
        "ms_rounds": rounds,
        "max_rel_err": {"a_vs_c": err(outs["a"], ref_c), "b_vs_c": err(outs["b"], ref_c),
                        "a_vs_oracle": err(outs["a"], gold), "b_vs_oracle": err(outs["b"], gold),
                        "c_vs_oracle": err(outs["c"], gold)},
        "a_equals_b": bool(torch.equal(outs["a"], outs["b"])),
        "profile_us_per_call": {"a": profile_a, "kernel": profile_kernel},
    }
    k = result["ms"]["kernel_graph"] * 1e-3
    result["kernel_rate"] = {"useful_tflop_per_s": flops / k / 1e12, "issued_tflop_per_s": issued / k / 1e12}
    return result


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
    vox = Voxelization(VS, PCR, P, (30000, 60000)).eval()
    clouds = [torch.from_numpy(S.radar_cloud(seed=s)).to(dev) for s in range(4)]
    result = {"card": card,
              "config": {"voxel_size": VS, "point_cloud_range": PCR, "max_points": P, "in_channels": 45,
                         "feat_channels": FEAT, "cloud": "synthetic.radar_cloud(seed=0..3)"},
              "batch1": run_batch(enc, vox, clouds[:1], args.window),
              "batch4": run_batch(enc, vox, clouds, args.window)}
    with open(os.path.join(args.out_dir, "radar_bench.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({k: {"ms": result[k]["ms"], "M": result[k]["M"], "R": result[k]["R"],
                          "err": result[k]["max_rel_err"]} for k in ("batch1", "batch4")} | {"card": card}))


if __name__ == "__main__":
    main()
