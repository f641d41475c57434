"""Training step of the PointPillars pillar net + scatter: forward + backward of (canvas * R).sum().

    python tools/pillars_train_bench.py OUT_DIR [--iters 10] [--rounds 3] [--batches 1,4]

Input: synthetic.lidar_cloud per sample, hard-voxelized with the shipped config's training settings (voxel
0.2 x 0.2 x 8, P = 20, max_voxels[0] = 30000) outside the timed window.  Three ways, alternated per round, median
of the rounds:
  torch   the torch restatement (PointPillarsEncoder.forward without voxel_num=) on the valid pillars, eager
  native  PointPillarsEncoder.forward(..., voxel_num=) on the [B * 30000, P, F] segments, eager
  graph   the native step captured as one CUDA graph and replayed
Each row also gives the peak memory of the torch and native steps.  The card name and power limit are read in the
same run.  Writes OUT_DIR/pillars_train_bench.json.  Needs a CUDA device."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
from torch.nn import functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200.pillar_encoder import PointPillarsEncoder  # noqa: E402
from bevfusion_b200.voxelize import Voxelization  # noqa: E402

VS, PCR, P, CAP = [0.2, 0.2, 8.0], [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], 20, 30000


def encoder(dev):
    enc = PointPillarsEncoder(
        dict(type="PillarFeatureNet", in_channels=5, feat_channels=[64, 64], with_distance=False, voxel_size=VS,
             point_cloud_range=PCR, norm_cfg=dict(type="BN1d", eps=1e-3, momentum=0.01)),
        dict(type="PointPillarsScatter", in_channels=64, output_shape=[512, 512]))
    return enc.to(dev).train()


def inputs(B, dev):
    vox = Voxelization(VS, PCR, P, (CAP, 60000)).train()
    seg_v = torch.zeros((B * CAP, P, 5), device=dev)
    seg_n = torch.zeros(B * CAP, dtype=torch.int32, device=dev)
    seg_c = torch.zeros((B * CAP, 4), dtype=torch.int32, device=dev)
    n_dev, fs, cs, ns = [], [], [], []
    for b in range(B):
        v, c, n = vox(torch.from_numpy(S.lidar_cloud(seed=b)).to(dev))
        c4 = F.pad(c, (1, 0), value=b)
        m = v.shape[0]
        seg_v[b * CAP:b * CAP + m], seg_n[b * CAP:b * CAP + m], seg_c[b * CAP:b * CAP + m] = v, n, c4
        n_dev.append(m)
        fs.append(v), cs.append(c4), ns.append(n)
    return (seg_v, seg_c, seg_n, torch.tensor(n_dev, dtype=torch.int32, device=dev)), \
        (torch.cat(fs), torch.cat(cs), torch.cat(ns))


def timed(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def peak_of(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", default="1,4")
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print("card:", card, flush=True)
    results = {"card": card, "rows": []}
    for B in [int(b) for b in args.batches.split(",")]:
        torch.manual_seed(0)
        enc, ref = encoder(dev), encoder(dev)
        ref.load_state_dict(enc.state_dict())
        (sv, sc, sn, n_dev), (fv, fc, fn) = inputs(B, dev)
        R = torch.randn((B, 64, 512, 512), device=dev)

        def step_torch():
            ref(fv, fc, B, fn).mul(R).sum().backward()

        def step_native():
            enc(sv, sc, B, sn, voxel_num=n_dev).mul(R).sum().backward()

        for _ in range(2):
            step_torch()
            step_native()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            step_native()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step_native()
        graph.replay()
        times = {"torch": [], "native": [], "graph": []}
        for _ in range(args.rounds):
            times["torch"].append(timed(step_torch, args.iters))
            times["native"].append(timed(step_native, args.iters))
            times["graph"].append(timed(graph.replay, args.iters))
        del graph
        L = enc.pts_voxel_encoder
        from bevfusion_b200 import _C
        row = {"batch": B, "pillars": int(fv.shape[0]),
               "slots_occupied": int(fn.clamp(max=P).sum()),
               "ms": {k: round(statistics.median(v), 3) for k, v in times.items()},
               "peak_mb": {"torch": round(peak_of(step_torch), 1), "native": round(peak_of(step_native), 1)},
               "state_plus_workspace_mb": round((_C.lib().bevb200_pillar_train_state_bytes(B * CAP, P)
                                                 + _C.lib().bevb200_pillar_train_workspace_bytes(B * CAP, P)) / 1e6, 1)}
        g = [p.grad for p in (L.pfn_layers[0].linear.weight, L.pfn_layers[1].linear.weight)]
        assert all(bool(torch.isfinite(x).all()) for x in g)
        print(json.dumps(row), flush=True)
        results["rows"].append(row)
        del enc, ref
        torch.cuda.empty_cache()
    with open(os.path.join(args.out_dir, "pillars_train_bench.json"), "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
