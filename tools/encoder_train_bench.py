"""Training step of the voxelnet 0.075 SparseEncoder: forward + backward of (out * R).sum().

    python tools/encoder_train_bench.py OUT_DIR [--iters 5] [--rounds 3] [--batches 1,4]

Input: synthetic.lidar_cloud through voxelize_mean_fused(sync=False) at the config's training max_voxels (120000)
per sample, batch 1 and 4 (the samples are voxelized one by one and concatenated, outside the timed window).
Three ways, alternated per round, median of the rounds:
  modular  the per-conv Python path (SparseEncoder.forward without num_voxels=), eager
  native   SparseEncoder.forward(..., num_voxels=) in training mode, eager
  graph    the native step captured as one CUDA graph and replayed
Each row also gives the peak memory of the step and EncoderPlan.train_state_bytes.  The card name and power limit
are read in the same run.  Writes OUT_DIR/encoder_train_bench.json.  Needs a CUDA device."""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200.sparse_encoder import voxelnet_0p075_encoder  # noqa: E402
from bevfusion_b200.voxelize import voxelize_mean_fused  # noqa: E402

MAX_VOXELS = 120000


def inputs(B, dev):
    L = S.LIDAR_C3
    feats, coors = [], []
    for b in range(B):
        pts = torch.from_numpy(S.lidar_cloud(seed=b)).to(dev)
        f, c, _, n = voxelize_mean_fused(pts, L["voxel_size"], L["point_cloud_range"], L["max_num_points"],
                                         MAX_VOXELS, batch_idx=b, sync=False)
        m = int(n.item())                       # set-up, outside the timed window
        feats.append(f[:m])
        coors.append(c[:m])
    feats, coors = torch.cat(feats), torch.cat(coors)
    return feats, coors, torch.tensor([feats.shape[0]], dtype=torch.int32, device=dev)


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
    return (torch.cuda.max_memory_allocated() - base) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--iters", type=int, default=5)
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
        enc = voxelnet_0p075_encoder().to(dev).train()
        mod = copy.deepcopy(enc)
        feats, coors, n_dev = inputs(B, dev)
        X, Y, Z = enc.plan().out_shape
        R = torch.randn((B, enc.plan().out_channels * Z, X, Y), device=dev)

        def step_modular():
            mod(feats.clone().requires_grad_(True), coors, B).mul(R).sum().backward()

        def step_native():
            enc(feats.clone().requires_grad_(True), coors, B, num_voxels=n_dev).mul(R).sum().backward()

        for _ in range(2):
            step_modular()
            step_native()
        static_x = feats.clone().requires_grad_(True)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            enc(static_x, coors, B, num_voxels=n_dev).mul(R).sum().backward()
        torch.cuda.current_stream().wait_stream(side)
        for p in enc.parameters():
            p.grad = None
        static_x.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            enc(static_x, coors, B, num_voxels=n_dev).mul(R).sum().backward()
        graph.replay()
        times = {"modular": [], "native": [], "graph": []}
        for _ in range(args.rounds):
            times["modular"].append(timed(step_modular, args.iters))
            times["native"].append(timed(step_native, args.iters))
            times["graph"].append(timed(graph.replay, args.iters))
        del graph
        row = {"batch": B, "voxels": int(feats.shape[0]),
               "ms": {k: round(statistics.median(v), 3) for k, v in times.items()},
               "peak_gb": {"modular": round(peak_of(step_modular), 2), "native": round(peak_of(step_native), 2)},
               "train_state_gb": round(enc.plan().train_state_bytes(feats.shape[0], B) / 1e9, 2),
               "backward_workspace_gb": round(enc.plan().backward_workspace_bytes(feats.shape[0], B) / 1e9, 2)}
        print(json.dumps(row), flush=True)
        results["rows"].append(row)
        del enc, mod
        torch.cuda.empty_cache()
    with open(os.path.join(args.out_dir, "encoder_train_bench.json"), "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
