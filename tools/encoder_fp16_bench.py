"""The voxelnet 0.075 SparseEncoder (the bench's encoder) at BF16x3 and at FP16 (precision=PREC_FP16).

    python tools/encoder_fp16_bench.py OUT_DIR [--window 1.0] [--rounds 3]

Input: the C3 cloud (synthetic.lidar_cloud(seed=0)) through voxelize_mean_fused at the bench's cap, one sample.
Per precision, each captured as one CUDA graph and replayed:
  eval   SparseEncoder.forward in eval mode under no_grad
  train  one training step: forward with num_voxels= and the backward of (out * R).sum()
The two precisions alternate over --rounds rounds; each row is the median of the rounds' mean CUDA-event times over
a window of at least --window seconds.  The result also gives the exact training-state and backward-workspace bytes
of both plans, the fp16 eval output's max and p99 difference from BF16x3 relative to absref, and, from a separate torch.profiler run, the device time per kernel of each eval forward and training step.  The card
name and power limit are read in the same run.  Writes OUT_DIR/encoder_fp16_bench.json.  Needs a CUDA device.

absref is the same encoder on absolute values: |features|, |W| and, per conv, the folded BN's |scale| and |shift|
(the residuals and ReLUs then add and pass non-negative values), run at BF16x3.  It bounds every product a cell's
value is made of, so |fp16 - bf16x3| / absref compares the two precisions where the sums cancel too.  Cells with
absref = 0 (no voxel) are left out."""
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
from bevfusion_b200.sparse_block import bn_scale_shift  # noqa: E402
from bevfusion_b200.sparse_encoder import voxelnet_0p075_encoder  # noqa: E402
from bevfusion_b200.spconv.ops import PREC_BF16X3, PREC_FP16  # noqa: E402
from bevfusion_b200.voxelize import voxelize_mean_fused  # noqa: E402

PRECS = {"bf16x3": PREC_BF16X3, "fp16": PREC_FP16}


def card_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (v.strip() for v in q.split(","))
    return {"name": name, "power_limit": power, "clocks_max_sm": clock}


def timed_ms(fn, window_s):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    n = max(10, int(window_s * 1e3 / max(start.elapsed_time(stop), 1e-3)) + 1)
    start.record()
    for _ in range(n):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / n


def graph_of(fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    return g, out


def kernel_us(fn, calls=10):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    times = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            times[e.name[:90]] = times.get(e.name[:90], 0.0) + e.device_time_total / calls
    return {"device_us_per_call": sum(times.values()),
            "kernels_us_per_call": dict(sorted(times.items(), key=lambda kv: -kv[1])[:16])}


def abs_encoder(enc):
    """a copy of the eval-mode encoder whose every conv computes |W| and whose BN folds to |scale|, |shift|"""
    a = voxelnet_0p075_encoder().to(enc.conv_out[0].weight.device).eval()   # a new module: no shared plan handle
    a.load_state_dict(enc.state_dict())
    for conv, bn, _, _ in a.plan().chain:
        s, t = bn_scale_shift(bn)
        conv.weight.data.abs_()
        bn.running_mean.zero_()
        bn.running_var.fill_(1.0 - bn.eps)                 # invstd = 1: the fold is (|s|, |t|) itself
        bn.weight.data.copy_(s.abs())
        bn.bias.data.copy_(t.abs())
    return a


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    dev = torch.device("cuda")
    L = S.LIDAR_C3
    pts = torch.from_numpy(S.lidar_cloud(seed=0)).to(dev)
    feats, coors, _, n_dev = voxelize_mean_fused(pts, L["voxel_size"], L["point_cloud_range"], L["max_num_points"],
                                                 L["max_voxels"][1], sync=False)
    torch.manual_seed(0)
    enc_eval = voxelnet_0p075_encoder().to(dev).eval()
    enc_train = copy.deepcopy(enc_eval).train()
    n_rows = feats.shape[0]

    def eval_fn(p):
        def fwd():
            with torch.no_grad():
                return enc_eval(feats, coors, 1, precision=p, num_voxels=n_dev)
        return fwd

    outs = {k: eval_fn(p)() for k, p in PRECS.items()}
    R = torch.randn(outs["bf16x3"].shape, device=dev, generator=torch.Generator(device=dev).manual_seed(1)) * 1e-2

    def train_fn(p):
        def step():
            out = enc_train(feats, coors, 1, num_voxels=n_dev, precision=p)
            (out.float() * R).sum().backward()
            return out
        return step

    fns = {}
    for k, p in PRECS.items():
        g, _ = graph_of(eval_fn(p))
        fns[("eval", k)] = g.replay
        g2, _ = graph_of(train_fn(p))
        fns[("train", k)] = g2.replay
    times = {key: [] for key in fns}
    for _ in range(args.rounds):
        for key, fn in fns.items():
            for _ in range(3):
                fn()
            times[key].append(timed_ms(fn, args.window))
    ref, got = outs["bf16x3"].double(), outs["fp16"].double()
    with torch.no_grad():
        absref = abs_encoder(enc_eval)(feats.abs(), coors, 1, precision=PREC_BF16X3, num_voxels=n_dev).double()
    live = absref > 0
    d = (got - ref).abs()[live] / absref[live]
    sizes = {}
    for k, p in PRECS.items():
        plan = enc_train.plan(p)
        sizes[k] = {"train_state_bytes": plan.train_state_bytes(n_rows, 1),
                    "backward_workspace_bytes": plan.backward_workspace_bytes(n_rows, 1)}
    prof = {"eval_" + k: kernel_us(eval_fn(p)) for k, p in PRECS.items()}
    prof.update({"train_" + k: kernel_us(train_fn(p)) for k, p in PRECS.items()})
    result = {
        "card": card_info(),
        "voxels": int(n_dev.item()),
        "ms_median": {"%s_%s" % key: statistics.median(v) for key, v in times.items()},
        "ms_rounds": {"%s_%s" % key: v for key, v in times.items()},
        "bytes": sizes,
        "fp16_vs_bf16x3_rel_absref": {"max": float(d.max()), "p99": float(torch.quantile(d[:2 ** 24].float(), 0.99)),
                                      "cells": int(live.sum())},
        "profile": prof,
    }
    path = os.path.join(args.out_dir, "encoder_fp16_bench.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({k: result[k] for k in ("card", "voxels", "ms_median", "bytes", "fp16_vs_bf16x3_rel_absref")}))


if __name__ == "__main__":
    main()
