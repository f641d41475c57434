"""BEV map segmentation, the default seg config (128 x 128 cells of 0.8 m -> 200 x 200 of 0.5 m, C = 512 as the
SECONDFPN concatenation, six classes), at batch 1 and 4.

    python tools/map_seg_bench.py OUT_DIR [--window 1.0]

kernels     the grid transform's forward and backward kernel alone (CUDA events over many launches) against the HBM
            floor B * C * (128^2 + 200^2) * 4 bytes / 3.35 TB/s computed from the shapes
step        transform -> 1 x 1 projection to the six classes -> six focal losses -> backward to the features ->
            IoU counts of the sigmoid at evaluate_map's seven thresholds:
  (a) reference: the reference's lines on CUDA tensors (F.interpolate / F.grid_sample with the grid built on the host
                 and copied, six per-class sigmoid_focal_loss calls, backward, and evaluate_map's counting with its
                 per-sample .cpu())
  (b) eager:     BEVGridTransform, map_seg_loss, backward, map_seg_counts
  (c) graph:     (b) captured as one CUDA graph and replayed
head        the whole BEVSegmentationHead training step (with the two 3 x 3 convs of the classifier) for scale:
            the reference's lines vs the native transform and losses, eager
Host clock around each step with a device synchronise for (a); CUDA events over windows of at least --window seconds
for the rest; the median of three alternating rounds.  The card name and power limit are read in the same run.
Writes OUT_DIR/map_seg_bench.json.  Needs a CUDA device."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from bevfusion_b200 import map_seg as MS  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402

DEV = torch.device("cuda:0")
C, K = 512, 6
HBM = 3.35e12
THR = torch.tensor(MS.THRESHOLDS)


def ref_transform(x, input_scope, output_scope):
    coords = []
    for (imin, imax, _), (omin, omax, ostep) in zip(input_scope, output_scope):
        v = torch.arange(omin + ostep / 2, omax, ostep)
        v = (v - imin) / (imax - imin) * 2 - 1
        coords.append(v.to(x.device))
    u, v = torch.meshgrid(coords, indexing="ij")
    grid = torch.stack([torch.stack([v, u], dim=-1)] * x.shape[0], dim=0)
    return F.grid_sample(x, grid, mode="bilinear", align_corners=False)


def ref_focal(inputs, targets):
    inputs, targets = inputs.float(), targets.float()
    p = torch.sigmoid(inputs)
    ce = F.binary_cross_entropy_with_logits(inputs, targets, reduction="none")
    p_t = p * targets + (1 - p) * (1 - targets)
    return (ce * ((1 - p_t) ** 2)).mean()


def ref_counts(probs, gts):
    tp, fp, fn = (torch.zeros(K, len(THR)) for _ in range(3))
    for b in range(probs.shape[0]):
        pred = probs[b].detach().cpu().reshape(K, -1)[:, :, None] >= THR
        label = gts[b].cpu().bool().reshape(K, -1)[:, :, None]
        tp += (pred & label).sum(dim=1)
        fp += (pred & ~label).sum(dim=1)
        fn += (~pred & label).sum(dim=1)
    return tp, fp, fn


def timed_events(fn, window):
    fn()
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    while time.perf_counter() - t0 < window:
        fn()
        n += 1
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / n


def timed_host(fn, window):
    fn()
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < window:
        fn()
        torch.cuda.synchronize()
        n += 1
    return (time.perf_counter() - t0) * 1e6 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--window", type=float, default=1.0)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    torch.backends.cudnn.benchmark = True
    cfg = S.MAP_SEG_CFG
    results = {"card": card, "cases": []}
    for B in (1, 4):
        feats = S.map_seg_features(seed=B, batch=B, channels=C).to(DEV)
        masks = S.map_seg_masks(seed=B, batch=B).to(DEV)
        proj = (torch.randn((K, C, 1, 1), generator=torch.Generator().manual_seed(0)) / C ** 0.5).to(DEV)
        t = MS.BEVGridTransform(**cfg)
        plan = t.plan(128, 128, DEV)
        y = t(feats)
        gy = torch.empty_like(y)
        gx = torch.empty_like(feats)

        def k_fwd():
            plan.fwd.run(feats, y, B * C)

        def k_bwd():
            plan.bwd.run(y, gx, B * C)

        def ref_step():
            x = feats.detach().requires_grad_()
            logits = F.conv2d(ref_transform(x, cfg["input_scope"], cfg["output_scope"]), proj)
            losses = [ref_focal(logits[:, k], masks[:, k]) for k in range(K)]
            g, = torch.autograd.grad(sum(losses), x)
            ref_counts(torch.sigmoid(logits.detach()), masks)
            return g

        counts = torch.zeros((3, K, len(THR)), dtype=torch.int64, device=DEV)

        def our_step():
            x = feats.detach().requires_grad_()
            logits = F.conv2d(t(x), proj)
            losses = MS.map_seg_loss(logits, masks, "focal", S.MAP_CLASSES)
            g, = torch.autograd.grad(sum(losses.values()), x)
            MS.map_seg_counts(torch.sigmoid(logits.detach()), masks, out=counts)
            return g

        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(3):
                our_step()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            our_step()

        ref_head = MS.BEVSegmentationHead(C, dict(cfg), list(S.MAP_CLASSES), "focal").to(DEV).train()
        our_head = MS.BEVSegmentationHead(C, dict(cfg), list(S.MAP_CLASSES), "focal").to(DEV).train()
        our_head.load_state_dict(ref_head.state_dict())

        def ref_head_step():
            x = feats.detach().requires_grad_()
            logits = ref_head.classifier(ref_transform(x, cfg["input_scope"], cfg["output_scope"]))
            sum(ref_focal(logits[:, k], masks[:, k]) for k in range(K)).backward()

        def our_head_step():
            x = feats.detach().requires_grad_()
            sum(our_head([x], masks).values()).backward()

        # the same answer before timing: the step's feature gradient against the reference's lines
        ga, gb = ref_step(), our_step()
        grad_rel = float((ga - gb).abs().max() / ga.abs().max())
        rounds = {k: [] for k in ("fwd_kernel_us", "bwd_kernel_us", "a_reference_us", "b_eager_us", "c_graph_us",
                                  "head_reference_us", "head_native_us")}
        for _ in range(3):
            rounds["fwd_kernel_us"].append(timed_events(k_fwd, args.window))
            rounds["bwd_kernel_us"].append(timed_events(k_bwd, args.window))
            rounds["a_reference_us"].append(timed_host(ref_step, args.window))
            rounds["b_eager_us"].append(timed_events(our_step, args.window))
            rounds["c_graph_us"].append(timed_events(graph.replay, args.window))
            rounds["head_reference_us"].append(timed_events(ref_head_step, args.window))
            rounds["head_native_us"].append(timed_events(our_head_step, args.window))
        floor = B * C * (128 * 128 + 200 * 200) * 4 / HBM * 1e6
        row = {"B": B, "C": C, "hbm_floor_us": round(floor, 1), "step_grad_max_rel_diff": grad_rel}
        row.update({k: round(statistics.median(v), 1) for k, v in rounds.items()})
        row["fwd_floor_share"] = round(floor / row["fwd_kernel_us"], 2)
        row["bwd_floor_share"] = round(floor / row["bwd_kernel_us"], 2)
        results["cases"].append(row)
        print(json.dumps(row), flush=True)
    with open(os.path.join(args.out_dir, "map_seg_bench.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(card)


if __name__ == "__main__":
    main()
