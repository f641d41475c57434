"""Training losses of both detection heads, forward + backward, at batch 1 and 4: CenterHead with the six nuScenes tasks
on the 128 x 128 map (synthetic.centerhead_head_outputs, targets from head_targets), TransFusion with ten classes,
200 proposals and one trained layer on the 180 x 180 dense heatmap (synthetic.transfusion_predictions +
transfusion_heatmap, targets from transfusion_assign_batched).

    python tools/head_losses_bench.py OUT_DIR [--window 1.0] [--profile]

(a) reference: the reference's loss lines (centerpoint.py:596-634, transfusion.py:616-711) restated on CUDA tensors
               with the mmdet losses restated in torch and the reference's .item() calls, then backward()
(b) eager:     head_losses.centerhead_loss / transfusion_loss, then backward()
(c) graph:     targets + loss + backward captured as one CUDA graph, replayed
Host clock around each step with a device synchronise at its end for (a); CUDA events over windows of at least
--window seconds for (b) and (c); the median of three alternating rounds.  The card name and power limit are read in
the same run.  --profile instead writes a torch.profiler table of per-kernel times of (b).  Writes
OUT_DIR/head_losses_bench.json (or head_losses_profile.txt).  Needs a CUDA device."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from bevfusion_b200 import head_losses as HL  # noqa: E402
from bevfusion_b200 import head_targets as HT  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200.transfusion_assign import transfusion_assign_batched  # noqa: E402
from make_head_losses_golden import FocalLoss, GaussianFocalLoss, L1Loss  # noqa: E402

DEV = torch.device("cuda:0")
CW = [1.0] * 8 + [0.2, 0.2]
TASKS = [[n for n, _ in t] for t in S.CENTERHEAD_TASKS]
CFG_CH = dict(point_cloud_range=[-54.0, -54.0, -5.0, 54.0, 54.0, 3.0], grid_size=[1024, 1024, 1],
              voxel_size=[108 / 1024, 108 / 1024, 0.2], out_size_factor=8, dense_reg=1, gaussian_overlap=0.1,
              max_objs=500, min_radius=2, code_weights=CW)


def ref_centerhead(preds, targets):
    heatmaps, anno_boxes, inds, masks = targets
    lc, lb = GaussianFocalLoss(), L1Loss(loss_weight=0.25)
    out = {}
    for t, pd in enumerate(preds):
        p = pd[0]
        hm = torch.clamp(p["heatmap"].sigmoid(), min=1e-4, max=1 - 1e-4)
        num_pos = heatmaps[t].eq(1).float().sum().item()
        out["heatmap/task%d" % t] = lc(hm, heatmaps[t], avg_factor=max(num_pos, 1))
        pred = torch.cat([p[k] for k in ("reg", "height", "dim", "rot", "vel")], 1).permute(0, 2, 3, 1).contiguous()
        pred = pred.view(pred.size(0), -1, pred.size(3))
        ind = inds[t]
        pred = pred.gather(1, ind.unsqueeze(2).expand(ind.size(0), ind.size(1), pred.size(2)))
        num = masks[t].float().sum()
        mask = masks[t].unsqueeze(2).expand_as(anno_boxes[t]).float() * (~torch.isnan(anno_boxes[t])).float()
        out["bbox/task%d" % t] = lb(pred, anno_boxes[t], mask * mask.new_tensor(CW), avg_factor=num + 1e-4)
    return out


def ref_transfusion(pd, targets, P):
    labels, label_weights, bbox_targets, bbox_weights, _, num_pos, _, _, heatmap = targets
    num_pos = int(num_pos.sum().item())
    out = {"loss_heatmap": GaussianFocalLoss()(torch.clamp(pd["dense_heatmap"].sigmoid(), min=1e-4, max=1 - 1e-4),
                                               heatmap, avg_factor=max(heatmap.eq(1).float().sum().item(), 1))}
    cols = slice(0, P)
    score = pd["heatmap"][..., cols].permute(0, 2, 1).reshape(-1, pd["heatmap"].shape[1])
    out["cls"] = FocalLoss()(score, labels[..., cols].reshape(-1), label_weights[..., cols].reshape(-1),
                             avg_factor=max(num_pos, 1))
    preds = torch.cat([pd[k][..., cols] for k in ("center", "height", "dim", "rot", "vel")], 1).permute(0, 2, 1)
    w = bbox_weights[:, cols] * bbox_weights.new_tensor(CW)
    out["bbox"] = L1Loss(loss_weight=0.25)(preds, bbox_targets[:, cols], w, avg_factor=max(num_pos, 1))
    return out


def setup(head, B):
    gt = S.gt_boxes(seed=B, batch=B)
    boxes, labels, counts = HT.pad_gt([b.to(DEV) for b in gt[0]], [l.to(DEV) for l in gt[1]])
    if head == "centerhead":
        outs = S.centerhead_head_outputs(B, B, gt=gt)
        leaves = [{k: v.to(DEV) for k, v in t.items()} for t in outs]

        def targets():
            return HT.centerhead_targets_batched(boxes, labels, counts, TASKS, CFG_CH)

        def loss(preds, tg):
            return HL.centerhead_loss(preds, tg, CFG_CH)

        def ref(preds, tg):
            return ref_centerhead(preds, tg)

        wrap = lambda d: [[x] for x in d]
    else:
        P = 200
        pr = S.transfusion_predictions(B, B, gt, num_proposals=P)
        pr["dense_heatmap"] = S.transfusion_heatmap(B, B, height=180, width=180, gt=gt)
        leaves = [{k: v.to(DEV) for k, v in pr.items()}]
        cfg = dict(S.TRANSFUSION_TRAIN_CFG, grid_size=[1440, 1440, 1], code_weights=CW)

        def targets():
            a = transfusion_assign_batched({k: v for k, v in leaves[0].items()}, boxes, labels, counts, 10, P, cfg,
                                           S.TRANSFUSION_CODER)
            return tuple(a) + (HT.transfusion_heatmap_targets_batched(boxes, labels, counts, 10, cfg),)

        def loss(preds, tg):
            return HL.transfusion_loss(preds, tg, P, 1, False, cfg)

        def ref(preds, tg):
            return ref_transfusion(preds[0][0], tg, P)

        wrap = lambda d: [[d[0]]]
    return leaves, targets, loss, ref, wrap


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
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    results = {"card": card, "cases": []}
    prof_rows = []
    for head in ("centerhead", "transfusion"):
        for B in (1, 4):
            leaves, targets, loss, ref, wrap = setup(head, B)
            tg = targets()

            def step(lossfn, tg_fn):
                preds = wrap([{k: v.detach().requires_grad_() for k, v in d.items()} for d in leaves])
                out = lossfn(preds, tg_fn())
                total = sum(v for k, v in out.items() if k != "matched_ious")
                return torch.autograd.grad(total, [v for p in preds for v in p[0].values()])

            run_a = lambda: step(ref, lambda: tg)
            run_b = lambda: step(loss, lambda: tg)
            if args.profile:
                from torch.profiler import ProfilerActivity, profile
                for _ in range(3):
                    run_b()
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(20):
                        run_b()
                    torch.cuda.synchronize()
                prof_rows.append("== %s B=%d (20 steps)\n%s" % (head, B, prof.key_averages().table(
                    sort_by="cuda_time_total", row_limit=15)))
                continue
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(2):
                    step(loss, targets)
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                step(loss, targets)
            rounds = {"a_reference_us": [], "b_eager_us": [], "c_graph_us": []}
            for _ in range(3):
                rounds["a_reference_us"].append(timed_host(run_a, args.window))
                rounds["b_eager_us"].append(timed_events(run_b, args.window))
                rounds["c_graph_us"].append(timed_events(g.replay, args.window))
            row = {"head": head, "B": B}
            row.update({k: round(statistics.median(v), 1) for k, v in rounds.items()})
            results["cases"].append(row)
            print(json.dumps(row), flush=True)
    if args.profile:
        with open(os.path.join(args.out_dir, "head_losses_profile.txt"), "w") as f:
            f.write(card + "\n" + "\n".join(prof_rows))
        return
    with open(os.path.join(args.out_dir, "head_losses_bench.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(card)


if __name__ == "__main__":
    main()
