"""TransFusionHead.get_targets at the shipped config (200 proposals, 10 classes, one decoder layer, the 128 x 128
map of grid 1024 / out_size_factor 8) on synthetic.gt_boxes (40-120 gts per sample) and
synthetic.transfusion_predictions, at batch 1 and 4:

    python tools/transfusion_targets_bench.py OUT_DIR [--window 1.0]
    python tools/transfusion_targets_bench.py OUT_DIR --profile

(a) reference: get_targets_single restated op for op on CUDA tensors, one sample at a time: decode, the
               HungarianAssigner3D cost, cost.cpu() and scipy's linear_sum_assignment, the targets, float(mean_iou),
               and the heatmap loop (tests/test_transfusion_assign_gpu.py and tools/head_targets_bench.py hold the
               restatements)
(b) eager:     bevfusion_b200.transfusion_assign.transfusion_targets (list form: padding, the assignment call, the
               heatmap call, one synchronisation)
(c) graph:     transfusion_assign_batched + transfusion_heatmap_targets_batched on padded inputs as one CUDA graph
               replay
Host clock with a device synchronise for (a) and (b), CUDA events over windows of at least --window seconds for
(c); the median of three alternating rounds.  Also whether (a) and (b) agree, the launches per batched call and the card
name / power limit read in the same run.  Writes OUT_DIR/transfusion_targets_bench.json.  With --profile, a run of
its own (no graphs, no timing) gives each kernel's device time under torch.profiler (mean of 20 calls) and the
solver's Dijkstra steps per segment, in OUT_DIR/transfusion_targets_profile.json.  Needs a CUDA device."""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bevfusion_b200 import _C  # noqa: E402
from bevfusion_b200 import head_targets as H  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200 import transfusion_assign as TA  # noqa: E402
from head_targets_bench import card_info, host_ms, ref_transfusion, timed_ms  # noqa: E402
from test_transfusion_assign_gpu import ref_get_targets  # noqa: E402

CFG, CODER = S.TRANSFUSION_TRAIN_CFG, S.TRANSFUSION_CODER
P, K = 200, 10


def bench(batch, window, dev):
    gb, gl = S.gt_boxes(seed=batch, batch=batch)
    pred = {k: v.to(dev) for k, v in S.transfusion_predictions(batch + 100, batch, (gb, gl)).items()}
    bl, ll = [b.to(dev) for b in gb], [l.to(dev) for l in gl]

    def ref():
        r = ref_get_targets(bl, ll, pred, P)
        return r, ref_transfusion(CFG, bl, ll)

    eager = lambda: TA.transfusion_targets(bl, ll, pred, K, P, CFG, CODER)                    # noqa: E731
    pb, pl, pc = H.pad_gt(bl, ll)

    def batched():
        return (TA.transfusion_assign_batched(pred, pb, pl, pc, K, P, CFG, CODER),
                H.transfusion_heatmap_targets_batched(pb, pl, pc, K, CFG))

    (a, a_hm), b = ref(), eager()
    agree = dict(labels_differing=int(sum(int((x != y).sum()) for x, y in zip(a["labels"], b[0]))),
                 num_pos_equal=sum(a["num_pos"]) == b[5],
                 matched_ious_abs_diff=abs(float(np.mean(a["mean_iou"])) - b[6]),
                 heatmap_cells_differing=int((a_hm != b[7]).sum()))
    _C.reset_launch_count()
    batched()
    launches = _C.launch_count()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        batched()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        batched()
    for _ in range(3):
        ref()
        eager()
        g.replay()
    rounds = dict(reference=[], eager=[], graph=[])
    for _ in range(3):
        rounds["reference"].append(host_ms(ref, 5))
        rounds["eager"].append(host_ms(eager, 50))
        rounds["graph"].append(timed_ms(g.replay, window))
    ms = {k: statistics.median(v) for k, v in rounds.items()}
    return dict(batch=batch, gts=[int(b.shape[0]) for b in bl], ms=ms, rounds=rounds, launches_per_call=launches,
                reference_vs_device=agree, speedup_eager=ms["reference"] / ms["eager"],
                speedup_graph=ms["reference"] / ms["graph"])


def profile_kernels(batch, dev):
    """Device time of each kernel of one batched call (mean of 20 under torch.profiler) and the solver's steps."""
    from torch.profiler import ProfilerActivity, profile
    gb, gl = S.gt_boxes(seed=batch, batch=batch)
    pred = {k: v.to(dev) for k, v in S.transfusion_predictions(batch + 100, batch, (gb, gl)).items()}
    pb, pl, pc = H.pad_gt([b.to(dev) for b in gb], [l.to(dev) for l in gl])
    _, ex = TA.transfusion_assign_batched(pred, pb, pl, pc, K, P, CFG, CODER, return_extras=True)
    steps = ex["steps"].cpu().tolist()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            TA.transfusion_assign_batched(pred, pb, pl, pc, K, P, CFG, CODER)
        torch.cuda.synchronize()
    us = {}
    for e in prof.events():
        for k in ("tf_cost_kernel", "lsap_kernel", "tf_targets_kernel"):
            if k in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
                us.setdefault(k, []).append(e.device_time_total)
    return dict(kernel_us={k: sum(v) / len(v) for k, v in us.items()}, kernel_calls={k: len(v) for k, v in us.items()},
                solver_steps=steps, gts=pc.cpu().tolist())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("transfusion_targets_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    os.makedirs(args.out_dir, exist_ok=True)
    if args.profile:
        result = dict(card=card_info(), profile=[])
        for batch in (1, 4):
            result["profile"].append(dict(batch=batch, **profile_kernels(batch, dev)))
            print(json.dumps(result["profile"][-1]), flush=True)
        name = "transfusion_targets_profile.json"
    else:
        result = dict(card=card_info(), runs=[])
        for batch in (1, 4):
            r = bench(batch, args.window, dev)
            result["runs"].append(r)
            print(json.dumps({k: r[k] for k in ("batch", "ms", "launches_per_call", "reference_vs_device")}),
                  flush=True)
        name = "transfusion_targets_bench.json"
    with open(os.path.join(args.out_dir, name), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
