"""TransFusionHead's query selection (transfusion.py:238-274 and :322-325: sigmoid, peak mask, top num_proposals,
labels / index, the query_heatmap_score gather) at the shipped config (10 classes, 200 proposals, nms_kernel_size 3,
nuScenes) on synthetic.transfusion_heatmap logits, at batch 1 and 4, on the 128 x 128 and 180 x 180 maps, in fp32 and
fp16:

    python tools/transfusion_proposals_bench.py OUT_DIR [--window 1.0]
    python tools/transfusion_proposals_bench.py OUT_DIR --profile

(a) reference: the reference's lines on CUDA tensors, its unstable full argsort included
               (tests/transfusion_proposals_oracle.torch_proposals with stable=False)
(b) eager:     bevfusion_b200.transfusion_proposals.transfusion_proposals
(c) graph:     (b) captured once and replayed as a CUDA graph
The query_feat / query_pos gathers, which the head keeps in both forms, are not timed.  CUDA events over windows of
at least --window seconds after a warm-up; the median of three alternating rounds.  Also whether (a) and (b) agree
(indices, and the selected values), whether (b) equals the stable restatement bit for bit, the candidates per sample
(masked values > 0 or NaN), the launches per call and the card name / power limit read in the same run.  Writes
OUT_DIR/transfusion_proposals_bench.json.  With --profile, a run of its own (no graphs, no timing) gives each
kernel's device time under torch.profiler (mean of 20 calls) in OUT_DIR/transfusion_proposals_profile.json.  Needs
a CUDA device."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bevfusion_b200 import _C  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200.transfusion_proposals import transfusion_proposals  # noqa: E402
from head_targets_bench import card_info, timed_ms  # noqa: E402
from transfusion_proposals_oracle import torch_proposals  # noqa: E402

K, KSIZE, DATASET = 200, 3, "nuScenes"
SHAPES = [(1, 128), (4, 128), (1, 180), (4, 180)]
DTYPES = {"fp32": torch.float32, "fp16": torch.float16}


def heatmap(batch, size, dtype, dev):
    return S.transfusion_heatmap(seed=batch * 1000 + size, batch=batch, height=size, width=size,
                                 dtype=dtype).to(dev)


def agreement(x, ref, dev_out):
    bits = torch.int16 if x.dtype == torch.float16 else torch.int32
    stable = torch_proposals(x, K, KSIZE, DATASET, stable=True)
    vals = lambda out: torch.gather(out[2], 1, out[0][:, None, :]).squeeze(1)   # noqa: E731
    return dict(indices_equal=bool(torch.equal(ref[0], dev_out[0]) and torch.equal(ref[1], dev_out[1])),
                selected_values_equal=bool(torch.equal(vals(ref).view(bits), vals(dev_out).view(bits))),
                stable_restatement_bit_equal=all(bool(torch.equal(a.view(bits) if a.is_floating_point() else a,
                                                                  b.view(bits) if b.is_floating_point() else b))
                                                 for a, b in zip(stable, dev_out)))


def bench(batch, size, dname, window, dev):
    x = heatmap(batch, size, DTYPES[dname], dev)
    ref = lambda: torch_proposals(x, K, KSIZE, DATASET, stable=False)           # noqa: E731
    eager = lambda: transfusion_proposals(x, K, KSIZE, DATASET)                  # noqa: E731
    a, b = ref(), eager()
    agree = agreement(x, a, b)
    candidates = _candidates(x).tolist()
    _C.reset_launch_count()
    eager()
    launches = _C.launch_count()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eager()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        eager()
    for _ in range(20):
        ref()
        eager()
        g.replay()
    rounds = dict(reference=[], eager=[], graph=[])
    for _ in range(3):
        rounds["reference"].append(timed_ms(ref, window))
        rounds["eager"].append(timed_ms(eager, window))
        rounds["graph"].append(timed_ms(g.replay, window))
    ms = {k: statistics.median(v) for k, v in rounds.items()}
    return dict(batch=batch, shape=[10, size, size], dtype=dname, num_proposals=K, candidates_per_sample=candidates,
                ms=ms, rounds=rounds, launches_per_call=launches, reference_vs_device=agree,
                speedup_eager=ms["reference"] / ms["eager"], speedup_graph=ms["reference"] / ms["graph"])


def _candidates(x):
    """Cells per sample whose masked value is > 0 or NaN (what the peak pass keeps), nuScenes exemptions."""
    s = x.sigmoid()
    local = torch.zeros_like(s)
    local[:, :, 1:-1, 1:-1] = torch.nn.functional.max_pool2d(s, 3, 1, 0)
    local[:, 8:10] = s[:, 8:10]
    mm = s * (s == local)
    return ((mm > 0) | torch.isnan(mm)).flatten(1).sum(1)


def profile_kernels(batch, size, dname, dev):
    from torch.profiler import ProfilerActivity, profile
    x = heatmap(batch, size, DTYPES[dname], dev)
    transfusion_proposals(x, K)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            transfusion_proposals(x, K)
        torch.cuda.synchronize()
    us = {}
    for e in prof.events():
        for k in ("tf_peak_kernel", "tf_select_kernel"):
            if k in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
                us.setdefault(k, []).append(e.device_time_total)
    return dict(kernel_us={k: sum(v) / len(v) for k, v in us.items()}, kernel_calls={k: len(v) for k, v in us.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("transfusion_proposals_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    os.makedirs(args.out_dir, exist_ok=True)
    if args.profile:
        result = dict(card=card_info(), profile=[])
        for dname in DTYPES:
            for batch, size in SHAPES:
                result["profile"].append(dict(batch=batch, size=size, dtype=dname,
                                              **profile_kernels(batch, size, dname, dev)))
                print(json.dumps(result["profile"][-1]), flush=True)
        name = "transfusion_proposals_profile.json"
    else:
        result = dict(card=card_info(), runs=[])
        for dname in DTYPES:
            for batch, size in SHAPES:
                r = bench(batch, size, dname, args.window, dev)
                result["runs"].append(r)
                print(json.dumps({k: r[k] for k in ("batch", "shape", "dtype", "ms", "launches_per_call",
                                                    "candidates_per_sample", "reference_vs_device")}), flush=True)
        name = "transfusion_proposals_bench.json"
    with open(os.path.join(args.out_dir, name), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
