"""The voxelnet 0.075 SparseEncoder's eval forward (the bench's encoder) at BF16x3, FP16 and INT8.

    python tools/encoder_int8_bench.py OUT_DIR [--window 1.0] [--rounds 3]

Input: the C3 cloud (synthetic.lidar_cloud(seed=0)) through voxelize_mean_fused at the bench's cap, one sample.  The
INT8 scales are calibrated (SparseEncoder.calibrate_int8) on the clouds of seeds 1 and 2, not on the timed one.
Each precision's eval forward (eval mode, no_grad, num_voxels=) is captured as one CUDA graph and replayed; the three
alternate over --rounds rounds, and each time is the median of the rounds' mean CUDA-event times over a window of
at least --window seconds.  Then, untimed: dense()'s relative L2 and max deviation of FP16 and INT8 from BF16x3 (max
relative to max |BF16x3|), and, from a torch.profiler run after the timing, the device time per kernel of each
forward.  The card name and power limit are read in the same run.  Writes OUT_DIR/encoder_int8_bench.json.  Needs a
CUDA device."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200.sparse_encoder import voxelnet_0p075_encoder  # noqa: E402
from bevfusion_b200.spconv.ops import PREC_BF16X3, PREC_FP16, PREC_INT8  # noqa: E402
from bevfusion_b200.voxelize import voxelize_mean_fused  # noqa: E402
from encoder_fp16_bench import card_info, graph_of, kernel_us, timed_ms  # noqa: E402

PRECS = {"bf16x3": PREC_BF16X3, "fp16": PREC_FP16, "int8": PREC_INT8}


def cloud(seed, dev):
    L = S.LIDAR_C3
    pts = torch.from_numpy(S.lidar_cloud(seed=seed)).to(dev)
    feats, coors, _, n_dev = voxelize_mean_fused(pts, L["voxel_size"], L["point_cloud_range"], L["max_num_points"],
                                                 L["max_voxels"][1], sync=False)
    return feats, coors, n_dev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    dev = torch.device("cuda")
    torch.manual_seed(0)
    enc = voxelnet_0p075_encoder().to(dev).eval()
    calib = []
    for seed in (1, 2):
        f, c, n = cloud(seed, dev)
        k = int(n.item())
        calib.append((f[:k], c[:k], 1))
    scales = enc.calibrate_int8(calib)
    feats, coors, n_dev = cloud(0, dev)

    def eval_fn(p):
        def fwd():
            with torch.no_grad():
                return enc(feats, coors, 1, precision=p, num_voxels=n_dev)
        return fwd

    outs = {k: eval_fn(p)().clone() for k, p in PRECS.items()}
    fns = {k: graph_of(eval_fn(p))[0].replay for k, p in PRECS.items()}
    times = {k: [] for k in fns}
    for _ in range(args.rounds):
        for k, fn in fns.items():
            for _ in range(3):
                fn()
            times[k].append(timed_ms(fn, args.window))
    ref = outs["bf16x3"].double()
    dev_stats = {}
    for k in ("fp16", "int8"):
        d = outs[k].double() - ref
        dev_stats[k] = {"rel_l2": float(d.norm() / ref.norm()), "max_abs": float(d.abs().max()),
                        "max_rel_to_max": float(d.abs().max() / ref.abs().max())}
    prof = {k: kernel_us(eval_fn(p)) for k, p in PRECS.items()}
    result = {
        "card": card_info(),
        "voxels": int(n_dev.item()),
        "int8_scales": [float(v) for v in scales],
        "eval_ms_median": {k: statistics.median(v) for k, v in times.items()},
        "eval_ms_rounds": times,
        "dense_deviation_from_bf16x3": dev_stats,
        "profile": prof,
    }
    path = os.path.join(args.out_dir, "encoder_int8_bench.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({k: result[k] for k in ("card", "voxels", "eval_ms_median", "dense_deviation_from_bf16x3")}))


if __name__ == "__main__":
    main()
