"""Training step of the camera lift: fused lift + pool forward + backward against the materialised path.

    python tools/lift_backward_bench.py OUT_DIR [--configs C2,C5] [--window 1.0]

(a) fused:        out = plan.lift_pool(depth, ctx);                       grads of depth and ctx from G
(b) materialised: out = plan.pool(depth.unsqueeze(-1) * ctx.unsqueeze(2)); the same grads through _PoolPerm and
                  torch's broadcast-multiply backward (the reference's get_cam_feats + bev_pool)
Reports CUDA-event times over a window of at least --window seconds after a warm-up (three alternating rounds, the
median is reported), peak memory of one step of each path, the backward kernel alone with its algorithmic bytes, the
largest relative difference between the gradients of (a) and (b), and the card name / power limit read in the same
run.  Writes OUT_DIR/lift_backward_bench.json.  Needs a CUDA device: there is no CPU path."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200.bev_pool import BEVPoolPlan  # noqa: E402


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
    return start.elapsed_time(stop) / n, n


def peak_bytes(fn):
    """peak allocation of one call of fn() above what was allocated before it (inputs, plan tables)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def max_rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


def run_config(name, dev, window_s):
    geom, cfg = S.camera_geometry(name, device=dev)
    plan = BEVPoolPlan(geom, cfg["xbound"], cfg["ybound"], cfg["zbound"])
    B, N, D, fH, fW, _ = geom.shape
    del geom
    C = cfg["C"]
    g = torch.Generator(device=dev).manual_seed(0)
    depth = torch.softmax(torch.randn(B, N, D, fH, fW, generator=g, device=dev), dim=2).contiguous()
    ctx = torch.randn(B, N, fH, fW, C, generator=g, device=dev)
    G = torch.randn(*plan.tables.dims, C, generator=g, device=dev)
    d = depth.clone().requires_grad_(True)
    c = ctx.clone().requires_grad_(True)

    def fused():
        return torch.autograd.grad(plan.lift_pool(d, c), (d, c), G)

    def materialised():
        return torch.autograd.grad(plan.pool(d.unsqueeze(-1) * c.unsqueeze(2)), (d, c), G)

    def backward_only():
        return plan._lift_pool_backward(G, depth, ctx, True, True)

    fa = fused()
    fb = materialised()
    diff = {"ddepth": max_rel(fa[0], fb[0]), "dctx": max_rel(fa[1], fb[1])}
    del fa, fb
    for fn in (fused, materialised, backward_only):   # warm-up
        for _ in range(3):
            fn()
    rounds = {"fused": [], "materialised": [], "backward_only": []}
    iters = {}
    for _ in range(3):
        for key, fn in (("fused", fused), ("materialised", materialised), ("backward_only", backward_only)):
            ms, n = timed_ms(fn, window_s)
            rounds[key].append(ms)
            iters[key] = n
    med = {k: sorted(v)[1] for k, v in rounds.items()}
    peak = {"fused": peak_bytes(fused), "materialised": peak_bytes(materialised)}
    n_seg = plan._lift_tables(B * N, D, fH, fW)[5]
    f32 = 4
    alg = {"G_rows_gathered": n_seg * C * f32, "depth_ctx_read": depth.numel() * f32 + ctx.numel() * f32,
           "ddepth_dctx_written": depth.numel() * f32 + ctx.numel() * f32}
    alg_total = sum(alg.values())
    return {
        "config": name, "shape": {"B": B, "N": N, "D": D, "fH": fH, "fW": fW, "C": C, "grid": list(plan.tables.dims)},
        "n_kept": plan.tables.n_kept, "n_segments": n_seg,
        "fwd_plus_bwd_ms": {"fused": round(med["fused"], 4), "materialised": round(med["materialised"], 4)},
        "speedup": round(med["materialised"] / med["fused"], 2),
        "backward_kernel_ms": round(med["backward_only"], 4),
        "backward_algorithmic_bytes": alg, "backward_algorithmic_MB": round(alg_total / 1e6, 2),
        "backward_GBps": round(alg_total / (med["backward_only"] * 1e-3) / 1e9, 1),
        "peak_MB_above_inputs": {k: round(v / 2**20, 1) for k, v in peak.items()},
        "peak_saving_MB": round((peak["materialised"] - peak["fused"]) / 2**20, 1),
        "grad_max_rel_diff_fused_vs_materialised": diff,
        "rounds_ms": {k: [round(x, 4) for x in v] for k, v in rounds.items()}, "iterations_per_window": iters,
    }


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("out_dir")
    ap.add_argument("--configs", default="C2,C5")
    ap.add_argument("--window", type=float, default=1.0, help="seconds of work per timed window")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lift_backward_bench: no CUDA device (this benchmark only runs on the GPU)")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"card": card_info(), "timing": "CUDA events, eager calls, mean over a window of >= %.1f s after a "
           "warm-up; median of 3 alternating rounds" % a.window, "results": []}
    for name in a.configs.split(","):
        r = run_config(name, dev, a.window)
        print(json.dumps(r), flush=True)
        res["results"].append(r)
        torch.cuda.empty_cache()
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "lift_backward_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["card"]))


if __name__ == "__main__":
    main()
