"""Camera view transform of an augmented training step: the BEV pooling plan rebuilt from new calibration every step.

    python tools/lss_rebuild_bench.py OUT_DIR [--steps 20] [--draws 50]

Every step gets its own calibration (seeded draws of the reference's augment2d / augment3d, synthetic.augmented_rig),
then runs the fused lift + pool and its backward:
(a) host-count: BEVPoolPlan.from_cameras + lift_pool + backward, eager (the plan build reads its counts back to the
    host and allocates its tables)
(b) sync-free:  plan.rebuild_ + lift_pool + backward on a from_cameras(..., sync=False) plan, eager
(c) (b) captured once in a CUDA graph; a step copies the calibration into the static inputs and replays
at C2 with B = 1 and 4 and at C5 with B = 1 (steps cycle through 8 calibrations; times are CUDA events around
--steps steps after a warm-up, median of three rounds).  Then, over --draws draws at C2 and C5 (B = 1), the segment
count of the column tables, its ratio to cameras * fW * D, and which form of the lift the default cap selects.
Prints the card name and power limit read in the same run; writes OUT_DIR/lss_rebuild_bench.json.  Needs a CUDA
device: there is no CPU path."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200.bev_pool import BEVPoolPlan  # noqa: E402
from bevfusion_b200.vtransform import create_frustum  # noqa: E402

KEYS = ("camera2lidar_rots", "camera2lidar_trans", "intrins", "post_rots", "post_trans", "extra_rots", "extra_trans")


def card_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (v.strip() for v in q.split(","))
    return {"name": name, "power_limit": power, "clocks_max_sm": clock}


def calibrations(cfg, batch, seeds, dev):
    out = []
    for s in seeds:
        r = S.augmented_rig(cfg["n_cam"], cfg["image_size"], batch, s)
        out.append([r[k].to(dev) for k in KEYS])
    return out


def step_ms(step, n_cal, steps):
    """median over three rounds of the mean CUDA-event time of one step (calibration i % n_cal at step i)"""
    rounds = []
    for _ in range(3):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for i in range(steps):
            step(i % n_cal)
        stop.record()
        stop.synchronize()
        rounds.append(start.elapsed_time(stop) / steps)
    return statistics.median(rounds)


def time_config(name, batch, steps, dev):
    cfg = S.CONFIGS[name]
    fr = create_frustum(cfg["image_size"], cfg["feature_size"], cfg["dbound"]).to(dev)
    bounds = (cfg["xbound"], cfg["ybound"], cfg["zbound"])
    cals = calibrations(cfg, batch, range(1000, 1008), dev)
    D, fH, fW = fr.shape[:3]
    N, C = cfg["n_cam"], cfg["C"]
    g = torch.Generator(device=dev).manual_seed(0)
    depth = torch.softmax(torch.randn(batch, N, D, fH, fW, generator=g, device=dev), dim=2).contiguous()
    depth.requires_grad_(True)
    ctx = torch.randn(batch, N, fH, fW, C, generator=g, device=dev).requires_grad_(True)

    def host_step(i):
        c = cals[i]
        plan = BEVPoolPlan.from_cameras(fr, *c[:5], *bounds, c[5], c[6])
        torch.autograd.grad(plan.lift_pool(depth, ctx), (depth, ctx), G)

    plan = BEVPoolPlan.from_cameras(fr, *cals[0][:5], *bounds, cals[0][5], cals[0][6], sync=False)
    G = torch.randn(*plan.tables.dims, C, generator=g, device=dev)

    def free_step(i):
        plan.rebuild_(*cals[i])
        torch.autograd.grad(plan.lift_pool(depth, ctx), (depth, ctx), G)

    static = [t.clone() for t in cals[0]]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for i in range(3):
            host_step(i)
            free_step(i)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        plan.rebuild_(*static)
        torch.autograd.grad(plan.lift_pool(depth, ctx), (depth, ctx), G)

    def graph_step(i):
        for dst, src in zip(static, cals[i]):
            dst.copy_(src)
        graph.replay()

    with torch.no_grad():
        graph_step(1)
    torch.cuda.synchronize()
    res = {}
    for _ in range(2):                     # alternate the three paths twice; keep the second pass
        res = {"a_host_count_eager_ms": step_ms(host_step, len(cals), steps),
               "b_sync_free_eager_ms": step_ms(free_step, len(cals), steps)}
        with torch.no_grad():
            res["c_sync_free_graph_ms"] = step_ms(graph_step, len(cals), steps)
    res.update(config=name, batch=batch, C=C, max_segments=plan.max_segments,
               c_over_a=round(res["c_sync_free_graph_ms"] / res["a_host_count_eager_ms"], 4))
    del graph, plan
    torch.cuda.empty_cache()
    return res


def segment_stats(name, draws, dev):
    cfg = S.CONFIGS[name]
    fr = create_frustum(cfg["image_size"], cfg["feature_size"], cfg["dbound"]).to(dev)
    bounds = (cfg["xbound"], cfg["ybound"], cfg["zbound"])
    D, fH, fW = fr.shape[:3]
    pairs = cfg["n_cam"] * fW * D
    c0 = calibrations(cfg, 1, [0], dev)[0]
    plan = BEVPoolPlan.from_cameras(fr, *c0[:5], *bounds, c0[5], c0[6], sync=False)
    counts, forms = [], []
    for seed in range(draws):
        plan.rebuild_(*calibrations(cfg, 1, [seed], dev)[0])
        n_seg, form = (int(v) for v in plan.tables.counts[2:4].tolist())
        counts.append(n_seg)
        forms.append(form)
    rig = S.camera_rig(cfg["n_cam"], cfg["image_size"], 1)
    plan.rebuild_(*[rig[k].to(dev) for k in KEYS[:5]])
    level_count = int(plan.tables.counts[2])
    return {"config": name, "draws": draws, "cameras_fW_D": pairs, "level_rig_segments": level_count,
            "min": min(counts), "median": int(statistics.median(counts)), "max": max(counts),
            "max_over_cameras_fW_D": round(max(counts) / pairs, 4), "default_cap": plan.max_segments,
            "draws_on_rows": sum(forms), "draws_on_columns": len(forms) - sum(forms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--draws", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lss_rebuild_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = card_info()
    print("card: %(name)s, power limit %(power_limit)s, max SM clock %(clocks_max_sm)s" % card)
    result = {"card": card, "segments": [], "steps": []}
    for name in ("C2", "C5"):
        st = segment_stats(name, args.draws, dev)
        print(json.dumps(st))
        result["segments"].append(st)
    for name, batch in (("C2", 1), ("C2", 4), ("C5", 1)):
        r = time_config(name, batch, args.steps, dev)
        print(json.dumps(r))
        result["steps"].append(r)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "lss_rebuild_bench.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
