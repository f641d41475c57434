"""CenterHead.get_bboxes, head outputs in and boxes out, for the camera+radar config (six nuScenes tasks on a
128 x 128 map, max_num 500, score_threshold 0.1, nms_type [circle, rotate, rotate, circle, rotate, rotate], per-class
nms_scale, post_max_size 83) on synthetic.centerhead_head_outputs at batch 1 and 4:

    python tools/centerhead_decode_bench.py OUT_DIR [--window 1.0]       timings -> OUT_DIR/centerhead_decode_bench.json
    python tools/centerhead_decode_bench.py OUT_DIR --profile            a torch.profiler run of its own ->
                                                                         OUT_DIR/centerhead_decode_profile.json

(a) restated:  the reference's lines on CUDA tensors (tests/centerhead_decode_oracle.py: per task sigmoid, exp, the
               coder's two top-k stages, gathers, masks and per-sample boolean indexing) + iou3d.centerhead_nms + merge
(b) eager:     centerhead_decode.centerhead_get_bboxes (one decode call, centerhead_nms_batched per task, one
               read-back)
(c) graph:     centerhead_get_bboxes_batched as one CUDA graph replay
(d) decode:    centerhead_decode_batched alone (its two kernels) as a CUDA graph replay
Timings are CUDA-event means over windows of at least --window seconds after a warm-up, three alternating rounds,
the median.  The profile run gives, per call of each row, the device time of every kernel and the numbers of kernel
launches and device-to-host copies.  Also: (b) against (a) (same rows; largest ulp distance of sizes and yaw), the
algorithmic bytes of the decode from the shapes, and the card's name and power limit read in the same run.  Reads
nothing outside the repository.  Needs a CUDA device."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bevfusion_b200 import centerhead_decode as CD  # noqa: E402
from bevfusion_b200 import iou3d  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402
import centerhead_decode_oracle as O  # noqa: E402

H = W = 128
NUM_CLASSES = [len(c) for c in S.CENTERHEAD_TASKS]
CODER = S.centerhead_coder_cfg(H, W, max_num=500, score_threshold=0.1)
TEST_CFG = dict(S.CENTERHEAD_TEST_CFG, nms_type=list(S.CENTERHEAD_RADAR_NMS_TYPE),
                nms_scale=[list(s) for s in S.CENTERHEAD_RADAR_NMS_SCALE])


def card_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (v.strip() for v in q.split(","))
    return {"name": name, "power_limit": power, "clocks_max_sm": clock}


def timed_ms(fn, window_s):
    """mean CUDA-event time of fn() over a window of at least window_s seconds (after the caller's warm-up)"""
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
    return start.elapsed_time(stop) / n


def profile_row(fn, calls=20):
    """per fn() call: device time of each kernel / copy (us), kernel launches and device-to-host copies"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    dev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    d2h = sum("DtoH" in e.name or "Device -> Host" in e.name for e in dev)
    kernels = sum("Memcpy" not in e.name and "Memset" not in e.name for e in dev)
    times = {}
    for e in dev:
        times[e.name[:80]] = times.get(e.name[:80], 0.0) + e.device_time_total / calls
    return {"kernel_launches_per_call": kernels / calls, "d2h_copies_per_call": d2h / calls,
            "device_us_per_call": sum(times.values()),
            "kernels_us_per_call": dict(sorted(times.items(), key=lambda kv: -kv[1])[:12])}


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


def ulp_distance(a, b):
    def key(x):
        i = x.contiguous().view(torch.int32).long()
        return torch.where(i < 0, -(i & 0x7fffffff), i)
    return int((key(a) - key(b)).abs().max()) if a.numel() else 0


def decode_bytes(batch, candidates):
    """algorithmic bytes of one decode: every heatmap read once, 8 bytes per candidate written and read about twice,
    max_num rows of 10 regression values and the score gathered, the outputs written"""
    K, S_ = CODER["max_num"], 6 * batch
    return {"heatmap_read": 4 * batch * sum(NUM_CLASSES) * H * W, "candidate_keys": 8 * 3 * candidates,
            "gathered_rows": 4 * 11 * K * S_, "outputs": 4 * (9 + 2) * K * S_ + 4 * S_}


def rows_for(batch):
    dev = torch.device("cuda:0")
    preds = [[{k: v.to(dev) for k, v in t.items()}] for t in S.centerhead_head_outputs(batch, batch, H, W)]
    tasks = [p[0] for p in preds]
    runs = {
        "a_restated": lambda: O.torch_get_bboxes(preds, CODER, TEST_CFG, NUM_CLASSES, True, iou3d.centerhead_nms),
        "b_eager": lambda: CD.centerhead_get_bboxes(preds, CODER, TEST_CFG, NUM_CLASSES),
        "c_batched": lambda: CD.centerhead_get_bboxes_batched(preds, CODER, TEST_CFG, NUM_CLASSES),
        "d_decode": lambda: CD.centerhead_decode_batched(tasks, CODER),
    }
    for fn in runs.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    return preds, tasks, runs


def run_batch(batch, window):
    preds, tasks, runs = rows_for(batch)
    want, got = runs["a_restated"](), runs["b_eager"]()
    same_rows = all(torch.equal(g[1], w[1]) and torch.equal(g[2], w[2]) for g, w in zip(got, want))
    ulp = max(ulp_distance(g[0], w[0]) for g, w in zip(got, want)) if same_rows else None
    graph_c, out_c = graph_of(runs["c_batched"])
    graph_d, out_d = graph_of(runs["d_decode"])
    graph_c.replay()
    torch.cuda.synchronize()
    eager_c = runs["c_batched"]()
    assert all(torch.equal(x, y) for x, y in zip(out_c, eager_c)), "graph replay differs from eager"
    timed = {"a_restated": runs["a_restated"], "b_eager": runs["b_eager"], "c_graph": graph_c.replay,
             "d_decode_graph": graph_d.replay}
    rounds = {k: [] for k in timed}
    for _ in range(3):
        for k, fn in timed.items():
            rounds[k].append(timed_ms(fn, window))
    counts = out_d[3]
    candidates = sum(int((t["heatmap"].sigmoid() > CODER["score_threshold"]).sum()) for t in tasks)
    return {"batch": batch, "ms": {k: statistics.median(v) for k, v in rounds.items()}, "rounds_ms": rounds,
            "b_rows_equal_a": same_rows, "b_boxes_max_ulp_from_a": ulp,
            "detections_per_sample": [len(g[1]) for g in got],
            "decoded_rows_per_task_sample": counts.tolist(), "candidates": candidates,
            "decode_bytes": decode_bytes(batch, candidates)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("centerhead_decode_bench needs a CUDA device: there is no CPU path")
    os.makedirs(args.out_dir, exist_ok=True)
    result = {"card": card_info(), "map": [H, W], "coder": CODER}
    if args.profile:
        result["runs"] = []
        for batch in (1, 4):
            _, _, runs = rows_for(batch)
            result["runs"].append({"batch": batch, **{k: profile_row(fn) for k, fn in runs.items()}})
        name = "centerhead_decode_profile.json"
    else:
        result["window_s"] = args.window
        result["runs"] = [run_batch(b, args.window) for b in (1, 4)]
        name = "centerhead_decode_bench.json"
    with open(os.path.join(args.out_dir, name), "w") as f:
        json.dump(result, f, indent=1)
    for r in result["runs"]:
        if args.profile:
            print(json.dumps({"batch": r["batch"], **{k: {m: v[m] for m in ("kernel_launches_per_call",
                                                                           "d2h_copies_per_call",
                                                                           "device_us_per_call")}
                                                      for k, v in r.items() if k != "batch"}}))
            print(json.dumps({"batch": r["batch"], "d_decode_kernels_us": r["d_decode"]["kernels_us_per_call"]}))
        else:
            print(json.dumps({k: r[k] for k in ("batch", "ms", "b_rows_equal_a", "b_boxes_max_ulp_from_a",
                                                "detections_per_sample", "candidates", "decode_bytes")}))
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
