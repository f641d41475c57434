"""The NMS step of CenterHead.get_bboxes for the camera+radar config (nms_type [circle, rotate, rotate, circle,
rotate, rotate], per-class nms_scale, nms_thr 0.2, pre_max_size 1000, post_max_size 83, min_radius
[4, 12, 10, 1, 0.85, 0.175]) over all six tasks, on synthetic.centerhead_detections at batch 1 and 4:

    python tools/nms_bench.py OUT_DIR [--window 1.0]

(a) eager:  bevfusion_b200.iou3d.centerhead_nms per task (one nms_batched call per task, one read of the
            kept counts per task to split the result per sample)
(b) graph:  the padded core (sort, pre-max cut, pair mask, suppression, for all six tasks) as one CUDA graph,
            inputs already padded and thresholded
(c) reference loop: per rotate (task, sample) the reference's own iou3d_cuda_ref.nms_gpu through iou3d_utils'
            call sequence (score threshold, nms_scale, xywhr2xyxyr, sort, pre-max cut, D2H mask copy and host
            loop in the op, post-max cut, post_center_limit_range), per circle (task, sample) a numba restatement
            of circle_nms on the host; only when oracle/_ref holds iou3d_cuda_ref
Reports CUDA-event times over windows of at least --window seconds after a warm-up, three alternating rounds,
the median; then a torch.profiler pass gives each kernel's device time per call of (a).  Also the largest IoU
error of boxes_iou_bev against float64 (tests/nms_oracle.py) and against iou3d_cuda_ref on the synthetic boxes,
and the card name / power limit read in the same run.  Writes OUT_DIR/nms_bench.json.  Needs a CUDA device."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bevfusion_b200 import iou3d  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402
import nms_oracle as O  # noqa: E402

CFG = S.CENTERHEAD_TEST_CFG
TYPES, SCALES = S.CENTERHEAD_RADAR_NMS_TYPE, S.CENTERHEAD_RADAR_NMS_SCALE


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
    return start.elapsed_time(stop) / n


def kernel_us(fn, calls=20):
    """mean device time per fn() call of each kernel / memset / copy, from torch.profiler in a pass of its own"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            out[e.key[:80]] = t / calls
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def circle_nms_host():
    import numba

    @numba.jit(nopython=True)
    def circle(dets, thresh, post_max_size):
        """greedy circle NMS over dets [N, 3] (x, y, score) sorted on the host, as box3d_nms.circle_nms does"""
        x, y = dets[:, 0], dets[:, 1]
        order = dets[:, 2].argsort()[::-1].astype(np.int32)
        n = dets.shape[0]
        suppressed = np.zeros(n, dtype=np.int32)
        keep = []
        for a in range(n):
            i = order[a]
            if suppressed[i] == 1:
                continue
            keep.append(i)
            for b in range(a + 1, n):
                j = order[b]
                if suppressed[j] == 1:
                    continue
                if (x[i] - x[j]) ** 2 + (y[i] - y[j]) ** 2 <= thresh:
                    suppressed[j] = 1
        return keep[:post_max_size]
    return circle


def reference_loop(ref, circle, dets_dev):
    """get_bboxes' per-(task, sample) NMS with the reference's own nms_gpu (iou3d_utils.py:24-48) and a host
    circle NMS (centerpoint.py:710-737, 768-884)."""
    out = []
    rng = torch.tensor(CFG["post_center_limit_range"], device=dets_dev[0][0]["bboxes"].device)
    for task_id, (nms_type, scale) in enumerate(zip(TYPES, SCALES)):
        for d in dets_dev[task_id]:
            boxes3d, scores, labels = d["bboxes"], d["scores"], d["labels"]
            if nms_type == "circle":
                dets = torch.cat([boxes3d[:, [0, 1]], scores.view(-1, 1)], dim=1)
                keep = torch.tensor(circle(dets.cpu().numpy(), CFG["min_radius"][task_id], CFG["post_max_size"]),
                                    dtype=torch.long, device=boxes3d.device)
                out.append((boxes3d[keep], scores[keep], labels[keep]))
                continue
            m = scores >= CFG["score_threshold"]
            s, b, lab = scores.masked_select(m), boxes3d[m], labels[m].long()
            if s.shape[0] == 0:
                out.append((b, s, lab))
                continue
            bev = b[:, [0, 1, 3, 4, 6]]
            for cls, sc in enumerate(scale):
                cur = bev[lab == cls]
                cur[:, [2, 3]] *= sc
                bev[lab == cls] = cur
            order = s.sort(0, descending=True)[1][:CFG["pre_max_size"]]
            xy = iou3d.xywhr2xyxyr(bev)[order].contiguous()
            keep = torch.zeros(xy.size(0), dtype=torch.long)
            num = ref.nms_gpu(xy, keep, CFG["nms_thr"], xy.device.index)
            sel = order[keep[:num].cuda(xy.device)][:CFG["post_max_size"]]
            sb = b[sel]
            mk = (sb[:, :3] >= rng[:3]).all(1) & (sb[:, :3] <= rng[3:]).all(1)
            out.append((sb[mk], s[sel][mk], lab[sel][mk]))
    return out


def padded_core_inputs(dets_dev):
    """per task: the padded, thresholded inputs of the nms_batched call centerhead_nms makes"""
    calls = []
    for task_id, (nms_type, scale) in enumerate(zip(TYPES, SCALES)):
        ds = dets_dev[task_id]
        dev = ds[0]["bboxes"].device
        n = max(d["bboxes"].shape[0] for d in ds)
        pb = torch.zeros(len(ds), n, 9, device=dev)
        ps = torch.full((len(ds), n), float("-inf"), device=dev)
        pl = torch.zeros(len(ds), n, dtype=torch.long, device=dev)
        for i, d in enumerate(ds):
            k = d["bboxes"].shape[0]
            pb[i, :k], ps[i, :k], pl[i, :k] = d["bboxes"], d["scores"], d["labels"]
        if nms_type == "circle":
            counts = torch.tensor([d["bboxes"].shape[0] for d in ds], dtype=torch.int32, device=dev)
            calls.append((pb[..., :2].contiguous(), ps, counts, "circle", CFG["min_radius"][task_id], None))
            continue
        live = ps >= CFG["score_threshold"]
        perm = torch.argsort((~live).to(torch.int8), dim=1, stable=True)
        bev = pb[..., [0, 1, 3, 4, 6]]
        bev[..., 2:4] *= torch.tensor(scale, device=dev)[pl.clamp(max=len(scale) - 1)][..., None]
        xy = iou3d.xywhr2xyxyr(bev).gather(1, perm[..., None].expand(-1, -1, 5)).contiguous()
        calls.append((xy, ps.gather(1, perm), live.sum(1, dtype=torch.int32), "rotate", CFG["nms_thr"],
                      CFG["pre_max_size"]))
    return calls


def iou_errors(dets, ref, dev):
    """largest |IoU - float64| and |IoU - reference op| over the rotate tasks' boxes of the first sample (the
    reference off the diagonal: it misses corners of some boxes compared with themselves far from the origin,
    counted separately)"""
    e64, eref, eref64, pairs, self_bad, self_n, sd = 0.0, 0.0, 0.0, 0, 0, 0, 0.0
    for task_id in (1, 2, 4, 5):
        d = dets[task_id][0]
        bev = d["bboxes"][:, [0, 1, 3, 4, 6]].clone()
        xy = iou3d.xywhr2xyxyr(bev).numpy()
        b = torch.from_numpy(xy).to(dev)
        got = iou3d.boxes_iou_bev(b, b).cpu().numpy()
        gold = O.iou_matrix(xy, xy)
        e64 = max(e64, float(np.abs(got - gold).max()))
        sd = max(sd, float(np.abs(np.diagonal(got) - 1).max()))
        pairs += int((gold > 0).sum())
        if ref is not None:
            r = torch.zeros(len(xy), len(xy), device=dev)
            ref.boxes_iou_bev_gpu(b, b, r)
            r = r.cpu().numpy()
            off = ~np.eye(len(xy), dtype=bool)
            eref = max(eref, float(np.abs(got - r)[off].max()))
            eref64 = max(eref64, float(np.abs(r - gold)[off].max()))
            self_bad += int((np.abs(np.diagonal(r) - 1) > 1e-3).sum())
            self_n += len(xy)
    return {"max_abs_err_vs_float64": e64, "overlapping_pairs": pairs,
            "max_abs_err_vs_reference_offdiag": eref if ref is not None else None,
            "reference_max_abs_err_vs_float64_offdiag": eref64 if ref is not None else None,
            "reference_self_iou_off_by_1e-3": [self_bad, self_n] if ref is not None else None,
            "self_iou_max_abs_err": sd}


def run_batch(batch, window, ref, circle):
    dev = torch.device("cuda:0")
    dets = S.centerhead_detections(seed=batch, batch=batch)
    dets_dev = [[{k: v.to(dev) for k, v in d.items()} for d in task] for task in dets]

    def run_a():
        return [iou3d.centerhead_nms(dets_dev[t], t, TYPES[t], CFG, SCALES[t], len(S.CENTERHEAD_TASKS[t]))
                for t in range(6)]

    calls = padded_core_inputs(dets_dev)

    def run_core():
        return [iou3d.nms_batched(b, s, c, m, th, pre, CFG["post_max_size"]) for b, s, c, m, th, pre in calls]

    for _ in range(3):
        run_a()
        run_core()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run_core()
    torch.cuda.current_stream().wait_stream(side)
    with torch.cuda.graph(graph):
        graph_out = run_core()
    graph.replay()
    eager_core = run_core()
    torch.cuda.synchronize()
    for (kg, cg), (ke, ce) in zip(graph_out, eager_core):
        assert torch.equal(kg, ke) and torch.equal(cg, ce), "graph replay differs from eager"
    runs = {"a_eager": run_a, "b_graph": graph.replay}
    if ref is not None:
        def run_c():
            return reference_loop(ref, circle, dets_dev)
        got = [x for t in run_a() for x in t]
        want = run_c()
        same = all(torch.equal(g["bboxes"], w[0]) and torch.equal(g["scores"], w[1]) and torch.equal(g["labels"], w[2])
                   for g, w in zip(got, want))
        runs["c_reference_loop"] = run_c
    else:
        same = None
    for fn in runs.values():
        fn()
    torch.cuda.synchronize()
    rounds = {k: [] for k in runs}
    for _ in range(3):
        for k, fn in runs.items():
            rounds[k].append(timed_ms(fn, window))
    return {
        "batch": batch,
        "boxes_per_task": [[int(d["bboxes"].shape[0]) for d in task] for task in dets],
        "ms": {k: statistics.median(v) for k, v in rounds.items()},
        "rounds_ms": rounds,
        "a_equals_c": same,
        "kernels_us_per_call_a": kernel_us(run_a),
        "iou": iou_errors(dets, ref, dev),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--window", type=float, default=1.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nms_bench needs a CUDA device: there is no CPU path")
    os.makedirs(args.out_dir, exist_ok=True)
    from conftest import ref_module
    ref = ref_module("iou3d_cuda_ref")
    try:
        circle = circle_nms_host()
    except ImportError:
        circle = None
    if circle is None:
        ref = None                                       # the reference loop needs its host circle NMS
    result = {"card": card_info(), "window_s": args.window, "reference_built": ref is not None,
              "runs": [run_batch(b, args.window, ref, circle) for b in (1, 4)]}
    with open(os.path.join(args.out_dir, "nms_bench.json"), "w") as f:
        json.dump(result, f, indent=1)
    for r in result["runs"]:
        print(json.dumps({"batch": r["batch"], "ms": r["ms"], "a_equals_c": r["a_equals_c"], "iou": r["iou"]}))
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
