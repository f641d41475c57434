"""Heatmap training targets of both detection heads on synthetic.gt_boxes (40-120 boxes per sample) at batch 1 and 4:
CenterHead with the six nuScenes tasks on the 128 x 128 map (grid 1024, out_size_factor 8), TransFusion with ten
classes on the 180 x 180 map (grid 1440, out_size_factor 8).

    python tools/head_targets_bench.py OUT_DIR [--window 1.0]

(a) reference loop: CenterHead.get_targets_single / the heatmap loop of TransFusionHead.get_targets_single
            (centerpoint.py:432-582, transfusion.py:526-573, gaussian.py) restated here op for op on CUDA tensors,
            one sample at a time, stacked as get_targets does
(b) eager:  bevfusion_b200.head_targets.centerhead_targets / transfusion_heatmap_targets (list form: padding,
            one native call)
(c) graph:  the batched form on padded inputs as one CUDA graph replay
Host clock around each batch with a device synchronise at its end for (a); CUDA events over windows of at least
--window seconds after a warm-up for (b) and (c); the median of three alternating rounds.  Also the kernel launches
per native call, whether (a) and (b) agree (heatmap cells, ind, mask), and the card name / power limit read in the
same run.  Writes OUT_DIR/head_targets_bench.json.  Needs a CUDA device."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from bevfusion_b200 import _C  # noqa: E402
from bevfusion_b200 import head_targets as H  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402

CFG_CH = dict(point_cloud_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], grid_size=[1024, 1024, 40],
              voxel_size=[0.1, 0.1, 0.2], out_size_factor=8, dense_reg=1, gaussian_overlap=0.1, max_objs=500,
              min_radius=2)
CFG_TF = dict(point_cloud_range=[-54.0, -54.0, -5.0, 54.0, 54.0, 3.0], grid_size=[1440, 1440, 41],
              voxel_size=[0.075, 0.075, 0.2], out_size_factor=8, gaussian_overlap=0.1, min_radius=2)
TASKS = [[n for n, _ in t] for t in S.CENTERHEAD_TASKS]


def card_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (v.strip() for v in q.split(","))
    return {"name": name, "power_limit": power, "clocks_max_sm": clock}


# ---- (a) the reference's per-object loop, restated on CUDA tensors -----------------------------------------------
def gaussian_2d(shape, sigma=1):
    m, n = [(ss - 1.0) / 2.0 for ss in shape]
    y, x = np.ogrid[-m:m + 1, -n:n + 1]
    h = np.exp(-(x * x + y * y) / (2 * sigma * sigma))
    h[h < np.finfo(h.dtype).eps * h.max()] = 0
    return h


def draw_heatmap_gaussian(heatmap, center, radius, k=1):
    diameter = 2 * radius + 1
    gaussian = gaussian_2d((diameter, diameter), sigma=diameter / 6)
    x, y = int(center[0]), int(center[1])
    height, width = heatmap.shape[0:2]
    left, right = min(x, radius), min(width - x, radius + 1)
    top, bottom = min(y, radius), min(height - y, radius + 1)
    masked_heatmap = heatmap[y - top:y + bottom, x - left:x + right]
    masked_gaussian = torch.from_numpy(gaussian[radius - top:radius + bottom, radius - left:radius + right]).to(
        heatmap.device, torch.float32)
    if min(masked_gaussian.shape) > 0 and min(masked_heatmap.shape) > 0:
        torch.max(masked_heatmap, masked_gaussian * k, out=masked_heatmap)
    return heatmap


def gaussian_radius(det_size, min_overlap=0.5):
    height, width = det_size
    a1 = 1
    b1 = height + width
    c1 = width * height * (1 - min_overlap) / (1 + min_overlap)
    r1 = (b1 + torch.sqrt(b1 ** 2 - 4 * a1 * c1)) / 2
    a2 = 4
    b2 = 2 * (height + width)
    c2 = (1 - min_overlap) * width * height
    r2 = (b2 + torch.sqrt(b2 ** 2 - 4 * a2 * c2)) / 2
    a3 = 4 * min_overlap
    b3 = -2 * min_overlap * (height + width)
    c3 = (min_overlap - 1) * width * height
    r3 = (b3 + torch.sqrt(b3 ** 2 - 4 * a3 * c3)) / 2
    return min(r1, r2, r3)


def gravity_boxes(t):
    c = t[:, :3].clone()
    c[:, 2] = t[:, 2] + t[:, 5] * 0.5
    return torch.cat((c, t[:, 3:]), dim=1)


def ref_centerhead_single(cfg, boxes, labels, norm_bbox=True):
    device = labels.device
    gt = gravity_boxes(boxes)
    max_objs = cfg["max_objs"] * cfg["dense_reg"]
    grid_size, pc_range = torch.tensor(cfg["grid_size"]), torch.tensor(cfg["point_cloud_range"])
    voxel_size = torch.tensor(cfg["voxel_size"])
    fms = torch.div(grid_size[:2], cfg["out_size_factor"], rounding_mode="trunc")
    task_masks, flag = [], 0
    for class_name in TASKS:
        task_masks.append([torch.where(labels == class_name.index(i) + flag) for i in class_name])
        flag += len(class_name)
    task_boxes, task_classes, flag2 = [], [], 0
    for mask in task_masks:
        task_boxes.append(torch.cat([gt[m] for m in mask], axis=0).to(device))
        task_classes.append(torch.cat([labels[m] + 1 - flag2 for m in mask]).long().to(device))
        flag2 += len(mask)
    heatmaps, anno_boxes, inds, masks = [], [], [], []
    for idx in range(len(TASKS)):
        heatmap = gt.new_zeros((len(TASKS[idx]), fms[1], fms[0]))
        anno_box = gt.new_zeros((max_objs, 10), dtype=torch.float32)
        ind = labels.new_zeros((max_objs), dtype=torch.int64)
        mask = gt.new_zeros((max_objs), dtype=torch.uint8)
        for k in range(min(task_boxes[idx].shape[0], max_objs)):
            cls_id = task_classes[idx][k] - 1
            width = task_boxes[idx][k][3] / voxel_size[0] / cfg["out_size_factor"]
            length = task_boxes[idx][k][4] / voxel_size[1] / cfg["out_size_factor"]
            if width > 0 and length > 0:
                radius = max(cfg["min_radius"], int(gaussian_radius((length, width), cfg["gaussian_overlap"])))
                x, y, z = task_boxes[idx][k][0], task_boxes[idx][k][1], task_boxes[idx][k][2]
                coor_x = (x - pc_range[0]) / voxel_size[0] / cfg["out_size_factor"]
                coor_y = (y - pc_range[1]) / voxel_size[1] / cfg["out_size_factor"]
                center = torch.tensor([coor_x, coor_y], dtype=torch.float32, device=device)
                center_int = center.to(torch.int32)
                if not (0 <= center_int[0] < fms[0] and 0 <= center_int[1] < fms[1]):
                    continue
                draw_heatmap_gaussian(heatmap[cls_id], center_int[[1, 0]], radius)
                x, y = center_int[0], center_int[1]
                ind[k] = x * fms[1] + y
                mask[k] = 1
                vx, vy = task_boxes[idx][k][7:]
                rot = task_boxes[idx][k][6]
                box_dim = task_boxes[idx][k][3:6]
                if norm_bbox:
                    box_dim = box_dim.log()
                anno_box[k] = torch.cat([center - torch.tensor([x, y], device=device), z.unsqueeze(0), box_dim,
                                         torch.sin(rot).unsqueeze(0), torch.cos(rot).unsqueeze(0), vx.unsqueeze(0),
                                         vy.unsqueeze(0)])
        heatmaps.append(heatmap)
        anno_boxes.append(anno_box)
        masks.append(mask)
        inds.append(ind)
    return heatmaps, anno_boxes, inds, masks


def ref_centerhead(cfg, boxes, labels):
    per = [ref_centerhead_single(cfg, b, l) for b, l in zip(boxes, labels)]
    return tuple([torch.stack([p[k][t] for p in per]) for t in range(len(TASKS))] for k in range(4))


def ref_transfusion_single(cfg, boxes, labels, num_classes=10):
    device = labels.device
    gt = gravity_boxes(boxes)
    grid_size, pc_range = torch.tensor(cfg["grid_size"]), torch.tensor(cfg["point_cloud_range"])
    voxel_size = torch.tensor(cfg["voxel_size"])
    fms = grid_size[:2] // cfg["out_size_factor"]
    heatmap = gt.new_zeros(num_classes, fms[1], fms[0])
    for idx in range(len(gt)):
        width = gt[idx][3] / voxel_size[0] / cfg["out_size_factor"]
        length = gt[idx][4] / voxel_size[1] / cfg["out_size_factor"]
        if width > 0 and length > 0:
            radius = max(cfg["min_radius"], int(gaussian_radius((length, width), cfg["gaussian_overlap"])))
            x, y = gt[idx][0], gt[idx][1]
            coor_x = (x - pc_range[0]) / voxel_size[0] / cfg["out_size_factor"]
            coor_y = (y - pc_range[1]) / voxel_size[1] / cfg["out_size_factor"]
            center = torch.tensor([coor_x, coor_y], dtype=torch.float32, device=device)
            center_int = center.to(torch.int32)
            draw_heatmap_gaussian(heatmap[labels[idx]], center_int[[1, 0]], radius)
    return heatmap


def ref_transfusion(cfg, boxes, labels):
    return torch.stack([ref_transfusion_single(cfg, b, l) for b, l in zip(boxes, labels)])


# ---- timing ---------------------------------------------------------------------------------------------------------
def host_ms(fn, reps):
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / reps


def timed_ms(fn, window_s):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    n = max(20, int(window_s * 1e3 / max(start.elapsed_time(stop), 1e-3)) + 1)
    start.record()
    for _ in range(n):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / n


def bench(head, batch, window, dev):
    bl, ll = S.gt_boxes(seed=batch, batch=batch)
    bl = [b.to(dev) for b in bl]
    ll = [l.to(dev) for l in ll]
    if head == "centerhead":
        cfg = CFG_CH
        ref = lambda: ref_centerhead(cfg, bl, ll)                                  # noqa: E731
        eager = lambda: H.centerhead_targets(bl, ll, TASKS, cfg)                   # noqa: E731
        pb, pl, pc = H.pad_gt(bl, ll)
        batched = lambda: H.centerhead_targets_batched(pb, pl, pc, TASKS, cfg)     # noqa: E731
    else:
        cfg = CFG_TF
        ref = lambda: ref_transfusion(cfg, bl, ll)                                 # noqa: E731
        eager = lambda: H.transfusion_heatmap_targets(bl, ll, 10, cfg)             # noqa: E731
        pb, pl, pc = H.pad_gt(bl, ll)
        batched = lambda: H.transfusion_heatmap_targets_batched(pb, pl, pc, 10, cfg)   # noqa: E731
    a, b = ref(), eager()
    torch.cuda.synchronize()
    if head == "centerhead":
        agree = dict(heatmap_cells_differing=int(sum((x != y).sum() for x, y in zip(a[0], b[0]))),
                     ind_equal=all(torch.equal(x, y) for x, y in zip(a[2], b[2])),
                     mask_equal=all(torch.equal(x, y) for x, y in zip(a[3], b[3])),
                     anno_max_abs=float(max((x - y).abs().max() for x, y in zip(a[1], b[1]))))
    else:
        agree = dict(heatmap_cells_differing=int((a != b).sum()))
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
    rounds = dict(reference_loop=[], eager=[], graph=[])
    for _ in range(3):
        rounds["reference_loop"].append(host_ms(ref, 5))
        rounds["eager"].append(timed_ms(eager, window))
        rounds["graph"].append(timed_ms(g.replay, window))
    ms = {k: statistics.median(v) for k, v in rounds.items()}
    return dict(head=head, batch=batch, boxes=[int(b.shape[0]) for b in bl], ms=ms, rounds=rounds,
                launches_per_call=launches, reference_vs_device=agree,
                speedup_eager=ms["reference_loop"] / ms["eager"], speedup_graph=ms["reference_loop"] / ms["graph"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--window", type=float, default=1.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("head_targets_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    os.makedirs(args.out_dir, exist_ok=True)
    result = dict(card=card_info(), runs=[])
    for head in ("centerhead", "transfusion"):
        for batch in (1, 4):
            r = bench(head, batch, args.window, dev)
            result["runs"].append(r)
            print(json.dumps({k: r[k] for k in ("head", "batch", "ms", "launches_per_call", "reference_vs_device")}))
    with open(os.path.join(args.out_dir, "head_targets_bench.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
