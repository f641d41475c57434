"""Generates tests/golden/head_targets_tiny.npz from the REFERENCE's own code, on the CPU:

  - mmdet3d/core/utils/gaussian.py, executed as it is;
  - CenterHead.get_targets_single (models/heads/bbox/centerpoint.py), pulled out with `ast` and called with a
    stub `self` (train_cfg, class_names, task_heads, norm_bbox) and a stub box class (tensor, gravity_center);
  - the dense-heatmap block of TransFusionHead.get_targets_single (models/heads/bbox/transfusion.py), the
    statements from `gt_bboxes_3d = torch.cat(...)` through the loop over boxes, taken the same way.

Cases (each a padded batch, see CASES):
  ch_six     the six nuScenes tasks, 128 x 128 map, norm_bbox on, 9-column boxes; sample 1 is empty
  ch_small   the six tasks on a non-square 80 x 64 map, norm_bbox off, 7-column boxes (the reference's output on
             the same boxes with zero velocity, velocity columns dropped), max_objs 6 with more cars than that
  tf_ten     TransFusion, 10 classes, 180 x 180 map, 9-column boxes
  tf_wide    TransFusion on a non-square 72 x 90 map, 7-column boxes
Every case mixes random nuScenes-like boxes with named ones: labels of no task (10, 11, -1; CenterHead only), zero
and negative sizes, NaN sizes, centres in (-1, 0) cells, exactly on the map border, and r - 1, r, r + 1 cells
outside it, clusters of same-class boxes whose gaussians overlap, and sizes whose fp32 radius lies just below or
just above an integer.

Run:  python tests/golden/make_head_targets_golden.py      (needs the reference tree)
"""
import ast
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import head_targets_oracle as O  # noqa: E402

REF = os.environ.get("BEVFUSION_REFERENCE", "/root/reference")
TASKS = [["car"], ["truck", "construction_vehicle"], ["bus", "trailer"], ["barrier"], ["motorcycle", "bicycle"],
         ["pedestrian", "traffic_cone"]]
SIZES = [(1.95, 4.6, 1.7), (2.5, 6.9, 2.8), (2.9, 6.4, 3.2), (2.9, 11.5, 3.5), (2.9, 12.0, 3.9), (2.5, 0.5, 1.0),
         (0.8, 2.1, 1.5), (0.6, 1.8, 1.3), (0.7, 0.7, 1.8), (0.3, 0.3, 1.1)]
CFG_SIX = dict(point_cloud_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], grid_size=[1024, 1024, 40],
               voxel_size=[0.1, 0.1, 0.2], out_size_factor=8, dense_reg=1, gaussian_overlap=0.1, max_objs=500,
               min_radius=2)
CFG_SMALL = dict(point_cloud_range=[-25.6, -25.6, -5.0, 25.6, 25.6, 3.0], grid_size=[320, 256, 1],
                 voxel_size=[0.16, 0.2, 8.0], out_size_factor=4, dense_reg=1, gaussian_overlap=0.1, max_objs=6,
                 min_radius=2)
CFG_TF = dict(point_cloud_range=[-54.0, -54.0, -5.0, 54.0, 54.0, 3.0], grid_size=[1440, 1440, 41],
              voxel_size=[0.075, 0.075, 0.2], out_size_factor=8, gaussian_overlap=0.1, min_radius=2)
CFG_TF_WIDE = dict(point_cloud_range=[-21.6, -27.0, -5.0, 21.6, 27.0, 3.0], grid_size=[288, 360, 1],
                   voxel_size=[0.15, 0.15, 8.0], out_size_factor=4, gaussian_overlap=0.2, min_radius=1)


def reference_functions():
    g = {}
    exec(open(REF + "/mmdet3d/core/utils/gaussian.py").read(), g)

    def method(path, cls_name, fn_name):
        tree = ast.parse(open(path).read())
        cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls_name)
        return next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == fn_name)

    ns = dict(torch=torch, draw_heatmap_gaussian=g["draw_heatmap_gaussian"], gaussian_radius=g["gaussian_radius"])
    fn = method(REF + "/mmdet3d/models/heads/bbox/centerpoint.py", "CenterHead", "get_targets_single")
    fn.decorator_list = []
    exec(compile(ast.Module([fn], []), "centerpoint.py", "exec"), ns)
    centerhead = ns["get_targets_single"]

    fn = method(REF + "/mmdet3d/models/heads/bbox/transfusion.py", "TransFusionHead", "get_targets_single")
    start = next(i for i, s in enumerate(fn.body) if isinstance(s, ast.Assign)
                 and ast.unparse(s.targets[0]) == "gt_bboxes_3d" and "gravity_center" in ast.unparse(s.value))
    stop = next(i for i, s in enumerate(fn.body) if i > start and isinstance(s, ast.For))
    body = fn.body[start:stop + 1] + [ast.parse("return heatmap").body[0]]
    args = ast.parse("def f(self, gt_bboxes_3d, gt_labels_3d, device): pass").body[0]
    args.body = body
    ns2 = dict(torch=torch, draw_heatmap_gaussian=g["draw_heatmap_gaussian"], gaussian_radius=g["gaussian_radius"])
    exec(compile(ast.fix_missing_locations(ast.Module([args], [])), "transfusion.py", "exec"), ns2)
    return centerhead, ns2["f"], g["gaussian_radius"]


class Boxes:
    """LiDARInstance3DBoxes as far as the targets use it."""

    def __init__(self, t):
        self.tensor = t

    @property
    def gravity_center(self):
        bottom = self.tensor[:, :3]
        c = torch.zeros_like(bottom)
        c[:, :2] = bottom[:, :2]
        c[:, 2] = bottom[:, 2] + self.tensor[:, 5] * 0.5
        return c

    def __len__(self):
        return self.tensor.shape[0]


def radius_of(gaussian_radius, cfg, dx, dy):
    vs, osf = torch.tensor(cfg["voxel_size"]), cfg["out_size_factor"]
    w = torch.tensor(dx, dtype=torch.float32) / vs[0] / osf
    l = torch.tensor(dy, dtype=torch.float32) / vs[1] / osf
    r = gaussian_radius((l, w), min_overlap=cfg["gaussian_overlap"])
    return max(cfg["min_radius"], int(r)), float(r)


def near_integer_sizes(cfg, rng, n=3):
    """Pairs of (dx, dy) whose fp32 radius lies just below and at or just above an integer >= min_radius + 1:
    for a random dy, the two adjacent fp32 values of dx between which int(r) steps (found by bisection on the
    fp32 bit patterns; r grows with dx)."""
    vs, osf, ov = cfg["voxel_size"], cfg["out_size_factor"], cfg["gaussian_overlap"]

    def radius(dx, dy):
        return O.gaussian_radius(np.float32(dy) / np.float32(vs[1]) / np.float32(osf),
                                 np.float32(dx) / np.float32(vs[0]) / np.float32(osf), ov)

    out = []
    for k in range(n):
        dy = np.float32(rng.uniform(3.0, 14.0))
        target = cfg["min_radius"] + 1 + k
        lo, hi = np.float32(0.01).view(np.int32), np.float32(400.0).view(np.int32)
        if not radius(hi.view(np.float32), dy) >= target:
            continue
        while hi - lo > 1:                                   # positive floats order as their bit patterns
            mid = np.int32((int(lo) + int(hi)) // 2)
            if radius(mid.view(np.float32), dy) >= target:
                hi = mid
            else:
                lo = mid
        out += [(float(lo.view(np.float32)), float(dy)), (float(hi.view(np.float32)), float(dy))]
    return out


def random_boxes(rng, n, cfg, num_labels):
    lab = rng.integers(0, num_labels, n)
    pc = cfg["point_cloud_range"]
    rows = []
    for l in lab:
        w, L, h = np.array(SIZES[l % 10]) * rng.uniform(0.8, 1.2, 3)
        x = rng.uniform(pc[0] - 3, pc[3] + 3)
        y = rng.uniform(pc[1] - 3, pc[4] + 3)
        rows.append([x, y, rng.uniform(-2, 1), w, L, h, rng.uniform(-np.pi, np.pi), *rng.normal(0, 3, 2)])
    return rows, lab.tolist()


def named_boxes(cfg, gaussian_radius, rng, centerhead):
    """The edge cases listed in the module docstring, as (rows, labels)."""
    pc, vs, osf = cfg["point_cloud_range"], cfg["voxel_size"], cfg["out_size_factor"]
    fx, fy = cfg["grid_size"][0] // osf, cfg["grid_size"][1] // osf
    cell_x, cell_y = vs[0] * osf, vs[1] * osf
    mid_x, mid_y = pc[0] + cell_x * (fx // 2 + 0.3), pc[1] + cell_y * (fy // 2 + 0.6)
    rows, labs = [], []

    def add(x, y, dx=1.95, dy=4.6, lab=0, yaw=0.4):
        rows.append([x, y, -1.0, dx, dy, 1.6, yaw, 1.5, -0.5])
        labs.append(lab)

    if centerhead:
        add(mid_x, mid_y, lab=10)                       # labels of no task
        add(mid_x, mid_y, lab=11)
        add(mid_x, mid_y, lab=-1)
    add(mid_x, mid_y, dx=0.0)                           # zero and negative sizes, NaN size
    add(mid_x, mid_y, dy=-1.0)
    add(mid_x, mid_y, dx=float("nan"))
    add(pc[0] - 0.5 * cell_x, mid_y, lab=1)             # centre in (-1, 0) cells on either axis
    add(mid_x, pc[1] - 0.25 * cell_y, lab=1)
    add(pc[0], pc[1], lab=2)                            # exactly on the low corner
    add(pc[0] + fx * cell_x, mid_y, lab=2)              # exactly on the far borders
    add(mid_x, pc[1] + fy * cell_y, lab=2)
    r, _ = radius_of(gaussian_radius, cfg, 1.95, 4.6)
    for k in (r - 1, r, r + 1):                         # r - 1, r, r + 1 cells outside each side
        add(pc[0] - (k + 0.5) * cell_x, mid_y, lab=3)
        add(pc[0] + (fx + k - 0.5) * cell_x, mid_y, lab=3)
        add(mid_x, pc[1] - (k + 0.5) * cell_y, lab=4)
        add(mid_x, pc[1] + (fy + k - 0.5) * cell_y, lab=4)
    for j in range(5):                                  # clusters of overlapping same-class gaussians
        add(mid_x + 0.37 * j * cell_x, mid_y - 0.29 * j * cell_y, lab=0, yaw=0.2 * j)
    for j in range(3):                                  # (pedestrians: drawn even where the cars pass max_objs)
        add(mid_x - (4.2 + 0.6 * j) * cell_x, mid_y + (3.1 + 0.45 * j) * cell_y, dx=0.7, dy=0.7, lab=8)
    for dx, dy in near_integer_sizes(cfg, rng):        # radii just below / above an integer
        add(rng.uniform(pc[0], pc[3]), rng.uniform(pc[1], pc[4]), dx=dx, dy=dy, lab=int(rng.integers(0, 10)))
    return rows, labs


def build_case(name, mode, cfg, norm_bbox, D, samples, centerhead, tfheat):
    B = len(samples)
    nmax = max([len(r) for r, _ in samples] + [1])
    boxes = np.zeros((B, nmax, D), np.float32)
    labels = np.zeros((B, nmax), np.int32)
    counts = np.array([len(r) for r, _ in samples], np.int32)
    out = {}
    for b, (rows, labs) in enumerate(samples):
        if rows:
            boxes[b, :len(rows)] = np.array(rows, np.float32)[:, :D]
            labels[b, :len(rows)] = labs
    if mode == "centerhead":
        M = cfg["max_objs"] * cfg["dense_reg"]
        self = types.SimpleNamespace(train_cfg=cfg, class_names=TASKS, task_heads=[None] * len(TASKS),
                                     norm_bbox=norm_bbox)
        res = [[], [], [], []]
        for b in range(B):
            t9 = np.zeros((counts[b], 9), np.float32)
            t9[:, :D] = boxes[b, :counts[b]]
            hm, ab, ind, m = centerhead(self, Boxes(torch.from_numpy(t9)), torch.from_numpy(labels[b, :counts[b]]).long())
            for k, v in enumerate((hm, ab, ind, m)):
                res[k].append(v)
        A = 10 if D == 9 else 8
        for t in range(len(TASKS)):
            out["%s_hm%d" % (name, t)] = torch.stack([res[0][b][t] for b in range(B)]).numpy()
        out[name + "_anno"] = np.stack([np.stack([res[1][b][t].numpy()[:, :A] for b in range(B)])
                                        for t in range(len(TASKS))])
        out[name + "_ind"] = np.stack([np.stack([res[2][b][t].numpy() for b in range(B)]) for t in range(len(TASKS))])
        out[name + "_mask"] = np.stack([np.stack([res[3][b][t].numpy() for b in range(B)]) for t in range(len(TASKS))])
        assert out[name + "_anno"].shape[2] == M
    else:
        self = types.SimpleNamespace(train_cfg=cfg, num_classes=10)
        hms = []
        for b in range(B):
            t9 = np.zeros((counts[b], 9), np.float32)
            t9[:, :D] = boxes[b, :counts[b]]
            hms.append(tfheat(self, Boxes(torch.from_numpy(t9)), torch.from_numpy(labels[b, :counts[b]]).long(), "cpu"))
        out[name + "_hm"] = torch.stack(hms).numpy()
    out.update({name + "_boxes": boxes, name + "_labels": labels, name + "_counts": counts,
                name + "_cfg": np.array(json.dumps(dict(cfg=cfg, mode=mode, norm_bbox=norm_bbox)))})
    return out


def main():
    centerhead, tfheat, gaussian_radius = reference_functions()
    rng = np.random.default_rng(20261016)
    data = {}
    cases = []
    # ch_six: named + 70 random boxes; an empty second sample
    rows, labs = named_boxes(CFG_SIX, gaussian_radius, rng, True)
    r2, l2 = random_boxes(rng, 70, CFG_SIX, 10)
    data.update(build_case("ch_six", "centerhead", CFG_SIX, True, 9, [(rows + r2, labs + l2), ([], [])],
                           centerhead, tfheat))
    cases.append("ch_six")
    # ch_small: more cars than max_objs, norm_bbox off, 7 columns
    rows, labs = named_boxes(CFG_SMALL, gaussian_radius, rng, True)
    r2, l2 = random_boxes(rng, 40, CFG_SMALL, 12)
    cars, cl = random_boxes(rng, 9, CFG_SMALL, 1)
    r3, l3 = random_boxes(rng, 25, CFG_SMALL, 10)
    data.update(build_case("ch_small", "centerhead", CFG_SMALL, False, 7,
                           [(cars + rows + r2, cl + labs + l2), (r3, l3)], centerhead, tfheat))
    cases.append("ch_small")
    # TransFusion
    rows, labs = named_boxes(CFG_TF, gaussian_radius, rng, False)
    r2, l2 = random_boxes(rng, 80, CFG_TF, 10)
    r3, l3 = random_boxes(rng, 3, CFG_TF, 10)
    data.update(build_case("tf_ten", "transfusion", CFG_TF, True, 9, [(rows + r2, labs + l2), (r3, l3)],
                           centerhead, tfheat))
    cases.append("tf_ten")
    rows, labs = named_boxes(CFG_TF_WIDE, gaussian_radius, rng, False)
    r2, l2 = random_boxes(rng, 30, CFG_TF_WIDE, 10)
    data.update(build_case("tf_wide", "transfusion", CFG_TF_WIDE, True, 7, [(rows + r2, labs + l2), ([], [])],
                           centerhead, tfheat))
    cases.append("tf_wide")
    data["cases"] = np.array(cases)
    path = os.path.join(HERE, "head_targets_tiny.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, sorted(data))


if __name__ == "__main__":
    main()
