"""Restatement of the CenterHead / TransFusionHead heatmap targets (centerpoint.py:432-582, transfusion.py:526-573,
core/utils/gaussian.py) in numpy, one object at a time: fp32 scalars in the reference's op order for the sizes,
radius and centre (each Python constant rounded to fp32 where it meets a tensor), float64 for the gaussian as
gaussian_2d builds it.  log / sin / cos of anno_box go through torch's CPU fp32 ops on tensors shaped as the
reference's, so they round as the reference's do.

targets(boxes, labels, counts, mode, task_classes, cfg, max_objs=0, norm_bbox=True) takes the padded batch and
returns dict(heatmaps=[per task [B, ncls_t, fy, fx]], anno, ind, mask ([T, B, M, A] / [T, B, M]), records
[B, Nmax, 4] (plane, row, col, radius; radius -1 where nothing is drawn), status)."""
import math

import numpy as np
import torch

F = np.float32
MAX_RADIUS = 2 ** 30


def fp32(v):
    return F(v)


def gaussian_radius(height, width, overlap):
    """gaussian.py:55-84 with fp32 0-d tensors height, width and a Python float overlap."""
    height, width = F(height), F(width)
    one_minus, one_plus = F(1 - overlap), F(1 + overlap)
    with np.errstate(all="ignore"):
        b1 = height + width
        c1 = width * height * one_minus / one_plus
        r1 = (b1 + np.sqrt(b1 * b1 - F(4) * c1)) / F(2)
        b2 = F(2) * (height + width)
        c2 = one_minus * width * height
        r2 = (b2 + np.sqrt(b2 * b2 - F(16) * c2)) / F(2)
        a3x4 = F(4 * (4 * overlap))
        b3 = F(-2 * overlap) * (height + width)
        c3 = F(overlap - 1) * width * height
        r3 = (b3 + np.sqrt(b3 * b3 - a3x4 * c3)) / F(2)
    r = r1
    if r2 < r:
        r = r2
    if r3 < r:
        r = r3
    return r


def gaussian_2d(radius):
    """gaussian.py:5-21 for a (2r+1)^2 window, float64."""
    d = 2 * radius + 1
    sigma = d / 6
    y, x = np.ogrid[-radius:radius + 1, -radius:radius + 1]
    h = np.exp(-(x * x + y * y) / (2 * sigma * sigma))
    h[h < np.finfo(h.dtype).eps * h.max()] = 0
    return h


def draw(plane, row, col, radius):
    """Max the fp32 gaussian into plane [H, W] over rows row +- radius, cols col +- radius, clipped to the plane
    (what draw_heatmap_gaussian's slicing draws at center (col, row))."""
    H, W = plane.shape
    r0, r1 = max(row - radius, 0), min(row + radius, H - 1)
    c0, c1 = max(col - radius, 0), min(col + radius, W - 1)
    if r0 > r1 or c0 > c1:
        return
    g = gaussian_2d(radius).astype(np.float32)
    sub = g[r0 - row + radius:r1 - row + radius + 1, c0 - col + radius:c1 - col + radius + 1]
    np.maximum(plane[r0:r1 + 1, c0:c1 + 1], sub, out=plane[r0:r1 + 1, c0:c1 + 1])


def trunc_i32(v):
    """float32 -> int32 toward zero, saturating (only finite values reach here)."""
    return int(max(min(math.trunc(float(v)), 2 ** 31 - 1), -2 ** 31))


def targets(boxes, labels, counts, mode, task_classes, cfg, max_objs=0, norm_bbox=True, label_table=None):
    boxes = np.asarray(boxes, np.float32)
    labels = np.asarray(labels)
    B, nmax, D = boxes.shape
    T = len(task_classes)
    osf = int(cfg["out_size_factor"])
    fx, fy = int(cfg["grid_size"][0]) // osf, int(cfg["grid_size"][1]) // osf
    pcx, pcy = F(cfg["point_cloud_range"][0]), F(cfg["point_cloud_range"][1])
    vsx, vsy = F(cfg["voxel_size"][0]), F(cfg["voxel_size"][1])
    ov, min_radius = float(cfg["gaussian_overlap"]), int(cfg["min_radius"])
    if label_table is None:
        label_table = [(t, c) for t, n in enumerate(task_classes) for c in range(n)]
    center = mode == "centerhead"
    A = 10 if D == 9 else 8
    heatmaps = [np.zeros((B, n, fy, fx), np.float32) for n in task_classes]
    anno = np.zeros((T, B, max_objs, A), np.float32)
    ind = np.zeros((T, B, max_objs), np.int64)
    mask = np.zeros((T, B, max_objs), np.uint8)
    records = np.full((B, nmax, 4), 0, np.int32)
    records[..., 3] = -1
    plane0 = np.concatenate([[0], np.cumsum([B * n for n in task_classes])])[:-1]
    status = 0
    for b in range(B):
        n = max(0, min(int(counts[b]), nmax))
        keys = [label_table[int(l)] if 0 <= int(l) < len(label_table) else (-1, 0) for l in labels[b, :n]]
        # CenterHead slots: by class in task order, then by original index (centerpoint.py:463-486)
        slots = {}
        if center:
            for t in range(T):
                order = [i for c in range(task_classes[t]) for i in range(n) if keys[i] == (t, c)]
                for s, i in enumerate(order):
                    slots[i] = s
        for i in range(n):
            t, c = keys[i]
            if center and (t < 0 or slots[i] >= max_objs):
                continue
            x, y, z, dx, dy, dz, yaw = boxes[b, i, :7]
            width = dx / vsx / F(osf)
            length = dy / vsy / F(osf)
            if not (width > 0 and length > 0):
                continue
            r = gaussian_radius(length, width, ov)
            if not (np.isfinite(r) and r < MAX_RADIUS) or t < 0:
                status += 1
                continue
            radius = max(min_radius, int(r))
            with np.errstate(all="ignore"):
                coor_x = (x - pcx) / vsx / F(osf)
                coor_y = (y - pcy) / vsy / F(osf)
            if not (np.isfinite(coor_x) and np.isfinite(coor_y)):
                continue
            cx, cy = trunc_i32(coor_x), trunc_i32(coor_y)
            if center and not (0 <= cx < fx and 0 <= cy < fy):
                continue
            records[b, i] = (plane0[t] + b * task_classes[t] + c, cx, cy, radius)
            draw(heatmaps[t][b, c], cx, cy, radius)
            if center:
                s = slots[i]
                ind[t, b, s] = cx * fy + cy
                mask[t, b, s] = 1
                dims = torch.from_numpy(boxes[b, i, 3:6].copy())
                if norm_bbox:
                    dims = dims.log()
                rot = torch.tensor(boxes[b, i, 6])
                row = [coor_x - F(cx), coor_y - F(cy), z + dz * F(0.5)] + dims.numpy().tolist() + \
                      [float(torch.sin(rot)), float(torch.cos(rot))]
                if A == 10:
                    row += [boxes[b, i, 7], boxes[b, i, 8]]
                anno[t, b, s] = np.array(row, np.float32)
    return dict(heatmaps=heatmaps, anno=anno, ind=ind, mask=mask, records=records, status=status)
