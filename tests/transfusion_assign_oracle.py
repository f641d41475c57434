"""A numpy restatement of TransFusionHead.get_targets without the heatmap (transfusion.py:357-525, 575), with the
HungarianAssigner3D cost (hungarian_assigner.py:82-142, mmdet's FocalLossCost) in fp32 op for op and scipy as the
solver.  The rotated BEV overlap is nms_oracle's float64 polygon clipping rounded to fp32.

    decode(center, height, dim, rot, coder)          TransFusionBBoxCoder.decode of one sample -> [N, 7] fp32
    cost_matrix(boxes, logits, gt, gt_labels, train_cfg, costs) -> (cost [P, G], iou [P, G]) fp32
    targets(gt, gt_labels, counts, preds, num_classes, num_proposals, train_cfg, coder, costs)
        -> dict(labels, label_weights, bbox_targets, bbox_weights, ious [B, N ...], num_pos [B], mean_iou [B],
                gt_inds [B, N] (matched gt + 1, 0 unmatched))

Scalar divisions follow torch on CUDA tensors: a Python-number divisor multiplies by the fp32 reciprocal of its
fp32 value.  A sample without gts is all negative (the reference raises there)."""
import os
import sys

import numpy as np
from scipy.optimize import linear_sum_assignment

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import nms_oracle  # noqa: E402

f32 = np.float32
COSTS = dict(cls_weight=0.15, alpha=0.25, gamma=2.0, reg_weight=0.25, iou_weight=0.25)   # transfusion/default.yaml


def decode(center, height, dim, rot, coder):
    """center [2, N], height [1, N], dim [3, N], rot [2, N] fp32 -> [N, 7] (x, y, z_bottom, dx, dy, dz, yaw)."""
    osf, vs, pc = f32(coder["out_size_factor"]), coder["voxel_size"], coder["pc_range"]
    x = center[0] * osf * f32(vs[0]) + f32(pc[0])
    y = center[1] * osf * f32(vs[1]) + f32(pc[1])
    d = np.exp(dim.astype(f32))
    z = height[0] - d[2] * f32(0.5)
    yaw = np.arctan2(rot[0], rot[1]).astype(f32)
    return np.stack([x, y, z, d[0], d[1], d[2], yaw], 1).astype(f32)


def xyxyr(b):
    hw, hh = b[:, 3] * f32(0.5), b[:, 4] * f32(0.5)
    return np.stack([b[:, 0] - hw, b[:, 1] - hh, b[:, 0] + hw, b[:, 1] + hh, b[:, 6]], 1).astype(f32)


def iou3d(a, b):
    """BaseInstance3DBoxes.overlaps(a, b) in fp32 (z is the bottom); the BEV overlap in float64 rounded."""
    bev = nms_oracle.iou_matrix(xyxyr(a), xyxyr(b), overlap=True).astype(f32)
    with np.errstate(invalid="ignore", over="ignore"):
        top = np.minimum((a[:, 2] + a[:, 5])[:, None], (b[:, 2] + b[:, 5])[None])
        bottom = np.maximum(a[:, 2][:, None], b[:, 2][None])
        h = top - bottom
        h = np.where(h < 0, f32(0), h)
        ov = bev * h
        va, vb = a[:, 3] * a[:, 4] * a[:, 5], b[:, 3] * b[:, 4] * b[:, 5]
        u = (va[:, None] + vb[None]) - ov
        u = np.where(u < f32(1e-8), f32(1e-8), u)
        return (ov / u).astype(f32)


def cost_matrix(boxes, logits, gt, gt_labels, train_cfg, costs=COSTS):
    """boxes [P, 7] decoded, logits [K, P], gt [G, 7 | 9], gt_labels [G] -> (cost, iou) [P, G] fp32, summed as
    cls + reg + iou."""
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        p = (f32(1) / (f32(1) + np.exp(-logits.T.astype(f32)))).astype(f32)
        q = f32(1) - p
        a = f32(costs["alpha"])
        neg = -np.log(q + f32(1e-12)) * f32(1 - costs["alpha"]) * (p * p)
        pos = -np.log(p + f32(1e-12)) * a * (q * q)
        cls = (pos[:, gt_labels] - neg[:, gt_labels]) * f32(costs["cls_weight"])
        rng = train_cfg["point_cloud_range"]
        start = np.array(rng[0:2], f32)
        span = np.array(rng[3:5], f32) - start
        nb = (boxes[:, :2] - start) / span
        ng = (gt[:, :2] - start) / span
        reg = (np.abs(nb[:, None, 0] - ng[None, :, 0]) + np.abs(nb[:, None, 1] - ng[None, :, 1])) * \
            f32(costs["reg_weight"])
        iou = iou3d(boxes, gt[:, :7])
        return ((cls + reg) + (-iou) * f32(costs["iou_weight"])).astype(f32), iou


def encode(gt, coder, code_size):
    osf, vs, pc = coder["out_size_factor"], coder["voxel_size"], coder["pc_range"]
    t = np.zeros((len(gt), code_size), f32)
    t[:, 0] = (gt[:, 0] - f32(pc[0])) * (f32(1) / f32(osf * vs[0]))
    t[:, 1] = (gt[:, 1] - f32(pc[1])) * (f32(1) / f32(osf * vs[1]))
    t[:, 2] = gt[:, 2] + gt[:, 5] * f32(0.5)
    t[:, 3:6] = np.log(gt[:, 3:6])
    t[:, 6] = np.sin(gt[:, 6])
    t[:, 7] = np.cos(gt[:, 6])
    if code_size == 10:
        t[:, 8:10] = gt[:, 7:9]
    return t


def targets(gt, gt_labels, counts, preds, num_classes, num_proposals, train_cfg, coder, costs=COSTS):
    """gt [B, Nmax, 7 | 9], gt_labels [B, Nmax], counts [B]; preds: dict of numpy [B, *, N] (heatmap, center,
    height, dim, rot)."""
    B, N = preds["heatmap"].shape[0], preds["heatmap"].shape[2]
    P, K = num_proposals, num_classes
    L = N // P
    code = int(coder.get("code_size", 8))
    pw = float(train_cfg.get("pos_weight", -1))
    out = dict(labels=np.full((B, N), K, np.int64), label_weights=np.ones((B, N), np.int64),
               bbox_targets=np.zeros((B, N, code), f32), bbox_weights=np.zeros((B, N, code), f32),
               ious=np.zeros((B, N), f32), num_pos=np.zeros(B, np.int64), mean_iou=np.zeros(B, f32),
               gt_inds=np.zeros((B, N), np.int64))
    for b in range(B):
        G = int(counts[b])
        g_b, l_b = gt[b, :G].astype(f32), gt_labels[b, :G].astype(np.int64)
        boxes = decode(preds["center"][b], preds["height"][b], preds["dim"][b], preds["rot"][b], coder)
        for layer in range(L):
            if G == 0:
                continue
            sl = slice(layer * P, (layer + 1) * P)
            cost, iou = cost_matrix(boxes[sl], preds["heatmap"][b][:, sl], g_b, l_b, train_cfg, costs)
            rows, cols = linear_sum_assignment(cost)
            n = rows + layer * P
            out["gt_inds"][b, n] = cols + 1
            out["labels"][b, n] = l_b[cols]
            if pw > 0:
                out["label_weights"][b, n] = int(pw)
            out["bbox_targets"][b, n] = encode(g_b[cols], coder, code)
            out["bbox_weights"][b, n] = 1
            out["ious"][b, n] = np.clip(iou[rows, cols], 0, 1)
        pos = out["gt_inds"][b] > 0
        out["num_pos"][b] = pos.sum()
        out["mean_iou"][b] = f32(out["ious"][b][pos].astype(np.float64).sum()) * (f32(1) / f32(max(pos.sum(), 1)))
    return out
