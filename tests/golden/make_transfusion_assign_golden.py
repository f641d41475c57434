"""Writes transfusion_assign_tiny.npz: TransFusionHead.get_targets (without the heatmap) on seeded synthetic inputs,
restated with torch CPU tensors in the reference's op order (transfusion_bbox_coder.py decode / encode,
hungarian_assigner.py:82-142 with mmdet's FocalLossCost, BaseInstance3DBoxes.overlaps, transfusion.py:485-525)
and scipy.optimize.linear_sum_assignment as the solver.  The rotated BEV overlap is nms_oracle's float64 polygon
clipping rounded to fp32.  Divisions by a Python number are written as torch computes them on CUDA tensors: a
multiply by the fp32 reciprocal of the divisor's fp32 value.

Cases: three samples with two decoder layers of 24 proposals: 10 gts (the solver transposes), 31 gts (more gts
than proposals) and none (all negative; the reference raises there)."""
import os
import sys

import numpy as np
import torch
from scipy.optimize import linear_sum_assignment

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, ".."))
import nms_oracle  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402

P, K, L = 24, 10, 2


def decode(c, h, d, r, coder):
    c, h, d = c.clone(), h.clone(), d.clone()
    c[0] = c[0] * coder["out_size_factor"] * coder["voxel_size"][0] + coder["pc_range"][0]
    c[1] = c[1] * coder["out_size_factor"] * coder["voxel_size"][1] + coder["pc_range"][1]
    d = d.exp()
    h = h - d[2:3] * 0.5
    yaw = torch.atan2(r[0:1], r[1:2])
    return torch.cat([c, h, d, yaw], 0).T


def overlaps(a, b):
    xa = torch.stack([a[:, 0] - a[:, 3] / 2, a[:, 1] - a[:, 4] / 2, a[:, 0] + a[:, 3] / 2, a[:, 1] + a[:, 4] / 2,
                      a[:, 6]], 1)
    xb = torch.stack([b[:, 0] - b[:, 3] / 2, b[:, 1] - b[:, 4] / 2, b[:, 0] + b[:, 3] / 2, b[:, 1] + b[:, 4] / 2,
                      b[:, 6]], 1)
    bev = torch.from_numpy(nms_oracle.iou_matrix(xa.numpy(), xb.numpy(), overlap=True).astype(np.float32))
    top = torch.min((a[:, 2] + a[:, 5]).view(-1, 1), (b[:, 2] + b[:, 5]).view(1, -1))
    bottom = torch.max(a[:, 2].view(-1, 1), b[:, 2].view(1, -1))
    ov = bev * torch.clamp(top - bottom, min=0)
    va, vb = (a[:, 3] * a[:, 4] * a[:, 5]).view(-1, 1), (b[:, 3] * b[:, 4] * b[:, 5]).view(1, -1)
    return ov / torch.clamp(va + vb - ov, min=1e-8)


def focal_cost(logits, gt_labels, alpha=0.25, gamma=2.0, weight=0.15, eps=1e-12):
    p = logits.sigmoid()
    neg = -(1 - p + eps).log() * (1 - alpha) * p.pow(gamma)
    pos = -(p + eps).log() * alpha * (1 - p).pow(gamma)
    return (pos[:, gt_labels] - neg[:, gt_labels]) * weight


def l1_cost(boxes, gt, cfg, weight=0.25):
    start = boxes.new(cfg["point_cloud_range"][0:2])
    span = boxes.new(cfg["point_cloud_range"][3:5]) - boxes.new(cfg["point_cloud_range"][0:2])
    return torch.cdist((boxes[:, :2] - start) / span, (gt[:, :2] - start) / span, p=1) * weight


def encode(gt, coder):
    t = torch.zeros((gt.shape[0], coder["code_size"]))
    for k in range(2):
        inv = np.float32(1) / np.float32(coder["out_size_factor"] * coder["voxel_size"][k])
        t[:, k] = (gt[:, k] - coder["pc_range"][k]) * float(inv)
    t[:, 3:6] = gt[:, 3:6].log()
    t[:, 2] = gt[:, 2] + gt[:, 5] * 0.5
    t[:, 6] = torch.sin(gt[:, 6])
    t[:, 7] = torch.cos(gt[:, 6])
    if coder["code_size"] == 10:
        t[:, 8:10] = gt[:, 7:]
    return t


def main():
    cfg, coder = S.TRANSFUSION_TRAIN_CFG, S.TRANSFUSION_CODER
    b0, l0 = S.gt_boxes(seed=11, batch=2, min_boxes=10, max_boxes=10)
    b1, l1 = S.gt_boxes(seed=12, batch=1, min_boxes=31, max_boxes=31)
    boxes, labels = [b0[0], b1[0], b0[1][:0]], [l0[0], l1[0], l0[1][:0]]
    preds = S.transfusion_predictions(7, 3, (boxes, labels), num_proposals=P, num_classes=K, layers=L)
    nmax = max(len(b) for b in boxes)
    N = L * P
    out = dict(labels=np.full((3, N), K, np.int64), label_weights=np.ones((3, N), np.int64),
               bbox_targets=np.zeros((3, N, 10), np.float32), bbox_weights=np.zeros((3, N, 10), np.float32),
               ious=np.zeros((3, N), np.float32), num_pos=np.zeros(3, np.int64), mean_iou=np.zeros(3, np.float32),
               gt_inds=np.zeros((3, N), np.int64))
    for b in range(3):
        gt, gl = boxes[b], labels[b]
        dec = decode(preds["center"][b], preds["height"][b], preds["dim"][b], preds["rot"][b], coder)
        if len(gt):
            for layer in range(L):
                sl = slice(layer * P, (layer + 1) * P)
                cost = focal_cost(preds["heatmap"][b][:, sl].T, gl) + l1_cost(dec[sl], gt, cfg) + \
                    (-overlaps(dec[sl], gt)) * 0.25
                iou = overlaps(dec[sl], gt)
                rows, cols = linear_sum_assignment(cost.numpy())
                n = rows + layer * P
                out["gt_inds"][b, n] = cols + 1
                out["labels"][b, n] = gl[cols].numpy()
                out["bbox_targets"][b, n] = encode(gt[cols], coder).numpy()
                out["bbox_weights"][b, n] = 1
                out["ious"][b, n] = torch.clamp(iou[rows, cols], 0, 1).numpy()
        pos = out["gt_inds"][b] > 0
        out["num_pos"][b] = pos.sum()
        s = torch.from_numpy(out["ious"][b][pos]).sum()
        out["mean_iou"][b] = float(s * float(np.float32(1) / np.float32(max(pos.sum(), 1))))
    pad_b = np.zeros((3, nmax, 9), np.float32)
    pad_l = np.zeros((3, nmax), np.int32)
    for b in range(3):
        pad_b[b, :len(boxes[b])] = boxes[b].numpy()
        pad_l[b, :len(boxes[b])] = labels[b].numpy()
    np.savez_compressed(os.path.join(HERE, "transfusion_assign_tiny.npz"), gt_boxes=pad_b, gt_labels=pad_l,
                        counts=np.array([len(b) for b in boxes], np.int32), num_proposals=P, num_classes=K,
                        **{"pred_" + k: v.numpy() for k, v in preds.items()}, **out)


if __name__ == "__main__":
    main()
