"""transfusion_assign -- the training-target assignment of TransFusionHead on the device
(csrc/transfusion_assign.cu): batched exact Hungarian matching and the whole get_targets, with no host round trip.

    linear_sum_assignment_batched(cost, row_counts=None, col_counts=None)
        -> (col4row [S, R], row4col [S, C]) int32: scipy.optimize.linear_sum_assignment of S fp32 matrices at once,
           bit for bit (ties included)
    transfusion_assign_batched(preds, boxes, labels, counts, num_classes, num_proposals, train_cfg, bbox_coder_cfg)
        -> (labels, label_weights, bbox_targets, bbox_weights, ious, num_pos, mean_iou, status), device tensors, no
           host synchronisation, CUDA-graph capturable
    transfusion_targets(gt_bboxes_3d, gt_labels_3d, preds_dict, num_classes, num_proposals, train_cfg,
                        bbox_coder_cfg)
        -> TransFusionHead.get_targets' 8-tuple (transfusion.py:357-406), heatmap from head_targets, after exactly
           one host synchronisation (num_pos an int, matched_ious a float)
    HungarianAssigner3D(...).assign(bboxes, gt_bboxes, gt_labels, cls_pred, train_cfg)
        -> AssignResult(num_gts, gt_inds, max_overlaps, labels), for callers that keep the reference's loop

Three launches per call (cost, solver, targets).  The cost is the reference's (FocalLossCost + BBoxBEVL1Cost +
IoU3DCost, hungarian_assigner.py:82-142) in fp32 with one rounding per op in its order; the solver is scipy's
rectangular_lsap.cpp restated in double, so the assignment is scipy's on that matrix.  The BEV overlap is
iou3d.boxes_overlap_bev's.

Scalar division follows what torch does on CUDA tensors: dividing by a Python number multiplies by the fp32
reciprocal of the number rounded to fp32 (BinaryDivTrueKernel.cu), so encode's x target is
(x - pc0) * fp32(1 / fp32(osf * vs0)) and mean_iou is sum * fp32(1 / num_pos); BBoxBEVL1Cost divides by a
tensor, which is a true division.

Deliberate deviations, where the reference raises:
- a sample with no gt gets all-negative targets (the reference fails at torch.cat([None]));
- a segment (sample, decoder layer) whose cost has a NaN or -inf entry, or a +inf pattern with no complete
  assignment, or a sample with a gt label outside [0, num_classes) (its cost column is NaN), gets no matches and
  sets bits of its sample's status word (STATUS); transfusion_targets raises ValueError after its synchronisation.
A proposal with a NaN yaw overlaps nothing in BEV (as in iou3d.boxes_overlap_bev).  GPU only: CPU tensors raise."""
import ctypes
from collections import namedtuple

import numpy as np
import torch

from . import _C
from .head_targets import _box_tensor, pad_gt, transfusion_heatmap_targets_batched

__all__ = ["linear_sum_assignment_batched", "transfusion_assign_batched", "transfusion_targets",
           "HungarianAssigner3D", "AssignResult", "STATUS", "MAX_SIZE"]

MAX_SIZE = 4096        # BEVB200_ASSIGN_MAX rows / columns per segment
MAX_SEGMENTS = 65535   # BEVB200_ASSIGN_MAX_SEGMENTS
MAX_CLASSES = 256      # BEVB200_ASSIGN_MAX_CLASSES
STATUS = {"invalid_cost": 1, "bad_label": 2, "infeasible": 4}   # BEVB200_ASSIGN_* bits

AssignResult = namedtuple("AssignResult", ["num_gts", "gt_inds", "max_overlaps", "labels"])


def linear_sum_assignment_batched(cost, row_counts=None, col_counts=None, return_status=False,
                                  return_steps=False):
    """scipy.optimize.linear_sum_assignment of S matrices in one launch.  cost [S, R, C] fp32 CUDA; segment s is
    its top-left row_counts[s] x col_counts[s] block (int32 CUDA [S], nullable: R / C).  Returns col4row [S, R]
    (the column of each row, -1 for none) and row4col [S, C] int32; scipy's (row_ind, col_ind) of segment s are
    the rows with col4row >= 0 and their columns.  With return_status also the int32 [S] status bits (nonzero:
    no matches, where scipy raises), with return_steps the solver's steps per segment."""
    _C.require_cuda(cost, "cost", torch.float32)
    if cost.dim() != 3:
        raise ValueError("cost must be [S, R, C], got %s" % (tuple(cost.shape),))
    S, R, C = cost.shape
    if R > MAX_SIZE or C > MAX_SIZE or S > MAX_SEGMENTS:
        raise ValueError("at most %d rows and columns and %d segments (got %s)" % (MAX_SIZE, MAX_SEGMENTS,
                                                                                 (S, R, C)))
    for name, c in (("row_counts", row_counts), ("col_counts", col_counts)):
        if c is not None:
            _C.require_cuda(c, name, torch.int32)
            if tuple(c.shape) != (S,) or c.device != cost.device:
                raise ValueError("%s must be [S] on the cost's device" % name)
    dev = cost.device
    col4row = torch.empty((S, R), dtype=torch.int32, device=dev)
    row4col = torch.empty((S, C), dtype=torch.int32, device=dev)
    status = torch.empty((S,), dtype=torch.int32, device=dev)
    steps = torch.empty((S,), dtype=torch.int32, device=dev) if return_steps else None
    _C.check(_C.lib().bevb200_lsap(_C.ptr(cost), _C.ptr(row_counts), _C.ptr(col_counts), S, R, C, _C.ptr(col4row),
                                   _C.ptr(row4col), _C.ptr(status), _C.ptr(steps), None, 0,
                                   _C.current_stream(dev)), "lsap")
    out = (col4row, row4col)
    if return_status:
        out += (status,)
    if return_steps:
        out += (steps,)
    return out


def _cost_params(train_cfg):
    """(cls_weight, alpha, gamma, reg_weight, iou_weight) from train_cfg['assigner'] (HungarianAssigner3D)."""
    a = train_cfg.get("assigner", {})
    if a.get("type", "HungarianAssigner3D") != "HungarianAssigner3D":
        raise ValueError("only HungarianAssigner3D is supported (got %s)" % a.get("type"))
    return _costs(a.get("cls_cost", dict(type="FocalLossCost")), a.get("reg_cost", dict(type="BBoxBEVL1Cost")),
                  a.get("iou_cost", dict(type="IoU3DCost")), a.get("iou_calculator"))


def _costs(cls_cost, reg_cost, iou_cost, iou_calculator=None):
    if cls_cost.get("type") != "FocalLossCost":
        raise ValueError("cls_cost must be FocalLossCost (got %s)" % cls_cost.get("type"))
    if reg_cost.get("type") != "BBoxBEVL1Cost" or iou_cost.get("type") != "IoU3DCost":
        raise ValueError("reg_cost must be BBoxBEVL1Cost and iou_cost IoU3DCost")
    if iou_calculator is not None and (iou_calculator.get("type", "BboxOverlaps3D") != "BboxOverlaps3D"
                                       or iou_calculator.get("coordinate", "lidar") != "lidar"):
        raise ValueError("iou_calculator must be BboxOverlaps3D in lidar coordinates")
    if float(cls_cost.get("eps", 1e-12)) != 1e-12:
        raise ValueError("FocalLossCost eps must be 1e-12")
    return (float(cls_cost.get("weight", 1.0)), float(cls_cost.get("alpha", 0.25)), float(cls_cost.get("gamma", 2)),
            float(reg_cost.get("weight", 1.0)), float(iou_cost.get("weight", 1.0)))


def _run(heatmap, center, height, dim, rot, decoded, boxes, labels, counts, num_classes, num_proposals,
         train_cfg, bbox_coder_cfg, extras=False, costs=None):
    _C.require_cuda(boxes, "boxes", torch.float32)
    _C.require_cuda(labels, "labels", torch.int32)
    _C.require_cuda(counts, "counts", torch.int32)
    if boxes.dim() != 3 or boxes.shape[2] not in (7, 9):
        raise ValueError("boxes must be [B, Nmax, 7 | 9], got %s" % (tuple(boxes.shape),))
    B, nmax, D = boxes.shape
    if tuple(labels.shape) != (B, nmax) or tuple(counts.shape) != (B,):
        raise ValueError("labels must be [B, Nmax] and counts [B] for boxes %s" % (tuple(boxes.shape),))
    K, P = int(num_classes), int(num_proposals)
    if not 1 <= K <= MAX_CLASSES:
        raise ValueError("num_classes must be in 1..%d" % MAX_CLASSES)
    _C.require_cuda(heatmap, "heatmap", torch.float32)
    if heatmap.dim() != 3 or heatmap.shape[0] != B or heatmap.shape[1] != K:
        raise ValueError("heatmap must be [B, num_classes, N], got %s" % (tuple(heatmap.shape),))
    N = heatmap.shape[2]
    if P < 1 or N % P:
        raise ValueError("the %d proposal columns are not whole layers of num_proposals %d" % (N, P))
    L = N // P
    if P > MAX_SIZE or nmax > MAX_SIZE or B * L > MAX_SEGMENTS:
        raise ValueError("at most %d proposals and gts per segment and %d segments" % (MAX_SIZE, MAX_SEGMENTS))
    if decoded is None:
        for name, t, rows in (("center", center, 2), ("height", height, 1), ("dim", dim, 3), ("rot", rot, 2)):
            _C.require_cuda(t, name, torch.float32)
            if tuple(t.shape) != (B, rows, N):
                raise ValueError("%s must be [B, %d, N] = %s, got %s" % (name, rows, (B, rows, N), tuple(t.shape)))
    else:
        _C.require_cuda(decoded, "decoded", torch.float32)
        if tuple(decoded.shape) != (B, N, D):
            raise ValueError("decoded boxes must be [B, N, %d]" % D)
    code_size = int(bbox_coder_cfg.get("code_size", 8))
    if code_size not in (8, 10) or (code_size == 10 and D != 9):
        raise ValueError("code_size must be 8, or 10 with 9-column boxes")
    dev = boxes.device
    for t in (heatmap, center, height, dim, rot, decoded, labels, counts):
        if t is not None and t.device != dev:
            raise ValueError("predictions and ground truth must be on one device")
    pc, vs, osf = bbox_coder_cfg["pc_range"], bbox_coder_cfg["voxel_size"], int(bbox_coder_cfg["out_size_factor"])
    rng = train_cfg["point_cloud_range"]
    cls_w, alpha, gamma, reg_w, iou_w = costs if costs is not None else _cost_params(train_cfg)
    pos_weight = float(train_cfg.get("pos_weight", -1))
    out_labels = torch.empty((B, N), dtype=torch.int64, device=dev)
    label_weights = torch.empty((B, N), dtype=torch.int64, device=dev)
    bbox_targets = torch.empty((B, N, code_size), dtype=torch.float32, device=dev)
    bbox_weights = torch.empty((B, N, code_size), dtype=torch.float32, device=dev)
    ious = torch.empty((B, N), dtype=torch.float32, device=dev)
    num_pos = torch.empty((B,), dtype=torch.int32, device=dev)
    mean_iou = torch.empty((B,), dtype=torch.float32, device=dev)
    status = torch.empty((B,), dtype=torch.int32, device=dev)
    gt_inds = max_overlaps = cost = steps = None
    if extras:
        gt_inds = torch.empty((B, N), dtype=torch.int64, device=dev)
        max_overlaps = torch.empty((B, N), dtype=torch.float32, device=dev)
        cost = torch.full((B * L, P, nmax), float("nan"), dtype=torch.float32, device=dev)
        steps = torch.empty((B * L,), dtype=torch.int32, device=dev)
    L_ = _C.lib()
    ws_bytes = L_.bevb200_transfusion_assign_workspace_bytes(B, L, P, nmax)
    ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
    _C.check(L_.bevb200_transfusion_assign(
        _C.ptr(heatmap), _C.ptr(center), _C.ptr(height), _C.ptr(dim), _C.ptr(rot), _C.ptr(decoded), B, L, P, K,
        _C.ptr(boxes), _C.ptr(labels), _C.ptr(counts), nmax, D, float(pc[0]), float(pc[1]), float(vs[0]),
        float(vs[1]), osf, code_size, float(rng[0]), float(rng[1]), float(rng[3]), float(rng[4]), cls_w, alpha,
        gamma, reg_w, iou_w, pos_weight, _C.ptr(out_labels), _C.ptr(label_weights), _C.ptr(bbox_targets),
        _C.ptr(bbox_weights), _C.ptr(ious), _C.ptr(num_pos), _C.ptr(mean_iou), _C.ptr(status), _C.ptr(gt_inds),
        _C.ptr(max_overlaps), _C.ptr(cost), _C.ptr(steps), _C.ptr(ws), ws_bytes, _C.current_stream(dev)),
        "transfusion_assign")
    out = (out_labels, label_weights, bbox_targets, bbox_weights, ious, num_pos, mean_iou, status)
    if extras:
        return out, dict(gt_inds=gt_inds, max_overlaps=max_overlaps, cost=cost, steps=steps)
    return out


def _pred(preds, key):
    t = preds[key]
    return t.detach().to(torch.float32).contiguous() if isinstance(t, torch.Tensor) else t


def transfusion_assign_batched(preds, boxes, labels, counts, num_classes, num_proposals, train_cfg,
                               bbox_coder_cfg, return_extras=False):
    """TransFusionHead.get_targets without the heatmap, from padded ground truth (boxes [B, Nmax, 7 | 9] fp32,
    labels [B, Nmax] int32, counts [B] int32, as head_targets.pad_gt gives them) and the head's raw predictions
    preds = dict(heatmap [B, K, N] logits, center [B, 2, N], height [B, 1, N], dim [B, 3, N], rot [B, 2, N]; vel is
    not needed), N = L * num_proposals for L decoder layers, each layer matched on its own.
    train_cfg: point_cloud_range, pos_weight and assigner (HungarianAssigner3D with FocalLossCost, BBoxBEVL1Cost,
    IoU3DCost); bbox_coder_cfg: pc_range, voxel_size, out_size_factor, code_size.
    Returns (labels [B, N] int64, label_weights [B, N] int64, bbox_targets [B, N, code_size], bbox_weights
    [B, N, code_size], ious [B, N], num_pos [B] int32, mean_iou [B] fp32, status [B] int32), all on the device,
    without host synchronisation.  With return_extras also dict(gt_inds, max_overlaps, cost [B * L, P, Nmax]
    proposal-major (NaN past each sample's count), steps [B * L] solver steps)."""
    heatmap = _pred(preds, "heatmap")
    return _run(heatmap, _pred(preds, "center"), _pred(preds, "height"), _pred(preds, "dim"), _pred(preds, "rot"),
                None, boxes, labels, counts, num_classes, num_proposals, train_cfg, bbox_coder_cfg, return_extras)


def transfusion_targets(gt_bboxes_3d, gt_labels_3d, preds_dict, num_classes, num_proposals, train_cfg,
                        bbox_coder_cfg):
    """TransFusionHead.get_targets(gt_bboxes_3d, gt_labels_3d, preds_dict) (transfusion.py:357-406): gt as in
    head_targets.pad_gt (boxes on the CPU or the labels' device, labels on the device); preds_dict the head's
    output for the batch (a dict, or the reference's list whose [0] is that dict).  Returns (labels,
    label_weights, bbox_targets, bbox_weights, ious, num_pos, matched_ious, heatmap) as the reference does, with
    num_pos an int and matched_ious a float: one host synchronisation reads num_pos, the per-sample mean ious and
    the status together.  Raises ValueError where the reference would raise (see the module docstring)."""
    if not isinstance(preds_dict, dict):
        preds_dict = preds_dict[0]
    boxes, labels, counts = pad_gt([_box_tensor(b) for b in gt_bboxes_3d], gt_labels_3d)
    out = transfusion_assign_batched(preds_dict, boxes, labels, counts, num_classes, num_proposals, train_cfg,
                                     bbox_coder_cfg)
    heatmap = transfusion_heatmap_targets_batched(boxes, labels, counts, num_classes, train_cfg)
    num_pos, mean_iou, status = out[5], out[6], out[7]
    host = torch.cat([num_pos, mean_iou.view(torch.int32), status]).cpu().numpy()   # the one synchronisation
    B = num_pos.shape[0]
    st = host[2 * B:]
    if st.any():
        bad = [b for b in range(B) if st[b]]
        raise ValueError("samples %s: the matching cost has NaN / -inf entries, no complete assignment, or a gt "
                         "label outside [0, %d) (status %s)" % (bad, num_classes, st[bad].tolist()))
    ious_mean = [float(v) for v in host[B:2 * B].view(np.float32)]
    return (out[0], out[1], out[2], out[3], out[4], int(np.sum(host[:B])), float(np.mean(ious_mean)), heatmap)


class HungarianAssigner3D:
    """hungarian_assigner.py:82-142 on the device: assign(bboxes [P, 7 | 9] decoded, gt_bboxes [G, 7 | 9],
    gt_labels [G], cls_pred [1, K, P] logits, train_cfg) -> AssignResult(num_gts, gt_inds int64 [P] (0 or gt + 1),
    max_overlaps fp32 [P], labels int64 [P] (-1 when unmatched)); with no gt, max_overlaps is None as in the
    reference.  No host synchronisation: a failed matrix gives no matches, and `last_status` holds the status word
    ([1] int32 on the device) of the latest call."""

    def __init__(self, cls_cost=dict(type="FocalLossCost", weight=1.0), reg_cost=dict(type="BBoxBEVL1Cost",
                 weight=1.0), iou_cost=dict(type="IoU3DCost", weight=1.0), iou_calculator=dict(type="BboxOverlaps3D")):
        self.costs = _costs(cls_cost, reg_cost, iou_cost, iou_calculator)
        self.last_status = None

    def assign(self, bboxes, gt_bboxes, gt_labels, cls_pred, train_cfg):
        num_gts, num_bboxes = gt_bboxes.size(0), bboxes.size(0)
        dev = bboxes.device
        if num_gts == 0 or num_bboxes == 0:
            gt_inds = torch.full((num_bboxes,), 0 if num_gts == 0 else -1, dtype=torch.long, device=dev)
            return AssignResult(num_gts, gt_inds, None, torch.full((num_bboxes,), -1, dtype=torch.long, device=dev))
        _C.require_cuda(bboxes, "bboxes", torch.float32, contiguous=False)
        boxes = gt_bboxes.to(dev, torch.float32)[None, :, :7].contiguous()
        labels = gt_labels.to(dev, torch.int32)[None].contiguous()
        counts = torch.full((1,), num_gts, dtype=torch.int32, device=dev)
        heat = cls_pred.detach().to(torch.float32).reshape(1, -1, num_bboxes).contiguous()
        coder = dict(pc_range=[0.0, 0.0], voxel_size=[1.0, 1.0], out_size_factor=1, code_size=8)   # encode unused
        out, ex = _run(heat, None, None, None, None, bboxes.detach()[None, :, :7].contiguous(), boxes, labels, counts,
                       heat.shape[1], num_bboxes, train_cfg, coder, extras=True, costs=self.costs)
        self.last_status = out[7]
        gt_inds = ex["gt_inds"][0]
        assigned = torch.where(gt_inds > 0, out[0][0], torch.full_like(out[0][0], -1))
        return AssignResult(num_gts, gt_inds, ex["max_overlaps"][0], assigned)
