"""iou3d -- rotated BEV IoU and NMS for the CenterHead box post-processing (csrc/box_nms.cu).

Mirrors of mmdet3d/ops/iou3d/iou3d_utils.py, same signatures, dtypes and devices:
    boxes_iou_bev(boxes_a, boxes_b)                                   -> [M, N] IoU
    nms_gpu(boxes, scores, thresh, pre_maxsize=None, post_max_size=None) -> int64 indices
    nms_normal_gpu(boxes, scores, thresh)                             -> int64 indices
and of core/post_processing/box3d_nms.py:
    circle_nms(dets, thresh, post_max_size=83)   dets a CUDA [N, 3] tensor (x, y, score) -> int64 CUDA indices

Batched forms with no host synchronisation (CUDA-graph capturable):
    nms_batched(boxes, scores, counts, mode, thresh, pre_max_size, post_max_size) -> (keep, keep_count)
    centerhead_nms(decoded, task_id, nms_type, test_cfg, nms_scale, num_classes=...)
                                              the NMS step of CenterHead.get_bboxes for one task over the batch

Boxes are [x1, y1, x2, y2, ry] fp32 (xywhr2xyxyr form).  The mirrors sort with the reference's own
`scores.sort(0, descending=True)`, so equal scores order as in the reference on the same torch.  circle_nms
sorts with torch too, where the reference uses numpy `argsort()[::-1]`: on equal scores the two orders may
differ, and so may the keep lists.  nms_batched and centerhead_nms sort stably, so equal scores keep their row
order; the reference sorts each list with torch's default sort, whose order of equal scores is not fixed, so on
tied scores their keep lists may differ from the reference's.  nms_gpu, nms_normal_gpu and circle_nms read the kept count back to size
their result (one device-to-host copy; the reference copies the whole pair mask).  GPU only: CPU tensors
raise."""
import torch

from . import _C

__all__ = ["boxes_iou_bev", "boxes_overlap_bev", "nms_gpu", "nms_normal_gpu", "circle_nms", "nms_batched",
           "centerhead_nms", "xywhr2xyxyr", "MODES"]

MODES = {"rotate": 0, "normal": 1, "circle": 2}   # BEVB200_NMS_ROTATE / _NORMAL / _CIRCLE
MAX_BOXES = 65536                                  # BEVB200_NMS_MAX_BOXES


def _dense(boxes_a, boxes_b, fn):
    _C.require_cuda(boxes_a, "boxes_a", torch.float32)
    _C.require_cuda(boxes_b, "boxes_b", torch.float32)
    if boxes_a.dim() != 2 or boxes_a.shape[1] != 5 or boxes_b.dim() != 2 or boxes_b.shape[1] != 5:
        raise ValueError("boxes must be [N, 5] ([x1, y1, x2, y2, ry])")
    out = torch.empty((boxes_a.shape[0], boxes_b.shape[0]), dtype=torch.float32, device=boxes_a.device)
    _C.check(fn(_C.ptr(boxes_a), boxes_a.shape[0], _C.ptr(boxes_b), boxes_b.shape[0], _C.ptr(out),
                _C.current_stream(boxes_a.device)), "boxes_bev")
    return out


def boxes_iou_bev(boxes_a, boxes_b):
    """Rotated BEV IoU of boxes_a [M, 5] and boxes_b [N, 5] -> [M, N] fp32 (iou3d_utils.py:6-21)."""
    return _dense(boxes_a.contiguous(), boxes_b.contiguous(), _C.lib().bevb200_boxes_iou_bev)


def boxes_overlap_bev(boxes_a, boxes_b):
    """Rotated BEV overlap area of boxes_a [M, 5] and boxes_b [N, 5] -> [M, N] fp32."""
    return _dense(boxes_a.contiguous(), boxes_b.contiguous(), _C.lib().bevb200_boxes_overlap_bev)


def _nms(sorted_boxes, counts, mode, thresh, post_max, order=None):
    """Native greedy NMS of [S, nmax, D] boxes sorted by score -> (keep [S, post_max] int64, keep_count [S])."""
    S, nmax = sorted_boxes.shape[0], sorted_boxes.shape[1]
    if nmax > MAX_BOXES:
        raise ValueError("NMS takes at most %d boxes per list (got %d)" % (MAX_BOXES, nmax))
    dev = sorted_boxes.device
    keep = torch.empty((S, post_max), dtype=torch.int64, device=dev)
    keep_count = torch.empty((S,), dtype=torch.int32, device=dev)
    L = _C.lib()
    ws_bytes = L.bevb200_nms_workspace_bytes(S, nmax)
    ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
    _C.check(L.bevb200_nms(_C.ptr(sorted_boxes), _C.ptr(counts), S, nmax, MODES[mode], float(thresh), post_max,
                           _C.ptr(order), _C.ptr(keep), _C.ptr(keep_count), _C.ptr(ws), ws_bytes,
                           _C.current_stream(dev)), "nms")
    return keep, keep_count


def _single(boxes, scores, thresh, mode, pre_maxsize=None, post_max_size=None):
    _C.require_cuda(boxes, "boxes", torch.float32, contiguous=False)
    _C.require_cuda(scores, "scores", contiguous=False)
    order = scores.sort(0, descending=True)[1]
    if pre_maxsize is not None:
        order = order[:pre_maxsize]
    boxes = boxes[order].contiguous()
    n = boxes.shape[0]
    post = n if post_max_size is None else max(0, min(int(post_max_size), n))
    keep, count = _nms(boxes[None], None, mode, thresh, post, order[None].contiguous())
    return keep[0, :int(count.item())]


def nms_gpu(boxes, scores, thresh, pre_maxsize=None, post_max_size=None):
    """Rotated NMS (iou3d_utils.py:24-48): boxes [N, 5] ([x1, y1, x2, y2, ry]), scores [N] -> kept indices
    (int64, on the boxes' device) in descending score order."""
    return _single(boxes, scores, thresh, "rotate", pre_maxsize, post_max_size)


def nms_normal_gpu(boxes, scores, thresh):
    """Axis-aligned NMS (iou3d_utils.py:51-68): the angle column is ignored."""
    return _single(boxes, scores, thresh, "normal")


def circle_nms(dets, thresh, post_max_size=83):
    """Circle NMS (box3d_nms.py:180-219) on a CUDA [N, 3] tensor (x, y, score): a detection is dropped when
    a kept, higher-scored centre lies at squared distance <= thresh.  Returns int64 CUDA indices."""
    _C.require_cuda(dets, "dets", torch.float32, contiguous=False)
    return _single(dets[:, :2], dets[:, 2], thresh, "circle", None, post_max_size)


def nms_batched(boxes, scores, counts, mode, thresh, pre_max_size=None, post_max_size=None):
    """Greedy NMS of S padded lists in one native call, without host synchronisation.

    boxes [S, Nmax, 5] fp32 ([x1, y1, x2, y2, ry]; for mode "circle" the first two columns are the
    centres), scores [S, Nmax], counts [S] int (list s is rows [0, counts[s])), mode "rotate", "normal" or
    "circle".  Each list is sorted by descending score (stable: equal scores keep their row order; pads
    last), cut to pre_max_size, suppressed, and cut to post_max_size.  Returns keep [S, P] int64 (row indices into the list, -1 padded, P = post_max_size, or
    min(pre_max_size, Nmax) when it is None) and keep_count [S] int32."""
    _C.require_cuda(boxes, "boxes", torch.float32, contiguous=False)
    _C.require_cuda(scores, "scores", contiguous=False)
    _C.require_cuda(counts, "counts", contiguous=False)
    if mode not in MODES:
        raise ValueError("mode must be one of %s" % sorted(MODES))
    S, nmax = scores.shape
    counts = counts.to(torch.int32)
    pad = torch.arange(nmax, device=scores.device)[None, :] >= counts[:, None].long()
    order = scores.masked_fill(pad, float("-inf")).sort(dim=1, descending=True, stable=True)[1]
    if pre_max_size is not None and pre_max_size < nmax:
        order = order[:, :pre_max_size]
        counts = counts.clamp(max=pre_max_size)
    order = order.contiguous()
    d = 2 if mode == "circle" else 5
    sorted_boxes = boxes[..., :d].gather(1, order[..., None].expand(-1, -1, d)).contiguous()
    post = order.shape[1] if post_max_size is None else int(post_max_size)
    return _nms(sorted_boxes, counts.contiguous(), mode, thresh, post, order)


def xywhr2xyxyr(boxes_xywhr):
    """[x, y, w, h, r] -> [x1, y1, x2, y2, r] (core/bbox/structures/utils.py:71-89)."""
    boxes = torch.zeros_like(boxes_xywhr)
    half_w = boxes_xywhr[..., 2] / 2
    half_h = boxes_xywhr[..., 3] / 2
    boxes[..., 0] = boxes_xywhr[..., 0] - half_w
    boxes[..., 1] = boxes_xywhr[..., 1] - half_h
    boxes[..., 2] = boxes_xywhr[..., 0] + half_w
    boxes[..., 3] = boxes_xywhr[..., 1] + half_h
    boxes[..., 4] = boxes_xywhr[..., 4]
    return boxes


def _pad(tensors, fill=0):
    n = max([t.shape[0] for t in tensors] + [1])
    out = tensors[0].new_full((len(tensors), n) + tuple(tensors[0].shape[1:]), fill)
    for i, t in enumerate(tensors):
        out[i, :t.shape[0]] = t
    return out


def centerhead_nms(decoded, task_id, nms_type, test_cfg, nms_scale=None, num_classes=None):
    """The NMS step of CenterHead.get_bboxes for one task (models/heads/bbox/centerpoint.py:710-737 for
    "circle", get_task_detections :768-884 otherwise) over every sample of the batch in one nms_batched call.

    decoded: list over samples of dicts(bboxes [n, code_size], scores [n], labels [n]) from
    bbox_coder.decode; test_cfg: the head's test_cfg (score_threshold, nms_thr, pre_max_size, post_max_size,
    post_center_limit_range, min_radius); nms_scale: the BEV size scales of this task, a list over its
    classes or one number for all (None, as when the config sets no nms_scale: 1.0); num_classes: the task's
    class count, `self.num_classes[task_id]` (num_class_with_bg, :670; with one class every label becomes 0,
    :804-811).  num_classes may be left out only when nms_scale is a per-class list, which get_bboxes builds
    with one entry per class (:650-666); then it is the list's length.  Without either the class count is
    unknown and ValueError is raised, rather than guessing one class and relabelling every box as class 0.
    Returns the reference's list of per-sample dict(bboxes, scores, labels).  The kept counts are read back
    once, to split the result per sample.  Lists are sorted stably (see nms_batched)."""
    if num_classes is None:
        if not isinstance(nms_scale, (list, tuple)):
            raise ValueError("centerhead_nms needs num_classes (self.num_classes[task_id]) unless nms_scale is a "
                             "per-class list")
        num_classes = len(nms_scale)
    num_classes = int(num_classes)
    if num_classes < 1:
        raise ValueError("num_classes must be >= 1")
    if nms_scale is None:
        nms_scale = [1.0] * int(num_classes)
    elif not isinstance(nms_scale, (list, tuple)):
        nms_scale = [float(nms_scale)] * int(num_classes)
    boxes = [d["bboxes"] for d in decoded]
    scores = [d["scores"] for d in decoded]
    labels = [d["labels"] for d in decoded]
    for b in boxes:
        _C.require_cuda(b, "bboxes", contiguous=False)
    dev, B = boxes[0].device, len(decoded)
    counts = torch.tensor([b.shape[0] for b in boxes], dtype=torch.int32).to(dev, non_blocking=True)
    pb, ps = _pad(boxes), _pad(scores, float("-inf"))
    post_max = int(test_cfg["post_max_size"])
    if nms_type == "circle":
        keep, kc = nms_batched(pb, ps, counts, "circle", test_cfg["min_radius"][task_id], None, post_max)
        pl = _pad(labels)
        valid = torch.arange(keep.shape[1], device=dev)[None, :] < kc[:, None].long()
    else:
        pl = _pad([l.long() if num_classes > 1 else torch.zeros_like(l, dtype=torch.long) for l in labels])
        live = torch.arange(pb.shape[1], device=dev)[None, :] < counts[:, None].long()
        thr = float(test_cfg["score_threshold"])
        if thr > 0.0:
            live &= ps >= torch.tensor([thr], device=dev).type_as(ps)
        # the rows above the score threshold, moved to the front of each list in their order
        perm = torch.argsort((~live).to(torch.int8), dim=1, stable=True)
        bev = pb[..., [0, 1, 3, 4, 6]]                     # LiDARInstance3DBoxes.bev
        table = torch.tensor(list(nms_scale) + [1.0], dtype=bev.dtype, device=dev)
        k = len(nms_scale)                                 # labels outside 0..k-1 keep their size, as in :829-832
        cls = torch.where((pl >= 0) & (pl < k), pl, torch.full_like(pl, k))
        bev[..., 2:4] *= table[cls][..., None]
        keep, kc = nms_batched(xywhr2xyxyr(bev).gather(1, perm[..., None].expand(-1, -1, 5)), ps.gather(1, perm),
                               live.sum(1, dtype=torch.int32), "rotate", test_cfg["nms_thr"],
                               test_cfg["pre_max_size"], post_max)
        keep = perm.gather(1, keep.clamp(min=0))
        valid = torch.arange(keep.shape[1], device=dev)[None, :] < kc[:, None].long()
        rng = test_cfg["post_center_limit_range"]
        if len(rng) > 0:
            rng = torch.tensor(rng, dtype=pb.dtype, device=dev)
            ctr = pb.gather(1, keep[..., None].expand(-1, -1, pb.shape[2]))[..., :3]
            valid &= (ctr >= rng[:3]).all(-1) & (ctr <= rng[3:]).all(-1)
    # compact the valid slots of every row to its front, keeping their order; one read of the lengths
    slot = torch.argsort((~valid).to(torch.int8), dim=1, stable=True)
    idx = keep.gather(1, slot).clamp(min=0)
    lengths = valid.sum(1).tolist()
    out = []
    for i in range(B):
        sel = idx[i, :lengths[i]]
        if nms_type == "circle":
            out.append(dict(bboxes=boxes[i][sel], scores=scores[i][sel], labels=labels[i][sel]))
        else:
            out.append(dict(bboxes=pb[i, sel], scores=ps[i, sel], labels=pl[i, sel]))
    return out
