"""centerhead_decode -- the CenterHead inference tail on the device (csrc/centerhead_decode.cu): head outputs in,
boxes out.  The first half of CenterHead.get_bboxes (models/heads/bbox/centerpoint.py:637-757) is
CenterPointBBoxCoder.decode (core/bbox/coders/centerpoint_bbox_coders.py:62-225); here every task and sample of a
frame is decoded by one native call of two launches, and the NMS step (iou3d.centerhead_nms_batched) and the merge of
the tasks run on its padded output, so the batched forms have no host synchronisation and can be captured in a CUDA
graph.

    centerhead_decode_batched(tasks, coder, heat_is_logit=True, dim_is_log=True)
        -> (boxes [T * B, K, code], scores [T * B, K], labels [T * B, K] fp32, counts [T * B] int32)
    CenterPointBBoxCoder(pc_range, out_size_factor, voxel_size, post_center_range=None, max_num=100,
                         score_threshold=None, code_size=9).decode(heat, rot_sine, rot_cosine, hei, dim, vel,
                                                                   reg=None, task_id=-1)
        -> the reference's list over samples of dict(bboxes, scores, labels); one read of the counts
    centerhead_get_bboxes_batched(preds_dicts, bbox_coder, test_cfg, num_classes, norm_bbox=True)
        -> (bboxes [B, T * post_max_size, code], scores, labels int32, counts [B] int32), no device-to-host copy
    centerhead_get_bboxes(preds_dicts, bbox_coder, test_cfg, num_classes, norm_bbox=True)
        -> the reference's list over samples of [bboxes [n, code], scores [n], labels [n] int32]; one read-back

Semantics (the C header has them in full).  Segment s = t * B + b.  Per segment the K = max_num largest of the
task's cat * H * W scores are taken in descending score, NaN first, ties by ascending flat index
c * H * W + row * W + col: the reference's per-class top-k followed by its top-k over cat * K, with stable sorts (its
own are unstable, so its order of equal scores is unspecified).  The reference names the map [B, N, W, H]: its `xs` is
the row and its `ys` the column; x = (row + reg[0]) * out_size_factor * voxel_size[0] + pc_range[0], each step one
fp32 rounding.  A selected row survives when score > score_threshold (strict; only when score_threshold is truthy:
None and 0.0 both mean no score mask) and its centre (x, y, height) lies within post_center_range, limits included.  A
NaN score takes one of the K places and is then dropped by the score mask.  Survivors are compacted to the front of
their segment in descending-score order; rows at and after the count are zero (scores 0, labels 0).  Labels are
float32, as the reference's decode returns them.  GPU only: CPU tensors raise."""
import ctypes

import torch

from . import _C, iou3d

__all__ = ["centerhead_decode_batched", "CenterPointBBoxCoder", "centerhead_get_bboxes_batched",
           "centerhead_get_bboxes", "workspace_bytes", "MAX_TASKS", "MAX_SEGMENTS", "MAX_CLASSES", "MAX_CELLS",
           "MAX_NUM"]

MAX_TASKS = 16             # BEVB200_DECODE_MAX_TASKS
MAX_SEGMENTS = 65535       # BEVB200_DECODE_MAX_SEGMENTS, T * B
MAX_CLASSES = 64           # BEVB200_DECODE_MAX_CLASSES, per task
MAX_CELLS = 1 << 24        # BEVB200_DECODE_MAX_CELLS, cat * H * W per task and sample
MAX_NUM = 4096             # BEVB200_DECODE_MAX_K

_MAPS = (("heatmap", None), ("reg", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2))   # name, channels


class CenterPointBBoxCoder:
    """The reference's bbox coder for CenterPoint (same constructor and decode signature), decoding on the device.

    pc_range, voxel_size: the first two entries are used; out_size_factor: the head's stride; post_center_range:
    six limits of the centre (decode raises NotImplementedError without it, as the reference does); max_num: rows
    kept per sample before the masks; score_threshold: strict lower bound of the score, off when None or 0;
    code_size: 9 with velocity, 7 without."""

    def __init__(self, pc_range, out_size_factor, voxel_size, post_center_range=None, max_num=100,
                 score_threshold=None, code_size=9):
        self.pc_range = pc_range
        self.out_size_factor = out_size_factor
        self.voxel_size = voxel_size
        self.post_center_range = post_center_range
        self.max_num = max_num
        self.score_threshold = score_threshold
        self.code_size = code_size

    def encode(self):
        pass

    def decode(self, heat, rot_sine, rot_cosine, hei, dim, vel, reg=None, task_id=-1):
        """heat [B, N, H, W] scores (already activated), rot_sine / rot_cosine / hei [B, 1, H, W], dim [B, 3, H, W]
        sizes (already activated), vel [B, 2, H, W] or None, reg [B, 2, H, W] or None -> list over samples of
        dict(bboxes [n, 9 or 7], scores [n], labels [n] float32).  The counts are read back once."""
        for name, t in (("rot_sine", rot_sine), ("rot_cosine", rot_cosine)):
            if not isinstance(t, torch.Tensor) or t.dim() != 4 or t.shape[1] != 1:
                raise ValueError("%s must be [B, 1, H, W]" % name)
        task = dict(heatmap=heat, height=hei, dim=dim, rot=torch.cat([rot_sine, rot_cosine], 1))
        if vel is not None:
            task["vel"] = vel
        if reg is not None:
            task["reg"] = reg
        boxes, scores, labels, counts = centerhead_decode_batched([task], self, heat_is_logit=False,
                                                                  dim_is_log=False)
        return [dict(bboxes=boxes[i, :n], scores=scores[i, :n], labels=labels[i, :n])
                for i, n in enumerate(counts.tolist())]


def workspace_bytes(num_classes, B, H, W):
    """Device workspace of one decode of tasks with these class counts, 0 for sizes beyond the limits."""
    cat = _C.host_array(ctypes.c_int, [int(c) for c in num_classes])
    return int(_C.lib().bevb200_centerhead_decode_workspace_bytes(len(cat), B, cat, H, W))


def _coder_field(coder, name):
    return coder[name] if isinstance(coder, dict) else getattr(coder, name)


def _validate(tasks, K):
    if not isinstance(tasks, (list, tuple)) or len(tasks) < 1:
        raise ValueError("tasks must be a non-empty list of dicts of head outputs")
    has = {name: [name in t and t[name] is not None for t in tasks] for name, _ in _MAPS}
    for name in ("heatmap", "height", "dim", "rot"):
        if not all(has[name]):
            raise ValueError("every task needs '%s'" % name)
    for name in ("reg", "vel"):
        if any(has[name]) and not all(has[name]):
            raise ValueError("'%s' must be present in every task or in none" % name)
    heat0 = tasks[0]["heatmap"]
    if not isinstance(heat0, torch.Tensor) or heat0.dim() != 4:
        raise ValueError("heatmap must be [B, cat, H, W]")
    B, _, H, W = heat0.shape
    for t in tasks:
        for name, ch in _MAPS:
            if not has[name][0]:
                continue
            m = t[name]
            if not isinstance(m, torch.Tensor):
                raise TypeError("%s must be a torch.Tensor" % name)
            if m.dim() != 4 or (m.shape[0], m.shape[2], m.shape[3]) != (B, H, W) or (ch and m.shape[1] != ch):
                raise ValueError("%s must be [B, %s, H, W] = [%d, %s, %d, %d] in every task, got %s"
                                 % (name, ch or "cat", B, ch or "cat", H, W, tuple(m.shape)))
            if m.dtype != torch.float32:
                raise ValueError("%s must be fp32, got %s" % (name, m.dtype))
    cats = [int(t["heatmap"].shape[1]) for t in tasks]
    if min(B, H, W, min(cats)) < 1:
        raise ValueError("empty heatmap %s" % (tuple(heat0.shape),))
    if K < 1 or K > H * W:
        raise ValueError("max_num must be in 1..H * W = %d (got %d)" % (H * W, K))
    if (len(tasks) > MAX_TASKS or len(tasks) * B > MAX_SEGMENTS or max(cats) > MAX_CLASSES
            or max(cats) * H * W > MAX_CELLS or K > MAX_NUM):
        raise ValueError("at most %d tasks, %d task-samples, %d classes and %d cells per task and sample and "
                         "max_num %d (got %d tasks of %s classes, B %d, %d x %d, max_num %d)"
                         % (MAX_TASKS, MAX_SEGMENTS, MAX_CLASSES, MAX_CELLS, MAX_NUM, len(tasks), cats, B, H, W, K))
    for t in tasks:
        for name, _ in _MAPS:
            if has[name][0] and not t[name].is_cuda:
                raise ValueError("%s must be a CUDA tensor: bevfusion_b200 has no CPU implementation" % name)
    return cats, B, H, W, has["reg"][0], has["vel"][0]


def centerhead_decode_batched(tasks, coder, heat_is_logit=True, dim_is_log=True, with_index=False):
    """Decode every task and sample of a frame in one native call, without host synchronisation.

    tasks: list over tasks of dicts of fp32 CUDA maps: heatmap [B, cat_t, H, W], height [B, 1, H, W],
    dim [B, 3, H, W], rot [B, 2, H, W] (sine, cosine), and in every task or in none reg [B, 2, H, W] and
    vel [B, 2, H, W]; all tasks share B, H, W.  coder: a CenterPointBBoxCoder, or a dict with its fields pc_range,
    out_size_factor, voxel_size, post_center_range, max_num, score_threshold.  heat_is_logit: the heatmaps are raw
    head outputs (sigmoid is applied); dim_is_log: so are the sizes (exp is applied, the head's norm_bbox).
    Returns boxes [T * B, K, 9 or 7], scores [T * B, K], labels [T * B, K] float32 and counts [T * B] int32, row
    s = t * B + b, K = max_num: the surviving rows first, in descending score, zeros after them.  with_index adds
    index [T * B, K] int32, each row's cell row * W + col.  Raises ValueError for what the limits or the shapes
    rule out and NotImplementedError without a post_center_range."""
    rng = _coder_field(coder, "post_center_range")
    if rng is None:
        raise NotImplementedError("Need to reorganize output as a batch, only support post_center_range is not "
                                  "None for now!")
    if len(rng) != 6:
        raise ValueError("post_center_range must have six entries")
    K = int(_coder_field(coder, "max_num"))
    cats, B, H, W, has_reg, has_vel = _validate(tasks, K)
    thr = _coder_field(coder, "score_threshold")
    pc, vs = _coder_field(coder, "pc_range"), _coder_field(coder, "voxel_size")
    T, dev = len(tasks), tasks[0]["heatmap"].device
    S, code = T * B, 9 if has_vel else 7
    maps = {name: [t[name].detach().contiguous() for t in tasks] for name, _ in _MAPS
            if name not in ("reg", "vel") or (has_reg if name == "reg" else has_vel)}
    table = {name: _C.host_array(ctypes.c_void_p, [m.data_ptr() for m in ms]) for name, ms in maps.items()}
    boxes = torch.empty((S, K, code), dtype=torch.float32, device=dev)
    scores = torch.empty((S, K), dtype=torch.float32, device=dev)
    labels = torch.empty((S, K), dtype=torch.float32, device=dev)
    index = torch.empty((S, K), dtype=torch.int32, device=dev) if with_index else None
    counts = torch.empty((S,), dtype=torch.int32, device=dev)
    cat = _C.host_array(ctypes.c_int, cats)
    L = _C.lib()
    ws_bytes = int(L.bevb200_centerhead_decode_workspace_bytes(T, B, cat, H, W))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _C.check(L.bevb200_centerhead_decode(
            table["heatmap"], table.get("reg"), table["height"], table["dim"], table["rot"], table.get("vel"), cat,
            T, B, H, W, K, int(bool(heat_is_logit)), int(bool(dim_is_log)),
            float(_coder_field(coder, "out_size_factor")), float(vs[0]), float(vs[1]), float(pc[0]), float(pc[1]),
            _C.host_array(ctypes.c_double, [float(v) for v in rng]), int(bool(thr)), float(thr) if thr else 0.0,
            _C.ptr(boxes), _C.ptr(scores), _C.ptr(labels), _C.ptr(index), _C.ptr(counts), _C.ptr(ws), ws_bytes,
            _C.current_stream(dev)), "centerhead_decode")
    if with_index:
        return boxes, scores, labels, counts, index
    return boxes, scores, labels, counts


def _per_task(test_cfg, num_classes):
    """get_bboxes' per-task nms_type and nms_scale lists (centerpoint.py:646-666)."""
    T = len(num_classes)
    types = test_cfg["nms_type"]
    if not isinstance(types, list):
        types = [types] * T
    if "nms_scale" in test_cfg:
        scales = test_cfg["nms_scale"]
        if not isinstance(scales, list):
            scales = [[scales] * num_classes[t] for t in range(T)]
    else:
        scales = [[1.0] * num_classes[t] for t in range(T)]
    if len(types) != T or len(scales) != T:
        raise ValueError("nms_type and nms_scale need one entry per task (%d)" % T)
    return types, scales


def centerhead_get_bboxes_batched(preds_dicts, bbox_coder, test_cfg, num_classes, norm_bbox=True):
    """CenterHead.get_bboxes (centerpoint.py:637-757) for all tasks and samples without a device-to-host copy.

    preds_dicts: the head's output, a sequence over tasks of one-element lists of dicts of raw fp32 CUDA maps
    (heatmap, reg, height, dim, rot and optionally vel); bbox_coder: the head's CenterPointBBoxCoder (or a dict of
    its fields); test_cfg: the head's test_cfg (nms_type, a name or a list over tasks; optionally nms_scale;
    score_threshold, nms_thr, pre_max_size, post_max_size, post_center_limit_range, min_radius); num_classes: the
    class count of every task; norm_bbox: the head's flag (dim holds log sizes).  One decode call, then per task
    the NMS step (iou3d.centerhead_nms_batched), then the merge: tasks concatenated in task order, z lowered by
    half the height, labels offset by the class counts of the earlier tasks and cast to int32.
    Returns bboxes [B, T * post_max_size, code], scores [B, T * post_max_size], labels int32 and counts [B] int32:
    sample b's detections are rows [0, counts[b]), zeros after them."""
    num_classes = [int(c) for c in num_classes]
    if len(preds_dicts) != len(num_classes):
        raise ValueError("preds_dicts has %d tasks, num_classes %d" % (len(preds_dicts), len(num_classes)))
    types, scales = _per_task(test_cfg, num_classes)
    tasks = [p[0] for p in preds_dicts]
    boxes, scores, labels, counts = centerhead_decode_batched(tasks, bbox_coder, True, norm_bbox)
    B = boxes.shape[0] // len(tasks)
    parts, flag = [], 0
    for t in range(len(tasks)):
        seg = slice(t * B, (t + 1) * B)
        bb, sc, lb, n = iou3d.centerhead_nms_batched(boxes[seg], scores[seg], labels[seg], counts[seg], t, types[t],
                                                     test_cfg, scales[t], num_classes[t])
        live = torch.arange(bb.shape[1], device=bb.device)[None, :] < n[:, None]
        parts.append((bb, sc, torch.where(live, lb + flag, torch.zeros_like(lb)).int(), live))
        flag += num_classes[t]
    bb, sc, lb, live = (torch.cat([p[i] for p in parts], 1) for i in range(4))
    # the live rows of every sample to its front, tasks in order
    slot = torch.argsort((~live).to(torch.int8), dim=1, stable=True)
    bb = bb.gather(1, slot[..., None].expand(-1, -1, bb.shape[2]))
    bb[..., 2] = bb[..., 2] - bb[..., 5] * 0.5
    return bb, sc.gather(1, slot), lb.gather(1, slot), live.sum(1, dtype=torch.int32)


def centerhead_get_bboxes(preds_dicts, bbox_coder, test_cfg, num_classes, norm_bbox=True):
    """CenterHead.get_bboxes in the reference's list form: per sample [bboxes [n, code], scores [n], labels [n]
    int32] (bboxes a plain tensor: there is no box_type_3d here).  centerhead_get_bboxes_batched followed by one
    read of the per-sample counts."""
    bb, sc, lb, counts = centerhead_get_bboxes_batched(preds_dicts, bbox_coder, test_cfg, num_classes, norm_bbox)
    return [[bb[i, :n], sc[i, :n], lb[i, :n]] for i, n in enumerate(counts.tolist())]
