"""head_targets -- the heatmap training targets of CenterHead and TransFusionHead on the device
(csrc/head_targets.cu), with no per-object host loop.

    centerhead_targets(gt_bboxes_3d, gt_labels_3d, tasks, train_cfg, norm_bbox=True)
        -> (heatmaps, anno_boxes, inds, masks), per-task lists stacked over the batch, as CenterHead.get_targets
           (models/heads/bbox/centerpoint.py:397-582)
    transfusion_heatmap_targets(gt_bboxes_3d, gt_labels_3d, num_classes, train_cfg)
        -> heatmap [B, ncls, fmap_y, fmap_x], the dense heatmap of TransFusionHead.get_targets (transfusion.py:526-573)
    centerhead_targets_batched / transfusion_heatmap_targets_batched
        the same from padded boxes [B, Nmax, 7 | 9], labels [B, Nmax] and device counts [B]; no host
        synchronisation, CUDA-graph capturable
    gaussian_radius(det_size, min_overlap), draw_heatmap_gaussian(heatmap, center, radius, k=1)
        mirrors of mmdet3d.core.utils.gaussian

One native call per batch: three launches (zero, assign, draw).  The list forms take the boxes on the CPU (where
the reference's data pipeline keeps them) or on the labels' CUDA device and pad them from host-known shapes, so they
add no synchronisation either.  Sizes, radii and centres are the reference's fp32 arithmetic op for
op and the gaussian is evaluated in double as gaussian_2d does, so the targets equal the reference's bit for bit
(the log / sin / cos of anno_box within 2 ulp).  With box_dim 7 anno_box has 8 columns (no velocity; the reference
would fail to unpack one).  Deviation: a box whose centre is not finite is skipped (the reference's float-to-int
conversion of NaN is undefined).  GPU only: CPU tensors raise."""
import ctypes

import torch

from . import _C

__all__ = ["centerhead_targets", "centerhead_targets_batched", "transfusion_heatmap_targets",
           "transfusion_heatmap_targets_batched", "gaussian_radius", "draw_heatmap_gaussian", "MODES"]

MODES = {"centerhead": 0, "transfusion": 1}   # BEVB200_HEAD_TARGETS_CENTERHEAD / _TRANSFUSION
MAX_BOXES = 4096                               # BEVB200_HEAD_TARGETS_MAX_BOXES
MAX_TASKS = 32                                 # BEVB200_HEAD_TARGETS_MAX_TASKS
MAX_LABELS = 256                               # BEVB200_HEAD_TARGETS_MAX_LABELS


def _fp32(v):
    """A Python number as the fp32 value torch.tensor([...]) would hold."""
    return float(torch.tensor(float(v), dtype=torch.float32))


def task_class_counts(tasks):
    """Classes per task from CenterHead's `tasks` config (dicts with class_names or num_class) or from lists of
    class names."""
    counts = []
    for t in tasks:
        if isinstance(t, dict):
            counts.append(len(t["class_names"]) if "class_names" in t else int(t["num_class"]))
        elif isinstance(t, int):
            counts.append(int(t))
        else:
            counts.append(len(t))
    if not counts or len(counts) > MAX_TASKS or min(counts) < 1:
        raise ValueError("tasks must give 1..%d tasks of at least one class each" % MAX_TASKS)
    return counts


def centerhead_label_table(task_classes):
    """Label -> (task, channel): label flag_t + c is class c of task t (centerpoint.py:463-471)."""
    return [(t, c) for t, n in enumerate(task_classes) for c in range(n)]


def _grid(train_cfg):
    osf = int(train_cfg["out_size_factor"])
    gs = train_cfg["grid_size"]
    pc, vs = train_cfg["point_cloud_range"], train_cfg["voxel_size"]
    return dict(pc_x=_fp32(pc[0]), pc_y=_fp32(pc[1]), vs_x=_fp32(vs[0]), vs_y=_fp32(vs[1]), osf=osf,
                fmap_x=int(gs[0]) // osf, fmap_y=int(gs[1]) // osf)


def _check_inputs(boxes, labels, counts):
    _C.require_cuda(boxes, "boxes", torch.float32)
    _C.require_cuda(labels, "labels", torch.int32)
    _C.require_cuda(counts, "counts", torch.int32)
    if boxes.dim() != 3 or boxes.shape[2] not in (7, 9):
        raise ValueError("boxes must be [B, Nmax, 7 | 9] (LiDARInstance3DBoxes.tensor rows), got %s"
                         % (tuple(boxes.shape),))
    B, nmax = boxes.shape[0], boxes.shape[1]
    if tuple(labels.shape) != (B, nmax) or tuple(counts.shape) != (B,):
        raise ValueError("labels must be [B, Nmax] and counts [B] for boxes %s" % (tuple(boxes.shape),))
    if nmax > MAX_BOXES:
        raise ValueError("at most %d boxes per sample (got %d)" % (MAX_BOXES, nmax))
    if boxes.device != labels.device or boxes.device != counts.device:
        raise ValueError("boxes, labels and counts must be on one device")


def _run(boxes, labels, counts, mode, task_classes, label_table, train_cfg, max_objs=0, norm_bbox=True):
    """One native call.  Returns (heatmap, anno_box, ind, mask, status, records): heatmap is the task-major
    flat buffer, records the [B, Nmax, 4] int32 draw records (plane, row, col, radius; radius -1: none)."""
    _check_inputs(boxes, labels, counts)
    if mode not in MODES:
        raise ValueError("mode must be one of %s" % sorted(MODES))
    if len(label_table) > MAX_LABELS:
        raise ValueError("at most %d labels" % MAX_LABELS)
    for t, c in label_table:
        if not (t == -1 or (0 <= t < len(task_classes) and 0 <= c < task_classes[t])):
            raise ValueError("bad label table entry (%d, %d)" % (t, c))
    g = _grid(train_cfg)
    if g["fmap_x"] < 1 or g["fmap_y"] < 1:
        raise ValueError("grid_size // out_size_factor must be >= 1")
    B, nmax, D = boxes.shape
    dev = boxes.device
    T = len(task_classes)
    heatmap = torch.empty((B * sum(task_classes) * g["fmap_y"] * g["fmap_x"],), dtype=torch.float32, device=dev)
    A = 10 if D == 9 else 8
    if mode == "centerhead":
        anno = torch.empty((T, B, max_objs, A), dtype=torch.float32, device=dev)
        ind = torch.empty((T, B, max_objs), dtype=torch.int64, device=dev)
        mask = torch.empty((T, B, max_objs), dtype=torch.uint8, device=dev)
    else:
        anno = ind = mask = None
    status = torch.empty((1,), dtype=torch.int32, device=dev)
    L = _C.lib()
    ws_bytes = L.bevb200_head_targets_workspace_bytes(B, nmax)
    records = torch.empty((max(ws_bytes // 16, 1), 4), dtype=torch.int32, device=dev)
    table = _C.host_array(ctypes.c_int32, [v for e in label_table for v in e] or [0])
    classes = _C.host_array(ctypes.c_int32, task_classes)
    _C.check(L.bevb200_head_targets(
        _C.ptr(boxes), _C.ptr(labels), _C.ptr(counts), B, nmax, D, ctypes.addressof(table), len(label_table),
        ctypes.addressof(classes), T, g["pc_x"], g["pc_y"], g["vs_x"], g["vs_y"], g["osf"], g["fmap_x"],
        g["fmap_y"], float(train_cfg["gaussian_overlap"]), int(train_cfg["min_radius"]), MODES[mode], max_objs,
        int(bool(norm_bbox)), _C.ptr(heatmap), _C.ptr(anno), _C.ptr(ind), _C.ptr(mask), _C.ptr(status),
        _C.ptr(records), ws_bytes, _C.current_stream(dev)), "head_targets")
    return heatmap, anno, ind, mask, status, records[:B * nmax].view(B, nmax, 4)


def _split_heatmap(flat, B, task_classes, fmap_y, fmap_x):
    out, off = [], 0
    for n in task_classes:
        size = B * n * fmap_y * fmap_x
        out.append(flat[off:off + size].view(B, n, fmap_y, fmap_x))
        off += size
    return out


def centerhead_targets_batched(boxes, labels, counts, tasks, train_cfg, norm_bbox=True, return_status=False):
    """CenterHead.get_targets from padded inputs: boxes [B, Nmax, 7 | 9] fp32, labels [B, Nmax] int32 and
    counts [B] int32, all on one CUDA device (sample b is rows [0, counts[b])).  tasks: the head's `tasks` config
    (or lists of class names); train_cfg: point_cloud_range, grid_size, voxel_size, out_size_factor, dense_reg,
    gaussian_overlap, max_objs, min_radius.  Returns (heatmaps, anno_boxes, inds, masks), lists over tasks of
    [B, ncls_t, fmap_y, fmap_x], [B, M, 10 | 8], int64 [B, M] and uint8 [B, M] (M = max_objs * dense_reg),
    each a contiguous view; with return_status also the int32 [1] status word (see the C header)."""
    task_classes = task_class_counts(tasks)
    g = _grid(train_cfg)
    M = int(train_cfg["max_objs"]) * int(train_cfg.get("dense_reg", 1))
    hm, anno, ind, mask, status, _ = _run(boxes, labels, counts, "centerhead", task_classes,
                                          centerhead_label_table(task_classes), train_cfg, M, norm_bbox)
    B = boxes.shape[0]
    out = (_split_heatmap(hm, B, task_classes, g["fmap_y"], g["fmap_x"]), list(anno.unbind(0)),
           list(ind.unbind(0)), list(mask.unbind(0)))
    return out + (status,) if return_status else out


def transfusion_heatmap_targets_batched(boxes, labels, counts, num_classes, train_cfg, return_status=False):
    """The dense heatmap of TransFusionHead.get_targets from padded inputs (see centerhead_targets_batched):
    [B, num_classes, fmap_y, fmap_x] fp32; with return_status also the status word (boxes skipped for a label
    outside [0, num_classes) or an infinite size)."""
    num_classes = int(num_classes)
    if not 1 <= num_classes <= MAX_LABELS:
        raise ValueError("num_classes must be in 1..%d" % MAX_LABELS)
    g = _grid(train_cfg)
    hm, _, _, _, status, _ = _run(boxes, labels, counts, "transfusion", [num_classes],
                                  [(0, c) for c in range(num_classes)], train_cfg)
    hm = hm.view(boxes.shape[0], num_classes, g["fmap_y"], g["fmap_x"])
    return (hm, status) if return_status else hm


def _box_tensor(b):
    return b.tensor if hasattr(b, "tensor") else b


def pad_gt(gt_bboxes_3d, gt_labels_3d):
    """Lists over samples of boxes [n_i, D] (tensors or objects with .tensor) and labels [n_i] -> the padded
    (boxes [B, Nmax, D] fp32, labels [B, Nmax] int32, counts [B] int32) on the labels' CUDA device.

    As in the reference's training step, the boxes may be on the CPU (the data pipeline keeps
    LiDARInstance3DBoxes there, formating.py:122-124, and get_targets_single moves them to the labels' device):
    boxes on the CPU are padded into one pinned host buffer and copied with one asynchronous transfer.  Boxes
    already on the labels' device are padded there.  The counts come from the host-known shapes, also through
    pinned memory: no synchronisation.  The labels must be CUDA tensors."""
    boxes = [_box_tensor(b) for b in gt_bboxes_3d]
    if len(boxes) == 0 or len(boxes) != len(gt_labels_3d):
        raise ValueError("need one box set and one label tensor per sample")
    dev = gt_labels_3d[0].device if isinstance(gt_labels_3d[0], torch.Tensor) else None
    for i, b in enumerate(boxes):
        _C.require_cuda(gt_labels_3d[i], "gt_labels_3d[%d]" % i, contiguous=False)
        if gt_labels_3d[i].device != dev:
            raise ValueError("gt_labels_3d must all be on one CUDA device")
        if not isinstance(b, torch.Tensor):
            raise TypeError("gt_bboxes_3d[%d] must be a tensor or have a .tensor attribute" % i)
        if b.device.type != "cpu" and b.device != dev:
            raise ValueError("gt_bboxes_3d[%d] is on %s; boxes must be on the CPU or on the labels' device %s"
                             % (i, b.device, dev))
        if b.dim() != 2 or b.shape[0] != gt_labels_3d[i].shape[0]:
            raise ValueError("sample %d: boxes [n, D] and labels [n] disagree" % i)
    D = boxes[0].shape[1]
    if any(b.shape[1] != D for b in boxes):
        raise ValueError("every sample's boxes must have the same number of columns")
    n = [b.shape[0] for b in boxes]
    B, nmax = len(boxes), max(n)
    host = [i for i, b in enumerate(boxes) if b.device.type == "cpu"]
    if host:
        staged = torch.zeros((B, nmax, D), dtype=torch.float32, pin_memory=True)
        for i in host:
            staged[i, :n[i]] = boxes[i]
        pb = staged.to(dev, non_blocking=True)
    else:
        pb = torch.zeros((B, nmax, D), dtype=torch.float32, device=dev)
    pl = torch.zeros((B, nmax), dtype=torch.int32, device=dev)
    for i, (b, l) in enumerate(zip(boxes, gt_labels_3d)):
        if n[i]:
            if b.device.type != "cpu":
                pb[i, :n[i]] = b
            pl[i, :n[i]] = l
    counts = torch.tensor(n, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
    return pb, pl, counts


def centerhead_targets(gt_bboxes_3d, gt_labels_3d, tasks, train_cfg, norm_bbox=True):
    """CenterHead.get_targets (centerpoint.py:397-430): gt_bboxes_3d a list over samples of LiDARInstance3DBoxes
    (or [n, 7 | 9] tensors), on the CPU as the reference's data pipeline delivers them or on the labels' device;
    gt_labels_3d a list of [n] CUDA label tensors (see pad_gt).  Returns (heatmaps, anno_boxes, inds, masks) as
    per-task lists stacked over the batch, on the labels' device."""
    return centerhead_targets_batched(*pad_gt(gt_bboxes_3d, gt_labels_3d), tasks, train_cfg, norm_bbox)


def transfusion_heatmap_targets(gt_bboxes_3d, gt_labels_3d, num_classes, train_cfg):
    """The `heatmap` of TransFusionHead.get_targets (transfusion.py:526-573, stacked over the batch):
    [B, num_classes, fmap_y, fmap_x] fp32 on the labels' device.  Boxes and labels as in centerhead_targets."""
    return transfusion_heatmap_targets_batched(*pad_gt(gt_bboxes_3d, gt_labels_3d), num_classes, train_cfg)


def gaussian_radius(det_size, min_overlap=0.5):
    """gaussian.py:55-84 on fp32 tensors (or numbers), elementwise: the radius the targets use before
    max(min_radius, int(r)).  Plain torch: this is the host-side helper, not the hot path.  The square roots are
    correctly rounded on every device, as in the kernel (torch's fp32 sqrt on CPU may be off by one ulp)."""
    height, width = (torch.as_tensor(v, dtype=torch.float32) for v in det_size)

    def sqrt(x):   # the float64 root of an fp32 value rounds to the correctly rounded fp32 root
        return torch.sqrt(x.double()).float()

    a1 = 1
    b1 = height + width
    c1 = width * height * (1 - min_overlap) / (1 + min_overlap)
    r1 = (b1 + sqrt(b1 ** 2 - 4 * a1 * c1)) / 2
    a2 = 4
    b2 = 2 * (height + width)
    c2 = (1 - min_overlap) * width * height
    r2 = (b2 + sqrt(b2 ** 2 - 4 * a2 * c2)) / 2
    a3 = 4 * min_overlap
    b3 = -2 * min_overlap * (height + width)
    c3 = (min_overlap - 1) * width * height
    r3 = (b3 + sqrt(b3 ** 2 - 4 * a3 * c3)) / 2
    r = torch.where(r2 < r1, r2, r1)              # Python's min(r1, r2, r3), NaN included
    return torch.where(r3 < r, r3, r)


def draw_heatmap_gaussian(heatmap, center, radius, k=1):
    """gaussian.py:24-52: every cell of the (2 radius + 1)^2 window at column int(center[0]), row int(center[1]),
    clipped to the [H, W] fp32 CUDA heatmap, becomes torch.max(cell, gaussian * k), as the reference's
    torch.max(masked_heatmap, masked_gaussian * k, out=masked_heatmap) does: cells where the gaussian is 0 are
    maxed with 0 too, k may be any number, and a NaN in the heatmap or in k propagates.  Runs the targets' draw
    kernel with one record.  `center` held on the device is read back (int(), as the reference does).  Returns
    heatmap."""
    _C.require_cuda(heatmap, "heatmap", torch.float32)
    if heatmap.dim() < 2:
        raise ValueError("heatmap must be [H, W]")
    if heatmap.dim() > 2:
        raise ValueError("heatmap must be one [H, W] plane")
    x, y, radius = int(center[0]), int(center[1]), int(radius)
    if not 0 <= radius < 2 ** 30:
        raise ValueError("radius must be in [0, 2^30)")
    x, y = (min(max(v, -2 ** 31), 2 ** 31 - 1) for v in (x, y))   # farther out draws nothing either way
    H, W = heatmap.shape
    _C.check(_C.lib().bevb200_draw_heatmap_gaussian(_C.ptr(heatmap), H, W, x, y, radius, float(k),
                                                     _C.current_stream(heatmap.device)), "draw_heatmap_gaussian")
    return heatmap
