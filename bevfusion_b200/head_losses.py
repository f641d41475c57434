"""head_losses -- the training losses of CenterHead and TransFusionHead and their gradients on the device
(csrc/head_losses.cu), with no host synchronisation.

    centerhead_loss(preds_dicts, targets, train_cfg, loss_cls=..., loss_bbox=..., return_status=False)
        -> CenterHead.loss's dict (models/heads/bbox/centerpoint.py:584-634): heatmap/task{t}, bbox/task{t}
    transfusion_loss(preds_dicts, targets, num_proposals, num_decoder_layers, auxiliary, train_cfg, loss_cls=...,
                     loss_bbox=..., loss_heatmap=..., return_status=False)
        -> TransFusionHead.loss's dict (transfusion.py:587-713): loss_heatmap, {prefix}_loss_cls,
           {prefix}_loss_bbox per trained layer, matched_ious

Both are torch.autograd.Functions over one native call per direction (forward: two launches; backward: two for
CenterHead, one for TransFusion): the gradients flow to every prediction tensor they read.  The values are 0-d fp32
device tensors; with return_status also the int32 [1] status word (STATUS bits: an `ind` outside the map on a
masked-in slot, a label outside [0, num_classes]; the entry is skipped, never read out of bounds).

Semantics are the reference's lines with mmdet 2.20's GaussianFocalLoss, FocalLoss(use_sigmoid=True) (mmcv 1.4's
sigmoid_focal_loss CUDA op) and L1Loss, reduction "mean" (the C header has the formulas).  clip_sigmoid is torch's
CUDA sigmoid in fp32 followed by the clamp to [fp32(1e-4), fp32(1 - 1e-4)], so the clamp decisions and the zero
gradients are the reference's.  The avg factors -- max(count(t == 1), 1), fp32(sum mask + 1e-4), max(sum num_pos, 1)
-- are formed on the device instead of the reference's .item().  Sums are taken in double in a fixed order: the
results are reproducible bit for bit.  Deviations: the inputs are not modified (the reference's sigmoid_ is in place
and overwrites the head's heatmap); fp16 predictions are widened to fp32 as force_fp32 does and their gradients come
back in fp16.  A NaN regression target gives a NaN bbox loss even where its weight is 0, as in the reference (its
gradient there is 0: torch's sgn(NaN) is 0).  Loss configs other than the three types above raise ValueError; there
is no fallback.  GPU only: CPU tensors raise."""
import ctypes

import torch

from . import _C

__all__ = ["centerhead_loss", "transfusion_loss", "STATUS", "MAX_TASKS", "MAX_OBJS", "MAX_LAYERS"]

STATUS = {"bad_ind": 1, "bad_label": 2}   # BEVB200_LOSS_BAD_IND / _BAD_LABEL
MAX_TASKS = 16                            # BEVB200_LOSS_MAX_TASKS
MAX_OBJS = 4096                           # BEVB200_LOSS_MAX_OBJS
MAX_LAYERS = 15                           # BEVB200_LOSS_MAX_LAYERS

_CH_MAPS = ("reg", "height", "dim", "rot", "vel")
_TF_MAPS = ("center", "height", "dim", "rot", "vel")
_MAP_CH = (2, 1, 3, 2, 2)


def _cfg(cfg, kind, defaults):
    """(loss_weight, alpha, gamma) of a loss config dict of type `kind`; anything else raises ValueError."""
    if not isinstance(cfg, dict) or cfg.get("type") != kind:
        raise ValueError("expected a %s config, got %r" % (kind, cfg))
    allowed = {"type", "reduction", "loss_weight"} | set(defaults)
    if kind == "FocalLoss":
        allowed.add("use_sigmoid")
        if not cfg.get("use_sigmoid", True):
            raise ValueError("FocalLoss needs use_sigmoid=True (the softmax form is not implemented)")
    extra = set(cfg) - allowed
    if extra:
        raise ValueError("%s: unsupported arguments %s" % (kind, sorted(extra)))
    if cfg.get("reduction", "mean") != "mean":
        raise ValueError("%s: only reduction='mean' is supported (got %r)" % (kind, cfg.get("reduction")))
    return (float(cfg.get("loss_weight", 1.0)),) + tuple(float(cfg.get(k, v)) for k, v in defaults.items())


def _gaussian(cfg):
    return _cfg(cfg, "GaussianFocalLoss", {"alpha": 2.0, "gamma": 4.0})


def _focal(cfg):
    return _cfg(cfg, "FocalLoss", {"gamma": 2.0, "alpha": 0.25})


def _l1(cfg):
    return _cfg(cfg, "L1Loss", {})[0]


def _code_weights(train_cfg, code):
    cw = train_cfg.get("code_weights", None)
    if cw is None or len(cw) != code:
        raise ValueError("train_cfg['code_weights'] must have %d entries (got %r)" % (code, cw))
    return _C.host_array(ctypes.c_float, [float(v) for v in cw])


def _pred(t, name):
    """A prediction as force_fp32 hands it on: fp32 and contiguous (autograd carries the cast back)."""
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % name)
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: bevfusion_b200 has no CPU implementation" % name)
    if t.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise TypeError("%s must be floating point, got %s" % (name, t.dtype))
    return t.float().contiguous()


def _target(t, name, dtype, shape, dev):
    _C.require_cuda(t, name, dtype, contiguous=False)
    if tuple(t.shape) != tuple(shape):
        raise ValueError("%s must be %s, got %s" % (name, tuple(shape), tuple(t.shape)))
    if t.device != dev:
        raise ValueError("%s must be on the predictions' device %s" % (name, dev))
    return t.contiguous()


def _grad_buffers(tensors):
    return [torch.empty_like(t) for t in tensors]


# ---- CenterHead ---------------------------------------------------------------------------------------------
class _CenterHeadLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, meta, *tensors):
        T, nm = meta["T"], meta["nmaps"]
        preds, tg = tensors[:T * (1 + nm)], tensors[T * (1 + nm):]
        dev = preds[0].device
        heat = [preds[t * (1 + nm)] for t in range(T)]
        maps = [[preds[t * (1 + nm) + 1 + k] for t in range(T)] for k in range(nm)]
        targ = [[tg[4 * t + i] for t in range(T)] for i in range(4)]
        L = _C.lib()
        losses = torch.empty((2 * T,), dtype=torch.float32, device=dev)
        avg = torch.empty((2 * T,), dtype=torch.float32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        ws_bytes = int(L.bevb200_centerhead_loss_workspace_bytes(T, meta["B"], meta["cat"], meta["H"], meta["W"],
                                                                 meta["M"], meta["code"]))
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _C.check(L.bevb200_centerhead_loss(*_ch_args(meta, heat, maps, targ), _C.ptr(losses), _C.ptr(avg),
                                               _C.ptr(status), _C.ptr(ws), ws_bytes, _C.current_stream(dev)),
                     "centerhead_loss")
        ctx.meta = meta
        ctx.save_for_backward(*tensors, avg)
        ctx.mark_non_differentiable(status)
        return losses, status

    @staticmethod
    def backward(ctx, grad_losses, _grad_status):
        meta = ctx.meta
        T, nm = meta["T"], meta["nmaps"]
        saved = ctx.saved_tensors
        tensors, avg = saved[:-1], saved[-1]
        preds, tg = tensors[:T * (1 + nm)], tensors[T * (1 + nm):]
        heat = [preds[t * (1 + nm)] for t in range(T)]
        maps = [[preds[t * (1 + nm) + 1 + k] for t in range(T)] for k in range(nm)]
        targ = [[tg[4 * t + i] for t in range(T)] for i in range(4)]
        g_heat = _grad_buffers(heat)
        g_maps = [_grad_buffers(m) for m in maps]
        tables = [_C.host_array(ctypes.c_void_p, [g.data_ptr() for g in gs]) for gs in [g_heat] + g_maps]
        if nm == 4:
            tables.append(None)
        dev = avg.device
        grad_losses = grad_losses.float().contiguous()
        with torch.cuda.device(dev):
            _C.check(_C.lib().bevb200_centerhead_loss_backward(*_ch_args(meta, heat, maps, targ), _C.ptr(grad_losses),
                                                               _C.ptr(avg), *tables, _C.current_stream(dev)),
                     "centerhead_loss_backward")
        grads = []
        for t in range(T):
            grads.append(g_heat[t])
            grads.extend(g_maps[k][t] for k in range(nm))
        return (None,) + tuple(grads) + (None,) * len(tg)


def _ch_args(meta, heat, maps, targ):
    tab = lambda ts: _C.host_array(ctypes.c_void_p, [t.data_ptr() for t in ts])
    map_tabs = [tab(m) for m in maps] + ([None] if len(maps) == 4 else [])
    return ([tab(heat)] + map_tabs + [tab(targ[0]), tab(targ[1]), tab(targ[2]), tab(targ[3]), meta["cat"], meta["T"],
            meta["B"], meta["H"], meta["W"], meta["M"], meta["code"], meta["cw"], meta["alpha"], meta["gamma"],
            meta["lw_cls"], meta["lw_bbox"]])


def centerhead_loss(preds_dicts, targets, train_cfg, loss_cls=dict(type="GaussianFocalLoss", reduction="mean"),
                    loss_bbox=dict(type="L1Loss", reduction="mean", loss_weight=0.25), return_status=False):
    """CenterHead.loss on the device.  preds_dicts: the head's output, a list over tasks of one-element lists of
    dicts of maps (heatmap [B, cat_t, H, W] logits, reg [B, 2, H, W], height [B, 1, H, W], dim [B, 3, H, W],
    rot [B, 2, H, W] and, with 10-column targets, vel [B, 2, H, W]; fp32 or fp16 CUDA tensors).  targets: the
    4-tuple (heatmaps, anno_boxes, inds, masks) of head_targets.centerhead_targets(_batched): per task
    [B, cat_t, H, W] fp32, [B, M, 10 | 8] fp32, [B, M] int64, [B, M] uint8 (or bool).  train_cfg: code_weights (one
    per anno_box column).  loss_cls: GaussianFocalLoss (alpha, gamma, loss_weight); loss_bbox: L1Loss (loss_weight).
    Returns dict(heatmap/task{t}, bbox/task{t}) of 0-d fp32 tensors in the reference's order, without a host
    synchronisation; with return_status also the status word."""
    lw_cls, alpha, gamma = _gaussian(loss_cls)
    lw_bbox = _l1(loss_bbox)
    heatmaps, anno_boxes, inds, masks = targets
    T = len(preds_dicts)
    if not 1 <= T <= MAX_TASKS or not (len(heatmaps) == len(anno_boxes) == len(inds) == len(masks) == T):
        raise ValueError("preds_dicts and the four target lists need the same 1..%d tasks" % MAX_TASKS)
    code = anno_boxes[0].shape[-1] if anno_boxes[0].dim() == 3 else 0
    if code not in (8, 10):
        raise ValueError("anno_box must be [B, M, 10 | 8], got %s" % (tuple(anno_boxes[0].shape),))
    nm = 5 if code == 10 else 4
    tasks = [p[0] if isinstance(p, (list, tuple)) else p for p in preds_dicts]
    h0 = _pred(tasks[0]["heatmap"], "heatmap")
    if h0.dim() != 4:
        raise ValueError("heatmap must be [B, cat, H, W]")
    B, _, H, W = h0.shape
    M = anno_boxes[0].shape[1]
    if not 1 <= M <= MAX_OBJS:
        raise ValueError("max_objs must be in 1..%d (got %d)" % (MAX_OBJS, M))
    dev = h0.device
    preds, tg, cats = [], [], []
    for t, task in enumerate(tasks):
        h = _pred(task["heatmap"], "heatmap")
        if h.dim() != 4 or (h.shape[0], h.shape[2], h.shape[3]) != (B, H, W) or h.shape[1] < 1 or h.device != dev:
            raise ValueError("heatmap of task %d must be [%d, cat, %d, %d] on %s, got %s" % (t, B, H, W, dev,
                                                                                           tuple(h.shape)))
        cats.append(int(h.shape[1]))
        preds.append(h)
        for name, ch in zip(_CH_MAPS[:nm], _MAP_CH):
            if name not in task:
                raise ValueError("task %d has no '%s' map (needed for %d-column targets)" % (t, name, code))
            m = _pred(task[name], name)
            if tuple(m.shape) != (B, ch, H, W) or m.device != dev:
                raise ValueError("%s of task %d must be %s on %s, got %s" % (name, t, (B, ch, H, W), dev,
                                                                              tuple(m.shape)))
            preds.append(m)
        mask = masks[t]
        if isinstance(mask, torch.Tensor) and mask.dtype == torch.bool:
            mask = mask.view(torch.uint8)
        tg += [_target(heatmaps[t], "heatmaps[%d]" % t, torch.float32, h.shape, dev),
               _target(anno_boxes[t], "anno_boxes[%d]" % t, torch.float32, (B, M, code), dev),
               _target(inds[t], "inds[%d]" % t, torch.int64, (B, M), dev),
               _target(mask, "masks[%d]" % t, torch.uint8, (B, M), dev)]
    meta = dict(T=T, B=B, H=H, W=W, M=M, code=code, nmaps=nm, cat=_C.host_array(ctypes.c_int, cats),
                cw=_code_weights(train_cfg, code), alpha=alpha, gamma=gamma, lw_cls=lw_cls, lw_bbox=lw_bbox)
    losses, status = _CenterHeadLoss.apply(meta, *preds, *tg)
    vals = losses.unbind(0)
    out = {}
    for t in range(T):
        out["heatmap/task%d" % t] = vals[2 * t]
        out["bbox/task%d" % t] = vals[2 * t + 1]
    return (out, status) if return_status else out


# ---- TransFusion --------------------------------------------------------------------------------------------
class _TransFusionLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, meta, *tensors):
        preds, tg = tensors[:2 + meta["nmaps"]], tensors[2 + meta["nmaps"]:]
        dev = preds[0].device
        L = _C.lib()
        losses = torch.empty((2 + 2 * meta["Lt"],), dtype=torch.float32, device=dev)
        avg = torch.empty((2,), dtype=torch.float32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        ws_bytes = int(L.bevb200_transfusion_loss_workspace_bytes(*meta["sizes"]))
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        dense_t, labels, lw, bt, bw, num_pos, mean_iou = tg
        with torch.cuda.device(dev):
            _C.check(L.bevb200_transfusion_loss(
                *_tf_inputs(meta, preds, tg), _C.ptr(num_pos), num_pos.numel(), _C.ptr(mean_iou), mean_iou.numel(),
                *meta["sizes"], meta["cw"], meta["focal"], meta["lws"], _C.ptr(losses), _C.ptr(avg), _C.ptr(status),
                _C.ptr(ws), ws_bytes, _C.current_stream(dev)), "transfusion_loss")
        ctx.meta = meta
        ctx.save_for_backward(*tensors, avg)
        ctx.mark_non_differentiable(status)
        return losses, status

    @staticmethod
    def backward(ctx, grad_losses, _grad_status):
        meta = ctx.meta
        saved = ctx.saved_tensors
        tensors, avg = saved[:-1], saved[-1]
        preds, tg = tensors[:2 + meta["nmaps"]], tensors[2 + meta["nmaps"]:]
        grads = _grad_buffers(preds)
        dev = avg.device
        grad_losses = grad_losses.float().contiguous()
        gp = [_C.ptr(g) for g in grads] + ([0] if meta["nmaps"] == 4 else [])
        with torch.cuda.device(dev):
            _C.check(_C.lib().bevb200_transfusion_loss_backward(
                *_tf_inputs(meta, preds, tg), *meta["sizes"], meta["cw"], meta["focal"], meta["lws"],
                _C.ptr(grad_losses), _C.ptr(avg), *gp, _C.current_stream(dev)), "transfusion_loss_backward")
        return (None,) + tuple(grads) + (None,) * len(tg)


def _tf_inputs(meta, preds, tg):
    dense, heat = preds[0], preds[1]
    maps = [_C.ptr(m) for m in preds[2:]] + ([0] if meta["nmaps"] == 4 else [])
    dense_t, labels, lw, bt, bw = tg[:5]
    return [_C.ptr(dense), _C.ptr(dense_t), _C.ptr(heat)] + maps + [_C.ptr(labels), _C.ptr(lw), _C.ptr(bt),
                                                                   _C.ptr(bw)]


def _prefix(idx, num_decoder_layers, auxiliary):
    if idx == num_decoder_layers - 1 or (idx == 0 and auxiliary is False):
        return "layer_-1"
    return "layer_%d" % idx


def transfusion_loss(preds_dicts, targets, num_proposals, num_decoder_layers, auxiliary, train_cfg,
                     loss_cls=dict(type="FocalLoss", use_sigmoid=True, gamma=2.0, alpha=0.25, reduction="mean",
                                   loss_weight=1.0),
                     loss_bbox=dict(type="L1Loss", reduction="mean", loss_weight=0.25),
                     loss_heatmap=dict(type="GaussianFocalLoss", reduction="mean", loss_weight=1.0),
                     return_status=False):
    """TransFusionHead.loss on the device.  preds_dicts: the head's output (the reference's [[dict]] or the dict):
    dense_heatmap [B, K, H, W] and heatmap [B, K, N] logits, center [B, 2, N], height [B, 1, N], dim [B, 3, N],
    rot [B, 2, N] and, with code_size 10, vel [B, 2, N] (fp32 or fp16 CUDA).  targets: either the device 9-tuple
    transfusion_assign_batched(...) + (heatmap,) -- labels, label_weights, bbox_targets, bbox_weights, ious,
    num_pos int32 [B], mean_iou fp32 [B], status, heatmap -- which keeps the whole step free of host
    synchronisation, or the reference's 8-tuple of get_targets (num_pos an int, matched_ious a float).  The cls and
    bbox terms of layer idx < (num_decoder_layers if auxiliary else 1) use proposal columns idx * num_proposals ..
    (idx + 1) * num_proposals, with avg factor max(sum num_pos, 1).  train_cfg: code_weights.  Returns the
    reference's dict of 0-d fp32 tensors (matched_ious the mean of the per-sample mean ious) in its order; with
    return_status also the status word."""
    lw_heat, ah, gh = _gaussian(loss_heatmap)
    lw_cls, gc, ac = _focal(loss_cls)
    lw_bbox = _l1(loss_bbox)
    pd = preds_dicts
    while isinstance(pd, (list, tuple)):
        pd = pd[0]
    if len(targets) == 9:
        labels, label_weights, bbox_targets, bbox_weights, _, num_pos, mean_iou, _, heatmap = targets
    elif len(targets) == 8:
        labels, label_weights, bbox_targets, bbox_weights, _, num_pos, mean_iou, heatmap = targets
    else:
        raise ValueError("targets must be transfusion_assign_batched's 8 tensors + (heatmap,) or get_targets' "
                         "8-tuple")
    dense = _pred(pd["dense_heatmap"], "dense_heatmap")
    heat = _pred(pd["heatmap"], "heatmap")
    if dense.dim() != 4 or heat.dim() != 3 or heat.shape[:2] != dense.shape[:2]:
        raise ValueError("dense_heatmap must be [B, K, H, W] and heatmap [B, K, N], got %s and %s"
                         % (tuple(dense.shape), tuple(heat.shape)))
    B, K, H, W = dense.shape
    N = heat.shape[2]
    dev = dense.device
    code = bbox_targets.shape[-1] if bbox_targets.dim() == 3 else 0
    if code not in (8, 10):
        raise ValueError("bbox_targets must be [B, N, 10 | 8], got %s" % (tuple(bbox_targets.shape),))
    nm = 5 if code == 10 else 4
    P, Lt = int(num_proposals), int(num_decoder_layers) if auxiliary else 1
    if P < 1 or N % P or not 1 <= Lt <= N // P:
        raise ValueError("heatmap's %d columns must be whole layers of num_proposals %d covering the %d trained "
                         "layers" % (N, P, Lt))
    if Lt > MAX_LAYERS:
        raise ValueError("at most %d trained decoder layers (got %d)" % (MAX_LAYERS, Lt))
    preds = [dense, heat]
    for name, ch in zip(_TF_MAPS[:nm], _MAP_CH):
        if name not in pd:
            raise ValueError("preds_dict has no '%s' (needed for code_size %d)" % (name, code))
        m = _pred(pd[name], name)
        if tuple(m.shape) != (B, ch, N) or m.device != dev:
            raise ValueError("%s must be %s on %s, got %s" % (name, (B, ch, N), dev, tuple(m.shape)))
        preds.append(m)
    if not isinstance(num_pos, torch.Tensor):
        num_pos = torch.tensor([int(num_pos)], dtype=torch.int32).to(dev)
    if not isinstance(mean_iou, torch.Tensor):
        mean_iou = torch.tensor([float(mean_iou)], dtype=torch.float32).to(dev)
    _C.require_cuda(num_pos, "num_pos", torch.int32)
    _C.require_cuda(mean_iou, "mean_iou", torch.float32)
    if num_pos.dim() != 1 or mean_iou.dim() != 1 or num_pos.numel() < 1 or mean_iou.numel() < 1:
        raise ValueError("num_pos and mean_iou must be non-empty 1-d tensors")
    tg = [_target(heatmap, "heatmap", torch.float32, (B, K, H, W), dev),
          _target(labels, "labels", torch.int64, (B, N), dev),
          _target(label_weights, "label_weights", torch.int64, (B, N), dev),
          _target(bbox_targets, "bbox_targets", torch.float32, (B, N, code), dev),
          _target(bbox_weights, "bbox_weights", torch.float32, (B, N, code), dev), num_pos, mean_iou]
    meta = dict(nmaps=nm, Lt=Lt, sizes=(B, K, H, W, N, P, Lt, code), cw=_code_weights(train_cfg, code),
                focal=_C.host_array(ctypes.c_double, [ah, gh, ac, gc]),
                lws=_C.host_array(ctypes.c_double, [lw_heat, lw_cls, lw_bbox]))
    losses, status = _TransFusionLoss.apply(meta, *preds, *tg)
    vals = losses.unbind(0)
    out = {"loss_heatmap": vals[0]}
    for idx in range(Lt):
        prefix = _prefix(idx, int(num_decoder_layers), auxiliary)
        out["%s_loss_cls" % prefix] = vals[1 + 2 * idx]
        out["%s_loss_bbox" % prefix] = vals[2 + 2 * idx]
    out["matched_ious"] = vals[1 + 2 * Lt].detach()
    return (out, status) if return_status else out
