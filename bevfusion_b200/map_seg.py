"""map_seg -- the BEV map segmentation head (BEVSegmentationHead, models/heads/segm/vanilla.py) and the IoU counts of
NuScenesDataset.evaluate_map (datasets/nuscenes_dataset.py:498-530) on the device (csrc/map_seg.cu).

    BEVGridTransform(input_scope=..., output_scope=..., prescale_factor=1)
        the reference's module: bilinear prescale (align_corners=False, torch's scale_factor source index) and
        bilinear grid_sample (zeros padding, align_corners=False) as one separable gather; backward is the gather form
        of the transposed operator, with no atomics, so gradients are reproducible bit for bit (torch's CUDA
        upsample and grid_sample backwards use atomicAdd and raise under torch.use_deterministic_algorithms)
    map_seg_loss(logits, target, loss, classes) -> {f"{name}/{loss}": 0-d fp32}   (focal or xent, mean)
    map_seg_counts(pred, gt, thresholds, out=None) -> int64 [3, K, T] tp / fp / fn, added into `out`
    map_seg_metrics(counts, classes, thresholds) -> evaluate_map's dict
    BEVSegmentationHead(in_channels, grid_transform, classes, loss)   drop-in, same state_dict names

The grid's per-axis tap tables are built once per (module, input size, device) on the host, in float32 with the
reference's op order, and uploaded once; a call then makes no host-to-device copy and no synchronisation and can be
captured in a CUDA graph.  Deliberate deviation: the counts are exact int64 where the reference adds them into
float32 tensors, which round once a count passes 2^24.  GPU only: CPU tensors raise."""
import ctypes
import math

import numpy as np
import torch
from torch import nn

from . import _C

__all__ = ["BEVGridTransform", "BEVSegmentationHead", "map_seg_loss", "map_seg_counts", "map_seg_metrics",
           "axis_coords", "axis_taps", "transpose_taps", "THRESHOLDS", "MAX_THRESHOLDS"]

THRESHOLDS = (0.35, 0.4, 0.45, 0.5, 0.55, 0.6, 0.65)   # evaluate_map's
MAX_THRESHOLDS = 16                                    # BEVB200_MAP_MAX_THRESHOLDS
_TARGET_TYPES = {torch.float32: 0, torch.uint8: 1, torch.bool: 1, torch.int64: 2}   # BEVB200_MAP_TARGET_*
_SMEM_LIMIT = 48 * 1024
_F = np.float32


# ---- tap tables (host) --------------------------------------------------------------------------------------------
def axis_coords(in_scope, out_scope):
    """The reference's normalised fp32 grid coordinates of one axis (BEVGridTransform.forward), computed the way it
    computes them: torch.arange and the normalisation in fp32 on the CPU."""
    imin, imax = in_scope[0], in_scope[1]
    omin, omax, ostep = out_scope
    if not ostep > 0 or not imax > imin:
        raise ValueError("scopes need imax > imin and a positive output step, got %r and %r" % (in_scope, out_scope))
    if omin + ostep / 2 >= omax:
        return np.zeros((0,), np.float32)
    v = torch.arange(omin + ostep / 2, omax, ostep)
    v = (v - imin) / (imax - imin) * 2 - 1
    return v.to(torch.float32).numpy()


def _prescale_taps(size, p):
    """torch's upsample_bilinear2d (align_corners=False, scale_factor p) along one axis: output size floor(size * p)
    and, per output index, ((i0, l0), (i1, l1)) in fp32."""
    out = int(math.floor(float(size) * p))
    rscale = _F(1.0 / p)
    taps = []
    for d in range(out):
        src = _F(rscale * _F(_F(d) + _F(0.5)))
        src = _F(src - _F(0.5))
        if src < 0:
            src = _F(0.0)
        i0 = int(src)
        i1 = i0 + (1 if i0 < size - 1 else 0)
        l1 = _F(src - _F(i0))
        l0 = _F(_F(1.0) - l1)
        taps.append(((i0, l0), (i1, l1)))
    return out, taps


def axis_taps(coords, size, prescale_factor=1):
    """Composite taps of one axis: for each output index the sorted list of (input index, fp32 weight), <= 4 entries;
    taps outside the (prescaled) input are dropped -- grid_sample's zeros padding.  `coords` are the normalised fp32
    grid coordinates, `size` the input length before the prescale."""
    p = prescale_factor
    if p != 1:
        psize, pre = _prescale_taps(size, p)
    else:
        psize, pre = size, None
    fsize = _F(psize)
    rows = []
    for c in np.asarray(coords, np.float32):
        ix = _F(_F(_F(c + _F(1.0)) * fsize) - _F(1.0))
        ix = _F(ix / _F(2.0))
        j0 = int(math.floor(ix))
        w1 = _F(ix - _F(j0))
        w0 = _F(_F(j0 + 1) - ix)
        acc = {}
        for j, w in ((j0, w0), (j0 + 1, w1)):
            if not 0 <= j < psize:
                continue
            if pre is None:
                acc[j] = _F(acc.get(j, _F(0.0)) + w)
            else:
                for i, lam in pre[j]:
                    acc[i] = _F(acc.get(i, _F(0.0)) + _F(w * lam))
        rows.append(sorted(acc.items()))
    return rows


def transpose_taps(rows, size):
    """For each input index 0..size-1 its (output index, weight) list in ascending output order."""
    cols = [[] for _ in range(size)]
    for o, taps in enumerate(rows):
        for i, w in taps:
            cols[i].append((o, w))
    return cols


def _csr(lists):
    ptr = np.zeros(len(lists) + 1, np.int32)
    ptr[1:] = np.cumsum([len(t) for t in lists])
    idx = np.array([i for t in lists for i, _ in t], np.int32)
    w = np.array([w for t in lists for _, w in t], np.float32)
    return ptr, idx, w


def _blocks(rows, R):
    """(first source row, number of source rows) of every block of R destination rows."""
    lo, cnt = [], []
    for b in range(0, len(rows), R):
        ids = [i for t in rows[b:b + R] for i, _ in t]
        lo.append(min(ids) if ids else 0)
        cnt.append(max(ids) - min(ids) + 1 if ids else 0)
    return np.array(lo, np.int32), np.array(cnt, np.int32)


class _Direction:
    """One direction of the transform as device CSR tables: dst [Hd, Wd] from src [Hs, Ws]."""

    def __init__(self, row_lists, col_lists, Hs, Ws, ints, floats):
        self.Hs, self.Ws, self.Hd, self.Wd = Hs, Ws, len(row_lists), len(col_lists)
        rp, ri, rw = _csr(row_lists)
        cp, ci, cw = _csr(col_lists)
        self.col_nnz = len(ci)
        L = _C.lib()
        for R in (16, 8, 4, 2, 1):
            lo, cnt = _blocks(row_lists, R)
            n_max = int(cnt.max()) if len(cnt) else 0
            if L.bevb200_map_grid_smem_bytes(Ws, self.Wd, self.col_nnz, n_max) <= _SMEM_LIMIT:
                break
        else:
            raise ValueError("grid transform of a %d x %d map to %d x %d needs more than %d bytes of shared memory"
                             % (Hs, Ws, self.Hd, self.Wd, _SMEM_LIMIT))
        self.R, self.n_max = R, n_max
        self._slots = {}
        for name, a in (("rp", rp), ("ri", ri), ("cp", cp), ("ci", ci), ("lo", lo), ("cnt", cnt)):
            self._slots[name] = ("i", len(ints), len(a))
            ints.append(a)
        for name, a in (("rw", rw), ("cw", cw)):
            self._slots[name] = ("f", len(floats), len(a))
            floats.append(a)

    def bind(self, ints, floats):
        """Device views of this direction's tables inside the uploaded int32 / fp32 buffers."""
        offs = {"i": np.cumsum([0] + [len(a) for a in ints[0]]), "f": np.cumsum([0] + [len(a) for a in floats[0]])}
        self.dev = {}
        for name, (kind, k, n) in self._slots.items():
            buf = ints[1] if kind == "i" else floats[1]
            o = int(offs[kind][k])
            self.dev[name] = buf[o:o + max(n, 1)]

    def run(self, src, dst, planes):
        d = self.dev
        with torch.cuda.device(src.device):
            _C.check(_C.lib().bevb200_map_grid_transform(
                _C.ptr(src), _C.ptr(dst), int(src.dtype == torch.float16), planes, self.Hs, self.Ws, self.Hd, self.Wd,
                _C.ptr(d["rp"]), _C.ptr(d["ri"]), _C.ptr(d["rw"]), _C.ptr(d["cp"]), _C.ptr(d["ci"]), _C.ptr(d["cw"]),
                self.col_nnz, _C.ptr(d["lo"]), _C.ptr(d["cnt"]), self.R, self.n_max,
                _C.current_stream(src.device)), "map_grid_transform")


def _upload(arrays, dtype, dev):
    a = np.concatenate([np.asarray(x, dtype) for x in arrays] + [np.zeros(1, dtype)])
    host = torch.from_numpy(a).pin_memory()
    return host, host.to(dev, non_blocking=True)   # the pinned copy is kept alive with the plan


class _GridPlan:
    """Forward and backward tables of one (scopes, prescale, input size) on one device."""

    def __init__(self, input_scope, output_scope, prescale_factor, H, W, dev):
        ry = axis_taps(axis_coords(input_scope[0], output_scope[0]), H, prescale_factor)
        rx = axis_taps(axis_coords(input_scope[1], output_scope[1]), W, prescale_factor)
        if not ry or not rx:
            raise ValueError("output_scope %r gives an empty output" % (output_scope,))
        self.H, self.W, self.Ho, self.Wo = H, W, len(ry), len(rx)
        ints, floats = [], []
        self.fwd = _Direction(ry, rx, H, W, ints, floats)
        self.bwd = _Direction(transpose_taps(ry, H), transpose_taps(rx, W), self.Ho, self.Wo, ints, floats)
        self._host_i, dev_i = _upload(ints, np.int32, dev)
        self._host_f, dev_f = _upload(floats, np.float32, dev)
        self.fwd.bind((ints, dev_i), (floats, dev_f))
        self.bwd.bind((ints, dev_i), (floats, dev_f))


class _GridTransformFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, plan):
        B, C = x.shape[:2]
        out = torch.empty((B, C, plan.Ho, plan.Wo), dtype=x.dtype, device=x.device)
        plan.fwd.run(x, out, B * C)
        ctx.plan = plan
        ctx.dtype = x.dtype
        return out

    @staticmethod
    def backward(ctx, g):
        plan = ctx.plan
        g = g.to(ctx.dtype).contiguous()
        B, C = g.shape[:2]
        gi = torch.empty((B, C, plan.H, plan.W), dtype=g.dtype, device=g.device)
        plan.bwd.run(g, gi, B * C)
        return gi, None


def _check_scope(scope, name):
    if len(scope) != 2 or any(len(s) != 3 for s in scope):
        raise ValueError("%s must be two (min, max, step) triples, got %r" % (name, scope))


class BEVGridTransform(nn.Module):
    """The reference's BEVGridTransform: input_scope / output_scope [(min, max, step)] * 2, index 0 the rows (H) and
    1 the columns (W); prescale_factor the bilinear pre-upsampling.  x: [B, C, H, W] fp32 or fp16 CUDA tensor."""

    def __init__(self, *, input_scope, output_scope, prescale_factor=1):
        super().__init__()
        _check_scope(input_scope, "input_scope")
        _check_scope(output_scope, "output_scope")
        if not prescale_factor > 0:
            raise ValueError("prescale_factor must be > 0, got %r" % (prescale_factor,))
        self.input_scope = input_scope
        self.output_scope = output_scope
        self.prescale_factor = prescale_factor
        self._plans = {}

    def plan(self, H, W, device):
        key = (int(H), int(W), torch.device(device))
        p = self._plans.get(key)
        if p is None:
            p = _GridPlan(self.input_scope, self.output_scope, self.prescale_factor, int(H), int(W), key[2])
            self._plans[key] = p
        return p

    def forward(self, x):
        _C.require_cuda(x, "x", contiguous=False)
        if x.dtype not in (torch.float32, torch.float16):
            raise TypeError("x must be fp32 or fp16, got %s" % x.dtype)
        if x.dim() != 4 or x.numel() == 0:
            raise ValueError("x must be a non-empty [B, C, H, W] map, got %s" % (tuple(x.shape),))
        plan = self.plan(x.shape[2], x.shape[3], x.device)
        return _GridTransformFn.apply(x.contiguous(), plan)


# ---- losses -------------------------------------------------------------------------------------------------------
def _map_pair(a, b, an, bn):
    _C.require_cuda(a, an, contiguous=False)
    _C.require_cuda(b, bn, contiguous=False)
    if a.dim() != 4 or tuple(a.shape) != tuple(b.shape) or a.numel() == 0:
        raise ValueError("%s and %s must be the same non-empty [B, K, H, W], got %s and %s"
                         % (an, bn, tuple(a.shape), tuple(b.shape)))
    if a.device != b.device:
        raise ValueError("%s must be on %s's device %s" % (bn, an, a.device))
    if a.dtype not in (torch.float32, torch.float16):
        raise TypeError("%s must be fp32 or fp16, got %s" % (an, a.dtype))
    if b.dtype not in _TARGET_TYPES:
        raise TypeError("%s must be int64, uint8, bool or fp32, got %s" % (bn, b.dtype))
    b = b.contiguous()
    return a.contiguous(), (b.view(torch.uint8) if b.dtype == torch.bool else b)


class _SegLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, focal):
        B, K, H, W = logits.shape
        dev = logits.device
        L = _C.lib()
        losses = torch.empty((K,), dtype=torch.float32, device=dev)
        ws_bytes = int(L.bevb200_map_seg_loss_workspace_bytes(B, K, H, W))
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _C.check(L.bevb200_map_seg_loss(_C.ptr(logits), int(logits.dtype == torch.float16), _C.ptr(target),
                                            _TARGET_TYPES[target.dtype], B, K, H, W, int(focal), _C.ptr(losses),
                                            _C.ptr(ws), ws_bytes, _C.current_stream(dev)), "map_seg_loss")
        ctx.save_for_backward(logits, target)
        ctx.focal = focal
        return losses

    @staticmethod
    def backward(ctx, grad_losses):
        logits, target = ctx.saved_tensors
        B, K, H, W = logits.shape
        dev = logits.device
        grad_losses = grad_losses.float().contiguous()
        g = torch.empty_like(logits)
        with torch.cuda.device(dev):
            _C.check(_C.lib().bevb200_map_seg_loss_backward(
                _C.ptr(logits), int(logits.dtype == torch.float16), _C.ptr(target), _TARGET_TYPES[target.dtype], B, K,
                H, W, int(ctx.focal), _C.ptr(grad_losses), _C.ptr(g), _C.current_stream(dev)), "map_seg_loss_backward")
        return g, None, None


def map_seg_loss(logits, target, loss, classes, reduction="mean"):
    """BEVSegmentationHead's training losses: for each class k, sigmoid_focal_loss (alpha=-1, gamma=2) or
    sigmoid_xent_loss of logits[:, k] against target[:, k], mean over B * H * W.  logits [B, K, H, W] fp32 or fp16
    (widened to fp32; the gradient comes back in the logits' dtype); target [B, K, H, W] int64, uint8, bool or fp32.
    Returns {f"{name}/{loss}": 0-d fp32} in class order, with no host synchronisation."""
    if loss not in ("focal", "xent"):
        raise ValueError("unsupported loss: %r" % (loss,))
    if reduction != "mean":
        raise ValueError("only reduction='mean' is supported, got %r" % (reduction,))
    logits, target = _map_pair(logits, target, "logits", "target")
    if len(classes) != logits.shape[1]:
        raise ValueError("%d classes for %d logit channels" % (len(classes), logits.shape[1]))
    vals = _SegLossFn.apply(logits, target, loss == "focal").unbind(0)
    return {"%s/%s" % (name, loss): v for name, v in zip(classes, vals)}


# ---- evaluation -----------------------------------------------------------------------------------------------------
def map_seg_counts(pred, gt, thresholds=THRESHOLDS, out=None):
    """evaluate_map's counts on the device: label = gt != 0, predicted = pred >= fp32 threshold (NaN: negative).
    pred [B, K, H, W] or one sample's [K, H, W], fp32 or fp16; gt the same shape, int64, uint8, bool or fp32.  ADDS
    tp, fp, fn into `out` (int64 [3, K, T] on pred's device; zeros if None) and returns it.  One launch, exact."""
    if isinstance(pred, torch.Tensor) and pred.dim() == 3:
        pred = pred.unsqueeze(0)
    if isinstance(gt, torch.Tensor) and gt.dim() == 3:
        gt = gt.unsqueeze(0)
    pred, gt = _map_pair(pred, gt, "pred", "gt")
    T = len(thresholds)
    if not 1 <= T <= MAX_THRESHOLDS:
        raise ValueError("1..%d thresholds, got %d" % (MAX_THRESHOLDS, T))
    B, K, H, W = pred.shape
    if out is None:
        out = torch.zeros((3, K, T), dtype=torch.int64, device=pred.device)
    _C.require_cuda(out, "out", torch.int64)
    if tuple(out.shape) != (3, K, T) or out.device != pred.device:
        raise ValueError("out must be int64 [3, %d, %d] on %s" % (K, T, pred.device))
    thr = _C.host_array(ctypes.c_float, [float(t) for t in thresholds])
    with torch.cuda.device(pred.device):
        _C.check(_C.lib().bevb200_map_seg_counts(_C.ptr(pred), int(pred.dtype == torch.float16), _C.ptr(gt),
                                                 _TARGET_TYPES[gt.dtype], B, K, H, W, thr, T, _C.ptr(out),
                                                 _C.current_stream(pred.device)), "map_seg_counts")
    return out


def map_seg_metrics(counts, classes, thresholds=THRESHOLDS):
    """evaluate_map's metric dict -- map/{name}/iou@max, map/{name}/iou@{t:.2f}, map/mean/iou@max -- from exact
    counts [3, K, T] (one device-to-host copy).  iou = tp / (tp + fp + fn + 1e-7) in float64."""
    c = counts.detach().cpu().numpy().astype(np.int64) if isinstance(counts, torch.Tensor) else np.asarray(counts)
    if c.shape != (3, len(classes), len(thresholds)):
        raise ValueError("counts must be [3, %d, %d], got %s" % (len(classes), len(thresholds), c.shape))
    tp, fp, fn = (c[i].astype(np.float64) for i in range(3))
    ious = tp / (tp + fp + fn + 1e-7)
    metrics = {}
    for k, name in enumerate(classes):
        metrics["map/%s/iou@max" % name] = float(ious[k].max())
        for t, iou in zip(thresholds, ious[k]):
            metrics["map/%s/iou@%.2f" % (name, float(np.float32(t)))] = float(iou)
    metrics["map/mean/iou@max"] = float(ious.max(axis=1).mean())
    return metrics


# ---- head -----------------------------------------------------------------------------------------------------------
class BEVSegmentationHead(nn.Module):
    """Drop-in BEVSegmentationHead: the reference's constructor, attribute and state_dict names (transform,
    classifier.0 .. classifier.6).  The classifier is plain torch; the transform and the losses are native.
    Training: forward(x, target) returns the loss dict; eval: torch.sigmoid of the logits."""

    def __init__(self, in_channels, grid_transform, classes, loss):
        super().__init__()
        self.in_channels = in_channels
        self.classes = classes
        self.loss = loss
        self.transform = BEVGridTransform(**grid_transform)
        self.classifier = nn.Sequential(
            nn.Conv2d(in_channels, in_channels, 3, padding=1, bias=False),
            nn.BatchNorm2d(in_channels),
            nn.ReLU(True),
            nn.Conv2d(in_channels, in_channels, 3, padding=1, bias=False),
            nn.BatchNorm2d(in_channels),
            nn.ReLU(True),
            nn.Conv2d(in_channels, len(classes), 1),
        )

    def forward(self, x, target=None):
        if isinstance(x, (list, tuple)):
            x = x[0]
        x = self.transform(x)
        x = self.classifier(x)
        if self.training:
            return map_seg_loss(x, target, self.loss, self.classes)
        return torch.sigmoid(x)
