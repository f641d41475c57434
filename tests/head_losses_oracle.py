"""Float64 restatement of the CenterHead / TransFusion training losses (centerpoint.py:584-634, transfusion.py:587-713
with mmdet 2.20's GaussianFocalLoss, mmcv 1.4's sigmoid_focal_loss and mmdet's l1_loss) and of their gradients, in
numpy.  Every gradient is the closed form of d loss / d logit or d loss / d prediction for an upstream gradient of 1
on every loss.

clip_sigmoid is the fp32 sigmoid clamped to the fp32 bounds, as the reference computes it on CUDA: pass `y32` (the
device's torch.sigmoid of the logits) to take it from the device, else it is numpy's fp32 1 / (1 + exp(-x)).  The
focal loss and its gradient are then evaluated in float64 at that fp32 p (near p = 1, 1 - p carries the sigmoid's
fp32 rounding, up to 2e-4 relative, which a float64 sigmoid would not share).  With f64=True the sigmoid, the
decision and the bounds are float64's (1e-4, 1 - 1e-4), as the reference's lines run in float64 on the CPU make them.

centerhead(preds, targets, code_weights, cls=(lw, alpha, gamma), bbox_lw) -> (losses dict, grads list of dicts)
transfusion(preds, targets, P, L, auxiliary, code_weights, heat=(lw, a, g), cls=(lw, a, g), bbox_lw)
    -> (losses dict, grads dict)"""
import numpy as np

LO, HI = float(np.float32(1e-4)), float(np.float32(1 - 1e-4))
FLT_MIN = float(np.finfo(np.float32).tiny)
CH_MAPS = (("reg", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2))
TF_MAPS = (("center", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2))


def sigmoid32(x):
    x = np.asarray(x, np.float32)
    with np.errstate(over="ignore"):
        return np.float32(1) / (np.float32(1) + np.exp(-x))


def gaussian_focal(x, t, alpha=2.0, gamma=4.0, y32=None, f64=False):
    """(loss sum, count(t == 1), d sum / d x) of gaussian_focal_loss(clip_sigmoid(x), t)."""
    x = np.asarray(x, np.float64)
    t64 = np.asarray(t, np.float64)
    with np.errstate(over="ignore"):
        y = 1.0 / (1.0 + np.exp(-x))
    if f64:
        passing = (y >= 1e-4) & (y <= 1 - 1e-4)
        p = np.clip(y, 1e-4, 1 - 1e-4)
    else:
        y32 = sigmoid32(x) if y32 is None else np.asarray(y32, np.float32)
        passing = (y32 >= np.float32(LO)) & (y32 <= np.float32(HI))
        y = y32.astype(np.float64)
        p = np.clip(y, LO, HI)
    q, eps = 1.0 - p, 1e-12
    pos = np.asarray(t, np.float32) == np.float32(1)
    nw = (1.0 - t64) ** gamma
    loss = -np.log(q + eps) * p ** alpha * nw + np.where(pos, -np.log(p + eps) * q ** alpha, 0.0)
    d = nw * (p ** alpha / (q + eps) - alpha * p ** (alpha - 1) * np.log(q + eps))
    d = d + np.where(pos, -q ** alpha / (p + eps) + alpha * q ** (alpha - 1) * np.log(p + eps), 0.0)
    grad = np.where(passing, d * y * (1 - y), 0.0)
    return loss.sum(), float(pos.sum()), grad


def sigmoid_focal(x, labels, weights, alpha=0.25, gamma=2.0, f64=False):
    """mmcv's sigmoid_focal_loss of logits x [R, K] against labels [R] (K: background) times weights [R]:
    (loss sum, d sum / d x).  Rows with labels outside [0, K] are skipped, as the device does.  p is the fp32 sigmoid
    mmcv's CUDA kernel computes (0 at x = -100, where a float64 sigmoid is 4e-44), or float64's with f64=True."""
    x = np.asarray(x, np.float64)
    R, K = x.shape
    labels = np.asarray(labels)
    ok = (labels >= 0) & (labels <= K)
    flag = labels[:, None] == np.arange(K)[None, :]
    with np.errstate(over="ignore"):
        p = 1.0 / (1.0 + np.exp(-x)) if f64 else sigmoid32(x).astype(np.float64)
    lp, lq = np.log(np.maximum(p, FLT_MIN)), np.log(np.maximum(1 - p, FLT_MIN))
    wp, wn = alpha * (1 - p) ** gamma, (1 - alpha) * p ** gamma
    loss = np.where(flag, -wp * lp, -wn * lq)
    grad = np.where(flag, -wp * (1 - p - gamma * p * lp), -wn * (gamma * (1 - p) * lq - p))
    w = (np.asarray(weights, np.float64) * ok)[:, None]
    return (loss * w).sum(), grad * w


def l1(pred, target, w):
    """(sum |pred - target| w, d / d pred); NaN targets give a NaN sum and a 0 gradient (torch's sgn(NaN))."""
    d = np.asarray(pred, np.float64) - np.asarray(target, np.float64)
    with np.errstate(invalid="ignore"):
        return (np.abs(d) * w).sum(), np.where(np.isnan(d), 0.0, np.sign(d)) * w


def centerhead(preds, targets, code_weights, cls=(1.0, 2.0, 4.0), bbox_lw=0.25, y32=None, f64=False):
    """preds: list over tasks of dicts of numpy maps; targets: (heatmaps, anno_boxes, inds, masks) lists.  y32: an
    optional list over tasks of the device's fp32 sigmoid of the heatmap."""
    heatmaps, annos, inds, masks = targets
    losses, grads = {}, []
    for t, pr in enumerate(preds):
        code = annos[t].shape[-1]
        maps = CH_MAPS[:4 if code == 8 else 5]
        s, n, gh = gaussian_focal(pr["heatmap"], heatmaps[t], cls[1], cls[2], None if y32 is None else y32[t], f64)
        avg = max(n, 1.0)
        losses["heatmap/task%d" % t] = cls[0] * s / avg
        g = {"heatmap": cls[0] * gh / avg}
        B, _, H, W = pr["heatmap"].shape
        full = np.concatenate([pr[k].reshape(B, c, H * W) for k, c in maps], 1).astype(np.float64)   # [B, code, HW]
        ind, mask = inds[t].astype(np.int64), masks[t].astype(np.float32)
        pred = np.take_along_axis(full, np.broadcast_to(ind[:, None, :], (B, code, ind.shape[1])), 2)
        pred = pred.transpose(0, 2, 1)                                                            # [B, M, code]
        anno = annos[t].astype(np.float32)
        w = (mask[..., None] * (~np.isnan(anno))).astype(np.float32) * np.asarray(code_weights, np.float32)
        s, gp = l1(pred, anno, w.astype(np.float64))
        num = float(np.float32(np.float32(mask.sum()) + np.float32(1e-4)))
        losses["bbox/task%d" % t] = bbox_lw * s / num
        gfull = np.zeros_like(full)
        for b in range(B):   # sgn * w adds exactly, so cells whose duplicate slots cancel are exactly 0
            np.add.at(gfull[b].T, ind[b], gp[b])
        gfull *= bbox_lw / num
        off = 0
        for k, c in maps:
            g[k] = gfull[:, off:off + c].reshape(B, c, H, W)
            off += c
        grads.append(g)
    return losses, grads


def prefix(idx, L, auxiliary):
    return "layer_-1" if idx == L - 1 or (idx == 0 and auxiliary is False) else "layer_%d" % idx


def transfusion(preds, targets, P, L, auxiliary, code_weights, heat=(1.0, 2.0, 4.0), cls=(1.0, 0.25, 2.0),
                bbox_lw=0.25, y32=None, f64=False):
    """preds: dict of numpy arrays (dense_heatmap, heatmap, center, height, dim, rot[, vel]); targets: labels,
    label_weights, bbox_targets, bbox_weights, num_pos (sum), mean_ious (list), heatmap."""
    labels, lweights, bt, bw, num_pos, mean_ious, hm = targets
    code = bt.shape[-1]
    maps = TF_MAPS[:4 if code == 8 else 5]
    s, n, gd = gaussian_focal(preds["dense_heatmap"], hm, heat[1], heat[2], y32, f64)
    out = {"loss_heatmap": heat[0] * s / max(n, 1.0)}
    grads = {"dense_heatmap": heat[0] * gd / max(n, 1.0)}
    logits = preds["heatmap"].astype(np.float64)
    B, K, N = logits.shape
    grads["heatmap"] = np.zeros((B, K, N))
    for k, c in maps:
        grads[k] = np.zeros((B, c, N))
    avg = float(max(num_pos, 1))
    box = np.concatenate([preds[k] for k, _ in maps], 1).astype(np.float64)     # [B, code, N]
    for idx in range(L if auxiliary else 1):
        cols = slice(idx * P, (idx + 1) * P)
        pre = prefix(idx, L, auxiliary)
        x = logits[:, :, cols].transpose(0, 2, 1).reshape(-1, K)
        s, g = sigmoid_focal(x, labels[:, cols].reshape(-1), lweights[:, cols].reshape(-1), cls[1], cls[2], f64)
        out[pre + "_loss_cls"] = cls[0] * s / avg
        grads["heatmap"][:, :, cols] = (cls[0] * g / avg).reshape(B, P, K).transpose(0, 2, 1)
        w = (bw[:, cols].astype(np.float32) * np.asarray(code_weights, np.float32)).astype(np.float64)
        s, g = l1(box[:, :, cols].transpose(0, 2, 1), bt[:, cols], w)
        out[pre + "_loss_bbox"] = bbox_lw * s / avg
        g = (bbox_lw * g / avg).transpose(0, 2, 1)
        off = 0
        for k, c in maps:
            grads[k][:, :, cols] = g[:, off:off + c]
            off += c
    out["matched_ious"] = float(np.mean(mean_ious))
    return out, grads


def boundary_logits(sigmoid32_fn, n=4096):
    """fp32 logits around the clamp bounds: for each bound, the two consecutive fp32 logits on either side of the
    first whose fp32 sigmoid (sigmoid32_fn: numpy's or the device's) reaches the bound, and, where some logits hit
    the bound exactly, the last of them with its neighbours.  Returns (logits fp32 array, their sigmoids)."""
    sel = []
    for bound, guess in ((LO, np.log(LO / (1 - LO))), (HI, np.log(HI / (1 - HI)))):
        x = np.float32(guess)
        xs = [x]
        for _ in range(n // 2):
            xs.append(np.nextafter(xs[-1], np.float32(np.inf)))
        down = [x]
        for _ in range(n // 2):
            down.append(np.nextafter(down[-1], np.float32(-np.inf)))
        xs = np.array(down[::-1] + xs[1:], np.float32)
        ys = np.asarray(sigmoid32_fn(xs), np.float32)
        i = int(np.argmax(ys >= np.float32(bound)))
        pick = list(range(i - 2, i + 2))
        at = np.nonzero(ys == np.float32(bound))[0]
        if len(at):
            pick += [at[-1] - 1, at[-1], at[-1] + 1]
        sel.append(xs[sorted(set(pick))])
    xs = np.concatenate(sel)
    return xs, np.asarray(sigmoid32_fn(xs), np.float32)
