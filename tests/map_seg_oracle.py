"""Float64 numpy restatement of BEVSegmentationHead's pieces (models/heads/segm/vanilla.py) and of evaluate_map's
counts (datasets/nuscenes_dataset.py:498-530).

The grid transform is written as dense per-axis matrices A_y [Ho, H] and A_x [Wo, W], out = A_y x A_x^T, whose
entries are float64 bilinear weights evaluated at the reference's fp32 sample coordinates: the fp32 normalised grid
(torch.arange and the normalisation in fp32), grid_sample's fp32 unnormalisation ((g + 1) * size - 1) / 2 and
upsample_bilinear2d's fp32 source index max(fp32(1 / p) * (d + 0.5) - 0.5, 0).  The backward is the transpose,
A_y^T g A_x."""
import math

import numpy as np

F32 = np.float32


def grid_coords(in_scope, out_scope):
    """Normalised fp32 grid coordinates of one axis: fp32(omin + ostep / 2 + i * ostep) for the reference's arange
    length, then (v - imin) / (imax - imin) * 2 - 1 in fp32."""
    imin, imax = in_scope[0], in_scope[1]
    omin, omax, ostep = out_scope
    start = omin + ostep / 2
    n = max(int(math.ceil((omax - start) / ostep)), 0)
    v = np.array([start + i * ostep for i in range(n)], np.float64).astype(F32)
    return ((v - F32(imin)) / F32(imax - imin) * F32(2) - F32(1)).astype(F32)


def prescale_matrix(size, p):
    """upsample_bilinear2d (align_corners=False, scale_factor p) along one axis: [floor(size p), size]."""
    out = int(math.floor(float(size) * p))
    A = np.zeros((out, size))
    r = F32(1.0 / p)
    for d in range(out):
        src = max(float(F32(F32(r * F32(d + 0.5)) - F32(0.5))), 0.0)
        i0 = int(src)
        i1 = min(i0 + 1, size - 1)
        lam = src - i0
        A[d, i0] += 1.0 - lam
        A[d, i1] += lam
    return A


def sample_matrix(coords, size):
    """grid_sample (bilinear, zeros, align_corners=False) along one axis: [len(coords), size]."""
    A = np.zeros((len(coords), size))
    for o, g in enumerate(np.asarray(coords, F32)):
        ix = float(F32(F32(F32(F32(g + F32(1)) * F32(size)) - F32(1)) / F32(2)))
        j0 = math.floor(ix)
        for j, w in ((j0, j0 + 1 - ix), (j0 + 1, ix - j0)):
            if 0 <= j < size:
                A[o, j] += w
    return A


def axis_matrix(in_scope, out_scope, size, p=1):
    c = grid_coords(in_scope, out_scope)
    if p == 1:
        return sample_matrix(c, size)
    P = prescale_matrix(size, p)
    return sample_matrix(c, P.shape[0]) @ P


def transform_matrices(input_scope, output_scope, H, W, p=1):
    return (axis_matrix(input_scope[0], output_scope[0], H, p), axis_matrix(input_scope[1], output_scope[1], W, p))


def grid_forward(x, Ay, Ax):
    return np.einsum("ih,bchw,jw->bcij", Ay, np.asarray(x, np.float64), Ax)


def grid_backward(g, Ay, Ax):
    return np.einsum("ih,bcij,jw->bchw", Ay, np.asarray(g, np.float64), Ax)


def _softplus_neg(x):
    """log(1 + exp(-x))"""
    return np.where(x > 0, np.log1p(np.exp(-np.abs(x))), -x + np.log1p(np.exp(-np.abs(x))))


def elementwise(x, t, loss):
    """(loss, d loss / d x) per element in float64: binary_cross_entropy_with_logits, or sigmoid_focal_loss with
    alpha = -1, gamma = 2."""
    x = np.asarray(x, np.float64)
    t = np.asarray(t, np.float64)
    p = 1.0 / (1.0 + np.exp(-x))
    q = 1.0 / (1.0 + np.exp(x))
    ce = (1.0 - t) * x + _softplus_neg(x)
    dce = (1.0 - t) * p - t * q
    if loss == "xent":
        return ce, dce
    m = t * q + (1.0 - t) * p
    return ce * m * m, dce * m * m + ce * 2.0 * m * (1.0 - 2.0 * t) * p * q


def losses(x, t, loss):
    """Per-class means [K]."""
    el, _ = elementwise(x, t, loss)
    return el.mean(axis=(0, 2, 3))


def loss_grad(x, t, loss, grad=None):
    """Gradient of sum_k grad[k] * loss_k (grad defaults to ones) with respect to the logits."""
    x = np.asarray(x, np.float64)
    B, K, H, W = x.shape
    _, d = elementwise(x, t, loss)
    g = np.ones(K) if grad is None else np.asarray(grad, np.float64)
    return d * g[None, :, None, None] / (B * H * W)


def counts(pred, gt, thresholds):
    """tp, fp, fn int64 [3, K, T] of pred >= fp32 threshold against gt != 0, summed over the batch."""
    pred = np.asarray(pred, np.float32)
    if pred.ndim == 3:
        pred, gt = pred[None], np.asarray(gt)[None]
    B, K = pred.shape[:2]
    p = pred.transpose(1, 0, 2, 3).reshape(K, -1)[:, :, None] >= np.asarray(thresholds, np.float32)[None, None]
    lab = (np.asarray(gt).transpose(1, 0, 2, 3).reshape(K, -1) != 0)[:, :, None]
    return np.stack([(p & lab).sum(1), (p & ~lab).sum(1), (~p & lab).sum(1)]).astype(np.int64)
