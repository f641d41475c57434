"""Restatements of TransFusionHead's query selection (transfusion.py:237-281 and :322-325) for the tests and the
benchmark.

    proposals(s, num_proposals, kernel_size, exempt)       numpy, from the sigmoid s [B, C, H, W] (numpy's exp is
                                                           not CUDA's, so the caller supplies s in x's dtype)
    torch_proposals(x, num_proposals, kernel_size, dataset, stable=True)
                                                           the reference's lines on torch tensors of any device,
                                                           with argsort(stable=stable)

Both return (labels [B, K] int64, index [B, K] int64, query_heatmap_score [B, C, K] in x's dtype).  Order: descending
masked value with NaN first, ties by ascending flat index (argsort(descending=True, stable=True))."""
import numpy as np
import torch
import torch.nn.functional as F

EXEMPT = {"nuScenes": (8, 9), "Waymo": (1, 2)}


def masked_plane(s, kernel_size, exempt):
    """m = s * (s == local_max) of the reference, in s's dtype (NaN propagates through the window maximum)."""
    B, C, H, W = s.shape
    p = kernel_size // 2
    local_max = np.zeros_like(s)
    win = np.lib.stride_tricks.sliding_window_view(s, (kernel_size, kernel_size), axis=(2, 3))
    local_max[:, :, p:H - p, p:W - p] = win.max(axis=(-2, -1))
    for c in exempt:
        local_max[:, c] = s[:, c]
    with np.errstate(invalid="ignore"):
        return s * (s == local_max).astype(s.dtype)


def proposals(s, num_proposals, kernel_size, exempt):
    B, C, H, W = s.shape
    m = masked_plane(s, kernel_size, exempt)
    flat = m.reshape(B, -1)
    idx = np.arange(flat.shape[1])
    top = np.empty((B, num_proposals), np.int64)
    for b in range(B):
        v = flat[b].astype(np.float64)
        nan = np.isnan(v)
        order = np.lexsort((idx, -np.where(nan, 0.0, v), ~nan))   # NaN first, value descending, index ascending
        top[b] = order[:num_proposals]
    labels, index = top // (H * W), top % (H * W)
    score = np.take_along_axis(m.reshape(B, C, H * W), np.broadcast_to(index[:, None, :], (B, C, num_proposals)),
                               axis=2)
    return labels, index, score


def torch_proposals(x, num_proposals, kernel_size, dataset, stable=True):
    """transfusion.py:238-274 and :322-325 on `x` (the dense heatmap), argsort(descending=True, stable=stable)."""
    batch_size = x.shape[0]
    heatmap = x.detach().sigmoid()
    padding = kernel_size // 2
    local_max = torch.zeros_like(heatmap)
    local_max_inner = F.max_pool2d(heatmap, kernel_size=kernel_size, stride=1, padding=0)
    local_max[:, :, padding:(-padding), padding:(-padding)] = local_max_inner
    for c in EXEMPT.get(dataset, ()):
        local_max[:, c] = F.max_pool2d(heatmap[:, c], kernel_size=1, stride=1, padding=0)
    heatmap = heatmap * (heatmap == local_max)
    heatmap = heatmap.view(batch_size, heatmap.shape[1], -1)
    top = heatmap.view(batch_size, -1).argsort(dim=-1, descending=True, stable=stable)[..., :num_proposals]
    labels = top // heatmap.shape[-1]
    index = top % heatmap.shape[-1]
    score = heatmap.gather(index=index[:, None, :].expand(-1, heatmap.shape[1], -1), dim=-1)
    return labels, index, score
