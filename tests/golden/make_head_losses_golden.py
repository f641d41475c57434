"""Generates tests/golden/head_losses_tiny.npz from the REFERENCE's own loss code, run in float64 on the CPU.

CenterHead.loss (centerpoint.py:584-634) with its _gather_feat and clip_sigmoid, and TransFusionHead.loss
(transfusion.py:587-713) with its clip_sigmoid, are extracted from the reference files and executed on a stand-in
`self` whose get_targets returns fixed targets.  mmcv and mmdet are not installed, so force_fp32 is a pass-through
decorator and the three loss classes are restated in torch from mmdet 2.20 / mmcv 1.4:
  GaussianFocalLoss  mmdet/models/losses/gaussian_focal_loss.py (alpha 2, gamma 4, eps 1e-12)
  FocalLoss          use_sigmoid=True on CUDA tensors: mmcv's sigmoid_focal_loss op, whose forward and backward
                     formulas are restated here as an autograd.Function (label K is the background; the row weight
                     multiplies the elementwise loss; sum / avg_factor)
  L1Loss             mmdet/models/losses/smooth_l1_loss.py l1_loss, weighted, sum / avg_factor
The reference's sigmoid_ is in place, so the heatmaps it receives are non-leaf copies of the leaves whose gradients
are recorded.  Cases: 2 samples, 6 tasks at 16 x 16 with duplicate inds, masked slots, exact-1 targets and saturated
logits (loss weights 1.0 / 0.25 and 1.5 / 0.4); TransFusion with 2 decoder layers, auxiliary on and off, code 10.

Run:  python tests/golden/make_head_losses_golden.py      (needs the reference tree)"""
import ast
import os

import numpy as np
import torch

REF = os.environ.get("BEVFUSION_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "head_losses_tiny.npz")
FLT_MIN = float(np.finfo(np.float32).tiny)


def force_fp32(apply_to=None, out_fp16=False):
    return lambda fn: fn


def _weight_reduce(loss, weight, avg_factor):
    if weight is not None:
        loss = loss * weight
    return loss.sum() / avg_factor


class GaussianFocalLoss:
    def __init__(self, alpha=2.0, gamma=4.0, reduction="mean", loss_weight=1.0):
        self.alpha, self.gamma, self.loss_weight = alpha, gamma, loss_weight

    def __call__(self, pred, target, weight=None, avg_factor=None):
        eps = 1e-12
        pos_weights = target.eq(1)
        neg_weights = (1 - target).pow(self.gamma)
        pos_loss = -(pred + eps).log() * (1 - pred).pow(self.alpha) * pos_weights
        neg_loss = -(1 - pred + eps).log() * pred.pow(self.alpha) * neg_weights
        return self.loss_weight * _weight_reduce(pos_loss + neg_loss, weight, avg_factor)


class _SigmoidFocal(torch.autograd.Function):
    """mmcv 1.4 sigmoid_focal_loss_cuda_kernel.cuh, forward and backward, no weight (reduction 'none')."""

    @staticmethod
    def forward(ctx, x, target, gamma, alpha):
        K = x.shape[1]
        flag = (target[:, None] == torch.arange(K, device=x.device)[None, :]).to(x.dtype)
        p = 1.0 / (1.0 + torch.exp(-x))
        term_p = (1.0 - p) ** gamma * torch.log(torch.clamp(p, min=FLT_MIN))
        term_n = p ** gamma * torch.log(torch.clamp(1.0 - p, min=FLT_MIN))
        ctx.save_for_backward(x, flag)
        ctx.gamma, ctx.alpha = gamma, alpha
        return -flag * alpha * term_p - (1 - flag) * (1.0 - alpha) * term_n

    @staticmethod
    def backward(ctx, grad):
        x, flag = ctx.saved_tensors
        g, a = ctx.gamma, ctx.alpha
        p = 1.0 / (1.0 + torch.exp(-x))
        term_p = (1.0 - p) ** g * (1.0 - p - g * p * torch.log(torch.clamp(p, min=FLT_MIN)))
        term_n = p ** g * (g * (1.0 - p) * torch.log(torch.clamp(1.0 - p, min=FLT_MIN)) - p)
        return grad * (-flag * a * term_p - (1 - flag) * (1.0 - a) * term_n), None, None, None


class FocalLoss:
    def __init__(self, use_sigmoid=True, gamma=2.0, alpha=0.25, reduction="mean", loss_weight=1.0):
        assert use_sigmoid
        self.gamma, self.alpha, self.loss_weight = gamma, alpha, loss_weight

    def __call__(self, pred, target, weight=None, avg_factor=None):
        loss = _SigmoidFocal.apply(pred, target, self.gamma, self.alpha)
        return self.loss_weight * _weight_reduce(loss, weight.view(-1, 1), avg_factor)


class L1Loss:
    def __init__(self, reduction="mean", loss_weight=1.0):
        self.loss_weight = loss_weight

    def __call__(self, pred, target, weight=None, avg_factor=None):
        return self.loss_weight * _weight_reduce(torch.abs(pred - target), weight, avg_factor)


def _load(path, functions, methods):
    """Module-level functions and class methods of a reference file, executed in one namespace."""
    tree = ast.parse(open(os.path.join(REF, path)).read())
    ns = dict(torch=torch, force_fp32=force_fp32, np=np)
    nodes = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in functions]
    for c in tree.body:
        if isinstance(c, ast.ClassDef) and c.name in methods:
            nodes += [n for n in c.body if isinstance(n, ast.FunctionDef) and n.name in methods[c.name]]
    exec(compile(ast.Module(nodes, []), "reference:" + path, "exec"), ns)
    return ns


class _Self:
    pass


def f32(a):
    """Inputs are fp32 values (the device reads them as such), held in float64 for the reference run."""
    return np.asarray(a, np.float32).astype(np.float64)


def centerhead_case(rng, B=2, H=16, W=16, M=8, cats=(1, 2, 2, 1, 2, 2), lw=(1.0, 0.25)):
    ns = _load("mmdet3d/models/heads/bbox/centerpoint.py", {"clip_sigmoid"}, {"CenterHead": {"loss", "_gather_feat"}})
    T = len(cats)
    leaves, heatmaps, annos, inds, masks = [], [], [], [], []
    for t in range(T):
        heat = rng.normal(-1.0, 2.0, (B, cats[t], H, W))
        heat.flat[rng.choice(heat.size, 6, replace=False)] = rng.choice([-100.0, 100.0], 6)
        maps = dict(heatmap=heat, reg=rng.uniform(0, 1, (B, 2, H, W)), height=rng.normal(0, 1, (B, 1, H, W)),
                    dim=rng.normal(0, 1, (B, 3, H, W)), rot=rng.normal(0, 1, (B, 2, H, W)),
                    vel=rng.normal(0, 1, (B, 2, H, W)))
        leaves.append({k: torch.tensor(f32(v), dtype=torch.float64, requires_grad=True) for k, v in maps.items()})
        hm = rng.uniform(0, 0.9, (B, cats[t], H, W)) ** 3
        hm.flat[rng.choice(hm.size, 5, replace=False)] = 1.0
        heatmaps.append(torch.tensor(f32(hm)))
        annos.append(torch.tensor(f32(rng.normal(0, 1, (B, M, 10)))))
        ind = rng.integers(0, H * W, (B, M))
        ind[:, 1] = ind[:, 0]                                     # two objects in one cell
        inds.append(torch.tensor(ind))
        mk = (rng.uniform(0, 1, (B, M)) < 0.7).astype(np.uint8)
        mk[:, :2] = 1
        mk[0, -1] = 0
        masks.append(torch.tensor(mk))
    me = _Self()
    me.get_targets = lambda gt_b, gt_l: (heatmaps, annos, inds, masks)
    me._gather_feat = ns["_gather_feat"].__get__(me)
    me.loss_cls = GaussianFocalLoss(loss_weight=lw[0])
    me.loss_bbox = L1Loss(loss_weight=lw[1])
    cw = [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.2, 0.2]
    me.train_cfg = dict(code_weights=cw)
    preds = [[{k: (v * 1.0) for k, v in leaf.items()}] for leaf in leaves]   # non-leaf: sigmoid_ is in place
    losses = ns["loss"](me, None, None, preds)
    sum(losses.values()).backward()
    out = {"cw": np.array(cw), "cats": np.array(cats), "lw": np.array(lw)}
    for t in range(T):
        for k, v in leaves[t].items():
            out["t%d_%s" % (t, k)] = v.detach().numpy().astype(np.float32)
            out["t%d_grad_%s" % (t, k)] = v.grad.numpy()
        out["t%d_target_heatmap" % t] = heatmaps[t].numpy().astype(np.float32)
        out["t%d_anno" % t] = annos[t].numpy().astype(np.float32)
        out["t%d_ind" % t] = inds[t].numpy()
        out["t%d_mask" % t] = masks[t].numpy()
    out["loss_keys"] = np.array(list(losses))
    out["loss_values"] = np.array([float(v.detach()) for v in losses.values()])
    return out


def transfusion_case(rng, auxiliary, B=2, K=3, H=8, W=8, P=5, L=2):
    ns = _load("mmdet3d/models/heads/bbox/transfusion.py", {"clip_sigmoid"}, {"TransFusionHead": {"loss"}})
    N = P * L
    dense = rng.normal(-1.0, 2.0, (B, K, H, W))
    dense.flat[:4] = [-100.0, 100.0, -100.0, 100.0]
    heat = rng.normal(-1.0, 2.0, (B, K, N))
    heat.flat[:2] = [-100.0, 100.0]
    raw = dict(dense_heatmap=dense, heatmap=heat, center=rng.normal(0, 3, (B, 2, N)),
               height=rng.normal(0, 1, (B, 1, N)), dim=rng.normal(0, 1, (B, 3, N)), rot=rng.normal(0, 1, (B, 2, N)),
               vel=rng.normal(0, 1, (B, 2, N)))
    leaves = {k: torch.tensor(f32(v), dtype=torch.float64, requires_grad=True) for k, v in raw.items()}
    labels = rng.integers(0, K + 1, (B, N))
    label_weights = (rng.uniform(0, 1, (B, N)) < 0.8).astype(np.int64)
    bbox_targets = f32(rng.normal(0, 1, (B, N, 10)))
    bbox_weights = (labels < K).astype(np.float64)[..., None] * np.ones(10)
    hm = f32(rng.uniform(0, 0.9, (B, K, H, W)) ** 3)
    hm.flat[rng.choice(hm.size, 4, replace=False)] = 1.0
    num_pos, matched_ious = int((labels < K).sum()), 0.375
    targets = (torch.tensor(labels), torch.tensor(label_weights), torch.tensor(bbox_targets),
               torch.tensor(bbox_weights), torch.zeros(B, N, dtype=torch.float64), num_pos, matched_ious,
               torch.tensor(hm))
    me = _Self()
    me.get_targets = lambda gt_b, gt_l, p: targets
    me.loss_heatmap = GaussianFocalLoss(loss_weight=1.0)
    me.loss_cls = FocalLoss(use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0)
    me.loss_bbox = L1Loss(loss_weight=0.25)
    cw = [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.2, 0.2]
    me.train_cfg = dict(code_weights=cw)
    me.num_proposals, me.num_decoder_layers, me.auxiliary, me.num_classes = P, L, auxiliary, K
    pd = {k: (v * 1.0) for k, v in leaves.items()}
    losses = ns["loss"](me, None, None, [[pd]])
    sum(v for k, v in losses.items() if k != "matched_ious").backward()
    out = {"cw": np.array(cw), "sizes": np.array([P, L, int(auxiliary)])}
    for k, v in leaves.items():
        out[k] = v.detach().numpy().astype(np.float32)
        out["grad_" + k] = v.grad.numpy()
    for name, v in zip(("labels", "label_weights", "bbox_targets", "bbox_weights"), targets[:4]):
        out[name] = v.numpy()
    out["num_pos"], out["matched_ious"], out["target_heatmap"] = num_pos, matched_ious, hm.astype(np.float32)
    out["loss_keys"] = np.array(list(losses))
    out["loss_values"] = np.array([float(v.detach()) for v in losses.values()])
    return out


def main():
    torch.set_default_dtype(torch.float64)
    rng = np.random.default_rng(20261016)
    data = {}
    for name, case in (("ch", centerhead_case(rng)), ("chw", centerhead_case(rng, lw=(1.5, 0.4))),
                       ("tf_aux", transfusion_case(rng, True)), ("tf_last", transfusion_case(rng, False))):
        data.update({"%s_%s" % (name, k): v for k, v in case.items()})
    np.savez_compressed(OUT, **data)
    print(OUT, len(data), "arrays")


if __name__ == "__main__":
    main()
