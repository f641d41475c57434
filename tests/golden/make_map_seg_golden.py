"""Generates tests/golden/map_seg_tiny.npz from the REFERENCE's own map-segmentation code, run on the CPU.

BEVGridTransform, sigmoid_xent_loss, sigmoid_focal_loss and BEVSegmentationHead (models/heads/segm/vanilla.py) and
NuScenesDataset.evaluate_map (datasets/nuscenes_dataset.py) are extracted from the reference files with `ast` and
executed as written, with three edits so that they run in float64 and expose their counts:
  - the grid coordinates keep the reference's fp32 values but take the input's dtype (grid_sample needs the two to
    match), so the transform and its gradient run in float64 at the fp32 sample coordinates;
  - the losses' .float() widening becomes .double();
  - evaluate_map also returns its tp / fp / fn tensors.
Cases: prescale 1, 2, 0.5 and 1.5 on a non-square scope pair; an output scope reaching outside the input (zeros
padding); both losses on saturated logits (+-30, +-100); a head (focal, prescale 2) in train and eval mode;
evaluate_map on predictions with exact threshold ties.

Run:  python tests/golden/make_map_seg_golden.py      (needs the reference tree)"""
import ast
import os
from typing import Any, Dict, List, Optional, Tuple, Union  # noqa: F401  (the reference's annotations)

import numpy as np
import torch
from torch import nn  # noqa: F401
from torch.nn import functional as F  # noqa: F401

REF = os.environ.get("BEVFUSION_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "map_seg_tiny.npz")

IN_SCOPE = [[-6.4, 6.4, 0.8], [-4.8, 4.8, 0.8]]            # 16 x 12 cells
OUT_SCOPE = [[-6.0, 6.0, 0.5], [-4.0, 4.0, 0.5]]           # 24 x 16
WIDE_SCOPE = [[-8.0, 8.0, 0.5], [-5.0, 6.0, 0.5]]          # 32 x 22, reaches outside the input
GEOMS = {"p1": (OUT_SCOPE, 1), "p2": (OUT_SCOPE, 2), "p05": (OUT_SCOPE, 0.5), "p15": (OUT_SCOPE, 1.5),
         "pad": (WIDE_SCOPE, 1), "pad2": (WIDE_SCOPE, 2)}
CLASSES = ["drivable_area", "ped_crossing", "divider"]


class _Edit(ast.NodeTransformer):
    def visit_Call(self, node):
        self.generic_visit(node)
        f = node.func
        if isinstance(f, ast.Attribute) and f.attr == "float" and not node.args:
            f.attr = "double"
        if (isinstance(f, ast.Attribute) and f.attr == "to" and len(node.args) == 1
                and ast.unparse(node.args[0]) == "x.device"):
            node.args.append(ast.parse("x.dtype").body[0].value)
        return node

    def visit_Return(self, node):
        if isinstance(node.value, ast.Name) and node.value.id == "metrics":
            node.value = ast.parse("(metrics, tp, fp, fn)").body[0].value
        return node


def _load():
    ns = dict(globals())
    nodes = []
    tree = ast.parse(open(os.path.join(REF, "mmdet3d/models/heads/segm/vanilla.py")).read())
    for n in tree.body:
        if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and n.name in (
                "sigmoid_xent_loss", "sigmoid_focal_loss", "BEVGridTransform", "BEVSegmentationHead"):
            n.decorator_list = []
            nodes.append(n)
    tree = ast.parse(open(os.path.join(REF, "mmdet3d/datasets/nuscenes_dataset.py")).read())
    for c in tree.body:
        if isinstance(c, ast.ClassDef) and c.name == "NuScenesDataset":
            nodes += [n for n in c.body if isinstance(n, ast.FunctionDef) and n.name == "evaluate_map"]
    mod = ast.fix_missing_locations(_Edit().visit(ast.Module(nodes, [])))
    exec(compile(mod, "reference", "exec"), ns)
    return ns


def main():
    R = _load()
    rng = np.random.default_rng(0)
    torch.manual_seed(0)
    out = {"classes": np.array(CLASSES), "in_scope": np.array(IN_SCOPE), "out_scope": np.array(OUT_SCOPE),
           "wide_scope": np.array(WIDE_SCOPE)}
    # grid transform, forward and the gradient of sum(out * r)
    x = rng.standard_normal((2, 3, 16, 12))
    out["grid_x"] = x
    for name, (oscope, p) in GEOMS.items():
        t = R["BEVGridTransform"](input_scope=IN_SCOPE, output_scope=oscope, prescale_factor=p)
        xt = torch.tensor(x, requires_grad=True)
        y = t(xt)
        r = torch.tensor(rng.standard_normal(tuple(y.shape)))
        (y * r).sum().backward()
        out["grid_%s_p" % name] = np.float64(p)
        out["grid_%s_out" % name] = y.detach().numpy()
        out["grid_%s_r" % name] = r.numpy()
        out["grid_%s_grad" % name] = xt.grad.numpy()
    # losses: per class, the reference head's loop; gradient of sum_k w_k loss_k
    logits = rng.standard_normal((2, 3, 10, 10)) * 3
    flat = logits.reshape(-1)
    flat[:8] = [30, -30, 100, -100, 30, -30, 100, -100]
    target = (rng.random((2, 3, 10, 10)) < 0.4).astype(np.int64)
    target[0, 2] = 0
    target[1, 2] = 1
    out["loss_logits"], out["loss_target"] = logits, target
    w = rng.random(3) + 0.5
    out["loss_w"] = w
    for loss in ("focal", "xent"):
        xl = torch.tensor(logits, requires_grad=True)
        tl = torch.tensor(target)
        fn = R["sigmoid_focal_loss"] if loss == "focal" else R["sigmoid_xent_loss"]
        vals = [fn(xl[:, k], tl[:, k]) for k in range(3)]
        sum(v * float(w[k]) for k, v in enumerate(vals)).backward()
        out["loss_%s_values" % loss] = np.array([float(v.detach()) for v in vals])
        out["loss_%s_grad" % loss] = xl.grad.numpy()
    # head: focal, prescale 2, train (losses, feature gradient) and eval (sigmoid)
    head = R["BEVSegmentationHead"](4, dict(input_scope=IN_SCOPE, output_scope=OUT_SCOPE, prescale_factor=2),
                                    CLASSES, "focal").double()
    with torch.no_grad():
        for m in head.classifier:
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.2, 0.2)
                m.running_mean.uniform_(-0.2, 0.2)
                m.running_var.uniform_(0.5, 1.5)
    feats = rng.standard_normal((2, 4, 16, 12))
    masks = (rng.random((2, 3, 24, 16)) < 0.3).astype(np.int64)
    state = {k: v.numpy().copy() for k, v in head.state_dict().items()}
    ft = torch.tensor(feats, requires_grad=True)
    head.train()
    hl = head([ft], torch.tensor(masks))
    sum(hl.values()).backward()
    out["head_keys"] = np.array(list(hl))
    out["head_losses"] = np.array([float(v.detach()) for v in hl.values()])
    out["head_grad"] = ft.grad.numpy()
    head.load_state_dict({k: torch.tensor(v) for k, v in state.items()})   # eval with the pre-step statistics
    head.eval()
    with torch.no_grad():
        out["head_eval"] = head([torch.tensor(feats)]).numpy()
    out["head_feats"], out["head_masks"] = feats, masks
    for k, v in state.items():
        out["head_state/" + k] = v
    # evaluate_map with ties at every threshold
    thr = np.array([0.35, 0.4, 0.45, 0.5, 0.55, 0.6, 0.65], np.float32)
    preds = rng.random((4, 3, 12, 12)).astype(np.float32)
    preds.reshape(-1)[::3] = rng.choice(thr, size=preds.size // 3 + 1)[:len(preds.reshape(-1)[::3])]
    preds[0, 0, 0, :3] = np.nan
    gts = (rng.random((4, 3, 12, 12)) < 0.5).astype(np.int64)

    class _Self:
        map_classes = CLASSES

    results = [dict(masks_bev=torch.tensor(preds[i]), gt_masks_bev=torch.tensor(gts[i])) for i in range(4)]
    metrics, tp, fp, fn = R["evaluate_map"](_Self(), results)
    out["eval_pred"], out["eval_gt"] = preds, gts
    out["eval_counts"] = np.stack([tp.numpy(), fp.numpy(), fn.numpy()]).astype(np.int64)
    out["eval_keys"] = np.array(list(metrics))
    out["eval_values"] = np.array(list(metrics.values()))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays")


if __name__ == "__main__":
    main()
