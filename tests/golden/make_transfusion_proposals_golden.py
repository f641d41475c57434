"""Generates tests/golden/transfusion_proposals_tiny.npz from the REFERENCE's own code, on the CPU: the query
selection of TransFusionHead.forward_single (models/heads/bbox/transfusion.py), the statements from
`heatmap = dense_heatmap.detach().sigmoid()` through `top_proposals_index = ...` and the value of the
`query_heatmap_score` assignment, pulled out with `ast` and run with a stub `self` (nms_kernel_size, test_cfg,
num_proposals, num_classes).

The reference calls the unstable argsort, whose tie order is not specified, so every case is checked to have no tie
among its top K masked values (and at least K positive peaks).  The file keeps each case's logits, the CPU sigmoid
the reference computed (the oracle's input) and the reference's labels, index and query_heatmap_score.

Cases (synthetic.transfusion_heatmap logits):
  nus    B 2, C 10, 24 x 24, k 3, nuScenes, K 40, fp32
  waymo  B 1, C 3, 11 x 17, k 5, Waymo, K 12, fp32
  none   B 1, C 4, 13 x 9, k 3, no exempt classes, K 10, fp32
  half   B 1, C 10, 16 x 20, k 3, nuScenes, K 16, fp16

Run:  python tests/golden/make_transfusion_proposals_golden.py      (needs the reference tree)
"""
import ast
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, ".."))
import transfusion_proposals_oracle as O  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402

REF = os.environ.get("BEVFUSION_REFERENCE", "/root/reference")
CASES = [("nus", 2, 10, 24, 24, 3, "nuScenes", 40, torch.float32),
         ("waymo", 1, 3, 11, 17, 5, "Waymo", 12, torch.float32),
         ("none", 1, 4, 13, 9, 3, "none", 10, torch.float32),
         ("half", 1, 10, 16, 20, 3, "nuScenes", 16, torch.float16)]


def reference_selection():
    tree = ast.parse(open(REF + "/mmdet3d/models/heads/bbox/transfusion.py").read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "TransFusionHead")
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "forward_single")
    src = [ast.unparse(s) for s in fn.body]
    start = next(i for i, s in enumerate(src) if s.startswith("heatmap = dense_heatmap.detach().sigmoid()"))
    stop = next(i for i, s in enumerate(src) if s.startswith("top_proposals_index ="))
    score = next(s for s in fn.body if isinstance(s, ast.Assign) and "query_heatmap_score" in ast.unparse(s.targets[0]))
    body = fn.body[start:stop + 1] + [
        ast.Assign(targets=[ast.Name("query_heatmap_score", ast.Store())], value=score.value, lineno=0),
        ast.parse("return heatmap_sigmoid, top_proposals_class, top_proposals_index, query_heatmap_score").body[0]]
    f = ast.parse("def f(self, dense_heatmap, batch_size):\n    heatmap_sigmoid = dense_heatmap.detach().sigmoid()"
                  ).body[0]
    f.body = f.body + body
    ns = dict(torch=torch, F=F)
    exec(compile(ast.fix_missing_locations(ast.Module([f], [])), "transfusion.py", "exec"), ns)
    return ns["f"]


def main():
    select = reference_selection()
    out = {}
    for name, B, C, H, W, k, dataset, K, dtype in CASES:
        x = S.transfusion_heatmap(seed=len(out) + 3, batch=B, num_classes=C, height=H, width=W, dtype=dtype,
                                  extent=20.0)
        stub = types.SimpleNamespace(nms_kernel_size=k, test_cfg=dict(dataset=dataset), num_proposals=K,
                                     num_classes=C)
        s, labels, index, score = select(stub, x, B)
        # the masked values of the top K and the one after: no two equal, all positive
        m = O.masked_plane(s.numpy(), k, O.EXEMPT.get(dataset, ())).reshape(B, -1).astype(np.float64)
        top = -np.sort(-m, axis=1)[:, :K + 1]
        assert (top > 0).all() and (top[:, :-1] > top[:, 1:]).all(), "%s: a tie in the top K" % name
        for key, v in dict(x=x, sigmoid=s, labels=labels, index=index, score=score).items():
            out["%s_%s" % (name, key)] = v.numpy()
        out["%s_cfg" % name] = np.array([k, K, {"nuScenes": 0, "Waymo": 1}.get(dataset, 2)], np.int64)
    np.savez_compressed(os.path.join(HERE, "transfusion_proposals_tiny.npz"), **out)


if __name__ == "__main__":
    main()
