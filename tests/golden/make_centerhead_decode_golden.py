"""Generates tests/golden/centerhead_decode_tiny.npz from the REFERENCE's own code, on the CPU: the class
CenterPointBBoxCoder of core/bbox/coders/centerpoint_bbox_coders.py, taken out of its module with `ast` (the module
imports mmdet, which is not needed for the class body: the base class is replaced by `object` and the registry
decorator dropped) and run on activated head outputs.

The reference calls the unstable torch.topk, whose tie order is not specified, so every case is checked to have no
tie among its top max_num + 1 scores.  The file keeps each case's activated maps (the oracle's input), the coder's
fields and the reference's per-sample bboxes / scores / labels, concatenated over samples, with their counts.

Cases (synthetic.centerhead_head_outputs, sigmoid and exp applied on CPU torch):
  two     task 1 (2 classes), B 2, 16 x 20, max_num 30, score_threshold 0.1, reg and vel
  plain   task 0 (1 class), B 1, 11 x 17, max_num 12, score_threshold None, no reg, no vel, a height range
  tight   task 5 (2 classes), B 1, 9 x 13, max_num 40, score_threshold 0.0, a post_center_range that cuts rows

Run:  python tests/golden/make_centerhead_decode_golden.py      (needs the reference tree)
"""
import ast
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from bevfusion_b200 import synthetic as S  # noqa: E402

REF = os.environ.get("BEVFUSION_REFERENCE", "/root/reference")
MAPS = ("heatmap", "reg", "height", "dim", "rot", "vel")
FIELDS = ("pc_range", "out_size_factor", "voxel_size", "post_center_range", "max_num", "score_threshold")
CASES = [("two", 1, 2, 16, 20, 30, 0.1, True, True, None),
         ("plain", 0, 1, 11, 17, 12, None, False, False, [-61.2, -61.2, -1.5, 61.2, 61.2, 1.0]),
         ("tight", 5, 1, 9, 13, 40, 0.0, True, True, [-30.0, -40.0, -1.0, 35.0, 30.0, 0.5])]


def reference_coder():
    tree = ast.parse(open(REF + "/mmdet3d/core/bbox/coders/centerpoint_bbox_coders.py").read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "CenterPointBBoxCoder")
    cls.bases, cls.decorator_list = [ast.Name("object", ast.Load())], []
    ns = dict(torch=torch)
    exec(compile(ast.fix_missing_locations(ast.Module([cls], [])), "centerpoint_bbox_coders.py", "exec"), ns)
    return ns["CenterPointBBoxCoder"]


def main():
    Coder = reference_coder()
    out = {}
    for name, task, B, H, W, K, thr, with_reg, with_vel, rng in CASES:
        raw = S.centerhead_head_outputs(seed=len(out) + 5, batch=B, height=H, width=W, extent=30.0)[task]
        cfg = S.centerhead_coder_cfg(H, W, extent=30.0, max_num=K, score_threshold=thr)
        if rng is not None:
            cfg["post_center_range"] = rng
        maps = dict(heatmap=raw["heatmap"].sigmoid(), reg=raw["reg"] if with_reg else None, height=raw["height"],
                    dim=torch.exp(raw["dim"]), rot=raw["rot"], vel=raw["vel"] if with_vel else None)
        top = maps["heatmap"].reshape(B, -1).double().sort(1, descending=True)[0][:, :K + 1]
        assert (top[:, :-1] > top[:, 1:]).all(), "%s: a tie in the top max_num + 1" % name
        coder = Coder(**{k: cfg[k] for k in FIELDS}, code_size=9 if with_vel else 7)
        got = coder.decode(maps["heatmap"], maps["rot"][:, 0:1], maps["rot"][:, 1:2], maps["height"], maps["dim"],
                           maps["vel"], reg=maps["reg"], task_id=task)
        assert 0 < sum(len(g["scores"]) for g in got) < B * K, "%s: the masks cut nothing or everything" % name
        for k in MAPS:
            if maps[k] is not None:
                out["%s_%s" % (name, k)] = maps[k].numpy()
        for k in ("pc_range", "voxel_size", "post_center_range"):
            out["%s_%s" % (name, k)] = np.array(cfg[k], np.float64)
        out["%s_cfg" % name] = np.array([cfg["out_size_factor"], K, -1.0 if thr is None else thr], np.float64)
        for k in ("bboxes", "scores", "labels"):
            out["%s_out_%s" % (name, k)] = torch.cat([g[k] for g in got]).numpy()
        out["%s_out_counts" % name] = np.array([len(g["scores"]) for g in got], np.int64)
    np.savez_compressed(os.path.join(HERE, "centerhead_decode_tiny.npz"), **out)


if __name__ == "__main__":
    main()
