"""The TransFusion assignment's specification on the CPU: the solver restatement (lsap_oracle) against scipy on
thousands of seeded matrices, the numpy restatement of get_targets (transfusion_assign_oracle) against the golden
fixture, and the C ABI's symbols."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
import lsap_oracle  # noqa: E402
import transfusion_assign_oracle as TO  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "transfusion_assign_tiny.npz")


def lsap_cases(seed, count, max_size=11):
    """Seeded fp32 matrices: random normal, small integers (ties everywhere), one decimal, and constant; every
    orientation."""
    rng = np.random.default_rng(seed)
    for t in range(count):
        r, c = (int(v) for v in rng.integers(1, max_size + 1, 2))
        kind = t % 4
        if kind == 0:
            m = rng.standard_normal((r, c))
        elif kind == 1:
            m = rng.integers(0, 3, (r, c))
        elif kind == 2:
            m = np.round(rng.standard_normal((r, c)), 1)
        else:
            m = np.full((r, c), float(rng.integers(-2, 3)))
        yield m.astype(np.float32)


def large_cases():
    rng = np.random.default_rng(5)
    for r, c in ((300, 200), (200, 300), (120, 200), (200, 200), (64, 64)):
        yield rng.standard_normal((r, c)).astype(np.float32)
        yield rng.integers(0, 4, (r, c)).astype(np.float32)


def test_lsap_oracle_equals_scipy_small():
    n = 0
    for m in lsap_cases(0, 3000):
        a, b = linear_sum_assignment(m)
        x, y = lsap_oracle.solve(m)
        assert np.array_equal(a, x) and np.array_equal(b, y), m
        n += 1
    assert n == 3000


def test_lsap_oracle_equals_scipy_large():
    for m in large_cases():
        a, b = linear_sum_assignment(m)
        x, y = lsap_oracle.solve(m)
        assert np.array_equal(a, x) and np.array_equal(b, y), m.shape


def test_lsap_oracle_edges():
    assert [len(v) for v in lsap_oracle.solve(np.zeros((0, 3), np.float32))] == [0, 0]
    with pytest.raises(ValueError):
        lsap_oracle.solve(np.array([[np.nan, 1.0]], np.float32))
    with pytest.raises(ValueError):
        lsap_oracle.solve(np.array([[-np.inf, 1.0]], np.float32))
    with pytest.raises(lsap_oracle.Infeasible):
        lsap_oracle.solve(np.array([[np.inf, np.inf], [1.0, 2.0]], np.float32))
    with pytest.raises(ValueError):
        linear_sum_assignment(np.array([[np.inf, np.inf], [1.0, 2.0]], np.float32))


def _golden_inputs(z):
    preds = {k[5:]: z[k] for k in z.files if k.startswith("pred_")}
    return z["gt_boxes"], z["gt_labels"], z["counts"], preds, int(z["num_classes"]), int(z["num_proposals"])


def test_oracle_reproduces_golden():
    z = np.load(GOLDEN)
    gt, gl, counts, preds, K, P = _golden_inputs(z)
    got = TO.targets(gt, gl, counts, preds, K, P, S.TRANSFUSION_TRAIN_CFG, S.TRANSFUSION_CODER)
    for k in ("gt_inds", "labels", "label_weights", "bbox_weights", "num_pos"):
        assert np.array_equal(got[k], z[k]), k
    bt, want = got["bbox_targets"], z["bbox_targets"]
    ulp = np.abs(bt.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    assert ulp.max() <= 2
    assert np.abs(got["ious"] - z["ious"]).max() <= 1e-6
    assert np.abs(got["mean_iou"] - z["mean_iou"]).max() <= 1e-6
    assert z["num_pos"].tolist() == [20, 48, 0]     # 10 gts x 2 layers, 24 proposals x 2 layers, no gt


def test_oracle_pos_weight_truncates():
    z = np.load(GOLDEN)
    gt, gl, counts, preds, K, P = _golden_inputs(z)
    cfg = dict(S.TRANSFUSION_TRAIN_CFG, pos_weight=2.7)
    got = TO.targets(gt, gl, counts, preds, K, P, cfg, S.TRANSFUSION_CODER)
    assert set(np.unique(got["label_weights"][got["gt_inds"] > 0]).tolist()) == {2}
    assert set(np.unique(got["label_weights"][got["gt_inds"] == 0]).tolist()) == {1}


def test_transfusion_predictions_shapes_and_ties():
    gt = S.gt_boxes(seed=3, batch=2)
    p = S.transfusion_predictions(1, 2, gt, num_proposals=200, num_classes=10, layers=2)
    assert tuple(p["heatmap"].shape) == (2, 10, 400) and tuple(p["center"].shape) == (2, 2, 400)
    assert tuple(p["height"].shape) == (2, 1, 400) and tuple(p["dim"].shape) == (2, 3, 400)
    cols = torch.cat([p[k][0] for k in ("heatmap", "center", "height", "dim", "rot")], 0).T[:200]
    assert len(torch.unique(cols, dim=0)) < 200          # exact duplicate proposals


def test_cabi_symbols_exported():
    from bevfusion_b200 import _C
    lib = ctypes.CDLL(_C.LIB_PATH)
    for name in ("bevb200_lsap", "bevb200_lsap_workspace_bytes", "bevb200_transfusion_assign",
                 "bevb200_transfusion_assign_workspace_bytes"):
        assert hasattr(lib, name), name
        assert name in _C.declared_symbols()
    L = _C.lib()
    assert L.bevb200_transfusion_assign_workspace_bytes(4, 1, 200, 120) >= 4 * 200 * 120 * 4
    assert L.bevb200_transfusion_assign_workspace_bytes(1, 1, 4097, 1) == 0
    assert L.bevb200_transfusion_assign_workspace_bytes(65536, 1, 8, 8) == 0
    assert L.bevb200_lsap_workspace_bytes(8, 200, 120) == 0


def test_ctypes_signatures_match_the_header():
    """ctypes passes an argument past its declared list with default conversion (a 32-bit int), so a short list
    corrupts the trailing pointers: every new binding declares exactly the header's parameter count."""
    import re
    from bevfusion_b200 import _C
    with open(_C.HEADER_PATH) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    for name in ("bevb200_lsap", "bevb200_lsap_workspace_bytes", "bevb200_transfusion_assign",
                 "bevb200_transfusion_assign_workspace_bytes"):
        params = re.search(r"\b%s\s*\(([^;]*?)\)\s*;" % name, text, re.S).group(1)
        assert len([a for a in params.split(",") if a.strip()]) == len(_C._SIGNATURES[name][1]), name


def test_python_refuses_cpu_tensors():
    from bevfusion_b200 import transfusion_assign as TA
    with pytest.raises(RuntimeError):
        TA.linear_sum_assignment_batched(torch.zeros((1, 2, 2)))
