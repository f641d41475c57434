"""CPU: the numpy restatement of the CenterHead / TransFusion heatmap targets (tests/head_targets_oracle.py) against
the fixture made from the reference's own code, bit for bit; the fixture covers the cases it is meant to; the
workspace query, the argument checks of the C ABI and the host-side validation of bevfusion_b200.head_targets.
No compute calls."""
import ctypes
import json
import os
import re

import numpy as np
import pytest
import torch

import head_targets_oracle as O

FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "head_targets_tiny.npz")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TASK_CLASSES = [1, 2, 2, 1, 2, 2]
SYMBOLS = ["bevb200_head_targets_workspace_bytes", "bevb200_head_targets", "bevb200_draw_heatmap_gaussian"]


def fixture():
    return np.load(FIX)


def case(d, name):
    meta = json.loads(str(d[name + "_cfg"]))
    return meta, d[name + "_boxes"], d[name + "_labels"], d[name + "_counts"]


def oracle_case(d, name):
    meta, boxes, labels, counts = case(d, name)
    cfg = meta["cfg"]
    if meta["mode"] == "centerhead":
        M = cfg["max_objs"] * cfg["dense_reg"]
        return meta, O.targets(boxes, labels, counts, "centerhead", TASK_CLASSES, cfg, M, meta["norm_bbox"])
    return meta, O.targets(boxes, labels, counts, "transfusion", [10], cfg)


def bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("name", ["ch_six", "ch_small", "tf_ten", "tf_wide"])
def test_oracle_matches_reference_bit_for_bit(name):
    d = fixture()
    meta, got = oracle_case(d, name)
    if meta["mode"] == "centerhead":
        for t in range(6):
            assert bits_equal(got["heatmaps"][t], d["%s_hm%d" % (name, t)]), t
        assert bits_equal(got["anno"], d[name + "_anno"])
        assert bits_equal(got["ind"], d[name + "_ind"])
        assert bits_equal(got["mask"], d[name + "_mask"])
    else:
        assert bits_equal(got["heatmaps"][0], d[name + "_hm"])
    assert got["status"] == 0      # the fixture holds nothing the reference would raise on


def test_fixture_covers_the_cases():
    d = fixture()
    assert sorted(d["cases"].tolist()) == ["ch_six", "ch_small", "tf_ten", "tf_wide"]
    dims = {}
    for name in d["cases"].tolist():
        meta, boxes, labels, counts = case(d, name)
        cfg = meta["cfg"]
        osf = cfg["out_size_factor"]
        fx, fy = cfg["grid_size"][0] // osf, cfg["grid_size"][1] // osf
        dims[name] = (boxes.shape[2], meta["norm_bbox"], fx == fy)
        assert 0 in counts.tolist() or name in ("ch_small", "tf_ten")
        live = np.arange(boxes.shape[1])[None, :] < counts[:, None]
        b, l = boxes[live], labels[live]
        assert (b[:, 3] == 0).any() and (b[:, 4] < 0).any() and np.isnan(b[:, 3]).any()
        cx = (b[:, 0] - np.float32(cfg["point_cloud_range"][0])) / np.float32(cfg["voxel_size"][0]) / np.float32(osf)
        assert ((cx > -1) & (cx < 0)).any() and (cx == 0).any() and (cx == fx).any()
        _, got = oracle_case(d, name)
        rec = got["records"][live]
        drawn = rec[:, 3] >= 0
        if meta["mode"] == "transfusion":
            # centres off the map that still draw (within r cells) and ones that do not
            assert (drawn & ((rec[:, 1] < 0) | (rec[:, 1] >= fy))).any()
        else:
            assert ((l >= 10) | (l < 0)).any()                                  # labels of no task
        w = b[:, 3] / np.float32(cfg["voxel_size"][0]) / np.float32(osf)
        ln = b[:, 4] / np.float32(cfg["voxel_size"][1]) / np.float32(osf)
        r = np.array([O.gaussian_radius(p, q, cfg["gaussian_overlap"]) for p, q in zip(ln, w) if p > 0 and q > 0])
        frac = r.astype(np.float64) - np.round(r)
        assert ((frac < 0) & (frac > -1e-5) & (r > 2.5)).any() and ((frac >= 0) & (frac < 1e-5) & (r > 2.5)).any()
        # overlapping same-class gaussians: two drawn records on one plane whose windows share a cell of the map
        q = rec[drawn]
        same = q[:, None, 0] == q[None, :, 0]
        reach = q[:, None, 3] + q[None, :, 3]
        near = (np.abs(q[:, None, 1] - q[None, :, 1]) <= reach) & (np.abs(q[:, None, 2] - q[None, :, 2]) <= reach)
        inside = (q[:, 1] >= 0) & (q[:, 1] < fy) & (q[:, 2] >= 0) & (q[:, 2] < fx)
        pair = np.triu(same & near & inside[:, None] & inside[None, :], 1)
        assert pair.any(), name
    assert dims["ch_six"] == (9, True, True) and dims["ch_small"] == (7, False, False)
    assert dims["tf_wide"][0] == 7 and not dims["tf_wide"][2]
    meta, boxes, labels, counts = case(d, "ch_small")
    assert (labels[0, :counts[0]] == 0).sum() > meta["cfg"]["max_objs"]   # more cars than max_objs


def test_oracle_radius_is_fp32_op_order():
    # the nuScenes car at 0.8 m cells: radius from the fp32 formula, min_radius applied after int()
    r = O.gaussian_radius(np.float32(4.6) / np.float32(0.1) / np.float32(8), np.float32(1.95) / np.float32(0.1)
                          / np.float32(8), 0.1)
    assert r.dtype == np.float32 and 0.5 < r < 2.0
    assert O.gaussian_radius(np.float32(0), np.float32(0), 0.1) == 0
    assert np.isnan(O.gaussian_radius(np.float32(np.inf), np.float32(1), 0.1))


def test_symbols_declared_and_exported():
    from bevfusion_b200 import _C
    declared = _C.declared_symbols()
    L = _C.lib()
    for name in SYMBOLS:
        assert name in declared and hasattr(L, name), name
    text = open(os.path.join(ROOT, "include", "bevfusion_b200.h")).read()
    for macro, value in (("CENTERHEAD", 0), ("TRANSFUSION", 1), ("MAX_BOXES", 4096), ("MAX_TASKS", 32),
                         ("MAX_LABELS", 256)):
        assert re.search(r"#define BEVB200_HEAD_TARGETS_%s %d\b" % (macro, value), text), macro


def _call(L, **kw):
    table = (ctypes.c_int32 * 20)(*[v for t, n in enumerate(TASK_CLASSES) for c in range(n) for v in (t, c)])
    classes = (ctypes.c_int32 * 6)(*TASK_CLASSES)
    st = ctypes.c_int32(0)
    a = dict(boxes=None, labels=None, counts=None, B=1, nmax=0, D=9, table=ctypes.addressof(table), nl=10,
             classes=ctypes.addressof(classes), nt=6, fx=128, fy=128, mode=0, max_objs=0, ws=None, ws_bytes=0,
             heatmap=1, status=ctypes.addressof(st))
    a.update(kw)
    return L.bevb200_head_targets(a["boxes"], a["labels"], a["counts"], a["B"], a["nmax"], a["D"], a["table"],
                                  a["nl"], a["classes"], a["nt"], -51.2, -51.2, 0.1, 0.1, 8, a["fx"], a["fy"], 0.1,
                                  2, a["mode"], a["max_objs"], 1, a["heatmap"], None, None, None, a["status"],
                                  a["ws"], a["ws_bytes"], None)


def test_workspace_and_argument_checks():
    from bevfusion_b200 import _C
    L = _C.lib()
    assert L.bevb200_head_targets_workspace_bytes(4, 120) >= 4 * 120 * 16
    assert L.bevb200_head_targets_workspace_bytes(1, 4096) >= 4096 * 16
    assert L.bevb200_head_targets_workspace_bytes(1, 4097) == 0
    assert L.bevb200_head_targets_workspace_bytes(-1, 10) == 0
    assert _call(L, nmax=4097) == -4                            # too many boxes per sample
    assert _call(L, mode=2) == -1                               # bad mode
    assert _call(L, D=8) == -1                                  # box_dim 7 or 9
    assert _call(L, mode=1) == -1                               # TransFusion takes one task
    assert _call(L, nt=33) == -1 and _call(L, nt=0) == -1
    assert _call(L, nl=257) == -1
    assert _call(L, fx=0) == -1
    assert _call(L, status=None) == -1
    bad = (ctypes.c_int32 * 2)(0, 1)                            # task 0 has one class
    assert _call(L, table=ctypes.addressof(bad), nl=1) == -1
    assert _call(L, nmax=10, boxes=1, labels=1) == -3           # workspace too small
    assert L.bevb200_draw_heatmap_gaussian(None, 4, 4, 0, 0, -1, 1.0, None) == -1
    assert L.bevb200_draw_heatmap_gaussian(None, 4, 4, 0, 0, 2 ** 30, 1.0, None) == -1     # radius too large
    assert L.bevb200_draw_heatmap_gaussian(None, 0, 4, 0, 0, 2, 1.0, None) == 0


def test_host_side_validation():
    from bevfusion_b200 import head_targets as H
    cfg = dict(point_cloud_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], grid_size=[1024, 1024, 40],
               voxel_size=[0.1, 0.1, 0.2], out_size_factor=8, dense_reg=1, gaussian_overlap=0.1, max_objs=500,
               min_radius=2)
    boxes, labels = [torch.zeros(3, 9)], [torch.zeros(3, dtype=torch.long)]
    with pytest.raises(RuntimeError):                           # CPU tensors raise: no CPU path
        H.centerhead_targets(boxes, labels, [["car"]], cfg)
    with pytest.raises(RuntimeError):
        H.transfusion_heatmap_targets(boxes, labels, 10, cfg)
    with pytest.raises(RuntimeError):
        H.centerhead_targets_batched(torch.zeros(1, 3, 9), torch.zeros(1, 3, dtype=torch.int32),
                                     torch.tensor([3], dtype=torch.int32), [["car"]], cfg)
    with pytest.raises(RuntimeError):
        H.draw_heatmap_gaussian(torch.zeros(8, 8), (2, 2), 2)
    with pytest.raises(ValueError):
        H.task_class_counts([])
    with pytest.raises(ValueError):
        H.task_class_counts([[]])
    with pytest.raises(ValueError):
        H.task_class_counts([["car"]] * 33)
    assert H.task_class_counts([dict(num_class=1, class_names=["car"]), dict(num_class=2, class_names=["a", "b"]),
                                ["x", "y"], 3]) == [1, 2, 2, 3]
    assert H.centerhead_label_table([1, 2]) == [(0, 0), (1, 0), (1, 1)]
    with pytest.raises(ValueError):
        H.pad_gt([], [])


def test_gaussian_radius_mirror_matches_oracle():
    from bevfusion_b200 import head_targets as H
    rng = np.random.default_rng(1)
    h = rng.uniform(0.1, 30, 500).astype(np.float32)
    w = rng.uniform(0.1, 30, 500).astype(np.float32)
    got = H.gaussian_radius((torch.from_numpy(h), torch.from_numpy(w)), 0.1).numpy()
    want = np.array([O.gaussian_radius(a, b, 0.1) for a, b in zip(h, w)], np.float32)
    assert bits_equal(got, want)
