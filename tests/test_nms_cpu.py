"""CPU: the float64 NMS checker (tests/nms_oracle.py) against the fixture made from the reference's own IoU
code, host loop and circle_nms; the workspace query and argument checks of the NMS C ABI; CPU tensors raise.
No compute calls."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import nms_oracle as O

FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nms_tiny.npz")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ["bevb200_boxes_iou_bev", "bevb200_boxes_overlap_bev", "bevb200_nms_workspace_bytes", "bevb200_nms"]


def fixture():
    return np.load(FIX)


def test_oracle_iou_matches_reference():
    d = fixture()
    got = np.array([O.iou_bev(p, q) for p, q in zip(d["iou_a"], d["iou_b"])])
    assert np.abs(got - d["iou_ref"]).max() <= 1e-4
    # the named degenerate pairs: identical, half-shifted, square vs pi/4, disjoint, shared edge, containment x2,
    # zero width, identical turned
    octagon = 2 * (np.sqrt(2) - 1)                                 # unit square against itself turned by pi/4
    want = [1.0, 1 / 3, octagon / (2 - octagon), 0.0, 0.0, 1 / 16, 1 / 16, 0.0, 1.0]
    n = int(d["iou_named"])
    assert np.abs(got[:n] - want).max() <= 1e-12
    assert np.abs(d["iou_ref"][:n] - want).max() <= 1e-6


def test_fixture_pins_rotation_sign():
    """A non-square box turned by r and by -r overlap a fixed box differently: the reference's sign decides."""
    a = [0.0, 0.0, 4.0, 1.0, 0.0]
    for r in (0.3, 0.7, 1.1):
        plus, minus = O.iou_bev(a, [1.0, 0.0, 5.0, 1.0, r]), O.iou_bev(a, [1.0, 0.0, 5.0, 1.0, -r])
        assert abs(plus - minus) < 1e-12        # mirror-symmetric pair: both signs agree here
    d = fixture()
    flipped = np.array([O.iou_bev(p, np.array([q[0], q[1], q[2], q[3], -q[4]])) for p, q in
                        zip(d["iou_a"], d["iou_b"])])
    # turning only the second box the other way changes many IoUs by far more than the tolerance
    assert (np.abs(flipped - d["iou_ref"]) > 1e-2).sum() > 50


def test_oracle_keep_lists_match_reference():
    d = fixture()
    for k in range(int(d["nms_cases"])):
        keep = O.nms(d["nms%d_boxes" % k], d["nms%d_scores" % k], float(d["nms%d_thresh" % k]))
        assert np.array_equal(keep, d["nms%d_keep" % k]), k


def test_fixture_covers_the_cases():
    d = fixture()
    sizes = {int(d["nms%d_boxes" % k].shape[0]) for k in range(int(d["nms_cases"]))}
    threshs = {float(d["nms%d_thresh" % k]) for k in range(int(d["nms_cases"]))}
    assert {1, 63, 64, 65, 500} <= sizes and {-0.1, 0.0, 1.0, 0.2} <= threshs
    yaws = np.concatenate([d["iou_b"][:, 4]] + [d["nms%d_boxes" % k][:, 4] for k in range(int(d["nms_cases"]))])
    assert (np.abs(yaws) > np.pi).any()
    ks = [len(d["nms%d_keep" % k]) for k in range(int(d["nms_cases"]))]
    assert min(ks) >= 1 and max(k for k, n in zip(ks, sizes) if n > 1) > 1


def test_oracle_circle_nms_matches_reference():
    d = fixture()
    for k in range(int(d["circle_cases"])):
        keep = O.circle_nms(d["circle%d_dets" % k], float(d["circle%d_thresh" % k]), int(d["circle%d_post" % k]))
        assert np.array_equal(keep, d["circle%d_keep" % k]), k


def test_check_greedy_flags_bad_lists():
    d = fixture()
    b, s = d["nms7_boxes"], d["nms7_scores"]
    order = O.sort_desc(s)
    iou = O.iou_matrix(b[order], b[order])
    good = O.greedy(iou, 0.2)
    assert O.check_greedy(iou, good, 0.2, 1e-4) == []
    assert O.check_greedy(iou, good[:-1], 0.2, 1e-4) != []                     # a box dropped without cause
    dropped = sorted(set(range(len(b))) - set(good))
    assert O.check_greedy(iou, sorted(good + dropped[:1]), 0.2, 1e-4) != []    # a suppressed box kept


def test_symbols_declared_and_exported():
    from bevfusion_b200 import _C
    declared = _C.declared_symbols()
    L = _C.lib()
    for name in SYMBOLS:
        assert name in declared and hasattr(L, name), name
    text = open(os.path.join(ROOT, "include", "bevfusion_b200.h")).read()
    for macro, value in (("ROTATE", 0), ("NORMAL", 1), ("CIRCLE", 2), ("MAX_BOXES", 65536)):
        assert re.search(r"#define BEVB200_NMS_%s %d\b" % (macro, value), text), macro


def test_workspace_and_argument_checks():
    from bevfusion_b200 import _C
    L = _C.lib()
    assert L.bevb200_nms_workspace_bytes(1, 64) >= 64 * 8
    assert L.bevb200_nms_workspace_bytes(24, 500) >= 24 * 500 * 8 * 8
    assert L.bevb200_nms_workspace_bytes(1, 65536) >= 65536 * 1024 * 8
    assert L.bevb200_nms_workspace_bytes(1, 65537) == 0
    assert L.bevb200_nms_workspace_bytes(-1, 10) == 0
    cnt = ctypes.c_int32(0)
    p = ctypes.addressof(cnt)
    # above 65,536 boxes per segment: unsupported, whatever else is passed
    assert L.bevb200_nms(None, None, 1, 65537, 0, 0.2, 10, None, None, p, None, 0, None) == -4
    assert L.bevb200_nms(None, None, 1, 64, 3, 0.2, 10, None, None, p, None, 0, None) == -1       # bad mode
    assert L.bevb200_nms(None, None, 1, 64, 0, 0.2, -1, None, None, p, None, 0, None) == -1       # bad post_max
    assert L.bevb200_nms(None, None, 0, 64, 0, 0.2, 10, None, None, None, None, 0, None) == 0     # nothing to do
    buf = (ctypes.c_int64 * 10)()
    assert L.bevb200_nms(1, None, 1, 64, 0, 0.2, 10, None, ctypes.addressof(buf), p, None, 0, None) == -3
    assert L.bevb200_boxes_iou_bev(None, -1, None, 3, None, None) == -1
    assert L.bevb200_boxes_iou_bev(None, 0, None, 3, None, None) == 0


def test_cpu_tensors_raise():
    from bevfusion_b200 import iou3d
    boxes, scores = torch.zeros(4, 5), torch.arange(4.0)
    with pytest.raises(RuntimeError):
        iou3d.boxes_iou_bev(boxes, boxes)
    with pytest.raises(RuntimeError):
        iou3d.nms_gpu(boxes, scores, 0.2)
    with pytest.raises(RuntimeError):
        iou3d.nms_normal_gpu(boxes, scores, 0.2)
    with pytest.raises(RuntimeError):
        iou3d.circle_nms(torch.zeros(4, 3), 1.0)
    with pytest.raises(RuntimeError):
        iou3d.nms_batched(boxes[None], scores[None], torch.tensor([4]), "rotate", 0.2)
    with pytest.raises(RuntimeError):
        iou3d.centerhead_nms([dict(bboxes=torch.zeros(4, 9), scores=scores, labels=torch.zeros(4))], 0, "rotate",
                             dict(post_max_size=83), [1.0])
