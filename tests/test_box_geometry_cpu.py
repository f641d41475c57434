"""CPU: the float64 checker (tests/nms_oracle.py) against closed forms on every box family of
tests/box_families.py: the rotated BEV overlap and IoU in both argument orders, and the 3D IoU of
BaseInstance3DBoxes.overlaps (BEV overlap times height overlap, over the clamped union) with the boxes side by
side in z, stacked touching, and stacked overlapping.  The GPU tests of those families compare the kernels with
this checker, so it is pinned here first."""
import numpy as np
import pytest

import box_families as F
import nms_oracle as O

N = 2000
EXACT = 1e-9


@pytest.fixture(scope="module")
def fams():
    return F.families(np.random.default_rng(7), N)


@pytest.mark.parametrize("name", F.NAMES)
def test_bev_overlap_and_iou_closed_forms(fams, name):
    A, B, ov, iou = fams[name]
    for X, Y in ((A, B), (B, A)):
        got_ov = np.array([O.overlap_bev(p, q) for p, q in zip(X, Y)])
        got_iou = np.array([O.iou_bev(p, q) for p, q in zip(X, Y)])
        assert np.abs(got_ov - ov).max() <= EXACT
        assert np.abs(got_iou - iou).max() <= EXACT
    assert np.array_equal(O.iou_matrix(A[:50], B[:50]).diagonal(), [O.iou_bev(p, q) for p, q in zip(A[:50], B[:50])])


def test_closed_forms_are_not_trivial(fams):
    """Each family holds the geometry it is named for."""
    for name in ("touch_end", "touch_side", "touch_corner", "zero_width"):
        assert (fams[name][2] == 0).all(), name
    for name in ("slide", "nested", "yaw_pi", "square_half_pi"):
        iou = fams[name][3]
        assert (iou > 0.05).mean() > 0.7, name
    inside = fams["corner_on_edge"][2] > 0
    assert 0.3 < inside.mean() < 0.7
    ulp = fams["yaw_ulp"][3]
    assert (ulp <= 1).all() and (ulp > 1 - 1e-3).all() and (ulp < 1).mean() > 0.9
    assert (fams["yaw_ulp"][0][:, 4] != fams["yaw_ulp"][1][:, 4]).all()


def test_turned_overlap_closed_form():
    """The small-turn octagon against the checker at angles large enough to see, on both sides of 0."""
    for w, l in F.SIZES:
        for theta in (1e-3, -1e-3, 1e-2):
            a = [-w / 2, -l / 2, w / 2, l / 2, 0.3]
            b = [-w / 2, -l / 2, w / 2, l / 2, 0.3 + theta]
            if max(w, l) * abs(theta) < 0.5 * min(w, l):
                assert abs(O.overlap_bev(a, b) - F.turned_overlap(w, l, theta)) <= EXACT, (w, l, theta)


def boxes3d(X, z, dz):
    return np.stack([(X[:, 0] + X[:, 2]) / 2, (X[:, 1] + X[:, 3]) / 2, z, X[:, 2] - X[:, 0], X[:, 3] - X[:, 1], dz,
                     X[:, 4]], 1)


@pytest.mark.parametrize("name", ["slide", "nested", "touch_side", "corner_on_edge", "yaw_ulp", "zero_width"])
def test_iou3d_closed_forms(fams, name):
    A, B, ov, iou = fams[name]
    A, B, ov, iou = A[:400], B[:400], ov[:400], iou[:400]
    n = len(A)
    rng = np.random.default_rng(3)
    sa, sb = (A[:, 2] - A[:, 0]) * (A[:, 3] - A[:, 1]), (B[:, 2] - B[:, 0]) * (B[:, 3] - B[:, 1])
    za, dza = rng.uniform(-3, 1, n), rng.uniform(0.5, 3, n)
    dzb = rng.uniform(0.5, 3, n)
    h = rng.uniform(0, 1, n) * np.minimum(dza, dzb)
    cases = {                                                       # z of b -> height overlap
        "level": (za, dza, dza),
        "on top, touching": (za + dza, dzb, np.zeros(n)),
        "below, touching": (za - dzb, dzb, np.zeros(n)),
        "on top, overlapping": (za + dza - h, dzb, h),
        "below, overlapping": (za - dzb + h, dzb, h),
    }
    for case, (zb, dz_b, hh) in cases.items():
        got = O.iou3d_matrix(boxes3d(A, za, dza), boxes3d(B, zb, dz_b))
        ov3 = ov * hh
        want = ov3 / np.maximum(sa * dza + sb * dz_b - ov3, 1e-8)
        assert np.abs(np.diagonal(got) - want).max() <= EXACT, case
        if case == "level":
            assert np.abs(np.diagonal(got) - iou).max() <= EXACT   # equal heights: the BEV IoU


def test_iou3d_identical_zero_and_nan():
    b = np.array([[10.0, -4.0, -1.0, 1.95, 4.6, 1.7, 0.4], [0.0, 0.0, 0.0, 0.0, 2.0, 1.0, 0.0]])
    got = O.iou3d_matrix(b, b)
    assert abs(got[0, 0] - 1) <= EXACT and got[1, 1] == 0 and got[0, 1] == 0     # zero width: union clamped
    nan = b.copy()
    nan[0, 6] = np.nan
    assert O.iou3d_matrix(nan, b)[0, 0] == 0                          # a NaN box overlaps nothing


def test_iou3d_forms_corners_in_the_boxes_dtype():
    """fp32 boxes: x -+ dx / 2 is rounded to fp32 before the float64 overlap, as torch rounds it."""
    b = np.array([[60.123, -47.77, -1.3, 1.95, 4.6, 1.7, 0.4]], np.float32)
    assert O.xywhr2xyxyr(b).dtype == np.float32
    x1 = np.float64(b[0, 0] - b[0, 3] / np.float32(2))
    assert O.xywhr2xyxyr(b)[0, 0] == x1 and x1 != np.float64(b[0, 0]) - np.float64(b[0, 3]) / 2
    # a box with itself: the BEV overlap is the rounded corners' area, the volumes use dx and dy themselves
    c = O.xywhr2xyxyr(b)[0].astype(np.float64)
    ov = (c[2] - c[0]) * (c[3] - c[1]) * np.float64(b[0, 5])
    v = np.prod(b[0, 3:6].astype(np.float64))
    assert abs(O.iou3d_matrix(b, b)[0, 0] - ov / (2 * v - ov)) <= 1e-12
