"""Float64 checker of bevfusion_b200.iou3d, written from the geometry (numpy only, no GPU):

    iou_bev(a, b) / overlap_bev(a, b)   rotated BEV IoU / overlap of two [x1, y1, x2, y2, ry] boxes: one
                                        rotated rectangle clipped by the other (Sutherland-Hodgman)
    iou_matrix(A, B)                    [M, N] of the above (pairs whose circumscribed circles are apart
                                        are 0 without clipping)
    iou3d_matrix(A, B)                  [M, N] 3D IoU of (x, y, z, dx, dy, dz, yaw) boxes, z the bottom
    greedy(iou, thresh)                 greedy keep list of score-sorted boxes given their IoU matrix
    nms(boxes, scores, thresh, pre, post)   nms_gpu's result (indices into boxes)
    circle_nms(dets, thresh, post)      circle NMS, squared distance <= thresh
    check_greedy(iou, keep, thresh, delta)  a keep list is a valid greedy NMS under tolerance delta

A box turned by r maps (x, y) to ((x-cx) cos r + (y-cy) sin r + cx, -(x-cx) sin r + (y-cy) cos r + cy),
the reference's convention (iou3d_kernel.cu:116-124).  IoU = overlap / max(sa + sb - overlap, 1e-8) with
sa, sb the unrotated extents' areas.  A box with a NaN coordinate overlaps nothing (IoU 0)."""
import numpy as np


def corners(box):
    x1, y1, x2, y2, r = [float(v) for v in box]
    cx, cy = (x1 + x2) / 2, (y1 + y2) / 2
    c, s = np.cos(r), np.sin(r)
    out = []
    for x, y in ((x1, y1), (x2, y1), (x2, y2), (x1, y2)):     # counter-clockwise; a rotation keeps that
        dx, dy = x - cx, y - cy
        out.append((dx * c + dy * s + cx, -dx * s + dy * c + cy))
    return out


def _area(poly):
    if len(poly) < 3:
        return 0.0
    a = 0.0
    for i in range(len(poly)):
        x0, y0 = poly[i]
        x1, y1 = poly[(i + 1) % len(poly)]
        a += x0 * y1 - x1 * y0
    return abs(a) / 2


def _clip(poly, e0, e1):
    """Keep the part of poly on the left of the directed line e0 -> e1."""
    def side(p):
        return (e1[0] - e0[0]) * (p[1] - e0[1]) - (e1[1] - e0[1]) * (p[0] - e0[0])
    out = []
    for i in range(len(poly)):
        p, q = poly[i], poly[(i + 1) % len(poly)]
        sp, sq = side(p), side(q)
        if sp >= 0:
            out.append(p)
        if (sp >= 0) != (sq >= 0):
            t = sp / (sp - sq)
            out.append((p[0] + t * (q[0] - p[0]), p[1] + t * (q[1] - p[1])))
    return out


def _apart(a, b):
    ra = 0.5 * np.hypot(a[2] - a[0], a[3] - a[1])
    rb = 0.5 * np.hypot(b[2] - b[0], b[3] - b[1])
    d = np.hypot((a[0] + a[2] - b[0] - b[2]) / 2, (a[1] + a[3] - b[1] - b[3]) / 2)
    return d > ra + rb


def overlap_bev(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if not (np.isfinite(a).all() and np.isfinite(b).all()) or _apart(a, b):
        return 0.0
    if (a[2] - a[0]) * (a[3] - a[1]) == 0 or (b[2] - b[0]) * (b[3] - b[1]) == 0:
        return 0.0                                  # exactly: clipping noise over a union of 1e-8 would not be
    poly = corners(a)
    cb = corners(b)
    for k in range(4):
        poly = _clip(poly, cb[k], cb[(k + 1) % 4])
        if not poly:
            return 0.0
    return _area(poly)


def iou_bev(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    ov = overlap_bev(a, b)
    sa = (a[2] - a[0]) * (a[3] - a[1])
    sb = (b[2] - b[0]) * (b[3] - b[1])
    u = sa + sb - ov
    return ov / (u if u > 1e-8 else 1e-8)


def iou_matrix(A, B, overlap=False):
    A, B = np.asarray(A, np.float64).reshape(-1, 5), np.asarray(B, np.float64).reshape(-1, 5)
    out = np.zeros((len(A), len(B)))
    if len(A) == 0 or len(B) == 0:
        return out
    ca, cb = (A[:, :2] + A[:, 2:4]) / 2, (B[:, :2] + B[:, 2:4]) / 2
    ra = 0.5 * np.hypot(A[:, 2] - A[:, 0], A[:, 3] - A[:, 1])
    rb = 0.5 * np.hypot(B[:, 2] - B[:, 0], B[:, 3] - B[:, 1])
    d = np.hypot(ca[:, None, 0] - cb[None, :, 0], ca[:, None, 1] - cb[None, :, 1])
    with np.errstate(invalid="ignore"):
        cand = ~(d > ra[:, None] + rb[None, :])        # NaN boxes stay candidates and give 0 below
    fn = overlap_bev if overlap else iou_bev
    for i, j in zip(*np.nonzero(cand)):
        out[i, j] = fn(A[i], B[j])
    return out


def xywhr2xyxyr(boxes):
    """[N, 7+] (x, y, z, dx, dy, dz, yaw, ...) boxes -> [N, 5] BEV [x1, y1, x2, y2, ry], in the boxes' own dtype
    (LiDARInstance3DBoxes.bev, then xywhr2xyxyr as torch computes it)."""
    b = np.asarray(boxes)
    hx, hy = b[:, 3] / 2, b[:, 4] / 2
    return np.stack([b[:, 0] - hx, b[:, 1] - hy, b[:, 0] + hx, b[:, 1] + hy, b[:, 6]], 1)


def iou3d_matrix(A, B):
    """[M, N] 3D IoU of (x, y, z, dx, dy, dz, yaw) boxes with z the bottom, as BaseInstance3DBoxes.overlaps
    (mode iou) defines it: the BEV overlap of the xyxyr boxes times the overlap of [z, z + dz], over
    max(va + vb - overlap, 1e-8).  The xyxyr corners and the tops z + dz are formed in the boxes' own dtype, as the
    reference's torch code forms them; everything after that is float64."""
    A, B = np.asarray(A).reshape(-1, np.shape(A)[-1]), np.asarray(B).reshape(-1, np.shape(B)[-1])
    bev = iou_matrix(xywhr2xyxyr(A), xywhr2xyxyr(B), overlap=True)
    top_a, top_b = (A[:, 2] + A[:, 5]).astype(np.float64), (B[:, 2] + B[:, 5]).astype(np.float64)
    A, B = A.astype(np.float64), B.astype(np.float64)
    h = np.minimum(top_a[:, None], top_b[None, :]) - np.maximum(A[:, None, 2], B[None, :, 2])
    ov = bev * np.where(h < 0, 0.0, h)                          # clamp(min=0); NaN stays
    va, vb = A[:, 3] * A[:, 4] * A[:, 5], B[:, 3] * B[:, 4] * B[:, 5]
    u = va[:, None] + vb[None, :] - ov
    return ov / np.where(u < 1e-8, 1e-8, u)


def greedy(iou, thresh):
    """Greedy NMS over boxes sorted by descending score: row i is dropped when iou[k, i] > thresh for an
    earlier kept k (the reference's host loop, iou3d.cpp:132-145)."""
    n = iou.shape[0]
    removed = np.zeros(n, bool)
    keep = []
    for i in range(n):
        if removed[i]:
            continue
        keep.append(i)
        removed[i + 1:] |= iou[i, i + 1:] > thresh
    return keep


def sort_desc(scores):
    return np.argsort(-np.asarray(scores, np.float64), kind="stable")


def nms(boxes, scores, thresh, pre_max_size=None, post_max_size=None):
    order = sort_desc(scores)
    if pre_max_size is not None:
        order = order[:pre_max_size]
    b = np.asarray(boxes, np.float64)[order]
    keep = order[greedy(iou_matrix(b, b), thresh)]
    return keep if post_max_size is None else keep[:post_max_size]


def circle_nms(dets, thresh, post_max_size=83):
    """Indices of the kept detections of dets [N, 3] (x, y, score): a detection is dropped when a kept,
    higher-scored centre lies at squared distance <= thresh (box3d_nms.py:180-219)."""
    dets = np.asarray(dets, np.float64)
    order = sort_desc(dets[:, 2])
    xy = dets[order, :2]
    d2 = ((xy[:, None, :] - xy[None, :, :]) ** 2).sum(-1)
    n = len(order)
    removed = np.zeros(n, bool)
    keep = []
    for i in range(n):
        if removed[i]:
            continue
        keep.append(i)
        removed[i + 1:] |= d2[i, i + 1:] <= thresh
    return order[np.array(keep, int)][:post_max_size]


def check_greedy(iou, keep, thresh, delta):
    """keep (sorted positions, ascending, not cut by a post_max) is a greedy NMS of the score-sorted boxes
    whose float64 IoU matrix is iou, up to delta: every kept box has IoU <= thresh + delta with each earlier
    kept box, and every dropped box has IoU > thresh - delta with some earlier kept box.  Returns the list
    of violations (empty when valid)."""
    bad = []
    keep = [int(k) for k in keep]
    if keep != sorted(set(keep)) or (keep and (keep[0] < 0 or keep[-1] >= iou.shape[0])):
        return [("keep list not ascending / out of range", keep)]
    kset, prev = set(keep), []
    for i in range(iou.shape[0]):
        hits = iou[prev, i] if prev else np.zeros(0)
        if i in kset:
            if (hits > thresh + delta).any():
                bad.append(("kept but overlapped", i))
            prev.append(i)
        elif not (hits > thresh - delta).any():
            bad.append(("dropped without cause", i))
    return bad
