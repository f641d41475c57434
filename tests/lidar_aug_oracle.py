"""Restatement of GlobalRotScaleTrans + RandomFlip3D + PointsRangeFilter + ObjectRangeFilter + ObjectNameFilter
(transforms_3d.py:195-232, 323-353, 534-636) on LiDARPoints, RadarPoints and LiDARInstance3DBoxes (base_points.py,
radar_points.py, lidar_points.py, base_box3d.py, lidar_box3d.py, utils.py:6-19), the checker of
bevfusion_b200.lidar_aug.

Every transform is written twice:
  exact=False  the reference's own torch CPU lines on plain tensors: `t[:, :3] = t[:, :3] @ rot_mat_T` on the strided
               view, `+= new_tensor(translation)`, `*= scale`, the flips, limit_period;
  exact=True   what the device evaluates: each output of a matmul is the fp32 FMA chain
               fma(p2, R[2][j], fma(p1, R[1][j], fma(p0, R[0][j], +0))) (all terms, the zero entries included),
               emulated in numpy with float64 round-to-odd (fma32), and every other operation one fp32 rounding.
The sines and cosines are torch's, computed once on the host in both forms: the device never evaluates them.
count_diff() counts the values where two results disagree (NaN equal to NaN, signed zeros distinct)."""
import hashlib
from fractions import Fraction

import numpy as np
import torch

SHIPPED_SCALE = [0.9, 1.1]                       # configs/nuscenes/default.yaml augment3d
SHIPPED_ROTATE = [-0.78539816, 0.78539816]
SHIPPED_TRANSLATE = 0.5
POINT_CLOUD_RANGE = [-54.0, -54.0, -5.0, 54.0, 54.0, 3.0]   # the transfusion camera+lidar config
OBJECT_CLASSES = ["car", "truck", "construction_vehicle", "bus", "trailer", "barrier", "motorcycle", "bicycle",
                  "pedestrian", "traffic_cone"]
RADAR_DIM = 45                                   # len(radar_use_dims) of configs/nuscenes/det/default.yaml
PI32 = np.float32(np.pi)
TWO_PI32 = np.float32(2 * np.pi)

f32, f64 = np.float32, np.float64


# ---- draws ------------------------------------------------------------------------------------------------------
def draw_tuple(draw):
    """(scale, theta, translation [3], flip_horizontal, flip_vertical) from a golden [7] row; scale NaN = no
    GlobalRotScaleTrans draw (is_train False)"""
    d = np.asarray(draw, np.float64)
    scale = None if np.isnan(d[0]) else float(d[0])
    return scale, float(d[1]), d[2:5].copy(), int(d[5]), int(d[6])


def rot_mats(theta):
    """(rot_mat_T of BasePoints.rotate(-theta), rot_mat_T of LiDARInstance3DBoxes.rotate(theta), fl32(theta)), as
    float32 [3, 3] numpy arrays, computed with the reference's torch CPU calls"""
    a = torch.tensor(-theta, dtype=torch.float32)
    s, c = torch.sin(a), torch.cos(a)
    pts = a.new_tensor([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T.contiguous()
    b = torch.tensor(theta, dtype=torch.float32)
    s, c = torch.sin(b), torch.cos(b)
    box = b.new_tensor([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    return pts.numpy(), box.numpy(), b.numpy()


# ---- the exact fp32 arithmetic ----------------------------------------------------------------------------------
def fma32(a, b, c):
    """fl32(a * b + c) rounded once, elementwise, for float32 arrays: a * b is exact in float64, the sum is taken in
    float64 with round-to-odd (which makes the second rounding to fp32 correct), then stored to fp32"""
    with np.errstate(all="ignore"):
        a, b, c = np.broadcast_arrays(np.asarray(a, f32), np.asarray(b, f32), np.asarray(c, f32))
        p = a.astype(f64) * b.astype(f64)
        s = p + c.astype(f64)
        bb = s - p
        e = (p - (s - bb)) + (c.astype(f64) - bb)       # TwoSum: the exact sum is s + e
        fix = np.isfinite(s) & np.isfinite(e) & (e != 0) & ((s.view(np.int64) & 1) == 0)
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
        return s.astype(f32)


def fma32_fraction(a, b, c):
    """the same for finite scalars, in exact rational arithmetic (the check of fma32)"""
    x = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    if x == 0:   # IEEE: -0 only for (-0 product) + (-0)
        neg_product = (a == 0 or b == 0) and bool(np.signbit(a)) != bool(np.signbit(b))
        return f32(-0.0) if neg_product and c == 0 and np.signbit(c) else f32(0.0)
    d = f32(float(x))
    cands = [d, np.nextafter(d, f32(np.inf)), np.nextafter(d, f32(-np.inf))]
    return min(cands, key=lambda v: (abs(Fraction(float(v)) - x), int(np.array(v, f32).view(np.int32)) & 1))


def chain(cols, R, exact):
    """[n, k] @ R [k, m] in fp32: torch's matmul (exact=False) or the FMA chain from +0 in k order (exact=True)"""
    if not exact:
        return (torch.from_numpy(np.ascontiguousarray(cols)) @ torch.from_numpy(R)).numpy()
    out = np.empty((cols.shape[0], R.shape[1]), f32)
    for j in range(R.shape[1]):
        acc = np.zeros(cols.shape[0], f32)
        for k in range(R.shape[0]):
            acc = fma32(cols[:, k], R[k, j], acc)
        out[:, j] = acc
    return out


# ---- the transforms ---------------------------------------------------------------------------------------------
def augment_points(points, draw, exact=False):
    """LiDARPoints: rotate(-theta), translate, scale, flip h, flip v ([n, d] fp32, copied)"""
    scale, theta, trans, fh, fv = draw
    t = torch.from_numpy(np.array(points, f32, copy=True))
    if scale is not None:
        R = rot_mats(theta)[0]
        if exact:
            x = t.numpy()
            x[:, :3] = chain(x[:, :3], R, True)
            x[:, :3] += f32(trans)
            x[:, :3] *= f32(scale)
        else:
            t[:, :3] = t[:, :3] @ torch.from_numpy(R)
            t[:, :3] += t.new_tensor(trans)
            t[:, :3] *= scale
    if fh:
        t[:, 1] = -t[:, 1]
    if fv:
        t[:, 0] = -t[:, 0]
    return t.numpy()


def augment_radar(radar, draw, exact=False):
    """RadarPoints: columns 0:3 as LiDAR's, columns 3:5 rotated by rot_mat_T[:2, :2] and scaled; flip h negates
    columns 1 and 4, flip v columns 0 and 3"""
    scale, theta, trans, fh, fv = draw
    t = torch.from_numpy(np.array(radar, f32, copy=True))
    if scale is not None:
        R = rot_mats(theta)[0]
        if exact:
            x = t.numpy()
            x[:, :3] = chain(x[:, :3], R, True)
            x[:, 3:5] = chain(x[:, 3:5], np.ascontiguousarray(R[:2, :2]), True)
            x[:, :3] += f32(trans)
            x[:, :3] *= f32(scale)
            x[:, 3:5] *= f32(scale)
        else:
            Rt = torch.from_numpy(R)
            t[:, :3] = t[:, :3] @ Rt
            t[:, 3:5] = t[:, 3:5] @ Rt[:2, :2]
            t[:, :3] += t.new_tensor(trans)
            t[:, :3] *= scale
            t[:, 3:5] *= scale
    if fh:
        t[:, 1] = -t[:, 1]
        t[:, 4] = -t[:, 4]
    if fv:
        t[:, 0] = -t[:, 0]
        t[:, 3] = -t[:, 3]
    return t.numpy()


def augment_boxes(boxes, draw, exact=False):
    """LiDARInstance3DBoxes [n, 7 | 9]: rotate(theta) (xyz, yaw += fl32(theta), velocity), translate, scale
    (columns :6 and 7:), flip h (columns 1::7, yaw = -yaw + pi), flip v (columns 0::7, yaw = -yaw)"""
    scale, theta, trans, fh, fv = draw
    t = torch.from_numpy(np.array(boxes, f32, copy=True))
    D = t.shape[1]
    if scale is not None:
        _, R, yaw = rot_mats(theta)
        if exact:
            x = t.numpy()
            x[:, :3] = chain(x[:, :3], R, True)
            x[:, 6] += yaw
            if D == 9:
                x[:, 7:9] = chain(x[:, 7:9], np.ascontiguousarray(R[:2, :2]), True)
            x[:, :3] += f32(trans)
            x[:, :6] *= f32(scale)
            x[:, 7:] *= f32(scale)
        else:
            Rt = torch.from_numpy(R)
            t[:, :3] = t[:, :3] @ Rt
            t[:, 6] += torch.from_numpy(yaw)
            if D == 9:
                t[:, 7:9] = t[:, 7:9] @ Rt[:2, :2]
            t[:, :3] += t.new_tensor(trans)
            t[:, :6] *= scale
            t[:, 7:] *= scale
    if fh:
        t[:, 1::7] = -t[:, 1::7]
        if exact:
            t.numpy()[:, 6] = -t.numpy()[:, 6] + PI32
        else:
            t[:, 6] = -t[:, 6] + np.pi
    if fv:
        t[:, 0::7] = -t[:, 0::7]
        t[:, 6] = -t[:, 6]
    return t.numpy()


def limit_yaw(boxes, exact=False):
    """limit_yaw(offset=0.5, period=2 * pi): yaw - floor(yaw / fl32(2 pi) + 0.5) * fl32(2 pi), each step in fp32"""
    b = np.array(boxes, f32, copy=True)
    if exact:
        with np.errstate(all="ignore"):
            y = b[:, 6]
            b[:, 6] = y - np.floor(y / TWO_PI32 + f32(0.5)) * TWO_PI32
    else:
        t = torch.from_numpy(b)
        t[:, 6] = t[:, 6] - torch.floor(t[:, 6] / (2 * np.pi) + 0.5) * (2 * np.pi)
    return b


def in_range_3d(points, rng):
    r = np.asarray(rng, f32)
    with np.errstate(invalid="ignore"):
        return ((points[:, 0] > r[0]) & (points[:, 1] > r[1]) & (points[:, 2] > r[2]) & (points[:, 0] < r[3])
                & (points[:, 1] < r[4]) & (points[:, 2] < r[5]))


def in_range_bev(xy, rng):
    r = np.asarray(rng, f32)
    with np.errstate(invalid="ignore"):
        return (xy[:, 0] > r[0]) & (xy[:, 1] > r[1]) & (xy[:, 0] < r[2]) & (xy[:, 1] < r[3])


RADAR_BEV_RANGE = [-55.0, -55.0, 55.0, 55.0]     # PointsRangeFilter's radar face (transforms_3d.py:610)


def boxes_filtered(boxes, labels, draw, point_cloud_range=POINT_CLOUD_RANGE, num_classes=len(OBJECT_CLASSES),
                   exact=False):
    """augment_boxes, then ObjectRangeFilter (strict fp32 in_range_bev, then limit_yaw) and ObjectNameFilter"""
    b = augment_boxes(boxes, draw, exact)
    r = np.asarray(point_cloud_range, f32)[[0, 1, 3, 4]]
    keep = in_range_bev(b[:, :2], r)
    b = limit_yaw(b[keep], exact)
    lab = np.asarray(labels)[keep]
    named = (lab >= 0) & (lab < num_classes)
    return b[named], lab[named]


def pipeline(points, radar, boxes, labels, masks, draw, point_cloud_range=POINT_CLOUD_RANGE,
             num_classes=len(OBJECT_CLASSES), exact=False):
    """one sample through the five transforms: (points, radar, boxes, labels, masks)"""
    p = augment_points(points, draw, exact)
    p = p[in_range_3d(p, point_cloud_range)]
    r = augment_radar(radar, draw, exact)
    r = r[in_range_bev(r[:, :2], RADAR_BEV_RANGE)]
    b, lab = boxes_filtered(boxes, labels, draw, point_cloud_range, num_classes, exact)
    m = np.asarray(masks)
    if draw[3]:
        m = m[:, :, ::-1]
    if draw[4]:
        m = m[:, ::-1, :]
    return p, r, b, lab, np.ascontiguousarray(m)


def lidar_aug_matrix(draw):
    """the reference's lidar_aug_matrix: GlobalRotScaleTrans' rotation.T * scale and translation * scale in
    float64 stored to fp32, then RandomFlip3D's rotation @ m[:3, :]"""
    scale, theta, trans, fh, fv = draw
    m = np.eye(4).astype(np.float32)
    if scale is not None:
        rotation = np.eye(3) @ rot_mats(theta)[1]
        m[:3, :3] = rotation.T * scale
        m[:3, 3] = np.asarray(trans) * scale
    rotation = np.eye(3)
    if fh:
        rotation = np.array([[1, 0, 0], [0, -1, 0], [0, 0, 1]]) @ rotation
    if fv:
        rotation = np.array([[-1, 0, 0], [0, 1, 0], [0, 0, 1]]) @ rotation
    m[:3, :] = rotation @ m[:3, :]
    return m


# ---- inputs -----------------------------------------------------------------------------------------------------
def sample_inputs(rng, n_points, n_radar, n_boxes):
    """(points [n, 5], radar [m, 45], boxes [k, 9], labels [k] int64 with -1 entries, masks [6, 16, 24] bool):
    nuScenes-like values reaching past every range face"""
    points = np.empty((n_points, 5), f32)
    points[:, :2] = rng.uniform(-62, 62, (n_points, 2))
    points[:, 2] = rng.uniform(-6, 4, n_points)
    points[:, 3] = rng.integers(0, 256, n_points)
    points[:, 4] = 0.0                                     # the key's time column
    radar = np.zeros((n_radar, RADAR_DIM), f32)
    radar[:, :2] = rng.uniform(-64, 64, (n_radar, 2))
    radar[:, 2] = rng.uniform(-1, 2, n_radar)
    radar[:, 3] = rng.uniform(-5, 40, n_radar)            # rcs
    radar[:, 4:6] = rng.normal(0, 6, (n_radar, 2))         # vx_comp, vy_comp
    radar[:, 6:] = rng.integers(0, 2, (n_radar, RADAR_DIM - 6))
    boxes = np.empty((n_boxes, 9), f32)
    boxes[:, :2] = rng.uniform(-60, 60, (n_boxes, 2))
    boxes[:, 2] = rng.uniform(-3, 1, n_boxes)
    boxes[:, 3:6] = rng.uniform(0.3, 12, (n_boxes, 3))
    boxes[:, 6] = rng.uniform(-np.pi, np.pi, n_boxes)
    boxes[:, 7:9] = rng.normal(0, 5, (n_boxes, 2))
    labels = rng.integers(-1, 10, n_boxes).astype(np.int64)
    masks = rng.random((6, 16, 24)) < 0.3
    return points, radar, boxes, labels, masks


def bulk_draws():
    """draws for the bulk check: the shipped limits, zero and limit angles, scale 1, every flip pair"""
    rng = np.random.default_rng(77)
    draws = []
    for k in range(8):
        theta = [0.0, SHIPPED_ROTATE[0], SHIPPED_ROTATE[1], np.pi, -np.pi / 2][k] if k < 5 else \
            float(rng.uniform(*SHIPPED_ROTATE))
        scale = 1.0 if k == 0 else float(rng.uniform(*SHIPPED_SCALE))
        trans = rng.normal(0, SHIPPED_TRANSLATE, 3) if k else np.zeros(3)
        draws.append((scale, theta, trans, k & 1, (k >> 1) & 1))
    return draws


def bulk_inputs(rows=12500):
    """(draw, points [rows, 5], radar [rows, 45], boxes7 [rows // 2, 7], boxes9 [rows, 9]) per bulk draw: 8 draws,
    so 10^5 LiDAR, radar and 9-column box rows; some rows hold +-0, +-inf, NaN, subnormals and +-pi yaws"""
    rng = np.random.default_rng(1234)
    for draw in bulk_draws():
        points, radar, boxes, _, _ = sample_inputs(rng, rows, rows, rows)
        special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-40, -1e-40, 3e38], f32)
        for a in (points, radar, boxes):
            idx = rng.integers(0, rows, 64)
            col = rng.integers(0, 5, 64)
            a[idx, col] = special[rng.integers(0, len(special), 64)]
        boxes[:8, 6] = [np.pi, -np.pi, PI32, -PI32, 3 * np.pi, np.nextafter(PI32, f32(0)), 0.0, -0.0]
        yield draw, points, radar, np.ascontiguousarray(boxes[:rows // 2, :7]), boxes


def canonical(a):
    """a copy with every NaN replaced by one quiet NaN (payloads and signs of NaNs are not compared)"""
    a = np.array(a, f32, copy=True)
    a[np.isnan(a)] = np.nan
    return a


def sha256_of(arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(canonical(a)).tobytes())
    return h.digest()


def count_diff(a, b):
    """values where a and b differ: bits compared, every NaN equal to every NaN; a shape mismatch counts all"""
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    if a.shape != b.shape:
        return max(a.size, b.size, 1)
    same = (a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))
    return int((~same).sum())
