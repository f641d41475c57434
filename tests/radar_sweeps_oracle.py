"""numpy / torch restatement of LoadRadarPointsMultiSweeps (mmdet3d/datasets/pipelines/loading.py:717-790, with
perform_encodings :629-653 and normalize_feats :711-715) and of the radar face of PointsRangeFilter
(transforms_3d.py:607-612, radar_points.py:92-107), the checker of bevfusion_b200.radar_sweeps.

The sweep's three transforms are computed twice: with numpy's `@` as the reference writes it (loading.py:749-764),
and as the float64 FMA chain fma(p2, R[j][2], fma(p1, R[j][1], fma(p0, R[j][0], +0))) evaluated exactly with
fractions.Fraction (float(Fraction) rounds correctly).  A value where the two disagree is a double-rounding case;
transforms_both() reports them."""
import os
from fractions import Fraction

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "radar_sweeps_tiny.npz")
GOLDEN_CASES = ("shipped", "nocomp", "norm", "all58")

ENCODING = [(3, "one-hot", 8), (11, "one-hot", 5), (14, "one-hot", 18), (15, "ordinal", 7), (0, "nusc-filter", 1)]
NORMALIZE_DIMS = [(3, 0, 50), (4, -100, 100), (5, -100, 100)]
BEV_RANGE = [-55.0, -55.0, 55.0, 55.0]
SHIPPED_USE_DIM = [0, 1, 2, 5, 8, 9] + list(range(18, 57))


def _chain(p, R, j):
    """fma(p2, R[j][2], fma(p1, R[j][1], fma(p0, R[j][0], +0.0))) for finite doubles, each fma rounded once; a zero
    result of x*y + acc is -0.0 iff x*y and acc are both -0.0 (IEEE, round to nearest)"""
    acc = 0.0
    for k in range(3):
        prod = Fraction(p[k]) * Fraction(float(R[j][k]))
        s = prod + Fraction(acc)
        if s == 0:
            prod_neg = prod == 0 and (np.signbit(p[k]) != np.signbit(float(R[j][k])))
            acc = -0.0 if (prod_neg and np.signbit(acc)) else 0.0
        else:
            acc = float(s)
    return acc


def transforms_numpy(raw, R, t, compensate_velocity, time_diff):
    """loading.py:744-772 as written: (xyz fp32 [n, 3] after += t and the compensation, velo [n, 2], velo_comp
    [n, 2])"""
    ps = np.copy(raw).reshape(-1, 18)
    td = np.ones((ps.shape[0], 1)) * time_diff
    velo_comp = np.concatenate((ps[:, 8:10], np.zeros((ps.shape[0], 1))), 1) @ np.asarray(R).T
    velo = np.concatenate((ps[:, 6:8], np.zeros((ps.shape[0], 1))), 1) @ np.asarray(R).T
    ps[:, :3] = ps[:, :3] @ np.asarray(R).T
    ps[:, :3] += np.asarray(t)
    if compensate_velocity:
        ps[:, :2] += velo_comp[:, :2] * td
    return ps[:, :3], velo[:, :2], velo_comp[:, :2]


def transforms_exact(raw, R, t, compensate_velocity, time_diff):
    """the same as the FMA chains, each float64 operation rounded once, in exact arithmetic"""
    n = raw.shape[0]
    xyz, velo, comp = np.empty((n, 3), np.float32), np.empty((n, 2)), np.empty((n, 2))
    for i in range(n):
        r = [float(v) for v in raw[i]]
        for j in range(3):
            a = np.float32(_chain(r[0:3], R, j))
            xyz[i, j] = np.float32(float(a) + float(t[j]))
        for j in range(2):
            velo[i, j] = _chain([r[6], r[7], 0.0], R, j)
            comp[i, j] = _chain([r[8], r[9], 0.0], R, j)
        if compensate_velocity:
            for j in range(2):
                xyz[i, j] = np.float32(float(xyz[i, j]) + comp[i, j] * time_diff)
    return xyz, velo, comp


def transforms_both(raw, R, t, compensate_velocity=True, time_diff=0.05):
    """(disagreements between numpy and the exact chains, counted over xyz, velo and velo_comp)"""
    a, b = transforms_numpy(raw, R, t, compensate_velocity, time_diff), \
        transforms_exact(raw, R, t, compensate_velocity, time_diff)
    return sum(int((x.view(np.int32 if x.dtype == np.float32 else np.int64)
                    != y.view(np.int32 if y.dtype == np.float32 else np.int64)).sum()) for x, y in zip(a, b))


def load_sweep(raw, R, t, time_diff, compensate_velocity, exact=False):
    """loading.py:741-772: one raw [n, 18] fp32 sweep -> its 19-column float64 rows"""
    ps = np.copy(raw).reshape(-1, 18)
    td = np.ones((ps.shape[0], 1)) * time_diff
    f = transforms_exact if exact else transforms_numpy
    xyz, velo, velo_comp = f(raw, R, t, compensate_velocity, time_diff)
    ps[:, :3] = xyz
    return np.concatenate([ps[:, :6], velo, velo_comp, ps[:, 10:], td], axis=1)


def perform_encodings(points, bad_category="raise"):
    """loading.py:629-653.  bad_category="zero": a one-hot source that is NaN or rounds outside [-w, w), where the
    reference raises IndexError, leaves that row's block zero instead (the device's documented behaviour)."""
    for idx, kind, dims in ENCODING:
        feat = points[:, idx]
        encoding = np.zeros((points.shape[0], dims))
        if kind == "one-hot":
            r = np.rint(feat)
            if bad_category == "raise":
                with np.errstate(invalid="ignore"):
                    encoding[np.arange(feat.shape[0]), r.astype(int)] = 1
            else:
                ok = (r >= -dims) & (r < dims)
                rows = np.nonzero(ok)[0]
                encoding[rows, r[rows].astype(int)] = 1
        elif kind == "ordinal":
            for i in range(dims):
                encoding[:, i] = (np.rint(feat) > i).astype(int)
        else:
            mask = (points[:, 14] == 0) & (points[:, 3] < 7) & (points[:, 11] == 3)
            encoding[mask, 0] = 1
        points = np.concatenate([points, encoding], axis=1)
    return points


def normalize_feats(points, normalize_dims):
    for dim, mn, mx in normalize_dims:
        points[:, dim] -= mn
        points[:, dim] /= (mx - mn)
    return points


def in_range_bev(tensor, point_range):
    return ((tensor[:, 0] > point_range[0]) & (tensor[:, 1] > point_range[1]) & (tensor[:, 0] < point_range[2])
            & (tensor[:, 1] < point_range[3]))


def multi_sweeps(raws, rotations, translations, time_diffs, use_dim, compensate_velocity=True, normalize=False,
                 normalize_dims=NORMALIZE_DIMS, bev_range=BEV_RANGE, exact=False, bad_category="raise"):
    """the sweeps of one sample in concatenation order -> the [n, len(use_dim)] fp32 cloud after PointsRangeFilter's
    radar face (bev_range None: before it)"""
    parts = [load_sweep(r, R, t, td, compensate_velocity, exact)
             for r, R, t, td in zip(raws, rotations, translations, time_diffs)]
    points = np.concatenate(parts, axis=0)
    points = perform_encodings(points, bad_category)
    points = points[:, use_dim]
    if normalize:
        with np.errstate(divide="ignore", invalid="ignore"):
            points = normalize_feats(points, normalize_dims)
    out = torch.as_tensor(points, dtype=torch.float32)
    if bev_range is not None:
        out = out[in_range_bev(out, bev_range)]
    return out.numpy()


def radar_pose(rng, k):
    """a nuScenes-like sensor2lidar pose of radar k: yaw around the car, small pitch / roll, mounted ~0.5-3.5 m out"""
    yaw = k * 2 * np.pi / 5 + rng.uniform(-0.3, 0.3)
    pitch, roll = rng.uniform(-0.02, 0.02), rng.uniform(-0.02, 0.02)
    cz, sz, cy, sy, cx, sx = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch), np.cos(roll), np.sin(roll)
    R = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) \
        @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    t = np.array([3.4 * np.cos(yaw) + rng.uniform(-0.1, 0.1), 1.0 * np.sin(yaw), 0.5 + rng.uniform(-0.05, 0.05)])
    return R, t


def radar_sweep(rng, n):
    """n raw radar rows (x y z dyn_prop id rcs vx vy vx_comp vy_comp is_quality_valid ambig_state x_rms y_rms
    invalid_state pdh0 vx_rms vy_rms), float32, as the nuScenes devkit reads them with filtering 'none'"""
    pts = np.zeros((n, 18), np.float32)
    r = rng.uniform(0.5, 80.0, n)
    az = rng.uniform(-1.0, 1.0, n)
    pts[:, 0], pts[:, 1] = r * np.cos(az), r * np.sin(az)
    pts[:, 2] = rng.uniform(-0.5, 1.5, n)
    pts[:, 3] = rng.integers(0, 8, n)
    pts[:, 4] = rng.integers(0, 120, n)
    pts[:, 5] = rng.uniform(-10, 40, n).round(1)
    pts[:, 6:10] = rng.normal(0, 5, (n, 4))
    pts[:, 10] = rng.integers(0, 2, n)
    pts[:, 11] = rng.integers(0, 5, n)
    pts[:, 12:14] = rng.integers(0, 32, (n, 2))
    pts[:, 14] = np.where(rng.random(n) < 0.7, 0, rng.integers(0, 18, n))
    pts[:, 15] = rng.integers(0, 8, n)
    pts[:, 16:18] = rng.integers(0, 32, (n, 2))
    return pts


def golden_case(z, case):
    """the inputs of one case of golden/radar_sweeps_tiny.npz, as multi_sweeps' keyword arguments"""
    counts = z[case + "_counts"]
    raws = np.split(z[case + "_raw"], np.cumsum(counts)[:-1])
    sweeps_num, comp, norm = (int(v) for v in z[case + "_flags"])
    return dict(raws=raws, rotations=list(z[case + "_rot"]), translations=list(z[case + "_trans"]),
                time_diffs=list(z[case + "_lag"]), use_dim=[int(c) for c in z[case + "_use_dim"]],
                compensate_velocity=bool(comp), normalize=bool(norm))
