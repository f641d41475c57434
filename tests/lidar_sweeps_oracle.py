"""numpy / torch restatement of LoadPointsFromMultiSweeps (mmdet3d/datasets/pipelines/loading.py:87-235) and
PointsRangeFilter (transforms_3d.py:585-614 with base_points.py:208-232), the checker of bevfusion_b200.lidar_sweeps.

The sweep transform is computed twice: with numpy's `@` as the reference writes it (loading.py:221-224), and as the
float64 FMA chain fl32(fma(p2, R[j][2], fma(p1, R[j][1], p0 * R[j][0]))) evaluated exactly with fractions.Fraction
(float(Fraction) rounds correctly).  A value where the two disagree after the fp32 store is a double-rounding case;
transform_both() reports them."""
from fractions import Fraction

import numpy as np
import torch


def remove_close(points, radius=1.0):
    """loading.py:152-170 on an [n, d] float32 array"""
    x_filt = np.abs(points[:, 0]) < radius
    y_filt = np.abs(points[:, 1]) < radius
    not_close = np.logical_not(np.logical_and(x_filt, y_filt))
    return points[not_close]


def transform_numpy(xyz, R, t):
    """loading.py:221-224: fp32 [n, 3] @ fp64 R.T, stored to fp32, += fp64 t, stored to fp32"""
    out = np.empty_like(xyz)
    out[:] = xyz @ np.asarray(R, np.float64).T
    out += np.asarray(t, np.float64)
    return out


def _fl(x):
    return float(x)  # Fraction -> nearest double


def transform_exact(xyz, R, t):
    """the same as the float64 FMA chain, each operation rounded once, in exact arithmetic"""
    R = [[Fraction(float(v)) for v in row] for row in np.asarray(R, np.float64)]
    t = [Fraction(float(v)) for v in np.asarray(t, np.float64)]
    out = np.empty_like(xyz)
    for i, (p0, p1, p2) in enumerate(xyz.tolist()):
        p0, p1, p2 = Fraction(p0), Fraction(p1), Fraction(p2)
        for j in range(3):
            a = _fl(p0 * R[j][0])
            b = _fl(p1 * R[j][1] + Fraction(a))
            c = _fl(p2 * R[j][2] + Fraction(b))
            out[i, j] = np.float32(_fl(Fraction(float(np.float32(c))) + t[j]))
    return out


def transform_both(xyz, R, t):
    """(numpy result, exact FMA-chain result, indices where they differ)"""
    a, b = transform_numpy(xyz, R, t), transform_exact(xyz, R, t)
    diff = np.nonzero(a.view(np.int32) != b.view(np.int32))
    return a, b, diff


def multi_sweeps(key_raw, sweeps_raw, rotations, translations, lags, use_dim, key_use_dim=None, sweeps_num=9,
                 pad_empty_sweeps=True, remove_close_on=True, point_cloud_range=None, exact=False):
    """key_raw [n, load_dim] as read from file, sweeps_raw the chosen sweeps in the order of `choices`.
    LoadPointsFromFile's use_dim (loading.py:405) then the sweep loader's (:187-188), then the sweeps (:189-231),
    then in_range_3d.  exact=True uses transform_exact instead of numpy's matmul."""
    load_dim = key_raw.shape[1]
    key_use_dim = list(range(load_dim)) if key_use_dim is None else list(key_use_dim)
    points = key_raw[:, key_use_dim][:, use_dim].copy()       # points[:, self.use_dim]
    points[:, 4] = 0                                          # points.tensor[:, 4] = 0
    parts = [points]
    if pad_empty_sweeps and len(sweeps_raw) == 0:
        for _ in range(sweeps_num):
            parts.append(remove_close(points) if remove_close_on else points)
    else:
        for raw, R, t, lag in zip(sweeps_raw, rotations, translations, lags):
            ps = np.copy(raw).reshape(-1, load_dim)
            if remove_close_on:
                ps = remove_close(ps)
            ps = ps[:, use_dim]
            if exact:
                ps[:, :3] = transform_exact(ps[:, :3], R, t)
            else:
                ps[:, :3] = ps[:, :3] @ np.asarray(R, np.float64).T
                ps[:, :3] += np.asarray(t, np.float64)
            ps[:, 4] = lag
            parts.append(ps)
    out = torch.from_numpy(np.concatenate(parts, 0))
    if point_cloud_range is not None:
        rng = np.array(point_cloud_range, dtype=np.float32)
        mask = ((out[:, 0] > rng[0]) & (out[:, 1] > rng[1]) & (out[:, 2] > rng[2])
                & (out[:, 0] < rng[3]) & (out[:, 1] < rng[4]) & (out[:, 2] < rng[5]))
        out = out[mask]
    return out.numpy()


def nuscenes_pose(rng, k):
    """a sensor2lidar rotation (small roll / pitch, yaw up to 0.1 rad) and translation of sweep k (ego motion about
    0.5 m per sweep), float64, like the nuScenes infos"""
    yaw, pitch, roll = rng.uniform(-0.1, 0.1), rng.uniform(-0.01, 0.01), rng.uniform(-0.01, 0.01)
    cz, sz, cy, sy, cx, sx = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch), np.cos(roll), np.sin(roll)
    R = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) \
        @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    t = np.array([-0.5 * k + rng.uniform(-0.05, 0.05), rng.uniform(-0.2, 0.2), rng.uniform(-0.02, 0.02)])
    return R, t


def nuscenes_sweep(rng, n, load_dim=5):
    """n raw rows of (x, y, z, intensity, ring, ...) float32: a 32-beam spin out to 70 m, some rows inside the
    remove_close square and some outside every range face"""
    r = rng.uniform(0.3, 70.0, n)
    az = rng.uniform(-np.pi, np.pi, n)
    pts = np.zeros((n, load_dim), np.float32)
    pts[:, 0], pts[:, 1] = r * np.cos(az), r * np.sin(az)
    pts[:, 2] = rng.uniform(-6.0, 4.0, n)
    pts[:, 3] = rng.uniform(0, 255, n).round()
    pts[:, 4] = rng.integers(0, 32, n)
    if load_dim > 5:
        pts[:, 5:] = rng.standard_normal((n, load_dim - 5))
    return pts
