"""CPU: the restatement of LoadPointsFromMultiSweeps + PointsRangeFilter (tests/lidar_sweeps_oracle.py) -- its numpy
and exact FMA-chain transforms agree on seeded nuScenes-like sweeps; choose_sweeps draws what the reference draws;
pad entries, key column maps, remove_close, range faces and NaN rows; the parameter block the device reads; the C
declarations, the workspace query and the argument checks made before any device work."""
import re

import numpy as np
import pytest
import torch

import lidar_sweeps_oracle as O

PCR = [-54.0, -54.0, -5.0, 54.0, 54.0, 3.0]     # voxelnet 0.075


def reference_choices(n, sweeps_num, test_mode):
    """loading.py:196-210 as written (load_augmented None)"""
    if n <= sweeps_num:
        return np.arange(n)
    elif test_mode:
        return np.arange(sweeps_num)
    return np.random.choice(n, sweeps_num, replace=False)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_numpy_and_fma_chain_transforms_agree(seed):
    rng = np.random.default_rng(seed)
    double_roundings = 0
    for k in range(1, 4):
        xyz = O.nuscenes_sweep(rng, 1500)[:, :3]
        R, t = O.nuscenes_pose(rng, k)
        a, b, diff = O.transform_both(xyz, R, t)
        double_roundings += len(diff[0])
    assert double_roundings == 0


def test_oracle_exact_mode_equals_numpy_mode():
    rng = np.random.default_rng(7)
    key = O.nuscenes_sweep(rng, 400)
    sweeps = [O.nuscenes_sweep(rng, 300 + 50 * k) for k in range(3)]
    poses = [O.nuscenes_pose(rng, k + 1) for k in range(3)]
    args = (key, sweeps, [p[0] for p in poses], [p[1] for p in poses], [0.05, 0.1, 0.15], [0, 1, 2, 3, 4])
    a = O.multi_sweeps(*args, point_cloud_range=PCR)
    b = O.multi_sweeps(*args, point_cloud_range=PCR, exact=True)
    assert a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


@pytest.mark.parametrize("n,sweeps_num,test_mode", [(0, 9, False), (3, 9, False), (9, 9, False), (10, 9, True),
                                                     (10, 9, False), (10, 0, False), (0, 0, False), (25, 9, False)])
def test_choose_sweeps_matches_the_reference_and_its_rng(n, sweeps_num, test_mode):
    from bevfusion_b200.lidar_sweeps import choose_sweeps
    np.random.seed(123)
    want = reference_choices(n, sweeps_num, test_mode)
    after_ref = np.random.random()
    np.random.seed(123)
    got = choose_sweeps(n, sweeps_num, test_mode)
    after = np.random.random()
    assert np.array_equal(got, want) and got.dtype == want.dtype
    assert after == after_ref     # the same RNG consumption, including 10 choose 9 and sweeps_num = 0


def test_sweeps_num_zero_consumes_the_rng():
    from bevfusion_b200.lidar_sweeps import choose_sweeps
    np.random.seed(5)
    fresh = np.random.random()
    np.random.seed(5)
    assert len(choose_sweeps(10, 0)) == 0
    assert np.random.random() != fresh


def test_time_lag_is_the_reference_difference():
    from bevfusion_b200.lidar_sweeps import time_lag
    ts, sts = 1533151603547590, 1533151603497534
    assert time_lag(ts, sts) == ts / 1e6 - sts / 1e6


def test_pad_entries_and_key_column_maps():
    rng = np.random.default_rng(3)
    key = O.nuscenes_sweep(rng, 200, load_dim=6)
    key[3:, 0] += np.where(key[3:, 0] < 0, -2.0, 2.0).astype(np.float32)
    key[:3, 0], key[:3, 1] = 0.5, -0.25                     # only these three inside the remove_close square
    out = O.multi_sweeps(key, [], [], [], [], [0, 1, 2, 3, 4], key_use_dim=[0, 1, 2, 3, 5], sweeps_num=3)
    # key rows, then three copies of the key through remove_close, all with time 0
    assert out.shape == (200 + 3 * 197, 5)
    assert np.array_equal(out[:200, :4], key[:, :4]) and np.array_equal(out[:200, 4], np.zeros(200, np.float32))
    assert not np.signbit(out[:, 4]).any()
    for k in range(3):
        assert np.array_equal(out[200 + 197 * k:200 + 197 * (k + 1), :4], key[3:, :4])
    # a permuted key map composes LoadPointsFromFile's use_dim with the sweep loader's
    out = O.multi_sweeps(key, [], [], [], [], [4, 2, 1, 0, 3], key_use_dim=[5, 0, 1, 2, 3], sweeps_num=0)
    assert np.array_equal(out[:, :4], key[:, [3, 1, 0, 5]])


def test_remove_close_boundaries():
    one_below = np.nextafter(np.float32(1), np.float32(0))
    rows = np.array([[1.0, 0.0], [0.0, 1.0], [-1.0, 0.5], [one_below, one_below], [-one_below, 0.0], [-0.0, -0.0],
                     [0.0, -1.0], [np.nan, 0.0]], np.float32)
    kept = O.remove_close(rows)
    # |x| or |y| exactly 1.0 is not close; nextafter(1, 0) and -0.0 are; NaN is never close
    assert kept.shape[0] == 5
    assert np.array_equal(kept[:4], rows[[0, 1, 2, 6]]) and np.isnan(kept[4, 0])


def test_range_faces_and_nan_rows():
    lo, hi = np.float32(-51.2), np.float32(51.2)
    assert float(hi) != 51.2                                  # the bound float32 cannot hold exactly
    pcr = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]
    inside = lambda v: np.nextafter(v, np.float32(0))       # one float32 ulp inside the face
    rows = []
    for axis, (a, b) in enumerate([(lo, hi), (lo, hi), (np.float32(-5.0), np.float32(3.0))]):
        for v, keep in [(a, False), (b, False), (inside(a), True), (inside(b), True)]:
            r = np.zeros(5, np.float32)
            r[axis] = v
            rows.append((r, keep))
    rows.append((np.array([np.nan, 0, 0, 0, 0], np.float32), False))
    rows.append((np.array([0, 0, np.nan, 0, 0], np.float32), False))
    key = np.stack([r for r, _ in rows])
    out = O.multi_sweeps(key, [], [], [], [], [0, 1, 2, 3, 4], sweeps_num=0, point_cloud_range=pcr)
    want = key[[k for k, (_, keep) in enumerate(rows) if keep]]
    assert np.array_equal(out, want)


def test_parameter_block_layout_matches_the_header():
    from bevfusion_b200 import _C
    from bevfusion_b200.lidar_sweeps import ENTRY_DTYPE, PARAMS_DTYPE, MAX_DIM
    with open(_C.HEADER_PATH) as f:
        header = f.read()
    define = lambda name: int(re.search(r"#define %s (\d+)" % name, header).group(1))
    assert ENTRY_DTYPE.itemsize == define("BEVB200_SWEEP_ENTRY_BYTES")
    assert PARAMS_DTYPE.itemsize == define("BEVB200_SWEEP_PARAMS_BYTES")
    assert MAX_DIM == define("BEVB200_SWEEP_MAX_DIM")
    assert [ENTRY_DTYPE.fields[k][1] for k in ("kind", "slot", "rotation", "translation", "lag")] == [0, 4, 8, 80, 104]


def test_c_symbols_are_declared_and_bound():
    from bevfusion_b200 import _C
    declared = _C.declared_symbols()
    with open(_C.HEADER_PATH) as f:
        header = f.read()
    for name in ("bevb200_lidar_sweeps_workspace_bytes", "bevb200_lidar_sweeps_assemble",
                 "bevb200_hard_voxelize_mean_dev"):
        assert name in declared and name in _C._SIGNATURES
        assert hasattr(_C.lib(), name)
        params = re.search(r"\b%s\(([^)]*)\)" % name, header).group(1).split(",")
        assert len(params) == len(_C._SIGNATURES[name][1]), name


def test_workspace_query():
    from bevfusion_b200 import _C
    q = _C.lib().bevb200_lidar_sweeps_workspace_bytes
    assert q(1, 10, 34720) >= 10 * 34 * 4                   # one int32 per 1024-row tile of every entry
    assert q(4, 10, 34720) >= 4 * 10 * 34 * 4 > q(1, 10, 34720)
    assert q(1, 100, 1024) < q(1, 100, 1025)
    assert q(0, 10, 34720) >= 0
    for bad in [(-1, 10, 100), (1, 0, 100), (1, 10, 0), (65536, 1, 1), (1, 2, 1 << 30)]:
        assert q(*bad) == 0, bad


def test_assemble_refuses_bad_arguments_before_any_device_work():
    from bevfusion_b200 import _C
    L = _C.lib()
    # every check runs before the first device call: these addresses are never touched
    base = dict(store=1, slots=2, slot_cap=100, load_dim=5, slot_rows=1, params=8, entries=128, batch=1,
                max_entries=10, out_dim=5, cap=100, out=1, counts=1, status=1, ws=1, ws_bytes=1 << 20, stream=0)
    order = list(base)
    for field, value in [("load_dim", 2), ("load_dim", 65), ("out_dim", 4), ("out_dim", 9), ("cap", 0),
                         ("slots", 0), ("max_entries", 0), ("status", 0), ("entries", 0), ("entries", 132),
                         ("ws_bytes", 4)]:
        args = dict(base, **{field: value})
        rc = L.bevb200_lidar_sweeps_assemble(*[args[k] for k in order])
        assert rc != 0, (field, value)
        assert "lidar_sweeps_assemble" in L.bevb200_last_error().decode()


def test_python_refusals():
    from bevfusion_b200.lidar_sweeps import SweepStore, _check_loader_options
    with pytest.raises(ValueError, match="CUDA"):
        SweepStore(2, 100, 5, device="cpu")
    with pytest.raises(ValueError, match="load_dim"):
        SweepStore(2, 100, 2, device="cuda")
    with pytest.raises(ValueError, match="reduce_beams"):
        _check_loader_options(16, None)
    with pytest.raises(ValueError, match="load_augmented"):
        _check_loader_options(None, "mvp")
    _check_loader_options(32, None)          # the shipped configs: 32 beams leave the points as they are
    _check_loader_options(None, None)


def test_voxelize_num_points_refuses_cpu_tensors():
    from bevfusion_b200.voxelize import voxelize_mean_fused
    with pytest.raises(RuntimeError, match="CUDA"):
        voxelize_mean_fused(torch.zeros(8, 5), [0.5] * 3, [0, 0, 0, 4, 4, 4], 5, 10,
                            num_points=torch.zeros(1, dtype=torch.int32))
