"""CPU: the restatement of LoadRadarPointsMultiSweeps + PointsRangeFilter's radar face (tests/radar_sweeps_oracle.py)
reproduces the reference's own outputs (golden/radar_sweeps_tiny.npz) bit for bit; its numpy and exact FMA-chain
transforms agree on seeded nuScenes-like sweeps; radar_entries chooses the sweeps and time lags the reference
chooses; the op codes use_dim composes into; the parameter block the device reads; the C declarations, the workspace
query and the argument checks made before any device work."""
import re

import numpy as np
import pytest

import radar_sweeps_oracle as O

GOLDEN, CASES, golden_case = O.GOLDEN, O.GOLDEN_CASES, O.golden_case


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("exact", [False, True])
def test_oracle_reproduces_the_reference(case, exact):
    z = np.load(GOLDEN)
    g = golden_case(z, case)
    for bev_range, key in ((O.BEV_RANGE, "_after"), (None, "_before")):
        got = O.multi_sweeps(g["raws"], g["rotations"], g["translations"], g["time_diffs"], g["use_dim"],
                             g["compensate_velocity"], g["normalize"], bev_range=bev_range, exact=exact)
        want = z[case + key]
        assert got.shape == want.shape and np.array_equal(got.view(np.int32), want.view(np.int32)), (case, key)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_numpy_and_fma_chain_transforms(seed):
    # counted, not assumed: a disagreement would be a double-rounding case that the device (the chain) and the
    # reference (numpy's dgemm) resolve differently
    rng = np.random.default_rng(seed)
    disagreements = 0
    for k in range(5):
        R, t = O.radar_pose(rng, k)
        disagreements += O.transforms_both(O.radar_sweep(rng, 1000), R, t, True, 0.05 * k)
    assert disagreements == 0


def reference_entries(radars_dict, sweeps_num):
    """loading.py:731-745 as written: (data_path, time_diff) of every loaded sweep"""
    out = []
    for key, sweeps in radars_dict.items():
        if len(sweeps) < sweeps_num:
            idxes = list(range(len(sweeps)))
        else:
            idxes = list(range(sweeps_num))
        ts = sweeps[0]['timestamp'] * 1e-6
        for idx in idxes:
            sweep = sweeps[idx]
            timestamp = sweep['timestamp'] * 1e-6
            out.append((sweep["data_path"], ts - timestamp))
    return out


def test_radar_entries_choose_the_reference_sweeps_and_lags():
    from bevfusion_b200.radar_sweeps import radar_entries
    rng = np.random.default_rng(4)
    t0 = 1533151603547590
    radars = {}
    for k, n in enumerate([6, 9, 1, 4, 6]):
        radars["RADAR_%d" % k] = [{"data_path": "r%d_%d" % (k, s), "timestamp": t0 - s * 75013 - k * 17,
                                   "sensor2lidar_rotation": np.eye(3), "sensor2lidar_translation": rng.normal(size=3)}
                                  for s in range(n)]
    slots = {}
    for sweeps_num in (0, 1, 6, 10):
        got = radar_entries(radars, sweeps_num, lambda s: slots.setdefault(s["data_path"], len(slots)))
        want = reference_entries(radars, sweeps_num)
        assert [next(p for p, v in slots.items() if v == e[0]) for e in got] == [w[0] for w in want]
        assert [e[3] for e in got] == [w[1] for w in want]        # the same float64 lags, bit for bit
    # the * 1e-6 form differs from LiDAR's / 1e6 on these stamps
    a, b = 1533151603547590, 1533151603472577
    assert any((a * 1e-6 - c * 1e-6) != (a / 1e6 - c / 1e6) for c in range(b, b + 200))
    with pytest.raises(IndexError):
        radar_entries(dict(radars, RADAR_EMPTY=[]), 6, lambda s: 0)
    with pytest.raises(IndexError):
        reference_entries(dict(radars, RADAR_EMPTY=[]), 6)


def test_column_ops():
    from bevfusion_b200 import radar_sweeps as RS
    ops, lo, span = RS.column_ops(O.SHIPPED_USE_DIM)
    kinds = ops & 0xff
    assert list(kinds[:6]) == [RS.OP_XYZ] * 3 + [RS.OP_RAW, RS.OP_VELO_COMP, RS.OP_VELO_COMP]
    assert kinds[6] == RS.OP_LAG and list(kinds[7:15]) == [RS.OP_ONE_HOT] * 8 and kinds[-1] == RS.OP_ORDINAL
    ops, lo, span = RS.column_ops(list(range(58)))
    assert (ops[57] & 0xff) == RS.OP_NUSC and (ops[49] >> 16) == 2 and ((ops[49] >> 8) & 0xff) == 17
    ops, lo, span = RS.column_ops([0, 1, 2, 3, 4, 5, -1, 5], True, [(3, 0, 50), (4, -100, 100), (-1, 0.1, 0.7)])
    assert [bool(o & RS.OP_NORMALIZE) for o in ops] == [False] * 3 + [True] * 2 + [False, False, True]
    assert span[7] == 0.7 - 0.1 and lo[4] == -100.0 and (ops[6] & 0xff) == RS.OP_NUSC
    for bad in ([0, 1], list(range(58)) + list(range(7)), [0, 1, 58]):
        with pytest.raises(ValueError):
            RS.column_ops(bad)
    with pytest.raises(ValueError, match="twice"):
        RS.column_ops([0, 1, 2, 3], True, [(3, 0, 50), (-1, 0, 1)])
    with pytest.raises(ValueError):
        RS.column_ops([0, 1, 2], True, [(3, 0, 50)])


def test_parameter_block_layout_matches_the_header():
    from bevfusion_b200 import _C
    from bevfusion_b200 import radar_sweeps as RS
    with open(_C.HEADER_PATH) as f:
        header = f.read()
    define = lambda name: int(re.search(r"#define %s \(?(\d+)" % name, header).group(1))
    assert RS.ENTRY_DTYPE.itemsize == define("BEVB200_RADAR_SWEEP_ENTRY_BYTES")
    assert RS.PARAMS_DTYPE.itemsize == define("BEVB200_RADAR_SWEEP_PARAMS_BYTES")
    assert RS.MAX_DIM == define("BEVB200_RADAR_SWEEP_MAX_DIM") and RS.LOAD_DIM == define("BEVB200_RADAR_LOAD_DIM")
    assert RS.BAD_CATEGORY == define("BEVB200_RADAR_SWEEPS_BAD_CATEGORY")
    for name in ("RAW", "XYZ", "VELO", "VELO_COMP", "LAG", "ONE_HOT", "ORDINAL", "NUSC"):
        assert getattr(RS, "OP_" + name) == define("BEVB200_RADAR_OP_" + name)
    assert RS.OP_NORMALIZE == 1 << 24 and "#define BEVB200_RADAR_OP_NORMALIZE (1 << 24)" in header
    assert [RS.ENTRY_DTYPE.fields[k][1] for k in ("kind", "slot", "rotation", "translation", "time_diff")] == \
        [0, 4, 8, 80, 104]
    assert [RS.PARAMS_DTYPE.fields[k][1] for k in ("norm_min", "norm_span", "ops", "compensate_velocity",
                                                    "has_range", "range")] == [0, 512, 1024, 1280, 1284, 1288]
    assert RS._ENTRIES_AT >= RS.PARAMS_DTYPE.itemsize and RS._ENTRIES_AT % 8 == 0


def test_c_symbols_are_declared_and_bound():
    from bevfusion_b200 import _C
    declared = _C.declared_symbols()
    with open(_C.HEADER_PATH) as f:
        header = f.read()
    for name in ("bevb200_radar_sweeps_workspace_bytes", "bevb200_radar_sweeps_assemble",
                 "bevb200_hard_voxelize_radar_dev"):
        assert name in declared and name in _C._SIGNATURES
        assert hasattr(_C.lib(), name)
        params = re.search(r"\b%s\(([^)]*)\)" % name, header).group(1).split(",")
        assert len(params) == len(_C._SIGNATURES[name][1]), name


def test_workspace_query():
    from bevfusion_b200 import _C
    q = _C.lib().bevb200_radar_sweeps_workspace_bytes
    assert q(1, 30, 200) >= 30 * 2 * 4                     # one int32 per 128-row tile of every entry
    assert q(4, 30, 200) >= 4 * 30 * 2 * 4
    assert q(1, 100, 128 * 64) < q(1, 100, 128 * 64 + 1)
    assert q(0, 30, 200) >= 0
    for bad in [(-1, 10, 100), (1, 0, 100), (1, 10, 0), (65536, 1, 1), (1, 65536, 1), (1, 2, 1 << 30)]:
        assert q(*bad) == 0, bad


def test_assemble_refuses_bad_arguments_before_any_device_work():
    from bevfusion_b200 import _C
    L = _C.lib()
    # every check runs before the first device call: these addresses are never touched
    base = dict(store=1, slots=2, slot_cap=100, slot_rows=1, params=8, entries=1536, batch=1, max_entries=30,
                out_dim=45, cap=100, out=1, counts=1, status=1, ws=1, ws_bytes=1 << 20, stream=0)
    order = list(base)
    for field, value in [("out_dim", 2), ("out_dim", 65), ("cap", 0), ("cap", 1 << 30), ("slots", 0),
                         ("max_entries", 0), ("slot_cap", 0), ("batch", 65536), ("status", 0), ("entries", 0),
                         ("entries", 1540), ("params", 4), ("ws_bytes", 4), ("ws", 0)]:
        args = dict(base, **{field: value})
        rc = L.bevb200_radar_sweeps_assemble(*[args[k] for k in order])
        assert rc != 0, (field, value)
        assert "radar_sweeps_assemble" in L.bevb200_last_error().decode()


def test_voxelize_radar_dev_refuses_bad_arguments():
    import ctypes
    from bevfusion_b200 import _C
    L = _C.lib()
    w4 = _C.host_array(ctypes.c_int, [128, 128, 128, 64])
    f3 = lambda *v: ctypes.cast(_C.host_array(ctypes.c_float, list(v)), ctypes.c_void_p)
    vn = ctypes.c_int32(0)
    call = lambda vs, rows=100, n_dev=None, p=20: L.bevb200_hard_voxelize_radar_dev(
        None, n_dev, rows, 45, vs, f3(-51.2, -51.2, -5.0, 51.2, 51.2, 3.0), p, 100, 4, w4, 0.8, 0.8, -50.8, -50.8,
        f3(-51.2, -51.2, -5.0), f3(102.4, 102.4, 8.0), None, None, 128, 128, ctypes.addressof(vn), None, 0, None)
    assert call(f3(0.8, 0.8, 8.0)) == -1                   # no device count
    assert call(f3(0.8, 0.8, 4.0), n_dev=8) == -4          # two cells high: not a pillar grid
    assert call(f3(0.8, 0.8, 8.0), n_dev=8, p=40) == -4    # P > 32
    assert call(f3(0.8, 0.8, 8.0), rows=-1, n_dev=8) == -1


def test_python_refusals():
    import torch
    from bevfusion_b200.radar_sweeps import RadarSweepStore
    from bevfusion_b200.radar_encoder import RadarEncoder
    from bevfusion_b200.voxelize import Voxelization
    with pytest.raises(ValueError, match="CUDA"):
        RadarSweepStore(2, 100, device="cpu")
    with pytest.raises(ValueError, match="positive"):
        RadarSweepStore(0, 100, device="cuda")
    enc = RadarEncoder(dict(type="RadarFeatureNet", in_channels=45, feat_channels=[128, 128, 128, 64],
                            voxel_size=[0.8, 0.8, 8], point_cloud_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]),
                       dict(type="PointPillarsScatter", in_channels=64, output_shape=[128, 128])).eval()
    vox = Voxelization([0.8, 0.8, 8], [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], 10, (30000, 60000)).eval()
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA"):
        enc.forward_points(torch.zeros(2, 10, 45), vox, num_points=torch.zeros(2, dtype=torch.int32))
