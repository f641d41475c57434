"""CPU: the host half of bevfusion_b200.lidar_aug and its oracle.

- GlobalRotScaleTrans / RandomFlip3D draw what the reference drew under the same seed (golden/lidar_aug_tiny.npz), in
  train and test mode, on numpy's global RNG and on a given RandomState; lidar_aug_matrix equals the reference's.
- The oracle (tests/lidar_aug_oracle.py), in its torch form and in its exact fp32 FMA-chain form, reproduces the
  reference's pipeline outputs and, on 10^5 rows each of LiDAR, radar and boxes, the reference classes' outputs
  (compared through the SHA-256 the generator stored, with the disagreement counts it recorded).
- fma32 against exact rational arithmetic; the records the host packs; the C layout and declarations; the argument
  checks made before any device work."""
import re

import numpy as np
import pytest
import torch

import lidar_aug_oracle as O

GOLDEN = "golden/lidar_aug_tiny.npz"
CASES = ["flip00", "flip01", "flip10", "flip11", "rot0", "test", "empty"]


@pytest.fixture(scope="module")
def z(golden_dir):
    import os
    return np.load(os.path.join(golden_dir, "lidar_aug_tiny.npz"))


def ref_draw(z, case):
    return O.draw_tuple(z[case + "_draw"])


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("own_rng", [False, True])
def test_draws_match_the_reference(z, case, own_rng):
    from bevfusion_b200.lidar_aug import GlobalRotScaleTrans, RandomFlip3D, draw_sample
    seed, is_train = int(z[case + "_seed"]), bool(z[case + "_is_train"])
    rng = np.random.RandomState(seed) if own_rng else None
    if not own_rng:
        np.random.seed(seed)
    d = draw_sample(GlobalRotScaleTrans(O.SHIPPED_SCALE, list(z[case + "_rot_lim"]), O.SHIPPED_TRANSLATE, is_train,
                                        rng=rng), RandomFlip3D(rng=rng))
    scale, theta, trans, fh, fv = ref_draw(z, case)
    if is_train:
        assert d.scale == scale and d.theta == theta and np.array_equal(d.translation, trans)
    else:
        assert d.scale is None and d.theta is None and d.translation is None
    assert (d.flip_horizontal, d.flip_vertical) == (bool(fh), bool(fv))


@pytest.mark.parametrize("case", CASES)
def test_matrix_matches_the_reference(z, case):
    from bevfusion_b200.lidar_aug import LidarAugDraw, lidar_aug_matrix
    d = LidarAugDraw(*ref_draw(z, case))
    m = lidar_aug_matrix(d)
    assert m.dtype == np.float32 and O.count_diff(m, z[case + "_matrix"]) == 0
    assert O.count_diff(O.lidar_aug_matrix(tuple(d)), m) == 0


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("exact", [False, True])
def test_oracle_reproduces_the_reference_pipeline(z, case, exact):
    got = O.pipeline(z[case + "_points_in"], z[case + "_radar_in"], z[case + "_boxes_in"], z[case + "_labels_in"],
                     z[case + "_masks_in"], ref_draw(z, case), exact=exact)
    for g, key in zip(got, ("points", "radar", "boxes", "labels", "masks")):
        want = z[case + "_" + key]
        if key in ("labels", "masks"):
            assert np.array_equal(g, want), key
        else:
            assert O.count_diff(g, want) == 0, key


@pytest.mark.parametrize("exact", [False, True])
def test_oracle_agrees_with_the_reference_classes_on_1e5_rows(z, exact):
    outputs = {"points": [], "radar": [], "boxes": []}
    for draw, points, radar, boxes7, boxes9 in O.bulk_inputs():
        outputs["points"].append(O.augment_points(points, draw, exact))
        outputs["radar"].append(O.augment_radar(radar, draw, exact))
        outputs["boxes"] += [O.limit_yaw(O.augment_boxes(boxes9, draw, exact), exact),
                             O.limit_yaw(O.augment_boxes(boxes7, draw, exact), exact)]
    for k, arrays in outputs.items():
        assert sum(len(a) for a in arrays) == int(z["bulk_rows_" + k]) >= 10 ** 5
        assert O.sha256_of(arrays) == z["bulk_sha256_" + k].tobytes(), k
        assert int(z["bulk_diff_" + k]) == 0 and int(z["bulk_diff_" + k + "_exact"]) == 0


def test_torch_and_exact_forms_agree_on_the_bulk_rows():
    # counted, not assumed: a disagreement would be a value that torch's CPU matmul and the device's FMA chain
    # round differently
    diffs = 0
    for draw, points, radar, boxes7, boxes9 in O.bulk_inputs(rows=4000):
        diffs += O.count_diff(O.augment_points(points, draw), O.augment_points(points, draw, True))
        diffs += O.count_diff(O.augment_radar(radar, draw), O.augment_radar(radar, draw, True))
        for b in (boxes7, boxes9):
            diffs += O.count_diff(O.limit_yaw(O.augment_boxes(b, draw)), O.limit_yaw(O.augment_boxes(b, draw, True),
                                                                                     True))
    assert diffs == 0


def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(9)
    a = (rng.normal(0, 50, 3000)).astype(np.float32)
    b = rng.uniform(-1, 1, 3000).astype(np.float32)
    c = (rng.normal(0, 50, 3000)).astype(np.float32)
    a[:40], b[:40], c[:40] = np.float32(-0.0), np.float32(0.5), np.float32(-0.0)
    c[40:80] = -(a[40:80].astype(np.float64) * b[40:80]).astype(np.float32)   # near-cancellations
    got = O.fma32(a, b, c)
    want = np.array([O.fma32_fraction(x, y, w) for x, y, w in zip(a, b, c)], np.float32)
    assert O.count_diff(got, want) == 0
    assert np.signbit(got[:40]).all()
    # the non-FMA evaluation (product rounded to fp32, then the sum) is a different function on these inputs
    assert O.count_diff((a * b) + c, want) > 0


@pytest.mark.parametrize("theta", [0.0, 0.3, -0.78539816, np.pi, 1e-8])
def test_records_hold_the_reference_scalars(theta):
    from bevfusion_b200.lidar_aug import LidarAugDraw, pack_record
    t = np.array([0.1, -0.2, 0.3])
    rec = pack_record(LidarAugDraw(1.05, theta, t, True, False))
    point_rot, box_rot, yaw = O.rot_mats(theta)
    assert O.count_diff(rec["point_rot"].reshape(3, 3), point_rot) == 0
    assert O.count_diff(rec["box_rot"].reshape(3, 3), box_rot) == 0
    assert rec["yaw_inc"] == yaw and rec["scale"] == np.float32(1.05)
    assert np.array_equal(rec["translation"], t.astype(np.float32))
    assert (rec["enabled"], rec["rot_scale_trans"], rec["flip_horizontal"], rec["flip_vertical"]) == (1, 1, 1, 0)
    off = pack_record(LidarAugDraw(None, None, None, False, True))
    assert (off["enabled"], off["rot_scale_trans"], off["flip_vertical"]) == (1, 0, 1)


def test_record_layout_and_declarations_match_the_header():
    from bevfusion_b200 import _C
    from bevfusion_b200 import lidar_aug as A
    with open(_C.HEADER_PATH) as f:
        header = f.read()
    define = lambda name: int(re.search(r"#define %s \(?(\d+)" % name, header).group(1))
    assert A.AUG_DTYPE.itemsize == define("BEVB200_LIDAR_AUG_BYTES")
    assert A.BAD_COUNT == define("BEVB200_BOX_AUG_BAD_COUNT")
    assert A.MAX_BOXES == define("BEVB200_HEAD_TARGETS_MAX_BOXES")
    assert [A.AUG_DTYPE.fields[k][1] for k in ("enabled", "rot_scale_trans", "flip_horizontal", "flip_vertical",
                                               "translation", "scale", "yaw_inc", "point_rot", "box_rot")] == \
        [0, 4, 8, 12, 16, 28, 32, 36, 72]
    declared = _C.declared_symbols()
    for name in ("bevb200_lidar_sweeps_assemble_aug", "bevb200_radar_sweeps_assemble_aug", "bevb200_box_aug"):
        assert name in declared and name in _C._SIGNATURES and hasattr(_C.lib(), name)
        params = re.search(r"\b%s\(([^)]*)\)" % name, header).group(1).split(",")
        assert len(params) == len(_C._SIGNATURES[name][1]), name
        floats = [i for i, p in enumerate(params) if p.split()[0] == "float" and "*" not in p]
        assert floats == [i for i, t in enumerate(_C._SIGNATURES[name][1]) if t is _C.c_float], name


def test_argument_checks_before_any_device_work():
    from bevfusion_b200 import _C
    L = _C.lib()
    st = 64   # a non-null address the checks never dereference
    for args in ((0, 0, 0, 1, 4, 8), (0, 0, 0, 1, 4097, 7), (0, 0, 0, -1, 4, 7), (0, 0, 0, 1, 4, 7, -1)):
        B, nmax, D = args[3], args[4], args[5]
        ncls = args[6] if len(args) > 6 else 10
        assert L.bevb200_box_aug(0, 0, 0, B, nmax, D, 0, -1.0, -1.0, 1.0, 1.0, ncls, 0, 0, 0, st, 0) == -1
    assert L.bevb200_box_aug(0, 0, 0, 1, 4, 7, 0, -1.0, -1.0, 1.0, 1.0, 10, 0, 0, 0, 0, 0) == -1
    # the radar augmentation reads output columns 3 and 4
    assert L.bevb200_radar_sweeps_assemble_aug(8, 1, 1, 8, 8, 8, 8, 1, 1, 4, 1, 8, 8, st, 8, 1 << 20, 0) == -1
    assert b"out_dim" in L.bevb200_last_error()
    # misaligned records
    assert L.bevb200_lidar_sweeps_assemble_aug(8, 1, 1, 5, 8, 8, 8, 9, 1, 1, 5, 1, 8, 8, st, 8, 1 << 20, 0) == -1


def test_no_cpu_block():
    from bevfusion_b200.lidar_aug import LidarAug
    with pytest.raises(ValueError):
        LidarAug(2, "cpu")
