"""CPU: ObjectPaste's host side against the reference (golden/object_paste_tiny.npz, made by the reference's own
DataBaseSampler, ObjectPaste.__call__, box_np_ops and numba box_collision_test).

- The package's DataBaseSampler + ObjectPaste and the oracle's sampler reproduce every case's draws exactly: the kept
  objects, the merged boxes and labels, the face planes, and (epoch gate) an untouched RNG.
- The oracle's removal and paste reproduce the reference's output cloud bit for bit.
- The vectorised box_collision_test has zero disagreements with the numba function on the fixture's adversarial pairs.
- The C ABI: the symbols, the struct sizes and the argument checks."""
import hashlib
import os
import re

import numpy as np
import pytest

import object_paste_oracle as O
from bevfusion_b200 import object_paste as P

CASES = O.CASES


@pytest.fixture(scope="module")
def z(golden_dir):
    return O.load_fixture(os.path.join(golden_dir, "object_paste_tiny.npz"))


def fixture_db(z, case):
    """{class: [info]} in the fixture's key order, each info with its id and raw rows"""
    keys = [str(k) for k in z[case + "_db_keys"]]
    off = z[case + "_db_offsets"]
    db = {k: [] for k in keys}
    for i, c in enumerate(z[case + "_db_class"]):
        db[keys[c]].append({"name": keys[c], "path": "obj_%04d.bin" % i, "id": i, "box3d_lidar": z[case + "_db_boxes"][i],
                            "difficulty": int(z[case + "_db_difficulty"][i]),
                            "num_points_in_gt": int(z[case + "_db_npts"][i]), "rows": z[case + "_db_rows"][off[i]:off[i + 1]]})
    return db


def settings(z, case):
    groups = {O.CLASSES[c]: int(n) for c, n in z[case + "_groups"]}
    prepare = O.SHIPPED_PREPARE if int(z[case + "_prepare"]) else {}
    epoch, stop = (int(v) for v in z[case + "_epoch"])
    return groups, prepare, epoch, None if stop == -9999 else stop


def frames(z, case):
    for j in range(int(z[case + "_frames"])):
        p = "%s_f%d_" % (case, j)
        yield p, z[p + "gt_boxes"], z[p + "gt_labels"]


def package_paste(z, case, rng=None):
    groups, prepare, epoch, stop = settings(z, case)
    if rng is None:
        np.random.seed(int(z[case + "_seed"]))
    sampler = P.DataBaseSampler(fixture_db(z, case), 1.0, prepare, groups, O.CLASSES, rng=rng)
    paste = P.ObjectPaste(sampler, stop)
    paste.set_epoch(epoch)
    return paste


@pytest.mark.parametrize("case", CASES)
def test_package_sampler_reproduces_the_reference(z, case):
    paste = package_paste(z, case)
    for p, gt, labels in frames(z, case):
        before = np.random.get_state()
        d = paste.draw(gt, labels)
        kept = [] if d is None else [i["id"] for i in d.infos]
        assert kept == z[p + "kept"].tolist()
        if d is not None:
            assert [paste.sampler.infos[i]["id"] for i in d.indices] == kept
            assert d.boxes.dtype == np.float32
            normal, dd = P.box_planes(d.boxes)
            assert O.count_diff(normal, z[p + "normal"]) == 0 and O.count_diff(dd, z[p + "d"]) == 0
        boxes, lab = P.ObjectPaste.merge(gt, labels, d)
        assert O.count_diff(boxes, z[p + "boxes"]) == 0 and np.array_equal(lab, z[p + "labels"])
        if case == "epoch_gate":
            after = np.random.get_state()
            assert d is None and int(z[p + "rng_unchanged"]) == 1
            assert np.array_equal(before[1], after[1]) and before[2] == after[2]


@pytest.mark.parametrize("case", CASES)
def test_package_sampler_on_a_random_state(z, case):
    # the same draws on a RandomState seeded as the global RNG was
    paste = package_paste(z, case, rng=np.random.RandomState(int(z[case + "_seed"])))
    for p, gt, labels in frames(z, case):
        d = paste.draw(gt, labels)
        assert ([] if d is None else [i["id"] for i in d.infos]) == z[p + "kept"].tolist()


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_reference(z, case):
    groups, prepare, epoch, stop = settings(z, case)
    np.random.seed(int(z[case + "_seed"]))
    db = fixture_db(z, case)
    sampler = O.Sampler(db, 1.0, prepare, groups)
    for p, gt, labels in frames(z, case):
        kept = [] if (stop is not None and epoch >= stop) else sampler.sample_all(gt, labels)
        assert [i["id"] for i in kept] == z[p + "kept"].tolist()
        boxes = np.stack([i["box3d_lidar"] for i in kept]) if kept else np.zeros((0, 9), np.float32)
        normal, d = z[p + "normal"], z[p + "d"]
        got = O.paste(z[p + "cloud"], [i["rows"] for i in kept], boxes, normal, d)
        assert O.count_diff(got, z[p + "points"]) == 0


def test_nan_rows_are_removed_only_when_something_is_pasted(z):
    cloud = z["shipped_f0_cloud"]
    nan = np.isnan(cloud[:, :3]).any(1)
    assert nan.any()
    assert not np.isnan(z["shipped_f0_points"][:, :3]).any()            # S >= 1: NaN rows go
    assert np.isnan(z["epoch_gate_f0_points"][:, :3]).any(1).sum() == nan.sum()   # S = 0: they stay


def test_vectorised_collision_test_matches_numba(z):
    n = int(z["bulk_pairs"])
    assert n >= 100000
    pairs = O.collision_pairs(np.random.default_rng(77), n)
    a = P.center_to_corner_box2d(pairs[:, 0, 0:2], pairs[:, 0, 3:5], pairs[:, 0, 6])
    b = P.center_to_corner_box2d(pairs[:, 1, 0:2], pairs[:, 1, 3:5], pairs[:, 1, 6])
    assert hashlib.sha256(a.tobytes() + b.tobytes()).digest() == z["bulk_corners_sha256"].tobytes()
    want = np.unpackbits(z["bulk_collide"])[:n].astype(bool)
    got = np.zeros(n, bool)
    for s in range(0, n, 250):
        got[s:s + 250] = np.diagonal(P.box_collision_test(a[s:s + 250], b[s:s + 250]))
    assert int((got != want).sum()) == 0
    assert 0.2 < want.mean() < 0.8
    # the oracle's pair-by-pair restatement on a slice
    assert all(O.collide(a[k], b[k]) == want[k] for k in range(0, n, 97))


def test_sample_2d_and_bad_boxes_raise():
    with pytest.raises(ValueError):
        P.ObjectPaste(None, sample_2d=True)
    db = {"car": [{"name": "car", "path": "x", "box3d_lidar": np.zeros(9), "difficulty": 0, "num_points_in_gt": 9}]}
    with pytest.raises(ValueError):
        P.DataBaseSampler(db, 1.0, {}, {"car": 1}, O.CLASSES)


def test_c_abi():
    from bevfusion_b200 import _C
    header = open(_C.HEADER_PATH).read()
    defs = dict(re.findall(r"#define (BEVB200_\w+) (\d+)", header))
    assert int(defs["BEVB200_PASTE_SAMPLE_BYTES"]) == P.SAMPLE_DTYPE.itemsize == 48
    assert int(defs["BEVB200_PASTE_OBJECT_BYTES"]) == P.OBJECT_DTYPE.itemsize == 112
    assert int(defs["BEVB200_SWEEPS_BAD_PASTE"]) == P.BAD_PASTE
    assert int(defs["BEVB200_PASTE_MAX_OBJECTS"]) == P.MAX_PASTE
    for name in ("bevb200_lidar_sweeps_assemble_paste", "bevb200_lidar_sweeps_paste_workspace_bytes"):
        assert name in _C.declared_symbols() and name in _C._SIGNATURES
    L = _C.lib()
    tiles = (34720 + 1023) // 1024
    assert L.bevb200_lidar_sweeps_paste_workspace_bytes(4, 10, 34720, 40, 4096) >= 4 * 50 * tiles * 4
    assert L.bevb200_lidar_sweeps_paste_workspace_bytes(4, 10, 100, 40, 5000) >= 4 * 50 * 5 * 4
    assert L.bevb200_lidar_sweeps_paste_workspace_bytes(4, 10, 100, 257, 10) == 0
    assert L.bevb200_lidar_sweeps_paste_workspace_bytes(4, 10, 100, 1, 0) == 0
    st = 8
    # max_paste out of range with a paste block: rejected before any launch
    assert L.bevb200_lidar_sweeps_assemble_paste(8, 1, 1, 5, 8, 8, 8, 0, 8, 1, 5, 8, 1, 1, 16, 16, 300, 1, 1, 5, 1,
                                                 8, 8, st, 8, 1 << 20, 0) == -1
