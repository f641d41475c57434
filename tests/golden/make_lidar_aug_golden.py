"""Generates tests/golden/lidar_aug_tiny.npz from the REFERENCE's own GlobalRotScaleTrans, RandomFlip3D,
PointsRangeFilter, ObjectRangeFilter and ObjectNameFilter (mmdet3d/datasets/pipelines/transforms_3d.py) acting on the
reference's LiDARPoints, RadarPoints and LiDARInstance3DBoxes (mmdet3d/core/points, mmdet3d/core/bbox/structures),
executed on the CPU with stubs for the modules those files import but these classes do not use (mmcv, mmdet's
PIPELINES, the CUDA ops, VoxelGenerator, box_np_ops).  Writes only lidar_aug_tiny.npz.

Pipeline cases (one sample each, numpy's global RNG seeded per case, the transforms called in pipeline order):
  flip00, flip01, flip10, flip11  is_train, the shipped augment3d limits, the seed searched so the two flip draws
                                  are (horizontal, vertical) as named
  rot0      rot_lim [0, 0] (the camera+radar config)
  test      is_train False: GlobalRotScaleTrans draws nothing, RandomFlip3D still draws
  empty     an empty box set
Each stores the inputs (a LiDAR cloud [n, 5], a radar cloud [m, 45] with the shipped radar_use_dims layout, 9-column
boxes with -1 labels, BEV masks), the reference's draws as it made them, and its outputs: points, radar, boxes,
labels, masks and lidar_aug_matrix.

Bulk check: the oracle (tests/lidar_aug_oracle.py) against the reference classes on seeded rows (bulk_inputs),
in both the torch and the exact fp32 FMA-chain forms.  The number of rows and the disagreement counts are stored
(they must be zero), with a SHA-256 of the reference's output bytes per group, so the CPU tests can re-derive the
same outputs from the oracle without the reference tree.

Run:  python tests/golden/make_lidar_aug_golden.py      (needs the reference tree)
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("BEVFUSION_REFERENCE", "/root/reference")
sys.path.insert(0, os.path.dirname(HERE))
import lidar_aug_oracle as O  # noqa: E402


def _exec(path, name, package):
    mod = types.ModuleType(name)
    mod.__package__ = package
    sys.modules[name] = mod
    exec(compile(open(path).read(), path, "exec"), mod.__dict__)
    return mod


def load_reference():
    """namespace with the reference's LiDARPoints, RadarPoints, LiDARInstance3DBoxes, GlobalRotScaleTrans,
    RandomFlip3D, PointsRangeFilter, ObjectRangeFilter, ObjectNameFilter"""
    def unused(*args, **kwargs):
        raise AssertionError("not used by these transforms")

    class Registry:
        def register_module(self, *args, **kwargs):
            return lambda cls: cls

    def stub(name, attrs=None, package=False):
        mod = types.ModuleType(name)
        mod.__dict__.update(attrs or {})
        if package:
            mod.__path__ = []
        sys.modules[name] = mod
        return mod

    stub("refpoints", package=True)
    for name in ("base_points", "lidar_points", "radar_points"):
        _exec(os.path.join(REF, "mmdet3d", "core", "points", name + ".py"), "refpoints." + name, "refpoints")
    BasePoints = sys.modules["refpoints.base_points"].BasePoints
    stub("mmdet3d", package=True)
    stub("mmdet3d.core", {"VoxelGenerator": unused}, package=True)
    stub("mmdet3d.core.points", {"BasePoints": BasePoints})
    stub("mmdet3d.ops", package=True)
    stub("mmdet3d.ops.roiaware_pool3d", {"points_in_boxes_gpu": unused})
    stub("mmdet3d.ops.iou3d", {"iou3d_cuda": None})
    stub("refboxes", package=True)
    for name in ("utils", "base_box3d", "lidar_box3d"):
        _exec(os.path.join(REF, "mmdet3d", "core", "bbox", "structures", name + ".py"), "refboxes." + name,
              "refboxes")
    Boxes = sys.modules["refboxes.lidar_box3d"].LiDARInstance3DBoxes
    stub("mmcv", {"is_tuple_of": unused})
    stub("mmcv.utils", {"build_from_cfg": unused})
    stub("mmdet3d.core.bbox", {"CameraInstance3DBoxes": type("CameraInstance3DBoxes", (), {}),
                               "DepthInstance3DBoxes": type("DepthInstance3DBoxes", (), {}),
                               "LiDARInstance3DBoxes": Boxes, "box_np_ops": None})
    stub("mmdet", package=True)
    stub("mmdet.datasets", package=True)
    stub("mmdet.datasets.builder", {"PIPELINES": Registry()})
    stub("refds", package=True)
    stub("refds.builder", {"OBJECTSAMPLERS": None})
    stub("refds.pipelines", package=True)
    stub("refds.pipelines.utils", {"noise_per_object_v3_": unused})
    path = os.path.join(REF, "mmdet3d", "datasets", "pipelines", "transforms_3d.py")
    ns = {"__name__": "refds.pipelines.transforms_3d", "__package__": "refds.pipelines"}
    exec(compile(open(path).read(), path, "exec"), ns)
    out = types.SimpleNamespace(**{k: ns[k] for k in ("GlobalRotScaleTrans", "RandomFlip3D", "PointsRangeFilter",
                                                       "ObjectRangeFilter", "ObjectNameFilter")})
    out.LiDARPoints = sys.modules["refpoints.lidar_points"].LiDARPoints
    out.RadarPoints = sys.modules["refpoints.radar_points"].RadarPoints
    out.LiDARInstance3DBoxes = Boxes
    return out


def run_pipeline(R, data, is_train, rot_lim, resize_lim=O.SHIPPED_SCALE, trans_lim=O.SHIPPED_TRANSLATE):
    """the five transforms in pipeline order on one sample dict; returns it with lidar_aug_matrix"""
    for t in (R.GlobalRotScaleTrans(resize_lim=resize_lim, rot_lim=rot_lim, trans_lim=trans_lim, is_train=is_train),
              R.RandomFlip3D(), R.PointsRangeFilter(O.POINT_CLOUD_RANGE),
              R.ObjectRangeFilter(O.POINT_CLOUD_RANGE), R.ObjectNameFilter(O.OBJECT_CLASSES)):
        data = t(data)
    return data


def sample(R, rng, n_points, n_radar, n_boxes):
    points, radar, boxes, labels, masks = O.sample_inputs(rng, n_points, n_radar, n_boxes)
    data = {"points": R.LiDARPoints(torch.from_numpy(points.copy()), points_dim=points.shape[1]),
            "radar": R.RadarPoints(torch.from_numpy(radar.copy()), points_dim=radar.shape[1]),
            "gt_bboxes_3d": R.LiDARInstance3DBoxes(torch.from_numpy(boxes.copy()), box_dim=9),
            "gt_labels_3d": labels.copy(), "gt_masks_bev": masks.copy()}
    return (points, radar, boxes, labels, masks), data


CASES = {
    "flip00": dict(is_train=True, rot_lim=O.SHIPPED_ROTATE, flips=(0, 0)),
    "flip01": dict(is_train=True, rot_lim=O.SHIPPED_ROTATE, flips=(0, 1)),
    "flip10": dict(is_train=True, rot_lim=O.SHIPPED_ROTATE, flips=(1, 0)),
    "flip11": dict(is_train=True, rot_lim=O.SHIPPED_ROTATE, flips=(1, 1)),
    "rot0": dict(is_train=True, rot_lim=[0.0, 0.0], flips=None),
    "test": dict(is_train=False, rot_lim=O.SHIPPED_ROTATE, flips=None),
    "empty": dict(is_train=True, rot_lim=O.SHIPPED_ROTATE, flips=None, n_boxes=0),
}


def flips_of_seed(seed, is_train):
    """the (horizontal, vertical) flips the two RandomFlip3D draws give after GlobalRotScaleTrans' draws"""
    st = np.random.RandomState(seed)
    if is_train:
        st.uniform(), st.uniform(), [st.normal(0, 1) for _ in range(3)]
    return int(st.choice([0, 1])), int(st.choice([0, 1]))


def pipeline_cases(R):
    out = {}
    rng = np.random.default_rng(4242)
    for case, cfg in CASES.items():
        inputs, data = sample(R, rng, 1500, 300, cfg.get("n_boxes", 60))
        seed = 100
        while cfg["flips"] is not None and flips_of_seed(seed, cfg["is_train"]) != cfg["flips"]:
            seed += 1
        np.random.seed(seed)
        draw_state = np.random.get_state()
        data = run_pipeline(R, data, cfg["is_train"], cfg["rot_lim"])
        np.random.set_state(draw_state)    # what the reference drew, read back through the same calls
        st = np.random
        scale = theta = np.nan
        trans = np.full(3, np.nan)
        if cfg["is_train"]:
            scale, theta = st.uniform(*O.SHIPPED_SCALE), st.uniform(*cfg["rot_lim"])
            trans = np.array([st.normal(0, O.SHIPPED_TRANSLATE) for _ in range(3)])
        fh, fv = st.choice([0, 1]), st.choice([0, 1])
        points, radar, boxes, labels, masks = inputs
        out.update({case + "_points_in": points, case + "_radar_in": radar, case + "_boxes_in": boxes,
                    case + "_labels_in": labels, case + "_masks_in": masks, case + "_seed": np.int64(seed),
                    case + "_is_train": np.int32(cfg["is_train"]), case + "_rot_lim": np.array(cfg["rot_lim"]),
                    case + "_draw": np.array([scale, theta, *trans, fh, fv], np.float64),
                    case + "_points": data["points"].tensor.numpy(), case + "_radar": data["radar"].tensor.numpy(),
                    case + "_boxes": data["gt_bboxes_3d"].tensor.numpy(),
                    case + "_labels": np.asarray(data["gt_labels_3d"], np.int64),
                    case + "_masks": data["gt_masks_bev"], case + "_matrix": data["lidar_aug_matrix"]})
        print(case, seed, (fh, fv), data["points"].tensor.shape, data["radar"].tensor.shape,
              data["gt_bboxes_3d"].tensor.shape)
    return out


def reference_stages(R, draw, points, radar, boxes):
    """the reference classes' rotate / translate / scale / flip on one draw, without the filters"""
    p = R.LiDARPoints(torch.from_numpy(points.copy()), points_dim=points.shape[1])
    r = R.RadarPoints(torch.from_numpy(radar.copy()), points_dim=radar.shape[1])
    b = R.LiDARInstance3DBoxes(torch.from_numpy(boxes.copy()), box_dim=boxes.shape[1])
    scale, theta, trans, fh, fv = draw
    p.rotate(-theta), p.translate(trans), p.scale(scale)
    r.rotate(-theta), r.translate(trans), r.scale(scale)
    b.rotate(theta), b.translate(trans), b.scale(scale)
    for flag, d in ((fh, "horizontal"), (fv, "vertical")):
        if flag:
            p.flip(d), r.flip(d), b.flip(d)
    b.limit_yaw(offset=0.5, period=2 * np.pi)
    return p.tensor.numpy(), r.tensor.numpy(), b.tensor.numpy()


def bulk(R):
    out, rows = {}, {"points": 0, "radar": 0, "boxes": 0}
    outputs = {k: [] for k in rows}
    diffs = {k: 0 for k in ("points", "radar", "boxes", "points_exact", "radar_exact", "boxes_exact")}
    for draw, points, radar, boxes7, boxes9 in O.bulk_inputs():
        want_p, want_r, want_b9 = reference_stages(R, draw, points, radar, boxes9)
        _, _, want_b7 = reference_stages(R, draw, points[:0], radar[:0], boxes7)
        for exact in (False, True):
            got_p = O.augment_points(points, draw, exact=exact)
            got_r = O.augment_radar(radar, draw, exact=exact)
            got_b9 = O.limit_yaw(O.augment_boxes(boxes9, draw, exact=exact), exact=exact)
            got_b7 = O.limit_yaw(O.augment_boxes(boxes7, draw, exact=exact), exact=exact)
            sfx = "_exact" if exact else ""
            diffs["points" + sfx] += O.count_diff(got_p, want_p)
            diffs["radar" + sfx] += O.count_diff(got_r, want_r)
            diffs["boxes" + sfx] += O.count_diff(got_b9, want_b9) + O.count_diff(got_b7, want_b7)
        for k, v in (("points", want_p), ("radar", want_r), ("boxes", want_b9), ("boxes", want_b7)):
            outputs[k].append(v)
            rows[k] += len(v)
    print("bulk rows", rows, "disagreements", diffs)
    assert not any(diffs.values()), diffs
    for k in rows:
        out["bulk_rows_" + k] = np.int64(rows[k])
        out["bulk_sha256_" + k] = np.frombuffer(O.sha256_of(outputs[k]), np.uint8)
    for k, v in diffs.items():
        out["bulk_diff_" + k] = np.int64(v)
    return out


def main():
    R = load_reference()
    out = pipeline_cases(R)
    out.update(bulk(R))
    np.savez_compressed(os.path.join(HERE, "lidar_aug_tiny.npz"), **out)


if __name__ == "__main__":
    main()
