"""Generates tests/golden/object_paste_tiny.npz from the REFERENCE's own DataBaseSampler / BatchSampler
(mmdet3d/datasets/pipelines/dbsampler.py), ObjectPaste.__call__ (transforms_3d.py), box_np_ops and
box_collision_test (pipelines/utils.py, through numba), acting on the reference's LiDARPoints and
LiDARInstance3DBoxes, with stubs for mmcv (load returns the synthetic dbinfos, build_from_cfg builds the sampler and a
LoadPointsFromFile that reads the .bin files as the reference's does) and np.long shimmed to np.int64.  Writes only
object_paste_tiny.npz.

Each case builds a seeded synthetic database (infos plus .bin files in a temporary directory), seeds numpy's global RNG,
constructs the reference's ObjectPaste (the class samplers' shuffles consume the RNG) and runs it on one or more frames
in order.  Stored per case: the database (boxes, classes, difficulty, num_points_in_gt, raw rows), the sampler
settings, the seed, and per frame the inputs (GT boxes, labels, cloud) and the reference's outputs (points, boxes,
labels, the kept objects' ids and face planes).  The inputs are regenerated from the seeds by
object_paste_oracle.case_inputs, so the file stores digests of them instead of the arrays, and stores the output cloud
as the mask of surviving input rows plus a digest of the whole output (object_paste_oracle.load_fixture rebuilds and
checks both).
  shipped       the shipped sample_groups and prepare filters
  exhaust       classes of 4 and 5 objects drawn 2 and 3 at a time over 3 frames: the remainder, reshuffle and reset
                path, with idx + num == n
  many_gt       more GT boxes of each class than its max (nothing of those classes is drawn)
  empty_gt      no GT boxes
  all_collide   a GT box containing every candidate (nothing kept: the cloud is returned untouched)
  contains_gt   every candidate contains a GT box (the other containment direction)
  pending       every candidate of a class at one spot: the first ones are rejected by later, still pending ones
  epoch_gate    epoch == stop_epoch: nothing drawn, the RNG state unchanged
Bulk check: box_collision_test on oracle.collision_pairs (>= 10^5 adversarial pairs), results stored as bits.

Run:  python tests/golden/make_object_paste_golden.py      (needs the reference tree and numba)
"""
import copy
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("BEVFUSION_REFERENCE", "/root/reference")
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import object_paste_oracle as O  # noqa: E402
import make_lidar_aug_golden as LG  # noqa: E402

if not hasattr(np, "long"):
    np.long = np.int64            # the reference's dbsampler and ObjectPaste use np.long

BULK_PAIRS = 120000


def load_reference():
    R = LG.load_reference()
    ns = R.GlobalRotScaleTrans.__init__.__globals__          # transforms_3d's module namespace

    def load(path, name, package):
        mod = types.ModuleType(name)
        mod.__package__ = package
        sys.modules[name] = mod
        exec(compile(open(path).read(), path, "exec"), mod.__dict__)
        return mod

    box_np_ops = load(os.path.join(REF, "mmdet3d", "core", "bbox", "box_np_ops.py"), "refbox_np_ops", None)
    sys.modules["mmdet3d.core.bbox"].box_np_ops = box_np_ops
    utils = load(os.path.join(REF, "mmdet3d", "datasets", "pipelines", "utils.py"), "refds.pipelines.utils",
                 "refds.pipelines")

    class Registry:
        def register_module(self, *args, **kwargs):
            return lambda cls: cls

    class LoadPointsFromFile:      # loading.py's LoadPointsFromFile for coord_type LIDAR and reduce_beams >= 32
        def __init__(self, coord_type, load_dim, use_dim, reduce_beams=None):
            self.load_dim = load_dim
            self.use_dim = list(range(use_dim)) if isinstance(use_dim, int) else use_dim

        def __call__(self, results):
            points = np.fromfile(results["lidar_path"], dtype=np.float32).reshape(-1, self.load_dim)
            points = points[:, self.use_dim]
            results["points"] = R.LiDARPoints(points, points_dim=points.shape[-1], attribute_dims=None)
            return results

    state = {}

    def build_from_cfg(cfg, registry):
        cfg = dict(cfg)
        kind = cfg.pop("type")
        return {"DataBaseSampler": lambda: ds.DataBaseSampler(**cfg),
                "LoadPointsFromFile": lambda: LoadPointsFromFile(**cfg)}[kind]()

    import logging
    sys.modules["mmcv"].load = lambda path: copy.deepcopy(state["infos"])
    sys.modules["mmcv"].build_from_cfg = build_from_cfg
    stub = types.ModuleType("mmdet.datasets")
    stub.PIPELINES = Registry()
    stub.__path__ = []
    sys.modules["mmdet.datasets"] = stub
    sys.modules["refds.builder"].OBJECTSAMPLERS = Registry()
    mu = types.ModuleType("mmdet3d.utils")
    mu.get_root_logger = lambda: logging.getLogger("ref")
    sys.modules["mmdet3d.utils"] = mu
    ds = load(os.path.join(REF, "mmdet3d", "datasets", "pipelines", "dbsampler.py"), "refds.pipelines.dbsampler",
              "refds.pipelines")
    ns["build_from_cfg"] = build_from_cfg
    ns["box_np_ops"] = box_np_ops
    R.ObjectPaste, R.box_np_ops, R.box_collision_test, R.state = ns["ObjectPaste"], box_np_ops, \
        utils.box_collision_test, state
    return R


def ref_planes(R, boxes):
    corners = R.box_np_ops.center_to_corner_box3d(boxes[:, :3], boxes[:, 3:6], boxes[:, 6], origin=(0.5, 0.5, 0),
                                                  axis=2)
    surfaces = R.box_np_ops.corner_to_surfaces_3d(corners)
    return R.box_np_ops.surface_equ_3d(surfaces[:, :, :3, :])


def run_case(R, case, seed):
    db, groups, prepare, frames, epoch, stop = O.case_inputs(case, seed)
    out = {case + "_groups": np.array([[O.CLASSES.index(c), n] for c, n in groups.items()], np.int32),
           case + "_prepare": np.int32(bool(prepare)),
           case + "_epoch": np.array([epoch, -9999 if stop is None else stop], np.int32),
           case + "_seed": np.int64(seed), case + "_frames": np.int32(len(frames)),
           case + "_inputs_sha256": O.inputs_digest(db, frames)}
    with tempfile.TemporaryDirectory() as root:
        R.state["infos"] = O.write_db(db, root)
        loaded = []
        np.random.seed(seed)
        paste = R.ObjectPaste(dict(dataset_root=root + "/", info_path="dbinfos.pkl", rate=1.0, prepare=prepare,
                                   classes=O.CLASSES, sample_groups=groups,
                                   points_loader=dict(type="LoadPointsFromFile", coord_type="LIDAR", load_dim=5,
                                                      use_dim=5, reduce_beams=32)), stop_epoch=stop)
        paste.set_epoch(epoch)
        sampler = paste.db_sampler
        load = sampler.points_loader.__call__
        sampler.points_loader = lambda results: (loaded.append(os.path.basename(results["lidar_path"])),
                                                 load(results))[1]
        for j, (gt, labels, cloud) in enumerate(frames):
            before = np.random.get_state()[1].copy(), np.random.get_state()[2]
            loaded.clear()
            data = {"points": R.LiDARPoints(torch.from_numpy(cloud.copy()), points_dim=5),
                    "gt_bboxes_3d": R.LiDARInstance3DBoxes(torch.from_numpy(gt.copy()), box_dim=9),
                    "gt_labels_3d": labels.copy()}
            data = paste(data)
            after = np.random.get_state()[1], np.random.get_state()[2]
            kept = [int(p[4:8]) for p in loaded]
            boxes = data["gt_bboxes_3d"].tensor.numpy()
            points = data["points"].tensor.numpy()
            normal, d = ref_planes(R, boxes[len(gt):]) if kept else (np.zeros((0, 6, 3), np.float32),
                                                                      np.zeros((0, 6), np.float32))
            # the reference's output is [the kept objects' rows, the surviving cloud rows]: store which cloud rows
            # survive and a digest of the whole output, and rebuild it from the regenerated inputs in the tests
            pasted = sum(int(db_row_count(db, k)) for k in kept)
            keep = np.zeros(len(cloud), bool)
            if kept:
                survivors = points[pasted:]
                keep = ~R.box_np_ops.points_in_rbbox(cloud[:, :3], boxes[len(gt):]).any(-1)
                assert O.count_diff(survivors, cloud[keep]) == 0
            else:
                keep[:] = True
            p = "%s_f%d_" % (case, j)
            out.update({p + "gt_boxes": gt, p + "gt_labels": labels, p + "keep": np.packbits(keep),
                        p + "points_sha256": O.digest(points), p + "boxes": boxes,
                        p + "labels": np.asarray(data["gt_labels_3d"], np.int64), p + "kept": np.array(kept, np.int64),
                        p + "normal": normal, p + "d": d,
                        p + "rng_unchanged": np.int32(np.array_equal(before[0], after[0]) and before[1] == after[1])})
            print(case, j, "gt", len(gt), "kept", kept, "points", cloud.shape, "->", points.shape)
    return out


def db_row_count(db, k):
    return next(len(i["rows"]) for v in db.values() for i in v if i["id"] == k)


def bulk(R):
    pairs = O.collision_pairs(np.random.default_rng(77), BULK_PAIRS)
    a = R.box_np_ops.center_to_corner_box2d(pairs[:, 0, 0:2], pairs[:, 0, 3:5], pairs[:, 0, 6])
    b = R.box_np_ops.center_to_corner_box2d(pairs[:, 1, 0:2], pairs[:, 1, 3:5], pairs[:, 1, 6])
    res = np.zeros(BULK_PAIRS, bool)
    chunk = 1000
    for s in range(0, BULK_PAIRS, chunk):         # each pair's test, in chunks of 1000 diagonal entries
        m = R.box_collision_test(a[s:s + chunk], b[s:s + chunk])
        res[s:s + chunk] = np.diagonal(m)
    print("bulk pairs", BULK_PAIRS, "colliding", int(res.sum()))
    import hashlib
    corners = hashlib.sha256(np.ascontiguousarray(a).tobytes() + np.ascontiguousarray(b).tobytes()).digest()
    return {"bulk_pairs": np.int64(BULK_PAIRS), "bulk_collide": np.packbits(res),
            "bulk_corners_sha256": np.frombuffer(corners, np.uint8)}


def main():
    R = load_reference()
    out = {}
    for k, case in enumerate(O.CASES):
        out.update(run_case(R, case, 1000 + k))
    out.update(bulk(R))
    np.savez_compressed(os.path.join(HERE, "object_paste_tiny.npz"), **out)


if __name__ == "__main__":
    main()
