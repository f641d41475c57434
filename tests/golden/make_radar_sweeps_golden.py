"""Generates tests/golden/radar_sweeps_tiny.npz from the REFERENCE's own LoadRadarPointsMultiSweeps.__call__
(mmdet3d/datasets/pipelines/loading.py) and RadarPoints.in_range_bev (mmdet3d/core/points/radar_points.py, on the
reference's BasePoints), executed on the CPU with stubs for the modules loading.py imports but the radar loader does
not use (mmcv, nuscenes, PIL, mmdet's PIPELINES and LoadAnnotations, mmdet3d.core.points' other names,
loading_utils).  _load_points is replaced by a lookup of the raw rows by data_path.  Writes only
radar_sweeps_tiny.npz.

Raw sweeps are nuScenes-like 18-column rows (tests/radar_sweeps_oracle.radar_sweep) under five seeded radar poses.
Cases (each one sample; results['radar'] in the listed radar order):
  shipped   the shipped config: sweeps_num 6, radar_use_dims (45 columns), compensate_velocity, no normalize; two
            radars have fewer than 6 sweeps, one has 8
  nocomp    compensate_velocity False, sweeps_num 3
  norm      normalize True with the default normalize_dims on use_dim [0, 1, 2, 3, 4, 5, 18]
  all58     use_dim = all 58 columns, compensate_velocity
Stored per case: the raw sweeps of each entry in concatenation order (raw_<case> [n_total, 18] with counts), the
poses and time lags the reference used, and its output before and after the radar range filter.

Run:  python tests/golden/make_radar_sweeps_golden.py      (needs the reference tree)
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("BEVFUSION_REFERENCE", "/root/reference")
sys.path.insert(0, os.path.dirname(HERE))
import radar_sweeps_oracle as O  # noqa: E402


def load_reference():
    def unused(*args, **kwargs):
        raise AssertionError("not used by the radar loader")

    class Registry:
        def register_module(self, *args, **kwargs):
            return lambda cls: cls

    # the reference's BasePoints and RadarPoints, in a stub package so radar_points' relative import resolves
    pts = types.ModuleType("refpoints")
    pts.__path__ = []
    sys.modules["refpoints"] = pts
    for name in ("base_points", "radar_points"):
        path = os.path.join(REF, "mmdet3d", "core", "points", name + ".py")
        mod = types.ModuleType("refpoints." + name)
        mod.__package__ = "refpoints"
        sys.modules[mod.__name__] = mod
        exec(compile(open(path).read(), path, "exec"), mod.__dict__)
    stubs = {"mmcv": {}, "PIL": {"Image": object}, "nuscenes": {}, "nuscenes.utils": {},
             "nuscenes.utils.data_classes": {"RadarPointCloud": object},
             "nuscenes.map_expansion": {}, "nuscenes.map_expansion.map_api": {"NuScenesMap": object,
                                                                               "locations": []},
             "mmdet3d": {}, "mmdet3d.core": {},
             "mmdet3d.core.points": {"RadarPoints": sys.modules["refpoints.radar_points"].RadarPoints,
                                     "BasePoints": sys.modules["refpoints.base_points"].BasePoints,
                                     "get_points_type": unused},
             "mmdet": {}, "mmdet.datasets": {}, "mmdet.datasets.builder": {"PIPELINES": Registry()},
             "mmdet.datasets.pipelines": {"LoadAnnotations": object},
             "refpipes": {}, "refpipes.loading_utils": {"load_augmented_point_cloud": unused,
                                                        "reduce_LiDAR_beams": unused}}
    for name, attrs in stubs.items():
        mod = types.ModuleType(name)
        mod.__dict__.update(attrs)
        if name == "refpipes":
            mod.__path__ = []
        sys.modules[name] = mod
    path = os.path.join(REF, "mmdet3d", "datasets", "pipelines", "loading.py")
    ns = {"__name__": "refpipes.loading", "__package__": "refpipes"}
    exec(compile(open(path).read(), path, "exec"), ns)
    return ns["LoadRadarPointsMultiSweeps"]


def make_info(rng, counts, t0=1533151603547590):
    """results['radar'] for radars with the given sweep counts: per sweep a data_path, a timestamp ~75 ms apart, a
    pose; raw rows keyed by data_path"""
    radars, raw = {}, {}
    for k, n_sweeps in enumerate(counts):
        R, t = O.radar_pose(rng, k)
        sweeps = []
        for s in range(n_sweeps):
            path = "radar%d_sweep%d" % (k, s)
            raw[path] = O.radar_sweep(rng, int(rng.integers(20, 90)))
            sweeps.append({"data_path": path, "timestamp": t0 - s * 74_987 - int(rng.integers(0, 3000)),
                           "sensor2lidar_rotation": R @ O.radar_pose(rng, k)[0] if s else R,
                           "sensor2lidar_translation": t + rng.uniform(-0.6, 0.0, 3) * s})
        radars["RADAR_%d" % k] = sweeps
    return radars, raw


CASES = {
    "shipped": dict(counts=[6, 4, 6, 8, 2], sweeps_num=6, use_dim=O.SHIPPED_USE_DIM, compensate_velocity=True,
                    normalize=False),
    "nocomp": dict(counts=[3, 5, 1, 3, 4], sweeps_num=3, use_dim=O.SHIPPED_USE_DIM, compensate_velocity=False,
                   normalize=False),
    "norm": dict(counts=[2, 2, 3, 1, 2], sweeps_num=6, use_dim=[0, 1, 2, 3, 4, 5, 18], compensate_velocity=True,
                 normalize=True),
    "all58": dict(counts=[6, 6, 5, 6, 6], sweeps_num=6, use_dim=list(range(58)), compensate_velocity=True,
                  normalize=False),
}


def main():
    Loader = load_reference()
    rng = np.random.default_rng(2026)
    out = {}
    for case, cfg in CASES.items():
        radars, raw = make_info(rng, cfg["counts"])
        loader = Loader(load_dim=18, use_dim=cfg["use_dim"], sweeps_num=cfg["sweeps_num"], max_num=2500,
                        compensate_velocity=cfg["compensate_velocity"], filtering="none", normalize=cfg["normalize"])
        loader._load_points = lambda path: raw[path]
        res = loader({"radar": radars})["radar"]
        before = res.tensor.numpy().copy()
        after = res.tensor[res.in_range_bev([-55.0, -55.0, 55.0, 55.0])].numpy()
        rows, rots, trans, lags, counts = [], [], [], [], []
        for sweeps in radars.values():          # the entries the reference loaded, in its order
            ts = sweeps[0]["timestamp"] * 1e-6
            for sweep in sweeps[:min(len(sweeps), cfg["sweeps_num"])]:
                rows.append(raw[sweep["data_path"]])
                counts.append(len(rows[-1]))
                rots.append(sweep["sensor2lidar_rotation"])
                trans.append(sweep["sensor2lidar_translation"])
                lags.append(ts - sweep["timestamp"] * 1e-6)
        out.update({case + "_raw": np.concatenate(rows), case + "_counts": np.array(counts, np.int32),
                    case + "_rot": np.array(rots), case + "_trans": np.array(trans), case + "_lag": np.array(lags),
                    case + "_use_dim": np.array(cfg["use_dim"], np.int32),
                    case + "_flags": np.array([cfg["sweeps_num"], cfg["compensate_velocity"], cfg["normalize"]],
                                              np.int32),
                    case + "_timestamps": np.array([[s["timestamp"] for s in sw] + [-1] * (8 - len(sw))
                                                    for sw in radars.values()], np.int64),
                    case + "_before": before, case + "_after": after})
        print(case, before.shape, after.shape)
    np.savez_compressed(os.path.join(HERE, "radar_sweeps_tiny.npz"), **out)


if __name__ == "__main__":
    main()
