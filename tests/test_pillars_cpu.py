"""CPU: the float64 pillar oracle against the reference fixture, the PointPillars module structure and
state_dict, and host-side argument checks of the pillar C ABI.  No compute calls."""
import ctypes
import os

import numpy as np
import pytest
import torch

from pillars_oracle import layers_from_state_dict, pillar_feature_net, pillars_scatter

FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pillars_tiny.npz")


def fixture():
    return np.load(FIX)


def oracle_run(d, name, train=False):
    sd = {str(k): d["%s__sd__%s" % (name, k)] for k in d[name + "__sd_keys"]}
    n_layers = 2 if name == "A" else 1
    vs, pcr = d["voxel_size"], d["point_cloud_range"]
    layers = layers_from_state_dict(sd, "pts_voxel_encoder.", n_layers)
    return pillar_feature_net(d["features"], d["num_voxels"], d["coors"], layers, vs[0], vs[1],
                              vs[0] / 2 + pcr[0], vs[1] / 2 + pcr[1], with_distance=name == "B", train=train)


@pytest.mark.parametrize("name", ["A", "B"])
def test_oracle_matches_reference_eval(name):
    d = fixture()
    out, _ = oracle_run(d, name)
    gold = d[name + "__eval"]
    assert np.abs(out - gold).max() <= 1e-12 * max(np.abs(gold).max(), 1.0)


@pytest.mark.parametrize("name", ["A", "B"])
def test_oracle_matches_reference_train(name):
    d = fixture()
    out, stats = oracle_run(d, name, train=True)
    gold = d[name + "__train"]
    assert np.abs(out - gold).max() <= 1e-12 * max(np.abs(gold).max(), 1.0)
    for i, (mu, var) in enumerate(stats):      # momentum 0.01 running-statistics update
        k = "%s__sd__pts_voxel_encoder.pfn_layers.%d.norm." % (name, i)
        assert np.allclose(0.99 * d[k + "running_mean"] + 0.01 * mu, d["%s__train_running_mean%d" % (name, i)],
                           rtol=0, atol=1e-12)
        assert np.allclose(0.99 * d[k + "running_var"] + 0.01 * var, d["%s__train_running_var%d" % (name, i)],
                           rtol=0, atol=1e-12)


def test_fixture_covers_every_count_and_padded_rows_matter():
    d = fixture()
    num, P = d["num_voxels"], int(d["P"])
    assert set(num.tolist()) == set(range(1, P + 1))
    # some scale is negative, so the padded-row / min-vs-max traps are exercised
    assert (d["A__sd__pts_voxel_encoder.pfn_layers.0.norm.weight"] < 0).any()
    assert (d["A__sd__pts_voxel_encoder.pfn_layers.1.norm.weight"] < 0).any()


def test_scatter_oracle_matches_reference():
    d = fixture()
    got = pillars_scatter(d["A__eval"], d["coors"], int(d["batch"]), int(d["nx"]), int(d["ny"]))
    assert np.array_equal(got, d["A__canvas"])


@pytest.mark.parametrize("name", ["A", "B"])
def test_state_dict_matches_reference(name):
    from bevfusion_b200.pillar_encoder import PointPillarsEncoder
    d = fixture()
    cfg = dict(feat_channels=[64, 64], with_distance=False) if name == "A" else \
        dict(feat_channels=[64], with_distance=True)
    enc = PointPillarsEncoder(
        dict(type="PillarFeatureNet", in_channels=5, voxel_size=list(d["voxel_size"]),
             point_cloud_range=list(d["point_cloud_range"]), norm_cfg=dict(type="BN1d", eps=1e-3, momentum=0.01),
             **cfg),
        dict(type="PointPillarsScatter", in_channels=64, output_shape=[int(d["nx"]), int(d["ny"])]))
    sd = enc.state_dict()
    keys = [str(k) for k in d[name + "__sd_keys"]]
    assert list(sd) == keys
    for k in keys:
        assert tuple(sd[k].shape) == d["%s__sd__%s" % (name, k)].shape, k
    enc.load_state_dict({k: torch.from_numpy(np.asarray(d["%s__sd__%s" % (name, k)])).float() for k in keys})
    bn = enc.pts_voxel_encoder.pfn_layers[0].norm
    assert bn.eps == 1e-3 and bn.momentum == 0.01


def test_cpu_tensors_raise():
    from bevfusion_b200.pillar_encoder import PillarFeatureNet, PointPillarsScatter
    net = PillarFeatureNet(5, [64, 64], voxel_size=(0.2, 0.2, 8), point_cloud_range=(-51.2, -51.2, -5, 51.2, 51.2, 3))
    with pytest.raises(RuntimeError):
        net(torch.zeros(4, 20, 5), torch.ones(4, dtype=torch.int32), torch.zeros(4, 4, dtype=torch.int32))
    with pytest.raises(RuntimeError):
        PointPillarsScatter(64, (8, 8))(torch.zeros(4, 64), torch.zeros(4, 4, dtype=torch.int32), 1)


def test_pillar_abi_rejects_bad_shapes():
    from bevfusion_b200 import _C
    L = _C.lib()
    assert L.bevb200_pillar_packed_bytes(5, 32, 64) > 0
    assert L.bevb200_pillar_packed_bytes(8, 32, 64) == L.bevb200_pillar_packed_bytes(3, 32, 64)
    for f, c1, c2 in [(9, 32, 64), (2, 32, 64), (5, 64, 64), (5, 32, 128), (5, 16, 64)]:
        assert L.bevb200_pillar_packed_bytes(f, c1, c2) == 0
        assert L.bevb200_pillar_pack_weights(None, None, None, None, None, None, f, c1, c2, None, None) == -4
    assert L.bevb200_pillar_pack_weights(None, None, None, None, None, None, 5, 32, 64, None, None) == -1
    g = [0.2, 0.2, -51.1, -51.1]
    for p, f in [(33, 5), (0, 5), (20, 9), (20, 2)]:      # P 1..32, F 3..8
        assert L.bevb200_pillar_features(None, None, None, 10, None, p, f, *g, None, None, None) == -4
    assert L.bevb200_pillar_features(None, None, None, 10, None, 20, 5, *g, None, None, None) == -1
    vs =_C.host_array(ctypes.c_float, [0.2, 0.2, 4.0])
    cr = _C.host_array(ctypes.c_float, [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0])
    vn = ctypes.c_int32(0)
    vp = lambda a: ctypes.cast(a, ctypes.c_void_p)
    # two cells high: not a pillar grid
    assert L.bevb200_hard_voxelize_pillars(None, 0, 5, vp(vs), vp(cr), 20, 100, *g, None, None, 512, 512,
                                           ctypes.addressof(vn), None, 0, None) == -4
    vs8 = _C.host_array(ctypes.c_float, [0.2, 0.2, 8.0])
    # canvas shape differs from the grid
    assert L.bevb200_hard_voxelize_pillars(None, 0, 5, vp(vs8), vp(cr), 20, 100, *g, None, None, 512, 256,
                                           ctypes.addressof(vn), None, 0, None) == -1
    assert L.bevb200_hard_voxelize_pillars(None, 0, 5, vp(vs8), vp(cr), 40, 100, *g, None, None, 512, 512,
                                           ctypes.addressof(vn), None, 0, None) == -4
