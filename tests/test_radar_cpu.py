"""CPU: the float64 radar oracle against the reference fixture, the radar encoder's module structure and
state_dict, and host-side argument checks of the radar C ABI.  No compute calls."""
import ctypes
import os

import numpy as np
import pytest
import torch

from radar_oracle import layers_from_state_dict, radar_feature_net, radar_scatter

FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "radar_tiny.npz")
CFG = {"A": dict(in_channels=45, feat_channels=[128, 128, 128, 64]), "B": dict(in_channels=18, feat_channels=[128, 64])}
NORM = dict(type="BN1d", eps=1e-3, momentum=0.01)


def fixture():
    return np.load(FIX)


def oracle_run(d, name, train=False):
    sd = {str(k): d["%s__sd__%s" % (name, k)] for k in d[name + "__sd_keys"]}
    vs, pcr = d["voxel_size"], d["point_cloud_range"]
    layers = layers_from_state_dict(sd, "pts_voxel_encoder.", len(CFG[name]["feat_channels"]))
    feats = d["features"][:, :, :CFG[name]["in_channels"]]
    return radar_feature_net(feats, d["num_voxels"], d["coors"], layers, vs[0], vs[1], vs[0] / 2 + pcr[0],
                             vs[1] / 2 + pcr[1], pcr, train=train)


def build(name, d):
    from bevfusion_b200.radar_encoder import RadarEncoder
    return RadarEncoder(
        dict(type="RadarFeatureNet", with_distance=False, voxel_size=list(d["voxel_size"]),
             point_cloud_range=list(d["point_cloud_range"]), norm_cfg=NORM, **CFG[name]),
        dict(type="PointPillarsScatter", in_channels=64, output_shape=[int(d["nx"]), int(d["ny"])]))


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
        k = "%s__sd__pts_voxel_encoder.rfn_layers.%d.norm." % (name, i)
        assert np.allclose(0.99 * d[k + "running_mean"] + 0.01 * mu, d["%s__train_running_mean%d" % (name, i)],
                           rtol=0, atol=1e-12)
        assert np.allclose(0.99 * d[k + "running_var"] + 0.01 * var, d["%s__train_running_var%d" % (name, i)],
                           rtol=0, atol=1e-12)


def test_oracle_does_not_modify_its_input():
    d = fixture()
    feats = np.array(d["features"], np.float64)
    before = feats.copy()
    sd = {str(k): d["A__sd__" + str(k)] for k in d["A__sd_keys"]}
    vs, pcr = d["voxel_size"], d["point_cloud_range"]
    radar_feature_net(feats, d["num_voxels"], d["coors"], layers_from_state_dict(sd, "pts_voxel_encoder.", 4),
                      vs[0], vs[1], vs[0] / 2 + pcr[0], vs[1] / 2 + pcr[1], pcr)
    assert np.array_equal(feats, before)


def test_fixture_covers_every_count_and_negative_scales():
    d = fixture()
    num, P = d["num_voxels"], int(d["P"])
    assert set(num.tolist()) == set(range(1, P + 1)) and (num == P).sum() >= 4
    for i in range(4):
        assert (d["A__sd__pts_voxel_encoder.rfn_layers.%d.norm.weight" % i] < 0).any()


def test_scatter_oracle_matches_reference():
    d = fixture()
    got = radar_scatter(d["A__eval"], d["coors"], int(d["batch"]), int(d["nx"]), int(d["ny"]))
    assert np.array_equal(got, d["A__canvas"])


@pytest.mark.parametrize("name", ["A", "B"])
def test_state_dict_matches_reference(name):
    d = fixture()
    enc = build(name, d)
    sd = enc.state_dict()
    keys = [str(k) for k in d[name + "__sd_keys"]]
    assert list(sd) == keys
    for k in keys:
        assert tuple(sd[k].shape) == d["%s__sd__%s" % (name, k)].shape, k
    enc.load_state_dict({k: torch.from_numpy(np.asarray(d["%s__sd__%s" % (name, k)])).float() for k in keys})
    bn = enc.pts_voxel_encoder.rfn_layers[0].norm
    assert bn.eps == 1e-3 and bn.momentum == 0.01
    layers = enc.pts_voxel_encoder.rfn_layers
    assert [l.last_vfe for l in layers] == [False] * (len(layers) - 1) + [True]


def test_unused_config_keys():
    from bevfusion_b200.radar_encoder import RadarEncoder
    d = fixture()
    vox = dict(type="RadarFeatureNet", in_channels=45, feat_channels=[128, 128, 128, 64])
    scat = dict(type="PointPillarsScatter", in_channels=64, output_shape=[128, 128])
    enc = RadarEncoder(vox, scat, pts_transformer_encoder=None, post_scatter=None, pts_bev_encoder=None)
    assert enc.pts_transformer_encoder is None and enc.post_scatter is None and enc.pts_bev_encoder is None
    for key in ("pts_transformer_encoder", "post_scatter", "pts_bev_encoder"):
        with pytest.raises(NotImplementedError):
            RadarEncoder(vox, scat, **{key: dict(type="Anything")})
    assert build("A", d).pts_voxel_encoder._with_distance is False


def test_cpu_tensors_raise():
    from bevfusion_b200.radar_encoder import RadarFeatureNet
    net = RadarFeatureNet(45, [128, 128, 128, 64], voxel_size=(0.8, 0.8, 8),
                          point_cloud_range=(-51.2, -51.2, -5, 51.2, 51.2, 3))
    with pytest.raises(RuntimeError):
        net(torch.zeros(4, 20, 45), torch.ones(4, dtype=torch.int32), torch.zeros(4, 4, dtype=torch.int32))


def widths(*w):
    return (ctypes.c_int * len(w))(*w)


def test_radar_abi_rejects_bad_shapes():
    from bevfusion_b200 import _C
    L = _C.lib()
    shipped = L.bevb200_radar_packed_bytes(45, 4, widths(128, 128, 128, 64))
    # bf16 hi | lo fragments of 48x128 + 2 x 128x128 + 128x64 weights, folded BN, the virtual row
    assert shipped == 4 * (48 * 128 + 2 * 128 * 128 + 128 * 64) + 4 * 2 * (3 * 128 + 64) + 4 * 64
    assert L.bevb200_radar_packed_bytes(18, 2, widths(128, 64)) > 0
    assert L.bevb200_radar_packed_bytes(3, 1, widths(16)) > 0
    assert L.bevb200_radar_packed_bytes(126, 1, widths(128)) > 0
    bad = [(45, 5, widths(128, 128, 128, 64, 64)), (45, 0, widths(64)), (45, 2, widths(128, 100)),
           (45, 2, widths(144, 64)), (45, 1, widths(8)), (2, 1, widths(64)), (127, 1, widths(64)),
           (45, 1, None)]
    for f, n, w in bad:
        assert L.bevb200_radar_packed_bytes(f, n, w) == 0
        assert L.bevb200_radar_pack_weights(None, None, None, f, n, w, None, None) == -4
    assert L.bevb200_radar_pack_weights(None, None, None, 45, 4, widths(128, 128, 128, 64), None, None) == -1
    g = [0.8, 0.8, -50.8, -50.8]
    lo = _C.host_array(ctypes.c_float, [-51.2, -51.2, -5.0])
    span = _C.host_array(ctypes.c_float, [102.4, 102.4, 8.0])
    vp = lambda a: ctypes.cast(a, ctypes.c_void_p)
    w4 = widths(128, 128, 128, 64)
    for p in (33, 0):                                      # P 1..32
        assert L.bevb200_radar_features(None, None, None, 10, None, p, 45, 4, w4, *g, vp(lo), vp(span), None, None,
                                        None, 0, None) == -4
        assert L.bevb200_radar_features_workspace_bytes(10, p) == 0
    assert L.bevb200_radar_features(None, None, None, 10, None, 20, 45, 5, widths(128, 128, 128, 64, 64), *g,
                                    vp(lo), vp(span), None, None, None, 0, None) == -4
    assert L.bevb200_radar_features(None, None, None, 10, None, 20, 45, 4, w4, *g, vp(lo), vp(span), None, None,
                                    None, 0, None) == -1
    assert L.bevb200_radar_features_workspace_bytes(10, 20) >= 10 * 20 * 16
    assert L.bevb200_hard_voxelize_radar_workspace_bytes(1000, 20) > L.bevb200_hard_voxelize_workspace_bytes(1000, 20)
    vs = _C.host_array(ctypes.c_float, [0.8, 0.8, 4.0])
    vs8 = _C.host_array(ctypes.c_float, [0.8, 0.8, 8.0])
    cr = _C.host_array(ctypes.c_float, [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0])
    vn = ctypes.c_int32(0)
    call = lambda vsz, p, nx, ny, w=w4, n=4: L.bevb200_hard_voxelize_radar(
        None, 0, 45, vp(vsz), vp(cr), p, 100, n, w, *g, vp(lo), vp(span), None, None, nx, ny, ctypes.addressof(vn),
        None, 0, None)
    assert call(vs, 20, 128, 128) == -4                     # two cells high: not a pillar grid
    assert call(vs8, 20, 128, 64) == -1                     # canvas shape differs from the grid
    assert call(vs8, 40, 128, 128) == -4                    # P > 32
    assert call(vs8, 20, 128, 128, widths(128, 100), 2) == -4
