"""GPU: the radar encoder (native BF16x3 radar kernel, fused voxelize + radar net + scatter, torch path)
against the reference fixture and the float64 oracle; <= 1e-4 of max |ref| unless a test says otherwise."""
import copy
import os

import numpy as np
import pytest
import torch

from radar_oracle import layers_from_state_dict, radar_feature_net

pytestmark = pytest.mark.gpu

FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "radar_tiny.npz")
VS, PCR, P = [0.8, 0.8, 8.0], [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], 20
NORM = dict(type="BN1d", eps=1e-3, momentum=0.01)
SHIPPED = dict(in_channels=45, feat_channels=[128, 128, 128, 64])


def rel_err(got, gold):
    return float(np.abs(np.asarray(got, np.float64) - gold).max() / max(np.abs(gold).max(), 1e-30))


def make_encoder(dev, seed=0, in_channels=45, feat_channels=(128, 128, 128, 64), vs=VS, pcr=PCR, shift_bias=0.0,
                 with_distance=False):
    from bevfusion_b200.radar_encoder import RadarEncoder
    nx, ny = round((pcr[3] - pcr[0]) / vs[0]), round((pcr[4] - pcr[1]) / vs[1])
    enc = RadarEncoder(
        dict(type="RadarFeatureNet", in_channels=in_channels, feat_channels=list(feat_channels),
             with_distance=with_distance, voxel_size=vs, point_cloud_range=pcr, norm_cfg=NORM),
        dict(type="PointPillarsScatter", in_channels=feat_channels[-1], output_shape=[nx, ny]))
    g = torch.Generator().manual_seed(seed)
    for layer in enc.pts_voxel_encoder.rfn_layers:
        w, bn, u = layer.linear.weight, layer.norm, layer.units
        w.data = torch.randn(tuple(w.shape), generator=g) / np.sqrt(w.shape[1])
        sign = torch.where(torch.rand(u, generator=g) < 0.25, -1.0, 1.0)
        bn.weight.data = sign * (0.5 + torch.rand(u, generator=g))
        bn.bias.data = torch.rand(u, generator=g) - 0.5 + shift_bias
        bn.running_mean.data = 0.6 * torch.rand(u, generator=g) - 0.3
        bn.running_var.data = 0.5 + 1.5 * torch.rand(u, generator=g)
    return enc.to(dev).eval()


def oracle_of(net, feats, num, coors):
    sd = {k: v.detach().double().cpu().numpy() for k, v in net.state_dict().items()}
    out, _ = radar_feature_net(feats, num, coors, layers_from_state_dict(sd, "", len(net.rfn_layers)),
                               net.vx, net.vy, net.x_offset, net.y_offset, net.pc_range)
    return out


def voxelizer(p=P):
    from bevfusion_b200.voxelize import Voxelization
    return Voxelization(VS, PCR, p, (30000, 60000)).eval()


def radar(dev, seed=0):
    from bevfusion_b200 import synthetic as S
    return torch.from_numpy(S.radar_cloud(seed=seed)).to(dev)


def batch_voxels(dev, seeds=(1, 2)):
    from bevfusion_b200.voxelize import voxelize_batch
    return voxelize_batch([radar(dev, s) for s in seeds], voxelizer(), voxelize_reduce=False)


@pytest.mark.parametrize("name", ["A", "B"])
def test_native_matches_reference_fixture(cuda, name):
    d = np.load(FIX)
    cfg = SHIPPED if name == "A" else dict(in_channels=18, feat_channels=[128, 64])
    enc = make_encoder(cuda, vs=list(d["voxel_size"]), pcr=list(d["point_cloud_range"]), **cfg)
    enc.load_state_dict({str(k): torch.from_numpy(np.asarray(d[name + "__sd__" + str(k)])).float()
                         for k in d[name + "__sd_keys"]})
    feats = torch.from_numpy(d["features"][:, :, :cfg["in_channels"]]).float().contiguous().to(cuda)
    num = torch.from_numpy(d["num_voxels"]).to(cuda)
    coors = torch.from_numpy(d["coors"]).to(cuda)
    with torch.no_grad():
        assert enc.pts_voxel_encoder._use_native(feats)
        rows = enc.pts_voxel_encoder(feats, num, coors)
        canvas = enc(feats, coors, torch.tensor(int(d["batch"])), num)
    e_rows = rel_err(rows.cpu().numpy(), d[name + "__eval"])
    print("fixture %s: rows %.2e" % (name, e_rows))
    assert e_rows <= 1e-4
    if name == "A":
        assert rel_err(canvas.cpu().numpy(), d["A__canvas"]) <= 1e-4


def test_native_matches_oracle_on_radar_cloud(cuda):
    enc = make_encoder(cuda, seed=1)
    net = enc.pts_voxel_encoder
    v, c4, n = batch_voxels(cuda)
    nn_ = n.cpu().numpy()
    assert (nn_ < P).any() and (nn_ == P).any() and (c4[:, 0] == 1).any()
    with torch.no_grad():
        assert net._use_native(v)
        out = net(v, n, c4)
    gold = oracle_of(net, v.cpu().numpy(), nn_, c4.cpu().numpy())
    err = rel_err(out.cpu().numpy(), gold)
    print("radar cloud: M=%d, n<P %d, n==P %d, err %.2e" % (len(nn_), (nn_ < P).sum(), (nn_ == P).sum(), err))
    assert err <= 1e-4


def test_virtual_row_decides_the_max(cuda):
    """A large BN shift makes the virtual row (the zero row through all four layers) the largest row for
    some channels.  Pillars with n < P must include it, pillars with n == P must not."""
    enc = make_encoder(cuda, seed=2, shift_bias=1.5)
    net = enc.pts_voxel_encoder
    v, c4, n = batch_voxels(cuda, seeds=(3, 4))
    with torch.no_grad():
        out = net(v, n, c4).cpu().numpy()
    vv, nn_, cc = v.cpu().numpy(), n.cpu().numpy(), c4.cpu().numpy()
    gold = oracle_of(net, vv, nn_, cc)
    assert rel_err(out, gold) <= 1e-4
    part, full = np.nonzero(nn_ < P)[0], np.nonzero(nn_ == P)[0]
    assert len(part) and len(full)
    one = part[nn_[part] == 1]
    no_pad = oracle_of(net, vv[one][:, :1], nn_[one], cc[one])             # P = n: no padded row
    assert np.abs(no_pad - gold[one]).max() > 1e-2 * np.abs(gold).max()
    extra = np.concatenate([vv[full], np.zeros_like(vv[full][:, :1])], axis=1)  # P + 1 slots: one padded row
    with_pad = oracle_of(net, extra, nn_[full], cc[full])
    assert np.abs(with_pad - gold[full]).max() > 1e-2 * np.abs(gold).max()


def test_forward_points_bit_equal_to_module_path(cuda):
    from bevfusion_b200.voxelize import voxelize_batch
    enc = make_encoder(cuda, seed=4)
    vox = voxelizer()
    clouds = [radar(cuda, 5), radar(cuda, 6)[:2000].contiguous()]
    with torch.no_grad():
        fused, vnum = enc.forward_points(clouds, vox, return_voxel_num=True)
        feats, coords, sizes = voxelize_batch(clouds, vox, voxelize_reduce=False)
        ref = enc(feats, coords, coords[-1, 0] + 1, sizes)
        again = enc.forward_points(clouds, vox)
    assert tuple(fused.shape) == (2, 64, 128, 128)
    assert vnum.tolist() == [int((coords[:, 0] == k).sum()) for k in range(2)]
    assert bool(torch.equal(fused, ref))
    assert bool(torch.equal(fused, again))
    with torch.no_grad():
        r1 = enc.pts_voxel_encoder(feats, sizes, coords)
        r2 = enc.pts_voxel_encoder(feats, sizes, coords)
    assert bool(torch.equal(r1, r2))


def test_forward_points_cuda_graph(cuda):
    """forward_points has no host synchronisation: captured once on a NaN-padded point buffer (NaN
    points are dropped by the voxelizer), replayed on clouds of different sizes."""
    enc = make_encoder(cuda, seed=7)
    vox = voxelizer()
    clouds = [radar(cuda, s)[:k].contiguous() for s, k in ((8, 3400), (9, 2200), (10, 700))]
    buf = torch.full((max(p.shape[0] for p in clouds) + 100, 45), float("nan"), device=cuda)
    with torch.no_grad():
        enc.forward_points([buf], vox)                       # warm-up: packed weights, allocator
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = enc.forward_points([buf], vox)
        for pts in clouds:
            buf.fill_(float("nan"))
            buf[:pts.shape[0]].copy_(pts)
            g.replay()
            torch.cuda.synchronize()
            eager = enc.forward_points([pts], vox)
            assert bool(torch.equal(out, eager)), pts.shape[0]


def test_nan_and_inf_in_feature_columns(cuda):
    """NaN -> 0 and +-inf -> +-FLT_MAX in real slots; anything in padded slots -> 0 (nan_to_num after the
    mask).  The infinities sit in the rcs column, whose layer-1 weights are made tiny so the rows stay finite."""
    enc = make_encoder(cuda, seed=13)
    net = enc.pts_voxel_encoder
    with torch.no_grad():
        net.rfn_layers[0].linear.weight[:, 3] = 2.0 ** -124   # exact in bf16: FLT_MAX * w is about 16
    v, c4, n = batch_voxels(cuda, seeds=(14,))
    v = v.clone()
    rng = np.random.default_rng(0)
    nn_ = n.cpu().numpy()
    rows = rng.choice(len(nn_), 300, replace=False)
    v[rows, 0, 10] = float("nan")
    v[rows[:100], 0, 3] = float("inf")
    v[rows[100:200], 0, 3] = -float("inf")
    part = np.nonzero(nn_ < P)[0][:200]
    v[part, P - 1, 5] = float("nan")
    v[part, P - 1, 3] = float("inf")
    with torch.no_grad():
        native = net(v, n, c4)
        ref = net._forward_torch(v, n, c4)
    assert bool(torch.isfinite(ref).all())
    assert rel_err(native.cpu().numpy(), ref.double().cpu().numpy()) <= 1e-4


def test_features_not_modified_and_cudnn_untouched(cuda):
    enc = make_encoder(cuda, seed=15)
    net = enc.pts_voxel_encoder
    v, c4, n = batch_voxels(cuda, seeds=(16,))
    before = v.clone()
    torch.backends.cudnn.enabled = False
    try:
        with torch.no_grad():
            net(v, n, c4)                                     # native
        net.train()
        net(v, n, c4)                                         # torch restatement, train mode
        net.eval()
        assert torch.backends.cudnn.enabled is False
    finally:
        torch.backends.cudnn.enabled = True
    assert bool(torch.equal(v, before))


@pytest.mark.parametrize("case", ["empty", "out_of_range"])
def test_empty_cloud_gives_zero_canvas(cuda, case):
    enc = make_encoder(cuda, seed=17)
    pts = torch.zeros((0, 45), device=cuda) if case == "empty" else radar(cuda, 18)[:500].clone()
    if case == "out_of_range":
        pts[:, 0] = 80.0
    with torch.no_grad():
        canvas, vnum = enc.forward_points([pts], voxelizer(), return_voxel_num=True)
    assert int(vnum[0]) == 0 and not bool(canvas.any())


@pytest.mark.parametrize("case", ["five_layers", "width_100", "p40"])
def test_unsupported_shape_takes_torch_path(cuda, case):
    fc = {"five_layers": (128, 128, 128, 64, 64), "width_100": (128, 100, 64)}.get(case, (128, 128, 128, 64))
    enc = make_encoder(cuda, seed=12, feat_channels=fc)
    net = enc.pts_voxel_encoder
    rng = np.random.default_rng(0)
    p = 40 if case == "p40" else P
    m = 300
    num = rng.integers(1, p + 1, size=m).astype(np.int32)
    feats = np.zeros((m, p, 45), np.float32)
    for v in range(m):
        feats[v, :num[v]] = rng.uniform(-2, 2, size=(num[v], 45))
    coors = np.stack([np.zeros(m), rng.integers(0, 128, m), rng.integers(0, 128, m), np.zeros(m)], 1).astype(np.int32)
    t = lambda a: torch.from_numpy(a).to(cuda)
    assert not net._use_native(t(feats))
    with torch.no_grad():
        out = net(t(feats), t(num), t(coors))
    assert rel_err(out.cpu().numpy(), oracle_of(net, feats, num, coors)) <= 1e-4
    with pytest.raises(ValueError):
        with torch.no_grad():
            enc.forward_points([radar(cuda)], voxelizer(p))


def test_with_distance_changes_nothing(cuda):
    a = make_encoder(cuda, seed=19)
    b = make_encoder(cuda, seed=19, with_distance=True)
    v, c4, n = batch_voxels(cuda, seeds=(20,))
    with torch.no_grad():
        assert b.pts_voxel_encoder._use_native(v)
        assert bool(torch.equal(a.pts_voxel_encoder(v, n, c4), b.pts_voxel_encoder(v, n, c4)))


def test_train_mode_forward_backward_vs_float64(cuda):
    d = np.load(FIX)
    enc = make_encoder(cuda, seed=11, vs=list(d["voxel_size"]), pcr=list(d["point_cloud_range"])).train()
    enc64 = copy.deepcopy(enc).double()
    x = torch.from_numpy(d["features"]).double().to(cuda)
    num = torch.from_numpy(d["num_voxels"]).to(cuda)
    coors = torch.from_numpy(d["coors"]).to(cuda)
    x32 = x.float().requires_grad_()
    x64 = x.clone().requires_grad_()
    g = torch.randn(int(d["batch"]), 64, int(d["nx"]), int(d["ny"]), device=cuda, dtype=torch.float64)
    y32 = enc(x32, coors, int(d["batch"]), num)
    (y32 * g.float()).sum().backward()
    # float64 copy: the net in float64, the scatter restated (the library's dense() is fp32)
    rows64 = enc64.pts_voxel_encoder(x64, num, coors)
    c = coors.long()
    (rows64 * g[c[:, 0], :, c[:, 1], c[:, 2]]).sum().backward()
    y64 = torch.zeros_like(g)
    y64[c[:, 0], :, c[:, 1], c[:, 2]] = rows64.detach()
    assert rel_err(y32.detach().cpu().numpy(), y64.cpu().numpy()) <= 1e-5
    assert rel_err(x32.grad.cpu().numpy(), x64.grad.cpu().numpy()) <= 1e-4
    for (name, p32), p64 in zip(enc.named_parameters(), enc64.parameters()):
        assert rel_err(p32.grad.cpu().numpy(), p64.grad.cpu().numpy()) <= 1e-4, name
    for (name, b32), b64 in zip(enc.named_buffers(), enc64.buffers()):
        assert rel_err(b32.cpu().numpy(), b64.cpu().numpy()) <= 1e-5, name
    # and the train-mode forward is the reference's (fixture, from the same inputs in float64)
    enc.load_state_dict({str(k): torch.from_numpy(np.asarray(d["A__sd__" + str(k)])) for k in d["A__sd_keys"]})
    with torch.no_grad():
        rows = enc.pts_voxel_encoder(x.float(), num, coors)
    assert rel_err(rows.cpu().numpy(), d["A__train"]) <= 1e-4
