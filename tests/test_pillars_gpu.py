"""GPU: the PointPillars encoder (native pillar kernel, fused voxelize + pillar net + scatter, torch
path) against the reference fixture and the float64 oracle; <= 1e-4 of max |ref| (BASELINE.json
north_star) unless a test says otherwise."""
import copy
import os

import numpy as np
import pytest
import torch
from torch.nn import functional as F

from pillars_oracle import layers_from_state_dict, pillar_feature_net, pillars_scatter

pytestmark = pytest.mark.gpu

FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pillars_tiny.npz")
VS, PCR, P = [0.2, 0.2, 8.0], [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], 20
NORM = dict(type="BN1d", eps=1e-3, momentum=0.01)


def rel_err(got, gold):
    return float(np.abs(np.asarray(got, np.float64) - gold).max() / max(np.abs(gold).max(), 1e-30))


def make_encoder(dev, seed=0, feat_channels=(64, 64), with_distance=False, vs=VS, pcr=PCR, shift_bias=0.0):
    from bevfusion_b200.pillar_encoder import PointPillarsEncoder
    nx, ny = round((pcr[3] - pcr[0]) / vs[0]), round((pcr[4] - pcr[1]) / vs[1])
    enc = PointPillarsEncoder(
        dict(type="PillarFeatureNet", in_channels=5, feat_channels=list(feat_channels), with_distance=with_distance,
             voxel_size=vs, point_cloud_range=pcr, norm_cfg=NORM),
        dict(type="PointPillarsScatter", in_channels=64, output_shape=[nx, ny]))
    g = torch.Generator().manual_seed(seed)
    for layer in enc.pts_voxel_encoder.pfn_layers:
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
    out, _ = pillar_feature_net(feats, num, coors, layers_from_state_dict(sd, "", len(net.pfn_layers)),
                                net.vx, net.vy, net.x_offset, net.y_offset, with_distance=net._with_distance)
    return out


def voxelize(points):
    from bevfusion_b200.voxelize import Voxelization
    return Voxelization(VS, PCR, P, (30000, 60000)).eval()(points)


def lidar(dev, seed=0):
    from bevfusion_b200 import synthetic as S
    return torch.from_numpy(S.lidar_cloud(seed=seed)).to(dev)


def test_native_matches_reference_fixture(cuda):
    d = np.load(FIX)
    enc = make_encoder(cuda, vs=list(d["voxel_size"]), pcr=list(d["point_cloud_range"]))
    enc.load_state_dict({str(k): torch.from_numpy(np.asarray(d["A__sd__" + str(k)])).float()
                         for k in d["A__sd_keys"]})
    feats = torch.from_numpy(d["features"]).float().to(cuda)
    num = torch.from_numpy(d["num_voxels"]).to(cuda)
    coors = torch.from_numpy(d["coors"]).to(cuda)
    with torch.no_grad():
        rows = enc.pts_voxel_encoder(feats, num, coors)
        canvas = enc(feats, coors, torch.tensor(int(d["batch"])), num)
    e_rows, e_canvas = rel_err(rows.cpu().numpy(), d["A__eval"]), rel_err(canvas.cpu().numpy(), d["A__canvas"])
    print("fixture: rows %.2e canvas %.2e" % (e_rows, e_canvas))
    assert e_rows <= 1e-4 and e_canvas <= 1e-4


def test_native_matches_oracle_on_lidar_cloud(cuda):
    enc = make_encoder(cuda, seed=1)
    net = enc.pts_voxel_encoder
    v, c, n = voxelize(lidar(cuda))
    nn_ = n.cpu().numpy()
    assert (nn_ < P).any() and (nn_ == P).any()
    c4 = F.pad(c, (1, 0), value=0)
    with torch.no_grad():
        assert net._use_native(v)
        out = net(v, n, c4)
    gold = oracle_of(net, v.cpu().numpy(), nn_, c4.cpu().numpy())
    err = rel_err(out.cpu().numpy(), gold)
    print("lidar cloud: M=%d, n<P %d, n==P %d, err %.2e" % (len(nn_), (nn_ < P).sum(), (nn_ == P).sum(), err))
    assert err <= 1e-4


def test_padded_row_decides_the_max(cuda):
    """A large BN shift makes relu(shift1) -- the layer-1 row of the padded slots -- the largest row
    for some channels.  Pillars with n < P must include it, pillars with n == P must not."""
    enc = make_encoder(cuda, seed=2, shift_bias=1.5)
    net = enc.pts_voxel_encoder
    v, c, n = voxelize(lidar(cuda, seed=3))
    c4 = F.pad(c, (1, 0), value=0)
    with torch.no_grad():
        out = net(v, n, c4).cpu().numpy()
    vv, nn_, cc = v.cpu().numpy(), n.cpu().numpy(), c4.cpu().numpy()
    gold = oracle_of(net, vv, nn_, cc)
    assert rel_err(out, gold) <= 1e-4
    part, full = np.nonzero(nn_ < P)[0][:2000], np.nonzero(nn_ == P)[0][:2000]
    assert len(part) and len(full)
    # without the padded row (P = n) the partial pillars change ...
    one = np.nonzero(nn_[part] == 1)[0]
    no_pad = oracle_of(net, vv[part][one][:, :1], nn_[part][one], cc[part][one])
    assert np.abs(no_pad - gold[part][one]).max() > 1e-2 * np.abs(gold).max()
    # ... and adding one to the full pillars (P + 1 slots) changes them
    extra = np.concatenate([vv[full], np.zeros_like(vv[full][:, :1])], axis=1)
    with_pad = oracle_of(net, extra, nn_[full], cc[full])
    assert np.abs(with_pad - gold[full]).max() > 1e-2 * np.abs(gold).max()


def test_forward_points_bit_equal_to_module_path(cuda):
    from bevfusion_b200.voxelize import Voxelization, voxelize_batch
    enc = make_encoder(cuda, seed=4)
    vox = Voxelization(VS, PCR, P, (30000, 60000)).eval()
    clouds = [lidar(cuda, seed=5), lidar(cuda, seed=6)[:150000].contiguous()]
    with torch.no_grad():
        fused = enc.forward_points(clouds, vox)
        feats, coords, sizes = voxelize_batch(clouds, vox, voxelize_reduce=False)
        ref = enc(feats, coords, coords[-1, 0] + 1, sizes)
        again = enc.forward_points(clouds, vox)
    assert tuple(fused.shape) == (2, 64, 512, 512)
    assert bool(torch.equal(fused, ref))
    assert bool(torch.equal(fused, again))
    with torch.no_grad():
        r1 = enc.pts_voxel_encoder(feats, sizes, coords)
        r2 = enc.pts_voxel_encoder(feats, sizes, coords)
    assert bool(torch.equal(r1, r2))


def test_forward_points_cuda_graph(cuda):
    """forward_points has no host synchronisation: captured once on a NaN-padded point buffer (NaN
    points are dropped by the voxelizer), replayed on clouds of different sizes."""
    from bevfusion_b200.voxelize import Voxelization
    enc = make_encoder(cuda, seed=7)
    vox = Voxelization(VS, PCR, P, (30000, 60000)).eval()
    clouds = [lidar(cuda, seed=s)[:k].contiguous() for s, k in ((8, 290000), (9, 200000), (10, 90000))]
    buf = torch.full((max(p.shape[0] for p in clouds) + 1000, 5), float("nan"), device=cuda)
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


def test_train_mode_forward_backward_vs_float64(cuda):
    d = np.load(FIX)
    enc = make_encoder(cuda, seed=11, vs=list(d["voxel_size"]), pcr=list(d["point_cloud_range"])).train()
    enc64 = copy.deepcopy(enc).double()
    x = torch.from_numpy(d["features"]).to(cuda)
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


@pytest.mark.parametrize("case", ["distance", "one_layer", "p40"])
def test_unsupported_shape_takes_torch_path(cuda, case):
    kw = dict(with_distance=True) if case == "distance" else dict(feat_channels=(64,)) if case == "one_layer" else {}
    enc = make_encoder(cuda, seed=12, **kw)
    net = enc.pts_voxel_encoder
    rng = np.random.default_rng(0)
    p = 40 if case == "p40" else P
    m = 300
    num = rng.integers(1, p + 1, size=m).astype(np.int32)
    feats = np.zeros((m, p, 5), np.float32)
    for v in range(m):
        feats[v, :num[v]] = rng.uniform(-2, 2, size=(num[v], 5))
    coors = np.stack([np.zeros(m), rng.integers(0, 512, m), rng.integers(0, 512, m), np.zeros(m)], 1).astype(np.int32)
    t = lambda a: torch.from_numpy(a).to(cuda)
    assert not net._use_native(t(feats))
    with torch.no_grad():
        out = net(t(feats), t(num), t(coors))
    assert rel_err(out.cpu().numpy(), oracle_of(net, feats, num, coors)) <= 1e-4
    if case == "p40":
        with pytest.raises(ValueError):
            from bevfusion_b200.voxelize import Voxelization
            with torch.no_grad():
                enc.forward_points([lidar(cuda)], Voxelization(VS, PCR, 40, (30000, 60000)).eval())


def test_scatter_matches_oracle(cuda):
    d = np.load(FIX)
    from bevfusion_b200.pillar_encoder import PointPillarsScatter
    s = PointPillarsScatter(64, (int(d["nx"]), int(d["ny"])))
    rows = torch.from_numpy(d["A__eval"]).float().to(cuda)
    out = s(rows, torch.from_numpy(d["coors"]).to(cuda), torch.tensor(int(d["batch"])))
    gold = pillars_scatter(d["A__eval"].astype(np.float32), d["coors"], int(d["batch"]), int(d["nx"]), int(d["ny"]))
    assert np.array_equal(out.cpu().numpy(), gold.astype(np.float32))
