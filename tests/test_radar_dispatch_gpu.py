"""GPU tests of the native radar feature net (radar.cu, BF16x3 mma.sync) on every chain, shape and row source it
accepts, against the float64 oracle (tests/radar_oracle.py) fed the module's state_dict.

Both row sources are driven through the C ABI with the test's own buffers:
  * rows   bevb200_radar_features: [M, P, F] voxels -> radar_rows_table_kernel -> radar_tiles_kernel -> [M, C] rows
  * fused  bevb200_hard_voxelize_radar: points -> voxelizer front -> radar_points_table_kernel -> radar_tiles_kernel
           -> [C, nx, ny] canvas
The rows output is NaN-prefilled (the call zeroes it), the canvas zero-prefilled (the caller zeroes it); both sit
between guard words, the workspace has a 4 KiB canary behind it, each call runs twice and must be bit-identical
(atomicMax on int bits), the fused canvas equals the rows form on the same voxelization bit for bit, and
RadarFeatureNet.forward / forward_points return the same bits.  Error bound: 1e-4 of max |float64| (BF16x3 keeps
about 16 significant bits of each operand).

Chains put each of the 8 widths once as a hidden layer and once as the last, at 1..4 layers, widening and narrowing;
F covers layer-0 K of 16 (F = 3, 14), 32 (15, 16), 48 (45) and 128 (126).  Geometry as the pillar tests: 0.16 x 0.2 m
cells on a 440 x 400 grid."""
import ctypes

import numpy as np
import pytest
import torch
from torch.nn import functional as Fn

from bevfusion_b200 import _C
from radar_oracle import layers_from_state_dict, radar_feature_net
from test_pillars_dispatch_gpu import (NORM, NUM_SMS, NX, NY, PCR, VS, cloud, guarded, guards_intact, rows_inputs,
                                       run_twice, same_bits, voxelizer, workspace)

pytestmark = pytest.mark.gpu

EINVAL, EWORKSPACE, EUNSUPPORTED = -1, -3, -4
BOUND = 1e-4
SHIPPED = [128, 128, 128, 64]
TILE_ROWS = NUM_SMS * 8 * 4 * 16            # rows the tile kernel's grid covers before its stride loop (67,584)
# (widths, F, P): every width hidden and last, 1..4 layers, widening and narrowing
CHAINS = [([16], 3, 1), ([32, 48], 14, 2), ([48, 96, 128], 15, 17), ([64, 80, 96], 16, 20),
          ([112, 128, 16, 32], 126, 32), ([128, 80], 45, 17), ([16, 112], 14, 32), (SHIPPED, 45, 20)]
F_SWEEP = [([80, 48], F, 20) for F in (3, 14, 15, 16, 45, 126)]
P_SWEEP = [([32, 112, 64], 15, P) for P in (1, 2, 17, 20, 32)]
CASES = CHAINS + F_SWEEP + P_SWEEP


def case_id(c):
    return "%s-F%d-P%d" % ("x".join(map(str, c[0])), c[1], c[2])


def rel_err(got, ref, what, bound=BOUND):
    got = got.double().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    assert np.isfinite(got).all(), "%s: non-finite output" % what
    err = float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))
    print("[radar %s] max |err| / max |float64| = %.3g" % (what, err))
    assert err <= bound, "%s: %.3g > %.1g" % (what, err, bound)
    return err


# ---------------------------------------------------------------------------------------------------- inputs
def make_encoder(dev, widths, F, seed=0, shift_bias=0.0):
    from bevfusion_b200.radar_encoder import RadarEncoder
    enc = RadarEncoder(
        dict(type="RadarFeatureNet", in_channels=F, feat_channels=list(widths), voxel_size=VS, point_cloud_range=PCR,
             norm_cfg=NORM),
        dict(type="PointPillarsScatter", in_channels=widths[-1], output_shape=[NX, NY]))
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for layer in enc.pts_voxel_encoder.rfn_layers:
            w, bn, u = layer.linear.weight, layer.norm, layer.units
            w.copy_(torch.randn(tuple(w.shape), generator=g) / np.sqrt(w.shape[1]))
            sign = torch.where(torch.rand(u, generator=g) < 0.25, -1.0, 1.0)
            bn.weight.copy_(sign * (0.5 + torch.rand(u, generator=g)))
            bn.bias.copy_(torch.rand(u, generator=g) - 0.5 + shift_bias)
            bn.running_mean.copy_(0.6 * torch.rand(u, generator=g) - 0.3)
            bn.running_var.copy_(0.5 + 1.5 * torch.rand(u, generator=g))
    return enc.to(dev).eval()


def radar_rows(dev, M, P, F, seed, counts=None, lo=(0, 0), hi=(NX, NY), pad=0.0):
    """rows_inputs with n = 0 pillars allowed and `pad` in the slots >= n (never read)."""
    rng = np.random.default_rng(seed + 1)
    if counts is None:
        counts = rng.integers(0, P + 1, M)
        counts[:4] = [0, 1, max(P - 1, 1), P][:M]
    feats, num, coors = rows_inputs(dev, M, P, F, seed, counts=counts, lo=lo, hi=hi)
    feats[torch.arange(P, device=dev)[None, :] >= num[:, None].long()] = pad
    return feats, num, coors


def oracle(net, feats, num, coors):
    sd = {k: v.detach().double().cpu().numpy() for k, v in net.state_dict().items()}
    out, _ = radar_feature_net(feats.cpu().numpy(), num.cpu().numpy(), coors.cpu().numpy(),
                               layers_from_state_dict(sd, "", len(net.rfn_layers)), net.vx, net.vy, net.x_offset,
                               net.y_offset, net.pc_range)
    return out


def widths_arg(widths):
    return (ctypes.c_int * len(widths))(*widths)


# ---------------------------------------------------------------------------------------------------- drivers
def rows_call(net, feats, num, coors, cap, nd, P, F, widths, packed, out, ws, ws_bytes):
    geom, _keep = net._geometry()
    dev = out.device
    return _C.lib().bevb200_radar_features(_C.ptr(feats), _C.ptr(num), _C.ptr(coors), cap, _C.ptr(nd), P, F,
                                           len(widths), widths_arg(widths), *geom, _C.ptr(packed), _C.ptr(out),
                                           _C.ptr(ws), ws_bytes, _C.current_stream(dev))


def rows_driver(net, feats, num, coors, n_dev=None):
    dev = feats.device
    cap, P, F = feats.shape
    widths = [l.units for l in net.rfn_layers]
    nbytes = _C.lib().bevb200_radar_features_workspace_bytes(cap, P)
    ws, pattern = workspace(nbytes, dev)
    buf, out = guarded((cap, widths[-1]), dev)
    nd = None if n_dev is None else torch.tensor([n_dev], dtype=torch.int32, device=dev)
    packed = net.packed_weights()
    fn = lambda: rows_call(net, feats, num, coors, cap, nd, P, F, widths, packed, out, ws, nbytes)
    return run_twice(fn, [(out, float("nan"))], [buf], ws, nbytes, pattern)[0]


def fused_call(net, pts, P, max_voxels, widths, canvas, vnum, ws, ws_bytes, F=None):
    vs, cr = _C.host_array(ctypes.c_float, VS), _C.host_array(ctypes.c_float, PCR)
    geom, _keep = net._geometry()
    return _C.lib().bevb200_hard_voxelize_radar(
        _C.ptr(pts), int(pts.shape[0]), int(pts.shape[1]) if F is None else F, ctypes.cast(vs, ctypes.c_void_p),
        ctypes.cast(cr, ctypes.c_void_p), P, max_voxels, len(widths), widths_arg(widths), *geom,
        _C.ptr(net.packed_weights()), _C.ptr(canvas), NX, NY, _C.ptr(vnum), _C.ptr(ws), ws_bytes,
        _C.current_stream(canvas.device))


def fused_driver(net, pts, P, max_voxels):
    dev = pts.device
    widths = [l.units for l in net.rfn_layers]
    nbytes = _C.lib().bevb200_hard_voxelize_radar_workspace_bytes(int(pts.shape[0]), P)
    ws, pattern = workspace(nbytes, dev)
    buf, canvas = guarded((widths[-1], NX, NY), dev)
    vnum = torch.empty(1, dtype=torch.int32, device=dev)
    got, vn = run_twice(lambda: fused_call(net, pts, P, max_voxels, widths, canvas, vnum, ws, nbytes),
                        [(canvas, 0.0), (vnum, -7)], [buf], ws, nbytes, pattern)
    return got, int(vn[0])


def check_rows(enc, feats, num, coors, what, n_dev=None):
    net = enc.pts_voxel_encoder
    got = rows_driver(net, feats, num, coors, n_dev)
    err = rel_err(got, oracle(net, feats, num, coors), what)
    with torch.no_grad():
        assert net._use_native(feats)
        assert same_bits(net(feats, num, coors), got), "RadarFeatureNet.forward differs from the C ABI"
    return got, err


def check_fused(enc, pts, P, max_voxels, what):
    """fused canvas == rows form on the same voxelization scattered into zeros (bit for bit), rows vs float64,
    forward_points returns the same bits and voxel_num"""
    net = enc.pts_voxel_encoder
    C = net.rfn_layers[-1].units
    vox = voxelizer(P, max_voxels)
    with torch.no_grad():
        v, c, n = vox(pts)
    M = int(n.shape[0])
    got, vnum = fused_driver(net, pts, P, max_voxels)
    assert vnum == M
    expect = torch.zeros((C, NX, NY), device=pts.device)
    err = 0.0
    if M:
        c4 = Fn.pad(c, (1, 0), value=0)
        rows = rows_driver(net, v, n, c4)
        err = rel_err(rows, oracle(net, v, n, c4), what)
        cl = c.long()
        expect[:, cl[:, 0], cl[:, 1]] = rows.t()
    assert same_bits(got, expect), "fused canvas differs from the rows form on the same voxelization"
    with torch.no_grad():
        py, pvn = enc.forward_points([pts], vox, return_voxel_num=True)
    assert same_bits(py[0], got) and int(pvn[0]) == M, "forward_points differs from the C ABI"
    return n.cpu().numpy(), err


# ---------------------------------------------------------------------------------------------------- matrix
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_rows_every_chain(cuda, case):
    """Rows form: pillars of 0, 1, P - 1 and P points (n = 0 gets the virtual row alone)."""
    widths, F, P = case
    enc = make_encoder(cuda, widths, F, seed=F + P + len(widths))
    feats, num, coors = radar_rows(cuda, 600, P, F, seed=F * 7 + P)
    check_rows(enc, feats, num, coors, "rows " + case_id(case))


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_fused_every_chain(cuda, case):
    widths, F, P = case
    enc = make_encoder(cuda, widths, F, seed=F + P + len(widths) + 1)
    pts = cloud(cuda, 5000, F, P, seed=F * 7 + P)
    n, _ = check_fused(enc, pts, P, 30000, "fused " + case_id(case))
    assert (n == 1).any() and (n == P).any()


def test_chains_cover_every_width_hidden_and_last():
    hidden = {w for c, _, _ in CHAINS for w in c[:-1]}
    last = {c[-1] for c, _, _ in CHAINS}
    assert hidden == last == set(range(16, 129, 16))
    assert {len(c) for c, _, _ in CHAINS} == {1, 2, 3, 4}
    assert any(a < b for c, _, _ in CHAINS for a, b in zip(c, c[1:]))
    assert any(a > b for c, _, _ in CHAINS for a, b in zip(c, c[1:]))
    assert {(F + 2 + 15) // 16 * 16 for _, F, _ in CASES} == {16, 32, 48, 128}


# ---------------------------------------------------------------------------------------------------- row counts
TOTALS = {"1": [1], "15": [5, 0, 10], "16": [9, 7], "17": [1] * 17,
          "span": [8, 32, 32, 3, 29, 0, 16]}       # rows 8..39 cross tiles 0-2, 40..71 tiles 2-4


@pytest.mark.parametrize("name", list(TOTALS))
def test_rows_total_rows_and_tile_spans(cuda, name):
    """Total rows of 1, 15, 16 and 17, and pillars crossing two and three 16-row tiles.  All pillars sit in one warp
    of the table kernel, so their rows are laid out in pillar order."""
    counts = TOTALS[name]
    P = 32
    enc = make_encoder(cuda, [48, 32], 14, seed=len(counts))
    feats, num, coors = radar_rows(cuda, len(counts), P, 14, seed=len(counts), counts=counts)
    if name != "span":
        assert sum(counts) == int(name)
    check_rows(enc, feats, num, coors, "rows total %s" % name)


def test_rows_tile_stride_loop(cuda):
    """4000 pillars of n = P = 32: 128,000 rows, past the 67,584 the tile kernel's grid holds."""
    enc = make_encoder(cuda, [64, 32], 16, seed=21)
    feats, num, coors = radar_rows(cuda, 4000, 32, 16, seed=21, counts=np.full(4000, 32))
    assert 4000 * 32 > TILE_ROWS
    check_rows(enc, feats, num, coors, "rows 128000 rows stride loop")


def test_fused_large_cloud(cuda):
    """A cloud whose real rows exceed the tile kernel's grid and whose 32-point words exceed the table kernel's."""
    enc = make_encoder(cuda, [96, 48], 14, seed=22)
    n_pts = NUM_SMS * 16 * 8 * 32 + 20000
    pts = cloud(cuda, n_pts, 14, 32, seed=22, hot=100, region=(90, 70), spread=2000)
    n, _ = check_fused(enc, pts, 32, 60000, "fused %d points stride loops" % n_pts)
    assert int(np.minimum(n, 32).sum()) > TILE_ROWS


# ---------------------------------------------------------------------------------------------------- header claims
def test_rows_padded_slots_never_read(cuda):
    """NaN in slots >= n changes nothing, bit for bit."""
    enc = make_encoder(cuda, [64, 80, 96], 16, seed=23)
    net = enc.pts_voxel_encoder
    feats, num, coors = radar_rows(cuda, 500, 20, 16, seed=23)
    nan_feats, _, _ = radar_rows(cuda, 500, 20, 16, seed=23, pad=float("nan"))
    assert bool(torch.isnan(nan_feats).any())
    assert same_bits(rows_driver(net, nan_feats, num, coors), rows_driver(net, feats, num, coors))


def test_rows_n_dev(cuda):
    """out_rows is zeroed; pillars v < min(*n_dev, cap) are computed, rows at or past *n_dev are 0."""
    enc = make_encoder(cuda, [128, 80], 45, seed=24)
    net = enc.pts_voxel_encoder
    feats, num, coors = radar_rows(cuda, 300, 20, 45, seed=24)
    full = rows_driver(net, feats, num, coors)
    for nd in (0, 1, 123, 299, 300, 1000):
        got = rows_driver(net, feats, num, coors, n_dev=nd)
        k = min(nd, 300)
        assert same_bits(got[:k], full[:k]), nd
        assert bool((got[k:] == 0).all()) and not bool(torch.signbit(got[k:]).any()), nd


@pytest.mark.parametrize("widths,F", [(SHIPPED, 45), ([16, 112], 14)])
def test_rows_coordinates_past_int16(cuda, widths, F):
    """Pillar indices in [32768, 60000] on both axes: the centre offsets use the full coordinates."""
    enc = make_encoder(cuda, widths, F, seed=25)
    feats, num, coors = radar_rows(cuda, 500, 20, F, seed=25, lo=(32768, 32768), hi=(60001, 60001))
    check_rows(enc, feats, num, coors, "rows coords >= 32768 %s" % "x".join(map(str, widths)))


def test_fused_max_voxels_binding(cuda):
    """A non-shipped chain, F and P with max_voxels below the pillar count: voxel_num is the cap and the canvas holds
    the first max_voxels pillars."""
    enc = make_encoder(cuda, [112, 128, 16, 32], 15, seed=26)
    pts = cloud(cuda, 8000, 15, 17, seed=26)
    with torch.no_grad():
        total = int(voxelizer(17, 100000)(pts)[2].shape[0])
    n, _ = check_fused(enc, pts, 17, 350, "fused max_voxels=350 of %d" % total)
    assert total > 350 and n.size == 350


@pytest.mark.parametrize("case", ["empty", "out_of_range"])
def test_fused_no_pillar(cuda, case):
    enc = make_encoder(cuda, [32, 48], 14, seed=27)
    if case == "empty":
        pts = torch.zeros((0, 14), device=cuda)
    else:
        pts = cloud(cuda, 500, 14, 20, seed=27, hot=5).clone()
        pts[:, 1] = 45.0
    got, vnum = fused_driver(enc.pts_voxel_encoder, pts, 20, 30000)
    assert vnum == 0 and not bool(got.any())


# ---------------------------------------------------------------------------------------------------- refusals
def test_refusals_leave_outputs_untouched(cuda):
    """Just outside the accepted space (widths 8, 100 and 144, five layers, F = 2 and 127, P = 0 and 33) both forms
    return BEVB200_EUNSUPPORTED and write nothing, and native_supported / _use_native agree with the C gate there and
    at the accepted corners; a workspace one byte short is refused and writes nothing."""
    from bevfusion_b200.radar_encoder import RadarFeatureNet
    enc = make_encoder(cuda, [32, 48], 14, seed=28)
    net = enc.pts_voxel_encoder
    packed = net.packed_weights()
    pts = cloud(cuda, 3000, 14, 20, seed=28)
    probes = [([8], 14, 20), ([128, 100], 14, 20), ([144], 14, 20), ([64] * 5, 14, 20), ([64], 127, 20),
              ([64], 2, 20), ([64], 14, 0), ([64], 14, 33),
              ([16], 3, 1), ([128] * 4, 126, 32)]
    for widths, F, P in probes:
        ok = (1 <= len(widths) <= 4 and all(w % 16 == 0 and 16 <= w <= 128 for w in widths) and 3 <= F <= 126
              and 1 <= P <= 32)
        probe = RadarFeatureNet(F, widths, voxel_size=VS, point_cloud_range=PCR, norm_cfg=NORM).to(cuda).eval()
        feats = torch.zeros((40, P, F), device=cuda)
        with torch.no_grad():
            assert probe.native_supported(P) == ok and probe._use_native(feats) == ok, (widths, F, P)
        if ok:
            continue
        num = torch.ones(40, dtype=torch.int32, device=cuda)
        coors = torch.zeros((40, 4), dtype=torch.int32, device=cuda)
        buf, out = guarded((40, widths[-1]), cuda)
        out.fill_(float("nan"))
        ws = torch.empty(1 << 20, dtype=torch.uint8, device=cuda)
        rc = rows_call(net, feats, num, coors, 40, None, P, F, widths, packed, out, ws, ws.numel())
        torch.cuda.synchronize()
        assert rc == EUNSUPPORTED and bool(torch.isnan(out).all()) and guards_intact(buf), (widths, F, P, rc)
        p = torch.zeros((100, max(F, 3)), device=cuda)
        p[:, :3] = pts[:100, :3]
        buf, canvas = guarded((widths[-1], NX, NY), cuda)
        canvas.fill_(float("nan"))
        vnum = torch.full((1,), -7, dtype=torch.int32, device=cuda)
        rc = fused_call(net, p, P, 30000, widths, canvas, vnum, ws, ws.numel(), F)
        torch.cuda.synchronize()
        assert rc == EUNSUPPORTED and bool(torch.isnan(canvas).all()) and int(vnum[0]) == -7, (widths, F, P, rc)
    L = _C.lib()
    widths = [32, 48]
    feats, num, coors = radar_rows(cuda, 200, 20, 14, seed=28)
    need = L.bevb200_radar_features_workspace_bytes(200, 20)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda)
    buf, out = guarded((200, 48), cuda)
    out.fill_(float("nan"))
    rc = rows_call(net, feats, num, coors, 200, None, 20, 14, widths, packed, out, ws, need - 1)
    torch.cuda.synchronize()
    assert rc in (EINVAL, EWORKSPACE) and bool(torch.isnan(out).all()) and guards_intact(buf), rc
    need = L.bevb200_hard_voxelize_radar_workspace_bytes(int(pts.shape[0]), 20)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda)
    buf, canvas = guarded((48, NX, NY), cuda)
    canvas.fill_(float("nan"))
    vnum = torch.full((1,), -7, dtype=torch.int32, device=cuda)
    rc = fused_call(net, pts, 20, 30000, widths, canvas, vnum, ws, need - 1)
    torch.cuda.synchronize()
    assert rc in (EINVAL, EWORKSPACE) and bool(torch.isnan(canvas).all()) and int(vnum[0]) == -7, rc


# ---------------------------------------------------------------------------------------------------- BN re-fold
def test_bn_refold_after_train_mode_forward(cuda):
    """eval native forward, train-mode forwards under no_grad (BN recalibration: the statistics move, no parameter
    does), eval again: the native forward follows the new statistics."""
    enc = make_encoder(cuda, SHIPPED, 45, seed=29)
    net = enc.pts_voxel_encoder
    feats, num, coors = radar_rows(cuda, 600, 20, 45, seed=29)
    before = oracle(net, feats, num, coors)
    with torch.no_grad():
        rel_err(net(feats, num, coors), before, "BN re-fold, before")
        net.train()
        for _ in range(3):
            net(feats, num, coors)
        net.eval()
        got = net(feats, num, coors)
    after = oracle(net, feats, num, coors)
    moved = float(np.abs(after - before).max() / np.abs(before).max())
    assert moved > 100 * BOUND, "the statistics moved too little for a stale fold to show (%.2g)" % moved
    rel_err(got, after, "BN re-fold, after the train-mode forwards (they moved the output by %.2g)" % moved)
