"""GPU tests of the native pillar feature net (pillars.cu) on every shape and row source it accepts, against the float64
oracle (tests/pillars_oracle.py) fed the module's state_dict.

Both row sources are driven through the C ABI with the test's own buffers:
  * rows   bevb200_pillar_features: [M, P, F] voxels -> [M, 64] rows (pillar_rows_kernel)
  * fused  bevb200_hard_voxelize_pillars: points -> voxelizer front -> pillar_canvas_kernel -> [64, nx, ny] canvas
Every output is NaN-prefilled and sits between guard words, the workspace has a 4 KiB canary behind it, each call runs
twice and must be bit-identical (exact fp32, no atomics), and PillarFeatureNet.forward / forward_points must return the
same bits.  The rows form writes exactly rows v < min(*n_dev, cap); the fused form writes exactly its pillars' cells,
and equals the rows form on the same voxelization bit for bit.  Error bound: 1e-5 of max |float64| (fp32 FMA
throughout).

Geometry: x 0..70.4 m at 0.16 m, y -40..40 m at 0.2 m (a 440 x 400 grid), so a swap of vx / vy, of x_off / y_off or of
the canvas axes fails."""
import ctypes

import numpy as np
import pytest
import torch
from torch.nn import functional as Fn

from bevfusion_b200 import _C
from pillars_oracle import layers_from_state_dict, pillar_feature_net

pytestmark = pytest.mark.gpu

EWORKSPACE, EUNSUPPORTED = -3, -4
VS, PCR = [0.16, 0.2, 4.0], [0.0, -40.0, -3.0, 70.4, 40.0, 1.0]
NX, NY = 440, 400
NORM = dict(type="BN1d", eps=1e-3, momentum=0.01)
BOUND = 1e-5
FS, PS = (3, 4, 5, 8), (1, 2, 20, 31, 32)
NUM_SMS, WARPS = 132, 4
CANVAS_WORDS = NUM_SMS * 16 * WARPS          # 32-point words the canvas kernel covers before its stride loop
ROWS_PILLARS = NUM_SMS * 16 * WARPS          # pillars the rows kernel covers before its stride loop
CANARY = 4096
GUARD = 1024
GUARD_BITS = int(np.array([0xffc0dead], np.uint32).view(np.int32)[0])   # a negative NaN: no store leaves it


# ---------------------------------------------------------------------------------------------------- harness
def guarded(shape, dev):
    """(buffer, view): `shape` fp32 between two GUARD-word guards."""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), GUARD_BITS, dtype=torch.int32, device=dev).view(torch.float32)
    return buf, buf[GUARD:GUARD + n].view(shape)


def guards_intact(buf):
    b = buf.view(torch.int32)
    return bool((b[:GUARD] == GUARD_BITS).all()) and bool((b[-GUARD:] == GUARD_BITS).all())


def workspace(nbytes, dev):
    ws = torch.empty(int(nbytes) + CANARY, dtype=torch.uint8, device=dev)
    pattern = ((torch.arange(CANARY, device=dev) * 7 + 3) % 256).to(torch.uint8)
    ws[int(nbytes):] = pattern
    return ws, pattern


def run_twice(fn, prefill, guards=(), ws=None, nbytes=0, pattern=None):
    """fn() twice, each over fresh prefills [(tensor, value)]: both succeed and agree bit for bit, the guards and the
    workspace canary are intact.  Returns clones of the prefilled tensors after the first run."""
    res = []
    for _ in range(2):
        for t, v in prefill:
            t.fill_(v)
        torch.cuda.synchronize()
        rc = fn()
        torch.cuda.synchronize()
        assert rc == 0, _C.lib().bevb200_last_error()
        res.append([t.clone() for t, _ in prefill])
    for a, b in zip(*res):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "not bit-reproducible"
    for g in guards:
        assert guards_intact(g), "a write outside the output"
    if ws is not None:
        assert torch.equal(ws[nbytes:], pattern), "workspace canary overwritten"
    return res[0]


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def rel_err(got, ref, what, bound=BOUND):
    got = got.double().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    assert np.isfinite(got).all(), "%s: non-finite output" % what
    err = float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))
    print("[pillars %s] max |err| / max |float64| = %.3g" % (what, err))
    assert err <= bound, "%s: %.3g > %.1g" % (what, err, bound)
    return err


# ---------------------------------------------------------------------------------------------------- inputs
def make_encoder(dev, F, seed=0, shift_bias=0.0):
    from bevfusion_b200.pillar_encoder import PointPillarsEncoder
    enc = PointPillarsEncoder(
        dict(type="PillarFeatureNet", in_channels=F, feat_channels=[64, 64], voxel_size=VS, point_cloud_range=PCR,
             norm_cfg=NORM),
        dict(type="PointPillarsScatter", in_channels=64, output_shape=[NX, NY]))
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for layer in enc.pts_voxel_encoder.pfn_layers:
            w, bn, u = layer.linear.weight, layer.norm, layer.units
            w.copy_(torch.randn(tuple(w.shape), generator=g) / np.sqrt(w.shape[1]))
            sign = torch.where(torch.rand(u, generator=g) < 0.25, -1.0, 1.0)
            bn.weight.copy_(sign * (0.5 + torch.rand(u, generator=g)))
            bn.bias.copy_(torch.rand(u, generator=g) - 0.5 + shift_bias)
            bn.running_mean.copy_(0.6 * torch.rand(u, generator=g) - 0.3)
            bn.running_var.copy_(0.5 + 1.5 * torch.rand(u, generator=g))
    return enc.to(dev).eval()


def rows_inputs(dev, M, P, F, seed, counts=None, lo=(0, 0), hi=(NX, NY)):
    """[M, P, F] voxels of points inside their pillars (x, y, z), N(0, 1) extra features; padded slots hold finite
    non-zero values (the reference's mean sums all P slots).  Counts include 1, P - 1 and P unless given."""
    rng = np.random.default_rng(seed)
    if counts is None:
        counts = rng.integers(1, P + 1, M)
        counts[:3] = [1, max(P - 1, 1), P][:M]
    num = np.asarray(counts, np.int32)
    cx, cy = rng.integers(lo[0], hi[0], M), rng.integers(lo[1], hi[1], M)
    coors = np.stack([rng.integers(0, 2, M), cx, cy, np.zeros(M, np.int64)], 1).astype(np.int32)
    x = (cx[:, None] + rng.random((M, P))) * VS[0] + PCR[0]
    y = (cy[:, None] + rng.random((M, P))) * VS[1] + PCR[1]
    z = rng.uniform(PCR[2], PCR[5], (M, P))
    feats = np.concatenate([np.stack([x, y, z], 2), rng.standard_normal((M, P, F - 3))], 2).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return t(feats), t(num), t(coors)


def cloud(dev, n, F, P, seed, hot=60, region=(40, 40), spread=0):
    """n points: `hot` cells with P .. P + 19 points (pillars at and over the cap), the rest uniform over a region x
    region cell block (pillars of 1 .. P - 1 points) and `spread` over the whole grid (mostly single points); 2% of the
    points out of range on one of the axes; shuffled."""
    rng = np.random.default_rng(seed)
    k = rng.integers(P, P + 20, hot)
    cx = [np.repeat(rng.integers(0, NX, hot), k)]
    cy = [np.repeat(rng.integers(0, NY, hot), k)]
    rest = n - int(k.sum()) - spread
    assert rest >= 0
    x0, y0 = rng.integers(0, NX - region[0]), rng.integers(0, NY - region[1])
    cx += [x0 + rng.integers(0, region[0], rest), rng.integers(0, NX, spread)]
    cy += [y0 + rng.integers(0, region[1], rest), rng.integers(0, NY, spread)]
    cx, cy = np.concatenate(cx), np.concatenate(cy)
    pts = np.zeros((n, F), np.float32)
    pts[:, 0] = (cx + rng.uniform(0.02, 0.98, n)) * VS[0] + PCR[0]
    pts[:, 1] = (cy + rng.uniform(0.02, 0.98, n)) * VS[1] + PCR[1]
    pts[:, 2] = rng.uniform(PCR[2] + 0.01, PCR[5] - 0.01, n)
    pts[:, 3:] = rng.standard_normal((n, F - 3))
    out = rng.choice(n, n // 50, replace=False)
    axis = rng.integers(0, 3, out.size)
    pts[out, axis] = np.where(rng.random(out.size) < 0.5, -100.0, 100.0)
    return torch.from_numpy(pts[rng.permutation(n)]).to(dev)


def oracle(net, feats, num, coors):
    sd = {k: v.detach().double().cpu().numpy() for k, v in net.state_dict().items()}
    out, _ = pillar_feature_net(feats.cpu().numpy(), num.cpu().numpy(), coors.cpu().numpy(),
                                layers_from_state_dict(sd, "", 2), net.vx, net.vy, net.x_offset, net.y_offset)
    return out


def voxelizer(P, max_voxels):
    from bevfusion_b200.voxelize import Voxelization
    return Voxelization(VS, PCR, P, (max_voxels, max_voxels)).eval()


# ---------------------------------------------------------------------------------------------------- drivers
def rows_driver(net, feats, num, coors, n_dev=None):
    L = _C.lib()
    dev = feats.device
    cap, P, F = feats.shape
    buf, out = guarded((cap, 64), dev)
    packed = net.packed_weights()
    nd = None if n_dev is None else torch.tensor([n_dev], dtype=torch.int32, device=dev)
    fn = lambda: L.bevb200_pillar_features(_C.ptr(feats), _C.ptr(num), _C.ptr(coors), cap, _C.ptr(nd), P, F,
                                           *net._geometry(), _C.ptr(packed), _C.ptr(out), _C.current_stream(dev))
    return run_twice(fn, [(out, float("nan"))], [buf])[0]


def fused_call(net, pts, P, max_voxels, canvas, vnum, ws, ws_bytes, F=None):
    vs, cr = _C.host_array(ctypes.c_float, VS), _C.host_array(ctypes.c_float, PCR)
    dev = canvas.device
    return _C.lib().bevb200_hard_voxelize_pillars(
        _C.ptr(pts), int(pts.shape[0]), int(pts.shape[1]) if F is None else F, ctypes.cast(vs, ctypes.c_void_p),
        ctypes.cast(cr, ctypes.c_void_p), P, max_voxels, *net._geometry(), _C.ptr(net.packed_weights()),
        _C.ptr(canvas), NX, NY, _C.ptr(vnum), _C.ptr(ws), ws_bytes, _C.current_stream(dev))


def fused_driver(net, pts, P, max_voxels):
    """-> (canvas [64, NX, NY], NaN where not written; voxel_num)"""
    dev = pts.device
    nbytes = _C.lib().bevb200_hard_voxelize_workspace_bytes(int(pts.shape[0]), P)
    ws, pattern = workspace(nbytes, dev)
    buf, canvas = guarded((64, NX, NY), dev)
    vnum = torch.empty(1, dtype=torch.int32, device=dev)
    got, vn = run_twice(lambda: fused_call(net, pts, P, max_voxels, canvas, vnum, ws, nbytes),
                        [(canvas, float("nan")), (vnum, -7)], [buf], ws, nbytes, pattern)
    return got, int(vn[0])


def check_rows(enc, feats, num, coors, what):
    """rows form vs float64 and vs PillarFeatureNet.forward"""
    net = enc.pts_voxel_encoder
    got = rows_driver(net, feats, num, coors)
    err = rel_err(got, oracle(net, feats, num, coors), what)
    with torch.no_grad():
        assert net._use_native(feats)
        assert same_bits(net(feats, num, coors), got), "PillarFeatureNet.forward differs from the C ABI"
    return got, err


def check_fused(enc, pts, P, max_voxels, what):
    """fused form == rows form on the same voxelization (bit for bit, unwritten cells NaN), rows vs float64, and
    forward_points returns the same bits with every other cell +0."""
    net = enc.pts_voxel_encoder
    vox = voxelizer(P, max_voxels)
    with torch.no_grad():
        v, c, n = vox(pts)
    M = int(n.shape[0])
    c4 = Fn.pad(c, (1, 0), value=0)
    got, vnum = fused_driver(net, pts, P, max_voxels)
    assert vnum == M
    expect = torch.full((64, NX, NY), float("nan"), device=pts.device)
    err = 0.0
    if M:
        rows = rows_driver(net, v, n, c4)
        err = rel_err(rows, oracle(net, v, n, c4), what)
        cl = c.long()
        expect[:, cl[:, 0], cl[:, 1]] = rows.t()
    assert same_bits(got, expect), "fused canvas differs from the rows form on the same voxelization"
    with torch.no_grad():
        py = enc.forward_points([pts], vox)[0]
    written = ~torch.isnan(expect)
    assert same_bits(py[written], got[written]), "forward_points differs from the C ABI"
    empty = py[~written]
    assert bool((empty == 0).all()) and not bool(torch.signbit(empty).any()), "a cell without pillar is not +0"
    return n.cpu().numpy(), err


# ---------------------------------------------------------------------------------------------------- shape matrix
@pytest.mark.parametrize("P", PS)
@pytest.mark.parametrize("F", FS)
def test_rows_every_shape(cuda, F, P):
    """Rows form at every F and P: pillars with n = 1, P - 1 and P, finite non-zero values in the padded slots."""
    enc = make_encoder(cuda, F, seed=F * 100 + P)
    feats, num, coors = rows_inputs(cuda, 700, P, F, seed=P + 10 * F)
    check_rows(enc, feats, num, coors, "rows F=%d P=%d" % (F, P))


@pytest.mark.parametrize("P", PS)
@pytest.mark.parametrize("F", FS)
def test_fused_every_shape(cuda, F, P):
    """Fused form at every F and P on a cloud with pillars of 1 point, of 1 .. P - 1 points, of P and of more."""
    enc = make_encoder(cuda, F, seed=F * 100 + P + 1)
    pts = cloud(cuda, 6000, F, P, seed=P + 10 * F)
    n, _ = check_fused(enc, pts, P, 30000, "fused F=%d P=%d" % (F, P))
    assert (n == 1).any() and (n == P).any() and (P <= 2 or ((n > 1) & (n < P)).any())


@pytest.mark.parametrize("P", [31, 32])
def test_virtual_row_decides_the_max(cuda, P):
    """A large BN shift makes the padded slots' layer-1 row relu(t1) the largest for some channels.  Pillars with
    n = P - 1 (the virtual row in the last slot) and n = 1 must include it, pillars with n = P must not."""
    enc = make_encoder(cuda, 4, seed=P, shift_bias=1.5)
    net = enc.pts_voxel_encoder
    feats, num, coors = rows_inputs(cuda, 600, P, 4, seed=P, counts=np.resize([1, P - 1, P], 600))
    got, _ = check_rows(enc, feats, num, coors, "rows virtual row P=%d" % P)
    got = got.double().cpu().numpy()
    for n in (1, P - 1):     # without the virtual row (P = n slots) these pillars change, far beyond the error bound
        sel = torch.nonzero(num == n)[:, 0]
        no_pad = oracle(net, feats[sel][:, :n], num[sel], coors[sel])
        assert np.abs(no_pad - got[sel.cpu().numpy()]).max() > 100 * BOUND * np.abs(got).max(), n


# ---------------------------------------------------------------------------------------------------- edges
def test_rows_n_dev(cuda):
    """Pillars v < min(*n_dev, cap) are computed, rows at or past *n_dev stay untouched (NaN)."""
    enc = make_encoder(cuda, 5, seed=3)
    net = enc.pts_voxel_encoder
    feats, num, coors = rows_inputs(cuda, 300, 20, 5, seed=3)
    full = rows_driver(net, feats, num, coors)
    for nd in (0, 1, 123, 299, 300, 1000):
        got = rows_driver(net, feats, num, coors, n_dev=nd)
        k = min(nd, 300)
        assert same_bits(got[:k], full[:k]), nd
        assert bool(torch.isnan(got[k:]).all()), "row past *n_dev = %d written" % nd


def test_rows_coordinates_past_int16(cuda):
    """Pillar indices in [32768, 60000] on both axes (any coors the rows form is given)."""
    enc = make_encoder(cuda, 5, seed=5)
    feats, num, coors = rows_inputs(cuda, 500, 20, 5, seed=5, lo=(32768, 32768), hi=(60001, 60001))
    check_rows(enc, feats, num, coors, "rows coords >= 32768")


def test_rows_stride_loop(cuda):
    """More pillars than the rows kernel's grid holds warps: the grid-stride loop."""
    enc = make_encoder(cuda, 4, seed=6)
    M = ROWS_PILLARS + 1500
    feats, num, coors = rows_inputs(cuda, M, 20, 4, seed=6)
    check_rows(enc, feats, num, coors, "rows M=%d stride loop" % M)


def test_fused_max_voxels_binding(cuda):
    """max_voxels below the pillar count: voxel_num is the cap and the canvas holds the first max_voxels pillars."""
    enc = make_encoder(cuda, 5, seed=7)
    pts = cloud(cuda, 8000, 5, 20, seed=7)
    with torch.no_grad():
        total = int(voxelizer(20, 100000)(pts)[2].shape[0])
    n, _ = check_fused(enc, pts, 20, 400, "fused max_voxels=400 of %d" % total)
    assert total > 400 and n.size == 400


@pytest.mark.parametrize("case", ["empty", "out_of_range"])
def test_fused_no_pillar(cuda, case):
    """No point, or none in range: voxel_num 0 and nothing written; forward_points gives a zero canvas."""
    enc = make_encoder(cuda, 5, seed=8)
    if case == "empty":
        pts = torch.zeros((0, 5), device=cuda)
    else:
        pts = cloud(cuda, 500, 5, 20, seed=8, hot=5).clone()
        pts[:, 0] = 75.0
    got, vnum = fused_driver(enc.pts_voxel_encoder, pts, 20, 30000)
    assert vnum == 0 and bool(torch.isnan(got).all())
    with torch.no_grad():
        py = enc.forward_points([pts], voxelizer(20, 30000))
    assert not bool(py.any())


def test_fused_stride_loop(cuda):
    """A cloud of more 32-point words than the canvas kernel's grid holds warps (and more pillars than the rows kernel's
    grid): both grid-stride loops, against each other and float64."""
    enc = make_encoder(cuda, 5, seed=9)
    n_pts = CANVAS_WORDS * 32 + 30000
    pts = cloud(cuda, n_pts, 5, 20, seed=9, hot=200, region=(110, 90), spread=3000)
    n, _ = check_fused(enc, pts, 20, 60000, "fused %d points stride loop" % n_pts)
    assert n.size > ROWS_PILLARS


# ---------------------------------------------------------------------------------------------------- refusals
def test_refusals_leave_outputs_untouched(cuda):
    """Just outside the accepted space (F 2 and 9, P 0 and 33) both forms return BEVB200_EUNSUPPORTED and write
    nothing; native_supported / _use_native agree with the C gate there and at the accepted corners; a fused
    workspace one byte short gives BEVB200_EWORKSPACE and writes nothing."""
    from bevfusion_b200.pillar_encoder import PillarFeatureNet
    L = _C.lib()
    enc = make_encoder(cuda, 5, seed=10)
    net = enc.pts_voxel_encoder
    packed = net.packed_weights()
    pts = cloud(cuda, 3000, 5, 20, seed=10)
    for F, P in [(2, 20), (9, 20), (5, 0), (5, 33), (3, 1), (8, 32)]:
        ok = 3 <= F <= 8 and 1 <= P <= 32
        probe = PillarFeatureNet(F, [64, 64], voxel_size=VS, point_cloud_range=PCR, norm_cfg=NORM).to(cuda).eval()
        feats = torch.zeros((40, P, F), device=cuda)
        with torch.no_grad():
            assert probe.native_supported(P) == ok and probe._use_native(feats) == ok, (F, P)
        if ok:
            continue
        num = torch.ones(40, dtype=torch.int32, device=cuda)
        coors = torch.zeros((40, 4), dtype=torch.int32, device=cuda)
        buf, out = guarded((40, 64), cuda)
        out.fill_(float("nan"))
        rc = L.bevb200_pillar_features(_C.ptr(feats), _C.ptr(num), _C.ptr(coors), 40, None, P, F, *net._geometry(),
                                       _C.ptr(packed), _C.ptr(out), _C.current_stream(cuda))
        torch.cuda.synchronize()
        assert rc == EUNSUPPORTED and bool(torch.isnan(out).all()) and guards_intact(buf), (F, P, rc)
        p = torch.zeros((100, max(F, 3)), device=cuda)
        p[:, :3] = pts[:100, :3]
        buf, canvas = guarded((64, NX, NY), cuda)
        canvas.fill_(float("nan"))
        vnum = torch.full((1,), -7, dtype=torch.int32, device=cuda)
        ws = torch.empty(1 << 20, dtype=torch.uint8, device=cuda)
        rc = fused_call(net, p, P, 30000, canvas, vnum, ws, ws.numel(), F)
        torch.cuda.synchronize()
        assert rc == EUNSUPPORTED and bool(torch.isnan(canvas).all()) and int(vnum[0]) == -7, (F, P, rc)
    need = L.bevb200_hard_voxelize_workspace_bytes(int(pts.shape[0]), 20)
    buf, canvas = guarded((64, NX, NY), cuda)
    canvas.fill_(float("nan"))
    vnum = torch.full((1,), -7, dtype=torch.int32, device=cuda)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda)
    rc = fused_call(net, pts, 20, 30000, canvas, vnum, ws, need - 1)
    torch.cuda.synchronize()
    assert rc == EWORKSPACE and bool(torch.isnan(canvas).all()) and int(vnum[0]) == -7 and guards_intact(buf)


# ---------------------------------------------------------------------------------------------------- BN re-fold
def test_bn_refold_after_train_mode_forward(cuda):
    """eval native forward, train-mode forwards under no_grad (BN recalibration: the statistics move, no parameter
    does), eval again: the native forward follows the new statistics."""
    enc = make_encoder(cuda, 5, seed=11)
    net = enc.pts_voxel_encoder
    feats, num, coors = rows_inputs(cuda, 600, 20, 5, seed=11)
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
