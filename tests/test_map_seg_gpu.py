"""The map-segmentation head on the H100: the grid transform forward and backward against the float64 oracle (run
as float64 matmuls on the device) and against torch's F.interpolate + F.grid_sample lines on CUDA; the per-class
losses and gradients against the oracle and the reference fixture; the IoU counts exactly against numpy and the
reference's evaluate_map; the drop-in head; launch counts, repeatability, a sync-free deterministic training step and
one CUDA graph of a whole training step."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import map_seg_oracle as O  # noqa: E402
from bevfusion_b200 import _C  # noqa: E402
from bevfusion_b200 import map_seg as MS  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden", "map_seg_tiny.npz")
EPS32 = 2.0 ** -23
EPS16 = 2.0 ** -10
FIX_IN = [[-6.4, 6.4, 0.8], [-4.8, 4.8, 0.8]]
FIX_OUT = [[-6.0, 6.0, 0.5], [-4.0, 4.0, 0.5]]
FIX_WIDE = [[-8.0, 8.0, 0.5], [-5.0, 6.0, 0.5]]
# name -> (input_scope, output_scope, prescale, H, W)
GEOMS = {
    "default": (S.MAP_SEG_CFG["input_scope"], S.MAP_SEG_CFG["output_scope"], 1, 128, 128),
    "p1": (FIX_IN, FIX_OUT, 1, 16, 12), "p2": (FIX_IN, FIX_OUT, 2, 16, 12), "p05": (FIX_IN, FIX_OUT, 0.5, 16, 12),
    "p15": (FIX_IN, FIX_OUT, 1.5, 16, 12), "pad": (FIX_IN, FIX_WIDE, 1, 16, 12), "pad2": (FIX_IN, FIX_WIDE, 2, 16, 12),
}


@pytest.fixture(autouse=True)
def _no_tf32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def torch_lines(x, input_scope, output_scope, p):
    """The reference's BEVGridTransform.forward, on x's device."""
    if p != 1:
        x = F.interpolate(x, scale_factor=p, mode="bilinear", align_corners=False)
    coords = []
    for (imin, imax, _), (omin, omax, ostep) in zip(input_scope, output_scope):
        v = torch.arange(omin + ostep / 2, omax, ostep)
        v = (v - imin) / (imax - imin) * 2 - 1
        coords.append(v.to(x.device))
    u, v = torch.meshgrid(coords, indexing="ij")
    grid = torch.stack([torch.stack([v, u], dim=-1)] * x.shape[0], dim=0)
    return F.grid_sample(x, grid, mode="bilinear", align_corners=False)


def mats(name, dev):
    isc, osc, p, H, W = GEOMS[name]
    Ay, Ax = O.transform_matrices(isc, osc, H, W, p)
    return torch.from_numpy(Ay).to(dev), torch.from_numpy(Ax).to(dev)


def fwd64(x, Ay, Ax):
    return Ay @ x.double() @ Ax.T, Ay.abs() @ x.double().abs() @ Ax.abs().T


def bwd64(g, Ay, Ax):
    return Ay.T @ g.double() @ Ax, Ay.abs().T @ g.double().abs() @ Ax.abs()


def inputs(name, B, C, dtype, dev, seed=0):
    _, _, _, H, W = GEOMS[name]
    gen = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn((B, C, H, W), generator=gen).to(dev, dtype)


# ---- grid transform --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("B,C", [(1, 512), (4, 512), (1, 80), (4, 80), (1, 7), (4, 7)])
@pytest.mark.parametrize("name", list(GEOMS))
def test_grid_forward(cuda, name, B, C, dtype):
    if name != "default" and C == 512 and B == 4:
        pytest.skip("the tiny geometries run at C 512 with B 1")
    isc, osc, p, H, W = GEOMS[name]
    x = inputs(name, B, C, dtype, cuda)
    t = MS.BEVGridTransform(input_scope=isc, output_scope=osc, prescale_factor=p)
    y = t(x)
    assert y.dtype == dtype and y.shape == (B, C, len(MS.axis_coords(isc[0], osc[0])),
                                             len(MS.axis_coords(isc[1], osc[1])))
    want, scale = fwd64(x, *mats(name, cuda))
    err = (y.double() - want).abs()
    bound = 8 * EPS32 * scale + (EPS16 * want.abs() + 2.0 ** -24 if dtype == torch.float16 else 0)
    assert bool((err <= bound).all()), float((err - bound).max())
    if dtype == torch.float32:
        ref = torch_lines(x, isc, osc, p)
        assert float((y - ref).abs().max()) <= 1e-5 * float(ref.abs().max())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("B,C", [(1, 512), (4, 80), (1, 7)])
@pytest.mark.parametrize("name", list(GEOMS))
def test_grid_backward(cuda, name, B, C, dtype):
    isc, osc, p, H, W = GEOMS[name]
    x = inputs(name, B, C, dtype, cuda).requires_grad_(True)
    t = MS.BEVGridTransform(input_scope=isc, output_scope=osc, prescale_factor=p)
    y = t(x)
    g = torch.randn(y.shape, generator=torch.Generator(device="cpu").manual_seed(2)).to(cuda, dtype)
    (gi,) = torch.autograd.grad(y, x, g)
    assert gi.dtype == dtype
    Ay, Ax = mats(name, cuda)
    want, scale = bwd64(g, Ay, Ax)
    err = (gi.double() - want).abs()
    bound = 8 * EPS32 * scale + (EPS16 * want.abs() + 2.0 ** -24 if dtype == torch.float16 else 0)
    assert bool((err <= bound).all()), float((err - bound).max())
    # rows and columns no tap reaches are exactly zero
    dead_r, dead_c = (Ay != 0).sum(0) == 0, (Ax != 0).sum(0) == 0
    assert bool((gi[:, :, dead_r, :] == 0).all()) and bool((gi[:, :, :, dead_c] == 0).all())
    if name == "default":                             # input rows / columns 0 and 127 feed no output
        assert bool(dead_r[[0, 127]].all() and dead_c[[0, 127]].all())
    # repeated calls are bit-identical
    for _ in range(2):
        (again,) = torch.autograd.grad(t(x), x, g)
        assert torch.equal(again, gi)
    if dtype == torch.float32:
        xr = x.detach().clone().requires_grad_(True)
        (ref,) = torch.autograd.grad(torch_lines(xr, isc, osc, p), xr, g)
        assert float((gi - ref).abs().max()) <= 1e-5 * float(ref.abs().max())


def test_grid_transform_follows_channels_last_and_views(cuda):
    isc, osc, p, H, W = GEOMS["p2"]
    x = inputs("p2", 2, 6, torch.float32, cuda)
    t = MS.BEVGridTransform(input_scope=isc, output_scope=osc, prescale_factor=p)
    want = t(x)
    assert torch.equal(t(x.to(memory_format=torch.channels_last)), want)
    assert torch.equal(t(torch.cat([x, x], 1)[:, 6:]), want)


# ---- losses ------------------------------------------------------------------------------------------------------
def _loss_case(kind, dev, seed=0):
    gen = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn((2, 4, 33, 31), generator=gen) * 4
    t = (torch.rand((2, 4, 33, 31), generator=gen) < 0.35).long()
    flat = x.view(-1)
    flat[:16] = torch.tensor([30.0, -30, 100, -100] * 4)
    t.view(-1)[:16] = torch.tensor([0, 1] * 8)
    if kind == "zeros":
        t[:, 1] = 0
    elif kind == "ones":
        t[:, 2] = 1
    elif kind == "soft":
        t = torch.rand((2, 4, 33, 31), generator=gen)
    return x.to(dev), t.to(dev)


@pytest.mark.parametrize("ttype", [torch.int64, torch.uint8, torch.bool, torch.float32])
@pytest.mark.parametrize("xtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("loss", ["focal", "xent"])
@pytest.mark.parametrize("kind", ["random", "zeros", "ones"])
def test_losses_against_oracle(cuda, kind, loss, xtype, ttype):
    x, t = _loss_case(kind, cuda)
    x = x.to(xtype).requires_grad_(True)
    tt = t.to(ttype)
    classes = ["c%d" % k for k in range(4)]
    out = MS.map_seg_loss(x, tt, loss, classes)
    assert list(out) == ["c%d/%s" % (k, loss) for k in range(4)]
    got = torch.stack(list(out.values()))
    assert got.dtype == torch.float32 and all(v.dim() == 0 for v in out.values())
    xn, tn = x.detach().double().cpu().numpy(), tt.double().cpu().numpy()
    np.testing.assert_allclose(got.detach().cpu().numpy(), O.losses(xn, tn, loss), rtol=2e-6, atol=0)
    w = torch.tensor([1.0, 0.5, 2.0, -1.0], device=cuda)
    (gx,) = torch.autograd.grad((got * w).sum(), x)
    assert gx.dtype == xtype
    want = O.loss_grad(xn, tn, loss, w.cpu().numpy())
    # fp16: one fp16 rounding, subnormals included (the gradients are O(1 / (B H W)))
    tol = 1e-5 * np.abs(want).max() + (EPS16 * np.abs(want) + 2.0 ** -25 if xtype == torch.float16 else 0)
    assert np.all(np.abs(gx.double().cpu().numpy() - want) <= tol)


@pytest.mark.parametrize("loss", ["focal", "xent"])
def test_soft_targets(cuda, loss):
    x, t = _loss_case("soft", cuda)
    x.requires_grad_(True)
    got = torch.stack(list(MS.map_seg_loss(x, t, loss, list("abcd")).values()))
    xn, tn = x.detach().double().cpu().numpy(), t.double().cpu().numpy()
    np.testing.assert_allclose(got.detach().cpu().numpy(), O.losses(xn, tn, loss), rtol=2e-6, atol=0)
    (gx,) = torch.autograd.grad(got.sum(), x)
    want = O.loss_grad(xn, tn, loss)
    assert np.abs(gx.double().cpu().numpy() - want).max() <= 1e-5 * np.abs(want).max()


@pytest.mark.parametrize("loss", ["focal", "xent"])
def test_losses_against_fixture(cuda, loss):
    g = np.load(GOLDEN)
    x = torch.tensor(g["loss_logits"], dtype=torch.float32, device=cuda, requires_grad=True)
    t = torch.tensor(g["loss_target"], device=cuda)
    got = torch.stack(list(MS.map_seg_loss(x, t, loss, list(g["classes"])).values()))
    np.testing.assert_allclose(got.detach().cpu().numpy(), g["loss_%s_values" % loss], rtol=2e-6, atol=0)
    (gx,) = torch.autograd.grad((got * torch.tensor(g["loss_w"], device=cuda, dtype=torch.float32)).sum(), x)
    want = g["loss_%s_grad" % loss]
    assert np.abs(gx.double().cpu().numpy() - want).max() <= 1e-5 * np.abs(want).max()


def test_loss_is_repeatable(cuda):
    x, t = _loss_case("random", cuda)
    x.requires_grad_(True)
    a = torch.stack(list(MS.map_seg_loss(x, t, "focal", list("abcd")).values()))
    (ga,) = torch.autograd.grad(a.sum(), x)
    for _ in range(2):
        b = torch.stack(list(MS.map_seg_loss(x, t, "focal", list("abcd")).values()))
        (gb,) = torch.autograd.grad(b.sum(), x)
        assert torch.equal(a, b) and torch.equal(ga, gb)


# ---- counts ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gtype", [torch.int64, torch.uint8, torch.bool, torch.float32])
@pytest.mark.parametrize("ptype", [torch.float32, torch.float16])
@pytest.mark.parametrize("ties", [False, True])
def test_counts_exact(cuda, ties, ptype, gtype):
    rng = np.random.default_rng(5)
    pred = rng.random((3, 5, 97, 61)).astype(np.float32)
    if ties:
        pred = rng.choice(np.float32([0.3, 0.35, 0.4, 0.45, 0.5, 0.55, 0.6, 0.65, 0.7]), pred.shape)
        pred[0, 0, 0, :4] = np.nan
    pred = pred.astype(np.float16 if ptype == torch.float16 else np.float32)
    gt = (rng.random((3, 5, 97, 61)) < 0.4)
    gtt = torch.from_numpy(gt).to(cuda, gtype)
    if gtype == torch.float32:
        gtt[0, 0, 0, 0] = float("nan")
        gt[0, 0, 0, 0] = True
    out = MS.map_seg_counts(torch.from_numpy(pred).to(cuda), gtt)
    assert out.dtype == torch.int64 and out.shape == (3, 5, 7)
    np.testing.assert_array_equal(out.cpu().numpy(), O.counts(pred.astype(np.float32), gt, MS.THRESHOLDS))
    # per-sample calls add into the same counters
    acc = torch.zeros_like(out)
    for b in range(3):
        MS.map_seg_counts(torch.from_numpy(pred[b]).to(cuda), gtt[b], out=acc)
    assert torch.equal(acc, out)


def test_counts_match_reference_evaluate_map(cuda):
    g = np.load(GOLDEN)
    out = None
    for b in range(g["eval_pred"].shape[0]):
        out = MS.map_seg_counts(torch.from_numpy(g["eval_pred"][b]).to(cuda), torch.from_numpy(g["eval_gt"][b])
                                .to(cuda), out=out)
    np.testing.assert_array_equal(out.cpu().numpy(), g["eval_counts"])
    m = MS.map_seg_metrics(out, list(g["classes"]))
    assert list(m) == list(g["eval_keys"])
    np.testing.assert_allclose(list(m.values()), g["eval_values"], rtol=1e-6, atol=1e-7)


def test_counts_exact_past_2_pow_24(cuda):
    pred = torch.zeros((8, 2, 200, 200), device=cuda)
    pred[:, :, :, :150] = 0.9
    gt = torch.zeros((8, 2, 200, 200), dtype=torch.uint8, device=cuda)
    gt[:, :, :, 50:] = 1
    out = torch.zeros((3, 2, 7), dtype=torch.int64, device=cuda)
    calls = 120
    for _ in range(calls):
        MS.map_seg_counts(pred, gt, out=out)
    per = 8 * 200
    tp, fp, fn = calls * per * 100, calls * per * 50, calls * per * 50
    assert tp > 2 ** 24
    want = torch.tensor([tp, fp, fn], dtype=torch.int64)[:, None, None].expand(3, 2, 7)
    assert torch.equal(out.cpu(), want)


# ---- head --------------------------------------------------------------------------------------------------------
def _fixture_head(g, dev):
    head = MS.BEVSegmentationHead(4, dict(input_scope=g["in_scope"].tolist(), output_scope=g["out_scope"].tolist(),
                                          prescale_factor=2), list(g["classes"]), "focal")
    keys = [k[len("head_state/"):] for k in g.files if k.startswith("head_state/")]
    head.load_state_dict({k: torch.from_numpy(g["head_state/" + k]).float() for k in keys})
    return head.to(dev)


def test_head_matches_reference_fixture(cuda):
    g = np.load(GOLDEN)
    head = _fixture_head(g, cuda).train()
    x = torch.tensor(g["head_feats"], dtype=torch.float32, device=cuda, requires_grad=True)
    losses = head([x], torch.tensor(g["head_masks"], device=cuda))
    assert list(losses) == list(g["head_keys"])
    got = torch.stack(list(losses.values()))
    # the classifier runs in fp32 (cuDNN, no TF32) against the fixture's float64
    np.testing.assert_allclose(got.detach().cpu().numpy(), g["head_losses"], rtol=1e-5, atol=0)
    (gx,) = torch.autograd.grad(got.sum(), x)
    want = g["head_grad"]
    assert np.abs(gx.double().cpu().numpy() - want).max() <= 1e-4 * np.abs(want).max()
    head = _fixture_head(g, cuda).eval()
    with torch.no_grad():
        y = head(torch.tensor(g["head_feats"], dtype=torch.float32, device=cuda))
    assert np.abs(y.double().cpu().numpy() - g["head_eval"]).max() <= 1e-5


def test_launch_counts(cuda):
    isc, osc, p, H, W = GEOMS["default"]
    t = MS.BEVGridTransform(input_scope=isc, output_scope=osc, prescale_factor=p)
    x = inputs("default", 1, 8, torch.float32, cuda).requires_grad_(True)
    t(x)                                                    # tables built and uploaded once
    _C.reset_launch_count()
    y = t(x)
    assert _C.launch_count() == 1
    with torch.autograd.set_multithreading_enabled(False):   # the launch counter is per host thread
        y.backward(torch.ones_like(y))
    assert _C.launch_count() == 2
    logits = torch.randn((1, 6, 200, 200), device=cuda, requires_grad=True)
    target = S.map_seg_masks(0, 1).to(cuda)
    _C.reset_launch_count()
    tot = sum(MS.map_seg_loss(logits, target, "focal", S.MAP_CLASSES).values())
    assert _C.launch_count() == 2
    with torch.autograd.set_multithreading_enabled(False):
        tot.backward()
    assert _C.launch_count() == 3
    _C.reset_launch_count()
    MS.map_seg_counts(torch.sigmoid(logits.detach()), target)
    assert _C.launch_count() == 1


def test_training_step_is_sync_free_and_deterministic(cuda):
    script = textwrap.dedent("""
        import sys, torch
        sys.path.insert(0, %r)
        from bevfusion_b200 import map_seg as MS, synthetic as S
        torch.use_deterministic_algorithms(True)
        torch.backends.cudnn.benchmark = False
        dev = torch.device("cuda:0")
        torch.manual_seed(0)
        head = MS.BEVSegmentationHead(64, dict(S.MAP_SEG_CFG, prescale_factor=2), list(S.MAP_CLASSES), "focal")
        head = head.to(dev).train()
        x = S.map_seg_features(0, 2, 64).to(dev).requires_grad_(True)
        t = S.map_seg_masks(0, 2).to(dev)
        def step():
            x.grad = None
            head.zero_grad(set_to_none=True)
            sum(head([x], t).values()).backward()
            c = MS.map_seg_counts(torch.sigmoid(x.grad[:, :6, :100, :100].repeat(1, 1, 2, 2)), t)
            return [x.grad.clone()] + [p.grad.clone() for p in head.parameters()] + [c]
        step()
        torch.cuda.set_sync_debug_mode("error")
        a = step()
        b = step()
        torch.cuda.set_sync_debug_mode(0)
        assert all(torch.equal(u, v) for u, v in zip(a, b))
        print("ok")
    """ % os.path.abspath(ROOT))
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


def test_training_step_graph_replay(cuda):
    torch.manual_seed(0)
    torch.backends.cudnn.deterministic = True
    head = MS.BEVSegmentationHead(32, dict(S.MAP_SEG_CFG), list(S.MAP_CLASSES), "focal").to(cuda).train()
    x = S.map_seg_features(0, 2, 32).to(cuda).requires_grad_(True)
    targets = [S.map_seg_masks(s, 2).to(cuda) for s in range(3)]
    t = targets[0].clone()
    params = list(head.parameters())

    def step():
        x.grad = None
        for p in params:
            p.grad = None
        losses = head([x], t)
        torch.stack(list(losses.values())).sum().backward()
        return torch.stack(list(losses.values())).detach()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(s)
    eager = []
    for tg in targets:
        t.copy_(tg)
        lv = step()
        eager.append([lv, x.grad.clone()] + [p.grad.clone() for p in params])
    x.grad = None
    for p in params:
        p.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        losses = head([x], t)
        static_loss = torch.stack(list(losses.values()))
        static_loss.sum().backward()
    for tg, want in zip(targets, eager):
        t.copy_(tg)
        graph.replay()
        torch.cuda.synchronize()
        got = [static_loss, x.grad] + [p.grad for p in params]
        assert all(torch.equal(u, v) for u, v in zip(got, want))
    torch.backends.cudnn.deterministic = False
