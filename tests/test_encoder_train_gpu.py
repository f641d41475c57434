"""GPU tests of the native SparseEncoder training path (bevb200_encoder_forward_train / _backward through
EncoderPlan.forward_train and SparseEncoder.forward(..., num_voxels=) in training mode): against a float64 twin,
against the modular training path, with a device count below the row count, sync-free and deterministic, as one
CUDA graph with voxelization and an optimizer step, and on its edge cases."""
import copy

import pytest
import torch

from bevfusion_b200 import _C
from bevfusion_b200 import encoder_plan
from bevfusion_b200 import synthetic as S
from bevfusion_b200.sparse_encoder import SparseEncoder
from bevfusion_b200.spconv import ops as sp_ops
from bevfusion_b200.voxelize import Voxelization, voxelize_mean, voxelize_mean_fused
from encoder_train_oracle import rel, twin_forward

pytestmark = pytest.mark.gpu

# the bf16x3 bounds of the modular training step against float64 (test_spconv_backward_gpu.TRAIN_BOUNDS)
BOUNDS = {"input": 1e-4, "conv": 1e-4, "bn": 1e-4, "stats": 6e-5}
SHAPE = [320, 320, 41]
RANGE = [-12.0, -12.0, -5.0, 12.0, 12.0, 3.0]


def _c3_voxels(dev, seed=0):
    L = S.LIDAR_C3
    pts = torch.from_numpy(S.lidar_cloud(seed=seed)).to(dev)
    vox = Voxelization(L["voxel_size"], RANGE, L["max_num_points"], L["max_voxels"])
    return voxelize_mean(*vox.eval()(pts), 0)


def _randomise_bn(m):
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm1d):
            mod.running_mean.normal_(0, 0.1); mod.running_var.uniform_(0.5, 1.5)
            mod.weight.data.uniform_(0.8, 1.2); mod.bias.data.normal_(0, 0.1)
    return m


def _basicblock(dev):
    torch.manual_seed(0)
    return _randomise_bn(SparseEncoder(in_channels=5, sparse_shape=SHAPE, output_channels=128,
                                       encoder_channels=((16, 16, 32), (32, 32, 64), (64, 64, 128), (128, 128)),
                                       encoder_paddings=((0, 0, 1), (0, 0, 1), (0, 0, (1, 1, 0)), (0, 0)),
                                       block_type="basicblock").to(dev)).train()


def _conv_module(dev):
    torch.manual_seed(1)
    return _randomise_bn(SparseEncoder(in_channels=5, sparse_shape=SHAPE).to(dev)).train()


def _two_samples(dev):
    """B = 2: the C3 cloud, and a near-empty second sample (3 voxels)."""
    f0, c0 = _c3_voxels(dev)
    f1, c1 = f0[:3].clone(), c0[:3].clone()
    c1[:, 0] = 1
    return torch.cat([f0, f1]), torch.cat([c0, c1])


def _out_shape(m, B):
    X, Y, Z = m.plan().out_shape
    return (B, m.plan().out_channels * Z, X, Y)


def _count(n, dev):
    return torch.tensor([n], dtype=torch.int32, device=dev)


def _params(plan):
    return ([cv.weight for cv, _, _, _ in plan.chain], [bn.weight for _, bn, _, _ in plan.chain],
            [bn.bias for _, bn, _, _ in plan.chain])


def _native_masks(m, feats, coors, B, n_dev):
    """The ReLU masks of a training forward of `m` on these inputs, read from its saved state (on a copy: the
    forward is deterministic, so the masks are those of the run under test)."""
    probe = copy.deepcopy(m)
    plan = probe.plan()
    with torch.no_grad():
        _, state = plan._forward_train_native(feats, coors, B, n_dev, None, True, *_params(plan))
    counts = [int(v) for v in plan.status[1:].tolist()]
    return [plan.saved_rows(state, feats.shape[0], B, i)[1][:counts[plan.level_of(i)]] > 0
            for i in range(len(plan.chain))]


def _step(m, feats, coors, B, n_dev, R, grad_input=True):
    x = feats.detach().clone().requires_grad_(grad_input)
    out = m(x, coors, B, num_voxels=n_dev)
    (out * R).sum().backward()
    return out.detach(), x.grad


def _grads(m):
    return {k: p.grad.clone() for k, p in m.named_parameters()}


def _stats(m):
    return {k: b.clone() for k, b in m.named_buffers()}


def _compare(rows_fn, bounds):
    bad = [(kind, name, l2) for kind, name, l2 in rows_fn if not l2 <= bounds[kind]]
    assert not bad, bad


@pytest.mark.parametrize("case", ["basicblock_b1", "conv_module_b2"])
def test_native_train_vs_float64(cuda, case):
    if case == "basicblock_b1":
        m, B = _basicblock(cuda), 1
        feats, coors = _c3_voxels(cuda)
    else:
        m, B = _conv_module(cuda), 2
        feats, coors = _two_samples(cuda)
    n_dev = _count(feats.shape[0], cuda)
    masks = _native_masks(m, feats, coors, B, n_dev)
    twin = copy.deepcopy(m).double()
    before = _stats(m)
    R = torch.randn(_out_shape(m, B), device=cuda, generator=torch.Generator(device=cuda).manual_seed(1))
    out, gx = _step(m, feats, coors, B, n_dev, R)

    chain64 = encoder_plan._chain_of(twin)
    x64 = feats.detach().double().requires_grad_(True)
    out64 = twin_forward(chain64, x64, coors, B, SHAPE, masks, [(bn.weight, bn.bias) for _, bn, _, _ in chain64],
                         [(bn.running_mean, bn.running_var, bn.num_batches_tracked) for _, bn, _, _ in chain64])
    (out64 * R.double()).sum().backward()
    assert rel(out, out64.detach())[1] <= 1e-4
    rows = [("input", "features", rel(gx, x64.grad)[0])]
    p64 = dict(twin.named_parameters())
    for name, p in m.named_parameters():
        rows.append(("bn" if p.dim() == 1 else "conv", name, rel(p.grad, p64[name].grad)[0]))
    b64 = dict(twin.named_buffers())
    for name, b in m.named_buffers():
        if name.endswith(("running_mean", "running_var")):
            rows.append(("stats", name, rel(b - before[name], b64[name].detach() - before[name].double())[0]))
        elif name.endswith("num_batches_tracked"):
            assert int(b) == int(b64[name]) == int(before[name]) + 1, name
    for kind in BOUNDS:
        print("%s: worst %-5s rel L2 %.2e" % (case, kind, max(l2 for k, _, l2 in rows if k == kind)))
    _compare(rows, BOUNDS)


def test_native_train_vs_modular(cuda):
    m = _basicblock(cuda)
    feats, coors = _c3_voxels(cuda)
    mod = copy.deepcopy(m)
    before = _stats(m)
    # the modular ReLUs apply the native run's masks: an element within rounding of 0 may fall on the other side of
    # the kink in either run, and one flip moves the gradients below it by far more than any kernel error
    masks = iter(_native_masks(m, feats, coors, 1, _count(feats.shape[0], cuda)))
    hooks = []
    for relu in (r for r in mod.modules() if isinstance(r, torch.nn.ReLU)):
        relu.inplace = False
        hooks.append(relu.register_forward_hook(lambda _, inp, out: inp[0] * next(masks)))
    x = feats.clone().requires_grad_(True)
    try:
        out_mod = mod(x, coors, 1)                               # no num_voxels: the modular path
    finally:
        for h in hooks:
            h.remove()
    assert next(masks, None) is None
    R = torch.randn(out_mod.shape, device=cuda, generator=torch.Generator(device=cuda).manual_seed(2))
    (out_mod * R).sum().backward()
    out, gx = _step(m, feats, coors, 1, _count(feats.shape[0], cuda), R)
    assert rel(out, out_mod.detach())[1] <= 1e-4
    rows = [("input", "features", rel(gx, x.grad)[0])]
    pm = dict(mod.named_parameters())
    for name, p in m.named_parameters():
        rows.append(("bn" if p.dim() == 1 else "conv", name, rel(p.grad, pm[name].grad)[0]))
    bm = dict(mod.named_buffers())
    for name, b in m.named_buffers():
        if name.endswith(("running_mean", "running_var")):
            rows.append(("stats", name, rel(b - before[name], bm[name] - before[name])[0]))
        else:
            assert torch.equal(b, bm[name]), name
    _compare(rows, BOUNDS)


def test_device_count_below_rows(cuda):
    m = _basicblock(cuda)
    feats, coors = _c3_voxels(cuda)
    n = feats.shape[0]
    pad = 1000
    fp = torch.cat([feats, torch.full((pad, feats.shape[1]), float("nan"), device=cuda)])
    cp = torch.cat([coors, torch.full((pad, 4), 100000, dtype=torch.int32, device=cuda)])
    ref = copy.deepcopy(m)
    before = _stats(m)
    R = torch.randn(_out_shape(m, 1), device=cuda, generator=torch.Generator(device=cuda).manual_seed(3))
    out_ref, g_ref = _step(ref, feats, coors, 1, _count(n, cuda), R)
    out, g = _step(m, fp, cp, 1, _count(n, cuda), R)
    assert out.shape == out_ref.shape
    assert rel(out, out_ref)[1] <= 1e-4
    assert bool(torch.isfinite(g).all()) and bool((g[n:] == 0).all())
    rows = [("input", "features", rel(g[:n], g_ref)[0])]
    pr = dict(ref.named_parameters())
    rows += [("bn" if p.dim() == 1 else "conv", k, rel(p.grad, pr[k].grad)[0]) for k, p in m.named_parameters()]
    br = dict(ref.named_buffers())
    for k, b in m.named_buffers():
        if k.endswith(("running_mean", "running_var")):
            rows.append(("stats", k, rel(b - before[k], br[k] - before[k])[0]))
    _compare(rows, BOUNDS)


def test_sync_free_and_deterministic(cuda):
    m = _basicblock(cuda)
    feats, coors = _c3_voxels(cuda)
    n_dev = _count(feats.shape[0], cuda)
    m2 = copy.deepcopy(m)
    R = torch.randn(_out_shape(m, 1), device=cuda, generator=torch.Generator(device=cuda).manual_seed(4))
    _step(m, feats, coors, 1, n_dev, R)                          # warm: plan, streams, allocator
    m.zero_grad(set_to_none=True)
    m.load_state_dict(m2.state_dict())
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out1, g1 = _step(m, feats, coors, 1, n_dev, R)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    out2, g2 = _step(m2, feats, coors, 1, n_dev, R)
    assert torch.equal(out1, out2) and torch.equal(g1, g2)
    p2, b2 = dict(m2.named_parameters()), dict(m2.named_buffers())
    for k, p in m.named_parameters():
        assert torch.equal(p.grad, p2[k].grad), k
    for k, b in m.named_buffers():
        assert torch.equal(b, b2[k]), k


def test_graph_replay_matches_eager(cuda):
    L = S.LIDAR_C3
    clouds = [torch.from_numpy(S.lidar_cloud(seed=s)[:150000]).to(cuda) for s in (5, 6, 7)]
    m = _basicblock(cuda)
    eager = copy.deepcopy(m)
    R = torch.randn(_out_shape(m, 1), device=cuda, generator=torch.Generator(device=cuda).manual_seed(5))

    def step(model, opt, pts):
        f, c, _, n_dev = voxelize_mean_fused(pts, L["voxel_size"], RANGE, L["max_num_points"], 60000, sync=False)
        out = model(f, c, 1, num_voxels=n_dev)
        (out * R).sum().backward()
        opt.step()
        return out

    opt = torch.optim.SGD(m.parameters(), lr=1e-3, momentum=0.9)
    opt_e = torch.optim.SGD(eager.parameters(), lr=1e-3, momentum=0.9)
    static = clouds[0].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                                # warm-up step, on both copies
        step(m, opt, static)
    torch.cuda.current_stream().wait_stream(side)
    step(eager, opt_e, static)
    m.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_g = step(m, opt, static)
    outs = []
    for pts in clouds:
        static.copy_(pts)
        graph.replay()
        outs.append(out_g.clone())
    for pts, og in zip(clouds, outs):
        eager.zero_grad(set_to_none=True)
        oe = step(eager, opt_e, pts)
        assert torch.equal(og, oe.detach())
    pe, be = dict(eager.named_parameters()), dict(eager.named_buffers())
    for k, p in m.named_parameters():
        assert torch.equal(p.detach(), pe[k].detach()), k
    for k, b in m.named_buffers():
        assert torch.equal(b, be[k]), k


def test_gradient_accumulation(cuda):
    m = _basicblock(cuda)
    fa, ca = _c3_voxels(cuda, seed=0)
    fb, cb = _c3_voxels(cuda, seed=1)
    single = copy.deepcopy(m)
    R = torch.randn(_out_shape(m, 1), device=cuda, generator=torch.Generator(device=cuda).manual_seed(6))
    xa, xb = fa.clone().requires_grad_(True), fb.clone().requires_grad_(True)
    oa = m(xa, ca, 1, num_voxels=_count(fa.shape[0], cuda))
    ob = m(xb, cb, 1, num_voxels=_count(fb.shape[0], cuda))
    ((oa * R).sum() + (ob * R).sum()).backward()
    _, ga = _step(single, fa, ca, 1, _count(fa.shape[0], cuda), R)
    g1 = _grads(single)
    single.zero_grad(set_to_none=True)
    _, gb = _step(single, fb, cb, 1, _count(fb.shape[0], cuda), R)
    g2 = _grads(single)
    assert torch.equal(xa.grad, ga) and torch.equal(xb.grad, gb)
    for k, p in m.named_parameters():
        assert torch.allclose(p.grad, g1[k] + g2[k], rtol=1e-6, atol=0), k


def test_no_input_gradient_skips_work(cuda):
    m = _basicblock(cuda)
    feats, coors = _c3_voxels(cuda)
    n_dev = _count(feats.shape[0], cuda)
    R = torch.randn(_out_shape(m, 1), device=cuda)
    x = feats.clone()                                            # no requires_grad: no input gradient
    (m(x, coors, 1, num_voxels=n_dev) * R).sum().backward()
    assert x.grad is None and m.conv_input[0].weight.grad is not None
    # the launch counter is per host thread and autograd runs backwards on its own: count the native call here
    plan = m.plan()
    weights, bn_w, bn_b = _params(plan)
    with torch.no_grad():
        _, state = plan._forward_train_native(feats, coors, 1, n_dev, None, True, weights, bn_w, bn_b)
    launches = []
    for need_input in (True, False):
        _C.reset_launch_count()
        gfeat, _, _, _ = plan._backward_native(state, feats.shape[0], 1, None, R, weights, need_input)
        launches.append(_C.launch_count())
        assert (gfeat is not None) == need_input
    print("backward launches with / without the input gradient: %d / %d" % tuple(launches))
    assert launches[1] < launches[0]


def test_weight_updated_in_place_raises(cuda):
    m = _basicblock(cuda)
    feats, coors = _c3_voxels(cuda)
    out = m(feats.clone().requires_grad_(True), coors, 1, num_voxels=_count(feats.shape[0], cuda))
    with torch.no_grad():
        m.conv_input[0].weight.mul_(1.01)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        out.sum().backward()


def test_cap_truncation_sets_status(cuda):
    m = _basicblock(cuda)
    feats, coors = _c3_voxels(cuda)
    plan = m.plan()
    caps = [0] * plan.n_levels
    caps[1] = 64
    x = feats.clone().requires_grad_(True)
    out = plan.forward_train(x, coors, 1, n_voxels_dev=_count(feats.shape[0], cuda), level_caps=caps)
    out.sum().backward()
    st = plan.status.tolist()
    assert st[0] & 1 and st[2] == 64
    assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(x.grad).all())


@pytest.mark.parametrize("n", [1, 0])
def test_fewer_than_two_rows(cuda, n):
    m = _basicblock(cuda)
    feats, coors = _c3_voxels(cuda)
    before_bn = [(bn.running_mean.clone(), bn.running_var.clone()) for _, bn, _, _ in m.plan().chain]
    x = feats.clone().requires_grad_(True)
    out = m(x, coors, 1, num_voxels=_count(n, cuda))
    (out * torch.randn_like(out)).sum().backward()
    plan = m.plan()
    st = plan.status.tolist()
    assert st[0] & 2 and st[1] == n
    assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(x.grad).all())
    assert all(bool(torch.isfinite(p.grad).all()) for p in m.parameters())
    for i, (_, bn, _, _) in enumerate(plan.chain):
        if st[1 + plan.level_of(i)] < 2:                         # levels with < 2 rows leave their BN alone
            assert torch.equal(bn.running_mean, before_bn[i][0]) and torch.equal(bn.running_var, before_bn[i][1])
            assert int(bn.num_batches_tracked) == 0


def test_refusals(cuda):
    feats, coors = _c3_voxels(cuda)
    n_dev = _count(feats.shape[0], cuda)

    def raises(m, **kw):
        f = kw.pop("feats", feats)
        with pytest.raises(ValueError):
            m(f, coors, 1, num_voxels=n_dev, **kw)

    raises(_basicblock(cuda), precision=sp_ops.PREC_FP32)
    raises(_basicblock(cuda), feats=feats.half())
    raises(_basicblock(cuda).half())
    m = _basicblock(cuda)
    m.conv_input[0].bias = torch.nn.Parameter(torch.zeros(16, device=cuda))
    raises(m)
    raises(_basicblock(cuda), out=torch.empty((1, 256, 40, 40), device=cuda))
    m = _basicblock(cuda)
    m.conv_input[1].momentum = None
    raises(m)
    torch.manual_seed(0)
    raises(SparseEncoder(5, SHAPE, order=("conv", "act", "norm")).to(cuda).train())


def test_eval_after_training_refolds(cuda):
    m = _basicblock(cuda)
    feats, coors = _c3_voxels(cuda)
    m.eval()
    with torch.no_grad():
        m(feats, coors, 1)                                       # the eval plan folds the initial statistics
    m.train()
    opt = torch.optim.SGD(m.parameters(), lr=1e-3)
    for s in (1, 2):
        f, c = _c3_voxels(cuda, seed=s)
        out = m(f, c, 1, num_voxels=_count(f.shape[0], cuda))
        out.square().mean().backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
    m.eval()
    with torch.no_grad():
        y = m(feats, coors, 1)
    twin = _basicblock(cuda).double()                           # (the plan's native handle does not deep-copy)
    twin.load_state_dict(m.state_dict())
    chain64 = encoder_plan._chain_of(twin)
    y64 = twin_forward(chain64, feats.double(), coors, 1, SHAPE, None,
                       [(bn.weight, bn.bias) for _, bn, _, _ in chain64],
                       [(bn.running_mean, bn.running_var, bn.num_batches_tracked) for _, bn, _, _ in chain64],
                       train=False)
    assert rel(y, y64.detach())[1] <= 1e-4
    assert all(int(bn.num_batches_tracked) == 2 for _, bn, _, _ in m.plan().chain)
