"""GPU tests of the SparseEncoder's fp16 precision (SparseEncoder.forward(..., precision=PREC_FP16)): the native plan's
eval forward, training forward and whole-encoder backward on fp16 operands, against the float64 oracle of
encoder_fp16_oracle (bounds and their constants derived there; every case prints its worst ratio).

  * Training forward, conv by conv from the saved state: z16 against the float64 conv of the conv's saved fp16 input
    and fp16(W); the running statistics against float64 of the saved z16; y16 against float64 BN, residual and ReLU
    of the saved z16; dense() equal to the last y16 bit for bit.
  * Backward against a float64 twin that runs through exactly the saved z16 / y16 values and the run's ReLU masks.
  * Eval forward against a float64 twin that rounds to fp16 where the plan rounds, on chains of 1 to 3 stages and
    the voxelnet chain.
  * These module chains cover Cout 16 / 32 (mma.sync), Cout 64 / 128 on both sides of the wgmma K-block threshold,
    first convs with c_in 5, 16 and 128, SubM and strided convs and residuals from two convs back (SparseBasicBlock).
    The raw chains of encoder_train_cases (residuals from one conv back and on the last conv, a strided first conv,
    k2 s2 convs) and the row-count boundaries run in test_encoder_fp16_edges_gpu.py.
  * Half weights against fp32 master weights, GradScaler overflow, precision isolation, sync-free capture in a CUDA
    graph, bit reproducibility and the refusals."""
import copy
import ctypes

import numpy as np
import pytest
import torch

from bevfusion_b200 import _C
from bevfusion_b200.sparse_encoder import SparseEncoder
from bevfusion_b200.spconv.ops import PREC_BF16X3, PREC_FP16
from encoder_fp16_oracle import (bwd_bounds, c_eval, check_train_forward, dense64, eval_twin, fp16_round,
                                 module_convs, rulebooks, twin_backward)
from encoder_train_oracle import rel
from half_oracle import check

pytestmark = pytest.mark.gpu


def _randomise_bn(m, seed):
    g = torch.Generator().manual_seed(seed)
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm1d):
            n = mod.num_features
            mod.running_mean.copy_(torch.randn(n, generator=g) * 0.1)
            mod.running_var.copy_(torch.rand(n, generator=g) + 0.5)
            mod.weight.data.copy_(torch.rand(n, generator=g) * 0.4 + 0.8)
            mod.bias.data.copy_(torch.randn(n, generator=g) * 0.1)
    return m


def voxelnet(shape):
    return SparseEncoder(in_channels=5, sparse_shape=shape, output_channels=128,
                         encoder_channels=((16, 16, 32), (32, 32, 64), (64, 64, 128), (128, 128)),
                         encoder_paddings=((0, 0, 1), (0, 0, 1), (0, 0, (1, 1, 0)), (0, 0)), block_type="basicblock")


def stages(shape, depth, in_channels=5, base=16):
    """conv_module chains of `depth` stages: SubM and strided convs, Cout 16 / 32 / 64"""
    ch = ((base,), (32, 32, 32), (64, 64, 64))[:depth]
    return SparseEncoder(in_channels, shape, base_channels=base, encoder_channels=ch,
                         encoder_paddings=((1,), (1, 1, 1), (1, 1, 1))[:depth])


def wide(shape, in_channels):
    """Cout 64 / 128 chains: with c_in 16 the first conv (27 x 16 channels: 14 K blocks of 32) and conv_out
    (3 x 128: 12) run on mma.sync, the 64 / 128-channel SubMs (>= 54 blocks) on wgmma"""
    return SparseEncoder(in_channels, shape, base_channels=64, output_channels=128,
                         encoder_channels=((64,), (128, 128)), encoder_paddings=((1,), (1, 1)))


CASES = {
    # name: (builder, shape, batch, voxels per sample)
    "voxelnet-b2": (lambda s: voxelnet(s), [48, 48, 41], 2, 1500),
    "stages3-cin5": (lambda s: stages(s, 3), [40, 40, 41], 1, 1200),
    "wide-cin16": (lambda s: wide(s, 16), [32, 32, 21], 1, 800),
    "wide-cin128": (lambda s: wide(s, 128), [32, 32, 21], 1, 600),
}


def _coors(shape, B, n, seed):
    rng = np.random.default_rng(seed)
    X, Y, Z = shape
    rows = []
    for b in range(B):
        flat = rng.choice(X * Y * Z, size=n, replace=False)
        rows.append(np.stack([np.full(n, b), flat // (Y * Z), (flat // Z) % Y, flat % Z], 1))
    return np.concatenate(rows).astype(np.int32)


def _make(case, dev, seed=0, half_features=False):
    build, shape, B, n = CASES[case]
    torch.manual_seed(seed)
    m = _randomise_bn(build(shape), seed).to(dev)
    coors = _coors(shape, B, n, seed)
    g = torch.Generator().manual_seed(seed + 1)
    feats = torch.randn(coors.shape[0], m.in_channels, generator=g)
    feats = (feats.half() if half_features else feats).to(dev)
    return m, feats, coors, shape, B


def _params(plan):
    return ([cv.weight for cv, _, _, _ in plan.chain], [bn.weight for _, bn, _, _ in plan.chain],
            [bn.bias for _, bn, _, _ in plan.chain])


def _probe(m, feats, coors_dev, B, n_dev):
    """a training forward of a copy of m (the step is deterministic, so its state is the run's): (dense, saved
    [(z16, y16)] per conv over the valid rows, running statistics before / after, the plan)"""
    probe = copy.deepcopy(m).train()
    plan = probe.plan(PREC_FP16)
    before = [(bn.running_mean.clone(), bn.running_var.clone()) for _, bn, _, _ in plan.chain]
    with torch.no_grad():
        out, state = plan._forward_train_native(feats, coors_dev, B, n_dev, None, True, *_params(plan))
    counts = [int(v) for v in plan.status[1:].tolist()]
    saved = []
    for i in range(len(plan.chain)):
        z, y = plan.saved_rows(state, feats.shape[0], B, i)
        k = counts[plan.level_of(i)]
        saved.append((z[:k].double().cpu(), y[:k].double().cpu()))
    after = [(bn.running_mean.clone(), bn.running_var.clone()) for _, bn, _, _ in plan.chain]
    return out, saved, before, after, plan


def _bns(plan):
    return [(bn.weight, bn.bias, bn.eps, bn.momentum) for _, bn, _, _ in plan.chain]


@pytest.mark.parametrize("case", list(CASES))
def test_train_forward_per_conv(cuda, case):
    m, feats, coors, shape, B = _make(case, cuda, half_features=case.endswith("128"))
    cd = torch.from_numpy(coors).to(cuda)
    n_dev = torch.tensor([coors.shape[0]], dtype=torch.int32, device=cuda)
    out, saved, before, after, plan = _probe(m, feats, cd, B, n_dev)
    assert out.dtype == torch.float16
    convs = module_convs(plan)
    rbs = rulebooks(convs, coors, B, shape)
    worst = check_train_forward(convs, fp16_round(feats.double().cpu()), [cv.weight for cv, _, _, _ in plan.chain],
                                _bns(plan), saved, before, after, rbs, case)
    assert torch.equal(out.double().cpu(), dense64(saved[-1][1], rbs[-1][0], B, rbs[-1][2]))
    print("%s: worst ratio %s" % (case, {k: round(v, 3) for k, v in worst.items()}))


@pytest.mark.parametrize("case", list(CASES))
def test_backward_vs_float64(cuda, case):
    m, feats, coors, shape, B = _make(case, cuda, seed=3)
    m.train()
    cd = torch.from_numpy(coors).to(cuda)
    n_dev = torch.tensor([coors.shape[0]], dtype=torch.int32, device=cuda)
    _, saved, _, _, plan = _probe(m, feats, cd, B, n_dev)
    x = feats.detach().clone().requires_grad_(True)
    out = m(x, cd, B, num_voxels=n_dev, precision=PREC_FP16)
    R = fp16_round(torch.randn(out.shape, generator=torch.Generator().manual_seed(9), dtype=torch.float64))
    (out.float() * R.float().to(cuda)).sum().backward()
    convs = module_convs(plan)
    rbs = rulebooks(convs, coors, B, shape)
    gx, gw, gg, gb = twin_backward(convs, rbs, fp16_round(feats.double().cpu()),
                                   [cv.weight for cv, _, _, _ in plan.chain], _bns(plan), saved, R, B)
    bound, bound_x = bwd_bounds(len(plan.chain))
    rows = [("input", x.grad, gx, bound_x)]
    for i, (conv, bn, _, _) in enumerate(m.plan(PREC_FP16).chain):
        rows += [("conv %d" % i, conv.weight.grad.reshape(gw[i].shape), gw[i], bound),
                 ("bn weight %d" % i, bn.weight.grad, gg[i], bound), ("bn bias %d" % i, bn.bias.grad, gb[i], bound)]
    worst = 0.0
    for name, got, want, b in rows:
        assert got.dtype == torch.float32
        assert bool(torch.isfinite(got).all()), name
        l2, _ = rel(got.cpu(), want)
        worst = max(worst, l2 / b)
        assert l2 <= b, (name, l2, b)
    print("%s: worst rel L2 / bound = %.3f" % (case, worst))


@pytest.mark.parametrize("case", ["depth1", "depth2", "depth3", "voxelnet"])
def test_eval_forward_vs_twin(cuda, case):
    shape = [40, 40, 41]
    torch.manual_seed(4)
    m = voxelnet(shape) if case == "voxelnet" else stages(shape, int(case[-1]))
    m = _randomise_bn(m, 4).to(cuda).eval()
    coors = _coors(shape, 2, 1000, 4)
    feats = torch.randn(coors.shape[0], 5, generator=torch.Generator().manual_seed(5)).to(cuda)
    with torch.no_grad():
        out = m(feats, torch.from_numpy(coors).to(cuda), 2, precision=PREC_FP16)
    assert out.dtype == torch.float16
    ref, absref = eval_twin(m.plan(PREC_FP16), feats, coors, 2, shape)
    depth = len(m.plan(PREC_FP16).chain)
    print("%s: worst ratio %.3f" % (case, check(out.cpu(), ref, absref, case, c_eval(depth))))


def test_half_weights_equal_master(cuda):
    """model.half() (half weights, BN widened) and fp32 master weights holding the same fp16 values train alike"""
    m, feats, coors, _, B = _make("stages3-cin5", cuda, seed=6)
    for p in m.parameters():
        p.data.copy_(p.data.half().float())
    for b in m.buffers():
        if b.dtype == torch.float32:
            b.copy_(b.half().float())
    h = copy.deepcopy(m).half()
    cd = torch.from_numpy(coors).to(cuda)
    n_dev = torch.tensor([coors.shape[0]], dtype=torch.int32, device=cuda)
    outs = []
    for mod in (m, h):
        mod.train()
        o = mod(feats.half(), cd, B, num_voxels=n_dev, precision=PREC_FP16)
        o.float().sum().backward()
        outs.append(o)
    assert torch.equal(outs[0], outs[1])
    for (k, p), (_, q) in zip(m.named_parameters(), h.named_parameters()):
        assert q.grad.dtype == torch.float16
        assert torch.equal(p.grad.half(), q.grad), k


def test_gradscaler_skips_overflow(cuda):
    """A gradient that overflows inside the backward gives non-finite gradients: the scaler skips the step and lowers
    its scale, and the next step with the same scaler trains normally.  The dense gradient is finite in fp16; the
    overflow is the kernel's rounding of the last BN's dz = gamma invstd (g - ...): conv_out's weights shrunk by 1e-3
    make its variance far below eps, so invstd ~ eps^-1/2 ~ 32, and gamma = 8 puts dz past 65504 at a scale of 2^12."""
    m, feats, coors, _, B = _make("stages3-cin5", cuda, seed=7)
    m.train()
    m.conv_out[0].weight.data.mul_(1e-3)
    m.conv_out[1].weight.data.fill_(8.0)
    cd = torch.from_numpy(coors).to(cuda)
    n_dev = torch.tensor([coors.shape[0]], dtype=torch.int32, device=cuda)
    opt = torch.optim.SGD(m.parameters(), lr=1e-3)
    scale = 2.0 ** 12
    scaler = torch.amp.GradScaler("cuda", init_scale=scale, backoff_factor=2.0 ** -12, growth_interval=2000)
    before = {k: p.detach().clone() for k, p in m.named_parameters()}
    X, Y, Z = m.plan(PREC_FP16).out_shape
    R = torch.randn((B, m.plan(PREC_FP16).out_channels * Z, X, Y), generator=torch.Generator().manual_seed(3)).clamp(-3, 3).half().float().to(cuda)
    assert float((R * scale).abs().max()) < 65504                 # the dense gradient itself is finite in fp16

    def step():
        out = m(feats, cd, B, num_voxels=n_dev, precision=PREC_FP16)
        scaler.scale((out.float() * R).sum()).backward()

    step()
    assert not all(bool(torch.isfinite(p.grad).all()) for p in m.parameters())
    scaler.step(opt)
    scaler.update()
    assert scaler.get_scale() == 1.0
    for k, p in m.named_parameters():
        assert torch.equal(p.detach(), before[k]), k               # the step was skipped
    opt.zero_grad(set_to_none=True)
    step()
    assert all(bool(torch.isfinite(p.grad).all()) for p in m.parameters())
    scaler.step(opt)
    scaler.update()
    assert scaler.get_scale() == 1.0
    assert any(not torch.equal(p.detach(), before[k]) for k, p in m.named_parameters())


def test_precision_isolation(cuda):
    """an fp16 step, then a bf16x3 step on the same module: the bf16x3 step is the one a fresh module makes"""
    m, feats, coors, _, B = _make("stages3-cin5", cuda, seed=8)
    ref = copy.deepcopy(m).train()
    m.train()
    cd = torch.from_numpy(coors).to(cuda)
    n_dev = torch.tensor([coors.shape[0]], dtype=torch.int32, device=cuda)
    with torch.no_grad():
        m(feats, cd, B, num_voxels=n_dev, precision=PREC_FP16)
    for a, b in zip(m.buffers(), ref.buffers()):            # undo the fp16 step's running statistics
        a.copy_(b)
    outs = []
    for mod in (m, ref):
        o = mod(feats, cd, B, num_voxels=n_dev, precision=PREC_BF16X3)
        o.sum().backward()
        outs.append(o)
    assert outs[0].dtype == torch.float32 and torch.equal(outs[0], outs[1])
    for (k, p), (_, q) in zip(m.named_parameters(), ref.named_parameters()):
        assert torch.equal(p.grad, q.grad), k
    m.eval(); ref.eval()
    with torch.no_grad():
        e16 = m(feats, cd, B, precision=PREC_FP16)
        e3 = m(feats, cd, B, precision=PREC_BF16X3)
        assert torch.equal(e3, ref(feats, cd, B, precision=PREC_BF16X3))
        assert torch.equal(e16, m(feats, cd, B, precision=PREC_FP16))


def test_sync_free_graph_and_reproducible(cuda):
    from bevfusion_b200 import synthetic as S
    from bevfusion_b200.voxelize import voxelize_mean_fused
    L = S.LIDAR_C3
    rng = [-12.0, -12.0, -5.0, 12.0, 12.0, 3.0]
    clouds = [torch.from_numpy(S.lidar_cloud(seed=s)[:60000]).to(cuda) for s in (1, 2)]
    torch.manual_seed(10)
    m = _randomise_bn(SparseEncoder(5, [320, 320, 41]), 10).to(cuda).train()
    eager = copy.deepcopy(m)
    R = None

    def step(model, opt, pts):
        f, c, _, n_dev = voxelize_mean_fused(pts, L["voxel_size"], rng, L["max_num_points"], 30000, sync=False)
        out = model(f, c, 1, num_voxels=n_dev, precision=PREC_FP16)
        (out.float() * R).sum().backward()
        opt.step()
        return out

    opt = torch.optim.SGD(m.parameters(), lr=1e-3, momentum=0.9)
    opt_e = torch.optim.SGD(eager.parameters(), lr=1e-3, momentum=0.9)
    static = clouds[0].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    X, Y, Z = m.plan(PREC_FP16).out_shape
    R = torch.randn((1, 128 * Z, X, Y), device=cuda, generator=torch.Generator(device=cuda).manual_seed(2)) * 1e-3
    with torch.cuda.stream(side):
        step(m, opt, static)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.set_sync_debug_mode("error")
    try:
        step(eager, opt_e, static)                               # no device-to-host sync inside the step
    finally:
        torch.cuda.set_sync_debug_mode("default")
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
        assert torch.equal(og, step(eager, opt_e, pts).detach())
    for (k, p), (_, q) in zip(m.named_parameters(), eager.named_parameters()):
        assert torch.equal(p.detach(), q.detach()), k
    for (k, b), (_, c) in zip(m.named_buffers(), eager.named_buffers()):
        assert torch.equal(b, c), k


def test_refusals_write_nothing(cuda):
    m, feats, coors, _, B = _make("stages3-cin5", cuda, seed=11)
    cd = torch.from_numpy(coors).to(cuda)
    n_dev = torch.tensor([coors.shape[0]], dtype=torch.int32, device=cuda)
    buffers = {k: b.clone() for k, b in m.named_buffers()}

    def raises(mod, match, **kw):
        with pytest.raises(ValueError, match=match):
            mod(feats, cd, B, precision=PREC_FP16, **kw)
        for k, b in mod.named_buffers():
            assert torch.equal(b, buffers[k]), k

    m.train()
    raises(m, "num_voxels")                                    # training without num_voxels
    raises(m, "out=", num_voxels=n_dev, out=torch.empty(1, device=cuda))
    mb = copy.deepcopy(m)
    mb.conv_input[0].bias = torch.nn.Parameter(torch.zeros(16, device=cuda))
    raises(mb, "bias", num_voxels=n_dev)
    mm = copy.deepcopy(m)
    mm.conv_input[1].momentum = None
    raises(mm, "momentum", num_voxels=n_dev)
    m.eval()
    raises(m, "fused", fused=False)                            # the per-conv ops have no fp16 form
    raises(m, "no_grad")                                       # eval with grad enabled
    mo = SparseEncoder(5, [40, 40, 41], base_channels=24).to(cuda).eval()   # 24 channels: no tensor-core form
    with torch.no_grad(), pytest.raises(ValueError, match="chain"):
        mo(feats, cd, B, precision=PREC_FP16)
    with torch.no_grad(), pytest.raises(ValueError, match="half"):
        m(feats, cd, B, precision=PREC_FP16, out=torch.empty(1, device=cuda))


def test_wrong_precision_calls_write_nothing(cuda):
    """an fp16 plan refuses the fp32 calls, a bf16x3 plan the _f16 calls: BEVB200_EINVAL, the output untouched"""
    m, feats, coors, _, B = _make("stages3-cin5", cuda, seed=12)
    m.eval()
    cd = torch.from_numpy(coors).to(cuda)
    L = _C.lib()
    for plan, fwd in ((m.plan(PREC_FP16), L.bevb200_encoder_forward), (m.plan(), L.bevb200_encoder_forward_f16)):
        n = feats.shape[0]
        ws = torch.empty(L.bevb200_encoder_workspace_bytes(plan._h, n, B, None) + 256, dtype=torch.uint8, device=cuda)
        params = torch.zeros(max(L.bevb200_encoder_param_bytes(plan._h), 256), dtype=torch.uint8, device=cuda)
        out = torch.full((B * 4096,), 7.0, device=cuda)
        status = torch.full((1 + plan.n_levels,), -3, dtype=torch.int32, device=cuda)
        rc = fwd(plan._h, _C.ptr(params), _C.ptr(feats), _C.ptr(cd), n, None, B, None, _C.ptr(out), 0,
                 _C.ptr(status), _C.ptr(ws), ws.numel(), _C.current_stream(cuda), None)
        torch.cuda.synchronize()
        assert rc == -1
        assert bool((out == 7.0).all()) and bool((status == -3).all())
