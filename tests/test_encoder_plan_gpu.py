"""GPU tests of the native SparseEncoder plan (bevb200_encoder_*, encoder_plan.py) against float64.

  * Every chain encoder_plan.supported() accepts: the voxelnet chain (basicblock), the default SparseEncoder
    (SECOND-style conv_module blocks, a (0, 1, 1) padding in stage 4, no residuals) and a basicblock chain with
    in_channels 4 and a conv bias, on small grids and on odd ones (site bitmaps ending partway through a word,
    voxels on every border face and in the very last site, an empty sample, unsorted rows).  Each is compared with
    an eval-mode float64 twin (tests/encoder_oracle.py): dense output within 1e-4 of max |float64|, the per-level
    row counts in plan.status exact, empty samples and inactive cells exactly 0.
  * Raw C-ABI chains built with bevb200_encoder_create / _set_conv / _forward, against float64 convs on
    ops.get_rulebook tables: residuals from one and two convs back and on the last conv, an all-SubM chain and a
    strided first conv.  (A residual from further back is refused by bevb200_encoder_create:
    test_encoder_plan_cpu.py.)
  * The packed parameters follow the module: after a training step, after load_state_dict, and after train-mode
    forwards that move only the BN statistics (also through the per-conv loop)."""
import copy
import ctypes

import numpy as np
import pytest
import torch

from bevfusion_b200 import _C
from encoder_oracle import conv_nbr, dense_zmajor, encoder_forward, epilogue

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------- helpers
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


def voxelnet(shape, seed=0):
    """the voxelnet_0p075 encoder on another grid"""
    from bevfusion_b200.sparse_encoder import SparseEncoder
    torch.manual_seed(seed)
    m = SparseEncoder(in_channels=5, sparse_shape=shape, output_channels=128,
                      encoder_channels=((16, 16, 32), (32, 32, 64), (64, 64, 128), (128, 128)),
                      encoder_paddings=((0, 0, 1), (0, 0, 1), (0, 0, (1, 1, 0)), (0, 0)), block_type="basicblock")
    return _randomise_bn(m, seed)


def default_encoder(shape, seed=0):
    """SparseEncoder(5, shape) with every default: conv_module blocks, stage 4 padded (0, 1, 1), no residual"""
    from bevfusion_b200.sparse_encoder import SparseEncoder
    torch.manual_seed(seed)
    return _randomise_bn(SparseEncoder(5, shape), seed)


def basic_with_bias(shape, seed=0):
    """a three-stage basicblock chain on 4 input channels, with a bias on conv_input's conv"""
    from bevfusion_b200.sparse_encoder import SparseEncoder
    torch.manual_seed(seed)
    m = SparseEncoder(in_channels=4, sparse_shape=shape, output_channels=128,
                      encoder_channels=((16, 16, 32), (32, 32, 64), (64, 64)),
                      encoder_paddings=((0, 0, 1), (0, 0, 1), (0, 0)), block_type="basicblock")
    m.conv_input[0].bias = torch.nn.Parameter(torch.randn(16) * 0.3)
    return _randomise_bn(m, seed)


CHAINS = {"voxelnet": voxelnet, "default": default_encoder, "basic-bias": basic_with_bias}


def random_coors(shape, B, n, seed):
    rng = np.random.default_rng(seed)
    X, Y, Z = shape
    flat = rng.choice(B * X * Y * Z, size=n, replace=False)
    z = flat % Z; y = (flat // Z) % Y; x = (flat // (Z * Y)) % X; b = flat // (Z * Y * X)
    return np.stack([b, x, y, z], 1).astype(np.int32)


def odd_coors(shape, B, n, seed, empty=1):
    """n random voxels of B samples, sample `empty` left out, plus voxels on all six border faces of every other
    sample and the last site of the last sample; rows shuffled (not batch-sorted)."""
    rng = np.random.default_rng(seed)
    X, Y, Z = shape
    idx = random_coors(shape, B, n, seed)
    border = []
    for b in range(B):
        if b == empty:
            continue
        for _ in range(6):
            x, y, z = rng.integers(0, X), rng.integers(0, Y), rng.integers(0, Z)
            border += [[b, 0, y, z], [b, X - 1, y, z], [b, x, 0, z], [b, x, Y - 1, z], [b, x, y, 0], [b, x, y, Z - 1]]
    border.append([B - 1, X - 1, Y - 1, Z - 1])
    idx = np.concatenate([idx[idx[:, 0] != empty], np.array(border, np.int32)])
    idx = np.unique(idx, axis=0)
    return idx[rng.permutation(idx.shape[0])]


def twin_of(m):
    """eval-mode float64 copy of m (without its native plan, which owns a C handle, nor its rulebook side streams)"""
    plan, m._plan = m._plan, None
    streams = m.__dict__.pop("_rulebook_streams", None)
    try:
        t = copy.deepcopy(m)
    finally:
        m._plan = plan
        if streams is not None:
            m._rulebook_streams = streams
    return t.double().eval()


def check_plan(m, feats, coors, B, what, empty=()):
    """the native plan on (feats, coors) vs the float64 twin of m: returns the relative error"""
    from bevfusion_b200 import encoder_plan
    m.eval()
    assert encoder_plan.supported(m)
    plan = m.plan()
    with torch.no_grad():
        got = plan.forward(feats, coors, B)
    want, active, rows = encoder_forward(twin_of(m), feats.double(), coors, B)
    assert got.shape == want.shape
    err = float((got.double() - want).abs().max() / want.abs().max())
    status = plan.status.cpu().tolist()
    print("%-28s %6d voxels  rows per level %s  max |float64| %.3g  rel err %.2e" % (
        what, coors.shape[0], rows, float(want.abs().max()), err))
    assert err <= 1e-4, "%s: rel err %.3e" % (what, err)
    assert status[0] == 0 and status[1:] == rows, "%s: rows per level %s, float64 %s" % (what, status[1:], rows)
    assert not bool(got[~active].any()), "%s: an inactive cell is not 0" % what
    for b in empty:
        assert not bool(got[b].any()), "%s: empty sample %d is not 0" % (what, b)
    return err


# ---------------------------------------------------------------------------------------------------- chains
# (small grid, odd grid): the odd one's site bitmaps end partway through a word (the voxelnet chain's k(1,1,3)
# s(1,1,2) conv_out needs z >= 25 there)
GRIDS = {"voxelnet": ([96, 88, 41], [57, 43, 41]), "default": ([96, 88, 21], [57, 43, 23]),
         "basic-bias": ([96, 88, 21], [57, 43, 23])}


@pytest.mark.parametrize("chain", list(CHAINS))
def test_plan_vs_float64_small_grid(cuda, chain):
    shape = GRIDS[chain][0]
    m = CHAINS[chain](shape).to(cuda)
    B = 2
    coors = torch.from_numpy(random_coors([shape[0], shape[1], shape[2] - 1], B, 6000, seed=3)).to(cuda)
    g = torch.Generator(device=cuda).manual_seed(1)
    feats = torch.randn(coors.shape[0], m.in_channels, device=cuda, generator=g)
    check_plan(m, feats, coors, B, chain + " " + "x".join(map(str, shape)))


@pytest.mark.parametrize("chain", list(CHAINS))
def test_plan_vs_float64_odd_grid(cuda, chain):
    shape = GRIDS[chain][1]
    m = CHAINS[chain](shape, seed=2).to(cuda)
    B = 3
    coors = torch.from_numpy(odd_coors(shape, B, 5000, seed=4)).to(cuda)
    assert shape[0] * shape[1] * shape[2] % 32 != 0
    g = torch.Generator(device=cuda).manual_seed(5)
    feats = torch.randn(coors.shape[0], m.in_channels, device=cuda, generator=g)
    check_plan(m, feats, coors, B, chain + " odd " + "x".join(map(str, shape)), empty=(1,))


def test_plan_follows_parameter_updates(cuda):
    """The packed parameters are re-made when a weight, BN parameter or BN statistic changes: after a train-mode
    step (SGD step and the BN statistics update) and after load_state_dict."""
    shape, B = [64, 56, 41], 2
    m = voxelnet(shape, seed=6).to(cuda)
    coors = torch.from_numpy(random_coors([64, 56, 40], B, 4000, seed=7)).to(cuda)
    feats = torch.randn(coors.shape[0], 5, device=cuda, generator=torch.Generator(device=cuda).manual_seed(8))
    check_plan(m, feats, coors, B, "before the step")
    with torch.no_grad():
        before = m.plan().forward(feats, coors, B).clone()

    m.train()
    opt = torch.optim.SGD(m.parameters(), lr=0.5)
    out = m(feats, coors, B)
    R = torch.randn(out.shape, device=cuda, generator=torch.Generator(device=cuda).manual_seed(9))
    (out * R).sum().backward()
    torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)          # a step of norm 0.5: the net stays in fp32 range
    opt.step()
    check_plan(m, feats, coors, B, "after a training step")
    with torch.no_grad():
        after = m.plan().forward(feats, coors, B)
    change = float((after - before).abs().max() / before.abs().max())
    print("the step moved the output by %.2e of max |output|" % change)
    assert change > 1e-3, "the step changed too little for a stale parameter image to show"

    m.load_state_dict(voxelnet(shape, seed=10).state_dict())
    check_plan(m, feats, coors, B, "after load_state_dict")


@pytest.mark.parametrize("path", ["loop", "plan"])
def test_bn_refold_after_train_mode_forward(cuda, path):
    """eval forward, train-mode forwards under no_grad (BN recalibration: the statistics move, no parameter does), eval
    again: the per-conv loop (bn_scale_shift) and the native plan (its packed parameters) follow the new statistics."""
    shape, B = [64, 56, 41], 2
    m = voxelnet(shape, seed=12).to(cuda)
    m.native_plan = path == "plan"
    coors = torch.from_numpy(random_coors([64, 56, 40], B, 4000, seed=13)).to(cuda)
    feats = torch.randn(coors.shape[0], 5, device=cuda, generator=torch.Generator(device=cuda).manual_seed(14))
    m.eval()
    with torch.no_grad():
        before = m(feats, coors, B).clone()
        m.train()
        for _ in range(3):
            m(feats, coors, B)
        m.eval()
        got = m(feats, coors, B)
    assert bool(m._plan) == (path == "plan")
    want, _, _ = encoder_forward(twin_of(m), feats.double(), coors, B)
    moved = float((want - before.double()).abs().max() / want.abs().max())
    err = float((got.double() - want).abs().max() / want.abs().max())
    print("%s: the train-mode forwards moved the output by %.2e, rel err %.2e" % (path, moved, err))
    assert moved > 1e-3, "the statistics moved too little for a stale fold to show"
    assert err <= 1e-4, "%s: rel err %.3e after the statistics moved" % (path, err)


# ---------------------------------------------------------------------------------------------------- raw C ABI
def conv(cin, cout, subm=True, res=-1, relu=True, scale=True, shift=True, ks=3, stride=2, pad=1):
    return dict(cin=cin, cout=cout, subm=subm, res=res, relu=relu, scale=scale, shift=shift,
                ks=[ks] * 3 if isinstance(ks, int) else ks, stride=[1] * 3 if subm else [stride] * 3,
                pad=[pad] * 3)


def create(in_channels, shape, convs):
    """bevb200_encoder_create -> (return code, handle or None)"""
    from bevfusion_b200.encoder_plan import _ConvDesc
    arr = (_ConvDesc * len(convs))()
    for a, c in zip(arr, convs):
        a.c_in, a.c_out, a.subm, a.relu, a.residual_from = c["cin"], c["cout"], int(c["subm"]), int(c["relu"]), c["res"]
        for k in range(3):
            a.ksize[k], a.stride[k], a.padding[k], a.dilation[k] = c["ks"][k], c["stride"][k], c["pad"][k], 1
    h = ctypes.c_void_p()
    rc = _C.lib().bevb200_encoder_create(in_channels, (ctypes.c_int32 * 3)(*shape), arr, len(convs), ctypes.byref(h))
    return rc, (h if rc == 0 else None)


def run_raw_chain(cuda, in_channels, shape, B, convs, n, seed):
    """The chain through the C ABI on n random voxels (unsorted) vs float64 convs on ops.get_rulebook tables.
    -> (relative error, rows per level)"""
    from bevfusion_b200.spconv import ops
    L = _C.lib()
    gen = torch.Generator(device=cuda).manual_seed(seed)
    coors = torch.from_numpy(random_coors(shape, B, n, seed)).to(cuda)
    feats = torch.randn(n, in_channels, device=cuda, generator=gen)
    params = []
    for c in convs:
        kv = int(np.prod(c["ks"]))
        params.append((torch.randn(kv, c["cin"], c["cout"], device=cuda, generator=gen) / (kv * c["cin"]) ** 0.5,
                       torch.rand(c["cout"], device=cuda, generator=gen) + 0.5 if c["scale"] else None,
                       torch.randn(c["cout"], device=cuda, generator=gen) * 0.2 if c["shift"] else None))
    rc, h = create(in_channels, shape, convs)
    assert rc == 0, L.bevb200_last_error()
    stream = _C.current_stream(cuda)
    try:
        pbuf = torch.empty(max(L.bevb200_encoder_param_bytes(h), 256), dtype=torch.uint8, device=cuda)
        for i, (w, s, t) in enumerate(params):
            _C.check(L.bevb200_encoder_set_conv(h, i, _C.ptr(w), _C.ptr(s), _C.ptr(t), _C.ptr(pbuf), pbuf.numel(),
                                                stream), "encoder_set_conv")
        ws = torch.empty(L.bevb200_encoder_workspace_bytes(h, n, B, None), dtype=torch.uint8, device=cuda)
        oshape, oc = (ctypes.c_int32 * 3)(), ctypes.c_int32()
        _C.check(L.bevb200_encoder_output_shape(h, oshape, ctypes.byref(oc)), "encoder_output_shape")
        X, Y, Z = list(oshape)
        out = torch.full((B, oc.value * Z, X, Y), float("nan"), device=cuda)
        status = torch.full((1 + L.bevb200_encoder_num_levels(h),), -1, dtype=torch.int32, device=cuda)
        _C.check(L.bevb200_encoder_forward(h, _C.ptr(pbuf), _C.ptr(feats), _C.ptr(coors), n, None, B, None,
                                           _C.ptr(out), 0, _C.ptr(status), _C.ptr(ws), ws.numel(), stream, None),
                 "encoder_forward")
        torch.cuda.synchronize()
    finally:
        L.bevb200_encoder_destroy(h)

    idx, cur, rows, outs = coors, list(shape), [n], []
    x = feats
    for c, (w, s, t) in zip(convs, params):
        rb, oshape_c = ops.get_rulebook(idx, B, cur, c["ks"], c["stride"], c["pad"], 1, 0, c["subm"])
        x = epilogue(conv_nbr(x, w, rb.nbr), s, t, outs[c["res"]] if c["res"] >= 0 else None, c["relu"])
        outs.append(x)
        if not c["subm"]:
            idx, cur = rb.outids, oshape_c
            rows.append(int(rb.n_out))
    want = dense_zmajor(x, idx, B, cur)
    assert list(oshape) == cur and out.shape == want.shape
    err = float((out.double() - want).abs().max() / want.abs().max())
    assert status.cpu().tolist() == [0] + rows
    active = dense_zmajor(torch.ones_like(x), idx, B, cur) != 0
    assert not bool(out[~active].any())
    return err, rows


RAW_CHAINS = {
    # conv 2 adds conv 1's output (its own input), then a strided conv closes the level
    "residual-previous": (5, [conv(5, 16), conv(16, 16), conv(16, 16, res=1), conv(16, 32, subm=False)]),
    # conv 2 adds conv 0's output: the split image it overwrites (the SparseBasicBlock case)
    "residual-two-back": (5, [conv(5, 16), conv(16, 16, scale=False), conv(16, 16, res=0), conv(16, 32, subm=False)]),
    # the last conv (fp32 rows only) adds the strided conv's output on level 1
    "residual-on-last": (5, [conv(5, 16), conv(16, 32, subm=False), conv(32, 32, shift=False), conv(32, 32, res=1)]),
    # one level: dense() scatters the caller's rows; Cin 7 is padded to 16
    "all-subm": (7, [conv(7, 16, relu=False), conv(16, 32), conv(32, 32, res=1, scale=False, shift=False)]),
    # level 0 holds only the input image
    "strided-first": (5, [conv(5, 16, subm=False), conv(16, 16), conv(16, 16, res=0, relu=False)]),
}


@pytest.mark.parametrize("chain", list(RAW_CHAINS))
def test_raw_chain_vs_float64(cuda, chain):
    in_channels, convs = RAW_CHAINS[chain]
    err, rows = run_raw_chain(cuda, in_channels, [40, 36, 15], 2, convs, 3000, seed=len(chain))
    print("raw chain %-18s rows per level %s  rel err %.2e" % (chain, rows, err))
    assert err <= 1e-4

