"""GPU tests of the sparse conv's fp16 paths against float64, at one fp16 rounding (tests/half_oracle.py).

Mixed-precision training hands SparseEncoder half voxel features (the reference's SparseEncoder.forward is
auto_fp16).  Every half path widens to fp32, runs the fp32 kernels and narrows once, so each result must be within
ulp16(ref) + C_BF16X3 * absref of the float64 conv of the half-rounded inputs; every case prints its worst ratio.

  * The half entry points of the python `sparse_conv_ext` stand-in -- indice_conv_half, fused_indice_conv_half and
    indice_conv_backward_half -- on the channel pairs, kernel volumes and row counts of the forward and backward
    dispatch tables, with reference [K, 2, N] pairs and with a Rulebook, and the compiled drop-in module, which must
    give bit-for-bit the same tensors.  Mixed dtypes: the output is half when the features or the filters are; each
    gradient has the dtype of its tensor.  Out-grads scaled by 2^k like a dynamic loss scaler's, results past 65504
    (inf of the right sign), NaN and inf inputs (as on the fp32 path).
  * Real rulebooks: SubM k3, the encoder's strided k3 s2 convs and conv_out's (1, 1, 3) s(1, 1, 2).
  * SubMConv3d / SparseConv3d / SparseBasicBlock with half weights and with fp32 weights on half features: grad
    enabled, torch.no_grad(), the fused BN + ReLU epilogue and the fused residual; SparseConvTensor.dense() in half.
  * A voxelnet-chain SparseEncoder with half features: eval mode (every conv checked on its own half input through
    forward hooks, the output dtype, the fp32 native plan untouched) and a training step (every filter gradient
    checked on the conv's own input and out-grad, end to end against a float64 twin)."""
import copy

import numpy as np
import pytest
import torch

from encoder_oracle import conv_nbr, dense_zmajor, epilogue
from half_oracle import C_BF16X3, check, ulp
from test_spconv_backward_gpu import DISPATCH as BWD_DISPATCH
from test_spconv_backward_gpu import _twin_forward, random_table, reference
from test_spconv_forward_gpu import DISPATCH as FWD_DISPATCH

pytestmark = pytest.mark.gpu

H, F = torch.float16, torch.float32
DTYPES = {"half": (H, H), "half-f/fp32-w": (H, F), "fp32-f/half-w": (F, H)}


@pytest.fixture(scope="module")
def shim():
    from bevfusion_b200.shims import build as shim_build
    return shim_build.load_module("sparse_conv_ext")


# (cin, cout, kv, n_out) of the dispatch tables' BF16x3 rows (the half entry points run BF16x3); the forward table
# holds (prec, cin, cout, kv, family, mis, n_out), the backward one (prec, cin, cout, kv, n_out, geom, misalign)
FWD_SHAPES = sorted({(v[1], v[2], v[3], v[6]) for v in (p.values for p in FWD_DISPATCH) if v[0] == 3})
BWD_SHAPES = sorted({(v[1], v[2], v[3], v[4]) for v in (p.values for p in BWD_DISPATCH) if v[0] == 3})
# row counts around the 128-row (SIMT, mma.sync) and 256-row (wgmma) output tiles, the 32-row filter-gradient tile
ROW_SHAPES = [(cin, cout, 27, n) for cin, cout in ((32, 32), (64, 64), (16, 48)) for n in (127, 128, 129, 255, 256, 257)]


def _table(kv, n_out, gen):
    """injective neighbour table (the reference pairs layout can hold it), 40 % of the entries missing, one offset
    without pairs, and every 13th output row from row 6 on with no neighbour at all"""
    n_in = n_out + n_out // 8 + 16
    nbr = random_table(kv, n_in, n_out, gen, junk=False)
    nbr[:, 6::13] = -1
    return nbr, n_in


def _inputs(cin, cout, kv, n_in, gen, fdt, wdt, fscale=1.0, wscale=1.0):
    dev = gen.device
    f = (torch.randn(n_in, cin, device=dev, generator=gen) * fscale).to(fdt)
    w = (torch.randn(kv, cin, cout, device=dev, generator=gen) * wscale / (cin * kv) ** 0.5).to(wdt)
    b = (torch.randn(cout, device=dev, generator=gen) * 0.5).to(wdt)
    return f, w, b


def _out_dtype(*ts):
    return H if any(t.dtype == H for t in ts) else F


# ---------------------------------------------------------------------------------------------------- forward
def forward_case(shim, cin, cout, kv, n_out, seed, fdt, wdt, fscale=1.0, wscale=1.0):
    from bevfusion_b200.spconv import ops
    cuda = torch.device("cuda:0")
    gen = torch.Generator(device=cuda).manual_seed(seed)
    nbr, n_in = _table(kv, n_out, gen)
    rb = ops.Rulebook(None, nbr, n_in, n_out, kv)
    pairs, num = rb.pairs()
    f, w, b = _inputs(cin, cout, kv, n_in, gen, fdt, wdt, fscale, wscale)
    ext = ops.sparse_conv_ext
    want_dt = _out_dtype(f, w)
    tag = "%d->%d k%d n_out %d %s/%s" % (cin, cout, kv, n_out, str(fdt)[6:], str(wdt)[6:])
    ref = conv_nbr(f, w, nbr)
    absref = conv_nbr(f.abs(), w.abs(), nbr)
    empty = ~(nbr >= 0).any(0)
    assert bool(empty.any()) or n_out <= 6
    ratios = []
    for name, bias in (("indice_conv_half", None), ("fused_indice_conv_half", b)):
        args = () if bias is None else (bias,)
        got = getattr(ext, name)(f, w, *args, pairs, num, n_out, 0, 1)
        assert got.dtype == want_dt, "%s %s: dtype %s" % (name, tag, got.dtype)
        assert torch.equal(getattr(ext, name)(f, w, *args, rb, None, n_out, 0, 1), got), \
            "%s %s: a Rulebook and reference pairs give different results" % (name, tag)
        assert torch.equal(getattr(shim, name)(f, w, *args, pairs, num, n_out, 0, 1), got), \
            "%s %s: the compiled module differs from the python stand-in" % (name, tag)
        r, a = (ref, absref) if bias is None else (ref + bias.double(), absref + bias.double().abs())
        ratios.append(check(got, r, a, "%s %s" % (name, tag)))
        # rows with no neighbour: exactly 0, or the bias narrowed once
        want = torch.zeros(cout, device=cuda) if bias is None else bias.float()
        assert torch.equal(got[empty], want.to(want_dt).expand(int(empty.sum()), cout)), \
            "%s %s: a row with no neighbour is not 0 / the bias" % (name, tag)
    print("forward %-32s worst |got - ref| / bound: conv %.3f  fused bias %.3f" % (tag, *ratios))
    return ratios


@pytest.mark.parametrize("cin,cout,kv,n_out", FWD_SHAPES + ROW_SHAPES)
def test_forward_entry_points_dispatch(shim, cuda, cin, cout, kv, n_out):
    forward_case(shim, cin, cout, kv, n_out, 7 * cin + cout + kv + n_out, H, H)


@pytest.mark.parametrize("dtypes", ["half-f/fp32-w", "fp32-f/half-w"])
@pytest.mark.parametrize("cin,cout,kv,n_out", [(5, 16, 27, 2000), (32, 32, 27, 2000), (64, 128, 27, 2000)])
def test_forward_entry_points_mixed_dtypes(shim, cuda, cin, cout, kv, n_out, dtypes):
    forward_case(shim, cin, cout, kv, n_out, cin + cout + len(dtypes), *DTYPES[dtypes])


@pytest.mark.parametrize("cin,cout", [(32, 64), (64, 128)])
def test_forward_overflow_is_signed_inf(shim, cuda, cin, cout):
    """features up to ~5000 and weights 30x the usual: hundreds of sums leave the fp16 range and must be +-inf
    (what a loss scaler looks for), the rest within the bound"""
    forward_case(shim, cin, cout, 27, 2000, 3 + cin, H, H, fscale=1000.0, wscale=30.0)
    from bevfusion_b200.spconv import ops
    gen = torch.Generator(device=cuda).manual_seed(3 + cin)
    nbr, n_in = _table(27, 2000, gen)
    f, w, _ = _inputs(cin, cout, 27, n_in, gen, H, H, 1000.0, 30.0)
    got = ops.sparse_conv_ext.indice_conv_half(f, w, ops.Rulebook(None, nbr, n_in, 2000, 27), None, 2000, 0, 1)
    ref = conv_nbr(f, w, nbr)
    n_pos, n_neg = int((ref > 7e4).sum()), int((ref < -7e4).sum())
    assert n_pos > 10 and n_neg > 10, "the case does not overflow"
    assert bool((got[ref > 7e4] == float("inf")).all()) and bool((got[ref < -7e4] == -float("inf")).all())
    assert not bool(torch.isnan(got).any())


def test_forward_nan_inf_inputs_as_fp32(shim, cuda):
    """NaN and +-inf features and a NaN filter entry: the half path gives NaN / inf exactly where the fp32 path run
    on the widened tensors does, and finite results where it is finite"""
    from bevfusion_b200.spconv import ops
    gen = torch.Generator(device=cuda).manual_seed(11)
    nbr, n_in = _table(27, 1500, gen)
    f, w, b = _inputs(32, 64, 27, n_in, gen, H, H)
    f[3, 5], f[40, 0], f[77, 31] = float("nan"), float("inf"), -float("inf")
    w[13, 2, 7] = float("nan")
    rb = ops.Rulebook(None, nbr, n_in, 1500, 27)
    pairs, num = rb.pairs()
    for name, args in (("indice_conv_half", ()), ("fused_indice_conv_half", (b,))):
        got = getattr(ops.sparse_conv_ext, name)(f, w, *args, rb, None, 1500, 0, 1)
        want = getattr(ops.sparse_conv_ext, name.replace("half", "fp32"))(
            f.float(), w.float(), *(a.float() for a in args), rb, None, 1500, 0, 1)
        assert got.dtype == H and want.dtype == F
        assert int(torch.isnan(want).sum()) > 0 and int(torch.isnan(want).all(1).sum()) < 1500
        assert torch.equal(torch.isnan(got), torch.isnan(want)), name
        assert torch.equal(torch.isinf(got), torch.isinf(want)) and torch.equal(got[torch.isinf(got)].float(),
                                                                               want[torch.isinf(want)]), name
        fin = torch.isfinite(want)
        assert torch.equal(got[fin], want[fin].half()), name      # same kernel, narrowed once
        assert torch.equal(torch.isnan(getattr(shim, name)(f, w, *args, pairs, num, 1500, 0, 1)), torch.isnan(got))


# ---------------------------------------------------------------------------------------------------- backward
def backward_case(shim, cin, cout, kv, n_out, seed, fdt, wdt, k=0, gscale=2.0 ** -12, fscale=1.0):
    """out_grad = randn * gscale * 2^k (a loss-scaled gradient of a loss near 1)"""
    from bevfusion_b200.spconv import ops
    cuda = torch.device("cuda:0")
    gen = torch.Generator(device=cuda).manual_seed(seed)
    nbr, n_in = _table(kv, n_out, gen)
    rb = ops.Rulebook(None, nbr, n_in, n_out, kv)
    pairs, num = rb.pairs()
    f, w, _ = _inputs(cin, cout, kv, n_in, gen, fdt, wdt, fscale)
    g = (torch.randn(n_out, cout, device=cuda, generator=gen) * gscale * 2.0 ** k).to(_out_dtype(f, w))
    tag = "%d->%d k%d n_out %d %s/%s 2^%d" % (cin, cout, kv, n_out, str(fdt)[6:], str(wdt)[6:], k)
    ext = ops.sparse_conv_ext
    din, dw = ext.indice_conv_backward_half(f, w, g, pairs, num, 0, 1)
    assert din.dtype == f.dtype and dw.dtype == w.dtype, "%s: dtypes %s %s" % (tag, din.dtype, dw.dtype)
    assert dw.shape == w.shape and din.shape == f.shape
    d2 = ext.indice_conv_backward_half(f, w, g, rb, None, 0, 1)
    assert torch.equal(d2[0], din) and torch.equal(d2[1], dw), "%s: Rulebook and pairs differ" % tag
    d3 = shim.indice_conv_backward_half(f, w, g, pairs, num, 0, 1)
    assert torch.equal(d3[0], din) and torch.equal(d3[1], dw), "%s: the compiled module differs" % tag
    ref_din, ref_dw, fed = reference(f, w, g, nbr)
    abs_din, abs_dw, _ = reference(f.abs(), w.abs(), g.abs(), nbr)
    assert bool((din[~fed] == 0).all()), "%s: an input row nothing feeds has a gradient" % tag
    r = (check(din, ref_din, abs_din, "input grad " + tag), check(dw, ref_dw, abs_dw, "filter grad " + tag))
    print("backward %-38s worst |got - ref| / bound: dIn %.3f  dW %.3f" % (tag, *r))
    return ref_dw, dw


@pytest.mark.parametrize("k", [0, 8, 16])
@pytest.mark.parametrize("cin,cout,kv,n_out", BWD_SHAPES)
def test_backward_entry_points_dispatch(shim, cuda, cin, cout, kv, n_out, k):
    backward_case(shim, cin, cout, kv, n_out, 5 * cin + cout + kv + k, H, H, k)


@pytest.mark.parametrize("n_out", [1, 31, 32, 33, 2047, 2049])
def test_backward_entry_points_row_counts(shim, cuda, n_out):
    backward_case(shim, 32, 64, 27, n_out, n_out, H, H, 8)


@pytest.mark.parametrize("dtypes", ["half-f/fp32-w", "fp32-f/half-w"])
@pytest.mark.parametrize("cin,cout", [(5, 16), (32, 64), (128, 128)])
def test_backward_entry_points_mixed_dtypes(shim, cuda, cin, cout, dtypes):
    backward_case(shim, cin, cout, 27, 3000, cin * 3 + cout, *DTYPES[dtypes], k=8)


def test_backward_filter_grad_overflow_is_inf(shim, cuda):
    """loss scale 2^16 on features around 32: some filter-gradient sums pass 65520 and must be +-inf in fp16 (the
    loss scaler then halves the scale); with fp32 filters the same sums stay finite"""
    ref_dw, dw = backward_case(shim, 32, 64, 27, 3000, 99, H, H, k=16, fscale=32.0)
    assert int((ref_dw.abs() > 7e4).sum()) > 10, "the case does not overflow"
    assert bool(torch.isinf(dw[ref_dw.abs() > 7e4]).all())
    ref_dw32, dw32 = backward_case(shim, 32, 64, 27, 3000, 99, H, F, k=16, fscale=32.0)
    assert bool(torch.isfinite(dw32).all())


# ---------------------------------------------------------------------------------------------------- real rulebooks
GEOMS = {"subm_k3": ([3, 3, 3], [1, 1, 1], [1, 1, 1], True),
         "conv_k3s2p1": ([3, 3, 3], [2, 2, 2], [1, 1, 1], False),
         "conv_k3s2p110": ([3, 3, 3], [2, 2, 2], [1, 1, 0], False),
         "conv_k113s112": ([1, 1, 3], [1, 1, 2], [0, 0, 0], False)}
CHANNELS = [(5, 16), (16, 16), (32, 64), (64, 128), (128, 128)]


@pytest.mark.parametrize("cin,cout", CHANNELS)
@pytest.mark.parametrize("geom", list(GEOMS))
def test_entry_points_on_rulebooks(shim, cuda, geom, cin, cout):
    from bevfusion_b200.spconv import ops
    ks, st, pd, subm = GEOMS[geom]
    shape, B, n = [40, 36, 11], 2, 5000
    rng = np.random.default_rng(cin + cout)
    flat = rng.choice(B * shape[0] * shape[1] * shape[2], size=n, replace=False)
    idx = np.stack([flat // (shape[0] * shape[1] * shape[2]), (flat // (shape[1] * shape[2])) % shape[0],
                    (flat // shape[2]) % shape[1], flat % shape[2]], 1).astype(np.int32)
    idx = torch.from_numpy(idx).to(cuda)
    outids, pairs, num = ops.get_indice_pairs(idx, B, shape, ks, st, pd, 1, 0, subm)
    rb, _ = ops.get_rulebook(idx, B, shape, ks, st, pd, 1, 0, subm)
    n_out, kv = outids.shape[0], rb.kernel_volume
    gen = torch.Generator(device=cuda).manual_seed(cin * cout)
    f, w, b = _inputs(cin, cout, kv, n, gen, H, H)
    w = w.reshape(*ks, cin, cout)
    ext = ops.sparse_conv_ext
    got = ext.fused_indice_conv_half(f, w, b, pairs, num, n_out, 0, int(subm))
    assert torch.equal(ext.fused_indice_conv_half(f, w, b, rb, None, n_out, 0, int(subm)), got)
    assert torch.equal(shim.fused_indice_conv_half(f, w, b, pairs, num, n_out, 0, int(subm)), got)
    ref = conv_nbr(f, w, rb.nbr) + b.double()
    absref = conv_nbr(f.abs(), w.abs(), rb.nbr) + b.double().abs()
    r_fwd = check(got, ref, absref, "forward %s %d->%d" % (geom, cin, cout))
    g = (torch.randn(n_out, cout, device=cuda, generator=gen) * 2.0 ** -4).half()
    din, dw = ext.indice_conv_backward_half(f, w, g, pairs, num, 0, int(subm))
    d2 = ext.indice_conv_backward_half(f, w, g, rb, None, 0, int(subm))
    d3 = shim.indice_conv_backward_half(f, w, g, pairs, num, 0, int(subm))
    assert all(torch.equal(a, c) for a, c in zip((din, dw), d2)) and all(torch.equal(a, c) for a, c in zip((din, dw), d3))
    ref_din, ref_dw, _ = reference(f, w.reshape(kv, cin, cout), g, rb.nbr)
    abs_din, abs_dw, _ = reference(f.abs(), w.abs().reshape(kv, cin, cout), g.abs(), rb.nbr)
    r_din = check(din, ref_din, abs_din, "input grad %s" % geom)
    r_dw = check(dw.reshape(kv, cin, cout), ref_dw, abs_dw, "filter grad %s" % geom)
    print("%-14s %3d -> %3d  n_in %d n_out %d  worst ratio: forward %.3f  dIn %.3f  dW %.3f" % (
        geom, cin, cout, n, n_out, r_fwd, r_din, r_dw))


# ---------------------------------------------------------------------------------------------------- modules
def _sparse_input(cuda, cin, n=3000, shape=(30, 28, 9), B=2, seed=0):
    from bevfusion_b200 import spconv
    rng = np.random.default_rng(seed)
    X, Y, Z = shape
    flat = rng.choice(B * X * Y * Z, size=n, replace=False)
    idx = np.stack([flat // (X * Y * Z), (flat // (Y * Z)) % X, (flat // Z) % Y, flat % Z], 1).astype(np.int32)
    f = torch.from_numpy(rng.standard_normal((n, cin)).astype(np.float32)).to(cuda).half()
    return lambda: spconv.SparseConvTensor(f, torch.from_numpy(idx).to(cuda), list(shape), B)


def _random_bn(c, seed, cuda):
    bn = torch.nn.BatchNorm1d(c, eps=1e-3).to(cuda).eval()
    gen = torch.Generator().manual_seed(seed)
    bn.running_mean.copy_(torch.randn(c, generator=gen) * 0.3)
    bn.running_var.copy_(torch.rand(c, generator=gen) + 0.5)
    bn.weight.data.copy_(torch.rand(c, generator=gen) + 0.5)
    bn.bias.data.copy_(torch.randn(c, generator=gen) * 0.3)
    return bn


def _conv_ref(mod, x_features, nbr):
    """float64 conv of the module on (half) input rows, and its |.| twin"""
    w = mod.weight.detach()
    ref, absref = conv_nbr(x_features, w, nbr), conv_nbr(x_features.abs(), w.abs(), nbr)
    if mod.bias is not None:
        ref, absref = ref + mod.bias.detach().double(), absref + mod.bias.detach().double().abs()
    return ref, absref


@pytest.mark.parametrize("weights", ["half", "fp32"])
@pytest.mark.parametrize("kind", ["SubMConv3d", "SparseConv3d"])
def test_conv_module_four_modes(cuda, kind, weights):
    """grad enabled, no_grad, fused BN + ReLU: one conv, its output narrowed once (the unfused BN + ReLU after it run
    in fp32 and narrow once more); all against float64"""
    from bevfusion_b200 import spconv
    from bevfusion_b200.sparse_block import bn_scale_shift
    torch.manual_seed(1)
    cin, cout = 16, 32
    conv = (spconv.SubMConv3d(cin, cout, 3, padding=1, bias=True) if kind == "SubMConv3d"
            else spconv.SparseConv3d(cin, cout, 3, stride=2, padding=1, bias=True)).to(cuda)
    if weights == "half":
        conv.half()
    bn = _random_bn(cout, 2, cuda)                  # BN stays fp32 (mmcv's patch_norm_fp32)
    s, t = bn_scale_shift(bn)
    make = _sparse_input(cuda, cin)
    y_grad = conv(make())                           # grad enabled: the autograd function
    with torch.no_grad():
        y_nograd = conv(make())
        y_fused = conv(make(), scale=s, shift=t, relu=True)
    nbr = conv._rulebook(make())[0].nbr
    ref, absref = _conv_ref(conv, make().features, nbr)
    b64 = conv.bias.detach().double()
    r = []
    # grad enabled: the conv is narrowed, then `+= bias` narrows again (the reference's order): two roundings
    assert y_grad.features.dtype == H
    two = ulp(ref - b64, H) + C_BF16X3 * absref + ulp(ref, H)
    r.append(float(((y_grad.features.detach().double() - ref).abs() / two).max()))
    assert r[-1] <= 1.0, "%s %s grad: %.3f of two roundings" % (kind, weights, r[-1])
    # no_grad: the bias folds into the epilogue, one rounding
    assert y_nograd.features.dtype == H
    r.append(check(y_nograd.features, ref, absref, "%s %s no_grad" % (kind, weights)))
    # unfused BN + ReLU in fp32 on the narrowed conv, narrowed again: two roundings, the first scaled by |s|
    s64, t64 = s.double(), t.double()
    z64 = (ref * s64 + t64).clamp_min(0)
    z = torch.relu(bn(y_nograd.features.float())).half()
    err = (z.double() - z64).abs()
    two = s64.abs() * (ulp(ref, H) + C_BF16X3 * absref) + ulp(z64, H)
    r.append(float((err / two).max()))
    assert r[-1] <= 1.0, "unfused conv + BN + ReLU: %.3f of two roundings" % r[-1]
    assert y_fused.features.dtype == H
    r.append(check(y_fused.features, z64, absref * s64.abs() + t64.abs(), "%s %s fused" % (kind, weights)))
    print("%-12s weights %-4s worst ratio: grad %.3f  no_grad %.3f  unfused BN+ReLU %.3f  fused %.3f" % (
        kind, weights, *r))


@pytest.mark.parametrize("weights", ["half", "fp32"])
def test_basic_block_fused_residual(cuda, weights):
    """SparseBasicBlock.forward_fused on half features: each conv's epilogue (BN, residual, ReLU) narrowed once,
    checked on the conv's own half input; the unfused forward agrees within the roundings it adds"""
    from bevfusion_b200.sparse_block import SparseBasicBlock, bn_scale_shift
    torch.manual_seed(3)
    c = 32
    blk = SparseBasicBlock(c, c, norm_cfg=dict(type="BN1d", eps=1e-3), conv_cfg=dict(type="SubMConv3d")).to(cuda)
    blk.bn1 = _random_bn(c, 4, cuda)
    blk.bn2 = _random_bn(c, 5, cuda)
    blk.eval()
    if weights == "half":
        blk.conv1.half()
        blk.conv2.half()
    make = _sparse_input(cuda, c, seed=6)
    with torch.no_grad():
        x = make()
        out = blk.forward_fused(x)
        s1, t1 = bn_scale_shift(blk.norm1)
        s2, t2 = bn_scale_shift(blk.norm2)
        mid = blk.conv1(x, scale=s1, shift=t1, relu=True)
    assert out.features.dtype == H and mid.features.dtype == H
    nbr = blk.conv1._rulebook(x)[0].nbr
    ref1, abs1 = _conv_ref(blk.conv1, x.features, nbr)
    r1 = check(mid.features, epilogue(ref1, s1, t1, None, True), abs1 * s1.double().abs() + t1.double().abs(),
               "block conv1 " + weights)
    ref2, abs2 = _conv_ref(blk.conv2, mid.features, nbr)
    r2 = check(out.features, epilogue(ref2, s2, t2, x.features, True),
               abs2 * s2.double().abs() + t2.double().abs() + x.features.double().abs(), "block conv2 + residual " + weights)
    print("SparseBasicBlock weights %-4s fused worst ratio: conv1 %.3f  conv2 + residual %.3f" % (weights, r1, r2))


def test_dense_keeps_half(cuda):
    """SparseConvTensor.dense() returns the features' dtype, exactly the scattered rows, and a gradient of that
    dtype (the reference's scatter_nd allocates in updates.dtype)"""
    make = _sparse_input(cuda, 16, n=500, shape=(10, 9, 5), seed=8)
    x = make()
    f = x.features.clone().requires_grad_(True)
    x.features = f
    d = x.dense()
    assert d.dtype == H and tuple(d.shape) == (2, 16, 10, 9, 5)
    li = x.indices.long()
    want = torch.zeros(2, 10, 9, 5, 16, dtype=H, device=cuda)
    want[li[:, 0], li[:, 1], li[:, 2], li[:, 3]] = f.detach()
    assert torch.equal(d, want.permute(0, 4, 1, 2, 3))
    assert x.dense(channels_first=False).dtype == H
    g = torch.randn(d.shape, device=cuda).half()
    (d.float() * g.float()).sum().backward()
    assert f.grad.dtype == H
    assert torch.equal(f.grad, g[li[:, 0], :, li[:, 1], li[:, 2], li[:, 3]])


# ---------------------------------------------------------------------------------------------------- encoder
def _voxelnet(cuda, shape, seed=0):
    from bevfusion_b200.sparse_encoder import SparseEncoder
    torch.manual_seed(seed)
    m = SparseEncoder(in_channels=5, sparse_shape=shape, output_channels=128,
                      encoder_channels=((16, 16, 32), (32, 32, 64), (64, 64, 128), (128, 128)),
                      encoder_paddings=((0, 0, 1), (0, 0, 1), (0, 0, (1, 1, 0)), (0, 0)), block_type="basicblock")
    g = torch.Generator().manual_seed(seed)
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm1d):
            n = mod.num_features
            mod.running_mean.copy_(torch.randn(n, generator=g) * 0.1)
            mod.running_var.copy_(torch.rand(n, generator=g) + 0.5)
            mod.weight.data.copy_(torch.rand(n, generator=g) * 0.4 + 0.8)
            mod.bias.data.copy_(torch.randn(n, generator=g) * 0.1)
    return m.to(cuda)


def _voxels(cuda, shape, n, seed, B=1):
    rng = np.random.default_rng(seed)
    X, Y, Z = shape
    flat = np.sort(rng.choice(B * X * Y * Z, size=n, replace=False))
    idx = np.stack([flat // (X * Y * Z), (flat // (Y * Z)) % X, (flat // Z) % Y, flat % Z], 1).astype(np.int32)
    feats = torch.from_numpy(rng.standard_normal((n, 5)).astype(np.float32)).to(cuda)
    return feats, torch.from_numpy(idx).to(cuda)


def _halve_convs(m):
    """the convs in half, BatchNorm in fp32: mmcv's wrap_fp16_model (model.half() + patch_norm_fp32)"""
    for conv in m._conv_sequence():
        conv.half()
    return m


def _conv_hooks(m, checks):
    """forward hooks on every conv: its output against float64 on its own (half) input rows and epilogue"""
    def hook(mod, args, kwargs, out):
        x = args[0]
        nbr = mod._rulebook(x)[0].nbr
        ref, absref = _conv_ref(mod, x.features, nbr)
        scale, shift, res, relu = (kwargs.get(k) for k in ("scale", "shift", "residual", "relu"))
        s = torch.ones_like(ref[0]) if scale is None else scale.double()
        # the fp32 epilogue errs relative to |acc * s|, |shift| and |residual|
        absepi = epilogue(absref * s.abs(), None, None if shift is None else shift.abs(), None if res is None else res.abs())
        r = check(out.features.detach(), epilogue(ref, scale, shift, res, bool(relu)), absepi,
                  "conv %d (%d -> %d)" % (len(checks), mod.in_channels, mod.out_channels))
        checks.append((mod.in_channels, mod.out_channels, int(nbr.shape[1]), r, out.features.dtype))
    return [mod.register_forward_hook(hook, with_kwargs=True) for mod in m._conv_sequence()]


@pytest.mark.parametrize("weights", ["half", "fp32"])
def test_encoder_eval_half(cuda, weights):
    """eval mode, half voxel features: the fused per-conv path (each conv checked on its own input), output in half
    and exactly the scatter of conv_out's rows; fp32 input still takes the native plan, unchanged by the half run"""
    from bevfusion_b200 import encoder_plan
    shape = [160, 160, 41]
    m = _voxelnet(cuda, shape).eval()
    feats, coors = _voxels(cuda, shape, 12000, seed=1)
    calls = []
    orig = encoder_plan.EncoderPlan.forward

    def counting(self, *a, **k):
        calls.append(1)
        return orig(self, *a, **k)

    encoder_plan.EncoderPlan.forward = counting
    try:
        with torch.no_grad():
            if weights == "half":
                ref32 = None
                _halve_convs(m)
            else:
                ref32 = m(feats, coors, 1)
                assert len(calls) == 1 and ref32.dtype == F
            checks = []
            hooks = _conv_hooks(m, checks)
            try:
                got = m(feats.half(), coors, 1)
            finally:
                for h in hooks:
                    h.remove()
            if ref32 is not None:
                assert torch.equal(m(feats, coors, 1), ref32), "the half run changed the fp32 result"
                assert len(calls) == 2
            else:
                assert not calls, "half weights on the native plan"
    finally:
        encoder_plan.EncoderPlan.forward = orig
    assert got.dtype == H and len(checks) == 21
    assert all(dt == H for *_, dt in checks)
    for cin, cout, n_out, r, _ in checks:
        print("  eval %-4s conv %3d -> %3d  n_out %6d  worst ratio %.3f" % (weights, cin, cout, n_out, r))
    print("eval, weights %s: worst ratio over 21 convs %.3f" % (weights, max(c[3] for c in checks)))


@pytest.mark.parametrize("weights", ["half", "fp32"])
def test_encoder_training_step_half(cuda, weights):
    """forward + backward with half voxel features: every filter gradient against float64 on the conv's own input
    rows and out-grad (one rounding to the weight's dtype); the output and gradients end to end against the float64
    twin, with the device's ReLU masks -- loose, printed"""
    shape = [160, 160, 41]
    m = _voxelnet(cuda, shape, seed=2)
    feats, coors = _voxels(cuda, shape, 12000, seed=3)
    if weights == "half":
        _halve_convs(m)
    twin = copy.deepcopy(m).double().train()          # on the weights as the device has them
    m.train()
    saved = []

    def hook(mod, args, out):
        saved.append((mod, args[0].features.detach(), mod._rulebook(args[0])[0].nbr, out.features))
        out.features.retain_grad()

    hooks = [mod.register_forward_hook(hook) for mod in m._conv_sequence()]
    masks = []
    hooks += [mod.register_forward_hook(lambda mod, inp, out: masks.append(out.detach() > 0))
              for mod in m.modules() if isinstance(mod, torch.nn.ReLU)]
    x = feats.half().requires_grad_(True)
    try:
        out = m(x, coors, 1)
    finally:
        for h in hooks:
            h.remove()
    assert out.dtype == H and len(saved) == 21 and len(masks) == 21
    R = torch.randn(out.shape, device=cuda, generator=torch.Generator(device=cuda).manual_seed(1))
    (out.float() * R).sum().backward()
    assert x.grad.dtype == H
    assert all(bool(torch.isfinite(o.grad).all()) for *_, o in saved), "the half gradients overflowed"
    worst = 0.0
    for i, (mod, f, nbr, o) in enumerate(saved):
        w = mod.weight
        assert w.grad.dtype == w.dtype
        g = o.grad
        kv = nbr.shape[0]
        _, absdw, _ = reference(f.abs(), w.detach().abs().reshape(kv, mod.in_channels, mod.out_channels), g.abs(), nbr)
        _, refdw, _ = reference(f, w.detach().reshape(kv, mod.in_channels, mod.out_channels), g, nbr)
        r = check(w.grad.reshape(kv, mod.in_channels, mod.out_channels), refdw, absdw,
                  "filter grad of conv %d (%d -> %d)" % (i, mod.in_channels, mod.out_channels))
        worst = max(worst, r)
        print("  train %-4s conv %2d %3d -> %3d  n_out %6d  dW worst ratio %.3f" % (
            weights, i, mod.in_channels, mod.out_channels, nbr.shape[1], r))
    print("training step, weights %s: worst filter-gradient ratio over 21 convs %.3f" % (weights, worst))
    # end to end: the float64 twin on the half-rounded features, with the device's ReLU masks
    x64 = x.detach().double().requires_grad_(True)
    flips = []
    out64 = _twin_forward(twin, x64, coors, 1, shape, masks, flips)
    (out64 * R.double()).sum().backward()
    rel = lambda a, b: float((a.double() - b).norm() / b.norm().clamp_min(1e-300))
    e_out, e_in = rel(out.detach(), out64.detach()), rel(x.grad, x64.grad)
    p64 = dict(twin.named_parameters())
    e_conv = max(rel(mod.weight.grad, p64[n + ".weight"].grad) for n, mod in m.named_modules()
                 if mod in [s[0] for s in saved])
    print("training step, weights %s, end to end rel L2: output %.2e  input grad %.2e  worst conv grad %.2e" % (
        weights, e_out, e_in, e_conv))
    # about 10x what an H100 80GB HBM3 (700 W) measured with either weight dtype: output 3.0e-3, input gradient
    # 1.3e-3, worst conv gradient 3.0e-3 -- the fp16 roundings of 21 layers, not a kernel error (the per-layer checks)
    assert e_out <= 3e-2 and e_in <= 1.5e-2 and e_conv <= 3e-2
