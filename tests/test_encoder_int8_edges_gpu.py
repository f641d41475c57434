"""GPU tests of the INT8 plan at the edges of its contract (include/bevfusion_b200.h, DESIGN.md 4.25): every case of
encoder_int8_cases must give a dense() bit-equal to the exact oracle (encoder_int8_oracle.run_chain) and the expected
status -- the instances no other test launches, saturation (scales a quarter too small, calibrated on another seed,
r_out = +inf, fl(v r_out) overflowing), rounding ties of the u8 and weight quantizers, accumulators past 2^24 on
wgmma, the last conv's half overflowing, one- and two-conv chains, NaN / +-inf features on valid rows, and level row
counts on both sides of a second persistent tile.  Then the module: calibrate_int8 over several batches (one of
them empty), a dead conv, fp32 features, out= as a channel slice, and an empty sample in the batch."""
import numpy as np
import pytest
import torch

from bevfusion_b200.encoder_plan import _chain_of
from bevfusion_b200.spconv.ops import PREC_INT8
from encoder_int8_cases import CASES, TILE_CASES
from test_encoder_fp16_gpu import _coors, _randomise_bn, voxelnet
from test_encoder_int8_gpu import _check_exact, _grid, _module_oracle

pytestmark = pytest.mark.gpu


def _run_case(cuda, build):
    raw, rows = build(cuda)
    status = _check_exact(raw)
    if rows is not None:
        assert status[1:] == rows


@pytest.mark.parametrize("case", list(CASES))
def test_edge_case_bit_equal(cuda, case):
    _run_case(cuda, CASES[case][1])


@pytest.mark.parametrize("case", list(TILE_CASES))
def test_persistent_tiles_bit_equal(cuda, case):
    _run_case(cuda, TILE_CASES[case])


# ---- the module ------------------------------------------------------------------------------------------------
SHAPE = [48, 48, 41]


def _module(cuda, seed):
    torch.manual_seed(seed)
    m = _randomise_bn(voxelnet(SHAPE), seed)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        w = m.conv_input[0].weight
        w.copy_(_grid(w, 2.0 ** -8, 1.0, g) * 0.25)
    return m.to(cuda).eval(), g


def _batch(cuda, g, B, n, seed, samples=None):
    """exact-grid fp16 features of n voxels in each of `samples` (default all B)"""
    samples = list(range(B)) if samples is None else samples
    coors = _coors(SHAPE, len(samples), n, seed)
    coors[:, 0] = np.asarray(samples)[coors[:, 0]]
    f = _grid(torch.empty(coors.shape[0], 5), 2.0 ** -4, 8.0, g).half()
    return f, coors, B


def _forward(m, cuda, f, coors, B, **kw):
    with torch.no_grad():
        return m(f.to(cuda), torch.from_numpy(coors).to(cuda), B, precision=PREC_INT8, **kw)


def _assert_oracle(m, cuda, f, coors, B):
    out = _forward(m, cuda, f, coors, B)
    want, _, _ = _module_oracle(m, f, coors, B, SHAPE, exact=True)
    got = out.double().cpu()
    assert got.shape == want.shape
    assert torch.equal(got, want), "%d cells differ" % int((got != want).sum())
    return out


def test_calibration_over_batches_is_the_max_of_single_batches(cuda):
    """fl(amax / 255) is monotone in amax, so the scales of several batches are the elementwise max of each batch's
    own; a batch with no voxels adds nothing (alone it leaves every conv dead: scale 1)"""
    m, g = _module(cuda, 3)
    batches = [_batch(cuda, g, 2, 900, 4), _batch(cuda, g, 1, 0, 5), _batch(cuda, g, 3, 600, 6)]
    dev = [(f.float().to(cuda), torch.from_numpy(c).to(cuda), B) for f, c, B in batches]
    single = [m.calibrate_int8([b]) for b in dev]
    assert torch.equal(single[1], torch.ones_like(single[1]))
    every = m.calibrate_int8(dev)
    assert torch.equal(every, torch.maximum(single[0], single[2]))
    assert torch.equal(m.int8_scales(), every)


def test_dead_conv_scale_one_and_forward_exact(cuda):
    m, g = _module(cuda, 7)
    dead = 4                                            # encoder_layers[0][1].conv2: a residual conv
    with torch.no_grad():
        _chain_of(m)[dead][1].bias.fill_(-1e4)
    f, coors, B = _batch(cuda, g, 2, 1500, 8)
    scales = m.calibrate_int8([(f.float().to(cuda), torch.from_numpy(coors).to(cuda), B)])
    assert float(scales[dead]) == 1.0 and bool((scales[:dead] != 1.0).all())
    _assert_oracle(m, cuda, f, coors, B)


def test_fp32_features_equal_their_fp16_rounding(cuda):
    m, g = _module(cuda, 11)
    f, coors, B = _batch(cuda, g, 2, 1500, 12)
    f32 = f.float() + torch.randn(f.shape, generator=g) * 2.0 ** -9           # not on the fp16 grid
    m.calibrate_int8([(f32.to(cuda), torch.from_numpy(coors).to(cuda), B)])
    a = _forward(m, cuda, f32, coors, B)
    b = _forward(m, cuda, f32.half(), coors, B)
    assert torch.equal(a, b)


def test_out_channel_slice_of_a_wider_tensor(cuda):
    m, g = _module(cuda, 13)
    f, coors, B = _batch(cuda, g, 2, 1500, 14)
    m.calibrate_int8([(f.float().to(cuda), torch.from_numpy(coors).to(cuda), B)])
    want = _forward(m, cuda, f, coors, B)
    C = want.shape[1]
    wide = torch.full((B, 40 + C + 24, want.shape[2], want.shape[3]), 3.0, dtype=torch.float16, device=cuda)
    got = _forward(m, cuda, f, coors, B, out=wide[:, 40:40 + C])
    torch.cuda.synchronize()
    assert got.data_ptr() == wide[:, 40:40 + C].data_ptr()
    assert torch.equal(wide[:, 40:40 + C], want)
    assert bool((wide[:, :40] == 3.0).all()) and bool((wide[:, 40 + C:] == 3.0).all())


def test_empty_middle_sample(cuda):
    m, g = _module(cuda, 17)
    f, coors, B = _batch(cuda, g, 3, 1200, 18, samples=[0, 2])
    m.calibrate_int8([(f.float().to(cuda), torch.from_numpy(coors).to(cuda), B)])
    out = _assert_oracle(m, cuda, f, coors, B)
    assert bool((out[1] == 0).all()) and bool((out[0] != 0).any()) and bool((out[2] != 0).any())
