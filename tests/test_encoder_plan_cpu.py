"""Host logic of the native SparseEncoder plan (bevb200_encoder_*): chain extraction, level shapes, row
caps and workspace arithmetic.  No device is touched."""
import ctypes

import pytest

from bevfusion_b200 import _C
from bevfusion_b200.encoder_plan import EncoderPlan, _chain_of, supported
from bevfusion_b200.sparse_encoder import SparseEncoder, voxelnet_0p075_encoder


def test_chain_matches_the_reference_encoder_structure():
    enc = voxelnet_0p075_encoder()
    chain = _chain_of(enc)
    assert len(chain) == 21                                   # 17 SubM + 4 strided (sparse_encoder.py:113-124)
    subm = [c[0].subm for c in chain]
    assert subm.count(False) == 4 and [i for i, s in enumerate(subm) if not s] == [5, 10, 15, 20]
    # SparseBasicBlock: conv2 adds the block input = the output of the conv before conv1 (sparse_block.py:94-110)
    res = [c[3] for c in chain]
    assert res[:6] == [-1, -1, 0, -1, 2, -1] and res[6:11] == [-1, 5, -1, 7, -1]
    assert all(c[2] for c in chain)                           # every conv is followed by BN + ReLU
    assert supported(enc)


def test_plan_levels_caps_and_workspace():
    enc = voxelnet_0p075_encoder()
    plan = EncoderPlan(enc)
    assert plan.n_levels == 5
    assert plan.out_shape == [180, 180, 2] and plan.out_channels == 128   # -> [B, 256, 180, 180]
    caps = plan.level_caps(160000, 1)
    # k3 s2: <= 8 outputs per input, <= 1 per site; conv_out k(1,1,3) s(1,1,2): <= 2 per input
    assert caps == [160000, 1280000, min(8 * 1280000, 360 * 360 * 11), 180 * 180 * 5, 180 * 180 * 2]
    tight = plan.level_caps(160000, 1, [0, 400000, 250000, 90000, 0])
    assert tight == [160000, 400000, 250000, 90000, 180 * 180 * 2]
    L = _C.lib()
    full = L.bevb200_encoder_workspace_bytes(plan._h, 160000, 1, None)
    small = L.bevb200_encoder_workspace_bytes(plan._h, 160000, 1, plan._caps_arg([0, 400000, 250000, 90000, 0]))
    assert 0 < small < full
    # the level-0 bitmap alone: 1440*1440*41 sites, 8 bytes per 32 sites
    assert small > 1440 * 1440 * 41 // 32 * 8
    assert L.bevb200_encoder_param_bytes(plan._h) >= sum(
        L.bevb200_spconv_split_weight_bytes(c[0].in_channels, c[0].out_channels, 27 if i < 20 else 3)
        for i, c in enumerate(_chain_of(enc)))


def test_create_rejects_bad_chains():
    from bevfusion_b200.encoder_plan import _ConvDesc
    L = _C.lib()

    def make(descs):
        arr = (_ConvDesc * len(descs))()
        for a, (cin, cout, subm, res) in zip(arr, descs):
            a.c_in, a.c_out, a.subm, a.relu, a.residual_from = cin, cout, subm, 1, res
            for k in range(3):
                a.ksize[k], a.stride[k], a.padding[k], a.dilation[k] = 3, 2 - subm, 1, 1
        h = ctypes.c_void_p()
        rc = L.bevb200_encoder_create(5, (ctypes.c_int32 * 3)(64, 64, 9), arr, len(descs), ctypes.byref(h))
        if rc == 0:
            L.bevb200_encoder_destroy(h)
        return rc

    assert make([(5, 16, 1, -1), (16, 16, 1, -1)]) == 0
    assert make([(5, 16, 1, -1), (32, 32, 1, -1)]) != 0          # c_in does not chain
    assert make([(5, 24, 1, -1)]) != 0                            # no tensor-core form for 24 channels
    assert make([(5, 16, 1, -1), (16, 32, 0, 0)]) != 0            # residual across levels / widths
    assert make([(5, 16, 1, 0)]) != 0                             # residual_from must be earlier
    # a level's two split images alternate: a residual from two convs back is the furthest that survives
    assert make([(5, 16, 1, -1), (16, 16, 1, -1), (16, 16, 1, 0)]) == 0
    assert make([(5, 16, 1, -1), (16, 16, 1, -1), (16, 16, 1, -1), (16, 16, 1, 0)]) != 0
    assert b"two previous convs" in L.bevb200_last_error()


def test_bn_fold_follows_train_mode_statistics():
    """A train-mode BN forward moves running_mean / running_var in place; the cached fold (bn_scale_shift, and the
    caches keyed on bn_fold_key) must see it even though no optimizer step touched a parameter."""
    import torch
    from bevfusion_b200.sparse_block import _bn_scale_shift, bn_fold_key, bn_scale_shift
    g = torch.Generator().manual_seed(0)
    bn = torch.nn.BatchNorm1d(16, eps=1e-3, momentum=0.01).eval()
    s0, t0 = (v.clone() for v in bn_scale_shift(bn))
    key = bn_fold_key(bn)
    bn.train()
    with torch.no_grad():
        bn(torch.randn(256, 16, generator=g) * 3.0 + 2.0)
    bn.eval()
    assert bn_fold_key(bn) != key
    s1, t1 = bn_scale_shift(bn)
    es, et = _bn_scale_shift(bn)
    assert torch.equal(s1, es) and torch.equal(t1, et)
    assert not torch.equal(s1, s0) and not torch.equal(t1, t0)
    assert bn_scale_shift(bn)[0] is s1                             # unchanged statistics: the cached fold


def test_unsupported_orders_fall_back():
    enc = SparseEncoder(5, [64, 64, 9], order=("norm", "act", "conv"))
    assert not supported(enc)
