"""CPU tests of the SparseEncoder's INT8 precision: the constant, the INT8 plan's size queries against their layout
formula, the refusals that need no device (training entries first, chains without ReLU, the wrong packing call), the
oracle's quantizers against torch on ties, zero, saturation, +inf and NaN, and a state_dict untouched by the scales."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from bevfusion_b200 import _C
from bevfusion_b200.sparse_encoder import voxelnet_0p075_encoder
from bevfusion_b200.spconv import ops
from encoder_int8_oracle import quant_u8, quant_weight
from test_encoder_fp16_cpu import CHAIN, _align, _create, _sizes

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "bevfusion_b200.h")
BEVB200_EINVAL = -1


def test_precision_constant():
    text = open(HEADER).read()
    assert int(re.search(r"#define BEVB200_PREC_INT8 (\d+)", text).group(1)) == ops.PREC_INT8 == 6
    assert sorted(ops._PREC_NAMES) == ["bf16x3", "fp32", "tf32", "tf32x3"]


def test_set_precision_int8_round_trip():
    L = _C.lib()
    h = _create()
    try:
        before = _sizes(h)
        for p in (ops.PREC_FP32, ops.PREC_TF32X3, ops.PREC_TF32, 5, 7, -1):
            assert L.bevb200_encoder_set_precision(h, p) == BEVB200_EINVAL
        assert _sizes(h) == before and L.bevb200_encoder_precision(h) == ops.PREC_BF16X3
        assert L.bevb200_encoder_set_precision(None, ops.PREC_INT8) == BEVB200_EINVAL
        # back and forth: the layout follows the precision
        for p in (ops.PREC_INT8, ops.PREC_FP16, ops.PREC_BF16X3):
            assert L.bevb200_encoder_set_precision(h, p) == 0 and L.bevb200_encoder_precision(h) == p
        assert _sizes(h) == before
    finally:
        L.bevb200_encoder_destroy(h)


def test_int8_needs_relu_everywhere():
    from test_encoder_fp16_cpu import _Conv
    L = _C.lib()
    descs = (_Conv * 2)()
    for d, (ci, co, relu) in zip(descs, [(5, 16, 1), (16, 32, 0)]):
        d.c_in, d.c_out, d.subm, d.relu, d.residual_from = ci, co, 1, relu, -1
        for k in range(3):
            d.ksize[k], d.stride[k], d.padding[k], d.dilation[k] = 3, 1, 1, 1
    h = ctypes.c_void_p()
    assert L.bevb200_encoder_create(5, (ctypes.c_int32 * 3)(16, 16, 9), descs, 2, ctypes.byref(h)) == 0
    try:
        assert L.bevb200_encoder_set_precision(h, ops.PREC_INT8) == BEVB200_EINVAL
        assert "ReLU" in L.bevb200_last_error().decode()
        assert L.bevb200_encoder_precision(h) == ops.PREC_BF16X3
    finally:
        L.bevb200_encoder_destroy(h)


def test_int8_sizes_match_layout():
    """param_bytes: per conv the weight image (conv 0: fp16, K blocks of 64 channels; the others: s8, K blocks of
    128), a, shift and [r_out, s_res, s_w], each 256-byte aligned.  workspace_bytes: the FP16 plan's, with each
    level's two images at the INT8 row width (level 0: the fp16 features or the u8 outputs, whichever is wider; the
    last conv excluded) and one fp16 image of the last conv."""
    L = _C.lib()
    h8, h16 = _create(ops.PREC_INT8), _create(ops.PREC_FP16)
    try:
        want = 0
        for i, (ci, co, _, _, ks) in enumerate(CHAIN):
            ce = max(16, 1 << (ci - 1).bit_length())
            kv = ks[0] * ks[1] * ks[2]
            per_block = 64 if i == 0 else 128
            want += _align((kv * ce + per_block - 1) // per_block * co * 128) + 2 * _align(co * 4) + _align((2 + co) * 4)
        assert L.bevb200_encoder_param_bytes(h8) == want
        n, B = 5000, 2
        caps = (ctypes.c_int32 * 4)()
        assert L.bevb200_encoder_level_caps(h8, n, B, None, caps) == 0
        levels = [0, 1, 1, 1, 2, 3]
        c_max = [16, 32, 64, 128]
        rb8 = [16 * 2, 0, 0, 0]
        for l, (_, co, *_r) in zip(levels[:-1], CHAIN[:-1]):
            rb8[l] = max(rb8[l], co)
        diff = sum(2 * (_align(caps[l] * rb8[l]) - _align(caps[l] * c_max[l] * 2)) for l in range(4))
        diff += _align(caps[3] * CHAIN[-1][1] * 2)
        assert (L.bevb200_encoder_workspace_bytes(h8, n, B, None) - L.bevb200_encoder_workspace_bytes(h16, n, B, None)
                == diff)
        # no training layout
        assert L.bevb200_encoder_train_state_bytes(h8, n, B, None) == 0
        assert L.bevb200_encoder_backward_workspace_bytes(h8, n, B, None) == 0
    finally:
        L.bevb200_encoder_destroy(h8)
        L.bevb200_encoder_destroy(h16)


def test_training_entries_refuse_int8_first():
    """Every pointer is null: the error names the INT8 plan, not the arguments.  Nothing can reach a device."""
    L = _C.lib()
    h = _create(ops.PREC_INT8)
    try:
        trn = (None,) * 4 + (100, None, 1, None, None, 0, None, None, 0, None, None)
        bwd = (None, None, 0, 100, 1, None, None, 0, None, None, None, None, None, 0, None)
        for fn, args in ((L.bevb200_encoder_forward_train, trn), (L.bevb200_encoder_forward_train_f16, trn),
                         (L.bevb200_encoder_backward, bwd), (L.bevb200_encoder_backward_f16, bwd)):
            assert fn(h, *args) == BEVB200_EINVAL
            assert "INT8" in L.bevb200_last_error().decode()
        assert L.bevb200_encoder_train_saved(h, 0, 0, None, -1, None, None) == BEVB200_EINVAL
        assert "INT8" in L.bevb200_last_error().decode()
        # the eval forward is the _f16 one; set_conv is the other precisions' packing call
        fwd = (None,) * 3 + (100, None, 1, None, None, 0, None, None, 0, None, None)
        assert L.bevb200_encoder_forward(h, *fwd) == BEVB200_EINVAL
        assert "_f16 calls" in L.bevb200_last_error().decode()
        assert L.bevb200_encoder_set_conv(h, 0, None, None, None, None, 0, None) == BEVB200_EINVAL
        assert "set_conv_int8" in L.bevb200_last_error().decode()
    finally:
        L.bevb200_encoder_destroy(h)


def test_set_conv_int8_refusals():
    L = _C.lib()
    h16, h8 = _create(ops.PREC_FP16), _create(ops.PREC_INT8)
    try:
        assert L.bevb200_encoder_set_conv_int8(h16, 0, None, None, None, 1.0, 1.0, 1.0, None, 0, None) == BEVB200_EINVAL
        assert "PREC_INT8" in L.bevb200_last_error().decode()
        pb = L.bevb200_encoder_param_bytes(h8)
        fake = ctypes.c_void_p(4096)    # never dereferenced: the scales are checked first
        for conv, s_in, s_out, s_res in ((1, 0.0, 1.0, 1.0), (1, 1.0, float("inf"), 1.0), (0, 1.0, -1.0, 1.0),
                                         (3, 1.0, 1.0, float("nan")), (2, float("nan"), 1.0, 1.0)):
            assert L.bevb200_encoder_set_conv_int8(h8, conv, fake, None, None, s_in, s_out, s_res, fake, pb,
                                                   None) == BEVB200_EINVAL
            assert "scales" in L.bevb200_last_error().decode()
    finally:
        L.bevb200_encoder_destroy(h16)
        L.bevb200_encoder_destroy(h8)


def test_u8_quantizer_matches_torch():
    r = 1.0
    vals = [0.0, -0.0, 0.5, 1.5, 2.5, 3.5, 126.5, 127.5, 253.5, 254.5, 254.49998, 255.0, 255.5, 256.0, 1e30,
            float("inf"), float("nan"), -1.0, -float("inf"), 1e-30, 0.49999997]
    v = np.array(vals, np.float32)
    got = quant_u8(v, r)
    t = torch.from_numpy(v) * r
    want = torch.round(torch.nan_to_num(t, nan=0.0, posinf=float("inf")).clamp(0, 255)).long().numpy()
    assert got.tolist() == want.tolist()
    assert got[15] == 255 and got[16] == 0                    # +inf saturates, NaN becomes 0
    assert got[2:6].tolist() == [0, 2, 2, 4]                  # ties to even
    # the scale multiplies first, in fp32
    v2 = np.array([1.0, 2.0, 3.0], np.float32)
    r2 = np.float32(1.0) / np.float32(0.012)
    assert quant_u8(v2, r2).tolist() == torch.round(torch.from_numpy(v2) * torch.tensor(r2)).long().tolist()


def test_weight_quantizer_matches_torch():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(27, 16, 32, generator=g)
    w[:, :, 3] = 0.0                                          # an all-zero channel: s_w = 1
    w[:, :, 4] = w[:, :, 4].clamp(-1, 1)
    w[0, 0, 4], w[1, 1, 4] = 1.27, -1.27                      # max 1.27: s_w = 0.01, q = +-127
    w[2, 2, 4] = 0.005                                        # a tie of W / s_w
    s, q = quant_weight(w.numpy())
    s_t = torch.where(w.abs().amax((0, 1)) > 0, w.abs().amax((0, 1)) / 127, torch.ones(32))
    q_t = torch.round(w / s_t).clamp(-127, 127).long()
    assert np.array_equal(s, s_t.numpy()) and np.array_equal(q, q_t.numpy())
    assert s[3] == 1.0 and (q[:, :, 3] == 0).all()
    assert q[0, 0, 4] == 127 and q[1, 1, 4] == -127
    assert np.abs(q).max() <= 127


def test_state_dict_unchanged_by_scales():
    m = voxelnet_0p075_encoder()
    keys = list(m.state_dict())
    from bevfusion_b200.encoder_plan import _chain_of
    n = len(_chain_of(m))
    assert m.int8_scales() is None
    m.set_int8_scales(torch.linspace(0.01, 0.2, n))
    assert list(m.state_dict()) == keys
    assert torch.equal(m.int8_scales(), torch.linspace(0.01, 0.2, n))
    fresh = voxelnet_0p075_encoder()
    fresh.load_state_dict(m.state_dict(), strict=True)
    for bad in (torch.ones(n - 1), torch.zeros(n), torch.full((n,), float("nan"))):
        with pytest.raises(ValueError):
            m.set_int8_scales(bad)
