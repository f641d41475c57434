"""CPU tests of the SparseEncoder's fp16 precision: the constant and the precision names, the fp16 plan's size
queries against their layout formula (and below BF16x3's), the BEVB200_EINVAL paths that need no device, and the
float64 oracle's fp16 rounding against torch.half on boundary values."""
import ctypes
import os
import re

import pytest
import torch

from bevfusion_b200 import _C
from bevfusion_b200.spconv import ops
from encoder_fp16_oracle import fp16_round

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "bevfusion_b200.h")
BEVB200_EINVAL = -1


def test_precision_constant_and_names(monkeypatch):
    text = open(HEADER).read()
    assert int(re.search(r"#define BEVB200_PREC_FP16 (\d+)", text).group(1)) == ops.PREC_FP16 == 4
    assert ops.PREC_FP16 not in (ops.PREC_FP32, ops.PREC_TF32X3, ops.PREC_TF32, ops.PREC_BF16X3)
    assert sorted(ops._PREC_NAMES) == ["bf16x3", "fp32", "tf32", "tf32x3"]     # the environment names stay four
    monkeypatch.setenv("BEVB200_SPCONV_PRECISION", "fp16")
    with pytest.raises(KeyError):
        ops.default_precision()


class _Conv(ctypes.Structure):
    _fields_ = [("c_in", ctypes.c_int32), ("c_out", ctypes.c_int32), ("ksize", ctypes.c_int32 * 3),
                ("stride", ctypes.c_int32 * 3), ("padding", ctypes.c_int32 * 3), ("dilation", ctypes.c_int32 * 3),
                ("subm", ctypes.c_int32), ("relu", ctypes.c_int32), ("residual_from", ctypes.c_int32)]


# c_in, c_out, subm, residual_from: a SubM, a strided conv, a residual block, conv_out (k 1,1,3 s 1,1,2)
CHAIN = [(5, 16, 1, -1, (3, 3, 3)), (16, 32, 0, -1, (3, 3, 3)), (32, 32, 1, -1, (3, 3, 3)), (32, 32, 1, 1, (3, 3, 3)),
         (32, 64, 0, -1, (3, 3, 3)), (64, 128, 0, -1, (1, 1, 3))]


def _create(precision=None):
    L = _C.lib()
    descs = (_Conv * len(CHAIN))()
    for d, (ci, co, subm, res, ks) in zip(descs, CHAIN):
        d.c_in, d.c_out, d.subm, d.relu, d.residual_from = ci, co, subm, 1, res
        for k in range(3):
            d.ksize[k], d.dilation[k] = ks[k], 1
            d.stride[k] = 1 if subm else (2 if ks[k] == 3 or k == 2 else 1)
            d.padding[k] = 1 if ks[k] == 3 else 0
    h = ctypes.c_void_p()
    shape = (ctypes.c_int32 * 3)(64, 64, 41)
    assert L.bevb200_encoder_create(5, shape, descs, len(CHAIN), ctypes.byref(h)) == 0
    if precision is not None:
        assert L.bevb200_encoder_set_precision(h, precision) == 0
    return h


def _sizes(h, n=5000, B=2):
    L = _C.lib()
    return (L.bevb200_encoder_param_bytes(h), L.bevb200_encoder_workspace_bytes(h, n, B, None),
            L.bevb200_encoder_train_state_bytes(h, n, B, None),
            L.bevb200_encoder_backward_workspace_bytes(h, n, B, None))


def _align(x):
    return (x + 255) // 256 * 256


def test_sizes_fp16_below_bf16x3():
    L = _C.lib()
    h3, h16 = _create(), _create(ops.PREC_FP16)
    try:
        assert L.bevb200_encoder_precision(h3) == ops.PREC_BF16X3
        assert L.bevb200_encoder_precision(h16) == ops.PREC_FP16
        s3, s16 = _sizes(h3), _sizes(h16)
        for a, b in zip(s16, s3):
            assert 0 < a < b
        # the parameter buffer: per conv the fp16 weight image (K blocks of 64 channels, Cout rows of 128 B), then
        # scale and shift, each 256-byte aligned
        want = 0
        for ci, co, _, _, ks in CHAIN:
            ce = max(16, 1 << (ci - 1).bit_length())
            kv = ks[0] * ks[1] * ks[2]
            want += _align((kv * ce + 63) // 64 * co * 128) + 2 * _align(co * 4)
        assert s16[0] == want
        # the training state: z16 and y16 are [cap, c_out] half per conv, the level-0 image [cap, c_eff] half, and no
        # fp32 rows of the last conv; both layouts share the rulebooks, the parameters' alignment and the partials
        caps = (ctypes.c_int32 * 8)()
        assert L.bevb200_encoder_level_caps(h16, 5000, 2, None, caps) == 0
        levels = [0, 1, 1, 1, 2, 3]
        rows16 = _align(5000 * 16 * 2) + sum(2 * _align(caps[l] * co * 2) for l, (_, co, *_r) in zip(levels, CHAIN))
        rows3 = (_align(5000 * 16 * 4) + sum(2 * _align(caps[l] * co * 4) for l, (_, co, *_r) in zip(levels, CHAIN))
                 + _align(caps[3] * 128 * 4))
        assert s3[2] - s16[2] == (rows3 - rows16) + (s3[0] - s16[0])
    finally:
        L.bevb200_encoder_destroy(h3)
        L.bevb200_encoder_destroy(h16)


def test_set_precision_refuses_other_precisions():
    L = _C.lib()
    h = _create()
    try:
        before = _sizes(h)
        for p in (ops.PREC_FP32, ops.PREC_TF32X3, ops.PREC_TF32, 5, -1):
            assert L.bevb200_encoder_set_precision(h, p) == BEVB200_EINVAL
        assert _sizes(h) == before and L.bevb200_encoder_precision(h) == ops.PREC_BF16X3
        assert L.bevb200_encoder_set_precision(None, ops.PREC_FP16) == BEVB200_EINVAL
        # back and forth: the layout follows the precision
        assert L.bevb200_encoder_set_precision(h, ops.PREC_FP16) == 0
        assert L.bevb200_encoder_set_precision(h, ops.PREC_BF16X3) == 0
        assert _sizes(h) == before
    finally:
        L.bevb200_encoder_destroy(h)


def test_wrong_precision_refused_first():
    """A call of the wrong precision family is refused before any other argument is read: every pointer is null
    here, and the error names the precision, not the null arguments.  Nothing can reach a device."""
    L = _C.lib()
    h3, h16 = _create(), _create(ops.PREC_FP16)
    try:
        fwd = (None,) * 3 + (100, None, 1, None, None, 0, None, None, 0, None, None)
        trn = (None,) * 4 + (100, None, 1, None, None, 0, None, None, 0, None, None)
        bwd = (None, None, 0, 100, 1, None, None, 0, None, None, None, None, None, 0, None)
        calls = [(L.bevb200_encoder_forward, h16, fwd), (L.bevb200_encoder_forward_f16, h3, fwd),
                 (L.bevb200_encoder_forward_train, h16, trn), (L.bevb200_encoder_forward_train_f16, h3, trn),
                 (L.bevb200_encoder_backward, h16, bwd), (L.bevb200_encoder_backward_f16, h3, bwd)]
        for fn, h, args in calls:
            assert fn(h, *args) == BEVB200_EINVAL
            msg = L.bevb200_last_error().decode()
            assert "_f16 calls" in msg, msg
        # the right family with the same null arguments fails on them instead
        assert L.bevb200_encoder_forward(h3, *fwd) == BEVB200_EINVAL
        assert "_f16 calls" not in L.bevb200_last_error().decode()
    finally:
        L.bevb200_encoder_destroy(h3)
        L.bevb200_encoder_destroy(h16)


def test_fp16_rounding_oracle_matches_torch_half():
    vals = [0.0, -0.0, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -26, 2.0 ** -26, 2.0 ** -14, 2.0 ** -14 - 2.0 ** -25,
            2.0 ** -14 - 2.0 ** -24, 65504.0, 65519.999, 65520.0, 65536.0, 1e6, 1.0 + 2.0 ** -11,
            1.0 + 3 * 2.0 ** -11, 2048.0 + 1.0, 2048.0 + 3.0, 1.0 / 3.0, 0.1, 5e-8, 6e-8]
    x = torch.tensor(vals + [-v for v in vals], dtype=torch.float64)
    x = torch.cat([x, torch.randn(20000, dtype=torch.float64) * torch.exp2(torch.randint(-26, 17, (20000,)).double())])
    # fp32 values, as the device rounds fp32 to fp16 (torch.half of a double may round twice, through fp32)
    x = x.float().double()
    got = fp16_round(x)
    want = x.float().to(torch.float16).double()  # IEEE round to nearest even, overflow to inf
    assert torch.equal(torch.isinf(got), torch.isinf(want))
    assert torch.equal(got, want)
    nan = fp16_round(torch.tensor([float("nan")], dtype=torch.float64))
    assert bool(torch.isnan(nan).all())
