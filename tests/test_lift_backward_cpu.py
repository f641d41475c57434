"""CPU: host-side contract of the fused lift + pool backward entry points (size queries, argument validation, no
CPU fallback).  Every call below returns before the library touches a device."""
import pytest
import torch

CHANNELS = (16, 32, 64, 80, 96, 128, 160, 256)
EINVAL, EWORKSPACE = -1, -3
FAKE = 1 << 20          # a 16-byte-aligned stand-in address: validation fails before anything is dereferenced


def _lib():
    from bevfusion_b200 import _C
    return _C.lib()


def test_workspace_queries():
    L = _lib()
    cols = L.bevb200_bev_pool_lift_columns_backward_workspace_bytes
    pix = L.bevb200_bev_pool_lift_backward_workspace_bytes
    # bad sizes / unsupported channel counts -> 0
    assert cols(-1, 10, 80) == 0 and cols(10, -1, 80) == 0 and cols(10, 10, 0) == 0 and cols(10, 10, 20) == 0
    assert pix(-1, 80) == 0 and pix(100, 7) == 0 and pix(100, 512) == 0
    for c in CHANNELS:
        assert cols(0, 0, c) > 0 and pix(0, c) > 0
        # one segment cell (int32) per segment / one cell per frustum point
        assert cols(62000, 40000, c) >= 62000 * 4
        assert cols(124000, 40000, c) >= cols(62000, 40000, c) + 62000 * 4
        assert pix(2_000_000, c) >= 2_000_000 * 4
        assert pix(4_000_000, c) > pix(2_000_000, c)
    # never shrinks with the channel count
    sizes = [cols(62000, 40000, c) for c in CHANNELS]
    assert sizes == sorted(sizes)


def _cols_call(c=80, fh=32, ws_bytes=1 << 20, out_grad=FAKE, depth=FAKE, ctx=FAKE, seg_key=FAKE, ddepth=FAKE,
               dctx=FAKE, n_segments=100, workspace=FAKE):
    return _lib().bevb200_bev_pool_lift_columns_backward(
        1, 1, 360, 360, 1000, c, 50, out_grad, depth, ctx, 6, 118, fh, 88, FAKE, FAKE, FAKE, seg_key, FAKE,
        n_segments, ddepth, dctx, workspace, ws_bytes, 0)


def _pix_call(c=80, ws_bytes=1 << 30, out_grad=FAKE, depth=FAKE, ctx=FAKE, perm=FAKE, ddepth=FAKE, dctx=FAKE,
              workspace=FAKE):
    n_total = 2 * 10 * 72 * 8
    return _lib().bevb200_bev_pool_lift_backward(
        1, 1, 64, 64, 1000, n_total, c, 50, out_grad, depth, ctx, 10, 72 * 8, perm, FAKE, FAKE, FAKE, ddepth, dctx,
        workspace, ws_bytes, 0)


def test_column_backward_validation():
    for c in (0, 20, 48, 512, 81):
        assert _cols_call(c=c) == EINVAL
    assert _cols_call(fh=65) == EINVAL                      # the segment mask is 64 bits: the pixel kernel's case
    assert _cols_call(out_grad=0) == EINVAL
    assert _cols_call(seg_key=0) == EINVAL
    assert _cols_call(ctx=0) == EINVAL                      # ddepth needs ctx
    assert _cols_call(depth=0) == EINVAL                    # dctx needs depth
    assert _cols_call(ctx=FAKE + 4) == EINVAL               # 16-byte alignment
    assert _cols_call(dctx=FAKE + 8) == EINVAL
    assert _cols_call(out_grad=FAKE + 4) == EINVAL
    assert _cols_call(n_segments=-1) == EINVAL
    assert _cols_call(ws_bytes=16) == EWORKSPACE
    assert _cols_call(workspace=0) == EWORKSPACE
    assert _cols_call(ddepth=0, dctx=0) == 0               # nothing requested: nothing to do


def test_pixel_backward_validation():
    for c in (0, 20, 48, 512):
        assert _pix_call(c=c) == EINVAL
    assert _pix_call(out_grad=0) == EINVAL
    assert _pix_call(perm=0) == EINVAL
    assert _pix_call(ctx=0) == EINVAL
    assert _pix_call(depth=0) == EINVAL
    assert _pix_call(ctx=FAKE + 4) == EINVAL
    assert _pix_call(ws_bytes=16) == EWORKSPACE
    assert _pix_call(workspace=0) == EWORKSPACE
    assert _pix_call(ddepth=0, dctx=0) == 0
    from bevfusion_b200 import _C
    assert b"workspace" in _C.lib().bevb200_last_error()


def test_lift_pool_rejects_cpu_tensors():
    from bevfusion_b200.bev_pool import BEVPoolPlan
    plan = BEVPoolPlan.__new__(BEVPoolPlan)      # no tables needed: the inputs are rejected first
    depth = torch.rand(1, 2, 4, 8, 6)
    ctx = torch.rand(1, 2, 8, 6, 16)
    with pytest.raises(RuntimeError):
        plan.lift_pool(depth, ctx)
    with pytest.raises(RuntimeError):
        plan.lift_pool(depth.requires_grad_(True), ctx.requires_grad_(True))
