"""The head losses' specification on the CPU: the float64 restatement (head_losses_oracle) against the fixture written
by the reference's own CenterHead.loss / TransFusionHead.loss; the clamp-boundary generator; the loss-config and
argument validation of head_losses; the C entry points' host-side refusals and workspace queries."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
import head_losses_oracle as O  # noqa: E402
from bevfusion_b200 import _C  # noqa: E402
from bevfusion_b200 import head_losses as HL  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "head_losses_tiny.npz")
CH_KEYS = ("heatmap", "reg", "height", "dim", "rot", "vel")
TF_KEYS = ("dense_heatmap", "heatmap", "center", "height", "dim", "rot", "vel")


def golden_centerhead(g, name):
    T = len(g[name + "_cats"])
    preds = [{k: g["%s_t%d_%s" % (name, t, k)] for k in CH_KEYS} for t in range(T)]
    targets = tuple([g["%s_t%d_%s" % (name, t, k)] for t in range(T)]
                    for k in ("target_heatmap", "anno", "ind", "mask"))
    grads = [{k: g["%s_t%d_grad_%s" % (name, t, k)] for k in CH_KEYS} for t in range(T)]
    losses = dict(zip(g[name + "_loss_keys"], g[name + "_loss_values"]))
    return preds, targets, grads, losses


def golden_transfusion(g, name):
    preds = {k: g["%s_%s" % (name, k)] for k in TF_KEYS}
    targets = (g[name + "_labels"], g[name + "_label_weights"], g[name + "_bbox_targets"], g[name + "_bbox_weights"],
               int(g[name + "_num_pos"]), [float(g[name + "_matched_ious"])], g[name + "_target_heatmap"])
    grads = {k: g["%s_grad_%s" % (name, k)] for k in TF_KEYS}
    losses = dict(zip(g[name + "_loss_keys"], g[name + "_loss_values"]))
    P, L, aux = (int(v) for v in g[name + "_sizes"])
    return preds, targets, grads, losses, P, L, bool(aux)


def close(got, want, rtol):
    for k in want:
        np.testing.assert_allclose(got[k], want[k], rtol=rtol, atol=0, err_msg=k)


def grads_close(got, want, tol):
    for k in want:
        scale = max(np.abs(want[k]).max(), 1e-30)
        np.testing.assert_allclose(got[k], want[k], rtol=0, atol=tol * scale, err_msg=k)
        np.testing.assert_array_equal(got[k] == 0, want[k] == 0, err_msg=k + " zero set")


@pytest.mark.parametrize("name", ["ch", "chw"])
def test_oracle_reproduces_reference_centerhead(name):
    g = np.load(GOLDEN)
    preds, targets, grads, losses = golden_centerhead(g, name)
    assert list(losses) == ["%s/task%d" % (k, t) for t in range(6) for k in ("heatmap", "bbox")]
    lw = g[name + "_lw"]
    got, ggot = O.centerhead(preds, targets, g[name + "_cw"], cls=(lw[0], 2.0, 4.0), bbox_lw=lw[1], f64=True)
    close(got, losses, 1e-7)
    for t in range(6):
        grads_close(ggot[t], grads[t], 1e-7)


@pytest.mark.parametrize("name", ["tf_aux", "tf_last"])
def test_oracle_reproduces_reference_transfusion(name):
    g = np.load(GOLDEN)
    preds, targets, grads, losses, P, L, aux = golden_transfusion(g, name)
    got, ggot = O.transfusion(preds, targets, P, L, aux, g[name + "_cw"], f64=True)
    assert list(got) == list(losses)
    close(got, losses, 1e-7)
    grads_close(ggot, grads, 1e-7)


def test_fixture_covers_its_cases():
    """Duplicate inds on masked slots, masked-out slots, exact-1 targets, saturated logits, untrained columns."""
    g = np.load(GOLDEN)
    for t in range(6):
        ind, mask = g["ch_t%d_ind" % t], g["ch_t%d_mask" % t]
        assert (ind[:, 0] == ind[:, 1]).all() and (mask[:, :2] == 1).all() and (mask == 0).any()
        assert (g["ch_t%d_target_heatmap" % t] == 1).sum() == 5
        assert (np.abs(g["ch_t%d_heatmap" % t]) == 100).sum() == 6
        assert (g["ch_t%d_grad_heatmap" % t][np.abs(g["ch_t%d_heatmap" % t]) == 100] == 0).all()
    assert (g["tf_last_grad_heatmap"][:, :, 5:] == 0).all() and (g["tf_aux_grad_heatmap"][:, :, 5:] != 0).any()
    assert (g["tf_aux_labels"] == 3).any() and (g["tf_aux_label_weights"] == 0).any()


def test_boundary_generator_reaches_the_bounds():
    xs, ys = O.boundary_logits(O.sigmoid32)
    lo, hi = np.float32(O.LO), np.float32(O.HI)
    assert (ys < lo).any() and (ys >= lo).any() and (ys[:4] < lo).sum() == 2
    assert (ys == hi).any() and (ys > hi).any() and (ys[(ys > lo) & (ys < hi)]).size > 0
    assert np.all(np.diff(xs[:4]) > 0)


def test_oracle_edge_semantics():
    # a target one ulp below 1 is not positive; NaN targets make the L1 NaN with a 0 gradient
    s, n, _ = O.gaussian_focal(np.zeros(3), np.array([1.0, np.nextafter(np.float32(1), np.float32(0)), 0.5],
                                                      np.float32))
    assert n == 1.0 and np.isfinite(s)
    s, g = O.l1(np.array([1.0, 2.0]), np.array([np.nan, 1.0]), np.array([0.0, 1.0]))
    assert np.isnan(s) and g.tolist() == [0.0, 1.0]
    # saturated logits in the sigmoid focal loss stay finite
    s, g = O.sigmoid_focal(np.array([[100.0, -100.0]]), np.array([0]), np.array([1]))
    assert np.isfinite(s) and np.isfinite(g).all()


CPU = torch.zeros(1)


@pytest.mark.parametrize("cfg", [dict(type="GaussianFocalLoss", reduction="sum"), dict(type="FocalLoss"),
                                 dict(type="GaussianFocalLoss", beta=1.0), "GaussianFocalLoss"])
def test_centerhead_refuses_unsupported_cls_config(cfg):
    with pytest.raises(ValueError):
        HL.centerhead_loss([[{}]], ([CPU], [CPU], [CPU], [CPU]), dict(code_weights=[1.0] * 10), loss_cls=cfg)


@pytest.mark.parametrize("kw", [dict(loss_cls=dict(type="FocalLoss", use_sigmoid=False)),
                                dict(loss_cls=dict(type="VarifocalLoss", use_sigmoid=True)),
                                dict(loss_bbox=dict(type="SmoothL1Loss")),
                                dict(loss_bbox=dict(type="L1Loss", reduction="none")),
                                dict(loss_heatmap=dict(type="FocalLoss", use_sigmoid=True))])
def test_transfusion_refuses_unsupported_configs(kw):
    with pytest.raises(ValueError):
        HL.transfusion_loss([[{}]], (CPU,) * 8, 5, 2, True, dict(code_weights=[1.0] * 10), **kw)


def test_cpu_tensors_are_refused():
    B, H, W, M = 1, 4, 4, 2
    task = dict(heatmap=torch.zeros(B, 1, H, W), reg=torch.zeros(B, 2, H, W), height=torch.zeros(B, 1, H, W),
                dim=torch.zeros(B, 3, H, W), rot=torch.zeros(B, 2, H, W), vel=torch.zeros(B, 2, H, W))
    targets = ([torch.zeros(B, 1, H, W)], [torch.zeros(B, M, 10)], [torch.zeros(B, M, dtype=torch.int64)],
               [torch.zeros(B, M, dtype=torch.uint8)])
    with pytest.raises(RuntimeError, match="CUDA"):
        HL.centerhead_loss([[task]], targets, dict(code_weights=[1.0] * 10))


def test_abi_symbols_declared_and_bound():
    names = ["bevb200_centerhead_loss_workspace_bytes", "bevb200_centerhead_loss", "bevb200_centerhead_loss_backward",
             "bevb200_transfusion_loss_workspace_bytes", "bevb200_transfusion_loss",
             "bevb200_transfusion_loss_backward"]
    declared = _C.declared_symbols()
    for n in names:
        assert n in declared and n in _C._SIGNATURES
        getattr(_C.lib(), n)


def test_workspace_queries():
    L = _C.lib()
    cat = _C.host_array(ctypes.c_int, [1, 2, 2, 1, 2, 2])
    # parts: one per 1024-cell heat tile and one per (task, sample), 24 bytes each, 256-byte aligned
    tiles = sum(-(-4 * c * 128 * 128 // 1024) for c in [1, 2, 2, 1, 2, 2]) + 6 * 4
    assert L.bevb200_centerhead_loss_workspace_bytes(6, 4, cat, 128, 128, 500, 10) == -(-tiles * 24 // 256) * 256
    assert L.bevb200_centerhead_loss_workspace_bytes(6, 4, cat, 128, 128, 500, 9) == 0
    assert L.bevb200_centerhead_loss_workspace_bytes(6, 4, cat, 128, 128, HL.MAX_OBJS + 1, 10) == 0
    assert L.bevb200_centerhead_loss_workspace_bytes(0, 4, cat, 128, 128, 500, 10) == 0
    assert L.bevb200_transfusion_loss_workspace_bytes(4, 10, 180, 180, 400, 200, 2, 10) > 0
    assert L.bevb200_transfusion_loss_workspace_bytes(4, 10, 180, 180, 401, 200, 2, 10) == 0
    assert L.bevb200_transfusion_loss_workspace_bytes(4, 10, 180, 180, 400, 200, 3, 10) == 0
    assert L.bevb200_transfusion_loss_workspace_bytes(1, 10, 8, 8, 16 * 5, 5, 16, 10) == 0


def test_entry_points_refuse_on_the_host():
    L = _C.lib()
    cat = _C.host_array(ctypes.c_int, [1])
    nul = [None] * 11
    rc = L.bevb200_centerhead_loss(*nul[:10], cat, 1, 1, 4, 4, 2, 10, None, 2.0, 4.0, 1.0, 0.25, None, None, None,
                                   None, 0, None)
    assert rc == -1 and b"null" in L.bevb200_last_error()
    cat17 = _C.host_array(ctypes.c_int, [1] * 17)
    rc = L.bevb200_centerhead_loss(*nul[:10], cat17, 17, 1, 4, 4, 2, 10, None, 2.0, 4.0, 1.0, 0.25, None, None, None,
                                   None, 0, None)
    assert rc == -4
    rc = L.bevb200_transfusion_loss(*[None] * 13, 1, None, 1, 1, 10, 8, 8, 10, 5, 2, 10, None, None, None, None,
                                    None, None, None, 0, None)
    assert rc == -1 and b"null" in L.bevb200_last_error()
    rc = L.bevb200_transfusion_loss(*[None] * 13, 1, None, 1, 1, 10, 8, 8, 11, 5, 2, 10, None, None, None, None,
                                    None, None, None, 0, None)
    assert rc == -1 and b"multiple" in L.bevb200_last_error()
    rc = L.bevb200_transfusion_loss_backward(*[None] * 12, 1, 10, 8, 8, 100, 5, 16, 10, *[None] * 3, *[None] * 9,
                                             None)
    assert rc == -4
