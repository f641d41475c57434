"""The map-segmentation specification on the CPU: the float64 restatement (map_seg_oracle) against the fixture written
by the reference's own BEVGridTransform, losses, BEVSegmentationHead and evaluate_map; the host tap and CSR tables
against the oracle, with the default config's figures; argument refusals; the C entry points' host-side checks."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
import map_seg_oracle as O  # noqa: E402
from bevfusion_b200 import _C  # noqa: E402
from bevfusion_b200 import map_seg as MS  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "map_seg_tiny.npz")
GEOMS = ("p1", "p2", "p05", "p15", "pad", "pad2")


def geometry(g, name):
    osc = (g["wide_scope"] if name.startswith("pad") else g["out_scope"]).tolist()
    return g["in_scope"].tolist(), osc, float(g["grid_%s_p" % name])


def dense(rows, size):
    A = np.zeros((len(rows), size))
    for o, taps in enumerate(rows):
        for i, w in taps:
            A[o, i] += w
    return A


@pytest.mark.parametrize("name", GEOMS)
def test_oracle_reproduces_reference_grid_transform(name):
    g = np.load(GOLDEN)
    isc, osc, p = geometry(g, name)
    Ay, Ax = O.transform_matrices(isc, osc, 16, 12, p)
    y = O.grid_forward(g["grid_x"], Ay, Ax)
    want = g["grid_%s_out" % name]
    assert y.shape == want.shape
    # the fixture unnormalises the fp32 grid in float64; the oracle in fp32 as the CUDA op does
    np.testing.assert_allclose(y, want, rtol=0, atol=2e-6 * np.abs(want).max())
    gx = O.grid_backward(g["grid_%s_r" % name], Ay, Ax)
    np.testing.assert_allclose(gx, g["grid_%s_grad" % name], rtol=0, atol=2e-6 * np.abs(gx).max())


def test_fixture_covers_its_cases():
    g = np.load(GOLDEN)
    assert sorted(float(g["grid_%s_p" % n]) for n in GEOMS) == [0.5, 1, 1, 1.5, 2, 2]
    isc, osc, _ = geometry(g, "p1")
    assert isc[0] != isc[1] and osc[0] != osc[1]                           # non-square scope pair
    Ay, Ax = O.transform_matrices(*geometry(g, "pad")[:2], 16, 12)
    assert (np.abs(Ay).sum(1) == 0).any() and (np.abs(Ax).sum(1) == 0).any()   # outputs wholly in the padding
    assert np.isin(np.abs(g["loss_logits"]), [30, 100]).sum() == 8
    thr = np.float32([0.35, 0.4, 0.45, 0.5, 0.55, 0.6, 0.65])
    assert all((g["eval_pred"] == t).any() for t in thr)
    assert np.isnan(g["eval_pred"]).any()


@pytest.mark.parametrize("loss", ["focal", "xent"])
def test_oracle_reproduces_reference_losses(loss):
    g = np.load(GOLDEN)
    v = O.losses(g["loss_logits"], g["loss_target"], loss)
    np.testing.assert_allclose(v, g["loss_%s_values" % loss], rtol=1e-12, atol=0)
    d = O.loss_grad(g["loss_logits"], g["loss_target"], loss, g["loss_w"])
    np.testing.assert_allclose(d, g["loss_%s_grad" % loss], rtol=0, atol=1e-12 * np.abs(d).max())


def test_oracle_reproduces_reference_counts_and_metrics():
    g = np.load(GOLDEN)
    c = O.counts(g["eval_pred"], g["eval_gt"], MS.THRESHOLDS)
    np.testing.assert_array_equal(c, g["eval_counts"])
    m = MS.map_seg_metrics(torch.from_numpy(c), list(g["classes"]))
    assert list(m) == list(g["eval_keys"])
    np.testing.assert_allclose(list(m.values()), g["eval_values"], rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("name", GEOMS)
def test_host_tables_match_oracle(name):
    g = np.load(GOLDEN)
    isc, osc, p = geometry(g, name)
    for axis, size in ((0, 16), (1, 12)):
        rows = MS.axis_taps(MS.axis_coords(isc[axis], osc[axis]), size, p)
        want = O.axis_matrix(isc[axis], osc[axis], size, p)
        assert all(len(t) <= 4 for t in rows)
        assert all([i for i, _ in t] == sorted({i for i, _ in t}) for t in rows)
        np.testing.assert_allclose(dense(rows, size), want, rtol=0, atol=1e-6)
        cols = MS.transpose_taps(rows, size)
        np.testing.assert_array_equal(dense(cols, len(rows)), dense(rows, size).T)
        assert all([o for o, _ in t] == sorted(o for o, _ in t) for t in cols)


def test_default_config_tables():
    cfg = S.MAP_SEG_CFG
    for axis in (0, 1):
        c = MS.axis_coords(cfg["input_scope"][axis], cfg["output_scope"][axis])
        assert len(c) == 200
        rows = MS.axis_taps(c, 128)
        # output index i samples the input at 1.3125 + 0.625 i
        for i, taps in enumerate(rows):
            (i0, w0), (i1, w1) = taps
            assert i1 == i0 + 1
            assert abs(i0 + w1 - (1.3125 + 0.625 * i)) < 2e-5 and abs(w0 + w1 - 1) < 1e-6
        assert rows[0] == [(1, np.float32(0.6875)), (2, np.float32(0.3125))]
        ids = [i for t in rows for i, _ in t]
        assert min(ids) == 1 and max(ids) == 126
        cols = MS.transpose_taps(rows, 128)
        assert max(len(t) for t in cols) == 4 and not cols[0] and not cols[127]


def test_output_length_is_the_reference_arange():
    for osc in ([-50, 50, 0.5], [-50, 50, 0.3], [-1.0, 1.0, 0.7], [0.0, 3.0, 1.0]):
        n = len(torch.arange(osc[0] + osc[2] / 2, osc[1], osc[2]))
        assert len(MS.axis_coords([-51.2, 51.2, 0.8], osc)) == n == len(O.grid_coords([-51.2, 51.2, 0.8], osc))


def test_refusals():
    x = torch.zeros((1, 2, 8, 8))
    t = MS.BEVGridTransform(input_scope=[[-1, 1, 0.25]] * 2, output_scope=[[-1, 1, 0.25]] * 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        t(x)
    with pytest.raises(RuntimeError, match="CUDA"):
        MS.map_seg_loss(x, x, "focal", ["a", "b"])
    with pytest.raises(RuntimeError, match="CUDA"):
        MS.map_seg_counts(x, x)
    with pytest.raises(ValueError, match="unsupported loss"):
        MS.map_seg_loss(x, x, "dice", ["a", "b"])
    with pytest.raises(ValueError, match="mean"):
        MS.map_seg_loss(x, x, "focal", ["a", "b"], reduction="sum")
    empty = MS.BEVGridTransform(input_scope=[[-1, 1, 0.25]] * 2, output_scope=[[1, 1, 0.5], [-1, 1, 0.5]])
    with pytest.raises(ValueError, match="empty"):
        empty.plan(8, 8, "cpu")
    with pytest.raises(ValueError):
        MS.BEVGridTransform(input_scope=[[-1, 1, 0.25]], output_scope=[[-1, 1, 0.25]] * 2)
    with pytest.raises(ValueError):
        MS.BEVGridTransform(input_scope=[[-1, 1, 0.25]] * 2, output_scope=[[-1, 1, 0.25]] * 2, prescale_factor=0)
    with pytest.raises(ValueError):
        MS.map_seg_metrics(torch.zeros((3, 2, 7), dtype=torch.int64), ["a"])


def test_head_has_reference_state_dict_names():
    g = np.load(GOLDEN)
    head = MS.BEVSegmentationHead(4, dict(input_scope=g["in_scope"].tolist(), output_scope=g["out_scope"].tolist(),
                                          prescale_factor=2), list(g["classes"]), "focal")
    want = sorted(k[len("head_state/"):] for k in g.files if k.startswith("head_state/"))
    assert sorted(head.state_dict()) == want
    head.load_state_dict({k: torch.from_numpy(g["head_state/" + k]).float() for k in want})
    assert isinstance(head.transform, MS.BEVGridTransform) and head.transform.prescale_factor == 2


def test_synthetic_generators_are_seeded():
    a, b = S.map_seg_masks(3, 2), S.map_seg_masks(3, 2)
    assert a.shape == (2, 6, 200, 200) and a.dtype == torch.int64 and torch.equal(a, b)
    frac = a.float().mean((0, 2, 3))
    assert 0.05 < frac[0] < 0.7 and (frac > 0).all()
    x = S.map_seg_features(1, 1, 8, 16, 16)
    assert x.shape == (1, 8, 16, 16) and torch.equal(x, S.map_seg_features(1, 1, 8, 16, 16)) and (x >= 0).all()


def test_abi_symbols_declared_and_bound():
    names = ["bevb200_map_grid_smem_bytes", "bevb200_map_grid_transform", "bevb200_map_seg_loss_workspace_bytes",
             "bevb200_map_seg_loss", "bevb200_map_seg_loss_backward", "bevb200_map_seg_counts"]
    declared = _C.declared_symbols()
    for n in names:
        assert n in declared and n in _C._SIGNATURES
        getattr(_C.lib(), n)


def test_queries_and_host_refusals():
    L = _C.lib()
    # double partial per (1024-element tile, class, sample), 256-byte aligned
    assert L.bevb200_map_seg_loss_workspace_bytes(4, 6, 200, 200) == -(-4 * 6 * 40 * 8 // 256) * 256
    assert L.bevb200_map_seg_loss_workspace_bytes(0, 6, 200, 200) == 0
    assert L.bevb200_map_grid_smem_bytes(128, 200, 400, 12) == 816 + 3200 + 12 * 328 * 4
    fake = 256
    rc = L.bevb200_map_seg_loss(None, 0, None, 0, 1, 1, 4, 4, 1, None, None, 0, None)
    assert rc == -1 and b"null" in L.bevb200_last_error()
    rc = L.bevb200_map_seg_loss(fake, 0, fake, 0, 1, 1, 64, 64, 1, fake, fake, 8, None)
    assert rc == -3
    rc = L.bevb200_map_seg_loss_backward(fake, 0, fake, 0, 0, 1, 4, 4, 1, fake, fake, None)
    assert rc == -1
    thr = _C.host_array(ctypes.c_float, [0.5] * 17)
    assert L.bevb200_map_seg_counts(fake, 0, fake, 0, 1, 1, 4, 4, thr, 17, fake, None) == -1
    assert L.bevb200_map_seg_counts(fake, 0, fake, 0, 1, 1, 4, 4, thr, 0, fake, None) == -1
    args = [fake, fake, 0, 1, 8, 8, 8, 8] + [fake] * 6 + [4, fake, fake, 8]
    assert L.bevb200_map_grid_transform(*args, 8000, None) == -1                  # more block rows than the source
    wide = [fake, fake, 0, 1, 4000, 4000, 4000, 4000] + [fake] * 6 + [16000, fake, fake, 8]
    assert L.bevb200_map_grid_transform(*wide, 8, None) == -4                       # shared memory over 48 KiB
    assert L.bevb200_map_grid_transform(None, *args[1:], 4, None) == -1
