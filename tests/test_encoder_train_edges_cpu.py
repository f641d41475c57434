"""Host side of the training-step boundary cases (encoder_train_cases.py) and of the raw float64 oracle: the
constants are read from the kernels, every builder lands exactly on its boundary (rows per level from the CPU
rulebook oracle), and the oracle's BatchNorm, with its rule for fewer than 2 rows, agrees with torch's.  No device
is touched."""
import os
import re

import numpy as np
import pytest
import torch

import encoder_train_cases as C
from encoder_train_oracle import bn_train_rows, raw_rulebook, raw_train_forward

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "bevfusion_b200", "csrc")


def _rows_per_level(convs, coors, B, shape):
    idx, shape, rows = coors, list(shape), [int(coors.shape[0])]
    for c in convs:
        oidx, _, oshape = raw_rulebook(idx, B, shape, c)
        if not c["subm"]:
            rows.append(int(oidx.shape[0]))
        idx, shape = oidx, oshape
    return rows


def test_constants_read_from_the_kernels():
    with open(os.path.join(CSRC, "encoder.cu")) as f:
        enc = f.read()
    with open(os.path.join(CSRC, "spconv_wgrad_tc.cu")) as f:
        wgt = f.read()
    assert re.search(r"constexpr int kStatRows = %d;" % C.STAT_ROWS, enc)
    assert re.search(r"constexpr int kWgtRows = %d;" % C.WGT_ROWS, wgt)
    assert C.STAT_ROWS >= 2 and C.WGT_ROWS >= 2
    assert C.stat_counts() == [C.STAT_ROWS - 1, C.STAT_ROWS, C.STAT_ROWS + 1,
                               2 * C.STAT_ROWS - 1, 2 * C.STAT_ROWS, 2 * C.STAT_ROWS + 1]
    assert sorted(set(v % C.WGT_ROWS for v in C.tile_counts())) == [0, 1, C.WGT_ROWS - 1]


@pytest.mark.parametrize("c", [16, 128])
@pytest.mark.parametrize("n", C.stat_counts())
def test_stat_case_lands_on_every_level(c, n):
    cin, convs, shape, B, coors, rows = C.stat_case(c, n)
    assert len(np.unique(coors, axis=0)) == n
    assert _rows_per_level(convs, coors, B, shape) == rows == [n, n, n]


@pytest.mark.parametrize("n", C.tile_counts() + [2, 5, 300])
def test_lattice_one_level(n):
    cin, convs = C.TILE_CHAIN
    shape, B = [40, 36, 15], 2
    coors, rows = C.lattice_coors(shape, B, n, 1, seed=n)
    assert _rows_per_level(convs, coors, B, shape) == rows == [n, n]


def test_block_shares_one_cell():
    cin, convs = C.ONE_ROW_CHAIN
    coors, rows = C.block_coors([12, 10, 8])
    assert _rows_per_level(convs, coors, 1, [12, 10, 8]) == rows == [8, 1]
    coors, rows = C.block_coors([12, 10, 8], extra=5)
    assert _rows_per_level(convs, coors, 3, [12, 10, 8]) == rows == [13, 6]


def test_chains_are_well_formed():
    for name, (cin, convs) in list(C.TRAIN_RAW.items()) + [("one-row", C.ONE_ROW_CHAIN), ("tile", C.TILE_CHAIN),
                                                            ("stat16", C.stat_chain(16)), ("stat128", C.stat_chain(128))]:
        prev = cin
        for i, c in enumerate(convs):
            assert c["cin"] == prev, name
            assert c["res"] < 0 or (i - 2 <= c["res"] < i and convs[c["res"]]["cout"] == c["cout"]), name
            prev = c["cout"]
        assert C.n_strided(convs) >= 1, name


def _bn(n_ch, seed):
    torch.manual_seed(seed)
    bn = torch.nn.BatchNorm1d(n_ch, eps=1e-3, momentum=0.1).double().train()
    bn.running_mean.normal_(0, 0.1)
    bn.running_var.uniform_(0.5, 1.5)
    bn.weight.data.uniform_(0.8, 1.2)
    bn.bias.data.normal_(0, 0.1)
    return bn


@pytest.mark.parametrize("n", [2, 3, C.STAT_ROWS + 1])
def test_bn_rows_match_torch(n):
    bn = _bn(16, n)
    x = (torch.randn(n, 16, dtype=torch.float64) * 2 + 0.5).requires_grad_(True)
    x2 = x.detach().clone().requires_grad_(True)
    w = bn.weight.detach().clone().requires_grad_(True)
    b = bn.bias.detach().clone().requires_grad_(True)
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    y, moved = bn_train_rows(x, w, b, rm, rv, bn.eps, bn.momentum)
    want = bn(x2)
    assert moved
    assert torch.allclose(y, want, rtol=1e-12, atol=1e-12)
    assert torch.allclose(rm, bn.running_mean, rtol=1e-12, atol=1e-14)
    assert torch.allclose(rv, bn.running_var, rtol=1e-12, atol=1e-14)
    R = torch.randn(n, 16, dtype=torch.float64)
    (y * R).sum().backward()
    (want * R).sum().backward()
    assert torch.allclose(x.grad, x2.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(w.grad, bn.weight.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(b.grad, bn.bias.grad, rtol=1e-10, atol=1e-12)


def test_bn_one_row_rule():
    """torch refuses one row in training; the rule gives beta, leaves the statistics, and passes exactly no
    gradient to the row or to gamma"""
    bn = _bn(16, 1)
    x = torch.randn(1, 16, dtype=torch.float64, requires_grad=True)
    with pytest.raises(ValueError):
        bn(x)
    w = bn.weight.detach().clone().requires_grad_(True)
    b = bn.bias.detach().clone().requires_grad_(True)
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    y, moved = bn_train_rows(x, w, b, rm, rv, bn.eps, bn.momentum)
    assert not moved and torch.equal(rm, bn.running_mean) and torch.equal(rv, bn.running_var)
    assert torch.equal(y.detach(), b.detach()[None])
    (y * torch.randn(1, 16, dtype=torch.float64)).sum().backward()
    assert bool((x.grad == 0).all()) and bool((w.grad == 0).all()) and bool((b.grad != 0).all())
    y0, moved0 = bn_train_rows(x[:0], w, b, rm, rv, bn.eps, bn.momentum)
    assert y0.shape == (0, 16) and not moved0


def test_raw_oracle_step_counts_and_canvas():
    """a one-row last level through raw_train_forward: num_batches_tracked moves on level 0 only, and the canvas
    form holds the dense output in the first C*Z*X*Y floats of every sample"""
    cin, convs = C.ONE_ROW_CHAIN
    shape, B = [12, 10, 8], 2
    coors, rows = C.block_coors(shape)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(8, cin, dtype=torch.float64, generator=g)
    ws = [torch.randn(int(np.prod(c["ks"])), c["cin"], c["cout"], dtype=torch.float64, generator=g) * 0.2
          for c in convs]
    params = [(torch.ones(c["cout"], dtype=torch.float64), torch.zeros(c["cout"], dtype=torch.float64))
              for c in convs]
    masks = [torch.ones(8 if i < 2 else 1, c["cout"], dtype=torch.bool) for i, c in enumerate(convs)]

    def bufs():
        return [[torch.zeros(c["cout"], dtype=torch.float64), torch.ones(c["cout"], dtype=torch.float64), 0]
                for c in convs]

    b1 = bufs()
    dense, got_rows = raw_train_forward(convs, x, coors, B, shape, ws, params, b1, masks, 1e-3, 0.1)
    assert got_rows == rows == [8, 1]
    assert [b[2] for b in b1] == [1, 1, 0, 0, 0]
    assert all(torch.equal(b[0], torch.zeros_like(b[0])) for b in b1[2:])
    canvas, _ = raw_train_forward(convs, x, coors, B, shape, ws, params, bufs(), masks, 1e-3, 0.1,
                                  out_batch_stride=dense[0].numel() + 7)
    assert torch.equal(canvas[:, :dense[0].numel()].reshape(dense.shape), dense)
    assert not bool(canvas[:, dense[0].numel():].any())
