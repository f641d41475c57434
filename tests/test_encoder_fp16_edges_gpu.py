"""GPU tests of the SparseEncoder's fp16 training step (bevb200_encoder_forward_train_f16 / _backward_f16) on every
raw chain of encoder_train_cases and across its chunk, tile and row-count boundaries, against the float64 oracle of
encoder_fp16_oracle (per conv from the saved state: z16, running statistics, y16; dense() bit-equal to the last y16;
the backward against the straight-through twin with the run's ReLU masks).

  * Chains: every TRAIN_RAW chain -- residuals from one conv back, from two back, on the last conv (whose image, in
    fp16, is one of its level's two alternating buffers, as is its residual source), a strided first conv, a
    residual block on every level, c_out 16 on level 1, a 128-channel SubM, first convs of 7 / 20 / 40 channels.
  * Counts: every level at k * kStatRows + {-1, 0, 1} for Cout 16 and 128; level 1 at kWgtRows * m + {-1, 0, 1}
    and at 63 / 64 / 65 and 255 / 256 / 257; 2 rows; 1 row (a k2 s2 p0 conv over one 2x2x2 block:
    BEVB200_ENCODER_FEW_ROWS, running statistics left alone, exactly-zero gradients behind it).
  * A device count below the cap: NaN feature rows past it at coordinates outside the grid, on a residual chain and
    under a cap of hundreds of filter-gradient tiles; the feature gradient rows past the count are 0.
  * The state and the workspace at exactly their queried sizes inside canary-filled buffers."""
import ctypes

import numpy as np
import pytest
import torch

from bevfusion_b200 import _C
from bevfusion_b200.encoder_plan import _BNDesc
from bevfusion_b200.spconv.ops import PREC_FP16
from encoder_fp16_oracle import bwd_bounds, check_train_forward, dense64, fp16_round, rulebooks, twin_backward
from encoder_train_cases import (ONE_ROW_CHAIN, STAT_ROWS, TILE_CHAIN, TRAIN_RAW, WGT_ROWS, block_coors,
                                 lattice_coors, stat_case, stat_counts, tile_counts)
from encoder_train_oracle import rel
from test_encoder_plan_gpu import create, random_coors
from test_encoder_train_edges_gpu import _arr, _guard_intact, _guarded

pytestmark = pytest.mark.gpu

EPS, MOMENTUM = 1e-3, 0.1
FEW_ROWS = 2


class RawF16:
    """One raw conv chain on an fp16 plan through the C ABI, on exactly-sized state / workspace.  Rows past n_valid
    (up to n_rows) are NaN features at coordinates outside the grid."""

    def __init__(self, dev, cin, shape, B, convs, coors, n_rows=None, seed=0):
        self.dev, self.cin, self.shape, self.B, self.convs = dev, cin, list(shape), B, convs
        self.coors = np.ascontiguousarray(coors, dtype=np.int32)
        self.n_valid = self.coors.shape[0]
        self.n_rows = n_rows or self.n_valid
        L = self.L = _C.lib()
        g = torch.Generator().manual_seed(seed)
        feats = torch.randn(self.n_valid, cin, generator=g).half()
        self.feats = torch.cat([feats, torch.full((self.n_rows - self.n_valid, cin), float("nan")).half()]).to(dev)
        pad = np.full((self.n_rows - self.n_valid, 4), 100000, np.int32)
        self.coors_dev = torch.from_numpy(np.concatenate([self.coors, pad])).to(dev)
        self.n_dev = torch.tensor([self.n_valid], dtype=torch.int32, device=dev)
        self.w, self.gamma, self.beta, self.rm, self.rv = [], [], [], [], []
        for c in convs:
            kv = int(np.prod(c["ks"]))
            self.w.append((torch.randn(kv, c["cin"], c["cout"], generator=g) / (kv * c["cin"]) ** 0.5).to(dev))
            self.gamma.append((torch.rand(c["cout"], generator=g) * 0.4 + 0.8).to(dev))
            self.beta.append((torch.randn(c["cout"], generator=g) * 0.1).to(dev))
            self.rm.append((torch.randn(c["cout"], generator=g) * 0.1).to(dev))
            self.rv.append((torch.rand(c["cout"], generator=g) + 0.5).to(dev))
        self.nbt = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in convs]
        self.before = [(m.clone(), v.clone()) for m, v in zip(self.rm, self.rv)]
        rc, self.h = create(cin, shape, convs)
        assert rc == 0, L.bevb200_last_error()
        _C.check(L.bevb200_encoder_set_precision(self.h, PREC_FP16), "encoder_set_precision")
        self.n_levels = L.bevb200_encoder_num_levels(self.h)
        oshape, oc = (ctypes.c_int32 * 3)(), ctypes.c_int32()
        _C.check(L.bevb200_encoder_output_shape(self.h, oshape, ctypes.byref(oc)), "encoder_output_shape")
        X, Y, Z = list(oshape)
        self.out_shape = (B, oc.value * Z, X, Y)
        caps = (ctypes.c_int32 * self.n_levels)()
        _C.check(L.bevb200_encoder_level_caps(self.h, self.n_rows, B, None, caps), "encoder_level_caps")
        self.level_caps = list(caps)
        self.state_bytes = L.bevb200_encoder_train_state_bytes(self.h, self.n_rows, B, None)
        self.state_buf, self.state = _guarded(self.state_bytes, dev)
        self.ws_bytes = L.bevb200_encoder_backward_workspace_bytes(self.h, self.n_rows, B, None)
        self.ws_buf, self.ws = _guarded(self.ws_bytes, dev)

    def close(self):
        if self.h is not None:
            self.L.bevb200_encoder_destroy(self.h)
            self.h = None

    def _bn(self):
        descs = (_BNDesc * len(self.convs))()
        for i, d in enumerate(descs):
            d.weight, d.bias = _C.ptr(self.gamma[i]), _C.ptr(self.beta[i])
            d.running_mean, d.running_var = _C.ptr(self.rm[i]), _C.ptr(self.rv[i])
            d.num_batches_tracked = _C.ptr(self.nbt[i])
            d.eps, d.momentum = EPS, MOMENTUM
        return descs

    def forward(self):
        self.out = torch.full(self.out_shape, float("nan"), dtype=torch.float16, device=self.dev)
        self.status = torch.full((1 + self.n_levels,), -1, dtype=torch.int32, device=self.dev)
        rc = self.L.bevb200_encoder_forward_train_f16(
            self.h, _arr(self.w), self._bn(), _C.ptr(self.feats), _C.ptr(self.coors_dev), self.n_rows,
            _C.ptr(self.n_dev), self.B, None, _C.ptr(self.out), 0, _C.ptr(self.status), _C.ptr(self.state),
            self.state_bytes, _C.current_stream(self.dev), None)
        _C.check(rc, "encoder_forward_train_f16")
        torch.cuda.synchronize()
        return self.status.cpu().tolist()

    def saved(self):
        """[(z16, y16)] of every conv over its level's valid rows, float64"""
        st = self.status.cpu().tolist()
        out, level = [], 0
        for i, c in enumerate(self.convs):
            level += 0 if c["subm"] else 1
            zo, yo = ctypes.c_size_t(), ctypes.c_size_t()
            _C.check(self.L.bevb200_encoder_train_saved(self.h, self.n_rows, self.B, None, i, ctypes.byref(zo),
                                                        ctypes.byref(yo)), "encoder_train_saved")
            n, cc = st[1 + level], c["cout"]
            z = self.state[zo.value:zo.value + n * cc * 2].view(torch.float16).view(n, cc)
            y = self.state[yo.value:yo.value + n * cc * 2].view(torch.float16).view(n, cc)
            out.append((z.double().cpu(), y.double().cpu()))
        return out

    def backward(self, R):
        gf = torch.full((self.n_rows, self.cin), float("nan"), dtype=torch.float16, device=self.dev)
        gw = [torch.full_like(w, float("nan")) for w in self.w]
        gg = [torch.full_like(v, float("nan")) for v in self.gamma]
        gb = [torch.full_like(v, float("nan")) for v in self.beta]
        rc = self.L.bevb200_encoder_backward_f16(
            self.h, _arr(self.w), _C.ptr(self.state), self.state_bytes, self.n_rows, self.B, None,
            _C.ptr(R.half().to(self.dev)), 0, _C.ptr(gf), _arr(gw), _arr(gg), _arr(gb), _C.ptr(self.ws),
            self.ws_bytes, _C.current_stream(self.dev))
        torch.cuda.synchronize()
        return rc, {"features": gf.cpu(), "w": [t.cpu() for t in gw], "gamma": [t.cpu() for t in gg],
                    "beta": [t.cpu() for t in gb]}


def check_step(run, what, flags=0, seed=1):
    """forward + backward of an fp16 run against float64 -> (status, native gradients, float64 gradients)"""
    st = run.forward()
    saved = run.saved()
    n = run.n_valid
    rbs = rulebooks(run.convs, run.coors, run.B, run.shape)
    rows = [n] + [int(oidx.shape[0]) for c, (oidx, _, _) in zip(run.convs, rbs) if not c["subm"]]
    assert st == [flags] + rows, "%s: status %s, float64 rows %s" % (what, st, rows)
    x16 = run.feats[:n].double().cpu()
    bns = [(g, b, EPS, MOMENTUM) for g, b in zip(run.gamma, run.beta)]
    after = [(m.clone(), v.clone()) for m, v in zip(run.rm, run.rv)]
    worst = check_train_forward(run.convs, x16, run.w, bns, saved, run.before, after, rbs, what)
    assert torch.equal(run.out.double().cpu(), dense64(saved[-1][1], rbs[-1][0], run.B, rbs[-1][2])), what
    for i, (zy, (oidx, _, _)) in enumerate(zip(saved, rbs)):
        assert int(run.nbt[i]) == (1 if zy[0].shape[0] >= 2 else 0), (what, i)
    R = fp16_round(torch.randn(run.out_shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64))
    rc, got = run.backward(R)
    assert rc == 0, run.L.bevb200_last_error()
    gx, gw, gg, gb = twin_backward(run.convs, rbs, x16, run.w, bns, saved, R, run.B)
    assert bool((got["features"][n:] == 0).all()), "%s: gradient rows past the count are not 0" % what
    bound, bound_x = bwd_bounds(len(run.convs))
    table = [("features", got["features"][:n], gx, bound_x)]
    for i in range(len(run.convs)):
        table += [("w%d" % i, got["w"][i], gw[i], bound), ("gamma%d" % i, got["gamma"][i], gg[i], bound),
                  ("beta%d" % i, got["beta"][i], gb[i], bound)]
    ratios = []
    for name, g, want, b in table:
        assert bool(torch.isfinite(g).all()), (what, name)
        l2 = rel(g, want)[0]
        assert l2 <= b, (what, name, l2, b)
        ratios.append(l2 / b)
    assert _guard_intact(run.state_buf, run.state_bytes) and _guard_intact(run.ws_buf, run.ws_bytes), what
    print("%-32s rows %s  worst ratio %s  backward rel L2 / bound %.3f" % (
        what, rows, {k: round(v, 3) for k, v in worst.items()}, max(ratios)))
    return st, got, (gx, gw, gg, gb)


def _run(cuda, cin, convs, shape, B, coors, what, **kw):
    run = RawF16(cuda, cin, shape, B, convs, coors, **kw)
    try:
        return run, check_step(run, what)
    finally:
        run.close()


@pytest.mark.parametrize("chain", list(TRAIN_RAW))
def test_raw_chain_fp16(cuda, chain):
    cin, convs = TRAIN_RAW[chain]
    shape, B = [40, 36, 15], 2
    _run(cuda, cin, convs, shape, B, random_coors(shape, B, 3000, seed=len(chain)), chain, seed=len(chain))


@pytest.mark.parametrize("chain", ["residual-previous", "residual-on-last"])
def test_device_count_below_cap(cuda, chain):
    cin, convs = TRAIN_RAW[chain]
    shape, B = [40, 36, 15], 2
    _run(cuda, cin, convs, shape, B, random_coors(shape, B, 2500, seed=11), chain + " n_dev < cap", n_rows=2637)


@pytest.mark.parametrize("c", [16, 128])
@pytest.mark.parametrize("n", stat_counts())
def test_stat_chunk_counts(cuda, c, n):
    cin, convs, shape, B, coors, rows = stat_case(c, n)
    assert rows == [n] * 3
    _run(cuda, cin, convs, shape, B, coors, "stats c%d n=%d (chunk %d)" % (c, n, STAT_ROWS))


@pytest.mark.parametrize("n", tile_counts() + [63, 64, 65, 255, 256, 257, 2])
def test_level_counts(cuda, n):
    """level 1 holds n rows: on kWgtRows tile edges, at 63 / 64 / 65 and 255 / 256 / 257, and 2"""
    cin, convs = TILE_CHAIN
    shape, B = [40, 36, 15], 2
    coors, rows = lattice_coors(shape, B, n, 1, seed=n)
    run, (st, _, _) = _run(cuda, cin, convs, shape, B, coors, "level counts n=%d (tile %d)" % (n, WGT_ROWS))
    assert st[1:] == [n, n]


def test_count_below_one_tile_under_a_large_cap(cuda):
    cin, convs = TILE_CHAIN
    shape, B = [80, 72, 31], 2
    coors, _ = lattice_coors(shape, B, 5, 1, seed=5)
    run, _ = _run(cuda, cin, convs, shape, B, coors, "5 rows under cap", n_rows=4096)
    assert run.level_caps[1] // WGT_ROWS >= 200, run.level_caps


def test_one_row_on_the_last_level(cuda):
    """8 voxels of one 2x2x2 block through a k2 s2 p0 conv: level 1 holds one row.  The flag is set, level 1's
    running statistics stay, and every gradient that reaches level 0 through level 1's BN is exactly 0."""
    cin, convs = ONE_ROW_CHAIN
    shape, B = [12, 10, 8], 1
    coors, rows = block_coors(shape)
    assert rows == [8, 1]
    run = RawF16(cuda, cin, shape, B, convs, coors, seed=4)
    try:
        st, got, _ = check_step(run, "one row on level 1", flags=FEW_ROWS)
        for i, lv in enumerate([0, 0, 1, 1, 1]):
            m0, v0 = run.before[i]
            assert (torch.equal(run.rm[i], m0) and torch.equal(run.rv[i], v0)) == (lv == 1), i
            assert bool((got["w"][i] == 0).all()) and bool((got["gamma"][i] == 0).all()), i
            if lv == 0:
                assert bool((got["beta"][i] == 0).all()), i
        assert bool((got["features"] == 0).all())
        assert bool((got["beta"][4] != 0).any())
    finally:
        run.close()
