"""GPU tests of the SparseEncoder's INT8 precision (SparseEncoder.forward(..., precision=PREC_INT8)) against the numpy
restatement of its contract in encoder_int8_oracle.

  * Exact chains: conv-0 features on a 2^-4 grid (|x| <= 8) and weights on a 2^-8 grid (|w| <= 1), so conv 0's fp32
    sums are exact in any order and dense() must equal the oracle bit for bit: voxelnet at B = 2, every raw chain of
    encoder_train_cases with a ReLU after each conv (chains that lack one get it: residuals one and two convs back and
    on the last conv, a strided first conv, a residual block on every level, Cout 16 on level 1, a 128-channel SubM,
    first convs of 7 / 20 / 40 channels, k2 s2 over one 2x2x2 block), both sides of the wgmma threshold, every level
    at 1, 63 / 64 / 65 and 255 / 256 / 257 rows, and a device row count below the cap (NaN rows past it).
  * Random features, on short lattice chains: every dense() cell outside the rows the oracle taints is bit-equal; the
    tainted fraction prints.
  * Calibration against a float64 run of the chain; a CUDA-graph replay against eager, sync-free; the refusals."""
import ctypes

import numpy as np
import pytest
import torch

from bevfusion_b200 import _C
from bevfusion_b200.sparse_block import bn_scale_shift
from bevfusion_b200.spconv.ops import PREC_INT8
from encoder_fp16_oracle import conv64, module_convs, rulebooks
from encoder_int8_oracle import chain_scales, run_chain
from encoder_train_cases import ONE_ROW_CHAIN, TILE_CHAIN, TRAIN_RAW, block_coors, lattice_coors, n_strided
from test_encoder_fp16_gpu import _coors, _randomise_bn, voxelnet
from test_encoder_plan_gpu import create

pytestmark = pytest.mark.gpu


def _grid(t, step, lim, g):
    return (torch.randint(-int(lim / step), int(lim / step) + 1, t.shape, generator=g).float() * step)


def _with_relu(convs):
    return [dict(c, relu=True) for c in convs]


INT8_RAW = {k: (cin, _with_relu(convs)) for k, (cin, convs) in TRAIN_RAW.items()}
INT8_RAW["k2s2-one-block"] = (ONE_ROW_CHAIN[0], _with_relu(ONE_ROW_CHAIN[1]))
INT8_RAW["tile"] = (TILE_CHAIN[0], _with_relu(TILE_CHAIN[1]))


class RawI8:
    """One raw conv chain on an INT8 plan through the C ABI.  Rows past n_valid (up to n_rows) are NaN features at
    coordinates outside the grid.

    Optional overrides of the seeded draws (which are made all the same, so the other values do not move): feats
    (fp32 [n_valid, cin], rounded to fp16), and per conv index the dicts weights (fp32 [K, cin, cout]), bn_scales
    and shifts (fp32 [cout] or None); s_act replaces chain_scales, and its None entries are chosen by one pass of the
    oracle (encoder_int8_oracle.run_chain)."""

    def __init__(self, dev, cin, shape, B, convs, coors, n_rows=None, seed=0, exact=True, feats=None, weights=None,
                 bn_scales=None, shifts=None, s_act=None):
        self.dev, self.cin, self.shape, self.B, self.convs = dev, cin, list(shape), B, convs
        self.coors = np.ascontiguousarray(coors, dtype=np.int32)
        self.n_valid = self.coors.shape[0]
        self.n_rows = n_rows or self.n_valid
        g = torch.Generator().manual_seed(seed)
        f = _grid(torch.empty(self.n_valid, cin), 2.0 ** -4, 8.0, g) if exact else torch.randn(self.n_valid, cin, generator=g)
        self.feats16 = f.half()
        self.w, self.s, self.t = [], [], []
        for i, c in enumerate(convs):
            kv = int(np.prod(c["ks"]))
            w = torch.randn(kv, c["cin"], c["cout"], generator=g) / (kv * c["cin"]) ** 0.5
            self.w.append(_grid(w, 2.0 ** -8, 1.0, g) * 0.25 if i == 0 else w)
            self.s.append(torch.rand(c["cout"], generator=g) + 0.5 if c.get("scale", True) else None)
            self.t.append(torch.randn(c["cout"], generator=g) * 0.2 if c.get("shift", True) else None)
        if feats is not None:
            self.feats16 = torch.as_tensor(feats, dtype=torch.float32).half()
        for dst, src in ((self.w, weights), (self.s, bn_scales), (self.t, shifts)):
            for i, v in (src or {}).items():
                dst[i] = None if v is None else torch.as_tensor(v, dtype=torch.float32)
        self._stats = None
        if s_act is not None:
            self.s_act = list(s_act)
            if any(v is None for v in self.s_act):
                self.stats()
            return
        self.s_act = chain_scales(convs, self.feats16.numpy(), self.coors, B, shape, [w.numpy() for w in self.w],
                                  [None if s is None else s.numpy() for s in self.s],
                                  [None if t is None else t.numpy() for t in self.t])

    def run(self):
        L, dev = _C.lib(), self.dev
        rc, h = create(self.cin, self.shape, self.convs)
        assert rc == 0, L.bevb200_last_error()
        try:
            _C.check(L.bevb200_encoder_set_precision(h, PREC_INT8), "encoder_set_precision")
            stream = _C.current_stream(dev)
            pbuf = torch.empty(L.bevb200_encoder_param_bytes(h), dtype=torch.uint8, device=dev)
            keep = []
            for i, c in enumerate(self.convs):
                w, s, t = [None if x is None else x.to(dev) for x in (self.w[i], self.s[i], self.t[i])]
                keep += [w, s, t]
                _C.check(L.bevb200_encoder_set_conv_int8(
                    h, i, _C.ptr(w), _C.ptr(s), _C.ptr(t), self.s_act[i - 1] if i else 1.0, self.s_act[i],
                    self.s_act[c["res"]] if c["res"] >= 0 else 1.0, _C.ptr(pbuf), pbuf.numel(), stream), "set_conv_int8")
            nan = torch.full((self.n_rows - self.n_valid, self.cin), float("nan")).half()
            feats = torch.cat([self.feats16, nan]).to(dev)
            pad = np.full((self.n_rows - self.n_valid, 4), 100000, np.int32)
            coors = torch.from_numpy(np.concatenate([self.coors, pad])).to(dev)
            n_dev = torch.tensor([self.n_valid], dtype=torch.int32, device=dev)
            ws = torch.empty(L.bevb200_encoder_workspace_bytes(h, self.n_rows, self.B, None), dtype=torch.uint8,
                             device=dev)
            oshape, oc = (ctypes.c_int32 * 3)(), ctypes.c_int32()
            _C.check(L.bevb200_encoder_output_shape(h, oshape, ctypes.byref(oc)), "encoder_output_shape")
            X, Y, Z = list(oshape)
            out = torch.full((self.B, oc.value * Z, X, Y), float("nan"), dtype=torch.float16, device=dev)
            status = torch.full((1 + L.bevb200_encoder_num_levels(h),), -1, dtype=torch.int32, device=dev)
            _C.check(L.bevb200_encoder_forward_f16(h, _C.ptr(pbuf), _C.ptr(feats), _C.ptr(coors), self.n_rows,
                                                   _C.ptr(n_dev), self.B, None, _C.ptr(out), 0, _C.ptr(status),
                                                   _C.ptr(ws), ws.numel(), stream, None), "encoder_forward_f16")
            torch.cuda.synchronize()
            return out, status.cpu().tolist()
        finally:
            L.bevb200_encoder_destroy(h)

    def oracle(self, exact=True, stats=None):
        if exact and stats is None and self._stats is not None:
            return self._stats[1]
        return run_chain(self.convs, self.feats16.numpy(), self.coors, self.B, self.shape,
                         [w.numpy() for w in self.w], [None if s is None else s.numpy() for s in self.s],
                         [None if t is None else t.numpy() for t in self.t], self.s_act, exact=exact, stats=stats)

    def stats(self):
        """the exact oracle's per-conv stats (encoder_int8_oracle.STAT_KEYS); fixes the s_act it chose"""
        if self._stats is None:
            st = []
            res = self.oracle(stats=st)
            self.s_act = [d["s_act"] for d in st]
            self._stats = (st, res)
        return self._stats[0]


def _check_exact(raw):
    out, status = raw.run()
    want, _, _ = raw.oracle()
    assert status[0] == 0
    got = out.double().cpu()
    assert got.shape == want.shape
    bad = got != want
    assert not bool(bad.any()), "%d of %d cells differ (max %g)" % (int(bad.sum()), bad.numel(),
                                                                    float((got - want).abs().max()))
    return status


@pytest.mark.parametrize("chain", list(INT8_RAW))
def test_exact_raw_chain(cuda, chain):
    cin, convs = INT8_RAW[chain]
    shape, B = [40, 36, 20], 2                    # even: the k2 s2 p0 conv keeps every lattice site
    if chain == "k2s2-one-block":
        coors, rows = block_coors(shape, extra=40)
    else:
        coors, rows = lattice_coors(shape, B, 700, n_strided(convs), seed=3)
    status = _check_exact(RawI8(cuda, cin, shape, B, convs, coors, seed=4))
    assert status[1:] == rows


@pytest.mark.parametrize("n", [1, 63, 64, 65, 255, 256, 257])
def test_exact_row_counts(cuda, n):
    """every level of the tile chain (mma.sync and wgmma instances) at n rows"""
    cin, convs = INT8_RAW["tile"]
    shape, B = [64, 64, 41], 2
    coors, rows = lattice_coors(shape, B, n, n_strided(convs), seed=n)
    assert _check_exact(RawI8(cuda, cin, shape, B, convs, coors, seed=n))[1:] == rows


@pytest.mark.parametrize("chain", ["residual-two-back", "tile"])
def test_exact_device_count_below_cap(cuda, chain):
    cin, convs = INT8_RAW[chain]
    shape, B = [40, 36, 21], 2
    coors, rows = lattice_coors(shape, B, 500, n_strided(convs), seed=7)
    assert _check_exact(RawI8(cuda, cin, shape, B, convs, coors, n_rows=900, seed=8))[1:] == rows


def _module_case(cuda, exact, seed=0):
    shape, B = [48, 48, 41], 2
    torch.manual_seed(seed)
    m = _randomise_bn(voxelnet(shape), seed)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        conv0 = m.conv_input[0].weight
        conv0.copy_(_grid(conv0, 2.0 ** -8, 1.0, g) * 0.25 if exact else conv0)
    m = m.to(cuda).eval()
    coors = _coors(shape, B, 1500, seed)
    f = _grid(torch.empty(coors.shape[0], 5), 2.0 ** -4, 8.0, g) if exact else torch.randn(coors.shape[0], 5, generator=g)
    return m, f.half(), coors, shape, B


def _module_oracle(m, feats16, coors, B, shape, exact):
    plan = m.plan(PREC_INT8)
    convs = module_convs(plan)
    w, sc, sh = [], [], []
    for conv, bn, _, _ in plan.chain:
        s, t = bn_scale_shift(bn)
        w.append(conv.weight.detach().float().cpu().reshape(-1, conv.in_channels, conv.out_channels).numpy())
        sc.append(s.float().cpu().numpy())
        sh.append(t.float().cpu().numpy())
    return run_chain(convs, feats16.numpy(), coors, B, shape, w, sc, sh, [float(v) for v in m.int8_scales()],
                     exact=exact)


def test_exact_voxelnet_b2(cuda):
    m, feats16, coors, shape, B = _module_case(cuda, exact=True)
    cd = torch.from_numpy(coors).to(cuda)
    keys = list(m.state_dict())
    m.calibrate_int8([(feats16.float().to(cuda), cd, B)])
    assert list(m.state_dict()) == keys
    with torch.no_grad():
        out = m(feats16.to(cuda), cd, B, precision=PREC_INT8)
    want, _, _ = _module_oracle(m, feats16, coors, B, shape, exact=True)
    got = out.double().cpu()
    assert out.dtype == torch.float16 and got.shape == want.shape
    assert torch.equal(got, want), "%d cells differ" % int((got != want).sum())


@pytest.mark.parametrize("chain", ["residual-two-back", "tile"])
def test_random_features_untainted_bit_equal(cuda, chain):
    """seeded N(0, 1) features: conv 0's fp32 sums may fall either side of a rounding tie, so only the rows the
    oracle leaves untainted are compared (a 3x3x3 rulebook spreads taint to every neighbour, so the chains are the
    short lattice ones, where a tie taints few rows)"""
    cin, convs = INT8_RAW[chain]
    shape, B = [40, 36, 20], 2
    coors, _ = lattice_coors(shape, B, 700, n_strided(convs), seed=21)
    raw = RawI8(cuda, cin, shape, B, convs, coors, seed=22, exact=False)
    out, status = raw.run()
    want, tainted, frac = raw.oracle(exact=False)
    got = out.double().cpu()
    print("%s: tainted fraction of the last level's rows %.4f" % (chain, frac))
    keep = ~tainted
    assert frac < 0.5 and bool((keep & (want != 0)).any())
    assert torch.equal(got[keep], want[keep]), "%d untainted cells differ" % int((got[keep] != want[keep]).sum())


def test_calibration_matches_float64(cuda):
    m, feats16, coors, shape, B = _module_case(cuda, exact=False, seed=9)
    x = feats16.float()
    scales = m.calibrate_int8([(x.to(cuda), torch.from_numpy(coors).to(cuda), B)])
    plan = m.plan(PREC_INT8)
    convs = module_convs(plan)
    rbs = rulebooks(convs, coors, B, shape)
    h, outs, ref = x.double(), [], []
    for (conv, bn, relu, res), c, (oidx, pl, _) in zip(plan.chain, convs, rbs):
        s, t = bn_scale_shift(bn)
        z, _ = conv64(h, conv.weight.detach().double().cpu().reshape(-1, c["cin"], c["cout"]), pl, oidx.shape[0])
        y = z * s.double().cpu() + t.double().cpu()
        if res >= 0:
            y = y + outs[res]
        y = y.clamp_min(0)
        outs.append(y)
        ref.append(float(y.max()) / 255.0)
        h = y
    ref = torch.tensor(ref, dtype=torch.float64)
    err = ((scales.double() - ref).abs() / ref).max()
    print("calibration: max relative deviation from float64 %.3e" % float(err))
    assert float(err) <= 2e-4     # BF16x3 per-conv rounding (~1e-5 relative) over the 21-conv chain


def test_graph_replay_equals_eager_sync_free(cuda):
    m, feats16, coors, shape, B = _module_case(cuda, exact=False, seed=11)
    cd = torch.from_numpy(coors).to(cuda)
    f = feats16.to(cuda)
    m.calibrate_int8([(f.float(), cd, B)])
    n_dev = torch.tensor([coors.shape[0]], dtype=torch.int32, device=cuda)
    with torch.no_grad():
        eager = m(f, cd, B, precision=PREC_INT8, num_voxels=n_dev).clone()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            again = m(f, cd, B, precision=PREC_INT8, num_voxels=n_dev)     # no device-to-host sync inside
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert torch.equal(again, eager)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            m(f, cd, B, precision=PREC_INT8, num_voxels=n_dev)
        torch.cuda.current_stream().wait_stream(side)
        out = torch.full_like(eager, float("nan"))
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            m(f, cd, B, precision=PREC_INT8, num_voxels=n_dev, out=out)
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(out, eager)


def test_refusals_leave_output_unwritten(cuda):
    m, feats16, coors, shape, B = _module_case(cuda, exact=False, seed=13)
    cd = torch.from_numpy(coors).to(cuda)
    f = feats16.to(cuda)
    X, Y, Z = m.plan().out_shape
    out = torch.full((B, 128 * Z, X, Y), float("nan"), dtype=torch.float16, device=cuda)

    def refused(**kw):
        with pytest.raises(ValueError):
            m(f, cd, B, precision=PREC_INT8, out=out, **kw)
        torch.cuda.synchronize()
        assert bool(torch.isnan(out).all())

    with torch.no_grad():
        refused()                                             # before calibration
    m.calibrate_int8([(f.float(), cd, B)])
    with torch.no_grad():
        refused(fused=False)
        m.train()
        refused()
        m.eval()
    refused()                                                 # grad enabled
    with torch.no_grad():
        with pytest.raises(ValueError):
            m(f, cd, B, precision=PREC_INT8, out=torch.empty_like(out, dtype=torch.float32))
        assert bool(torch.isnan(out).all())
        # a chain with a conv that has no ReLU: conv_input without its activation
        from bevfusion_b200.sparse_encoder import SparseEncoder
        plain = SparseEncoder(5, shape, order=("conv", "norm", "act")).to(cuda).eval()
        plain.conv_input = torch.nn.Sequential(*list(plain.conv_input)[:2]).to(cuda)
        plain._int8_scales = torch.ones(8)
        with pytest.raises(ValueError):
            plain(f, cd, B, precision=PREC_INT8, out=out)
        torch.cuda.synchronize()
        assert bool(torch.isnan(out).all())
