"""GPU: the sync-free BEV pooling and fused-lift twins (*_dev) at their edges, against the host-count calls bit for bit
and against float64.

Part A (tests named *twin*) calls every twin through the C ABI on synthetic tables of capacity `cap` whose entries
past the device counts are in bounds but wrong (tests/bev_pool_sync_free_cases.py): n_kept on the TMA kernels'
warp-range boundaries for every tuned width, capacities n_kept, n_kept + 1 and ~3 n_kept, B*D = 1 (the kernels
zero-fill) and B*D > 1 (memset), the generic kernels, a status word naming the other lift form, the column-table prepare
at caps around the segment count with a canary behind the column tables, and the refusals.  A read past a count doubles
a row, adds a cell or reads NaN, so it fails the float64 bound without leaving any allocation.

Part B (tests named *plan*) runs BEVPoolPlan.from_cameras(..., sync=False): both lift forms at every tuned width,
feature heights around 64, one plan rebuilt through an empty grid, a half-empty one and one over the cap, CUDA graphs
of rebuild_ + pool / lift_pool + backward replayed over that sequence, C2 at B = 4 and C5, and NaN at dropped points.

Bounds: pooling L * 2^-24 * sum|x|, the lift (L + 1) * 2^-24 * sum|d * ctx|, gradients 1e-5 * max|gold|, empty cells
exactly +0.0.  Each float64 check prints its worst error as a fraction of its bound."""
import types

import numpy as np
import pytest
import torch

from bevfusion_b200 import _C
from bev_pool_sync_free_cases import (FEATURE_HEIGHTS, LAYOUTS, TUNED, UNTUNED, TwinTables, capacities, caps_around,
                                      counts_at, lift_dims, stale_segments)
from test_bev_pool_dispatch_gpu import (CANARY, Case, check_sums, grad_expected, lift_reference, misalign,
                                        pool_reference, workspace)
from test_bev_pool_sync_free_gpu import (assert_column_tables_equal, assert_tables_equal, calib, frustum, host_plan,
                                         host_rows, inputs, lift_step, plans, rig, same)
from test_lift_backward_gpu import assert_close, gold64

pytestmark = pytest.mark.gpu

EINVAL, EWORKSPACE = -1, -3
COLUMNS, ROWS = 0, 1
SLACK = 256             # the column-forward and both lift-backward queries report this much over what the call needs
TAIL = 64               # canary records behind seg_key / seg_mask / seg_slot


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def twice(fn, outs, ws=None, pattern=None, nbytes=0):
    """fn() over NaN-filled `outs`, twice: both runs succeed and agree bit for bit, and the canary behind the
    workspace is intact.  Returns clones of the first run's outputs."""
    res = []
    for _ in range(2):
        for o in outs:
            o.fill_(float("nan"))
        torch.cuda.synchronize()
        rc = fn()
        torch.cuda.synchronize()
        assert rc == 0, _C.lib().bevb200_last_error()
        res.append([o.clone() for o in outs])
    for a, b in zip(*res):
        assert same(a, b), "not bit-reproducible"
    if ws is not None:
        assert torch.equal(ws[nbytes:], pattern), "workspace canary overwritten"
    return res[0]


def status(form, dev):
    """int32 [2] = {n_segments, lift_form} on the device"""
    return torch.tensor([0, form], dtype=torch.int32, device=dev)


# ---------------------------------------------------------------------------------------------------- part A
class Twin:
    """A TwinTables case on the device, with the float64 references of the tables cut to the counts."""

    def __init__(self, dev, tb, lift=False):
        self.tb, self.dev, self.c = tb, dev, tb.c
        self.cap, self.n_kept, self.n_int, self.dims = tb.cap, tb.n_kept, tb.n_int, tb.dims
        g = lambda a: t(a).to(dev)
        self.perm, self.perm_stale = g(tb.perm), g(tb.perm_stale)
        self.geom, self.starts, self.lengths = g(tb.geom), g(tb.starts), g(tb.lengths)
        self.counts = torch.tensor([tb.n_kept, tb.n_int], dtype=torch.int32, device=dev)
        self.stream = _C.current_stream(dev)
        gen = torch.Generator(device=dev).manual_seed(tb.cap)
        if lift:
            self.cams, self.D, self.fH, self.fW = lift_dims(tb.cap)
            shape = (1, self.cams, self.D, self.fH, self.fW)
            self.depth = torch.rand(shape, generator=gen, device=dev).contiguous()
            self.ctx = torch.randn(1, self.cams, self.fH, self.fW, self.c, generator=gen, device=dev)
            self.depth_nan, self.ctx_nan = self.depth.clone(), self.ctx.clone()
            dropped = g(tb.nan_rows).long()
            self.depth_nan.view(-1)[dropped] = float("nan")
            self.depth.view(-1)[dropped] = 0.0
            kept = torch.zeros(tb.cap, dtype=torch.bool, device=dev)
            kept[self.perm[:tb.n_kept].long()] = True
            hw = self.fH * self.fW
            self.empty_px = ~kept.view(self.cams, self.D, hw).any(1).view(-1)
            self.ctx_nan.view(-1, self.c)[self.empty_px] = float("nan")
            self.ctx.view(-1, self.c)[self.empty_px] = 0.0
            self.dropped = dropped
        else:
            self.x = torch.randn(tb.cap, self.c, generator=gen, device=dev)
            self.x[g(tb.nan_rows).long()] = float("nan")
        self.G = torch.randn(*self.dims, self.c, generator=gen, device=dev)

    def shell(self, perm=None):
        """the dispatch test's Case over the tables cut to the counts (what pool_reference / grad_expected read)"""
        case = Case.__new__(Case)
        tb = self.tb
        case.dims, case.c, case.n, case.n_int, case.n_total = self.dims, self.c, self.n_kept, self.n_int, self.cap
        case.starts_np, case.lengths_np = tb.starts[:self.n_int], tb.lengths[:self.n_int]
        case.geom_np, case.perm_np = tb.geom[:self.n_kept], tb.perm
        case.x = getattr(self, "x", None)
        case.perm, case.geom, case.starts, case.lengths = perm, self.geom, self.starts, self.lengths
        return case

    def plan_shell(self):
        """what lift_reference / gold64 read of a plan"""
        tables = types.SimpleNamespace(dims=self.dims, geom=self.geom[:self.n_kept], perm=self.perm, n_kept=self.n_kept)
        return types.SimpleNamespace(tables=tables)


def ptr(x):
    return _C.ptr(x)


def pool_host(tw, x, out):
    L = _C.lib()
    nbytes = L.bevb200_bev_pool_workspace_bytes(tw.n_kept, tw.c)
    ws, pattern = workspace(nbytes, tw.dev)
    return twice(lambda: L.bevb200_bev_pool_perm(*tw.dims, tw.n_kept, tw.c, tw.n_int, ptr(x), ptr(tw.perm_stale),
                                                 ptr(tw.geom), ptr(tw.starts), ptr(tw.lengths), ptr(out), ptr(ws),
                                                 nbytes, tw.stream), [out], ws, pattern, nbytes)[0]


def pool_twin(tw, x, out, nbytes=None, counts=None):
    L = _C.lib()
    need = L.bevb200_bev_pool_dev_workspace_bytes(tw.cap, tw.c)
    ws, pattern = workspace(need, tw.dev)
    counts = tw.counts if counts is None else counts
    fn = lambda: L.bevb200_bev_pool_perm_dev(*tw.dims, tw.cap, tw.c, ptr(x), ptr(tw.perm_stale), ptr(tw.geom),
                                             ptr(tw.starts), ptr(tw.lengths), _C.ptr(counts), ptr(out), ptr(ws),
                                             need if nbytes is None else nbytes, tw.stream)
    if nbytes is not None:
        return fn
    return twice(fn, [out], ws, pattern, need)[0]


def grad_twin(tw, og, xg):
    L = _C.lib()
    return twice(lambda: L.bevb200_bev_pool_grad_perm_dev(*tw.dims, tw.cap, tw.c, ptr(og), ptr(tw.perm), ptr(tw.geom),
                                                          ptr(tw.starts), ptr(tw.lengths), ptr(tw.counts), ptr(xg),
                                                          tw.stream), [xg])[0]


def grad_host(tw, og, xg):
    L = _C.lib()
    return twice(lambda: L.bevb200_bev_pool_grad_perm(*tw.dims, tw.n_kept, tw.cap, tw.c, tw.n_int, ptr(og),
                                                      ptr(tw.perm), ptr(tw.geom), ptr(tw.starts), ptr(tw.lengths),
                                                      ptr(xg), tw.stream), [xg])[0]


def check_pool_twin(tw, what, mis=""):
    x = misalign(tw.x) if "x" in mis else tw.x
    out = torch.empty(*tw.dims, tw.c, device=tw.dev)
    if "o" in mis:
        out = misalign(out)
    got = pool_twin(tw, x, out)
    assert same(got, pool_host(tw, x, out)), "%s: differs from the host-count call" % what
    check_sums(got, *pool_reference(tw.shell()), 0, what)
    og = tw.G if "x" not in mis else misalign(tw.G)
    xg = torch.empty(tw.cap, tw.c, device=tw.dev)
    if "x" in mis:
        xg = misalign(xg)
    got = grad_twin(tw, og, xg)
    assert same(got, grad_host(tw, og, xg)), "%s: gradient differs from the host-count call" % what
    assert same(got, grad_expected(tw.shell(), tw.G)), "%s: gradient differs from the gather" % what


@pytest.mark.parametrize("c,n", [(c, n) for c in TUNED for n in counts_at(c)])
def test_pool_twins_at_range_boundaries(cuda, c, n):
    """bevb200_bev_pool_perm_dev / _grad_perm_dev with the device n_kept at 0, 1, 31..33 and around every k * R * 32:
    TMA forward (zero-filling at B*D = 1, memset at B = 2) and backward, each capacity"""
    for i, cap in enumerate(capacities(n)):
        for B in (1, 2):
            lay = LAYOUTS[(i + B + n) % len(LAYOUTS)]
            tw = Twin(cuda, TwinTables(n, cap, c, lay, seed=n + cap + B, B=B))
            check_pool_twin(tw, "pool twin C=%d n=%d cap=%d B=%d %s" % (c, n, cap, B, lay))


@pytest.mark.parametrize("c,mis", [(UNTUNED, ""), (80, "x"), (80, "o"), (256, "x")])
@pytest.mark.parametrize("n", [0, 1, 33, 9001])
def test_pool_twins_generic_kernels(cuda, c, mis, n):
    """an untuned width, and x / out / out_grad / x_grad 4 bytes off alignment: the generic kernels with device counts"""
    for cap in capacities(n):
        for B in (1, 2):
            tw = Twin(cuda, TwinTables(n, cap, c, "hot", seed=n + cap + B, B=B))
            check_pool_twin(tw, "pool twin generic C=%d mis=%s n=%d cap=%d B=%d" % (c, mis or "-", n, cap, B), mis)


@pytest.mark.parametrize("c", [16, 80, UNTUNED])
def test_pool_twins_with_points_but_no_interval(cuda, c):
    """n_kept > 0 with n_intervals == 0: a zero grid and zero gradients, as the host-count call gives"""
    for B in (1, 2):
        tw = Twin(cuda, TwinTables(5000, 9000, c, "hot", seed=B, B=B, no_intervals=True))
        check_pool_twin(tw, "pool twin no interval C=%d B=%d" % (c, B))


# ---- the row lift
def lift_rows_host(tw, depth, ctx, out):
    L = _C.lib()
    nbytes = L.bevb200_bev_pool_workspace_bytes(tw.n_kept, tw.c)
    ws, pattern = workspace(nbytes, tw.dev)
    return twice(lambda: L.bevb200_bev_pool_lift(*tw.dims, tw.n_kept, tw.c, tw.n_int, ptr(depth), ptr(ctx), tw.D,
                                                 tw.fH * tw.fW, ptr(tw.perm_stale), ptr(tw.geom), ptr(tw.starts),
                                                 ptr(tw.lengths), ptr(out), ptr(ws), nbytes, tw.stream),
                 [out], ws, pattern, nbytes)[0]


def lift_rows_twin(tw, depth, ctx, out, form=None, nbytes=None, counts=None):
    L = _C.lib()
    need = L.bevb200_bev_pool_dev_workspace_bytes(tw.cap, tw.c)
    ws, pattern = workspace(need, tw.dev)
    counts = tw.counts if counts is None else counts
    fn = lambda: L.bevb200_bev_pool_lift_dev(*tw.dims, tw.cap, tw.c, ptr(depth), ptr(ctx), tw.D, tw.fH * tw.fW,
                                             ptr(tw.perm_stale), ptr(tw.geom), ptr(tw.starts), ptr(tw.lengths),
                                             _C.ptr(counts), None if form is None else ptr(form) + 4, ptr(out),
                                             ptr(ws), need if nbytes is None else nbytes, tw.stream)
    if nbytes is not None:
        return fn
    return twice(fn, [out], ws, pattern, need)[0]


def lift_bwd_host(tw, depth, ctx, dd, dc):
    L = _C.lib()
    nbytes = L.bevb200_bev_pool_lift_backward_workspace_bytes(tw.cap, tw.c)
    ws, pattern = workspace(nbytes, tw.dev)
    return twice(lambda: L.bevb200_bev_pool_lift_backward(*tw.dims, tw.n_kept, tw.cap, tw.c, tw.n_int, ptr(tw.G),
                                                          ptr(depth), ptr(ctx), tw.D, tw.fH * tw.fW, ptr(tw.perm),
                                                          ptr(tw.geom), ptr(tw.starts), ptr(tw.lengths), ptr(dd),
                                                          ptr(dc), ptr(ws), nbytes, tw.stream),
                 [dd, dc], ws, pattern, nbytes)


def lift_bwd_twin(tw, depth, ctx, dd, dc, form=None, nbytes=None):
    L = _C.lib()
    need = L.bevb200_bev_pool_lift_backward_dev_workspace_bytes(tw.cap, tw.c)
    ws, pattern = workspace(need, tw.dev)
    fn = lambda: L.bevb200_bev_pool_lift_backward_dev(*tw.dims, tw.cap, tw.c, ptr(tw.G), ptr(depth), ptr(ctx), tw.D,
                                                      tw.fH * tw.fW, ptr(tw.perm), ptr(tw.geom), ptr(tw.starts),
                                                      ptr(tw.lengths), ptr(tw.counts),
                                                      None if form is None else ptr(form) + 4, ptr(dd), ptr(dc),
                                                      ptr(ws), need if nbytes is None else nbytes, tw.stream)
    if nbytes is not None:
        return fn
    return twice(fn, [dd, dc], ws, pattern, need)


def check_lift_float64(tw, out, dd, dc, what):
    """forward within (L + 1) * 2^-24 * sum|d * ctx|; gradients within 1e-5 * max|gold|; dropped points ddepth == 0
    and pixels without a kept point dctx == 0, exactly"""
    shell = tw.plan_shell()
    check_sums(out, *lift_reference(shell, tw.depth, tw.ctx), 1, what)
    assert bool((dd.view(-1)[tw.dropped] == 0).all()), "%s: ddepth of a dropped point is not 0" % what
    assert bool((dc.view(-1, tw.c)[tw.empty_px] == 0).all()), "%s: dctx of a pixel without a kept point" % what
    if tw.n_kept >= 32 and tw.n_int:
        # the gradient bound is relative to max|gold|: with a handful of points that maximum is one C-long dot
        # product, cancellation included, and the bit-equality with the host-count call is the check there
        gd, gc = gold64(shell, tw.depth, tw.ctx, tw.G)
        assert_close(dd, gd)
        assert_close(dc, gc)
    elif not (tw.n_kept and tw.n_int):
        assert not bool(dd.any()) and not bool(dc.any())


@pytest.mark.parametrize("c,n", [(c, n) for c in TUNED for n in counts_at(c, lift=True)])
def test_lift_row_twins_at_range_boundaries(cuda, c, n):
    """bevb200_bev_pool_lift_dev (status word NULL and ROWS) and _lift_backward_dev against the host-count row lift
    and float64, at every capacity and at B*D = 1 and 2; NaN depth at dropped points and NaN context at pixels
    without a kept point"""
    for i, cap in enumerate(capacities(n)):
        for B in (1, 2):
            lay = LAYOUTS[(i + B + n) % len(LAYOUTS)]
            tw = Twin(cuda, TwinTables(n, cap, c, lay, seed=n + cap + B, B=B, lift=True), lift=True)
            what = "lift rows twin C=%d n=%d cap=%d B=%d %s" % (c, n, cap, B, lay)
            out = torch.empty(*tw.dims, c, device=cuda)
            want = lift_rows_host(tw, tw.depth_nan, tw.ctx_nan, out)
            for form in (None, status(ROWS, cuda)):
                assert same(lift_rows_twin(tw, tw.depth_nan, tw.ctx_nan, out, form), want), what
            dd, dc = torch.empty_like(tw.depth), torch.empty_like(tw.ctx)
            wd, wc = lift_bwd_host(tw, tw.depth_nan, tw.ctx_nan, dd, dc)
            for form in (None, status(ROWS, cuda)):
                gd, gc = lift_bwd_twin(tw, tw.depth_nan, tw.ctx_nan, dd, dc, form)
                assert same(gd, wd) and same(gc, wc), what
            check_lift_float64(tw, want, wd, wc, what)


# ---- the column lift
def col_buffers(tw, max_segments, seg, rng):
    """column tables of a sync-free plan: seg_key / seg_mask / seg_slot of max_segments records + TAIL canary
    records, holding stale copies of real records; col_begin and interval_slot_begin of stale in-bounds values"""
    dev = tw.dev
    key, mask = stale_segments(seg["seg_key"].cpu().numpy(), seg["seg_mask"].cpu().numpy(), seg["n"],
                               max_segments, rng)
    canary64 = np.full(TAIL, 0x5A5A5A5A5A5A5A5A, np.int64)
    out = dict(seg_key=t(np.concatenate([key, canary64])).to(dev),
               seg_mask=t(np.concatenate([mask, canary64])).to(dev),
               seg_slot=t(np.concatenate([rng.integers(0, max_segments, max_segments),
                                          np.full(TAIL, 0x5A5A5A5A)]).astype(np.int32)).to(dev),
               col_begin=torch.zeros(tw.cams * tw.fW + 1, dtype=torch.int32, device=dev),
               ival_begin=t(rng.integers(0, max(seg["n"], 1), tw.cap + 1).astype(np.int32)).to(dev),
               status=status(COLUMNS, dev))
    out["tails"] = [out[k][max_segments:].clone() for k in ("seg_key", "seg_mask", "seg_slot")]
    return out


def host_prepare(tw):
    """bevb200_bev_pool_lift_prepare on the tables cut to the counts"""
    L = _C.lib()
    dev = tw.dev
    i32 = dict(dtype=torch.int32, device=dev)
    m = max(tw.n_kept, 1)
    seg = dict(col_begin=torch.empty(tw.cams * tw.fW + 1, **i32), seg_key=torch.empty(m, dtype=torch.int64, device=dev),
               seg_mask=torch.empty(m, dtype=torch.int64, device=dev), seg_slot=torch.empty(m, **i32),
               ival_begin=torch.empty(tw.n_int + 1, **i32))
    n_seg = torch.zeros(1, **i32)
    ws = torch.empty(L.bevb200_bev_pool_lift_prepare_workspace_bytes(tw.n_kept), dtype=torch.uint8, device=dev)
    rc = L.bevb200_bev_pool_lift_prepare(ptr(tw.perm_stale), ptr(tw.starts), tw.n_kept, tw.n_int, tw.cams, tw.D, tw.fH,
                                         tw.fW, ptr(seg["col_begin"]), ptr(seg["seg_key"]), ptr(seg["seg_mask"]),
                                         ptr(seg["seg_slot"]), ptr(seg["ival_begin"]), ptr(n_seg), ptr(ws), ws.numel(),
                                         tw.stream)
    assert rc == 0, L.bevb200_last_error()
    seg["n"] = int(n_seg.item())
    return seg


def prepare_twin(tw, sg, max_segments, nbytes=None, counts=None, form=True):
    L = _C.lib()
    need = L.bevb200_bev_pool_lift_prepare_dev_workspace_bytes(tw.cap, min(max(max_segments, 1), tw.cap))
    ws = torch.empty(need + CANARY, dtype=torch.uint8, device=tw.dev)
    ws[need:] = 0xA5
    counts = tw.counts if counts is None else counts
    fn = lambda: L.bevb200_bev_pool_lift_prepare_dev(
        ptr(tw.perm_stale), ptr(tw.starts), _C.ptr(counts), tw.cap, max_segments, tw.cams, tw.D, tw.fH, tw.fW,
        ptr(sg["col_begin"]), ptr(sg["seg_key"]), ptr(sg["seg_mask"]), ptr(sg["seg_slot"]), ptr(sg["ival_begin"]),
        ptr(sg["status"]), ptr(sg["status"]) + 4 if form else None, ptr(ws), need if nbytes is None else nbytes,
        tw.stream)
    if nbytes is not None:
        return fn
    rc = fn()
    torch.cuda.synchronize()
    assert rc == 0, L.bevb200_last_error()
    assert bool((ws[need:] == 0xA5).all()), "workspace canary overwritten"


def check_prepare(tw, sg, host, max_segments):
    """n_segments and lift_form exactly; the column tables equal the host-count prepare when the count fits; nothing
    written past max_segments"""
    n_seg, form = (int(v) for v in sg["status"].tolist())
    assert n_seg == host["n"], (n_seg, host["n"])
    fits = host["n"] <= max_segments
    assert form == (COLUMNS if fits else ROWS)
    for k, tail in zip(("seg_key", "seg_mask", "seg_slot"), sg["tails"]):
        assert torch.equal(sg[k][max_segments:], tail), "%s written past max_segments" % k
    if fits:
        n = host["n"]
        assert torch.equal(sg["col_begin"], host["col_begin"])
        assert torch.equal(sg["seg_key"][:n], host["seg_key"][:n]) and torch.equal(sg["seg_mask"][:n], host["seg_mask"][:n])
        assert torch.equal(sg["seg_slot"][:n], host["seg_slot"][:n])
        assert torch.equal(sg["ival_begin"][:tw.n_int + 1], host["ival_begin"][:tw.n_int + 1])
    return fits


def columns_host(tw, host, depth, ctx, out, dd, dc):
    L = _C.lib()
    n_seg = host["n"]
    nb = L.bevb200_bev_pool_lift_columns_workspace_bytes(n_seg, tw.n_int, tw.c)
    ws, pattern = workspace(nb, tw.dev)
    (fwd,) = twice(lambda: L.bevb200_bev_pool_lift_columns(
        *tw.dims, tw.n_kept, tw.c, tw.n_int, ptr(depth), ptr(ctx), tw.cams, tw.D, tw.fH, tw.fW, ptr(tw.geom),
        ptr(tw.starts), ptr(host["col_begin"]), ptr(host["seg_key"]), ptr(host["seg_mask"]), ptr(host["seg_slot"]),
        ptr(host["ival_begin"]), n_seg, ptr(out), ptr(ws), nb, tw.stream), [out], ws, pattern, nb)
    nb = L.bevb200_bev_pool_lift_columns_backward_workspace_bytes(n_seg, tw.n_int, tw.c)
    ws, pattern = workspace(nb, tw.dev)
    gd, gc = twice(lambda: L.bevb200_bev_pool_lift_columns_backward(
        *tw.dims, tw.n_kept, tw.c, tw.n_int, ptr(tw.G), ptr(depth), ptr(ctx), tw.cams, tw.D, tw.fH, tw.fW,
        ptr(tw.geom), ptr(tw.starts), ptr(host["col_begin"]), ptr(host["seg_key"]), ptr(host["seg_mask"]), n_seg,
        ptr(dd), ptr(dc), ptr(ws), nb, tw.stream), [dd, dc], ws, pattern, nb)
    return fwd, gd, gc


def columns_twin(tw, sg, max_segments, depth, ctx, out, nbytes=None, form=True, counts=None):
    L = _C.lib()
    need = L.bevb200_bev_pool_lift_columns_dev_workspace_bytes(max_segments, tw.cap, tw.c)
    ws, pattern = workspace(need, tw.dev)
    counts = tw.counts if counts is None else counts
    fn = lambda: L.bevb200_bev_pool_lift_columns_dev(
        *tw.dims, tw.cap, tw.c, ptr(depth), ptr(ctx), tw.cams, tw.D, tw.fH, tw.fW, ptr(tw.geom), ptr(tw.starts),
        ptr(sg["col_begin"]), ptr(sg["seg_key"]), ptr(sg["seg_mask"]), ptr(sg["seg_slot"]), ptr(sg["ival_begin"]),
        max_segments, _C.ptr(counts), ptr(sg["status"]) + 4 if form else None, ptr(out), ptr(ws),
        need if nbytes is None else nbytes, tw.stream)
    if nbytes is not None:
        return fn
    return twice(fn, [out], ws, pattern, need)[0]


def columns_bwd_twin(tw, sg, max_segments, depth, ctx, dd, dc, nbytes=None, form=True, counts=None):
    L = _C.lib()
    need = L.bevb200_bev_pool_lift_columns_backward_dev_workspace_bytes(max_segments, tw.c)
    ws, pattern = workspace(need, tw.dev)
    counts = tw.counts if counts is None else counts
    fn = lambda: L.bevb200_bev_pool_lift_columns_backward_dev(
        *tw.dims, tw.cap, tw.c, ptr(tw.G), ptr(depth), ptr(ctx), tw.cams, tw.D, tw.fH, tw.fW, ptr(tw.geom),
        ptr(tw.starts), ptr(sg["col_begin"]), ptr(sg["seg_key"]), ptr(sg["seg_mask"]), max_segments, _C.ptr(counts),
        ptr(sg["status"]), ptr(sg["status"]) + 4 if form else None, ptr(dd), ptr(dc), ptr(ws),
        need if nbytes is None else nbytes, tw.stream)
    if nbytes is not None:
        return fn
    return twice(fn, [dd, dc], ws, pattern, need)


def column_case(cuda, c, n, cap, B, lay):
    tw = Twin(cuda, TwinTables(n, cap, c, lay, seed=n + cap + B, B=B, lift=True), lift=True)
    host = host_prepare(tw)
    sg = col_buffers(tw, cap, host, np.random.default_rng(n + cap))
    prepare_twin(tw, sg, cap)
    assert check_prepare(tw, sg, host, cap)
    return tw, host, sg


@pytest.mark.parametrize("c,n", [(c, n) for c in TUNED for n in counts_at(c, lift=True)])
def test_lift_column_twins_at_range_boundaries(cuda, c, n):
    """bevb200_bev_pool_lift_prepare_dev (cap = capacity) + _lift_columns_dev + _lift_columns_backward_dev against the
    host-count prepare / columns / columns backward and float64, at every capacity and at B*D = 1 and 2"""
    for i, cap in enumerate(capacities(n)):
        for B in (1, 2):
            lay = LAYOUTS[(i + B + n) % len(LAYOUTS)]
            tw, host, sg = column_case(cuda, c, n, cap, B, lay)
            what = "lift columns twin C=%d n=%d cap=%d B=%d %s" % (c, n, cap, B, lay)
            out = torch.empty(*tw.dims, c, device=cuda)
            dd, dc = torch.empty_like(tw.depth), torch.empty_like(tw.ctx)
            want, wd, wc = columns_host(tw, host, tw.depth_nan, tw.ctx_nan, out, dd, dc)
            assert same(columns_twin(tw, sg, cap, tw.depth_nan, tw.ctx_nan, out), want), what
            gd, gc = columns_bwd_twin(tw, sg, cap, tw.depth_nan, tw.ctx_nan, dd, dc)
            assert same(gd, wd) and same(gc, wc), what
            check_lift_float64(tw, want, wd, wc, what)


@pytest.mark.parametrize("c", [16, 80, 256])
def test_lift_twins_with_points_but_no_interval(cuda, c):
    """n_kept > 0 with n_intervals == 0: both lift forms give a zero grid and zero gradients"""
    for B in (1, 2):
        tw = Twin(cuda, TwinTables(3000, 4096, c, "hot", seed=B, B=B, lift=True, no_intervals=True), lift=True)
        out = torch.empty(*tw.dims, c, device=cuda)
        assert not bool(lift_rows_twin(tw, tw.depth_nan, tw.ctx_nan, out, status(ROWS, cuda)).any())
        dd, dc = torch.empty_like(tw.depth), torch.empty_like(tw.ctx)
        for g in lift_bwd_twin(tw, tw.depth_nan, tw.ctx_nan, dd, dc, status(ROWS, cuda)):
            assert not bool(g.any())
        # column tables of an empty plan (prepare at n_kept = 0), read under counts {n_kept, 0}
        sg = col_buffers(tw, 64, dict(seg_key=torch.zeros(1), seg_mask=torch.zeros(1), n=0), np.random.default_rng(B))
        prepare_twin(tw, sg, 64, counts=torch.zeros(2, dtype=torch.int32, device=cuda))
        assert sg["status"].tolist() == [0, COLUMNS]
        got = columns_twin(tw, sg, 64, tw.depth_nan, tw.ctx_nan, out)
        assert not bool(got.any()) and not bool(torch.signbit(got).any())
        for g in columns_bwd_twin(tw, sg, 64, tw.depth_nan, tw.ctx_nan, dd, dc):
            assert not bool(g.any())


# ---- the form the status word does not name
@pytest.mark.parametrize("B,n", [(1, 5000), (2, 5000), (1, 0), (2, 0)])
def test_lift_twin_of_the_other_form_writes_nothing(cuda, B, n):
    """each lift twin with the status word naming the other form leaves every byte of its NaN-filled outputs: B*D = 1
    (the kernels would zero-fill), B*D > 1 (a memset would) and an empty grid"""
    c = 80
    tw, host, sg = column_case(cuda, c, n, n + 96, B, "hot")
    rows_word = status(ROWS, cuda)
    cols_word = sg["status"].clone()
    sg_rows = dict(sg, status=rows_word)

    def untouched(fn, outs):
        for o in outs:
            o.fill_(float("nan"))
        torch.cuda.synchronize()
        rc = fn()
        torch.cuda.synchronize()
        assert rc == 0, _C.lib().bevb200_last_error()
        for o in outs:
            assert bool(torch.isnan(o).all()), "the twin of the form not named wrote its output"

    out = torch.empty(*tw.dims, c, device=cuda)
    dd, dc = torch.empty_like(tw.depth), torch.empty_like(tw.ctx)
    L = _C.lib()
    need = L.bevb200_bev_pool_dev_workspace_bytes(tw.cap, c)
    untouched(lift_rows_twin(tw, tw.depth, tw.ctx, out, cols_word, nbytes=need), [out])
    need = L.bevb200_bev_pool_lift_backward_dev_workspace_bytes(tw.cap, c)
    untouched(lift_bwd_twin(tw, tw.depth, tw.ctx, dd, dc, cols_word, nbytes=need), [dd, dc])
    need = L.bevb200_bev_pool_lift_columns_dev_workspace_bytes(tw.cap, tw.cap, c)
    untouched(columns_twin(tw, sg_rows, tw.cap, tw.depth, tw.ctx, out, nbytes=need), [out])
    need = L.bevb200_bev_pool_lift_columns_backward_dev_workspace_bytes(tw.cap, c)
    untouched(columns_bwd_twin(tw, sg_rows, tw.cap, tw.depth, tw.ctx, dd, dc, nbytes=need), [dd, dc])


# ---- the column-table prepare at caps around the segment count
@pytest.mark.parametrize("cfg_name,batch,seed", [("tiny", 1, 50), ("tiny", 2, 51), ("C2", 1, 52)])
def test_prepare_twin_caps_around_the_segment_count(cuda, cfg_name, batch, seed):
    """bevb200_bev_pool_lift_prepare_dev on a real host plan's perm / starts with stale entries past the counts, at
    max_segments 1, n_seg - 1, n_seg, n_seg + 1 and the capacity: n_segments and lift_form exactly, the column tables
    of the host-count prepare when the count fits, and nothing written past max_segments"""
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS[cfg_name]
    fr = frustum(cuda, cfg)
    hp = host_plan(cfg, rig(cuda, cfg, batch, seed), fr)
    ht = hp.tables
    rng = np.random.default_rng(seed)
    cap = ht.n_total
    n, n_int = ht.n_kept, ht.n_intervals
    assert 0 < n < cap
    tw = types.SimpleNamespace(dev=cuda, cap=cap, n_kept=n, n_int=n_int, stream=_C.current_stream(cuda),
                               cams=batch * cfg["n_cam"], D=fr.shape[0], fH=fr.shape[1], fW=fr.shape[2])
    perm = ht.perm.clone()
    perm[n:] = ht.perm[torch.from_numpy(rng.integers(0, n, cap - n)).to(cuda)]
    starts = torch.from_numpy(rng.integers(0, n, cap).astype(np.int32)).to(cuda)
    starts[:n_int] = ht.starts
    tw.perm_stale, tw.starts = perm, starts
    tw.counts = torch.tensor([n, n_int], dtype=torch.int32, device=cuda)
    tw.perm = ht.perm
    host = host_prepare(tw)
    n_seg = host["n"]
    caps = caps_around(n_seg, cap)
    assert {1, n_seg - 1, n_seg, n_seg + 1, cap} <= set(caps)
    for max_segments in caps:
        sg = col_buffers(tw, max_segments, host, rng)
        prepare_twin(tw, sg, max_segments)
        fits = check_prepare(tw, sg, host, max_segments)
        assert fits == (max_segments >= n_seg)
        # again over the tables the first call left: a rebuild in place gives the same
        sg["status"].fill_(-7)
        prepare_twin(tw, sg, max_segments)
        assert check_prepare(tw, sg, host, max_segments) == fits


# ---- refusals
def test_twin_refusals_leave_outputs_and_tables_untouched(cuda):
    """every twin given a workspace one byte short of what it needs, a null counts_dev, the column twins a null
    lift_form, and max_segments outside [1, capacity]: the error code, NaN outputs and the tables bit-unchanged.
    The column-forward and lift-backward queries report SLACK bytes more than the call needs."""
    c, n, cap = 80, 5000, 6000
    tw, host, sg = column_case(cuda, c, n, cap, 2, "hot")
    tp = Twin(cuda, TwinTables(n, cap, c, "hot", seed=3, B=2))
    L = _C.lib()
    tables = [tw.perm_stale, tw.perm, tw.geom, tw.starts, tw.lengths, tw.counts, sg["col_begin"], sg["seg_key"],
              sg["seg_mask"], sg["seg_slot"], sg["ival_begin"], sg["status"], tp.perm_stale, tp.geom, tp.starts,
              tp.lengths, tp.counts]
    before = [x.clone() for x in tables]
    out = torch.empty(*tw.dims, c, device=cuda)
    dd, dc = torch.empty_like(tw.depth), torch.empty_like(tw.ctx)
    xg = torch.empty(cap, c, device=cuda)
    null = torch.empty(0)
    null_counts = types.SimpleNamespace(data_ptr=lambda: 0)
    need_pool = L.bevb200_bev_pool_dev_workspace_bytes(cap, c)
    need_cols = L.bevb200_bev_pool_lift_columns_dev_workspace_bytes(cap, cap, c) - SLACK
    need_cbwd = L.bevb200_bev_pool_lift_columns_backward_dev_workspace_bytes(cap, c) - SLACK
    need_rbwd = L.bevb200_bev_pool_lift_backward_dev_workspace_bytes(cap, c) - SLACK
    need_prep = L.bevb200_bev_pool_lift_prepare_dev_workspace_bytes(cap, cap)
    rows = status(ROWS, cuda)
    cases = [
        ("pool short", EWORKSPACE, pool_twin(tp, tp.x, out, nbytes=need_pool - 1), [out]),
        ("pool null counts", EINVAL, pool_twin(tp, tp.x, out, nbytes=need_pool, counts=null_counts), [out]),
        ("lift rows short", EWORKSPACE, lift_rows_twin(tw, tw.depth, tw.ctx, out, rows, nbytes=need_pool - 1), [out]),
        ("lift rows null counts", EINVAL,
         lift_rows_twin(tw, tw.depth, tw.ctx, out, rows, nbytes=need_pool, counts=null_counts), [out]),
        ("lift rows bwd short", EWORKSPACE, lift_bwd_twin(tw, tw.depth, tw.ctx, dd, dc, rows, nbytes=need_rbwd - 1),
         [dd, dc]),
        ("columns short", EWORKSPACE, columns_twin(tw, sg, cap, tw.depth, tw.ctx, out, nbytes=need_cols - 1), [out]),
        ("columns null form", EINVAL,
         columns_twin(tw, sg, cap, tw.depth, tw.ctx, out, nbytes=need_cols, form=False), [out]),
        ("columns null counts", EINVAL,
         columns_twin(tw, sg, cap, tw.depth, tw.ctx, out, nbytes=need_cols, counts=null_counts), [out]),
        ("columns cap 0", EINVAL, columns_twin(tw, sg, 0, tw.depth, tw.ctx, out, nbytes=need_cols), [out]),
        ("columns cap above capacity", EINVAL,
         columns_twin(tw, sg, cap + 1, tw.depth, tw.ctx, out, nbytes=need_cols + 4096), [out]),
        ("columns bwd short", EWORKSPACE,
         columns_bwd_twin(tw, sg, cap, tw.depth, tw.ctx, dd, dc, nbytes=need_cbwd - 1), [dd, dc]),
        ("columns bwd null form", EINVAL,
         columns_bwd_twin(tw, sg, cap, tw.depth, tw.ctx, dd, dc, nbytes=need_cbwd, form=False), [dd, dc]),
        ("columns bwd null counts", EINVAL,
         columns_bwd_twin(tw, sg, cap, tw.depth, tw.ctx, dd, dc, nbytes=need_cbwd, counts=null_counts), [dd, dc]),
        ("columns bwd cap 0", EINVAL, columns_bwd_twin(tw, sg, 0, tw.depth, tw.ctx, dd, dc, nbytes=need_cbwd),
         [dd, dc]),
        ("columns bwd cap above capacity", EINVAL,
         columns_bwd_twin(tw, sg, cap + 1, tw.depth, tw.ctx, dd, dc, nbytes=need_cbwd + 4096), [dd, dc]),
        ("prepare short", EWORKSPACE, prepare_twin(tw, sg, cap, nbytes=need_prep - 1), []),
        ("prepare null counts", EINVAL, prepare_twin(tw, sg, cap, nbytes=need_prep, counts=null_counts), []),
        ("prepare null form", EINVAL, prepare_twin(tw, sg, cap, nbytes=need_prep, form=False), []),
        ("prepare cap 0", EINVAL, prepare_twin(tw, sg, 0, nbytes=need_prep), []),
        ("prepare cap above capacity", EINVAL, prepare_twin(tw, sg, cap + 1, nbytes=need_prep), []),
    ]
    # the pooling backward twin takes no workspace: null counts only
    cases.append(("grad null counts", EINVAL,
                  lambda: L.bevb200_bev_pool_grad_perm_dev(*tp.dims, cap, c, ptr(tp.G), ptr(tp.perm), ptr(tp.geom),
                                                           ptr(tp.starts), ptr(tp.lengths), None, ptr(xg), tp.stream),
                  [xg]))
    cases.append(("lift rows bwd null counts", EINVAL,
                  lambda: L.bevb200_bev_pool_lift_backward_dev(*tw.dims, cap, c, ptr(tw.G), ptr(tw.depth), ptr(tw.ctx),
                                                               tw.D, tw.fH * tw.fW, ptr(tw.perm), ptr(tw.geom),
                                                               ptr(tw.starts), ptr(tw.lengths), None, ptr(rows) + 4,
                                                               ptr(dd), ptr(dc), ptr(null), 1 << 30, tw.stream),
                  [dd, dc]))
    for what, code, fn, outs in cases:
        for o in outs:
            o.fill_(float("nan"))
        torch.cuda.synchronize()
        rc = fn()
        torch.cuda.synchronize()
        assert rc == code, (what, rc, L.bevb200_last_error())
        for o in outs:
            assert bool(torch.isnan(o).all()), "%s: output written by a refused call" % what
        for a, b in zip(before, tables):
            assert torch.equal(a, b), "%s: a table changed under a refused call" % what


# ---------------------------------------------------------------------------------------------------- part B
def cut_case(host, x, C):
    """the dispatch test's Case over a host-count plan's tables (for pool_reference)"""
    ht = host.tables
    case = Case.__new__(Case)
    case.dims, case.c, case.n, case.n_int, case.n_total = ht.dims, C, ht.n_kept, ht.n_intervals, ht.n_total
    case.starts_np, case.lengths_np = ht.starts.cpu().numpy(), ht.lengths.cpu().numpy()
    case.geom_np, case.perm_np = ht.geom.cpu().numpy(), ht.perm.cpu().numpy()
    case.x = x.reshape(-1, C)
    return case


def pool_step(plan, x, G):
    xr = x.detach().clone().requires_grad_(True)
    out = plan.pool(xr)
    (xg,) = torch.autograd.grad(out, (xr,), G)
    return out.detach(), xg


def check_lift_against(host, dev, depth, ctx, G, what, rows=False):
    """dev.lift_pool forward and gradients bit-equal to the host-count plan's form (columns, or the row API), and
    within float64; zero ddepth at dropped points and zero dctx at pixels with no kept point"""
    want = host_rows(host, depth, ctx, G) if rows else lift_step(host, depth, ctx, G)
    got = lift_step(dev, depth, ctx, G)
    for a, b in zip(want, got):
        assert same(a, b), what
    out, dd, dc = got
    ht = host.tables
    if ht.n_kept == 0:
        assert not bool(out.any()) and not bool(dd.any()) and not bool(dc.any())
        return
    check_sums(out, *lift_reference(host, depth, ctx), 1, what)
    gd, gc = gold64(host, depth, ctx, G)
    assert_close(dd, gd)
    assert_close(dc, gc)
    del gd, gc
    B, N, D, fH, fW = depth.shape
    assert bool((dd.view(-1)[ht.perm[ht.n_kept:].long()] == 0).all()), what
    kept = torch.zeros(depth.numel(), dtype=torch.bool, device=depth.device)
    kept[ht.perm[:ht.n_kept].long()] = True
    empty_px = ~kept.view(B * N, D, fH * fW).any(1).view(-1)
    assert bool((dc.view(-1, dc.shape[-1])[empty_px] == 0).all()), what


@pytest.mark.parametrize("C", TUNED)
@pytest.mark.parametrize("batch", [1, 2])
def test_plan_both_lift_forms_at_every_width(cuda, C, batch):
    """the column form under the default cap and the row form forced by max_segments = n_seg - 1"""
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["tiny"]
    fr = frustum(cuda, cfg)
    r = rig(cuda, cfg, batch, seed=60 + C + batch)
    host, dev = plans(cuda, cfg, r, fr, max_segments=None)
    depth, ctx, G = inputs(cuda, dev, fr, C, seed=C)
    assert int(dev.tables.lift_form) == COLUMNS
    check_lift_against(host, dev, depth, ctx, G, "plan columns C=%d B=%d" % (C, batch))
    n_seg = int(dev.tables.n_segments)
    _, rows = plans(cuda, cfg, r, fr, max_segments=n_seg - 1)
    assert int(rows.tables.lift_form) == ROWS and int(rows.tables.n_segments) == n_seg
    check_lift_against(host, rows, depth, ctx, G, "plan rows C=%d B=%d" % (C, batch), rows=True)


@pytest.mark.parametrize("fH", FEATURE_HEIGHTS)
def test_plan_feature_heights_around_the_pixel_mask(cuda, fH):
    """fH = 64: the top bit of the segment mask is live and the form is columns; fH = 65: no column tables, rows"""
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["tiny"]
    fr = frustum(cuda, cfg, (fH, 8))
    host, dev = plans(cuda, cfg, rig(cuda, cfg, 1, seed=70 + fH), fr, max_segments=None)
    assert_tables_equal(host, dev)
    depth, ctx, G = inputs(cuda, dev, fr, 80, seed=fH)
    if fH > 64:
        assert dev.max_segments == 0 and int(dev.tables.lift_form) == ROWS
    else:
        assert assert_column_tables_equal(host, dev)
        if fH == 64:
            mask = dev._seg["seg_mask"][:int(dev.tables.n_segments)]
            assert bool((mask < 0).any()), "no segment covers pixel row 63"
    check_lift_against(host, dev, depth, ctx, G, "plan fH=%d" % fH)


def sequence(cuda, cfg, batch, fr):
    """[(name, rig)]: augmented draw A, every point off the grid, about half the points shifted off it, a draw over
    the cap, draw A again; and the cap (max_segments) that the draws other than the over-cap one fit"""
    B, N, D, fH, fW = batch, cfg["n_cam"], fr.shape[0], fr.shape[1], fr.shape[2]
    n_seg = lambda r: host_plan(cfg, r, fr)._lift_tables(B * N, D, fH, fW)[5]
    shift = torch.tensor([cfg["xbound"][1] / 2, 0.0, 0.0], device=cuda)
    draws = [(rig(cuda, cfg, batch, seed=s), rig(cuda, cfg, batch, seed=s, shift=shift)) for s in range(80, 88)]
    segs = [(n_seg(a), n_seg(h)) for a, h in draws]
    over = max(range(len(draws)), key=lambda i: segs[i][0])
    pick = min((i for i in range(len(draws)) if i != over), key=lambda i: max(segs[i]))
    a, half = draws[pick]
    cap = max(segs[pick])
    assert segs[over][0] > cap
    seq = [("A", a), ("off", rig(cuda, cfg, batch, seed=80, shift=1000.0)), ("half", half), ("over", draws[over][0]),
           ("A", a)]
    return seq, cap


@pytest.mark.parametrize("batch", [1, 2])
def test_plan_rebuild_sequence_in_place(cuda, batch):
    """one plan rebuilt through draw A, an empty grid, a half-empty grid, a draw over the cap and draw A again, with
    no allocation between: tables, pool and its gradient, lift_pool and both gradients after every rebuild_"""
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["tiny"]
    fr = frustum(cuda, cfg)
    seq, cap = sequence(cuda, cfg, batch, fr)
    _, plan = plans(cuda, cfg, seq[0][1], fr, max_segments=cap)
    depth, ctx, G = inputs(cuda, plan, fr, 64, seed=batch)
    x = (depth.unsqueeze(-1) * ctx.unsqueeze(2)).contiguous()
    ptrs = [plan.tables.perm.data_ptr(), plan._seg["seg_key"].data_ptr()]
    n_half = None
    for name, r in seq:
        plan.rebuild_(*calib(r))
        host = host_plan(cfg, r, fr)
        what = "plan rebuild %s B=%d" % (name, batch)
        assert [plan.tables.perm.data_ptr(), plan._seg["seg_key"].data_ptr()] == ptrs
        assert_tables_equal(host, plan)
        fits = assert_column_tables_equal(host, plan)
        assert fits == (name != "over"), what
        if name == "half":
            n_half = host.tables.n_kept
        for a, b in zip(pool_step(host, x, G), pool_step(plan, x, G)):
            assert same(a, b), what
        out, xg = pool_step(plan, x, G)
        check_sums(out, *pool_reference(cut_case(host, x, 64)), 0, what)
        check_lift_against(host, plan, depth, ctx, G, what, rows=not fits)
    assert 0 < n_half < host.tables.n_kept


def run_graph_sequence(cuda, cfg, batch, fr, lift):
    seq, cap = sequence(cuda, cfg, batch, fr)
    _, plan = plans(cuda, cfg, seq[0][1], fr, max_segments=cap)
    static = [v.clone() for v in calib(seq[0][1])]
    C = 64
    depth, ctx, G = inputs(cuda, plan, fr, C, seed=5)
    if lift:
        sd, sc = depth.clone().requires_grad_(True), ctx.clone().requires_grad_(True)
        args = (sd, sc)
    else:
        sx = (depth.unsqueeze(-1) * ctx.unsqueeze(2)).contiguous().requires_grad_(True)
        args = (sx,)

    def step():
        plan.rebuild_(*static)
        out = plan.lift_pool(sd, sc) if lift else plan.pool(sx)
        return (out,) + torch.autograd.grad(out, args, G)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        res = step()
    for name, r in seq[1:] + seq[:1]:
        with torch.no_grad():
            for dst, src in zip(static, calib(r)):
                dst.copy_(src)
        graph.replay()
        torch.cuda.synchronize()
        host = host_plan(cfg, r, fr)
        if lift:
            fits = name != "over"
            want = lift_step(host, depth, ctx, G) if fits else host_rows(host, depth, ctx, G)
        else:
            want = pool_step(host, args[0].detach(), G)
        for a, b in zip(want, res):
            assert same(a, b.detach()), "graph replay %s" % name


def test_plan_graph_of_rebuild_and_pool(cuda):
    """rebuild_ + pool + backward captured once and replayed over the sequence (empty grid included)"""
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["tiny"]
    run_graph_sequence(cuda, cfg, 1, frustum(cuda, cfg), lift=False)


def test_plan_graph_of_rebuild_and_lift_at_batch_2(cuda):
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["tiny"]
    run_graph_sequence(cuda, cfg, 2, frustum(cuda, cfg), lift=True)


@pytest.mark.parametrize("cfg_name,batch", [("C2", 4), ("C5", 1)])
def test_plan_larger_configurations(cuda, cfg_name, batch):
    """C2 at B = 4 with one augmentation draw per sample, C5 at B = 1 (fH = 64): columns under the default cap, lift
    forward and gradients bit-equal to the host-count plan and within float64"""
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS[cfg_name]
    fr = frustum(cuda, cfg)
    r = rig(cuda, cfg, batch, seed=90)
    assert not torch.equal(r["post_rots"][0], r["post_rots"][-1]) or batch == 1
    host, dev = plans(cuda, cfg, r, fr, max_segments=None)
    assert int(dev.tables.lift_form) == COLUMNS
    assert_tables_equal(host, dev)
    depth, ctx, G = inputs(cuda, dev, fr, 80, seed=9)
    check_lift_against(host, dev, depth, ctx, G, "plan %s B=%d" % (cfg_name, batch))
    torch.cuda.empty_cache()


def test_plan_default_cap_holds_augmented_c5(cuda):
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["C5"]
    fr = frustum(cuda, cfg)
    _, plan = plans(cuda, cfg, rig(cuda, cfg, 1, seed=100), fr, max_segments=None)
    for seed in range(100, 103):
        plan.rebuild_(*calib(rig(cuda, cfg, 1, seed=seed)))
        assert int(plan.tables.lift_form) == COLUMNS, (seed, int(plan.tables.n_segments), plan.max_segments)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("batch", [1, 2])
def test_plan_nan_at_dropped_points(cuda, batch):
    """NaN depth at every dropped frustum point (lift_pool) and NaN rows of x at dropped points (pool): the outputs
    equal the run with zeros there bit for bit, and every gradient is finite"""
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["tiny"]
    fr = frustum(cuda, cfg)
    _, dev = plans(cuda, cfg, rig(cuda, cfg, batch, seed=110), fr, max_segments=None)
    t = dev.tables
    n = int(t.n_kept)
    assert 0 < n < t.n_total
    dropped = t.perm[n:].long()
    depth, ctx, G = inputs(cuda, dev, fr, 80, seed=110)
    depth.view(-1)[dropped] = 0.0
    dn = depth.clone()
    dn.view(-1)[dropped] = float("nan")
    for form_cap in (None, int(t.n_segments) - 1):
        plan = dev if form_cap is None else plans(cuda, cfg, rig(cuda, cfg, batch, seed=110), fr, form_cap)[1]
        for a, b in zip(lift_step(plan, depth, ctx, G), lift_step(plan, dn, ctx, G)):
            assert same(a, b)
            assert bool(torch.isfinite(b).all())
    x = (depth.unsqueeze(-1) * ctx.unsqueeze(2)).contiguous()
    xn = x.clone()
    xn.view(-1, 80)[dropped] = float("nan")
    (o0, g0), (o1, g1) = pool_step(dev, x, G), pool_step(dev, xn, G)
    assert same(o0, o1) and same(g0, g1) and bool(torch.isfinite(g1).all())
