"""GPU: sync-free BEV pooling plans (BEVPoolPlan.from_cameras(..., sync=False) + rebuild_) under seeded draws of the
reference's training augmentation.  Tables, pooling, the fused lift (column and row form) and every gradient are
compared bit for bit with a host-count plan built from the same calibration; the status word's fallback to the row
kernels, the empty and single-cell grids, CUDA-graph capture of rebuild_ + lift_pool + backward with new calibration
at every replay, and the refusals of rebuild_."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

KEYS = ("camera2lidar_rots", "camera2lidar_trans", "intrins", "post_rots", "post_trans", "extra_rots", "extra_trans")


def rig(cuda, cfg, batch, seed, shift=None):
    from bevfusion_b200 import synthetic as S
    r = {k: v.to(cuda) for k, v in S.augmented_rig(cfg["n_cam"], cfg["image_size"], batch, seed).items()}
    if shift is not None:
        r["camera2lidar_trans"] = r["camera2lidar_trans"] + shift
    return r


def calib(r):
    return [r[k] for k in KEYS]


def frustum(cuda, cfg, feature_size=None):
    from bevfusion_b200.vtransform import create_frustum
    return create_frustum(cfg["image_size"], feature_size or cfg["feature_size"], cfg["dbound"]).to(cuda)


ALL = 1 << 30      # a column-table cap no rig reaches (clamped to the plan's frustum points)


def host_plan(cfg, r, fr, bounds=None):
    from bevfusion_b200.bev_pool import BEVPoolPlan
    xb, yb, zb = bounds or (cfg["xbound"], cfg["ybound"], cfg["zbound"])
    c = calib(r)
    return BEVPoolPlan.from_cameras(fr, *c[:5], xb, yb, zb, c[5], c[6])


def plans(cuda, cfg, r, fr, max_segments=ALL, bounds=None):
    """(host-count plan, sync-free plan) of one calibration"""
    from bevfusion_b200.bev_pool import BEVPoolPlan
    xb, yb, zb = bounds or (cfg["xbound"], cfg["ybound"], cfg["zbound"])
    c = calib(r)
    dev = BEVPoolPlan.from_cameras(fr, *c[:5], xb, yb, zb, c[5], c[6], sync=False, max_segments=max_segments)
    return host_plan(cfg, r, fr, bounds), dev


def inputs(cuda, plan, fr, C, seed):
    B, N = plan.B, plan._cams[1]
    D, fH, fW = fr.shape[:3]
    g = torch.Generator(device=cuda).manual_seed(seed)
    depth = torch.softmax(torch.randn(B, N, D, fH, fW, generator=g, device=cuda), dim=2).contiguous()
    ctx = torch.randn(B, N, fH, fW, C, generator=g, device=cuda)
    G = torch.randn(*plan.tables.dims, C, generator=g, device=cuda)
    return depth, ctx, G


def lift_step(plan, depth, ctx, G):
    d = depth.detach().clone().requires_grad_(True)
    c = ctx.detach().clone().requires_grad_(True)
    out = plan.lift_pool(d, c)
    gd, gc = torch.autograd.grad(out, (d, c), G)
    return out.detach(), gd, gc


def host_rows(host, depth, ctx, G):
    """the row form of the host-count API: BEVB200_LIFT_VARIANT=rows forward, bevb200_bev_pool_lift_backward"""
    from bevfusion_b200 import _C
    from bevfusion_b200.bev_pool import _ws
    os.environ["BEVB200_LIFT_VARIANT"] = "rows"
    try:
        with torch.no_grad():
            out = host.lift_pool(depth, ctx)
    finally:
        del os.environ["BEVB200_LIFT_VARIANT"]
    t = host.tables
    B, N, D, fH, fW = depth.shape
    c = ctx.shape[-1]
    L = _C.lib()
    dd, dc = torch.empty_like(depth), torch.empty_like(ctx)
    ws = _ws(L.bevb200_bev_pool_lift_backward_workspace_bytes(t.n_total, c), depth.device)
    rc = L.bevb200_bev_pool_lift_backward(*t.dims, t.n_kept, t.n_total, c, t.n_intervals, _C.ptr(G), _C.ptr(depth),
                                          _C.ptr(ctx), D, fH * fW, _C.ptr(t.perm), _C.ptr(t.geom), _C.ptr(t.starts),
                                          _C.ptr(t.lengths), _C.ptr(dd), _C.ptr(dc), _C.ptr(ws), ws.numel(),
                                          _C.current_stream(depth.device))
    _C.check(rc, "bev_pool_lift_backward")
    return out, dd, dc


def same(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def assert_tables_equal(host, dev):
    h, d = host.tables, dev.tables
    n_kept, n_int = int(d.n_kept), int(d.n_intervals)
    assert (n_kept, n_int) == (h.n_kept, h.n_intervals)
    assert torch.equal(d.perm, h.perm) and torch.equal(d.ranks, h.ranks)
    assert torch.equal(d.geom[:n_kept], h.geom)
    assert torch.equal(d.starts[:n_int], h.starts) and torch.equal(d.lengths[:n_int], h.lengths)


def assert_column_tables_equal(host, dev):
    """the column tables, when the host count fits under the plan's cap (else the status word says rows)"""
    B, N, D, fH, fW = dev._cams
    col_begin, seg_key, seg_mask, seg_slot, ival_begin, n_seg = host._lift_tables(B * N, D, fH, fW)
    assert int(dev.tables.n_segments) == n_seg
    if n_seg > dev.max_segments:
        assert int(dev.tables.lift_form) == 1
        return False
    assert int(dev.tables.lift_form) == 0
    sg = dev._seg
    n_int = host.tables.n_intervals
    assert torch.equal(sg["col_begin"], col_begin)
    if n_seg:
        assert torch.equal(sg["seg_key"][:n_seg], seg_key) and torch.equal(sg["seg_mask"][:n_seg], seg_mask)
        assert torch.equal(sg["seg_slot"][:n_seg], seg_slot)
    assert torch.equal(sg["ival_begin"][:n_int + 1], ival_begin[:n_int + 1])
    return True


@pytest.mark.parametrize("cfg_name", ["tiny", "C2"])
@pytest.mark.parametrize("batch", [1, 2, 4])
def test_tables_bit_equal_to_the_host_count_plan(cuda, cfg_name, batch):
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS[cfg_name]
    fr = frustum(cuda, cfg)
    host, dev = plans(cuda, cfg, rig(cuda, cfg, batch, seed=batch), fr)
    assert_tables_equal(host, dev)
    assert assert_column_tables_equal(host, dev)
    # rebuilt in place with another draw: the same again, in the same buffers
    perm_ptr = dev.tables.perm.data_ptr()
    r2 = rig(cuda, cfg, batch, seed=100 + batch)
    dev.rebuild_(*calib(r2))
    host2 = host_plan(cfg, r2, fr)
    assert dev.tables.perm.data_ptr() == perm_ptr
    assert_tables_equal(host2, dev)
    assert_column_tables_equal(host2, dev)


@pytest.mark.parametrize("C", [16, 32, 64, 80, 96, 128, 160, 256, 24])
def test_outputs_and_gradients_bit_equal(cuda, C):
    """every tuned channel width and one untuned one (24: generic pooling kernels; the fused lift has tuned widths
    only): pool and its x gradient, the column lift and its depth / ctx gradients"""
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["tiny"]
    fr = frustum(cuda, cfg)
    for batch in (1, 2):                                   # 1: zero-filling kernels; 2: pre-zeroed grid
        host, dev = plans(cuda, cfg, rig(cuda, cfg, batch, seed=C + batch), fr)
        depth, ctx, G = inputs(cuda, dev, fr, C, seed=C)
        x = (depth.unsqueeze(-1) * ctx.unsqueeze(2)).contiguous()
        outs = []
        for plan in (host, dev):
            xr = x.clone().requires_grad_(True)
            out = plan.pool(xr)
            (xg,) = torch.autograd.grad(out, (xr,), G)
            outs.append((out.detach(), xg))
        assert same(outs[0][0], outs[1][0]) and same(outs[0][1], outs[1][1])
        assert float(outs[0][0].abs().max()) > 0
        if C not in (16, 32, 64, 80, 96, 128, 160, 256):
            continue
        assert int(dev.tables.lift_form) == 0
        for a, b in zip(lift_step(host, depth, ctx, G), lift_step(dev, depth, ctx, G)):
            assert same(a, b)


def test_c2_outputs_bit_equal(cuda):
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["C2"]
    fr = frustum(cuda, cfg)
    host, dev = plans(cuda, cfg, rig(cuda, cfg, 2, seed=11), fr)
    depth, ctx, G = inputs(cuda, dev, fr, 80, seed=3)
    assert int(dev.tables.lift_form) == 0
    for a, b in zip(lift_step(host, depth, ctx, G), lift_step(dev, depth, ctx, G)):
        assert same(a, b)
    with torch.no_grad():
        assert same(host.lift(depth, ctx), dev.lift(depth, ctx))


def test_feature_height_above_64_runs_the_row_form(cuda):
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["tiny"]
    fr = frustum(cuda, cfg, (72, 8))
    host, dev = plans(cuda, cfg, rig(cuda, cfg, 1, seed=5), fr)
    assert int(dev.tables.lift_form) == 1 and dev.max_segments == 0
    assert_tables_equal(host, dev)
    depth, ctx, G = inputs(cuda, dev, fr, 80, seed=5)
    for a, b in zip(lift_step(host, depth, ctx, G), lift_step(dev, depth, ctx, G)):
        assert same(a, b)


@pytest.mark.parametrize("batch", [1, 2])
def test_no_point_in_the_grid(cuda, batch):
    """every frustum point off the grid (n_kept = 0): zero BEV map and zero gradients, as the host-count plan gives"""
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["tiny"]
    fr = frustum(cuda, cfg)
    host, dev = plans(cuda, cfg, rig(cuda, cfg, batch, seed=1, shift=1000.0), fr)
    assert host.tables.n_kept == 0 and int(dev.tables.n_kept) == 0 and int(dev.tables.n_intervals) == 0
    assert int(dev.tables.lift_form) == 0 and int(dev.tables.n_segments) == 0
    depth, ctx, G = inputs(cuda, dev, fr, 80, seed=1)
    for plan in (host, dev):                              # garbage in the outputs' memory must not survive
        torch.empty(64 << 20, device=cuda).fill_(float("nan"))
        out, gd, gc = lift_step(plan, depth, ctx, G)
        assert not bool(out.any()) and not bool(gd.any()) and not bool(gc.any())
        xr = (depth.unsqueeze(-1) * ctx.unsqueeze(2)).requires_grad_(True)
        out = plan.pool(xr)
        (xg,) = torch.autograd.grad(out, (xr,), G)
        assert not bool(out.any()) and not bool(xg.any())
    # the fallback forms of the empty grid are zero as well
    _, dev_rows = plans(cuda, cfg, rig(cuda, cfg, batch, seed=1, shift=1000.0), fr)
    dev_rows.tables.counts[3] = 1
    out, gd, gc = lift_step(dev_rows, depth, ctx, G)
    assert not bool(out.any()) and not bool(gd.any()) and not bool(gc.any())


def test_every_point_in_one_cell(cuda):
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["tiny"]
    fr = frustum(cuda, cfg)
    bounds = ((-200.0, 200.0, 400.0), (-200.0, 200.0, 400.0), (-1000.0, 1000.0, 2000.0))
    host, dev = plans(cuda, cfg, rig(cuda, cfg, 1, seed=2), fr, bounds=bounds)
    assert tuple(dev.tables.dims) == (1, 1, 1, 1)
    assert int(dev.tables.n_intervals) == 1 and int(dev.tables.n_kept) == dev.tables.n_total
    assert_tables_equal(host, dev)
    assert_column_tables_equal(host, dev)
    depth, ctx, G = inputs(cuda, dev, fr, 64, seed=2)
    for a, b in zip(lift_step(host, depth, ctx, G), lift_step(dev, depth, ctx, G)):
        assert same(a, b)
        assert bool(a.any())


@pytest.mark.parametrize("cfg_name,batch", [("tiny", 2), ("C2", 1)])
def test_fallback_to_the_row_kernels(cuda, cfg_name, batch):
    """max_segments below the true count: the status word reports the row form, and forward and backward equal the
    row path of the host-count API bit for bit"""
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS[cfg_name]
    fr = frustum(cuda, cfg)
    r = rig(cuda, cfg, batch, seed=9)
    B, N, D, fH, fW = batch, cfg["n_cam"], fr.shape[0], fr.shape[1], fr.shape[2]
    n_seg = host_plan(cfg, r, fr)._lift_tables(B * N, D, fH, fW)[5]
    host, dev = plans(cuda, cfg, r, fr, max_segments=n_seg // 2)
    assert int(dev.tables.n_segments) == n_seg and int(dev.tables.lift_form) == 1
    assert_tables_equal(host, dev)
    depth, ctx, G = inputs(cuda, dev, fr, 80, seed=9)
    for a, b in zip(host_rows(host, depth, ctx, G), lift_step(dev, depth, ctx, G)):
        assert same(a, b)
    # and a plan whose cap the count just fits runs the columns, equal to the host-count default
    _, fits = plans(cuda, cfg, r, fr, max_segments=n_seg)
    assert int(fits.tables.lift_form) == 0
    for a, b in zip(lift_step(host, depth, ctx, G), lift_step(fits, depth, ctx, G)):
        assert same(a, b)


def test_cuda_graph_replays_new_calibration(cuda):
    """capture rebuild_ + lift_pool + backward once, replay it with calibrations copied into the static inputs (one
    over the column cap): every replay equals an eager host-count plan of that calibration bit for bit"""
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["C2"]
    fr = frustum(cuda, cfg)
    rigs = [rig(cuda, cfg, 1, seed=s) for s in range(20, 26)]
    hosts = [host_plan(cfg, r, fr) for r in rigs]
    B, N, D, fH, fW = 1, cfg["n_cam"], fr.shape[0], fr.shape[1], fr.shape[2]
    n_seg = [h._lift_tables(B * N, D, fH, fW)[5] for h in hosts]
    over = max(range(len(rigs)), key=lambda i: n_seg[i])
    cap = max(n for i, n in enumerate(n_seg) if i != over)
    assert n_seg[over] > cap
    order = [i for i in range(len(rigs)) if i != over][:3] + [over]
    _, plan = plans(cuda, cfg, rigs[order[0]], fr, max_segments=cap)
    static = [t.clone() for t in calib(rigs[order[0]])]
    depth, ctx, G = inputs(cuda, plan, fr, 80, seed=4)
    sd, sc = depth.clone().requires_grad_(True), ctx.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            plan.rebuild_(*static)
            torch.autograd.grad(plan.lift_pool(sd, sc), (sd, sc), G)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):                         # a host synchronisation inside would fail the capture
        plan.rebuild_(*static)
        out = plan.lift_pool(sd, sc)
        gd, gc = torch.autograd.grad(out, (sd, sc), G)
    for i in order[1:] + order[:1]:
        with torch.no_grad():
            for dst, src in zip(static, calib(rigs[i])):
                dst.copy_(src)
        graph.replay()
        torch.cuda.synchronize()
        fits = n_seg[i] <= cap
        assert int(plan.tables.lift_form) == (0 if fits else 1)
        assert int(plan.tables.n_kept) == hosts[i].tables.n_kept
        want = lift_step(hosts[i], depth, ctx, G) if fits else host_rows(hosts[i], depth, ctx, G)
        for a, b in zip(want, (out.detach(), gd, gc)):
            assert same(a, b)


def test_default_cap_holds_augmented_c2(cuda):
    """the default max_segments (DESIGN.md section 4.24) keeps augmented C2 rigs on the column kernels"""
    from bevfusion_b200 import synthetic as S
    from bevfusion_b200.bev_pool import BEVPoolPlan
    cfg = S.CONFIGS["C2"]
    fr = frustum(cuda, cfg)
    c = calib(rig(cuda, cfg, 1, seed=30))
    plan = BEVPoolPlan.from_cameras(fr, *c[:5], cfg["xbound"], cfg["ybound"], cfg["zbound"], c[5], c[6], sync=False)
    for seed in range(30, 36):
        plan.rebuild_(*calib(rig(cuda, cfg, 1, seed=seed)))
        assert int(plan.tables.lift_form) == 0, (seed, int(plan.tables.n_segments), plan.max_segments)


def test_eager_step_does_not_synchronise(cuda):
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["tiny"]
    fr = frustum(cuda, cfg)
    r = rig(cuda, cfg, 2, seed=3)
    host, plan = plans(cuda, cfg, r, fr)
    depth, ctx, G = inputs(cuda, plan, fr, 80, seed=3)
    lift_step(plan, depth, ctx, G)                        # workspaces are allocated at first use
    x = (depth.unsqueeze(-1) * ctx.unsqueeze(2)).contiguous().requires_grad_(True)
    torch.autograd.grad(plan.pool(x), (x,), G)
    r2 = rig(cuda, cfg, 2, seed=4)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        plan.rebuild_(*calib(r2))
        out, gd, gc = lift_step(plan, depth, ctx, G)
        (xg,) = torch.autograd.grad(plan.pool(x), (x,), G)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    host2 = host_plan(cfg, r2, fr)
    for a, b in zip(lift_step(host2, depth, ctx, G), (out, gd, gc)):
        assert same(a, b)


def test_rebuild_refusals_leave_the_tables_untouched(cuda):
    from bevfusion_b200 import synthetic as S
    cfg = S.CONFIGS["tiny"]
    fr = frustum(cuda, cfg)
    r = rig(cuda, cfg, 2, seed=6)
    host, plan = plans(cuda, cfg, r, fr)
    t = plan.tables
    before = [x.clone() for x in (t.perm, t.geom, t.starts, t.lengths, t.counts, plan._seg["seg_key"],
                                  plan._seg["col_begin"])]
    other = calib(rig(cuda, cfg, 2, seed=7))
    bad = [
        (1, other[1][:1]),                                 # wrong batch
        (3, other[3][..., :2, :2]),                        # wrong matrix size
        (2, other[2].double()),                            # wrong dtype
        (0, other[0].cpu()),                               # wrong device
        (5, other[5].reshape(2, 9)),                       # extra_rots shape
    ]
    for k, v in bad:
        args = list(other)
        args[k] = v
        with pytest.raises(ValueError):
            plan.rebuild_(*args)
    torch.cuda.synchronize()
    after = (t.perm, t.geom, t.starts, t.lengths, t.counts, plan._seg["seg_key"], plan._seg["col_begin"])
    for a, b in zip(before, after):
        assert torch.equal(a, b)
    with pytest.raises(ValueError):
        host.rebuild_(*other)                              # a host-count plan has no rebuild
