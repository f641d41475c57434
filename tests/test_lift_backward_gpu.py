"""GPU: backward of the fused LSS lift + pool (BEVPoolPlan.lift_pool / lift).  Gradients of depth and ctx against a
float64 autograd of the materialised volume, the fp32 materialised path through plan.pool, and the reference's own
bev_pool backward kernel; bit reproducibility, unchanged forward, CUDA-graph capture.
Tolerances: gradients <= 1e-5 x max|gold|."""
import pytest
import torch

from conftest import ref_module

pytestmark = pytest.mark.gpu

TOL = 1e-5


def make_case(cuda, cfg_name, batch=1, C=None, seed=1, jitter=0.0, geom_fn=None):
    from bevfusion_b200 import synthetic as S
    from bevfusion_b200.bev_pool import BEVPoolPlan
    geom, cfg = S.camera_geometry(cfg_name, batch=batch, device=cuda)
    g = torch.Generator(device=cuda).manual_seed(seed)
    if jitter:
        geom = geom + torch.randn(geom.shape, generator=g, device=cuda) * jitter
    if geom_fn is not None:
        geom = geom_fn(geom)
    plan = BEVPoolPlan(geom.contiguous(), cfg["xbound"], cfg["ybound"], cfg["zbound"])
    B, N, D, fH, fW, _ = geom.shape
    C = C or cfg["C"]
    depth = torch.softmax(torch.randn(B, N, D, fH, fW, generator=g, device=cuda), dim=2).contiguous()
    ctx = torch.randn(B, N, fH, fW, C, generator=g, device=cuda)
    Bq, Dq, Hq, Wq = plan.tables.dims
    G = torch.randn(Bq, Dq, Hq, Wq, C, generator=g, device=cuda)
    return plan, depth, ctx, G


def fused_grads(plan, depth, ctx, G, want=(True, True)):
    d = depth.detach().clone().requires_grad_(want[0])
    c = ctx.detach().clone().requires_grad_(want[1])
    out = plan.lift_pool(d, c)
    inputs = [t for t, w in zip((d, c), want) if w]
    grads = torch.autograd.grad(out, inputs, G)
    return grads if len(grads) == 2 else grads[0]


def gold64(plan, depth, ctx, G):
    """float64 autograd of the materialised lift, pooled with index_add_ over the plan's perm / geom tables."""
    t = plan.tables
    Bq, Dq, Hq, Wq = t.dims
    C = ctx.shape[-1]
    d = depth.double().requires_grad_(True)
    c = ctx.double().requires_grad_(True)
    x = (d.unsqueeze(-1) * c.unsqueeze(2)).reshape(-1, C)
    gm = t.geom.long()
    cell = ((gm[:, 3] * Dq + gm[:, 2]) * Hq + gm[:, 0]) * Wq + gm[:, 1]
    out = torch.zeros(Bq * Dq * Hq * Wq, C, dtype=torch.float64, device=depth.device)
    out = out.index_add(0, cell, x[t.perm[:t.n_kept].long()])
    return torch.autograd.grad(out, (d, c), G.double().reshape(-1, C))


def assert_close(got, gold, tol=TOL):
    scale = float(gold.abs().max())
    assert scale > 0
    err = float((got.double() - gold.double()).abs().max())
    assert err <= tol * scale, (err, scale)


@pytest.mark.parametrize("cfg_name", ["tiny", "C2"])
def test_against_float64(cuda, cfg_name):
    plan, depth, ctx, G = make_case(cuda, cfg_name)
    dd, dc = fused_grads(plan, depth, ctx, G)
    gd, gc = gold64(plan, depth, ctx, G)
    assert dd.shape == depth.shape and dc.shape == ctx.shape
    assert_close(dd, gd)
    assert_close(dc, gc)


@pytest.mark.parametrize("cfg_name", ["tiny", "C2", "C5"])
def test_against_materialised_fp32(cuda, cfg_name):
    """C5: fH = 64, D = 200 -- more segments per column than one shared-memory chunk holds."""
    plan, depth, ctx, G = make_case(cuda, cfg_name)
    dd, dc = fused_grads(plan, depth, ctx, G)
    d = depth.clone().requires_grad_(True)
    c = ctx.clone().requires_grad_(True)
    out = plan.pool(d.unsqueeze(-1) * c.unsqueeze(2))
    gd, gc = torch.autograd.grad(out, (d, c), G)
    del out
    assert_close(dd, gd)
    assert_close(dc, gc)


def test_bit_reproducible(cuda):
    plan, depth, ctx, G = make_case(cuda, "C2")
    dd1, dc1 = fused_grads(plan, depth, ctx, G)
    dd2, dc2 = fused_grads(plan, depth, ctx, G)
    assert torch.equal(dd1, dd2) and torch.equal(dc1, dc2)


@pytest.mark.parametrize("cfg_name", ["tiny", "C2"])
def test_forward_unchanged(cuda, cfg_name):
    plan, depth, ctx, _ = make_case(cuda, cfg_name)
    with torch.no_grad():
        ref = plan.lift_pool(depth, ctx)
    out = plan.lift_pool(depth.clone().requires_grad_(True), ctx.clone().requires_grad_(True))
    assert out.requires_grad
    assert torch.equal(out.detach(), ref)


@pytest.mark.parametrize("batch", [1, 2])
def test_arbitrary_geometry_and_filtering(cuda, batch):
    """jittered frustum points: many partial-mask segments per column, points leave the grid.  Image columns 0..2
    of camera 0 are moved out of the grid entirely: their pixels keep no point at all."""
    def off_grid(geom):
        geom = geom.clone()
        geom[:, 0, :, :, 0:3, 0] += 100.0
        return geom

    plan, depth, ctx, G = make_case(cuda, "tiny", batch=batch, C=64, seed=7, jitter=1.5, geom_fn=off_grid)
    t = plan.tables
    B, N, D, fH, fW = depth.shape
    n_seg = plan._lift_tables(B * N, D, fH, fW)[5]
    assert n_seg > 0.5 * t.n_kept
    dd, dc = fused_grads(plan, depth, ctx, G)
    gd, gc = gold64(plan, depth, ctx, G)
    assert_close(dd, gd)
    assert_close(dc, gc)
    filtered = t.perm[t.n_kept:].long()
    assert filtered.numel() > 0
    assert bool((dd.reshape(-1)[filtered] == 0).all())
    kept = torch.zeros(B * N * D * fH * fW, dtype=torch.int32, device=cuda)
    kept[t.perm[:t.n_kept].long()] = 1
    empty_pixels = kept.view(B * N, D, fH * fW).sum(1).view(-1) == 0
    assert int(empty_pixels.sum()) >= batch * fH * 3
    assert bool((dc.reshape(-1, dc.shape[-1])[empty_pixels] == 0).all())


@pytest.mark.parametrize("C", [16, 32, 64, 80, 96, 128, 160, 256])
def test_every_channel_count(cuda, C):
    plan, depth, ctx, G = make_case(cuda, "tiny", C=C, seed=C)
    dd, dc = fused_grads(plan, depth, ctx, G)
    gd, gc = gold64(plan, depth, ctx, G)
    assert_close(dd, gd)
    assert_close(dc, gc)


def test_feature_height_above_64(cuda):
    """fH = 72: the segment mask cannot hold a column, the pixel backward runs (and the row forward)."""
    from bevfusion_b200 import synthetic as S
    from bevfusion_b200.bev_pool import BEVPoolPlan
    from bevfusion_b200.vtransform import create_frustum, get_geometry
    cfg = S.CONFIGS["tiny"]
    rig = {k: v.to(cuda) for k, v in S.camera_rig(cfg["n_cam"], cfg["image_size"], 1).items()}
    frustum = create_frustum(cfg["image_size"], (72, 8), cfg["dbound"]).to(cuda)
    geom = get_geometry(frustum, rig["camera2lidar_rots"], rig["camera2lidar_trans"], rig["intrins"],
                        rig["post_rots"], rig["post_trans"]).contiguous()
    plan = BEVPoolPlan(geom, cfg["xbound"], cfg["ybound"], cfg["zbound"])
    B, N, D, fH, fW, _ = geom.shape
    assert fH == 72
    g = torch.Generator(device=cuda).manual_seed(3)
    depth = torch.softmax(torch.randn(B, N, D, fH, fW, generator=g, device=cuda), dim=2).contiguous()
    ctx = torch.randn(B, N, fH, fW, 80, generator=g, device=cuda)
    G = torch.randn(*plan.tables.dims, 80, generator=g, device=cuda)
    dd, dc = fused_grads(plan, depth, ctx, G)
    gd, gc = gold64(plan, depth, ctx, G)
    assert_close(dd, gd)
    assert_close(dc, gc)
    assert getattr(plan, "_lift_cache", None) is None          # the column tables were never built
    dd2, dc2 = fused_grads(plan, depth, ctx, G)
    assert torch.equal(dd, dd2) and torch.equal(dc, dc2)


def test_one_gradient_at_a_time(cuda):
    plan, depth, ctx, G = make_case(cuda, "tiny")
    dd, dc = fused_grads(plan, depth, ctx, G)
    d = depth.clone().requires_grad_(True)
    c = ctx.clone()
    (plan.lift_pool(d, c) * G).sum().backward()
    assert c.grad is None and torch.equal(d.grad, dd)
    d = depth.clone()
    c = ctx.clone().requires_grad_(True)
    (plan.lift_pool(d, c) * G).sum().backward()
    assert d.grad is None and torch.equal(c.grad, dc)
    assert torch.equal(fused_grads(plan, depth, ctx, G, want=(True, False)), dd)
    assert torch.equal(fused_grads(plan, depth, ctx, G, want=(False, True)), dc)


def test_module_layout(cuda):
    """plan.lift (the [B, C*nz, nx, ny] module layout), also written into a channel slice of the fuser's input,
    backpropagates into depth and ctx exactly like lift_pool followed by torch's permute."""
    plan, depth, ctx, _ = make_case(cuda, "tiny", batch=2)
    B = depth.shape[0]
    Bq, Z, X, Y = plan.tables.dims
    C = ctx.shape[-1]
    W = torch.randn(B, Z * C, X, Y, device=cuda)
    d0, c0 = depth.clone().requires_grad_(True), ctx.clone().requires_grad_(True)
    ref = plan.lift_pool(d0, c0).permute(0, 1, 4, 2, 3).reshape(B, Z * C, X, Y)
    gd, gc = torch.autograd.grad(ref, (d0, c0), W)
    d1, c1 = depth.clone().requires_grad_(True), ctx.clone().requires_grad_(True)
    bev = plan.lift(d1, c1)
    assert torch.equal(bev.detach(), ref.detach())
    g1 = torch.autograd.grad(bev, (d1, c1), W)
    assert torch.equal(g1[0], gd) and torch.equal(g1[1], gc)
    d2, c2 = depth.clone().requires_grad_(True), ctx.clone().requires_grad_(True)
    buf = torch.zeros(B, Z * C + 16, X, Y, device=cuda)
    plan.lift(d2, c2, out=buf[:, :Z * C])
    Wbuf = torch.cat([W, torch.randn(B, 16, X, Y, device=cuda)], 1)
    g2 = torch.autograd.grad(buf, (d2, c2), Wbuf)
    assert torch.equal(g2[0], gd) and torch.equal(g2[1], gc)


def test_cuda_graph_capture(cuda):
    plan, depth, ctx, G = make_case(cuda, "C2")
    sd = depth.clone().requires_grad_(True)
    sc = ctx.clone().requires_grad_(True)
    sG = G.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                    # warm-up (builds the segment tables, which synchronise)
        for _ in range(2):
            torch.autograd.grad(plan.lift_pool(sd, sc), (sd, sc), sG)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = plan.lift_pool(sd, sc)
        gd, gc = torch.autograd.grad(out, (sd, sc), sG)
    _, depth2, ctx2, G2 = make_case(cuda, "C2", seed=5)
    with torch.no_grad():
        sd.copy_(depth2)
        sc.copy_(ctx2)
        sG.copy_(G2)
    graph.replay()
    torch.cuda.synchronize()
    ed, ec = fused_grads(plan, depth2, ctx2, G2)
    assert torch.equal(out.detach(), plan.lift_pool(depth2, ctx2))
    assert torch.equal(gd, ed) and torch.equal(gc, ec)


def test_against_reference_backward_kernel(cuda):
    """the reference's own bev_pool_backward (compiled into oracle/_ref) on the sorted kept rows, followed by the
    float64 backward of the lift's broadcast multiply, at C2."""
    ref = ref_module("bev_pool_ext_ref")
    if ref is None:
        pytest.skip("oracle/_ref not built")
    plan, depth, ctx, G = make_case(cuda, "C2")
    dd, dc = fused_grads(plan, depth, ctx, G)
    t = plan.tables
    Bq, Dq, Hq, Wq = t.dims
    torch.cuda.synchronize()
    xg = ref.bev_pool_backward(G.contiguous(), t.geom.contiguous(), t.lengths.contiguous(), t.starts.contiguous(),
                               Bq, Dq, Hq, Wq)                 # [n_kept, C], sorted rows (legacy default stream)
    torch.cuda.synchronize()
    B, N, D, fH, fW = depth.shape
    C = ctx.shape[-1]
    p = t.perm[:t.n_kept].long()
    pix = (p // (D * fH * fW)) * (fH * fW) + p % (fH * fW)
    xg = xg.double()
    gd = torch.zeros(depth.numel(), dtype=torch.float64, device=cuda)
    gd[p] = (xg * ctx.reshape(-1, C).double()[pix]).sum(1)
    gc = torch.zeros(B * N * fH * fW, C, dtype=torch.float64, device=cuda)
    gc.index_add_(0, pix, xg * depth.reshape(-1).double()[p].unsqueeze(1))
    assert_close(dd.reshape(-1), gd)
    assert_close(dc.reshape(-1, C), gc)
