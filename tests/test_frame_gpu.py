"""The frame bench.py times -- bench.HotPath.frame / frame_lift, captured as one CUDA graph and replayed -- against
float64 (tests/frame_oracle.py) and the reference's own CUDA kernels, at full size.

The frame runs the camera branch on a second stream, the encoder plan's rulebooks on a third, takes the voxel count
from the device (cap-sized voxel buffers whose tails are garbage), keeps workspaces and lift tables across calls and
captures, and writes into channel slices.  Every test here builds the frame through bench.HotPath, so it follows
whatever the benchmark times."""
import numpy as np
import pytest
import torch

import frame_oracle as FO
from conftest import ref_module

pytestmark = pytest.mark.gpu

SPIN_CYCLES = 200_000_000          # torch.cuda._sleep: about 0.1 s of one spinning thread, longer than a frame's launch


def _hotpath(device, seed, **kw):
    import bench
    return bench.HotPath(device, seed=seed, **kw)


def _sparse_cloud(seed, n, keep=0.4):
    """n points: the first keep * n of synthetic cloud `seed` (shuffled, so a thinner scene), the rest far outside
    the range (dropped).  Fewer voxels than the 160 k cap: the sync-free voxelizer's buffers get a garbage tail."""
    from bevfusion_b200 import synthetic as S
    p = S.lidar_cloud(seed=seed)[:int(keep * n)]
    pad = np.zeros((n - p.shape[0], p.shape[1]), np.float32)
    pad[:, 0] = 1.0e3
    return np.concatenate([p, pad])


class C2Frame:
    """one rank of `bench.py --gpus 2`: HotPath(seed), its inputs, and the float64 references of both branches"""

    def __init__(self, device, seed):
        self.seed, self.device = seed, device
        self.hp = hp = _hotpath(device, seed)
        self.x, self.pts = hp.device_inputs(seed=seed)
        self.pts_np = hp.points_host.numpy()
        self.cells = FO.CameraCells(hp.geom, hp.cfg)
        self.cam64 = FO.pool64(self.cells, FO.volume_rows(self.x), hp.cfg["C"], device)
        self.lid64 = FO.lidar64(hp.L, hp.encoder, self.pts_np, device)
        print("seed %d: float64 encoder at %d voxels (CPU-oracle rulebooks included) took %.1f s"
              % (seed, self.lid64["n"], self.lid64["seconds"]))


@pytest.fixture(scope="module", params=[0, 1], ids=["seed0", "seed1"])
def c2(cuda, request):
    f = C2Frame(cuda, request.param)
    yield f
    del f
    torch.cuda.empty_cache()


def _fused_voxels(hp, pts):
    from bevfusion_b200.voxelize import voxelize_mean_fused
    L = hp.L
    return voxelize_mean_fused(pts, L["voxel_size"], L["point_cloud_range"], L["max_num_points"], L["max_voxels"][1],
                               0, sync=False)


def _after_slow_producer(fn, srcs, prefilled=()):
    """fn(*bufs) issued on a non-default stream while a third stream, held busy by a spin, fills bufs from srcs;
    the consumer joins the producer with wait_stream only.  Buffers start at zero (indices in `prefilled` start
    as copies of their source).  A stage that ignores the caller's stream reads the zeros."""
    dev = srcs[0].device
    bufs = [s.clone() if i in prefilled else torch.zeros_like(s) for i, s in enumerate(srcs)]
    producer, consumer = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
    producer.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(producer):
        torch.cuda._sleep(SPIN_CYCLES)
        for b, s in zip(bufs, srcs):
            b.copy_(s)
    consumer.wait_stream(producer)
    with torch.cuda.stream(consumer):
        out = fn(*bufs)
    torch.cuda.synchronize(dev)
    return out


# ------------------------------------------------------------------------------------ the C2+C3 frame
def test_frame_replay_vs_float64(c2):
    """one graph replay of HotPath.frame: BEV map within the per-cell fp32 bound of the float64 pool (empty cells
    0), LiDAR map within 1e-4 x max of the float64 encoder, rows per level, overflow flag and voxel count exact"""
    hp = c2.hp
    g, gout = hp.capture(hp.frame, c2.x, c2.pts)
    hp.encoder.plan().status.fill_(-1)
    g.replay()
    torch.cuda.synchronize()
    bev, lidar = gout
    assert tuple(bev.shape) == (1, 80, 360, 360) and tuple(lidar.shape) == (1, 256, 180, 180)
    FO.check_pool(FO.bev_to_raw(bev, c2.cells.dims), c2.cam64, "frame bev (seed %d)" % c2.seed)
    FO.check_lidar(lidar, hp.encoder.plan().status, c2.lid64, "frame lidar (seed %d)" % c2.seed)
    assert hp.encoder.plan().status[1].item() == c2.lid64["n"]          # the device count reached the encoder
    feats, coords, num, nv = _fused_voxels(hp, c2.pts)
    FO.check_voxels(feats, coords, num, nv, c2.lid64, "sync-free voxelization (seed %d)" % c2.seed)
    del g, gout


def test_frame_graph_eager_and_staged_bit_equal(c2):
    """graph replay == eager frame() == hp.plan(x) then hp._lidar(points) on the default stream, bit for bit"""
    hp = c2.hp
    g, gout = hp.capture(hp.frame, c2.x, c2.pts)
    g.replay()
    torch.cuda.synchronize()
    replay = [t.clone() for t in gout]
    eager = hp.frame(c2.x, c2.pts)
    staged = (hp.plan(c2.x), hp._lidar(c2.pts))
    torch.cuda.synchronize()
    for name, r, e, s in zip(("bev", "lidar"), replay, eager, staged):
        assert torch.equal(r, e), "%s: graph replay != eager frame()" % name
        assert torch.equal(e, s), "%s: eager frame() != the stages run one after another" % name
    del g, gout


def test_frame_graph_replays_new_inputs(c2):
    """another rank's volume and a thinner cloud -- fewer voxels than the cap, so the voxel buffers have a garbage
    tail -- written into the captured buffers: the replay equals eager on them and its LiDAR map matches float64;
    the first inputs copied back give the first result again"""
    from bevfusion_b200 import synthetic as S
    hp = c2.hp
    x_buf, pts_buf = c2.x.clone(), c2.pts.clone()
    g, gout = hp.capture(hp.frame, x_buf, pts_buf)
    g.replay()
    torch.cuda.synchronize()
    first = [t.clone() for t in gout]
    other = 1 - c2.seed
    thin = _sparse_cloud(other, pts_buf.shape[0])
    x_buf.copy_(S.lifted_features("C2", device=c2.device, seed=other))
    pts_buf.copy_(torch.from_numpy(thin).to(c2.device))
    ref = FO.lidar64(hp.L, hp.encoder, thin, c2.device)
    assert ref["n"] < hp.L["max_voxels"][1] and ref["n"] != c2.lid64["n"]
    g.replay()
    torch.cuda.synchronize()
    replay = [t.clone() for t in gout]
    FO.check_lidar(replay[1], hp.encoder.plan().status, ref, "replay on a thinner cloud (seed %d)" % other)
    eager = hp.frame(x_buf, pts_buf)
    torch.cuda.synchronize()
    for name, r, e in zip(("bev", "lidar"), replay, eager):
        assert torch.equal(r, e), "%s: replay on new inputs != eager" % name
    x_buf.copy_(c2.x)
    pts_buf.copy_(c2.pts)
    g.replay()
    torch.cuda.synchronize()
    for name, r, e in zip(("bev", "lidar"), gout, first):
        assert torch.equal(r, e), "%s: replay on the first inputs again != first replay" % name
    del g, gout, x_buf, pts_buf


def test_frame_and_stages_follow_the_callers_stream(c2):
    """the frame and each of its stages issued on a non-default stream whose inputs come from a spinning producer
    stream equal the default-stream result"""
    hp = c2.hp
    want = hp.frame(c2.x, c2.pts)
    got = _after_slow_producer(hp.frame, [c2.x, c2.pts])
    for name, a, b in zip(("bev", "lidar"), got, want):
        assert torch.equal(a, b), "frame %s under a non-default stream" % name
    assert torch.equal(_after_slow_producer(hp.plan.pool, [c2.x]), hp.plan.pool(c2.x)), "BEVPoolPlan.pool"
    depth, ctx = hp.lift_inputs(c2.seed, c2.device)
    assert torch.equal(_after_slow_producer(hp.plan.lift, [depth, ctx]), hp.plan.lift(depth, ctx)), "BEVPoolPlan.lift"
    f, c, n, nv = _after_slow_producer(lambda p: _fused_voxels(hp, p), [c2.pts])
    wf, wc, wn, wnv = _fused_voxels(hp, c2.pts)
    m = int(wnv.item())
    assert int(nv.item()) == m and torch.equal(c[:m], wc[:m]) and torch.equal(n[:m], wn[:m]) \
        and torch.equal(f[:m], wf[:m]), "voxelize_mean_fused(sync=False)"
    plan = hp.encoder.plan()

    def encode(feats, coors, count):
        with torch.no_grad():
            return plan.forward(feats, coors, 1, n_voxels_dev=count)
    with torch.no_grad():
        want_enc = plan.forward(wf, wc, 1, n_voxels_dev=wnv)
    # coordinates start as the real ones, the count at 0: an encoder that reads early sees no voxels
    got_enc = _after_slow_producer(encode, [wf, wc, wnv], prefilled=(1,))
    assert torch.equal(got_enc, want_enc), "EncoderPlan.forward"


# ------------------------------------------------------------------------- fused lift frame, C4 write path
def test_frame_lift_replay_vs_float64(c2):
    """HotPath.frame_lift on the camera branch's real inputs: per-cell bound against the float64 pool of
    depth (x) ctx, LiDAR map against float64, graph replay == eager"""
    hp = c2.hp
    depth, ctx = hp.lift_inputs(c2.seed, c2.device)
    g, gout = hp.capture(hp.frame_lift, depth, ctx, c2.pts)
    g.replay()
    torch.cuda.synchronize()
    ref = FO.pool64(c2.cells, FO.lifted_rows(depth, ctx), hp.cfg["C"], c2.device)
    FO.check_pool(FO.bev_to_raw(gout[0], c2.cells.dims), ref, "frame_lift bev (seed %d)" % c2.seed, products=True)
    FO.check_lidar(gout[1], hp.encoder.plan().status, c2.lid64, "frame_lift lidar (seed %d)" % c2.seed)
    eager = hp.frame_lift(depth, ctx, c2.pts)
    torch.cuda.synchronize()
    for name, r, e in zip(("bev", "lidar"), gout, eager):
        assert torch.equal(r, e), "frame_lift %s: graph replay != eager" % name
    del g, gout


def test_lidar_written_into_fuser_slice_in_graph(c2):
    """hp._lidar(points, out=fuser_in[:, 80:]) captured as the C4 frame does: channels 80:336 equal the standalone
    output bit for bit, channels 0:80 keep their sentinel"""
    hp = c2.hp
    fuser_in = torch.full((1, 80 + 256, 180, 180), 7.25, device=c2.device)
    g, _ = hp.capture(lambda p: hp._lidar(p, out=fuser_in[:, 80:]), c2.pts)
    fuser_in.fill_(7.25)
    g.replay()
    torch.cuda.synchronize()
    alone = hp._lidar(c2.pts)
    assert torch.equal(fuser_in[:, 80:], alone)
    assert bool((fuser_in[:, :80] == 7.25).all())
    del g


# ------------------------------------------------------------------- graph-held workspaces outlive later calls
def _unique_coords(n, shape, seed):
    rng = np.random.default_rng(seed)
    flat = rng.choice(int(np.prod(shape)), size=n, replace=False)
    x, y, z = np.unravel_index(flat, shape)
    return np.stack([np.zeros(n, np.int64), x, y, z], 1).astype(np.int32)


def _span(t):
    return t.data_ptr(), t.data_ptr() + t.numel() * t.element_size()


def _assert_disjoint(tensors, held, what):
    """no tensor in `tensors` shares memory with the spans in `held` (memory a captured graph still uses)"""
    for i, t in enumerate(tensors):
        a, b = _span(t)
        assert not any(a < hi and lo < b for lo, hi in held), \
            "%s: tensor %d was given memory a captured graph still uses" % (what, i)


def test_encoder_plan_workspace_outlives_graph(cuda):
    """capture EncoderPlan.forward at n1 voxels, grow the workspace with an eager call at 4 n1, fill fresh tensors
    of the old workspace's size: none of them, nor the new workspace, gets the captured workspace's memory, and
    replaying the graph still equals eager at n1 and writes none of them"""
    from bevfusion_b200.sparse_encoder import voxelnet_0p075_encoder
    torch.manual_seed(3)
    m = voxelnet_0p075_encoder().to(cuda).eval()
    m.sparse_shape = [192, 192, 41]
    plan = m.plan()
    rng = np.random.default_rng(4)

    def inputs(n, seed):
        c = torch.from_numpy(_unique_coords(n, [192, 192, 40], seed)).to(cuda)
        return torch.from_numpy(rng.standard_normal((n, 5)).astype(np.float32)).to(cuda), c
    f1, c1 = inputs(6000, 1)
    f2, c2 = inputs(24000, 2)
    with torch.no_grad():
        want1 = plan.forward(f1, c1, 1).clone()
        ws1, held = plan._ws.numel(), [_span(plan._ws)]
        out1 = torch.empty_like(want1)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            plan.forward(f1, c1, 1, out=out1)
        out2 = plan.forward(f2, c2, 1)
    assert plan._ws.numel() > ws1                       # the eager call replaced the workspace
    out2_copy = out2.clone()
    sentinels = [torch.full((ws1,), 0xA5, dtype=torch.uint8, device=cuda) for _ in range(3)]
    sentinels += [torch.full((ws1 // 4,), -3.5, device=cuda) for _ in range(3)]
    keep = [s.clone() for s in sentinels]
    _assert_disjoint([plan._ws, out2] + sentinels, held, "workspace growth")
    out1.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out1, want1), "replay at n1 after the workspace grew"
    for i, (s, k) in enumerate(zip(sentinels, keep)):
        assert torch.equal(s, k), "replay wrote into tensor %d allocated after the workspace grew" % i
    assert torch.equal(out2, out2_copy)
    with torch.no_grad():
        assert torch.equal(plan.forward(f1, c1, 1), want1)
    del g


def test_lift_tables_outlive_graph(cuda):
    """capture BEVPoolPlan.lift_pool, call it eagerly with another (cameras, D, fH, fW) key so that the lift tables
    are rebuilt, fill fresh tensors of the old tables' sizes (zeros: harmless as indices): the replay still equals
    eager with the first key and the later call's output is untouched"""
    from bevfusion_b200 import synthetic as S
    from bevfusion_b200.bev_pool import BEVPoolPlan
    geom, cfg = S.camera_geometry("C2", device=cuda)
    plan = BEVPoolPlan(geom, cfg["xbound"], cfg["ybound"], cfg["zbound"])
    g0 = torch.Generator(device=cuda).manual_seed(5)
    depth1 = torch.softmax(torch.randn(1, 6, 118, 32, 88, generator=g0, device=cuda), dim=2).contiguous()
    ctx1 = torch.randn(1, 6, 32, 88, 80, generator=g0, device=cuda)
    with torch.no_grad():
        want1 = plan.lift_pool(depth1, ctx1).clone()
        shapes = [(t.numel(), t.dtype) for t in plan._lift_cache[1][:5]]
        held = [_span(t) for t in plan._lift_cache[1][:5]]
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out1 = plan.lift_pool(depth1, ctx1)
        depth2 = depth1.reshape(1, 12, 59, 32, 88)
        ctx2 = torch.randn(1, 12, 32, 88, 80, generator=g0, device=cuda)
        out2 = plan.lift_pool(depth2, ctx2)
    assert plan._lift_cache[0] == (12, 59, 32, 88)
    out2_copy = out2.clone()
    sentinels = [torch.zeros(n, dtype=dt, device=cuda) for n, dt in shapes for _ in range(2)]
    # checked before the replay: a graph must never read tables whose memory went to someone else
    _assert_disjoint([out2] + sentinels, held, "lift tables rebuilt")
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out1, want1), "replay with the first key after the lift tables were rebuilt"
    assert all(not bool(s.any()) for s in sentinels)
    assert torch.equal(out2, out2_copy)
    del g


# ----------------------------------------------------------------------------- the reference's CUDA kernels
def test_reference_kernels_on_the_frame_inputs(c2):
    """what bench.gpu_reference_leg times, on the frame's own inputs: the reference's voxels equal ours exactly, its
    BEV map is within the per-cell bound and its LiDAR map within 1e-4 x max of float64"""
    bev_ref, vl, sp = (ref_module(n) for n in ("bev_pool_ext_ref", "voxel_layer_ref", "sparse_conv_ext_ref"))
    if bev_ref is None or vl is None or sp is None:
        pytest.skip("oracle/_ref not built")
    from oracle.reference_pipeline import reference_encoder_forward
    hp, dev = c2.hp, c2.device
    t = hp.plan.tables
    xs = c2.x.reshape(-1, 80)[t.perm[:t.n_kept].long()].contiguous()
    torch.cuda.synchronize()
    out = bev_ref.bev_pool_forward(xs, t.geom, t.lengths, t.starts, *t.dims)       # legacy default stream
    torch.cuda.synchronize()
    del xs
    FO.check_pool(out, c2.cam64, "reference bev_pool_forward (seed %d)" % c2.seed)
    L = hp.L
    mv, mp = L["max_voxels"][1], L["max_num_points"]
    voxels = torch.zeros((mv, mp, 5), device=dev)
    coors = torch.zeros((mv, 3), dtype=torch.int32, device=dev)
    num = torch.zeros((mv,), dtype=torch.int32, device=dev)
    n = vl.hard_voxelize(c2.pts, voxels, coors, num, L["voxel_size"], L["point_cloud_range"], mp, mv, 3, True)
    torch.cuda.synchronize()
    _, oc, on, onv = _fused_voxels(hp, c2.pts)
    assert n == int(onv.item()) == c2.lid64["n"]
    assert torch.equal(coors[:n], oc[:n, 1:]) and torch.equal(num[:n], on[:n])
    feats = voxels[:n].sum(dim=1) / num[:n].type_as(voxels).view(-1, 1)
    coords = torch.nn.functional.pad(coors[:n], (1, 0), mode="constant", value=0)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            lid = reference_encoder_forward(sp, hp.encoder, feats, coords, 1)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    torch.cuda.synchronize()
    FO.check_dense(lid, c2.lid64, "reference encoder (seed %d)" % c2.seed)


# ------------------------------------------------------------------------------------ C5 stress configuration
def test_c5_vs_float64(cuda):
    """the C5 HotPath exactly as bench.c5_leg builds it (6 cam 64x176 features, D=200, 256x256 BEV, 4.3 GB volume;
    0.05 m voxels on 2160x2160x41): plan.pool and plan.lift within the per-cell bound of float64 (pooled in row
    slices), _lidar within 1e-4 x max of the float64 encoder with no level cap truncating"""
    lidar = dict(voxel_size=[0.05, 0.05, 0.2], point_cloud_range=[-54.0, -54.0, -5.0, 54.0, 54.0, 3.0],
                 max_num_points=10, max_voxels=(120000, 240000), sparse_shape=[2160, 2160, 41])
    hp = _hotpath(cuda, 0, cfg_name="C5", lidar=lidar)
    cells = FO.CameraCells(hp.geom, hp.cfg)
    x, pts = hp.device_inputs(seed=0)
    FO.check_pool(hp.plan.pool(x), FO.pool64(cells, FO.volume_rows(x), 80, cuda), "C5 pool")
    del x
    torch.cuda.empty_cache()
    depth, ctx = hp.lift_inputs(seed=0, device=cuda)
    FO.check_pool(FO.bev_to_raw(hp.plan.lift(depth, ctx), cells.dims),
                  FO.pool64(cells, FO.lifted_rows(depth, ctx), 80, cuda), "C5 lift", products=True)
    del depth, ctx
    ref = FO.lidar64(hp.L, hp.encoder, hp.points_host.numpy(), cuda)
    print("C5: float64 encoder at %d voxels (CPU-oracle rulebooks included) took %.1f s" % (ref["n"], ref["seconds"]))
    out = hp._lidar(pts)
    FO.check_lidar(out, hp.encoder.plan().status, ref, "C5 lidar")
    feats, coords, num, nv = _fused_voxels(hp, pts)
    FO.check_voxels(feats, coords, num, nv, ref, "C5 sync-free voxelization")
    del hp
    torch.cuda.empty_cache()
