"""Dev tool: small invocations of every kernel family, meant to run under compute-sanitizer."""
import os, sys
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import numpy as np, torch
import __graft_entry__ as g
g.smoke()
from bevfusion_b200.bev_pool import bev_pool, bev_pool_ext
from bevfusion_b200.spconv import ops
dev = torch.device("cuda:0")
rng = np.random.default_rng(0)
# drop-in bev_pool fwd+bwd with long intervals, odd channel count (generic kernel) and tuned width
for c in (80, 7):
    n, B, D, H, W = 5000, 2, 2, 9, 7
    coords = torch.from_numpy(np.stack([rng.integers(0, H, n), rng.integers(0, W, n), rng.integers(0, D, n),
                                        rng.integers(0, B, n)], 1)).to(dev)
    x = torch.randn(n, c, device=dev, requires_grad=True)
    out = bev_pool(x, coords, B, D, H, W)
    out.sum().backward()
# sparse conv fwd/bwd, all precisions, strided + subm
shape, Bn, n = [20, 18, 7], 2, 1500
vol = Bn * shape[0] * shape[1] * shape[2]
flat = rng.choice(vol, size=n, replace=False)
idx = np.stack([flat // (shape[0] * shape[1] * shape[2]), (flat // (shape[1] * shape[2])) % shape[0],
                (flat // shape[2]) % shape[1], flat % shape[2]], 1).astype(np.int32)
ti = torch.from_numpy(idx).to(dev)
for (cin, cout) in ((16, 32), (64, 64), (5, 16), (64, 128)):
    f = torch.randn(n, cin, device=dev)
    for subm, ks, st, pd in ((True, 3, 1, 1), (False, 3, 2, 1), (False, [1, 1, 3], [1, 1, 2], 0)):
        rb, _ = ops.get_rulebook(ti, Bn, shape, ks, st, pd, 1, 0, subm)
        kv = rb.nbr.shape[0]
        w = torch.randn(kv, cin, cout, device=dev)
        for prec in (0, 1, 2, 3):
            o = ops.sparse_conv(f, w, rb.nbr, rb.n_out, precision=prec)
        o = ops.sparse_conv(f, w, rb.nbr, rb.n_out, precision=3, packed=ops.pack_weights(w, 3))
        ops.sparse_conv_backward(f, w, torch.randn_like(o), rb.nbr, precision=1)
        ops.sparse_conv_backward(f, w, torch.randn_like(o), rb.nbr, precision=3)     # tensor-core filter gradient
        rb.pairs()
# tensor-core filter gradient at the remaining slab counts (32 / 128 channels on either side)
for (cin, cout) in ((32, 32), (32, 64), (128, 128), (64, 128)):
    f = torch.randn(n, cin, device=dev)
    rb, _ = ops.get_rulebook(ti, Bn, shape, 3, 1, 1, 1, 0, True)
    w = torch.randn(27, cin, cout, device=dev)
    ops.sparse_conv_backward(f, w, torch.randn(rb.n_out, cout, device=dev), rb.nbr, precision=3)
# fused voxelize + mean, DynamicScatter fwd / bwd (all reductions), LiDAR depth images, in-place layouts
from bevfusion_b200 import synthetic as S
from bevfusion_b200.scatter_points import dynamic_scatter
from bevfusion_b200.voxelize import voxel_layer, voxelize_mean_fused
from bevfusion_b200.vtransform import points_to_depth
vs, cr = [0.4, 0.5, 0.25], [-8.0, -6.0, -1.0, 8.0, 6.0, 3.0]
pts = torch.from_numpy(S.uniform_cloud(3000, seed=1, margin=1.0, rng_range=cr)).to(dev)
voxelize_mean_fused(pts, vs, cr, 4, 500, 1)
coors = torch.zeros(pts.shape[0], 3, dtype=torch.int32, device=dev)
voxel_layer.dynamic_voxelize(pts, coors, vs, cr, 3)
for red in ("sum", "mean", "max"):
    p = pts.clone().requires_grad_(True)
    vf, vc = dynamic_scatter(p, coors, red)
    vf.sum().backward()
M = S.lidar_camera_matrices(2, (64, 176), batch=1)
for kw in (dict(), dict(depth_input="one-hot", depth_bins=20, add_depth_features=True)):
    points_to_depth([pts], M["lidar2image"].to(dev), M["img_aug_matrix"].to(dev), M["lidar_aug_matrix"].to(dev), (64, 176), **kw)
buf = torch.zeros(2, 3 + 16 * 7, 20, 18, device=dev)
ops.sparse_to_dense(torch.randn(n, 16, device=dev), ti, Bn, shape, z_major=True, out=buf[:, 3:])
torch.cuda.synchronize()
print("sanitize_small ok")
