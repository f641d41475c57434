"""Dev tool: the nine sparse-conv layer shapes of the SparseEncoder on the real C3 rulebooks (synthetic
lidar_cloud(seed=0)), each run alone through bevb200_spconv_forward_split (BF16x3, the encoder's kernel).
Per shape: n_out, pairs, kernel time (CUDA events over >= 1 s windows), useful TFLOP/s (real pairs) and issued
TFLOP/s (dense-K implicit GEMM x 3 bf16 products), and the max relative difference against the exact-fp32
SIMT path (precision 0).
    python tools/conv_layers.py [--window SECONDS]"""
import argparse
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import torch  # noqa: E402

from bevfusion_b200 import _C, synthetic as S  # noqa: E402
from bevfusion_b200.spconv import ops  # noqa: E402
from bevfusion_b200.voxelize import Voxelization, voxelize_mean  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--window", type=float, default=1.0, help="seconds per timing window")
args = ap.parse_args()

dev = torch.device("cuda:0")
lib = _C.lib()
L = S.LIDAR_C3
pts = torch.from_numpy(S.lidar_cloud(seed=0)).to(dev)
vox = Voxelization(L["voxel_size"], L["point_cloud_range"], L["max_num_points"], L["max_voxels"]).eval()
v, c, n = vox(pts)
_, idx = voxelize_mean(v, c, n, 0)
shape = L["sparse_shape"]


def time_us(fn, window):
    """median over three windows of >= `window` seconds, each timed with CUDA events"""
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); torch.cuda.synchronize()
    reps = max(1, int(window * 1e3 / max(a.elapsed_time(b), 1e-3)))
    ts = []
    for _ in range(3):
        a.record()
        for _ in range(reps):
            fn()
        b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3 / reps)
    return sorted(ts)[1]


layers = [("conv_input", 5, 16, True, 3, 1, 1, 1), ("s1 subm", 16, 16, True, 3, 1, 1, 4),
          ("s1 down", 16, 32, False, 3, 2, 1, 1), ("s2 subm", 32, 32, True, 3, 1, 1, 4),
          ("s2 down", 32, 64, False, 3, 2, 1, 1), ("s3 subm", 64, 64, True, 3, 1, 1, 4),
          ("s3 down", 64, 128, False, 3, 2, [1, 1, 0], 1), ("s4 subm", 128, 128, True, 3, 1, 1, 4),
          ("conv_out", 128, 128, False, [1, 1, 3], [1, 1, 2], 0, 1)]
print(torch.cuda.get_device_name(0), flush=True)
print(f"{'layer':10s} {'cin->cout':>9s} {'n_out':>8s} {'pairs':>9s} {'us':>8s} {'useful TF/s':>11s} "
      f"{'issued TF/s':>11s} {'max rel diff':>12s}  launches", flush=True)
total = 0.0
for name, cin, cout, subm, ks, st, pd, mult in layers:
    rb, oshape = ops.get_rulebook(idx, 1, shape, ks, st, pd, 1, 0, subm)
    n_in, kv = idx.shape[0], rb.nbr.shape[0]
    g = torch.Generator(device=dev).manual_seed(cin * 1000 + cout)
    f = torch.randn(n_in, cin, device=dev, generator=g)
    w = torch.randn(kv, cin, cout, device=dev, generator=g) / (cin * kv) ** 0.5
    scale = torch.rand(cout, device=dev, generator=g) + 0.5
    shift = torch.randn(cout, device=dev, generator=g) * 0.1
    ce = lib.bevb200_spconv_split_channels(cin)
    fs = torch.empty((n_in, ce * 4), dtype=torch.uint8, device=dev)
    _C.check(lib.bevb200_spconv_split_rows(_C.ptr(f), n_in, 0, cin, _C.ptr(fs), _C.current_stream(dev)), "split_rows")
    pk = torch.empty(lib.bevb200_spconv_split_weight_bytes(cin, cout, kv), dtype=torch.uint8, device=dev)
    _C.check(lib.bevb200_spconv_pack_split_weights(_C.ptr(w), cin, cout, kv, _C.ptr(pk), _C.current_stream(dev)), "pack")
    out = torch.empty((rb.n_out, cout), device=dev)
    osp = torch.empty((rb.n_out, cout * 4), dtype=torch.uint8, device=dev)

    def run():
        _C.check(lib.bevb200_spconv_forward_split(_C.ptr(fs), _C.ptr(pk), _C.ptr(rb.nbr), rb.n_out, n_in, rb.n_out, 0,
                                                  ce, cout, kv, _C.ptr(scale), _C.ptr(shift), 0, 1, _C.ptr(out),
                                                  _C.ptr(osp), _C.current_stream(dev)), "forward_split")
    run()
    exact = ops.sparse_conv(f, w, rb.nbr, rb.n_out, scale, shift, None, True, precision=0)
    torch.cuda.synchronize()
    diff = (out - exact).abs().max().item() / max(exact.abs().max().item(), 1e-30)
    us = time_us(run, args.window)
    total += us * mult
    pairs = int((rb.nbr >= 0).sum())
    nkb = (kv * ce + 31) // 32
    useful = 2.0 * pairs * cin * cout / (us * 1e-6) / 1e12
    issued = 3 * 2.0 * rb.n_out * nkb * 32 * cout / (us * 1e-6) / 1e12
    print(f"{name:10s} {cin:4d}->{cout:<4d} {rb.n_out:8d} {pairs:9d} {us:8.1f} {useful:11.1f} {issued:11.1f} "
          f"{diff:12.2e}  x{mult}", flush=True)
    del exact, out, osp, fs, pk
    if not subm:
        idx, shape = rb.outids, oshape
print(f"sum over the 21 launches of a frame: {total / 1e3:.3f} ms", flush=True)
