"""Float64 references of the benchmarked frame (bench.HotPath.frame / frame_lift), for tests/test_frame_gpu.py.

  * camera branch: the frustum geometry quantised by the CPU oracle (oracle.quantize_filter, independent of the
    plan's tables), then the kept rows of the lifted volume -- or of depth (x) ctx formed in float64 -- pooled per
    cell with index_add_ on the device, in row slices.  Besides the float64 sum it keeps sum |row| and the row count
    of every cell: the per-cell fp32 error bound (oracle.fp32_sum_bound).
  * LiDAR branch: oracle.hard_voxelize (the C port) and the per-voxel mean in float64, then
    encoder_oracle.encoder_forward on a float64 copy of the encoder with rulebooks from the CPU oracle."""
import copy
import time

import numpy as np
import torch

import encoder_oracle
import oracle


class CameraCells:
    """Kept rows of a camera geometry [B, N, D, fH, fW, 3] and the pooled cell of each, as the CPU oracle
    quantises them; cells are numbered in the raw op layout [B, nz, nx, ny]."""

    def __init__(self, geom, cfg):
        dx, bx, nx = oracle.gen_dx_bx(cfg["xbound"], cfg["ybound"], cfg["zbound"])
        B = int(geom.shape[0])
        coords, kept = oracle.quantize_filter(geom.cpu().numpy(), dx, bx, nx, B)
        nz, X, Y = int(nx[2]), int(nx[0]), int(nx[1])
        rows = np.nonzero(kept)[0]
        c = coords[rows]
        self.rows = torch.from_numpy(rows)
        self.cell = torch.from_numpy(((c[:, 3] * nz + c[:, 2]) * X + c[:, 0]) * Y + c[:, 1])
        self.dims = (B, nz, X, Y)
        self.n_cells = B * nz * X * Y


def volume_rows(x):
    """rows r of the lifted volume x [B, N, D, fH, fW, C] in float64"""
    x2 = x.reshape(-1, x.shape[-1])
    return lambda r: x2[r].double()


def lifted_rows(depth, ctx):
    """rows r of depth.unsqueeze(-1) * ctx.unsqueeze(2) (depth [B, N, D, fH, fW], ctx [B, N, fH, fW, C]), the
    products formed in float64"""
    _, _, D, fH, fW = depth.shape
    d1 = depth.reshape(-1)
    c2 = ctx.reshape(-1, ctx.shape[-1])

    def rows(r):
        cam, hw = r // (D * fH * fW), r % (fH * fW)
        return d1[r].double().unsqueeze(1) * c2[cam * (fH * fW) + hw].double()
    return rows


def pool64(cells, row_values, C, device, chunk=1 << 21):
    """(sum, sum |.|, row count) per cell in float64 on the device, pooling the kept rows `chunk` at a time
    (the C5 volume is 4.3 GB: its float64 copy is never formed whole)."""
    s = torch.zeros(cells.n_cells, C, dtype=torch.float64, device=device)
    a = torch.zeros_like(s)
    cnt = torch.zeros(cells.n_cells, dtype=torch.float64, device=device)
    for i in range(0, cells.rows.numel(), chunk):
        r = cells.rows[i:i + chunk].to(device)
        k = cells.cell[i:i + chunk].to(device)
        v = row_values(r)
        s.index_add_(0, k, v)
        a.index_add_(0, k, v.abs())
        cnt.index_add_(0, k, torch.ones(k.numel(), dtype=torch.float64, device=device))
    return s, a, cnt


def check_pool(got, ref, what, products=False):
    """got: the raw op output [B, nz, nx, ny, C] (fp32).  Every element within the fp32 summation bound of its
    cell; cells no row reaches exactly 0.  products=True: each term is itself an fp32 product, one more rounding
    per term, i.e. the bound of count + 1 terms."""
    s, a, cnt = ref
    C = s.shape[1]
    g = got.reshape(-1, C)
    assert g.shape[0] == s.shape[0], what + ": cell count"
    empty = cnt == 0
    assert not bool(g[empty].any()), what + ": a cell no row reaches is not 0"
    terms = (cnt + 1.0) if products else cnt
    bound = oracle.fp32_sum_bound(a.cpu().numpy(), terms.cpu().numpy()[:, None])
    oracle.assert_within(g.cpu().numpy(), s.cpu().numpy(), bound, what)


def bev_to_raw(bev, dims):
    """[B, nz*C, nx, ny] module layout -> raw op layout [B, nz, nx, ny, C] (channel z*C + c)"""
    B, nz, X, Y = dims
    return bev.reshape(B, nz, -1, X, Y).permute(0, 1, 3, 4, 2)


def float64_encoder(encoder):
    """copy.deepcopy(encoder).double() without copying the native plan (it owns a library handle) or streams"""
    memo = {id(v): None for k, v in vars(encoder).items() if k in ("_plan", "_rulebook_streams")}
    return copy.deepcopy(encoder, memo).double().eval()


def lidar64(L, encoder, points, device):
    """The LiDAR branch in float64: hard voxelization by the C port, per-voxel mean, SparseEncoder.
    -> dict(coors (b, x, y, z) int32 [M, 4], num [M], mean [M, F] and abs_sum [M, F] float64, dense, active, rows,
    seconds: wall time of the float64 encoder, CPU rulebooks included)"""
    vox, c, num, m = oracle.hard_voxelize(points, L["voxel_size"], L["point_cloud_range"], L["max_num_points"],
                                          L["max_voxels"][1])
    mean = vox.astype(np.float64).sum(axis=1) / num.reshape(-1, 1)
    coors = np.concatenate([np.zeros((m, 1), np.int32), c], axis=1)
    m64 = float64_encoder(encoder)
    t0 = time.perf_counter()
    dense, active, rows = encoder_oracle.encoder_forward(m64, torch.from_numpy(mean).to(device),
                                                         torch.from_numpy(coors), 1)
    if torch.device(device).type == "cuda":
        torch.cuda.synchronize(device)
    return dict(coors=coors, num=num, mean=mean, abs_sum=np.abs(vox.astype(np.float64)).sum(axis=1), n=int(m),
                dense=dense, active=active.to(device), rows=rows,
                seconds=time.perf_counter() - t0)


def check_voxels(feats, coords, num, nv, ref, what):
    """the sync-free voxelizer's cap buffers against the C port: count and coordinates exact, the first nv rows'
    means within one fp32 mean of at most max_points terms"""
    n = int(nv.item())
    assert n == ref["n"], "%s: %d voxels, oracle %d" % (what, n, ref["n"])
    assert np.array_equal(coords[:n].cpu().numpy(), ref["coors"]), what + ": voxel coordinates"
    assert np.array_equal(num[:n].cpu().numpy(), ref["num"]), what + ": points per voxel"
    bound = oracle.fp32_sum_bound(ref["abs_sum"], ref["num"].reshape(-1, 1), mean_of=ref["mean"])
    oracle.assert_within(feats[:n].cpu().numpy(), ref["mean"], bound, what + ": voxel means")


def check_lidar(out, status, ref, what):
    """encoder output [1, 256, X, Y] and the plan's status word against the float64 restatement"""
    check_dense(out, ref, what)
    st = status.cpu().tolist()
    assert st[0] == 0, what + ": a level cap truncated the encoder (status %s)" % st
    assert st[1:] == ref["rows"], "%s: rows per level %s, float64 restatement %s" % (what, st[1:], ref["rows"])


def check_dense(out, ref, what):
    gold = ref["dense"]
    assert tuple(out.shape) == tuple(gold.shape), what + ": shape"
    scale = float(gold.abs().max())
    err = float((out.double() - gold).abs().max())
    assert err <= 1e-4 * scale, "%s: max error %g > 1e-4 x %g" % (what, err, scale)
    agree = float(((out != 0) == (gold != 0)).double().mean())
    assert agree >= 0.9999, "%s: non-zero pattern agrees on %.6f of the elements" % (what, agree)
    assert not bool(out[~ref["active"]].any()), what + ": an element of an inactive cell is not 0"
