"""oracle -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement (numpy + plain C, oracle/oracle.c) of the reference algorithms of the BEVFusion
hot path.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this package, and only as the checker / reported CPU baseline.  Nothing under
bevfusion_b200/ imports it.

Pinning (the reference tree ships no tests or golden vectors for this path, SURVEY.md section 4):
  * tests/golden/*.npz hold outputs of the reference's OWN code run in the build container:
    its compiled CPU extensions (oracle/_ref, built unmodified from /root/reference by
    oracle/build_ref.py) for voxelization and spconv, and its pure-torch QuickCumsum
    (mmdet3d/ops/bev_pool/bev_pool.py:9-35, the only CPU-capable bev_pool path) for pooling;
    tests/test_oracle_golden.py checks this oracle against them;
  * on the GPU box the tests additionally compare against the reference CUDA kernels
    themselves (oracle/_ref/*.so travel with the repo snapshot).

Each function cites the reference file:line it follows (paths relative to /root/reference).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")
_lib = None


def build():
    """Compile oracle.c -> liboracle.so (gcc, seconds)."""
    src = os.path.join(_HERE, "oracle.c")
    if not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-C", _HERE, "liboracle.so"])
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_LIB_PATH)
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _ivec(v):
    return (ctypes.c_int * len(v))(*[int(x) for x in v])


def _fvec(v):
    return (ctypes.c_float * len(v))(*[float(x) for x in v])


# ------------------------------------------------------------------------------------ bev_pool
def gen_dx_bx(xbound, ybound, zbound):
    """mmdet3d/models/vtransforms/base.py:15-21 (fp32 dx, bx; integer nx by truncation)."""
    rows = [xbound, ybound, zbound]
    dx = np.array([r[2] for r in rows], dtype=np.float32)
    bx = np.array([r[0] + r[2] / 2.0 for r in rows], dtype=np.float32)
    nx = np.array([int((r[1] - r[0]) / r[2]) for r in rows], dtype=np.int64)
    return dx, bx, nx


def quantize_filter(geom, dx, bx, nx, B):
    """base.py:149-169: ((geom - (bx - dx/2)) / dx).long(), batch index column, bounds mask.
    geom [N', 3] fp32 -> coords [N', 4] int64 (x, y, z, b), kept [N'] bool."""
    geom = _f32(geom).reshape(-1, 3)
    lower = (bx.astype(np.float32) - dx.astype(np.float32) / np.float32(2.0)).astype(np.float32)
    q = ((geom - lower) / dx.astype(np.float32))
    with np.errstate(invalid="ignore"):
        idx = np.trunc(q).astype(np.int64)  # .long(): truncation toward zero
    n = geom.shape[0]
    batch_ix = (np.arange(n, dtype=np.int64) // (n // B)).reshape(-1, 1)
    coords = np.concatenate([idx, batch_ix], axis=1)
    kept = ((coords[:, 0] >= 0) & (coords[:, 0] < nx[0]) & (coords[:, 1] >= 0)
            & (coords[:, 1] < nx[1]) & (coords[:, 2] >= 0) & (coords[:, 2] < nx[2])
            & np.isfinite(q).all(axis=1))
    return coords, kept


def ranks_of(coords, B, D, H, W):
    """mmdet3d/ops/bev_pool/bev_pool.py:87-92."""
    c = coords.astype(np.int64)
    return c[:, 0] * (W * D * B) + c[:, 1] * (D * B) + c[:, 2] * B + c[:, 3]


def sort_and_intervals(ranks):
    """bev_pool.py:93 (argsort; stable here) and :41-46 (interval table)."""
    order = np.argsort(ranks, kind="stable")
    rs = ranks[order]
    kept = np.ones(rs.shape[0], dtype=bool)
    kept[1:] = rs[1:] != rs[:-1]
    starts = np.nonzero(kept)[0].astype(np.int32)
    lengths = np.empty_like(starts)
    if starts.size:
        lengths[:-1] = starts[1:] - starts[:-1]
        lengths[-1] = rs.shape[0] - starts[-1]
    return order, rs, starts, lengths


def bev_pool_forward(x, geom_feats, interval_lengths, interval_starts, b, d, h, w, acc64=True):
    """bev_pool_forward, bev_pool_cpu.cpp:22-47 + kernel bev_pool_cuda.cu:20-42 -> [b,d,h,w,c]."""
    x, g = _f32(x), _i32(geom_feats)
    s, l = _i32(interval_starts), _i32(interval_lengths)
    n, c = x.shape
    out = np.zeros((b, d, h, w, c), dtype=np.float32)
    lib().oracle_bev_pool(int(b), int(d), int(h), int(w), int(n), int(c), int(s.shape[0]), _p(x),
                          _p(g), _p(s), _p(l), int(acc64), _p(out))
    return out


def bev_pool_backward(out_grad, geom_feats, interval_lengths, interval_starts, b, d, h, w):
    """bev_pool_backward, bev_pool_cpu.cpp:60-87 + kernel bev_pool_cuda.cu:61-84 -> [n, c]."""
    og, g = _f32(out_grad), _i32(geom_feats)
    s, l = _i32(interval_starts), _i32(interval_lengths)
    n, c = g.shape[0], og.shape[4]
    xg = np.zeros((n, c), dtype=np.float32)
    lib().oracle_bev_pool_grad(int(b), int(d), int(h), int(w), int(n), int(c), int(s.shape[0]),
                               _p(og), _p(g), _p(s), _p(l), _p(xg))
    return xg


def bev_pool(feats, coords, B, D, H, W, acc64=True):
    """bev_pool(), bev_pool.py:84-98 -> [B, C, D, H, W]."""
    ranks = ranks_of(coords, B, D, H, W)
    order, rs, starts, lengths = sort_and_intervals(ranks)
    x = _f32(feats)[order]
    g = coords[order].astype(np.int32)
    out = bev_pool_forward(x, g, lengths, starts, B, D, H, W, acc64)
    return np.ascontiguousarray(out.transpose(0, 4, 1, 2, 3))


def quick_cumsum(x_sorted, ranks_sorted):
    """QuickCumsum.forward, bev_pool.py:9-24 (the reference's only CPU-capable pooling path):
    fp32 cumsum, keep last row of each run, adjacent difference.  Returns [n_intervals, c]."""
    cs = np.cumsum(_f32(x_sorted), axis=0, dtype=np.float32)
    kept = np.ones(cs.shape[0], dtype=bool)
    kept[:-1] = ranks_sorted[1:] != ranks_sorted[:-1]
    cs = cs[kept]
    return np.concatenate([cs[:1], cs[1:] - cs[:-1]], axis=0)


# -------------------------------------------------------------------------------- voxelization
def hard_voxelize(points, voxel_size, coors_range, max_points, max_voxels):
    """hard_voxelize_cpu, voxelization_cpu.cpp:107-144 -> (voxels [M,P,F], coors [M,3] (x,y,z),
    num_points [M], voxel_num)."""
    pts = _f32(points)
    n, nf = pts.shape
    voxels = np.zeros((max_voxels, max_points, nf), dtype=np.float32)
    coors = np.zeros((max_voxels, 3), dtype=np.int32)
    num = np.zeros((max_voxels,), dtype=np.int32)
    m = lib().oracle_hard_voxelize(_p(pts), int(n), int(nf), _fvec(voxel_size), _fvec(coors_range),
                                   int(max_points), int(max_voxels), _p(voxels), _p(coors), _p(num))
    assert m >= 0
    return voxels[:m], coors[:m], num[:m], m


def dynamic_voxelize(points, voxel_size, coors_range):
    """dynamic_voxelize_cpu, voxelization_cpu.cpp:146-171 -> coors [N,3] (-1 rows when OOR)."""
    pts = _f32(points)
    n, nf = pts.shape
    coors = np.zeros((n, 3), dtype=np.int32)
    lib().oracle_dynamic_voxelize(_p(pts), int(n), int(nf), _fvec(voxel_size), _fvec(coors_range),
                                  _p(coors))
    return coors


def voxel_mean(voxels, num_points):
    """BEVFusion.voxelize, bevfusion.py:191-195: feats.sum(dim=1) / sizes."""
    return (voxels.astype(np.float64).sum(axis=1) / num_points.reshape(-1, 1)).astype(np.float32)


_U32 = 2.0 ** -24     # unit roundoff of fp32


def fp32_sum_bound(abs_sum, count, mean_of=None):
    """Error bound of a left-to-right fp32 sum of `count` terms whose absolute values add up to
    `abs_sum` (float64): |fl(sum) - sum| <= g * abs_sum, g = k / (1 - k), k = (count - 1) * 2^-24
    (Higham, Accuracy and Stability, eq. 4.4).  With `mean_of` (the float64 mean) the bound is the
    one of fl(fl(sum) / count): the sum's error over count, plus one rounding of the quotient."""
    count = np.asarray(count, np.float64)
    k = np.maximum(count - 1.0, 0.0) * _U32
    b = k / (1.0 - k) * np.asarray(abs_sum, np.float64)
    if mean_of is not None:
        b = b / count
        b = b + _U32 * (np.abs(mean_of) + b) + 2.0 ** -149
    return b


def assert_within(got, ref64, bound, what=""):
    """Per element: |got - ref64| <= bound where ref64 is finite; identical (inf / NaN included)
    where it is not."""
    got = np.asarray(got, np.float64)
    fin = np.isfinite(ref64)
    assert np.array_equal(got[~fin], ref64[~fin], equal_nan=True), what + ": non-finite elements differ"
    err = np.abs(got[fin] - ref64[fin])
    bad = ~(err <= bound[fin])
    assert not bad.any(), "%s: %d elements outside their bound, worst %g x bound" % (
        what, int(bad.sum()), float(np.nanmax(err[bad] / np.maximum(bound[fin][bad], 1e-300))))


def segment_reduce_f64(feats, seg, m, mean=False):
    """float64 sum (or mean) of the rows of feats [N, C] over segment ids seg [N] (-1 = skipped)
    -> (ref [m, C] float64, bound [m, C]): the fp32 result of adding each segment's rows one at
    a time, in any fixed order, lies within `bound` of `ref` (fp32_sum_bound)."""
    x = np.asarray(feats, np.float64)
    seg = np.asarray(seg, np.int64)
    keep = seg >= 0
    ref = np.zeros((m, x.shape[1]))
    mag = np.zeros((m, x.shape[1]))
    with np.errstate(invalid="ignore"):
        np.add.at(ref, seg[keep], x[keep])
        np.add.at(mag, seg[keep], np.abs(x[keep]))
    count = np.bincount(seg[keep], minlength=m).astype(np.float64)[:, None]
    if mean:
        with np.errstate(invalid="ignore", divide="ignore"):
            ref = ref / count
        return ref, fp32_sum_bound(mag, count, mean_of=ref)
    return ref, fp32_sum_bound(mag, count)


def dynamic_scatter(feats, coors, reduce_type="max"):
    """dynamic_point_to_voxel_forward (scatter_points_cuda.cu:187-241): rows with a negative
    entry are masked to -1 (:203), at::unique_dim sorts the rows lexicographically (:206-208) and
    the leading all -1 row is removed (:210-215); features are reduced per voxel (sum / mean in
    fp64 here, so the comparison with either GPU implementation is a tolerance one; max is exact).
    The reference's max is a CAS loop on fmaxf starting from -inf (:22-30, :223), so NaN features
    are ignored and a voxel holding only NaN reduces to -inf.
    Returns (reduced [M, C] f32, out_coors [M, ndim] i32, coors_map [N] i32, count [M] i32).
    PINNING: the reference has no CPU path for this op (voxelization.h:118); the restatement is
    checked on the GPU box against oracle/_ref's voxel_layer (tests/test_voxelize_gpu.py)."""
    feats = np.asarray(feats, np.float32)
    coors = np.asarray(coors, np.int32)
    n, c = feats.shape
    if n == 0:
        return feats.copy(), coors.copy(), np.zeros(0, np.int32), np.zeros(0, np.int32)
    clean = coors.copy()
    clean[(coors < 0).any(1)] = -1
    out_coors, inv, count = np.unique(clean, axis=0, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1).astype(np.int64)
    if out_coors[0, 0] < 0:
        out_coors, count, inv = out_coors[1:], count[1:], inv - 1
    m = out_coors.shape[0]
    keep = inv >= 0
    if reduce_type == "max":
        red = np.full((m, c), -np.inf, np.float32)
        np.fmax.at(red, inv[keep], feats[keep])     # fmaxf (:22-30): a NaN never replaces a number
    else:
        red = np.zeros((m, c), np.float64)
        np.add.at(red, inv[keep], feats[keep].astype(np.float64))
        if reduce_type == "mean":
            red = red / count[:, None]
        red = red.astype(np.float32)
    return red, out_coors.astype(np.int32), inv.astype(np.int32), count.astype(np.int32)


def dynamic_scatter_backward(grad_reduced, feats, reduced, coors_map, count, reduce_type="max"):
    """dynamic_point_to_voxel_backward (scatter_points_cuda.cu:243-315)."""
    feats = np.asarray(feats, np.float32)
    g = np.zeros_like(feats)
    keep = coors_map >= 0
    if reduce_type in ("sum", "mean"):
        g[keep] = grad_reduced[coors_map[keep]]
        if reduce_type == "mean":
            g[keep] /= count[coors_map[keep]][:, None].astype(np.float32)
        return g
    m, c = reduced.shape
    n = feats.shape[0]
    frm = np.full((m, c), n, np.int64)                       # :286 full(num_input)
    pts = np.nonzero(keep)[0]
    seg = np.asarray(coors_map, np.int64)[pts]
    hit = feats[pts] == np.asarray(reduced)[seg]             # :162 (NaN never equals the maximum)
    np.minimum.at(frm, seg, np.where(hit, pts[:, None], n))  # :163 smallest index attaining the max
    v, ch = np.nonzero(frm < n)
    g[frm[v, ch], ch] = np.asarray(grad_reduced)[v, ch]
    return g


# ----------------------------------------------------------------------------- depth images
def _dot3(m, x, y, z):
    f = np.float32
    return f(f(f(m[0] * x) + f(m[1] * y)) + f(m[2] * z))


def _inverse3(a):
    """3x3 inverse by the adjugate, fp32 op by op (stands in for torch.inverse, base.py:291)."""
    a = np.asarray(a, np.float32).reshape(9)
    f = np.float32
    c00 = f(f(a[4] * a[8]) - f(a[5] * a[7]))
    c01 = f(f(a[3] * a[8]) - f(a[5] * a[6]))
    c02 = f(f(a[3] * a[7]) - f(a[4] * a[6]))
    det = f(f(f(a[0] * c00) - f(a[1] * c01)) + f(a[2] * c02))
    inv = [c00 / det, f(f(a[2] * a[7]) - f(a[1] * a[8])) / det, f(f(a[1] * a[5]) - f(a[2] * a[4])) / det,
           f(-c01) / det, f(f(a[0] * a[8]) - f(a[2] * a[6])) / det, f(f(a[2] * a[3]) - f(a[0] * a[5])) / det,
           c02 / det, f(f(a[1] * a[6]) - f(a[0] * a[7])) / det, f(f(a[0] * a[4]) - f(a[1] * a[3])) / det]
    return np.asarray(inv, np.float32)


def points_to_depth(points, lidar2image, img_aug_matrix, lidar_aug_matrix, image_size,
                    depth_input="scalar", depth_bins=None, add_depth_features=False):
    """BaseDepthTransform.forward's depth image for ONE sample (base.py:279-329): points [N, F],
    lidar2image / img_aug_matrix [ncam, 4, 4], lidar_aug_matrix [4, 4] -> [ncam, channels, H, W].
    Every step is an explicit fp32 operation in the reference's order (inverse aug :290-293,
    lidar2image :295-296, clamp + divide :298-300, image aug :303-305, on-image test :309-314,
    .long() :316).  Colliding points: the last one (largest index) wins -- the sequential reading of
    the index_put at :319.  Like the reference after its in-place `cur_coords -= trans` (:290), the
    optional feature channels (:327-329) carry xyz minus the lidar-aug translation."""
    f = np.float32
    pts = np.asarray(points, np.float32)
    n, nf = pts.shape
    H, W = int(image_size[0]), int(image_size[1])
    la = np.asarray(lidar_aug_matrix, np.float32)
    l2i = np.asarray(lidar2image, np.float32)
    ia = np.asarray(img_aug_matrix, np.float32)
    ncam = l2i.shape[0]
    one_hot = depth_input == "one-hot"
    feat = nf if add_depth_features else 0
    channels = (int(depth_bins) if one_hot else 1) + feat
    depth = np.zeros((ncam, channels, H, W), np.float32)
    inv = _inverse3(la[:3, :3])
    with np.errstate(all="ignore"):
        x1, y1, z1 = (pts[:, 0] - la[0, 3]).astype(f), (pts[:, 1] - la[1, 3]).astype(f), (pts[:, 2] - la[2, 3]).astype(f)
        x2, y2, z2 = _dot3(inv[0:3], x1, y1, z1), _dot3(inv[3:6], x1, y1, z1), _dot3(inv[6:9], x1, y1, z1)
        shifted = pts.copy()
        shifted[:, 0], shifted[:, 1], shifted[:, 2] = x1, y1, z1
        for cam in range(ncam):
            L, A = l2i[cam], ia[cam]
            x3 = f(_dot3(L[0, :3], x2, y2, z2) + L[0, 3])
            y3 = f(_dot3(L[1, :3], x2, y2, z2) + L[1, 3])
            z3 = f(_dot3(L[2, :3], x2, y2, z2) + L[2, 3])
            z3 = np.minimum(np.maximum(z3, f(1e-5)), f(1e5)).astype(f)
            x3, y3 = (x3 / z3).astype(f), (y3 / z3).astype(f)
            u = f(_dot3(A[0, :3], x3, y3, z3) + A[0, 3])
            v = f(_dot3(A[1, :3], x3, y3, z3) + A[1, 3])
            on = (v < f(H)) & (v >= 0) & (u < f(W)) & (u >= 0)
            idx = np.nonzero(on)[0]                          # ascending: later points overwrite
            row, col = v[idx].astype(np.int64), u[idx].astype(np.int64)
            if one_hot:
                bins = np.minimum(z3[idx], f(depth_bins - 1)).astype(np.int64)
                depth[cam, bins, row, col] = 1.0
            else:
                depth[cam, 0, row, col] = z3[idx]           # numpy fancy assignment: last write wins
            if feat:
                depth[cam, channels - feat:, row, col] = shifted[idx]   # result dims: (point, channel)
    return depth


# ------------------------------------------------------------------------------------- spconv
def conv_output_size(input_size, kernel_size, stride, padding, dilation):
    """get_conv_output_size, mmdet3d/ops/spconv/ops.py:20-31."""
    return [(input_size[i] + 2 * padding[i] - dilation[i] * (kernel_size[i] - 1) - 1) // stride[i] + 1
            for i in range(len(input_size))]


def get_indice_pairs(indices, batch_size, spatial_shape, ksize, stride, padding, dilation, subm):
    """getIndicePair<3> CPU branch, spconv_ops.h:27-141 -> (outids [M,4], indice_pairs [K,2,N],
    indice_num [K], out_shape).  Strided convs number outputs in first-encounter order
    (geometry.h:144-194); the reference GPU path orders them by ascending flat index."""
    ind = _i32(indices)
    n = ind.shape[0]
    kvol = int(np.prod(ksize))
    pairs = np.full((kvol, 2, n), -1, dtype=np.int32)
    num = np.zeros((kvol,), dtype=np.int32)
    if subm:
        out_shape = list(spatial_shape)
        lib().oracle_indice_pairs_subm(_p(ind), n, _ivec(ksize), _ivec(dilation), _ivec(out_shape),
                                       _p(pairs), _p(num))
        return ind.copy(), pairs, num, out_shape
    out_shape = conv_output_size(spatial_shape, ksize, stride, padding, dilation)
    outids = np.zeros((max(n * kvol, 1), 4), dtype=np.int32)
    m = lib().oracle_indice_pairs_conv(_p(ind), n, _ivec(ksize), _ivec(stride), _ivec(padding),
                                       _ivec(dilation), _ivec(out_shape), _p(outids), _p(pairs),
                                       _p(num))
    assert m >= 0
    return outids[:m].copy(), pairs, num, out_shape


def indice_conv(features, filters, indice_pairs, indice_num, num_act_out, inverse=False,
                subm=False, acc64=True):
    """indiceConv<float>, spconv_ops.h:260-361 -> [num_act_out, Cout]."""
    f, w = _f32(features), _f32(filters)
    n_in, c_in = f.shape
    c_out = w.shape[-1]
    pairs, num = _i32(indice_pairs), _i32(indice_num)
    kvol, _, pdim = pairs.shape
    out = np.zeros((num_act_out, c_out), dtype=np.float32)
    lib().oracle_indice_conv(_p(f), _p(w), _p(pairs), _p(num), int(n_in), int(num_act_out),
                             int(c_in), int(c_out), int(kvol), int(pdim), int(subm), int(inverse),
                             int(acc64), _p(out))
    return out


def indice_conv_backward(features, filters, out_bp, indice_pairs, indice_num, inverse=False):
    """indiceConvBackward<float>, spconv_ops.h:363-456 -> (input_grad [N,Cin], filters_grad
    [K,Cin,Cout]) in float64 arithmetic: per offset k and pair (in, out):
    filters_grad[k] += f[in]^T (x) g[out];  input_grad[in] += g[out] @ W[k]^T."""
    f, g = features.astype(np.float64), out_bp.astype(np.float64)
    w = filters.reshape(-1, filters.shape[-2], filters.shape[-1]).astype(np.float64)
    din = np.zeros_like(f)
    dw = np.zeros_like(w)
    for k in range(w.shape[0]):
        n = int(indice_num[k])
        if n <= 0:
            continue
        a, b = indice_pairs[k, 1 if inverse else 0, :n], indice_pairs[k, 0 if inverse else 1, :n]
        dw[k] = f[a].T @ g[b]
        np.add.at(din, a, g[b] @ w[k].T)
    return din.astype(np.float32), dw.reshape(filters.shape).astype(np.float32)


def flat_index(outids, out_shape):
    """((b*X + x)*Y + y)*Z + z -- the order of the reference GPU rulebook (indice.cu.h:59-60)."""
    o = outids.astype(np.int64)
    return ((o[:, 0] * out_shape[0] + o[:, 1]) * out_shape[1] + o[:, 2]) * out_shape[2] + o[:, 3]


def sparse_conv(features, indices, batch_size, spatial_shape, filters, ksize, stride, padding,
                dilation, subm, acc64=True):
    """SparseConvolution.forward core (conv.py:152-216) with outputs re-ordered to ascending
    flat index for strided convs.  Returns (out_features, outids, out_shape)."""
    outids, pairs, num, out_shape = get_indice_pairs(indices, batch_size, spatial_shape, ksize,
                                                     stride, padding, dilation, subm)
    out = indice_conv(features, filters.reshape(-1, filters.shape[-2], filters.shape[-1]), pairs,
                      num, outids.shape[0], False, subm, acc64)
    if not subm:
        order = np.argsort(flat_index(outids, out_shape), kind="stable")
        out, outids = out[order], outids[order]
    return out, outids, out_shape


def dense(features, indices, batch_size, spatial_shape):
    """SparseConvTensor.dense(), structure.py:49-59 -> [B, C, X, Y, Z]."""
    X, Y, Z = spatial_shape
    c = features.shape[1]
    out = np.zeros((batch_size, X, Y, Z, c), dtype=features.dtype)
    idx = indices.astype(np.int64)
    out[idx[:, 0], idx[:, 1], idx[:, 2], idx[:, 3]] = features
    return np.ascontiguousarray(out.transpose(0, 4, 1, 2, 3))
