"""DynamicScatter at its edges: every key width, tile-boundary point counts, one voxel holding
every point, features full of ties, cancellation and infinities.  Voxel ids, counts and max are exact
against the oracle; sum / mean are held to the per-element bound of an ordered fp32 sum; the two max
backward implementations must agree bit for bit."""
import numpy as np
import pytest
import torch

import oracle
from conftest import ref_module

pytestmark = pytest.mark.gpu

SIZES = [1, 31, 4095, 4096, 4097, 8193, 100003]          # around the scan's 4096-element tiles
OCCUPANCY = ["one_voxel", "eight_per_voxel", "all_distinct", "all_invalid", "ends_invalid"]
FAMILIES = ["gauss", "quantised", "cancelling", "special"]
NDIMS = [1, 2, 3, 4]
CHANNELS = [1, 3, 5, 64, 128]
REDUCE = ["sum", "mean", "max"]
LARGE_N = 4096 * 1024 + 4097


def key_limit(ndim):
    """Coordinates must be below this: 20 bits per column, 15 with four columns."""
    return 1 << (20 if ndim <= 3 else 15)


def make_coors(n, ndim, occupancy, rng):
    """[n, ndim] int32 rows spread over the whole key range of every column."""
    lim = key_limit(ndim)
    space = lim ** ndim
    k = {"one_voxel": 1, "all_distinct": n}.get(occupancy, max(n // 8, 1))
    flat = np.unique(rng.integers(0, space, 2 * k + 64))
    while len(flat) < k:
        flat = np.unique(np.concatenate([flat, rng.integers(0, space, 2 * k)]))
    flat = rng.permutation(flat)[:k]
    ids = rng.permutation(n) if occupancy == "all_distinct" else rng.integers(0, k, n)
    f = flat[ids]
    cols = []
    for _ in range(ndim):
        cols.append(f % lim)
        f = f // lim
    coors = np.stack(cols[::-1], axis=1).astype(np.int32)
    if occupancy == "all_invalid":
        coors[np.arange(n), rng.integers(0, ndim, n)] = -1 - rng.integers(0, 5, n).astype(np.int32)
    elif occupancy == "ends_invalid":
        coors[0, 0] = -1
        coors[-1, ndim - 1] = -7
    return coors


def make_feats(n, c, family, rng):
    if family == "quantised":                                # 4 levels: ties in every voxel
        return rng.integers(0, 4, (n, c)).astype(np.float32) - 1.0
    x = rng.standard_normal((n, c)).astype(np.float32)
    if family == "cancelling":                               # +-1e6 in pairs, small terms between them
        big = np.where(np.arange(n) % 2 == 0, 1e6, -1e6).astype(np.float32)[:, None]
        x = np.where(rng.random((n, c)) < 0.5, big, x * np.float32(1e-3)).astype(np.float32)
    elif family == "special":
        x[:, 0] = -np.inf
        if c > 1:
            x[:, 1] = 2.5                                    # constant column: every point ties
        if c > 2:
            x[:, 2] = np.where(rng.random(n) < 0.5, 0.0, -0.0)
        if c > 3:
            x[rng.random(n) < 0.3, 3] = -np.inf
    return np.ascontiguousarray(x)


def cases():
    """One case per (size, occupancy); ndim, channels and family rotate so that every value of each
    meets every size and every occupancy."""
    out = []
    for i, n in enumerate(SIZES):
        for j, occ in enumerate(OCCUPANCY):
            t = i * len(OCCUPANCY) + j
            out.append((n, occ, NDIMS[(i + j) % 4], CHANNELS[(i + 2 * j) % 5], FAMILIES[t % 4]))
    return out


def case_id(c):
    return "n%d-%s-d%d-c%d-%s" % c


def build(case):
    n, occ, ndim, c, family = case
    rng = np.random.default_rng(n * 131 + ndim * 17 + c)
    return make_feats(n, c, family, rng), make_coors(n, ndim, occ, rng), rng


def order_preserving_permutation(seg, rng):
    """A random permutation of the points that keeps the order of the points INSIDE each voxel:
    row k of the permuted arrays is original row src[k]."""
    perm = rng.permutation(len(seg))
    pos = np.argsort(seg[perm], kind="stable")               # positions, grouped by voxel
    by_voxel = np.argsort(seg, kind="stable")                # points, grouped by voxel, ascending index
    src = np.empty(len(seg), np.int64)
    src[pos] = by_voxel
    return src


def forward(cuda, feats, coors, reduce_type):
    from bevfusion_b200.voxelize import voxel_layer
    return voxel_layer.dynamic_point_to_voxel_forward(
        torch.from_numpy(feats).to(cuda), torch.from_numpy(coors).to(cuda), reduce_type)


def assert_reduced(red, feats, g_map, m, reduce_type, g_red):
    if reduce_type == "max":
        assert np.array_equal(red, g_red)
    else:
        with np.errstate(invalid="ignore"):
            ref, bound = oracle.segment_reduce_f64(feats, g_map, m, mean=reduce_type == "mean")
        oracle.assert_within(red, ref, bound, reduce_type)


@pytest.mark.parametrize("reduce_type", REDUCE)
@pytest.mark.parametrize("case", cases(), ids=case_id)
def test_forward(cuda, case, reduce_type):
    feats, coors, rng = build(case)
    red, oc, cmap, cnt = forward(cuda, feats, coors, reduce_type)
    g_red, g_oc, g_map, g_cnt = oracle.dynamic_scatter(feats, coors, reduce_type)
    assert np.array_equal(oc.cpu().numpy(), g_oc)
    assert np.array_equal(cmap.cpu().numpy(), g_map)
    assert np.array_equal(cnt.cpu().numpy(), g_cnt)
    assert_reduced(red.cpu().numpy(), feats, g_map, len(g_cnt), reduce_type, g_red)
    # same bits again, and after moving points around without reordering any voxel's own points
    assert torch.equal(forward(cuda, feats, coors, reduce_type)[0].view(torch.int32), red.view(torch.int32))
    src = order_preserving_permutation(g_map, rng)
    red2, oc2, cmap2, cnt2 = forward(cuda, feats[src], coors[src], reduce_type)
    assert torch.equal(red2.view(torch.int32), red.view(torch.int32))
    assert torch.equal(oc2, oc) and torch.equal(cnt2, cnt)
    assert np.array_equal(cmap2.cpu().numpy(), g_map[src])


@pytest.mark.parametrize("reduce_type", REDUCE)
@pytest.mark.parametrize("case", cases(), ids=case_id)
def test_backward_stored_argmax_and_traceback(cuda, case, reduce_type):
    """The backward through autograd (max: the arg-max the forward stored) and through
    voxel_layer.dynamic_point_to_voxel_backward (max: atomicMin traceback) give the same bits, route
    each maximum's gradient to the smallest point index attaining it and leave dropped rows at 0."""
    from bevfusion_b200.scatter_points import dynamic_scatter
    from bevfusion_b200.voxelize import voxel_layer
    feats, coors, rng = build(case)
    f = torch.from_numpy(feats).to(cuda).requires_grad_(True)
    c = torch.from_numpy(coors).to(cuda)
    vf, vc = dynamic_scatter(f, c, reduce_type)
    w = torch.from_numpy(rng.standard_normal(tuple(vf.shape)).astype(np.float32)).to(cuda)
    vf.backward(w)
    red, oc, cmap, cnt = voxel_layer.dynamic_point_to_voxel_forward(f.detach(), c, reduce_type)
    assert torch.equal(vf.detach().view(torch.int32), red.view(torch.int32)) and torch.equal(vc, oc)
    grad = torch.full_like(f.detach(), float("nan"))
    voxel_layer.dynamic_point_to_voxel_backward(grad, w, f.detach(), red, cmap, cnt, reduce_type)
    assert torch.equal(grad.view(torch.int32), f.grad.view(torch.int32))
    g_red, _, g_map, g_cnt = oracle.dynamic_scatter(feats, coors, reduce_type)
    gold = oracle.dynamic_scatter_backward(w.cpu().numpy(), feats, g_red, g_map, g_cnt, reduce_type)
    got = grad.cpu().numpy()
    assert np.array_equal(got, gold)
    assert not got[g_map < 0].any()


@pytest.mark.parametrize("ndim", NDIMS)
def test_key_limits(cuda, ndim):
    """The largest legal value round-trips in every column; one past it raises instead of aliasing
    another voxel; a row that is too big AND negative is simply dropped."""
    lim = key_limit(ndim)
    rows = [[0] * ndim, [lim - 1] * ndim]
    for d in range(ndim):
        r = [d + 1] * ndim
        r[d] = lim - 1
        rows.append(r)
        r = [lim - 1] * ndim
        r[d] = d
        rows.append(r)
    coors = np.asarray(rows + rows[::-1], np.int32)
    feats = np.arange(len(coors), dtype=np.float32).reshape(-1, 1) + 1
    red, oc, cmap, cnt = forward(cuda, feats, coors, "sum")
    g_red, g_oc, g_map, g_cnt = oracle.dynamic_scatter(feats, coors, "sum")
    assert len(g_oc) == len(np.unique(np.asarray(rows), axis=0))
    assert np.array_equal(oc.cpu().numpy(), g_oc) and np.array_equal(cmap.cpu().numpy(), g_map)
    assert np.array_equal(red.cpu().numpy(), g_red)
    for d in range(ndim):
        for v in (lim, 2 ** 31 - 1):
            bad = coors.copy()
            bad[3, d] = v
            with pytest.raises(ValueError, match="exceed the key range"):
                forward(cuda, feats, bad, "sum")
    if ndim > 1:
        dropped = coors.copy()
        dropped[3, 0], dropped[3, 1] = lim, -1
        dropped[4, 0], dropped[4, ndim - 1] = -(2 ** 31), 2 ** 31 - 1
        red, oc, cmap, cnt = forward(cuda, feats, dropped, "sum")
        g = oracle.dynamic_scatter(feats, np.where(np.isin(np.arange(len(coors)), [3, 4])[:, None], -1, coors), "sum")
        assert np.array_equal(oc.cpu().numpy(), g[1]) and np.array_equal(cmap.cpu().numpy(), g[2])
        assert cmap[3].item() == -1 and cmap[4].item() == -1 and np.array_equal(red.cpu().numpy(), g[0])


def test_pin_max_ignores_nan_features(cuda):
    """max is the reference's fmaxf reduction: NaN features are skipped, a voxel holding only NaN
    reduces to -inf, and no NaN element ever receives a gradient -- on both backward paths.  sum and
    mean propagate NaN."""
    from bevfusion_b200.scatter_points import dynamic_scatter
    from bevfusion_b200.voxelize import voxel_layer
    nan, inf = float("nan"), float("inf")
    coors = np.array([[0, 0, 1]] * 4 + [[0, 0, 2]] * 2 + [[0, 0, 3]] * 2 + [[0, 0, 4]] * 3, np.int32)
    feats = np.array([[nan, 1.0], [1.0, nan], [nan, 3.0], [3.0, 3.0],          # voxel 0: max (3, 3) from points 3, 2
                      [nan, nan], [nan, 5.0],                                  # voxel 1: (-inf, 5) from -, 5
                      [nan, -inf], [-inf, nan],                                # voxel 2: (-inf, -inf) from 7, 6
                      [2.0, nan], [nan, nan], [2.0, nan]], np.float32)         # voxel 3: (2, -inf) from 8, -
    want = np.array([[3.0, 3.0], [-inf, 5.0], [-inf, -inf], [2.0, -inf]], np.float32)
    f = torch.from_numpy(feats).to(cuda).requires_grad_(True)
    c = torch.from_numpy(coors).to(cuda)
    vf, _ = dynamic_scatter(f, c, "max")
    assert np.array_equal(vf.detach().cpu().numpy(), want)
    assert np.array_equal(oracle.dynamic_scatter(feats, coors, "max")[0], want)
    w = torch.arange(1.0, 9.0, device=cuda).view(4, 2)
    vf.backward(w)
    gold = np.zeros_like(feats)
    gold[3, 0], gold[2, 1], gold[5, 1], gold[7, 0], gold[6, 1], gold[8, 0] = 1, 2, 4, 5, 6, 7
    assert np.array_equal(f.grad.cpu().numpy(), gold)
    red, oc, cmap, cnt = voxel_layer.dynamic_point_to_voxel_forward(f.detach(), c, "max")
    grad = torch.full_like(f.detach(), nan)
    voxel_layer.dynamic_point_to_voxel_backward(grad, w, f.detach(), red, cmap, cnt, "max")
    assert np.array_equal(grad.cpu().numpy(), gold)
    assert np.array_equal(oracle.dynamic_scatter_backward(w.cpu().numpy(), feats, want, cmap.cpu().numpy(),
                                                          cnt.cpu().numpy(), "max"), gold)
    for reduce_type in ("sum", "mean"):
        red = forward(cuda, feats, coors, reduce_type)[0].cpu().numpy()
        assert np.isnan(red).all()


def large_case():
    """LARGE_N points, one channel, three key columns, about a million distinct voxels, 1 % of
    the rows invalid.  Returns (feats, coors, flat voxel key per point with -1 for invalid rows)."""
    rng = np.random.default_rng(2024)
    ids = rng.integers(0, 1 << 20, LARGE_N)
    coors = np.stack([(ids >> 14) * 16383, ((ids >> 7) & 127) * 8191, (ids & 127) * 8191], axis=1).astype(np.int32)
    bad = rng.random(LARGE_N) < 0.01
    coors[bad, 1] = -1
    feats = rng.standard_normal((LARGE_N, 1)).astype(np.float32)
    return feats, coors, np.where(bad, -1, ids)


def test_more_than_4194304_points_reach_the_scan_carry_loop(cuda):
    """The device-wide scan handles 4096 elements per tile and scans the tile sums 1024 at a time
    with a running carry; DynamicScatter scans one element per point, so only a cloud of more than
    4096 * 1024 points enters the carry loop.  This is the only test that does."""
    feats, coors, ids = large_case()
    assert len(ids) > 4096 * 1024
    red, oc, cmap, cnt = forward(cuda, feats, coors, "sum")
    uniq, inv, count = np.unique(ids, return_inverse=True, return_counts=True)
    assert uniq[0] == -1
    uniq, count, inv = uniq[1:], count[1:], inv.reshape(-1) - 1
    assert len(uniq) > 1000000
    want = np.stack([(uniq >> 14) * 16383, ((uniq >> 7) & 127) * 8191, (uniq & 127) * 8191], axis=1)
    assert np.array_equal(oc.cpu().numpy(), want)
    assert np.array_equal(cmap.cpu().numpy(), inv)
    assert np.array_equal(cnt.cpu().numpy(), count)
    ref, bound = oracle.segment_reduce_f64(feats, inv, len(uniq))
    oracle.assert_within(red.cpu().numpy(), ref, bound, "sum")


@pytest.mark.parametrize("reduce_type", REDUCE)
def test_ties_vs_reference_cuda_extension(cuda, reduce_type):
    """Quantised features (ties in every voxel) through the reference's own forward and backward."""
    ref = ref_module("voxel_layer_ref")
    if ref is None:
        pytest.skip("oracle/_ref not built")
    from bevfusion_b200.voxelize import voxel_layer
    rng = np.random.default_rng(5)
    feats = torch.from_numpy(make_feats(20000, 5, "quantised", rng)).to(cuda)
    coors = torch.from_numpy(rng.integers(-1, 14, (20000, 3)).astype(np.int32)).to(cuda)
    r_red, r_oc, r_map, r_cnt = ref.dynamic_point_to_voxel_forward(feats, coors, reduce_type)
    red, oc, cmap, cnt = voxel_layer.dynamic_point_to_voxel_forward(feats, coors, reduce_type)
    assert torch.equal(oc, r_oc.int()) and torch.equal(cmap, r_map.int()) and torch.equal(cnt, r_cnt.int())
    if reduce_type == "max":
        assert torch.equal(red, r_red)
    else:                                                    # small integers: every order sums exactly
        assert float((red - r_red).abs().max()) <= 1e-6 * float(r_red.abs().max())
    g = torch.randn_like(red)
    r_grad = torch.zeros_like(feats)
    ref.dynamic_point_to_voxel_backward(r_grad, g, feats, r_red, r_map, r_cnt, reduce_type)
    grad = torch.full_like(feats, float("nan"))
    voxel_layer.dynamic_point_to_voxel_backward(grad, g, feats, red, cmap, cnt, reduce_type)
    if reduce_type == "max":
        assert torch.equal(grad, r_grad)
    else:
        assert float((grad - r_grad).abs().max()) <= 1e-6 * float(r_grad.abs().max())
