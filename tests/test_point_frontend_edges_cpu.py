"""CPU self-checks of the generators and float64 helpers behind the point front end's edge tests
(test_voxelize_edges_gpu, test_dynamic_scatter_edges_gpu, test_depthmap_edges_gpu): they reach what
they claim to reach, and the float64 references agree with the oracle where they can decide."""
import os

import numpy as np
import pytest

import oracle
import test_depthmap_edges_gpu as D
import test_dynamic_scatter_edges_gpu as S
import test_voxelize_edges_gpu as V


@pytest.mark.parametrize("geom", list(V.GEOMS))
def test_boundary_cloud_reaches_the_faces(geom):
    vs, cr, exact = V.GEOMS[geom]
    pts, is_probe = V.boundary_cloud(vs, cr, 5, seed=3)
    coors = oracle.dynamic_voxelize(pts, vs, cr)
    ref, decided = V.cells_f64(pts, vs, cr)
    if exact:
        assert np.array_equal(coors, ref)                    # no rounding anywhere: float64 decides every point
    else:
        assert 0 < (~decided).sum() <= is_probe.sum()
        assert np.array_equal(coors[decided], ref[decided])
    grid = V.grid_of(vs, cr)
    kept = coors[coors[:, 0] >= 0]
    assert (kept.min(0) == 0).all() and (kept.max(0) == grid - 1).all()        # first and last cell of every axis
    assert np.isnan(pts[:, :3]).any() and np.isinf(pts[:, :3]).any()
    if geom == "nondividing":                                # in range, beyond the rounded grid: dropped
        strip = (pts[:, 0] >= 9.95) & (pts[:, 0] < 10) & (pts[:, 1] < 9) & (pts[:, 2] < 9) & (pts[:, :3] >= 0).all(1)
        assert strip.any() and (coors[strip] == -1).all()


def test_scatter_cases_cover_every_value():
    cases = S.cases()
    for k, values in enumerate([S.SIZES, S.OCCUPANCY, S.NDIMS, S.CHANNELS, S.FAMILIES]):
        assert {c[k] for c in cases} == set(values)
    assert S.LARGE_N > 4096 * 1024
    rng = np.random.default_rng(0)
    feats, coors = S.make_feats(4096, 3, "quantised", rng), S.make_coors(4096, 3, "eight_per_voxel", rng)
    red, _, cmap, cnt = oracle.dynamic_scatter(feats, coors, "max")
    ties = np.zeros_like(red)
    np.add.at(ties, cmap, feats == red[cmap])
    assert (ties[cnt > 4] > 1).mean() > 0.5                  # most maxima are attained more than once
    for ndim in S.NDIMS:
        c = S.make_coors(20000, ndim, "all_distinct", rng)
        assert len(np.unique(c, axis=0)) == 20000 and c.min() >= 0
        assert (c.max(0) > 0.9 * S.key_limit(ndim)).all() and c.max() < S.key_limit(ndim)
    seg = rng.integers(-1, 50, 3000)
    src = S.order_preserving_permutation(seg, rng)
    assert sorted(src.tolist()) == list(range(3000)) and not np.array_equal(src, np.arange(3000))
    for v in range(-1, 50):
        assert (np.diff(src[seg[src] == v]) > 0).all()


def test_oracle_max_backward_matches_a_plain_loop():
    rng = np.random.default_rng(1)
    feats, coors = S.make_feats(500, 4, "quantised", rng), rng.integers(-1, 5, (500, 3)).astype(np.int32)
    feats[rng.random(feats.shape) < 0.1] = np.nan
    red, _, cmap, cnt = oracle.dynamic_scatter(feats, coors, "max")
    assert not np.isnan(red).any()
    w = rng.standard_normal(red.shape).astype(np.float32)
    gold = np.zeros_like(feats)
    for v in range(len(cnt)):
        for ch in range(4):
            hit = np.nonzero((cmap == v) & (feats[:, ch] == red[v, ch]))[0]
            if len(hit):
                gold[hit[0], ch] = w[v, ch]
    assert np.array_equal(oracle.dynamic_scatter_backward(w, feats, red, cmap, cnt, "max"), gold)


def test_ordered_fp32_sum_stays_inside_its_bound():
    rng = np.random.default_rng(2)
    x = S.make_feats(20001, 3, "cancelling", rng)
    seg = np.zeros(len(x), np.int64)
    ref, bound = oracle.segment_reduce_f64(x, seg, 1)
    got = np.cumsum(x, axis=0, dtype=np.float32)[-1:]        # numpy's cumsum adds one row at a time
    oracle.assert_within(got, ref, bound)
    assert (bound < 2e-3 * np.abs(x).sum(0)).all()
    wrong = got.copy()
    wrong[0, 1] += 2 * np.float32(bound[0, 1]) + np.spacing(wrong[0, 1])
    with pytest.raises(AssertionError):
        oracle.assert_within(wrong, ref, bound)


def test_float64_projection_agrees_with_the_oracle_on_the_golden_frame(golden_dir):
    g = np.load(os.path.join(golden_dir, "depth_tiny.npz"))
    for b, pts in enumerate([g["points0"], g["points1"]]):
        args = (g["lidar2image"][b], g["img_aug_matrix"][b], g["lidar_aug_matrix"][b], g["image_size"])
        gold = oracle.points_to_depth(pts, *args, add_depth_features=True)
        shifted = pts.copy()
        shifted[:, :3] -= g["lidar_aug_matrix"][b][:3, 3]
        exp = D.expected_depth_f64(pts, *args)
        share = D.assert_scalar_matches_f64(gold[:, 0], gold[:, 1:], shifted, exp)
        assert share < 0.01 and (exp[0] >= 0).sum() > 0
