"""CPU: the case builders of tests/test_bev_pool_sync_free_edges_gpu.py land exactly on their boundaries -- device
n_kept on the TMA kernels' warp-range edges at every tuned width, column-table caps n_seg +- 1, feature heights
straddling the 64-bit pixel mask -- and every table entry they put past the counts is in bounds."""
import pytest

from bev_pool_sync_free_cases import (FEATURE_HEIGHTS, LAYOUTS, TUNED, TwinTables, capacities, caps_around, counts_at,
                                      lift_dims, range_edges)
from test_bev_pool_dispatch_gpu import NUM_SMS, tma_split


@pytest.mark.parametrize("lift", [False, True])
@pytest.mark.parametrize("c", TUNED)
def test_counts_sit_on_the_range_edges(c, lift):
    warps, _ = tma_split(1, c, lift)
    R = NUM_SMS * warps
    edges = range_edges(c, lift)
    assert counts_at(c, lift)[:5] == [0, 1, 31, 32, 33]
    for k in (1, 2):
        below, at, above = edges[3 * (k - 1):3 * k]
        assert (below, at, above) == (k * R * 32 - 1, k * R * 32, k * R * 32 + 1)
        # at k * R * 32 the ranges hold exactly k stages: one row less fits them, one more adds a stage
        assert tma_split(at, c, lift)[1] == 32 * k and tma_split(below, c, lift)[1] == 32 * k
        assert tma_split(above, c, lift)[1] == 32 * (k + 1)
        assert -(-at // (32 * k)) == R and -(-below // (32 * k)) == R


def test_capacities_and_caps():
    assert capacities(0) == [1, 1, 5] and capacities(33) == [33, 34, 104]
    for n_seg, cap in ((2, 100), (500, 501), (700, 7040), (1, 10)):
        caps = caps_around(n_seg, cap)
        assert {n_seg - 1, n_seg, n_seg + 1} & set(range(1, cap + 1)) <= set(caps)
        assert caps[0] == 1 and caps[-1] == cap
        assert n_seg - 1 in caps or n_seg - 1 < 1
        assert n_seg + 1 in caps or n_seg + 1 > cap


def test_feature_heights_straddle_the_mask():
    assert [h for h in FEATURE_HEIGHTS if h <= 64] == [1, 63, 64] and max(FEATURE_HEIGHTS) == 65


@pytest.mark.parametrize("cap", [1, 5, 33, 34, 104, 4096, 6000, 33793, 101381])
def test_lift_dims_cover_the_capacity(cap):
    cams, D, fH, fW = lift_dims(cap)
    assert cams * D * fH * fW == cap and fH <= 64


@pytest.mark.parametrize("lay", LAYOUTS)
@pytest.mark.parametrize("n", [0, 1, 31, 33, 2111, 8449])
@pytest.mark.parametrize("B", [1, 2])
def test_stale_fills_are_in_bounds(lay, n, B):
    for cap in capacities(n):
        tb = TwinTables(n, cap, 80, lay, seed=n + cap, B=B)
        assert tb.stale_in_bounds()
        # the leading entries are a plan: intervals tile [0, n_kept) in ascending cell order
        s, L = tb.starts[:tb.n_int], tb.lengths[:tb.n_int]
        assert int(L.sum()) == n and (s[1:] == (s + L)[:-1]).all() and (n == 0 or s[0] == 0)
        B_, D, H, W = tb.dims
        g = tb.geom[s].astype(int)
        cells = ((g[:, 3] * D + g[:, 2]) * H + g[:, 0]) * W + g[:, 1]
        assert (cells[1:] > cells[:-1]).all()
        if cap > n:
            assert set(tb.nan_rows.tolist()).isdisjoint(tb.perm[:n].tolist())


def test_no_interval_tables_keep_their_points():
    tb = TwinTables(5000, 9000, 16, "hot", seed=1, no_intervals=True)
    assert tb.n_kept == 5000 and tb.n_int == 0 and tb.stale_in_bounds()
