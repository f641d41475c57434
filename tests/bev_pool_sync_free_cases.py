"""Case builders of the sync-free BEV pooling edge tests (tests/test_bev_pool_sync_free_edges_*.py): device counts on
the warp-range boundaries of the TMA kernels, column-table caps around a segment count, feature heights around the
64-bit pixel mask, and synthetic tables of capacity `cap` whose entries past the device counts are in bounds but wrong.
Pure numpy, so the CPU companion checks every builder without a GPU."""
import numpy as np

from test_bev_pool_dispatch_gpu import NUM_SMS, TUNED, decode, grid_for, layout, tma_split

UNTUNED = 24                                   # no TMA kernel: the generic pooling kernels
FEATURE_HEIGHTS = (1, 63, 64, 65)              # the segment mask holds 64 pixel rows
LAYOUTS = ("edges", "hot", "one")


def range_edges(c, lift=False, ks=(1, 2)):
    """n_kept at k * R * 32 - 1, k * R * 32 and k * R * 32 + 1, R = NUM_SMS * warps the TMA kernel's ranges: at
    k * R * 32 every range holds exactly k stages, one row more adds a stage to the rows per range"""
    warps, _ = tma_split(1, c, lift)
    R = NUM_SMS * warps
    return [k * R * 32 + d for k in ks for d in (-1, 0, 1)]


def counts_at(c, lift=False):
    return [0, 1, 31, 32, 33] + range_edges(c, lift)


def capacities(n_kept):
    """table capacities: exactly the count (1 when it is 0: a capacity is positive), one more, a few times more"""
    return [max(n_kept, 1), n_kept + 1, 3 * n_kept + 5]


def caps_around(n_seg, capacity):
    """max_segments 1, n_seg - 1, n_seg, n_seg + 1 and the capacity, those inside [1, capacity]"""
    return sorted({v for v in (1, n_seg - 1, n_seg, n_seg + 1, capacity) if 1 <= v <= capacity})


def lift_dims(cap):
    """(cameras, D, fH, fW) with cameras * D * fH * fW == cap: the synthetic frustum of a lift case, original point
    ((cam * D + d) * fH + h) * fW + w"""
    fh = next(f for f in (8, 4, 2, 1) if cap % f == 0)
    d = next(v for v in (4, 3, 2, 1) if (cap // fh) % v == 0)
    return 1, d, fh, cap // (fh * d)


class TwinTables:
    """Tables of capacity `cap` whose leading n_kept rows / n_int intervals are a valid plan (intervals tile
    [0, n_kept) in ascending cell order, as bevb200_bev_pool_prepare_* writes them), and whose entries past the counts
    hold in-bounds but wrong values:
      perm_stale[n_kept:]  indices of kept points (a read past n_kept doubles a row); perm is the true permutation,
                           perm[n_kept:] the dropped points, which the backward twins read as the filtered tail
      geom[n_kept:]        real cells of the grid
      starts / lengths[n_int:]  ranges inside [0, max(n_kept, 1))
    `nan_rows` are the original points no kept row references."""

    def __init__(self, n_kept, cap, c, lay="edges", seed=0, B=1, D=1, lift=False, no_intervals=False):
        assert cap >= max(n_kept, 1)
        rng = np.random.default_rng(seed)
        self.n_kept, self.cap, self.c = n_kept, cap, c
        _, rpw = tma_split(n_kept, c, lift)
        if n_kept:
            starts, lengths = layout(lay, n_kept, rpw, rng)
        else:
            starts, lengths = np.zeros(0, np.int64), np.zeros(0, np.int64)
        n_int = starts.size
        self.dims = grid_for(n_int, B, D)
        total = int(np.prod(self.dims))
        cells = np.sort(rng.choice(total, n_int, replace=False))
        row_cell = np.repeat(cells, lengths)
        self.perm = rng.permutation(cap).astype(np.int32)
        self.perm_stale = self.perm.copy()
        pool = self.perm[:n_kept] if n_kept else self.perm
        self.perm_stale[n_kept:] = pool[rng.integers(0, pool.size, cap - n_kept)]
        geom = np.empty((cap, 4), np.int32)
        geom[:n_kept] = decode(row_cell, self.dims).reshape(n_kept, 4)
        geom[n_kept:] = decode(rng.integers(0, total, cap - n_kept), self.dims).reshape(cap - n_kept, 4)
        self.geom = geom
        hi = max(n_kept, 1)
        s_stale = rng.integers(0, hi, cap - n_int)
        self.starts = np.concatenate([starts, s_stale]).astype(np.int32)
        self.lengths = np.concatenate([lengths, 1 + rng.integers(0, hi - s_stale)]).astype(np.int32)
        # n_kept > 0 with no interval: a state the sync-free entries accept (every output is zero)
        self.n_int = 0 if no_intervals else n_int
        self.nan_rows = self.perm[n_kept:]

    def stale_in_bounds(self):
        """every entry of every table addresses memory inside its allocation"""
        n, cap, hi = self.n_kept, self.cap, max(self.n_kept, 1)
        B, D, H, W = self.dims
        g = self.geom
        in_grid = ((g[:, 0] >= 0) & (g[:, 0] < H) & (g[:, 1] >= 0) & (g[:, 1] < W) & (g[:, 2] >= 0) & (g[:, 2] < D)
                   & (g[:, 3] >= 0) & (g[:, 3] < B))
        tail_s, tail_l = self.starts[self.n_int:], self.lengths[self.n_int:]
        kept = set(self.perm[:n].tolist()) if n else set(self.perm.tolist())
        return (bool(in_grid.all()) and bool(((self.perm_stale >= 0) & (self.perm_stale < cap)).all())
                and set(self.perm_stale[n:].tolist()) <= kept and sorted(self.perm.tolist()) == list(range(cap))
                and bool(((tail_s >= 0) & (tail_l >= 1) & (tail_s + tail_l <= hi)).all()))


def stale_segments(seg_key, seg_mask, n_seg, size, rng):
    """`size` segment records copied from the real ones (key 0 / mask 1 when there is none): what a column table
    holds past its count after an earlier rebuild"""
    if n_seg == 0:
        return np.zeros(size, np.int64), np.ones(size, np.int64)
    pick = rng.integers(0, n_seg, size)
    return seg_key[pick].copy(), seg_mask[pick].copy()
