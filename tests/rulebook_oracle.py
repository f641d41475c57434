"""Brute-force sparse-conv rulebook and rulebook test-case generators, for the rulebook tests.

  * brute_force: the neighbour table of one conv straight from the definition.  There is a pair (q, o) through
    kernel offset k iff  o * stride - pad + k * dil == q  on every axis and o lies inside the output grid.  SubM
    forces stride 1 and pad k // 2 (spconv_ops.h:76-79, make_geom in rulebook.cu) and keeps the rows as outputs;
    a strided conv's outputs are the reached sites in ascending flat index.  Returns the layout the library
    returns: (outids [n_out, 4], nbr [K, n_out] = input row or -1, out_shape).
  * oracle_nbr: the same table from the C restatement of the reference (oracle.get_indice_pairs), with its
    first-encounter output numbering mapped to ascending flat index.
  * site / row generators: rows at chosen flat sites of the bitmap grid (word edges, scan-tile edges, the last site,
    runs of empty tiles), and for strided convs input rows that reach chosen OUTPUT sites.

Duplicate coordinates are outside the contract (one row per (k, o)); the generators never make them."""
import numpy as np

import oracle

WORD_SITES = 32                      # one bitmap word
TILE_SITES = 4096 * WORD_SITES       # one tile of the rank scan (kSiteScanTile words)


# name -> (ksize, stride, padding, dilation, subm); stride and padding of SubM entries are ignored (forced)
GEOMS = {
    "subm_k3": ([3, 3, 3], [1, 1, 1], [1, 1, 1], [1, 1, 1], True),
    "subm_k5": ([5, 5, 5], [1, 1, 1], [2, 2, 2], [1, 1, 1], True),
    "subm_k113": ([1, 1, 3], [1, 1, 1], [0, 0, 1], [1, 1, 1], True),
    "subm_k331": ([3, 3, 1], [1, 1, 1], [1, 1, 0], [1, 1, 1], True),
    "subm_k3_dil2": ([3, 3, 3], [1, 1, 1], [1, 1, 1], [2, 2, 2], True),
    "subm_k3_dil3": ([3, 3, 3], [1, 1, 1], [1, 1, 1], [3, 3, 3], True),
    "conv_k3s2p0": ([3, 3, 3], [2, 2, 2], [0, 0, 0], [1, 1, 1], False),
    "conv_k3s2p1": ([3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1], False),
    "conv_k3s2p2": ([3, 3, 3], [2, 2, 2], [2, 2, 2], [1, 1, 1], False),
    "conv_k2s2p0": ([2, 2, 2], [2, 2, 2], [0, 0, 0], [1, 1, 1], False),
    "conv_k1s2p0": ([1, 1, 1], [2, 2, 2], [0, 0, 0], [1, 1, 1], False),
    "conv_k2s3p0": ([2, 2, 2], [3, 3, 3], [0, 0, 0], [1, 1, 1], False),
    "conv_k3s221p110": ([3, 3, 3], [2, 2, 1], [1, 1, 0], [1, 1, 1], False),
    "conv_k113s112": ([1, 1, 3], [1, 1, 2], [0, 0, 0], [1, 1, 1], False),
    "conv_k3s1p2_dil2": ([3, 3, 3], [1, 1, 1], [2, 2, 2], [2, 2, 2], False),
    "subm_k7": ([7, 7, 7], [1, 1, 1], [3, 3, 3], [1, 1, 1], True),
    "conv_k7s2p3": ([7, 7, 7], [2, 2, 2], [3, 3, 3], [1, 1, 1], False),
    "subm_k16": ([16, 16, 16], [1, 1, 1], [8, 8, 8], [1, 1, 1], True),
    "conv_k16s2p7": ([16, 16, 16], [2, 2, 2], [7, 7, 7], [1, 1, 1], False),
}


def _list3(v):
    return [int(x) for x in v] if isinstance(v, (list, tuple)) else [int(v)] * 3


def conv_geometry(spatial_shape, ksize, stride, padding, dilation, subm):
    """(out_shape, stride, pad) the conv runs with."""
    ks, dil = list(ksize), list(dilation)
    if subm:
        return list(spatial_shape), [1, 1, 1], [k // 2 for k in ks]
    st, pd = list(stride), list(padding)
    return oracle.conv_output_size(list(spatial_shape), ks, st, pd, dil), st, pd


def num_tiles(batch_size, shape):
    """scan tiles of the bitmap of a [B, X, Y, Z] grid."""
    words = -(-batch_size * int(np.prod(shape)) // WORD_SITES)
    return -(-words // 4096)


def flat_of(rows, shape):
    r = np.asarray(rows, np.int64).reshape(-1, 4)
    return ((r[:, 0] * shape[0] + r[:, 1]) * shape[1] + r[:, 2]) * shape[2] + r[:, 3]


def rows_of(flat, shape):
    """(b, x, y, z) int32 rows of flat sites of a [B, X, Y, Z] grid."""
    s = np.asarray(flat, np.int64)
    z = s % shape[2]; s = s // shape[2]
    y = s % shape[1]; s = s // shape[1]
    x = s % shape[0]; b = s // shape[0]
    return np.stack([b, x, y, z], 1).astype(np.int32)


def in_grid(rows, batch_size, shape):
    r = np.asarray(rows).reshape(-1, 4)
    ok = (r[:, 0] >= 0) & (r[:, 0] < batch_size)
    for a in range(3):
        ok &= (r[:, 1 + a] >= 0) & (r[:, 1 + a] < shape[a])
    return ok


def _offsets(ksize):
    """(k, kx, ky, kz) in the flat offset order k = (kx * ky_size + ky) * kz_size + kz."""
    for kx in range(ksize[0]):
        for ky in range(ksize[1]):
            for kz in range(ksize[2]):
                yield (kx * ksize[1] + ky) * ksize[2] + kz, (kx, ky, kz)


def brute_force(indices, batch_size, spatial_shape, ksize, stride, padding, dilation, subm):
    """-> (outids [n_out, 4] int32, nbr [K, n_out] int32, out_shape).

    Strided: every row of a batch in range feeds the outputs the definition gives, also a row outside the input
    grid (the reference scatters from its inputs).  SubM: the outputs are the rows; the inputs are the rows inside
    the grid, so a row outside it finds its in-grid neighbours but is nobody's neighbour."""
    idx = np.asarray(indices, np.int64).reshape(-1, 4)
    n = idx.shape[0]
    ks, dil = [int(v) for v in ksize], [int(v) for v in dilation]
    out_shape, st, pd = conv_geometry(spatial_shape, ks, stride, padding, dil, subm)
    kvol = int(np.prod(ks))
    bok = (idx[:, 0] >= 0) & (idx[:, 0] < batch_size)
    if subm:
        ing = in_grid(idx, batch_size, spatial_shape)
        site = flat_of(idx[ing], spatial_shape)
        order = np.argsort(site, kind="stable")
        site, row = site[order], np.nonzero(ing)[0][order]
        nbr = np.full((kvol, n), -1, np.int32)
        for k, kk in _offsets(ks):
            q = idx.copy()
            for a in range(3):
                q[:, 1 + a] = idx[:, 1 + a] - pd[a] + kk[a] * dil[a]
            ok = in_grid(q, batch_size, spatial_shape)
            s = flat_of(q[ok], spatial_shape)
            pos = np.minimum(np.searchsorted(site, s), max(site.size - 1, 0))
            hit = np.zeros(s.size, bool) if site.size == 0 else site[pos] == s
            col = np.nonzero(ok)[0][hit]
            nbr[k, col] = row[pos[hit]]
        return idx.astype(np.int32), nbr, out_shape
    # per axis and per offset: v = q + pad - k * dil must be >= 0, a multiple of the stride and v / stride in range
    reach = []
    for a in range(3):
        q = idx[:, 1 + a]
        per = []
        for kk in range(ks[a]):
            v = q + pd[a] - kk * dil[a]
            ok = (v >= 0) & (v % st[a] == 0) & (v // st[a] < out_shape[a])
            per.append((ok, v // st[a]))
        reach.append(per)
    hits = []
    for k, (kx, ky, kz) in _offsets(ks):
        ok = bok & reach[0][kx][0] & reach[1][ky][0] & reach[2][kz][0]
        rows = np.nonzero(ok)[0]
        o = np.stack([idx[rows, 0], reach[0][kx][1][rows], reach[1][ky][1][rows], reach[2][kz][1][rows]], 1)
        hits.append((k, rows, flat_of(o, out_shape)))
    flat = np.unique(np.concatenate([h[2] for h in hits])) if hits else np.zeros(0, np.int64)
    nbr = np.full((kvol, flat.size), -1, np.int32)
    for k, rows, s in hits:
        nbr[k, np.searchsorted(flat, s)] = rows
    return rows_of(flat, out_shape), nbr, out_shape


def oracle_nbr(indices, batch_size, spatial_shape, ksize, stride, padding, dilation, subm):
    """(outids, nbr, out_shape) from oracle.get_indice_pairs, outputs in ascending flat index for strided convs.
    Only for rows inside the grid: see the note in test_rulebook_cpu.py on rows outside it."""
    outids, pairs, num, out_shape = oracle.get_indice_pairs(indices, batch_size, spatial_shape, ksize, stride,
                                                            padding, dilation, subm)
    kvol = pairs.shape[0]
    if subm:
        rank = np.arange(outids.shape[0])
    else:
        flat = flat_of(outids, out_shape)
        order = np.argsort(flat, kind="stable")
        rank = np.empty_like(order)
        rank[order] = np.arange(order.size)
        outids = outids[order]
    nbr = np.full((kvol, outids.shape[0]), -1, np.int32)
    for k in range(kvol):
        nbr[k, rank[pairs[k, 1, :num[k]]]] = pairs[k, 0, :num[k]]
    return outids, nbr, out_shape


def pair_lists(nbr):
    """per offset: (inputs, outputs) of the valid entries, outputs ascending -- rb.pairs()'s order."""
    out = []
    for k in range(nbr.shape[0]):
        o = np.nonzero(nbr[k] >= 0)[0]
        out.append((nbr[k, o].astype(np.int32), o.astype(np.int32)))
    return out


def transpose(nbr, n_in):
    """nbr_t [K, n_in]: nbr_t[k, j] = the output row fed by input row j through k, or -1."""
    t = np.full((nbr.shape[0], n_in), -1, np.int32)
    for k in range(nbr.shape[0]):
        o = np.nonzero(nbr[k] >= 0)[0]
        t[k, nbr[k, o]] = o
    return t


# ---------------------------------------------------------------------------------------------------- generators
def edge_sites(batch_size, shape, rng, fill=2000, empty_tiles=()):
    """Sorted flat sites of a [B, X, Y, Z] bitmap grid: the first site, the corner block around the very last one,
    both sides of a few word edges (32w - 1, 32w), both sides of every scan-tile edge (t * TILE_SITES - 1,
    t * TILE_SITES), and `fill` random sites.  No site lands in a tile listed in `empty_tiles`."""
    total = batch_size * int(np.prod(shape))
    s = [0, total - 1]
    words = -(-total // WORD_SITES)
    for w in {1, 2, 3, words // 3, words // 2, words - 1}:
        if 0 < w < words:
            s += [WORD_SITES * w - 1, WORD_SITES * w]
    for t in range(1, num_tiles(batch_size, shape)):
        s += [t * TILE_SITES - 1, t * TILE_SITES]
    # the 4 x 4 x 4 corner block that ends the last sample: rows that look the very last site up (dilation <= 3)
    c = np.stack(np.meshgrid(*[np.arange(max(n - 4, 0), n) for n in shape], indexing="ij"), -1).reshape(-1, 3)
    s += flat_of(np.concatenate([np.full((c.shape[0], 1), batch_size - 1), c], 1), shape).tolist()
    s += rng.integers(0, total, fill).tolist()
    s = np.unique(np.asarray(s, np.int64))
    s = s[(s >= 0) & (s < total)]
    if len(empty_tiles):
        s = s[~np.isin(s // TILE_SITES, np.asarray(list(empty_tiles)))]
    return s


def rows_reaching(out_flat, batch_size, in_shape, out_shape, ksize, stride, padding, dilation):
    """Input rows (inside the input grid) of a strided conv that reach the given output sites: for each output o,
    q = o * stride - pad + k * dil for the first offset k that puts q inside the grid.  Sorted, unique."""
    o = rows_of(out_flat, out_shape).astype(np.int64)
    q = np.zeros_like(o)
    done = np.zeros(o.shape[0], bool)
    for _, kk in _offsets(ksize):
        cand = o.copy()
        for a in range(3):
            cand[:, 1 + a] = o[:, 1 + a] * stride[a] - padding[a] + kk[a] * dilation[a]
        take = ~done & in_grid(cand, batch_size, in_shape)
        q[take] = cand[take]
        done |= take
    return rows_of(np.unique(flat_of(q[done], in_shape)), in_shape)


def in_shape_for(out_shape, ksize, stride, padding, dilation, extra):
    """An input grid whose conv output grid is `out_shape`; extra[a] in [0, stride[a]) adds rows that round away."""
    s = [(out_shape[a] - 1) * stride[a] - 2 * padding[a] + dilation[a] * (ksize[a] - 1) + 1 + extra[a]
         for a in range(3)]
    assert oracle.conv_output_size(s, ksize, stride, padding, dilation) == list(out_shape)
    return s
