"""GPU: the sparse-conv rulebook (rulebook.cu through ops.get_rulebook), its pair converters and dense(), bit-exact
against the brute force of tests/rulebook_oracle.py, on every geometry the C ABI accepts and on grids of one to
~650 rank-scan tiles.  The brute force is pinned to the C oracle by tests/test_rulebook_cpu.py.

Every case compares n_out, outids and the whole neighbour table nbr[k, o], and asserts the contract the convs rely
on: an input row feeds at most one output per offset, the SubM centre tap is the identity and SubM offsets are
symmetric (where the geometry has a centre: odd kernels, dilation 1 -- SubM pads by k // 2 whatever the dilation,
as spconv_ops.h:76-79 does), and two calls give the same bits.  Strided grids are built on the OUTPUT grid, whose
bitmap is the one the scan ranks."""
import numpy as np
import pytest
import torch

import oracle
import rulebook_oracle as R
from conftest import ref_module

pytestmark = pytest.mark.gpu

GEOMS = R.GEOMS
SMALL = [g for g in GEOMS if np.prod(GEOMS[g][0]) <= 125]            # every grid
LARGE = [g for g in GEOMS if np.prod(GEOMS[g][0]) > 125]             # kernel volumes 343 and 4096

# name -> (batch, shape of the bitmap grid, sites to mark, tiles left empty, batch left empty)
GRIDS = {
    "odd_b1": (1, [37, 29, 13], 2500, (), None),
    "b3_empty_middle": (3, [41, 35, 11], 3000, (), 1),
    "tiles_exact": (3, [64, 64, 32], 20000, (), None),               # 3 tiles, the last one full
    "tiles_exact_plus_word": (1, [2731, 3, 32], 20000, (), None),    # 2 tiles + a one-word tile
    "multi_tile": (2, [257, 251, 21], 40000, range(4, 9), None),     # 21 tiles, 4..8 empty
}


def same(got, want, what):
    assert got.shape == want.shape, "%s: shape %s != %s" % (what, got.shape, want.shape)
    bad = np.argwhere(got != want)
    assert bad.size == 0, "%s: %d entries differ, first at %s: got %s, want %s" % (
        what, bad.shape[0], bad[0].tolist(), got[tuple(bad[0])], want[tuple(bad[0])])


def make_case(geom, grid, seed):
    """(rows, batch, input shape) whose conv marks the edge sites of GRIDS[grid] in its bitmap grid."""
    ks, st, pd, dil, subm = GEOMS[geom]
    B, gshape, fill, empty, skip = GRIDS[grid]
    rng = np.random.default_rng(seed)
    sites = R.edge_sites(B, gshape, rng, fill=fill, empty_tiles=empty)
    if skip is not None:
        sites = sites[R.rows_of(sites, gshape)[:, 0] != skip]
    if subm:
        rows, ishape = R.rows_of(sites, gshape), list(gshape)
    else:
        ishape = R.in_shape_for(gshape, ks, st, pd, dil, [st[a] - 1 if a != 1 else 0 for a in range(3)])
        rows = R.rows_reaching(sites, B, ishape, gshape, ks, st, pd, dil)
    return rows[rng.permutation(rows.shape[0])], B, ishape


def check_contract(nbr, n_in, geom, inside=None):
    """`inside`: SubM rows inside the grid (default all); a row outside it is not its own centre neighbour"""
    ks, _, _, dil, subm = geom
    kvol = nbr.shape[0]
    for k in range(kvol):
        v = nbr[k][nbr[k] >= 0]
        assert v.max(initial=0) < max(n_in, 1)
        assert np.unique(v).size == v.size, "an input row feeds two outputs through offset %d" % k
    if subm and all(d == 1 or k == 1 for k, d in zip(ks, dil)):
        c = ((ks[0] // 2) * ks[1] + ks[1] // 2) * ks[2] + ks[2] // 2
        want = np.arange(nbr.shape[1])
        if inside is not None:
            want[~inside] = -1
        assert np.array_equal(nbr[c], want), "SubM centre tap is not the identity"
    if subm and all(k % 2 == 1 for k in ks) and all(d == 1 for d in dil):
        for k in range(kvol):
            i = np.nonzero(nbr[k] >= 0)[0]
            assert np.array_equal(nbr[kvol - 1 - k][nbr[k][i]], i), "SubM symmetry broken at offset %d" % k


def run_case(cuda, rows, B, shape, geom, label):
    """get_rulebook twice == the brute force, exactly; returns (rulebook, brute-force nbr)."""
    from bevfusion_b200.spconv import ops
    ks, st, pd, dil, subm = GEOMS[geom] if isinstance(geom, str) else geom
    ti = torch.from_numpy(np.ascontiguousarray(rows, np.int32)).to(cuda)
    rb, oshape = ops.get_rulebook(ti, B, shape, ks, st, pd, dil, 0, subm)
    again, _ = ops.get_rulebook(ti.clone(), B, shape, ks, st, pd, dil, 0, subm)
    outids, nbr, want_shape = R.brute_force(rows, B, shape, ks, st, pd, dil, subm)
    assert oshape == want_shape, label
    assert rb.n_out == outids.shape[0], label
    same(rb.outids.cpu().numpy(), outids, label + " outids")
    got = rb.nbr.cpu().numpy()
    same(got, nbr, label + " nbr")
    assert torch.equal(again.outids, rb.outids) and torch.equal(again.nbr, rb.nbr), label + ": calls differ"
    check_contract(got, rows.shape[0], (ks, st, pd, dil, subm), R.in_grid(rows, B, shape))
    grid = shape if subm else oshape
    print("%-34s B %d in %-16s out %-16s tiles %4d  n_in %7d  n_out %7d  pairs %8d" % (
        label, B, shape, oshape, R.num_tiles(B, grid), rows.shape[0], rb.n_out, int((got >= 0).sum())))
    return rb, nbr


@pytest.mark.parametrize("grid", list(GRIDS))
@pytest.mark.parametrize("geom", SMALL)
def test_rulebook_vs_brute_force(cuda, geom, grid):
    rows, B, shape = make_case(geom, grid, seed=len(geom) * 31 + len(grid))
    run_case(cuda, rows, B, shape, geom, "%s / %s" % (geom, grid))


@pytest.mark.parametrize("geom", LARGE)
def test_large_kernels(cuda, geom):
    """kernel volumes 343 and 4096 (the limit), on an odd grid with an empty middle sample"""
    rng = np.random.default_rng(5)
    B, shape = 3, [23, 19, 21]
    n = 60 if np.prod(GEOMS[geom][0]) > 343 else 400
    flat = rng.choice(B * int(np.prod(shape)), size=3 * n, replace=False)
    rows = R.rows_of(flat, shape)
    rows = rows[rows[:, 0] != 1][:n]
    run_case(cuda, rows, B, shape, geom, geom)


def test_kernel_volume_above_limit_is_rejected(cuda):
    from bevfusion_b200._C import BevB200Error
    from bevfusion_b200.spconv import ops
    ti = torch.tensor([[0, 3, 3, 3]], dtype=torch.int32, device=cuda)
    with pytest.raises(BevB200Error, match="4096"):
        ops.get_rulebook(ti, 1, [40, 300, 8], [17, 241, 1], 1, 0, 1, 0, True)
    with pytest.raises(BevB200Error, match="4096"):
        ops.get_rulebook(ti, 1, [40, 300, 8], [17, 241, 1], 1, 0, 1, 0, False)


def test_rows_outside_grid_and_batch(cuda):
    """rows one step outside the grid feed border outputs of a strided conv (the reference's scatter); rows further
    out or of a batch out of range reach nothing; SubM looks only rows inside the grid up."""
    rng = np.random.default_rng(11)
    B, shape = 2, [19, 17, 9]
    rows = R.rows_of(rng.choice(B * int(np.prod(shape)), 600, replace=False), shape)
    extra = np.array([[0, -1, 0, 0], [1, 18, -1, 8], [0, 19, 16, 8], [1, 5, 17, 9], [0, -2, 3, 3],
                      [0, 3, 3, -3], [2, 3, 3, 3], [-1, 3, 3, 3], [1, 40, 3, 3]], np.int32)
    rows = np.concatenate([rows, extra])[rng.permutation(rows.shape[0] + extra.shape[0])]
    for geom in ("conv_k3s2p1", "conv_k3s2p2", "conv_k2s2p0", "subm_k3", "subm_k3_dil2"):
        run_case(cuda, rows, B, shape, geom, "outside rows / " + geom)


# --------------------------------------------------------------------------------------------- full C3 grid
@pytest.fixture(scope="module")
def c3_rows(cuda):
    from bevfusion_b200 import synthetic as S
    from bevfusion_b200.voxelize import Voxelization, voxelize_mean
    L = S.LIDAR_C3
    pts = torch.from_numpy(S.lidar_cloud(seed=0)).to(cuda)
    vox = Voxelization(L["voxel_size"], L["point_cloud_range"], L["max_num_points"], L["max_voxels"]).eval()
    _, idx = voxelize_mean(*vox(pts), 0)
    return idx, list(L["sparse_shape"])


C3_CHAIN = [("conv_input + stage 1 SubM", [3, 3, 3], 1, 1, True), ("stage 1 down", [3, 3, 3], 2, 1, False),
            ("stage 2 SubM", [3, 3, 3], 1, 1, True), ("stage 2 down", [3, 3, 3], 2, 1, False),
            ("stage 3 SubM", [3, 3, 3], 1, 1, True), ("stage 3 down", [3, 3, 3], 2, [1, 1, 0], False),
            ("stage 4 SubM", [3, 3, 3], 1, 1, True), ("conv_out", [1, 1, 3], [1, 1, 2], 0, False)]


def test_c3_encoder_chain(cuda, c3_rows):
    """the 4 SubM and 4 strided rulebooks of the C3 encoder on the full 1440 x 1440 x 41 grid (~650 tiles); the
    SubM rulebooks after a strided conv take the path that reuses its bitmap."""
    from bevfusion_b200 import _C
    from bevfusion_b200.spconv import ops
    idx, shape = c3_rows
    rows = idx.cpu().numpy()
    for name, ks, st, pd, subm in C3_CHAIN:
        ks, st, pd = R._list3(ks), R._list3(st), R._list3(pd)
        _C.reset_launch_count()
        rb, oshape = ops.get_rulebook(idx, 1, shape, ks, st, pd, [1, 1, 1], 0, subm)
        reused = _C.launch_count() == 1
        outids, nbr, want_shape = R.brute_force(rows, 1, shape, ks, st, pd, [1, 1, 1], subm)
        assert oshape == want_shape and rb.n_out == outids.shape[0], name
        same(rb.outids.cpu().numpy(), outids, name + " outids")
        got = rb.nbr.cpu().numpy()
        same(got, nbr, name + " nbr")
        check_contract(got, rows.shape[0], (ks, st, pd, [1, 1, 1], subm))
        assert reused == (subm and name != C3_CHAIN[0][0]), name
        print("C3 %-26s in %-16s out %-16s tiles %4d  n_in %7d  n_out %7d  pairs %8d%s" % (
            name, shape, oshape, R.num_tiles(1, shape if subm else oshape), rows.shape[0], rb.n_out,
            int((got >= 0).sum()), "  (reused bitmap)" if reused else ""))
        if not subm:
            idx, rows, shape = rb.outids, outids, oshape


# ------------------------------------------------------------------------------ SubM on a strided conv's rows
def strided_case(seed, B=2, out_shape=(257, 251, 21)):
    ks, st, pd, dil = [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1]
    rng = np.random.default_rng(seed)
    ishape = R.in_shape_for(list(out_shape), ks, st, pd, dil, [1, 0, 1])
    sites = R.edge_sites(B, list(out_shape), rng, fill=30000, empty_tiles=range(4, 9))
    rows = R.rows_reaching(sites, B, ishape, list(out_shape), ks, st, pd, dil)
    return rows[rng.permutation(rows.shape[0])], B, ishape


@pytest.mark.parametrize("ks,dil", [(3, 1), (3, 2), (5, 1), (5, 2)])
def test_subm_reuses_strided_bitmap(cuda, ks, dil):
    """bevb200_rulebook_fill_subm_sorted (the gather alone, on the strided conv's bitmap and ranks) == a fresh
    rulebook on a copy of the rows == the brute force == the C oracle"""
    from bevfusion_b200 import _C
    from bevfusion_b200.spconv import ops
    rows, B, ishape = strided_case(seed=ks * 10 + dil)
    rb, oshape = ops.get_rulebook(torch.from_numpy(rows).to(cuda), B, ishape, 3, 2, 1, 1, 0, False)
    assert getattr(rb.outids, "_b200_site_state", None) is not None
    _C.reset_launch_count()
    sub, _ = ops.get_rulebook(rb.outids, B, oshape, ks, 1, ks // 2, dil, 0, True)
    assert _C.launch_count() == 1                                     # the reused bitmap: one gather launch
    _C.reset_launch_count()
    fresh, _ = ops.get_rulebook(rb.outids.clone(), B, oshape, ks, 1, ks // 2, dil, 0, True)
    assert _C.launch_count() > 1
    assert torch.equal(sub.outids, rb.outids) and torch.equal(sub.nbr, fresh.nbr)
    outs = rb.outids.cpu().numpy()
    _, want, _ = R.brute_force(outs, B, oshape, [ks] * 3, [1] * 3, [ks // 2] * 3, [dil] * 3, True)
    same(sub.nbr.cpu().numpy(), want, "reused SubM nbr")
    _, o_nbr, _ = R.oracle_nbr(outs, B, oshape, [ks] * 3, [1] * 3, [ks // 2] * 3, [dil] * 3, True)
    same(want, o_nbr, "brute force vs oracle")
    check_contract(want, outs.shape[0], ([ks] * 3, [1] * 3, [ks // 2] * 3, [dil] * 3, True))
    print("reused SubM k%d dil %d  B %d grid %s tiles %d  n %d  pairs %d" % (
        ks, dil, B, oshape, R.num_tiles(B, oshape), outs.shape[0], int((want >= 0).sum())))


def test_subm_reuse_after_side_stream_build(cuda):
    """the strided rulebook built on a side stream: the SubM gather on the main stream waits on its event"""
    from bevfusion_b200 import _C
    from bevfusion_b200.spconv import ops
    rows, B, ishape = strided_case(seed=3)
    side = torch.cuda.Stream()
    ti = torch.from_numpy(rows).to(cuda)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        rb, oshape = ops.get_rulebook(ti, B, ishape, 3, 2, 1, 1, 0, False)
    _C.reset_launch_count()
    sub, _ = ops.get_rulebook(rb.outids, B, oshape, 3, 1, 1, 1, 0, True)
    assert _C.launch_count() == 1
    got = sub.nbr.cpu().numpy()
    torch.cuda.synchronize()
    outs = rb.outids.cpu().numpy()
    _, want, _ = R.brute_force(outs, B, oshape, [3] * 3, [1] * 3, [1] * 3, [1] * 3, True)
    same(got, want, "SubM after a side-stream strided build")


def test_subm_does_not_reuse_a_foreign_grid(cuda):
    """a site state of another spatial shape or batch size must not be reused"""
    from bevfusion_b200 import _C
    from bevfusion_b200.spconv import ops
    rows, B, ishape = strided_case(seed=4, B=2, out_shape=(97, 89, 21))
    rb, oshape = ops.get_rulebook(torch.from_numpy(rows).to(cuda), B, ishape, 3, 2, 1, 1, 0, False)
    outs = rb.outids.cpu().numpy()
    for b, shape in ((B, [oshape[0] + 1, oshape[1], oshape[2]]), (B, [oshape[0], oshape[1], oshape[2] + 3]),
                     (B + 1, oshape)):
        _C.reset_launch_count()
        sub, _ = ops.get_rulebook(rb.outids, b, shape, 3, 1, 1, 1, 0, True)
        assert _C.launch_count() > 1, (b, shape)
        _, want, _ = R.brute_force(outs, b, shape, [3] * 3, [1] * 3, [1] * 3, [1] * 3, True)
        same(sub.nbr.cpu().numpy(), want, "SubM on %d x %s" % (b, shape))


# ------------------------------------------------------------------------------------------- pair converters
@pytest.mark.parametrize("geom", ["conv_k3s2p1", "subm_k3", "conv_k2s3p0", "subm_k3_dil2"])
def test_pairs_round_trip(cuda, geom):
    """rb.pairs() == the C oracle's pairs in output order (compaction carried across 1024-row chunks, -1 tail);
    nbr_from_pairs rebuilds nbr, also from padded pairs with garbage past num[k]; inverse=True == the transpose"""
    from bevfusion_b200.spconv import ops
    ks, st, pd, dil, subm = GEOMS[geom]
    B, shape = 2, [97, 89, 21]
    rng = np.random.default_rng(len(geom))
    rows = R.rows_of(rng.choice(B * int(np.prod(shape)), 30000, replace=False), shape)
    rows = rows[rng.permutation(rows.shape[0])]
    rb, nbr = run_case(cuda, rows, B, shape, geom, "pairs / " + geom)
    n_in, n_out, kvol = rows.shape[0], rb.n_out, rb.kernel_volume
    assert n_out > 4 * 1024                                           # several 1024-row chunks per offset
    pairs, num = (t.cpu().numpy() for t in rb.pairs())
    _, _, o_num, _ = oracle.get_indice_pairs(rows, B, shape, ks, st, pd, dil, subm)
    same(num, o_num, "indice_num")
    _, o_nbr, _ = R.oracle_nbr(rows, B, shape, ks, st, pd, dil, subm)
    for k, (i, o) in enumerate(R.pair_lists(o_nbr)):
        assert num[k] == i.size
        same(pairs[k, 0, :num[k]], i, "pairs[%d] inputs" % k)
        same(pairs[k, 1, :num[k]], o, "pairs[%d] outputs" % k)
        assert np.all(np.diff(pairs[k, 1, :num[k]]) > 0)
        assert (pairs[k, :, num[k]:] == -1).all()
    tp, tn = rb.pairs()
    assert torch.equal(ops.nbr_from_pairs(tp, tn, n_out), rb.nbr)
    # pairs_dim > num[k], slots past num[k] full of in-range garbage
    pad = torch.empty((kvol, 2, n_in + 77), dtype=torch.int32)
    pad[:, 0] = torch.randint(0, n_in, (kvol, n_in + 77), dtype=torch.int32)
    pad[:, 1] = torch.randint(0, n_out, (kvol, n_in + 77), dtype=torch.int32)
    for k in range(kvol):
        pad[k, :, :num[k]] = torch.from_numpy(pairs[k, :, :num[k]])
    assert torch.equal(ops.nbr_from_pairs(pad.to(cuda), tn, n_out), rb.nbr)
    inv = ops.nbr_from_pairs(tp, tn, n_in, inverse=True)
    assert torch.equal(inv, ops.transpose_nbr(rb.nbr, n_in))
    same(inv.cpu().numpy(), R.transpose(nbr, n_in), "inverse nbr")
    inv_pad = ops.nbr_from_pairs(pad.to(cuda), tn, n_in, inverse=True)
    assert torch.equal(inv_pad, inv)


# ------------------------------------------------------------------------------------------------- dense()
def dense_want(feats, rows, B, shape, z_major):
    X, Y, Z = shape
    c = feats.shape[1]
    ok = torch.from_numpy(R.in_grid(rows, B, shape))
    r = torch.from_numpy(rows).long()[ok]
    d = torch.zeros(B, X, Y, Z, c).index_put((r[:, 0], r[:, 1], r[:, 2], r[:, 3]), feats[ok])
    if z_major:
        return d.permute(0, 4, 3, 1, 2).reshape(B, c * Z, X, Y)
    return d.permute(0, 4, 1, 2, 3).contiguous()


@pytest.mark.parametrize("z_major", [False, True])
@pytest.mark.parametrize("c", [1, 5, 31, 32, 33, 128])
def test_sparse_to_dense(cuda, c, z_major):
    from bevfusion_b200.spconv import ops
    B, shape = 3, [13, 11, 7]
    rng = np.random.default_rng(c)
    rows = R.rows_of(rng.choice(B * int(np.prod(shape)), 700, replace=False), shape)
    rows = rows[rows[:, 0] != 1]
    bad = np.array([[0, -1, 0, 0], [2, 13, 0, 0], [0, 0, 11, 0], [2, 0, 0, 7], [0, 0, 0, -1], [3, 0, 0, 0],
                    [-1, 1, 1, 1]], np.int32)
    rows = np.concatenate([rows, bad])[rng.permutation(rows.shape[0] + bad.shape[0])]
    feats = torch.from_numpy(rng.standard_normal((rows.shape[0], c)).astype(np.float32))
    want = dense_want(feats, rows, B, shape, z_major)
    f, ti = feats.to(cuda), torch.from_numpy(rows).to(cuda)
    got = ops.sparse_to_dense(f, ti, B, shape, z_major=z_major)
    assert torch.equal(got.cpu(), want)
    # a channel slice of a wider buffer: the slice is zeroed and written, the other channels keep their guard value
    lo, width = 3, want.shape[1]
    buf = torch.full((B, width + 9, *want.shape[2:]), 7.25, device=cuda)
    buf[:, lo:lo + width] = float("nan")
    ops.sparse_to_dense(f, ti, B, shape, z_major=z_major, out=buf[:, lo:lo + width])
    host = buf.cpu()
    assert torch.equal(host[:, lo:lo + width], want)
    assert (host[:, :lo] == 7.25).all() and (host[:, lo + width:] == 7.25).all()
    # no rows: a zero fill
    out = torch.full_like(got, float("nan"))
    ops.sparse_to_dense(f[:0], ti[:0], B, shape, z_major=z_major, out=out)
    assert not bool(out.any())
    print("dense c %3d z_major %d  B %d grid %s  rows %d (%d outside)" % (c, z_major, B, shape, rows.shape[0],
                                                                         bad.shape[0]))


# --------------------------------------------------------------------------------------- reference extension
def test_vs_reference_extension(cuda):
    """get_indice_pairs_3d of the reference's own GPU build: same outids, num and pair sets on a multi-tile grid,
    a dilated geometry and an even kernel"""
    ref = ref_module("sparse_conv_ext_ref")
    if ref is None:
        pytest.skip("oracle/_ref not built")
    from bevfusion_b200.spconv import ops
    cases = [("conv_k3s2p1", "multi_tile"), ("subm_k3", "multi_tile"), ("subm_k3_dil2", "odd_b1"),
             ("conv_k3s1p2_dil2", "b3_empty_middle"), ("conv_k2s2p0", "tiles_exact_plus_word")]
    for geom, grid in cases:
        ks, st, pd, dil, subm = GEOMS[geom]
        rows, B, shape = make_case(geom, grid, seed=7)
        ti = torch.from_numpy(rows).to(cuda)
        out_shape = shape if subm else oracle.conv_output_size(shape, ks, st, pd, dil)
        r_out, r_pairs, r_num = ref.get_indice_pairs_3d(ti, B, out_shape, shape, ks, st, pd, dil, [0, 0, 0],
                                                        int(subm), 0)
        outids, pairs, num = ops.get_indice_pairs(ti, B, shape, ks, st, pd, dil, 0, subm)
        label = "%s / %s" % (geom, grid)
        assert torch.equal(outids, r_out), label
        assert torch.equal(num, r_num), label
        pairs, num, r_pairs = pairs.cpu().numpy(), num.cpu().numpy(), r_pairs.cpu().numpy()
        for k in range(num.shape[0]):
            a = np.sort(pairs[k, 0, :num[k]].astype(np.int64) << 32 | pairs[k, 1, :num[k]])
            b = np.sort(r_pairs[k, 0, :num[k]].astype(np.int64) << 32 | r_pairs[k, 1, :num[k]])
            assert np.array_equal(a, b), "%s offset %d" % (label, k)
        print("reference %-34s tiles %4d  n_out %7d  pairs %8d" % (
            label, R.num_tiles(B, out_shape), outids.shape[0], int(num.sum())))
