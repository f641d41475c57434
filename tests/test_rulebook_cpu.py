"""CPU: the brute-force rulebook of tests/rulebook_oracle.py against the C restatement of the reference
(oracle.get_indice_pairs) on every geometry the GPU rulebook tests use, the case generators, and the argument
checks of the rulebook C ABI, which return before anything is launched.

Rows outside the grid.  get_valid_out_pos (oracle.c, from geometry.h:24-85) computes
    lowers = (q - (k - 1) * dil - 1 + stride + pad) / stride,   uppers = (q + pad) / stride
with C division, which truncates toward zero.  While q + pad >= 0 on every axis, uppers is exact and a lowers that
rounds up only drops negative candidates, so the enumeration is exact.  Two or more steps outside (q + pad < 0),
uppers rounds up to a site the row does not reach: k3 s2 p1 at q = -2 gives uppers = 0 and an offset term
q - 0 * stride + pad = -1, a pair under a negative offset.  The SubM oracle also keys its site map by the flat
index, which aliases a row outside the grid to another site.  So the oracle is only fed rows inside the grid; what
rows outside it do is defined by the brute force (a strided conv scatters from every row of a valid batch, SubM
only looks rows inside the grid up), and the one-step-outside case is pinned on the device by
test_spconv_gpu.py::test_rulebook_edge_cases."""
import numpy as np
import pytest

import oracle
import rulebook_oracle as R

GEOMS = R.GEOMS

EINVAL, EWORKSPACE = -1, -3


def random_rows(n, batch_size, shape, seed, skip_batch=None):
    rng = np.random.default_rng(seed)
    total = batch_size * int(np.prod(shape))
    flat = rng.choice(total, size=min(n, total), replace=False)
    rows = R.rows_of(np.sort(flat), shape)
    if skip_batch is not None:
        rows = rows[rows[:, 0] != skip_batch]
    return rows[rng.permutation(rows.shape[0])]


@pytest.mark.parametrize("name", list(GEOMS))
@pytest.mark.parametrize("grid", ["odd_b1", "b3_empty_middle"])
def test_brute_force_equals_oracle(name, grid):
    ks, st, pd, dil, subm = GEOMS[name]
    big = int(np.prod(ks)) > 27
    if grid == "odd_b1":
        B, shape, n, skip = 1, ([23, 19, 21] if big else [37, 29, 13]), (300 if big else 2500), None
    else:
        B, shape, n, skip = 3, ([21, 17, 19] if big else [41, 35, 11]), (300 if big else 3000), 1
    rows = random_rows(n, B, shape, seed=len(name) * 7 + B, skip_batch=skip)
    outids, nbr, oshape = R.brute_force(rows, B, shape, ks, st, pd, dil, subm)
    o_outids, o_nbr, o_shape = R.oracle_nbr(rows, B, shape, ks, st, pd, dil, subm)
    assert oshape == o_shape
    assert np.array_equal(outids, o_outids)
    assert np.array_equal(nbr, o_nbr)
    assert (nbr >= 0).sum() > 0
    if not subm:
        assert np.all(np.diff(R.flat_of(outids, oshape)) > 0)
        if skip is not None:
            assert not (outids[:, 0] == skip).any()


def test_brute_force_strided_rows_one_step_outside():
    """the pinned device behaviour (test_rulebook_edge_cases): k3 s2 p1, a row at x = -1 feeds output (0, 0, 0)
    through offset 4; SubM: a row outside finds its in-grid neighbour and is nobody's neighbour."""
    rows = np.array([[0, -1, 0, 0], [0, 0, 0, 0]], np.int32)
    outids, nbr, _ = R.brute_force(rows[:1], 1, [8, 8, 4], [3] * 3, [2] * 3, [1] * 3, [1] * 3, False)
    assert outids.tolist() == [[0, 0, 0, 0]]
    assert nbr[4, 0] == 0 and (np.delete(nbr[:, 0], 4) == -1).all()
    _, nbr, _ = R.brute_force(rows, 1, [8, 8, 4], [3] * 3, [1] * 3, [1] * 3, [1] * 3, True)
    assert nbr[22, 0] == 1 and (np.delete(nbr[:, 0], 22) == -1).all()
    assert nbr[13, 1] == 1 and (np.delete(nbr[:, 1], 13) == -1).all()
    # two steps outside reaches nothing by the definition; rows of a batch out of range reach nothing either
    far = np.array([[0, -2, 0, 0], [1, 0, 0, 0], [-1, 0, 0, 0]], np.int32)
    outids, nbr, _ = R.brute_force(far, 1, [8, 8, 4], [3] * 3, [2] * 3, [1] * 3, [1] * 3, False)
    assert outids.shape[0] == 0 and nbr.shape == (27, 0)


def test_oracle_truncation_quirk_two_steps_outside():
    """the arithmetic of get_valid_out_pos (C truncating division) at q = -2, k3 s2 p1, restated: uppers rounds up
    to 0 and the offset term comes out -1 -- why the oracle is never fed such rows."""
    def cdiv(a, b):
        return int(a / b)

    def enumerated(q, k, s, p):
        """the candidate outputs get_valid_out_pos keeps (val >= 0), with their offset terms (dilation 1)"""
        uppers, lowers = cdiv(q + p, s), cdiv(q - (k - 1) - 1 + s + p, s)
        return {(v, q - v * s + p) for v in range(lowers, uppers + 1) if v >= 0}

    k, s, p = 3, 2, 1
    assert (cdiv(-2 + p, s), cdiv(-2 - (k - 1) - 1 + s + p, s)) == (0, -1)
    assert enumerated(-2, k, s, p) == {(0, -1)}              # a pair under offset -1
    for q in (-1, 0, 1, 2, 5, 6):                            # q + pad >= 0: exactly the definition
        assert enumerated(q, k, s, p) == {(o, q + p - o * s) for o in range(0, 8) if 0 <= q + p - o * s < k}


def test_edge_sites_generator():
    rng = np.random.default_rng(0)
    B, shape = 2, [257, 251, 21]
    tiles = R.num_tiles(B, shape)
    assert 10 <= tiles <= 30
    s = R.edge_sites(B, shape, rng, fill=3000, empty_tiles=range(4, 9))
    total = B * int(np.prod(shape))
    assert s[0] == 0 and s[-1] == total - 1 and np.all(np.diff(s) > 0)
    for t in range(1, tiles):
        if t - 1 not in range(4, 9):
            assert t * R.TILE_SITES - 1 in s
        if t not in range(4, 9):
            assert t * R.TILE_SITES in s
    assert 31 in s and 32 in s
    assert not np.isin(s // R.TILE_SITES, np.arange(4, 9)).any()      # a run of five empty tiles
    rows = R.rows_of(s, shape)
    assert R.in_grid(rows, B, shape).all() and np.array_equal(R.flat_of(rows, shape), s)
    assert rows[-1].tolist() == [B - 1, shape[0] - 1, shape[1] - 1, shape[2] - 1]
    corner = rows[(rows[:, 0] == B - 1) & (rows[:, 1:] >= np.array(shape) - 4).all(1)]
    assert corner.shape[0] == 64                                        # every row that can reach the last site
    # exact multiples of a tile, and one word past
    assert B * int(np.prod(shape)) % R.WORD_SITES != 0                 # a partial last word
    assert 3 * 64 * 64 * 32 == 3 * R.TILE_SITES and R.num_tiles(3, [64, 64, 32]) == 3
    assert 2731 * 3 * 32 == 2 * R.TILE_SITES + R.WORD_SITES and R.num_tiles(1, [2731, 3, 32]) == 3


@pytest.mark.parametrize("name", [g for g in GEOMS if not GEOMS[g][4] and np.prod(GEOMS[g][0]) <= 27])
def test_rows_reaching_generator(name):
    """input rows derived from targeted OUTPUT sites really mark those sites."""
    ks, st, pd, dil, _ = GEOMS[name]
    rng = np.random.default_rng(1)
    B, oshape = 2, [45, 41, 9]
    ishape = R.in_shape_for(oshape, ks, st, pd, dil, [s - 1 for s in st])
    want = R.edge_sites(B, oshape, rng, fill=500)
    rows = R.rows_reaching(want, B, ishape, oshape, ks, st, pd, dil)
    assert R.in_grid(rows, B, ishape).all()
    assert np.unique(R.flat_of(rows, ishape)).size == rows.shape[0]
    outids, nbr, got_shape = R.brute_force(rows, B, ishape, ks, st, pd, dil, False)
    assert got_shape == oshape
    assert np.isin(want, R.flat_of(outids, oshape)).all()


def test_transpose_and_pair_lists():
    rows = random_rows(500, 1, [12, 11, 9], seed=3)
    _, nbr, _ = R.brute_force(rows, 1, [12, 11, 9], [3] * 3, [2] * 3, [1] * 3, [1] * 3, False)
    t = R.transpose(nbr, rows.shape[0])
    for k in range(nbr.shape[0]):
        o = np.nonzero(nbr[k] >= 0)[0]
        assert np.array_equal(t[k, nbr[k, o]], o)
        assert (t[k] >= 0).sum() == o.size
    for k, (i, o) in enumerate(R.pair_lists(nbr)):
        assert np.all(np.diff(o) > 0) and np.array_equal(nbr[k, o], i)


# ------------------------------------------------------------------------------------- C ABI argument checks
def _call_prepare(L, shape, oshape, ks, st, pd, dil, subm, ws_bytes=None, n_in=10, batch=1):
    from bevfusion_b200 import _C
    from bevfusion_b200.spconv.ops import _i32, _vp
    arrs = [_i32(v) for v in (shape, oshape, ks, st, pd, dil)]
    need = L.bevb200_rulebook_workspace_bytes(n_in, batch, _vp(arrs[1]))
    size = need if ws_bytes is None else ws_bytes
    # the checks return before anything touches a pointer: host addresses stand in for device ones
    dummy = _C.host_array(ctypes_int32(), [0] * 64)
    n_out = _C.host_array(ctypes_int32(), [0])
    args = [_vp(a) for a in arrs]
    return L.bevb200_rulebook_prepare(_vp(dummy), n_in, batch, *args, int(subm), _vp(n_out), _vp(dummy), size,
                                      None), need


def ctypes_int32():
    import ctypes
    return ctypes.c_int32


def test_cabi_rejects_bad_geometry_without_launching():
    from bevfusion_b200 import _C
    L = _C.lib()
    before = _C.launch_count()
    shape = [16, 16, 8]
    ok3 = ([3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1])
    rc, _ = _call_prepare(L, shape, [8, 8, 4], [3, 3, 3], [2, 0, 2], [1, 1, 1], [1, 1, 1], False)
    assert rc == EINVAL and b"geometry" in L.bevb200_last_error()              # stride 0
    rc, _ = _call_prepare(L, shape, [8, 8, 4], [3, 3, 3], [2, 2, 2], [1, -1, 1], [1, 1, 1], False)
    assert rc == EINVAL                                                          # negative padding
    rc, _ = _call_prepare(L, shape, [8, 8, 4], [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 0], False)
    assert rc == EINVAL                                                          # dilation 0
    rc, _ = _call_prepare(L, [40, 300, 8], [40, 300, 8], [17, 241, 1], [1, 1, 1], [8, 120, 0], [1, 1, 1], True)
    assert rc == EINVAL and b"4096" in L.bevb200_last_error()                   # kernel volume 4097
    rc, _ = _call_prepare(L, shape, [16, 16, 7], [3, 3, 3], [1, 1, 1], [1, 1, 1], [1, 1, 1], True)
    assert rc == EINVAL and b"SubM" in L.bevb200_last_error()                   # SubM changes the grid
    rc, _ = _call_prepare(L, shape, [8, 8, 4], *ok3, False, n_in=-1)
    assert rc == EINVAL                                                          # negative row count
    rc, _ = _call_prepare(L, shape, [8, 8, 4], *ok3, False, batch=0)
    assert rc == EINVAL                                                          # no batch
    rc, need = _call_prepare(L, shape, [8, 8, 4], *ok3, False, ws_bytes=0)
    assert rc == EWORKSPACE and need > 0
    rc, need = _call_prepare(L, shape, [8, 8, 4], *ok3, False, ws_bytes=need - 1)
    assert rc == EWORKSPACE and b"workspace" in L.bevb200_last_error()
    from bevfusion_b200.spconv.ops import _i32, _vp
    dummy = _C.host_array(ctypes_int32(), [0] * 64)
    rc = L.bevb200_rulebook_fill(_vp(dummy), 10, 1, _vp(_i32(shape)), _vp(_i32([8, 8, 4])), _vp(_i32([3] * 3)),
                                 _vp(_i32([2] * 3)), _vp(_i32([1] * 3)), _vp(_i32([1] * 3)), 0, 5, _vp(dummy),
                                 _vp(dummy), _vp(dummy), 8, None)
    assert rc == EWORKSPACE                                                      # fill checks the same workspace
    need = L.bevb200_rulebook_workspace_bytes(0, 1, _vp(_i32(shape)))          # the SubM gather: bitmap only
    rc = L.bevb200_rulebook_fill_subm_sorted(_vp(dummy), 10, 1, _vp(_i32(shape)), _vp(_i32([3] * 3)),
                                             _vp(_i32([1] * 3)), _vp(dummy), _vp(dummy), need - 1, None)
    assert rc == EWORKSPACE
    rc = L.bevb200_rulebook_fill_subm_sorted(_vp(dummy), 10, 1, _vp(_i32(shape)), _vp(_i32([3] * 3)),
                                             _vp(_i32([0, 1, 1])), _vp(dummy), _vp(dummy), need, None)
    assert rc == EINVAL
    assert _C.launch_count() == before
