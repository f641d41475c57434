"""GPU tests of BEV pooling and the fused LSS lift on every dispatch path, against a float64 reference built directly
from the interval table (starts / lengths / geom, and perm), never from the library's own interval logic.

Forward paths (bevpool.cu), each named by the branch it reaches and told apart by its launch count:
  * tma0    bevb200_bev_pool, tuned C:           bevpool_fwd_tma_kernel<Q, 0> (one bulk copy per stage) + fix-up
  * tma1z   bevb200_bev_pool_perm, tuned C, B*D = 1: bevpool_fwd_tma_kernel<Q, 1>, empty cells zeroed by the warps
  * tma1m   bevb200_bev_pool_perm, tuned C, B*D > 1: the same kernel after a memset of the grid
  * generic either entry, C not tuned or x / out off 16-byte alignment: bevpool_fwd_generic_kernel
  * v1      either entry under BEVB200_POOL_VARIANT=1 (read once per process, so in a subprocess):
            bevpool_fwd_kernel + bevpool_fwd_fixup_kernel
Backward: bevpool_bwd_kernel (tuned C) and bevpool_bwd_generic_kernel, through both entries.  Lift: the column form
(bevpool_lift.cu) and the rows form (bevpool_fwd_tma_kernel<Q, 2>).

Every driver call fills its output with NaN, puts a 4 KiB canary behind the queried workspace, runs twice and must be
bit-identical; the Python wrappers must return the same bits.  Pooling must stay within L * 2^-24 * sum|x_r| of the
float64 sum of each cell's L rows, the lift within (L + 1) * 2^-24 * sum|d_r * ctx_r| (each product is rounded to
fp32 first), so one dropped or doubled row fails in any cell.  Cells without an interval must be exactly +0.0.
Each case prints its path and worst error as a fraction of the bound."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from bevfusion_b200 import _C

pytestmark = pytest.mark.gpu

EINVAL, EWORKSPACE = -1, -3
TUNED = (16, 32, 64, 80, 96, 128, 160, 256)
U = 2.0 ** -24
CANARY = 4096
NUM_SMS = 132
K_LONG_ROWS = 256          # v1 kernel: intervals longer than this are cut at 128-row chunk boundaries
LAUNCHES = {"tma": 3, "generic": 1, "v1": 2}   # kernel launches of one forward call on each path
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ---------------------------------------------------------------------------------------------------- tables
def tma_split(n, c, lift=False):
    """(warps per CTA, rows per warp range) of bevpool_fwd_tma_kernel, restated from the launcher: 3 stages of 32 rows
    in at most 200 KiB of shared memory, at most 8 warps, NUM_SMS * warps ranges, rows per range rounded up to 32."""
    stage = 32 * c * 4 + (128 if lift else 0)
    warps = max(1, min(8, (200 * 1024) // (3 * stage)))
    rpw = -(-n // (NUM_SMS * warps))
    return warps, -(-rpw // 32) * 32


def tiling(bounds, n):
    starts = np.unique(np.asarray([0] + [b for b in bounds if 0 <= b < n], dtype=np.int64)) if n else np.zeros(0, np.int64)
    lengths = np.diff(np.append(starts, n))
    return starts, lengths


def layout(name, n, rpw, rng):
    """(starts, lengths) that tile [0, n)."""
    if name == "ones":
        return tiling(range(n), n)
    if name == "one":                           # every warp range holds only a head piece of the one interval
        return tiling([], n)
    if name == "edges":                         # boundaries at every range boundary R and at R - 1, R + 1
        b = [k * rpw + d for k in range(1, n // rpw + 1) for d in (-1, 0, 1)]
        return tiling(b + list(rng.integers(0, n, n // 50)), n)
    if name == "hot":                           # hot cells with intervals longer than 2 * rpw, between short ones
        b, pos = [], 0
        while pos < n:
            b.append(pos)
            pos += int(2 * rpw + rng.integers(1, rpw + 2)) if rng.random() < 0.15 else int(rng.integers(1, 40))
        return tiling(b, n)
    if name == "random":
        return tiling(list(rng.integers(0, max(n, 1), max(n // 3, 1))), n)
    raise ValueError(name)


def with_gaps(starts, lengths, rng):
    """A table that does not tile: no interval at row 0, rows missing inside intervals, a gap at the end."""
    starts, lengths = starts[1:].copy(), lengths[1:].copy()
    cut = rng.random(lengths.size) < 0.5
    lengths[cut] -= rng.integers(0, lengths[cut])
    if lengths.size:
        if lengths[-1] > 1:
            lengths[-1] //= 2
        else:
            starts, lengths = starts[:-1], lengths[:-1]
    return starts, lengths


def decode(cells, dims):
    """(x, y, z, b) of flat cells of [B, D, H, W]; cell -1 gives a coordinate outside the grid (cycling the axes)."""
    B, D, H, W = dims
    cells = np.asarray(cells, dtype=np.int64)
    g = np.stack([(cells // W) % H, cells % W, (cells // (W * H)) % D, cells // (W * H * D)], 1)
    bad = np.array([[H, 0, 0, 0], [0, W, 0, 0], [0, 0, D, 0], [0, 0, 0, B], [-1, 0, 0, 0], [0, 0, 0, -1]])
    out = np.nonzero(cells < 0)[0]
    g[out] = bad[np.arange(out.size) % len(bad)]
    return g.astype(np.int32)


def grid_for(n_int, B=1, D=1):
    side = int(np.ceil(np.sqrt((2 * n_int + 16) / (B * D))))
    return (B, D, side, side + 1)


class Case:
    """One pooling problem.  Sorted entry: x [n, c] are the sorted rows.  Perm entry: x [n_total, c] in original order
    and sorted row r is x[perm[r]]; perm[n:] are the filtered rows."""

    def __init__(self, dev, dims, c, n, starts, lengths, cells, rng, use_perm, extra=37):
        self.dims, self.c, self.n = tuple(dims), c, n
        self.starts_np, self.lengths_np = starts.astype(np.int32), lengths.astype(np.int32)
        self.n_int = starts.size
        # every row of an interval carries its cell; rows in gaps carry a random in-grid cell
        total = int(np.prod(dims))
        row_cell = rng.integers(0, total, n)
        for s, L, cl in zip(starts, lengths, cells):
            row_cell[s:s + max(int(L), 1)] = cl
        self.geom_np = decode(row_cell, dims).reshape(n, 4)
        self.perm_np = None
        n_rows = n
        if use_perm:
            n_rows = n + extra
            self.perm_np = rng.permutation(n_rows).astype(np.int32)
        self.x_np = rng.standard_normal((n_rows, c)).astype(np.float32)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        self.x, self.geom = t(self.x_np), t(self.geom_np).reshape(n, 4)
        self.starts, self.lengths = t(self.starts_np), t(self.lengths_np)
        self.perm = None if self.perm_np is None else t(self.perm_np)
        self.n_total = n_rows

    @property
    def entry(self):
        return "perm" if self.perm is not None else "sorted"


def make_case(dev, c, n, lay="edges", dims=None, use_perm=False, seed=0, gaps=False, bad_cells=0, cells=None, B=1, D=1):
    rng = np.random.default_rng(seed)
    _, rpw = tma_split(n, c)
    starts, lengths = layout(lay, n, rpw, rng)
    if gaps:
        starts, lengths = with_gaps(starts, lengths, rng)
    dims = dims or grid_for(starts.size, B, D)
    if cells is None:
        cells = np.sort(rng.choice(int(np.prod(dims)), starts.size, replace=False))
    cells = np.asarray(cells, dtype=np.int64).copy()
    if bad_cells:
        cells[rng.choice(cells.size, min(bad_cells, cells.size), replace=False)] = -1
    return Case(dev, dims, c, n, starts, lengths, cells, rng, use_perm)


# ---------------------------------------------------------------------------------------------------- reference
def covered(starts, lengths, n):
    """(row, owning interval) of every row inside [starts[i], starts[i] + lengths[i]) n [0, n)."""
    s, L = starts.astype(np.int64), lengths.astype(np.int64)
    ok = (L > 0) & (s >= 0) & (s < n)
    e = np.minimum(s + L, n)
    idx = np.nonzero(ok)[0]
    cnt = e[ok] - s[ok]
    first = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64)
    rows = np.repeat(s[ok] - first, cnt) + np.arange(int(cnt.sum()), dtype=np.int64)
    return rows, np.repeat(idx, cnt)


def cell_of(g, dims):
    B, D, H, W = dims
    g = g.astype(np.int64)
    x, y, z, b = g[:, 0], g[:, 1], g[:, 2], g[:, 3]
    ok = (x >= 0) & (x < H) & (y >= 0) & (y < W) & (z >= 0) & (z < D) & (b >= 0) & (b < B)
    return np.where(ok, ((b * D + z) * H + x) * W + y, -1)


def interval_cells(case):
    s = case.starts_np.astype(np.int64)
    inside = (s >= 0) & (s < case.n)
    cells = np.full(s.size, -1, dtype=np.int64)
    cells[inside] = cell_of(case.geom_np[s[inside]], case.dims)
    return cells


def pool_reference(case):
    """float64 sums, sums of |x| and row counts per cell; `has` marks the cells that head an interval."""
    dev = case.x.device
    total = int(np.prod(case.dims))
    rows, owner = covered(case.starts_np, case.lengths_np, case.n)
    icell = interval_cells(case)
    rc = icell[owner]
    keep = rc >= 0
    rows, rc = rows[keep], rc[keep]
    src = case.perm_np[rows] if case.perm_np is not None else rows
    src_t, rc_t = torch.from_numpy(src).to(dev), torch.from_numpy(rc).to(dev)
    v = case.x[src_t].double()
    ref = torch.zeros(total, case.c, dtype=torch.float64, device=dev).index_add_(0, rc_t, v)
    mag = torch.zeros(total, case.c, dtype=torch.float64, device=dev).index_add_(0, rc_t, v.abs())
    cnt = torch.from_numpy(np.bincount(rc, minlength=total).astype(np.float64)).to(dev)
    has = np.zeros(total, dtype=bool)
    has[icell[icell >= 0]] = True
    return ref, mag, cnt, torch.from_numpy(has).to(dev)


def check_sums(got, ref, mag, cnt, has, slack, what):
    """|got - ref| <= (cnt + slack) * 2^-24 * mag per element; cells without an interval exactly +0.0.
    Returns the worst error as a fraction of its bound."""
    c = ref.shape[1]
    got = got.reshape(-1, c)
    assert not bool(torch.isnan(got).any()), "%s: elements left unwritten (NaN)" % what
    err = (got.double() - ref).abs()
    bound = (cnt[:, None] + slack) * U * mag
    bad = err > bound
    assert not bool(bad.any()), "%s: %d elements out of bound, e.g. cell %d" % (
        what, int(bad.sum()), int(torch.nonzero(bad)[0, 0]))
    empty = got[~has]
    assert bool((empty == 0).all()) and not bool(torch.signbit(empty).any()), "%s: a cell without interval is not +0" % what
    pos = bound > 0
    worst = float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0
    print("[%s] worst error / bound = %.3g" % (what, worst))
    return worst


# ---------------------------------------------------------------------------------------------------- drivers
def misalign(t):
    """The same values 4 bytes past a 16-byte boundary (a fresh allocation is 256-byte aligned)."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    buf[1:] = t.flatten()
    v = buf[1:].view(t.shape)
    assert v.data_ptr() % 16 == 4
    return v


def workspace(nbytes, dev):
    ws = torch.empty(int(nbytes) + CANARY, dtype=torch.uint8, device=dev)
    pattern = ((torch.arange(CANARY, device=dev) * 7 + 3) % 256).to(torch.uint8)
    ws[int(nbytes):] = pattern
    return ws, pattern


def run_twice(fn, out, ws=None, pattern=None, nbytes=0, launches=None):
    """fn() into `out` twice over a NaN prefill: both runs succeed and agree bit for bit, the canary behind the
    workspace is intact, and (when given) each run issues `launches` kernels."""
    res = []
    for _ in range(2):
        out.fill_(float("nan"))
        torch.cuda.synchronize()
        _C.reset_launch_count()
        rc = fn()
        torch.cuda.synchronize()
        assert rc == 0, _C.lib().bevb200_last_error()
        if launches is not None:
            assert _C.launch_count() == launches, "ran %d kernels, expected %d" % (_C.launch_count(), launches)
        res.append(out.clone())
    assert torch.equal(res[0].view(torch.int32), res[1].view(torch.int32)), "not bit-reproducible"
    if ws is not None:
        assert torch.equal(ws[nbytes:], pattern), "workspace canary overwritten"
    return res[0]


def pool_driver(case, x=None, out=None, launches=None, ws_bytes=None):
    """bevb200_bev_pool (sorted case) or bevb200_bev_pool_perm through the C ABI."""
    L = _C.lib()
    x = case.x if x is None else x
    dev = x.device
    B, D, H, W = case.dims
    nbytes = L.bevb200_bev_pool_workspace_bytes(case.n, case.c)
    ws, pattern = workspace(nbytes, dev)
    if out is None:
        out = torch.empty(B, D, H, W, case.c, device=dev)
    size = nbytes if ws_bytes is None else ws_bytes
    common = (_C.ptr(case.geom), _C.ptr(case.starts), _C.ptr(case.lengths), _C.ptr(out), _C.ptr(ws), size,
              _C.current_stream(dev))
    if case.perm is None:
        fn = lambda: L.bevb200_bev_pool(B, D, H, W, case.n, case.c, case.n_int, _C.ptr(x), *common)
    else:
        fn = lambda: L.bevb200_bev_pool_perm(B, D, H, W, case.n, case.c, case.n_int, _C.ptr(x), _C.ptr(case.perm),
                                             *common)
    if ws_bytes is not None:      # one call, expected to be refused
        out.fill_(float("nan"))
        rc = fn()
        torch.cuda.synchronize()
        return rc, out
    return run_twice(fn, out, ws, pattern, nbytes, launches)


def plan_shell(case):
    """A BEVPoolPlan over the case's tables (what BEVPoolPlan.pool runs)."""
    from bevfusion_b200.bev_pool import BEVPoolPlan, _PoolTables
    plan = BEVPoolPlan.__new__(BEVPoolPlan)
    plan.tables = _PoolTables(None, case.perm, case.geom, case.starts, case.lengths, case.n, case.n_int,
                              case.n_total, case.dims)
    return plan


def wrapper_forward(case, x):
    from bevfusion_b200.bev_pool import bev_pool_ext
    if case.perm is None:
        return bev_pool_ext.bev_pool_forward(x, case.geom, case.lengths, case.starts, *case.dims)
    return plan_shell(case).pool(x)


def check_forward(case, path, what, mis=""):
    """Driver vs float64 and vs the Python wrapper.  mis: 'x' and / or 'o' (out) 4 bytes off alignment."""
    x = misalign(case.x) if "x" in mis else case.x
    B, D, H, W = case.dims
    out = misalign(torch.empty(B, D, H, W, case.c, device=x.device)) if "o" in mis else None
    got = pool_driver(case, x=x, out=out, launches=LAUNCHES[path] if case.n and case.n_int else 0)
    worst = check_sums(got, *pool_reference(case), 0, "%s %s" % (path, what))
    if "o" not in mis:
        py = wrapper_forward(case, x)
        assert torch.equal(py.view(torch.int32), got.view(torch.int32)), "Python wrapper differs from the C ABI"
    return worst


# ---------------------------------------------------------------------------------------------------- forward matrix
@pytest.mark.parametrize("c", TUNED)
@pytest.mark.parametrize("entry", ["sorted", "perm"])
def test_forward_every_tuned_width(cuda, c, entry):
    """tma0 (sorted) and tma1z (perm, B*D = 1) at every tuned C, with hot cells longer than 2 * rpw."""
    case = make_case(cuda, c, 20011, "hot", use_perm=entry == "perm", seed=c)
    assert case.lengths_np.max() > 2 * tma_split(case.n, c)[1]
    check_forward(case, "tma", "%s C=%d" % ({"sorted": "tma0", "perm": "tma1z"}[entry], c))


LAYOUTS = [("ones", 3000), ("one", 5000), ("edges", 20000), ("edges", 33825), ("edges", 70001), ("hot", 40000),
           ("random", 1), ("random", 31), ("random", 32), ("random", 33)]


@pytest.mark.parametrize("c", [16, 80, 256])
@pytest.mark.parametrize("lay,n", LAYOUTS)
@pytest.mark.parametrize("entry", ["sorted", "perm"])
def test_forward_interval_layouts(cuda, c, lay, n, entry):
    """Range boundaries of the TMA kernel: lengths 1, one interval over all rows, boundaries at R and R +- 1 while n
    sweeps the split, intervals longer than 2 * rpw, n < 32 and n around one stage, and rpw > 32."""
    case = make_case(cuda, c, n, lay, use_perm=entry == "perm", seed=n + c)
    check_forward(case, "tma", "%s C=%d %s n=%d" % ({"sorted": "tma0", "perm": "tma1z"}[entry], c, lay, n))


def test_forward_layouts_reach_rpw_above_32():
    assert all(tma_split(70001, c)[1] > 32 for c in (16, 80, 256))
    assert {tma_split(33825, 16)[1], tma_split(20000, 16)[1]} == {64, 32}


@pytest.mark.parametrize("c", [16, 80, 256])
@pytest.mark.parametrize("B,D", [(2, 1), (1, 2)])
def test_forward_perm_memset(cuda, c, B, D):
    """tma1m: B = 2 or nz = 2, the grid is zeroed by a memset and the kernel writes occupied cells only."""
    case = make_case(cuda, c, 30000, "hot", use_perm=True, seed=c + B, B=B, D=D)
    check_forward(case, "tma", "tma1m C=%d B=%d D=%d" % (c, B, D))


@pytest.mark.parametrize("entry", ["sorted", "perm"])
@pytest.mark.parametrize("c,mis", [(4, ""), (7, ""), (20, ""), (80, "x"), (80, "o"), (256, "x")])
def test_forward_generic(cuda, entry, c, mis):
    """The generic kernel: C not tuned, or x / out off 16-byte alignment at a tuned C."""
    case = make_case(cuda, c, 9001, "hot", use_perm=entry == "perm", seed=c)
    check_forward(case, "generic", "generic %s C=%d mis=%s" % (entry, c, mis or "-"), mis)


@pytest.mark.parametrize("c", [16, 80, 256])
@pytest.mark.parametrize("pattern", ["first_gt0", "last_lt_end", "gaps", "single", "both_ends"])
def test_zero_fill_edges(cuda, c, pattern):
    """tma1z over a NaN prefill: nothing but the pooling warps writes the grid, so every empty cell before the first
    interval, between intervals (gaps of one and of many cells) and after the last must come out +0."""
    rng = np.random.default_rng(c)
    n = 6000
    starts, _ = layout("random", n, 32, rng)
    n_int = starts.size if pattern != "single" else 1
    dims = (1, 1, 64, 67) if pattern != "gaps" else (1, 1, 100, 100)
    total = int(np.prod(dims))
    if pattern == "first_gt0":
        cells = 5 + np.arange(n_int)
    elif pattern == "last_lt_end":
        cells = np.arange(n_int)
    elif pattern == "gaps":                 # alternating gaps of exactly one cell and of many cells
        steps = np.where(np.arange(n_int) % 2 == 0, 2, 3 + rng.integers(1, 4, n_int))
        cells = np.cumsum(steps) - 2
        assert cells[-1] < total - 1
    elif pattern == "single":
        cells = np.array([total // 3])
    else:                                   # cell 0 and the last cell both occupied
        cells = np.concatenate([[0], np.sort(rng.choice(np.arange(1, total - 1), n_int - 2, replace=False)), [total - 1]])
    if pattern == "single":
        starts = np.array([0])
    lengths = np.diff(np.append(starts, n))
    case = Case(cuda, dims, c, n, starts, lengths, cells, rng, use_perm=True)
    check_forward(case, "tma", "tma1z C=%d zfill %s" % (c, pattern))


# ---------------------------------------------------------------------------------------------------- non-tiling
@pytest.mark.parametrize("c", [16, 80, 256, 20])
@pytest.mark.parametrize("lay,n", [("edges", 20000), ("hot", 40000), ("random", 33)])
def test_forward_non_tiling_tables(cuda, c, lay, n):
    """bevb200_bev_pool with a leading gap, rows missing inside intervals and a trailing gap: the forward sums
    x[s, s + L) only, as the reference kernel does, at a tuned C (tma0) and an untuned one (generic)."""
    case = make_case(cuda, c, n, lay, seed=n + c, gaps=True)
    assert case.starts_np[0] > 0 and case.starts_np[-1] + case.lengths_np[-1] < n
    check_forward(case, "tma" if c in TUNED else "generic", "%s C=%d non-tiling %s n=%d" % (
        "tma0" if c in TUNED else "generic", c, lay, n))


@pytest.mark.parametrize("c", [80, 20])
@pytest.mark.parametrize("entry", ["sorted", "perm"])
def test_forward_out_of_grid_rows(cuda, c, entry):
    """Intervals whose geom lies outside the grid on any axis are skipped (perm entry: B = 2, the memset path)."""
    case = make_case(cuda, c, 15000, "hot", use_perm=entry == "perm", seed=3, bad_cells=40, B=2)
    path = "tma" if c in TUNED else "generic"
    check_forward(case, path, "%s %s C=%d out-of-grid" % (path, entry, c))


# ---------------------------------------------------------------------------------------------------- v1 subprocess
V1_CHILD = r"""
import sys
import numpy as np
import torch
sys.path[:0] = [sys.argv[1], sys.argv[2]]
from bevfusion_b200 import _C
_C.LIB_PATH = sys.argv[5]
import test_bev_pool_dispatch_gpu as T
dev = torch.device("cuda:0")
src = np.load(sys.argv[3])
res = {}
for k in range(int(src["count"])):
    case = T.case_from_arrays(src, k, dev)
    res["out%d" % k] = T.pool_driver(case, launches=T.LAUNCHES["v1"]).cpu().numpy()
np.savez(sys.argv[4], **res)
"""


def v1_cases(dev):
    cases = []
    for c in TUNED:
        for entry in ("sorted", "perm"):
            cases.append(("v1 %s C=%d long" % (entry, c),
                          make_case(dev, c, 12000, "hot", use_perm=entry == "perm", seed=100 + c)))
    for c in (16, 80, 256):
        cases.append(("v1 sorted C=%d non-tiling" % c, make_case(dev, c, 20000, "hot", seed=7 + c, gaps=True)))
    cases.append(("v1 sorted C=80 out-of-grid", make_case(dev, 80, 15000, "hot", seed=3, bad_cells=40, B=2)))
    return cases


def case_from_arrays(src, k, dev):
    p = "c%d_" % k
    case = Case.__new__(Case)
    case.dims = tuple(int(v) for v in src[p + "dims"])
    case.c, case.n = int(src[p + "x"].shape[1]), int(src[p + "n"])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    case.x, case.geom = t(src[p + "x"]), t(src[p + "geom"]).reshape(case.n, 4)
    case.starts, case.lengths = t(src[p + "starts"]), t(src[p + "lengths"])
    case.n_int = int(src[p + "starts"].size)
    case.perm = t(src[p + "perm"]) if src[p + "perm"].size else None
    case.n_total = int(src[p + "x"].shape[0])
    return case


@pytest.fixture(scope="module")
def v1_results(cuda, tmp_path_factory):
    """Every v1 case run once in a child process with BEVB200_POOL_VARIANT=1, loading the same library."""
    cases = v1_cases(cuda)
    d = tmp_path_factory.mktemp("v1")
    arrays = {"count": np.array(len(cases))}
    for k, (_, cs) in enumerate(cases):
        p = "c%d_" % k
        arrays.update({p + "dims": np.array(cs.dims), p + "x": cs.x_np, p + "n": np.array(cs.n), p + "geom": cs.geom_np,
                       p + "starts": cs.starts_np, p + "lengths": cs.lengths_np,
                       p + "perm": cs.perm_np if cs.perm_np is not None else np.zeros(0, np.int32)})
    np.savez(d / "in.npz", **arrays)
    env = dict(os.environ, BEVB200_POOL_VARIANT="1")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", V1_CHILD, HERE, ROOT, str(d / "in.npz"), str(d / "out.npz"), _C.LIB_PATH]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = np.load(d / "out.npz")
    return [(name, cs, torch.from_numpy(out["out%d" % k]).to(cuda)) for k, (name, cs) in enumerate(cases)]


def test_forward_v1_register_kernel(cuda, v1_results):
    """bevpool_fwd_kernel at every tuned C through both entries, with intervals longer than kLongRows that cross
    128-row chunks, a non-tiling table and out-of-grid rows."""
    long_seen = False
    for name, case, got in v1_results:
        long_seen |= bool((case.lengths_np > K_LONG_ROWS).any() and
                          ((case.starts_np[case.lengths_np > K_LONG_ROWS] % 128) != 0).any())
        check_sums(got, *pool_reference(case), 0, name)
    assert long_seen


# ---------------------------------------------------------------------------------------------------- edges
@pytest.mark.parametrize("entry", ["sorted", "perm"])
@pytest.mark.parametrize("n,n_int", [(0, 0), (500, 0)])
def test_empty_tables_zero_the_grid(cuda, entry, n, n_int):
    rng = np.random.default_rng(0)
    case = Case(cuda, (1, 1, 16, 17), 80, n, np.zeros(0, np.int64), np.zeros(0, np.int64), [], rng,
                use_perm=entry == "perm")
    got = pool_driver(case, launches=0)
    assert bool((got == 0).all()) and not bool(torch.signbit(got).any())


def test_plan_entirely_outside_the_grid(cuda):
    """n_kept = 0: pool gives zeros, grad_perm zeroes every row (NaN prefills through the C ABI)."""
    from bevfusion_b200 import synthetic as S
    from bevfusion_b200.bev_pool import BEVPoolPlan
    geom, cfg = S.camera_geometry("tiny", device=cuda)
    plan = BEVPoolPlan((geom + 1000.0).contiguous(), cfg["xbound"], cfg["ybound"], cfg["zbound"])
    t = plan.tables
    assert t.n_kept == 0 and t.n_intervals == 0
    x = torch.randn(t.n_total, 80, device=cuda)
    assert bool((plan.pool(x) == 0).all())
    case = Case.__new__(Case)
    case.dims, case.c, case.n, case.n_int, case.n_total = t.dims, 80, 0, 0, t.n_total
    case.x, case.perm, case.geom, case.starts, case.lengths = x, t.perm, t.geom, t.starts, t.lengths
    got = pool_driver(case, launches=0)
    assert bool((got == 0).all())
    og = torch.randn(*t.dims, 80, device=cuda)
    xg = torch.empty(t.n_total, 80, device=cuda)
    L = _C.lib()
    got = run_twice(lambda: L.bevb200_bev_pool_grad_perm(*t.dims, 0, t.n_total, 80, 0, _C.ptr(og), _C.ptr(t.perm),
                                                         _C.ptr(t.geom), _C.ptr(t.starts), _C.ptr(t.lengths),
                                                         _C.ptr(xg), _C.current_stream(cuda)), xg)
    assert bool((got == 0).all())


@pytest.mark.parametrize("entry", ["sorted", "perm"])
@pytest.mark.parametrize("c", [80, 256])
def test_workspace_too_small_is_refused_before_writing(cuda, entry, c):
    case = make_case(cuda, c, 5000, "hot", use_perm=entry == "perm", seed=1)
    need = _C.lib().bevb200_bev_pool_workspace_bytes(case.n, c)
    for size in (need - 16, 0):
        rc, out = pool_driver(case, ws_bytes=size)
        assert rc == EWORKSPACE
        assert bool(torch.isnan(out).all()), "out was written by a refused call"


# ---------------------------------------------------------------------------------------------------- backward
def grad_expected(case, og):
    """x_grad: the gradient of the cell of each covered row with an in-grid interval; 0 for every other row."""
    c = case.c
    rows, owner = covered(case.starts_np, case.lengths_np, case.n)
    rc = interval_cells(case)[owner]
    keep = rc >= 0
    rows, rc = rows[keep], rc[keep]
    dst = case.perm_np[rows] if case.perm_np is not None else rows
    exp = torch.zeros(case.n_total, c, device=og.device)
    exp[torch.from_numpy(dst).to(og.device)] = og.reshape(-1, c)[torch.from_numpy(rc).to(og.device)]
    return exp


def grad_driver(case, og, xg):
    L = _C.lib()
    args = (_C.ptr(case.geom), _C.ptr(case.starts), _C.ptr(case.lengths), _C.ptr(xg), _C.current_stream(og.device))
    if case.perm is None:
        fn = lambda: L.bevb200_bev_pool_grad(*case.dims, case.n, case.c, case.n_int, _C.ptr(og), *args)
    else:
        fn = lambda: L.bevb200_bev_pool_grad_perm(*case.dims, case.n, case.n_total, case.c, case.n_int, _C.ptr(og),
                                                  _C.ptr(case.perm), *args)
    return run_twice(fn, xg)


@pytest.mark.parametrize("entry", ["sorted", "perm"])
@pytest.mark.parametrize("c,mis,gaps", [(cc, "", False) for cc in TUNED] + [
    (7, "", False), (20, "", False), (80, "g", False), (80, "x", False), (80, "", True), (20, "", True),
    (256, "", True)])
def test_backward(cuda, entry, c, mis, gaps):
    """bev_pool_grad / bev_pool_grad_perm: a copy, so bit-exact against the gather; rows outside every interval, rows
    of out-of-grid intervals and the filtered tail of perm are zero over a NaN prefill.  mis: out_grad ('g') or
    x_grad ('x') 4 bytes off alignment (the generic kernel)."""
    if gaps and entry == "perm":
        pytest.skip("perm tables come from bevb200_bev_pool_prepare_* and tile [0, n)")
    case = make_case(cuda, c, 20011, "hot", use_perm=entry == "perm", seed=c, gaps=gaps, bad_cells=5, B=2)
    g = torch.Generator(device=cuda).manual_seed(c)
    og = torch.randn(*case.dims, c, generator=g, device=cuda)
    if "g" in mis:
        og = misalign(og)
    xg = torch.empty(case.n_total, c, device=cuda)
    if "x" in mis:
        xg = misalign(xg)
    got = grad_driver(case, og, xg)
    exp = grad_expected(case, og)
    assert torch.equal(got.view(torch.int32), exp.view(torch.int32))
    if not mis:
        if case.perm is None:
            from bevfusion_b200.bev_pool import bev_pool_ext
            py = bev_pool_ext.bev_pool_backward(og, case.geom, case.lengths, case.starts, *case.dims)
        else:
            x = case.x.clone().requires_grad_(True)
            (plan_shell(case).pool(x) * og).sum().backward()
            py = x.grad
        assert torch.equal(py.view(torch.int32), got.view(torch.int32))


# ---------------------------------------------------------------------------------------------------- drop-in bev_pool
@pytest.mark.parametrize("c", [16, 80, 20])
def test_bev_pool_function_matches_driver(cuda, c):
    """bev_pool(feats, coords, ...) == the perm driver over the same prepared tables, bit for bit."""
    from bevfusion_b200.bev_pool import bev_pool, prepare_from_coords
    rng = np.random.default_rng(c)
    B, D, H, W, n = 1, 1, 30, 40, 20000
    coords = np.stack([rng.integers(-1, H + 1, n), rng.integers(0, W, n), rng.integers(0, D, n),
                       rng.integers(0, B, n)], 1)
    coords_t = torch.from_numpy(coords).to(cuda)
    feats = torch.from_numpy(rng.standard_normal((n, c)).astype(np.float32)).to(cuda)
    t = prepare_from_coords(coords_t, B, D, H, W)
    assert 0 < t.n_kept < n
    case = Case.__new__(Case)
    case.dims, case.c, case.n, case.n_int, case.n_total = t.dims, c, t.n_kept, t.n_intervals, n
    case.x, case.perm, case.geom, case.starts, case.lengths = feats, t.perm, t.geom, t.starts, t.lengths
    got = pool_driver(case, launches=LAUNCHES["tma" if c in TUNED else "generic"])
    py = bev_pool(feats, coords_t, B, D, H, W)
    assert torch.equal(py.permute(0, 2, 3, 4, 1).contiguous().view(torch.int32), got.view(torch.int32))


# ---------------------------------------------------------------------------------------------------- lift forward
def lift_geometry(dev, kind):
    from bevfusion_b200 import synthetic as S
    from bevfusion_b200.vtransform import create_frustum, get_geometry
    cfg = S.CONFIGS["tiny"]
    if kind == "fh72":
        rig = {k: v.to(dev) for k, v in S.camera_rig(cfg["n_cam"], cfg["image_size"], 1).items()}
        frustum = create_frustum(cfg["image_size"], (72, 8), cfg["dbound"]).to(dev)
        geom = get_geometry(frustum, rig["camera2lidar_rots"], rig["camera2lidar_trans"], rig["intrins"],
                            rig["post_rots"], rig["post_trans"])
    else:
        geom, _ = S.camera_geometry("tiny", batch=2 if kind == "b2" else 1, device=dev)
        if kind == "jitter":               # pixels of a column scatter over cells; columns 0..2 of camera 0 leave the grid
            g = torch.Generator(device=dev).manual_seed(7)
            geom = geom + torch.randn(geom.shape, generator=g, device=dev) * 1.5
            geom[:, 0, :, :, 0:3, 0] += 100.0
    return geom.contiguous(), cfg


def lift_reference(plan, depth, ctx):
    t = plan.tables
    C = ctx.shape[-1]
    total = int(np.prod(t.dims))
    x = (depth.double().unsqueeze(-1) * ctx.double().unsqueeze(2)).reshape(-1, C)
    cells = torch.from_numpy(cell_of(t.geom.cpu().numpy(), t.dims)).to(depth.device)
    assert bool((cells >= 0).all())
    v = x[t.perm[:t.n_kept].long()]
    ref = torch.zeros(total, C, dtype=torch.float64, device=depth.device).index_add_(0, cells, v)
    mag = torch.zeros(total, C, dtype=torch.float64, device=depth.device).index_add_(0, cells, v.abs())
    cnt = torch.bincount(cells, minlength=total).double()
    return ref, mag, cnt, cnt > 0


def lift_rows_driver(plan, depth, ctx):
    L = _C.lib()
    t = plan.tables
    B, N, D, fH, fW = depth.shape
    c = ctx.shape[-1]
    dev = depth.device
    nbytes = L.bevb200_bev_pool_workspace_bytes(t.n_kept, c)
    ws, pattern = workspace(nbytes, dev)
    out = torch.empty(*t.dims, c, device=dev)
    fn = lambda: L.bevb200_bev_pool_lift(*t.dims, t.n_kept, c, t.n_intervals, _C.ptr(depth), _C.ptr(ctx), D, fH * fW,
                                         _C.ptr(t.perm), _C.ptr(t.geom), _C.ptr(t.starts), _C.ptr(t.lengths),
                                         _C.ptr(out), _C.ptr(ws), nbytes, _C.current_stream(dev))
    return run_twice(fn, out, ws, pattern, nbytes, launches=3)


def lift_columns_driver(plan, depth, ctx, n_seg=None):
    L = _C.lib()
    t = plan.tables
    B, N, D, fH, fW = depth.shape
    c = ctx.shape[-1]
    dev = depth.device
    col_begin, seg_key, seg_mask, seg_slot, ival_begin, ns = plan._lift_tables(B * N, D, fH, fW)
    ns = ns if n_seg is None else n_seg
    nbytes = L.bevb200_bev_pool_lift_columns_workspace_bytes(ns, t.n_intervals, c)
    ws, pattern = workspace(nbytes, dev)
    out = torch.empty(*t.dims, c, device=dev)
    fn = lambda: L.bevb200_bev_pool_lift_columns(
        *t.dims, t.n_kept, c, t.n_intervals, _C.ptr(depth), _C.ptr(ctx), B * N, D, fH, fW, _C.ptr(t.geom),
        _C.ptr(t.starts), _C.ptr(col_begin), _C.ptr(seg_key), _C.ptr(seg_mask), _C.ptr(seg_slot), _C.ptr(ival_begin),
        ns, _C.ptr(out), _C.ptr(ws), nbytes, _C.current_stream(dev))
    return run_twice(fn, out, ws, pattern, nbytes, launches=3 if ns else 0)


def lift_inputs(dev, kind, c, seed):
    from bevfusion_b200.bev_pool import BEVPoolPlan
    geom, cfg = lift_geometry(dev, kind)
    plan = BEVPoolPlan(geom, cfg["xbound"], cfg["ybound"], cfg["zbound"])
    B, N, D, fH, fW, _ = geom.shape
    g = torch.Generator(device=dev).manual_seed(seed)
    depth = torch.softmax(torch.randn(B, N, D, fH, fW, generator=g, device=dev), dim=2).contiguous()
    ctx = torch.randn(B, N, fH, fW, c, generator=g, device=dev)
    return plan, depth, ctx


@pytest.mark.parametrize("c", TUNED)
@pytest.mark.parametrize("kind", ["b1", "b2", "jitter", "fh72"])
def test_lift_forward(cuda, monkeypatch, c, kind):
    """Column form and rows form (bevpool_fwd_tma_kernel<Q, 2>) against the float64 lift: tiny rig at B = 1 (the
    kernels zero the grid themselves) and B = 2 (memset), jittered geometry with columns off the grid, and fH = 72
    where only the rows form exists.  plan.lift_pool returns the driver's bits."""
    plan, depth, ctx = lift_inputs(cuda, kind, c, seed=c)
    if kind == "jitter":
        assert plan.tables.n_kept < plan.tables.n_total
    ref = lift_reference(plan, depth, ctx)
    monkeypatch.setenv("BEVB200_LIFT_VARIANT", "rows")
    rows = lift_rows_driver(plan, depth, ctx)
    check_sums(rows, *ref, 1, "lift rows C=%d %s" % (c, kind))
    assert torch.equal(plan.lift_pool(depth, ctx).view(torch.int32), rows.view(torch.int32))
    monkeypatch.delenv("BEVB200_LIFT_VARIANT")
    if kind == "fh72":
        assert getattr(plan, "_lift_cache", None) is None
        return
    cols = lift_columns_driver(plan, depth, ctx)
    check_sums(cols, *ref, 1, "lift columns C=%d %s" % (c, kind))
    assert torch.equal(plan.lift_pool(depth, ctx).view(torch.int32), cols.view(torch.int32))


def test_lift_untuned_width_is_refused(cuda, monkeypatch):
    plan, depth, ctx = lift_inputs(cuda, "b1", 20, seed=0)
    with pytest.raises(_C.BevB200Error):
        plan.lift_pool(depth, ctx)
    monkeypatch.setenv("BEVB200_LIFT_VARIANT", "rows")
    with pytest.raises(_C.BevB200Error):
        plan.lift_pool(depth, ctx)


def test_lift_columns_without_segments_zero_the_grid(cuda):
    """B = 1 with no segment: the cells kernel that zero-fills does not run, so the grid must be zeroed otherwise."""
    plan, depth, ctx = lift_inputs(cuda, "b1", 80, seed=0)
    got = lift_columns_driver(plan, depth, ctx, n_seg=0)
    assert bool((got == 0).all())


# ---------------------------------------------------------------------------------------------------- channels first
@pytest.mark.parametrize("batch,nz,rows,c", [(1, 1, 1, 1), (2, 3, 1023, 7), (1, 2, 4096, 80), (2, 1, 33, 256)])
def test_channels_first(cuda, batch, nz, rows, c):
    """[batch, nz, rows, c] -> [batch, nz*c, rows], bit-exact against permute, into a dense output and into a channel
    slice of a wider NaN-filled buffer (out_batch_stride) whose other channels stay NaN; a stride that is too small
    is refused."""
    L = _C.lib()
    g = torch.Generator(device=cuda).manual_seed(rows)
    x = torch.randn(batch, nz, rows, c, generator=g, device=cuda)
    exp = x.permute(0, 1, 3, 2).reshape(batch, nz * c, rows)
    out = torch.empty(batch, nz * c, rows, device=cuda)
    got = run_twice(lambda: L.bevb200_bev_channels_first(_C.ptr(x), _C.ptr(out), batch, nz, rows, c, 0,
                                                         _C.current_stream(cuda)), out, launches=1)
    assert torch.equal(got.view(torch.int32), exp.view(torch.int32))
    lo, extra = 3, 5
    wide = torch.empty(batch, lo + nz * c + extra, rows, device=cuda)
    stride = wide.shape[1] * rows
    got = run_twice(lambda: L.bevb200_bev_channels_first(_C.ptr(x), _C.ptr(wide[:, lo:]), batch, nz, rows, c, stride,
                                                         _C.current_stream(cuda)), wide, launches=1)
    assert torch.equal(got[:, lo:lo + nz * c].contiguous().view(torch.int32), exp.view(torch.int32))
    assert bool(torch.isnan(got[:, :lo]).all()) and bool(torch.isnan(got[:, lo + nz * c:]).all())
    wide.fill_(float("nan"))
    too_small = nz * rows * c - 1 or -1        # 0 would select the dense default
    rc = L.bevb200_bev_channels_first(_C.ptr(x), _C.ptr(wide), batch, nz, rows, c, too_small,
                                      _C.current_stream(cuda))
    torch.cuda.synchronize()
    assert rc == EINVAL and bool(torch.isnan(wide).all())
