"""Boundary cases of the PointPillars training step (csrc/pillars_train.cu), as numpy arrays for the C ABI
(bevb200_pillar_forward_train / _backward_train) and for the float64 oracle (pillars_train_oracle.train_step).

Every boundary is read from the source text of the constant that sets it, so a retune moves the cases with it:
kPtChunk (rows per double partial), kPtWarps (= kPfnWarps), kPfnMaxP / kPfnMaxF, kNumSMs and the two grid
multipliers of pt_launch (P1-P3 / B1 and B2 / B3).

Margins by construction.  fp32 and float64 must take the same side of every decision the step makes: each ReLU
of a kept row (real rows and the padding row kind A) and each layer-1 / layer-2 max whose value is > 0 (a max of 0
takes no gradient).  For every such quantity q, S(q) is the sum of the magnitudes of every term that enters it (the
decorated inputs with their centres, both linears, the BN mean and the propagated layer-1 magnitudes), and a
builder requires |q| >= delta and max - runner-up >= delta with delta = MARGIN_ULPS * 2^-24 * S(q).  The kernel
evaluates each q with at most 13 + 32 + 64 rounded terms (and a 32-lane mean), so its fp32 error stays below about
110 * 2^-24 * S(q); MARGIN_ULPS = 256 leaves a factor 2 above that.  A draw that misses a margin is redrawn from
the next seed.

Exact ties are built so that fp32 and float64 both see them bit for bit, and are the only ties allowed:
  (a) two real rows of one pillar differ only in one raw column whose W1 weight is 0 in one channel;
  (b) a real row whose only nonzero decorated column has zero W1 weights in every channel (a pillar centred at
      the origin, its cluster mean exactly 0), so it equals the padding row in both layers;
  (c) layer-2 channels whose pre-activation is < 0 on every row, or exactly 0 (gamma = beta = 0).

Large cases (chunk and grid counts, segments) draw K template pillars and give each pillar one of them: all
coordinates are dyadic, so the offsets from the pillar centre and the cluster mean are exact in both precisions,
and with W1's raw x / y columns at 0 every pillar of a template has bit-equal pre-activations.  The margins then
hold for 10^5 pillars as they do for K."""
import math
import os
import re

import numpy as np

from pillars_train_oracle import inside_canvas, slot_values, train_step

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "bevfusion_b200", "csrc")
SOURCES = ("pillars_train.cu", "pillars.cuh", "common.cuh")


def _read(fname):
    with open(os.path.join(CSRC, fname)) as f:
        return f.read()


def cu_int(name):
    """an integer constexpr of the pillar sources, declared alone or in a comma list; names inside resolve too"""
    for fname in SOURCES:
        m = re.search(r"constexpr\s+int\s+(?:[^;]*?[\s,])?%s\s*=\s*([^,;]+)[,;]" % re.escape(name), _read(fname))
        if m:
            expr = re.sub(r"\bk[A-Z]\w*\b", lambda t: str(cu_int(t.group(0))), m.group(1))
            if not re.fullmatch(r"[\d\s()+\-*/]+", expr):
                raise ValueError("%s: not an integer expression: %r" % (name, expr))
            return int(eval(expr.replace("/", "//"), {"__builtins__": {}}))   # noqa: S307  (digits, operators)
    raise KeyError(name)


def _grid_multipliers():
    m = re.search(r"kNumSMs\s*\*\s*\(kPass == kB2 \|\| kPass == kB3 \? (\d+) : (\d+)\)", _read("pillars_train.cu"))
    if m is None:
        raise KeyError("pt_launch grid")
    return int(m.group(1)), int(m.group(2))


CHUNK = cu_int("kPtChunk")
WARPS = cu_int("kPtWarps")
MAX_P, MAX_F = cu_int("kPfnMaxP"), cu_int("kPfnMaxF")
NUM_SMS = cu_int("kNumSMs")
GRID_B23, GRID_P13 = _grid_multipliers()          # chunks per grid: kNumSMs * these (B2 / B3, and P1-P3 / B1)
INT32_MAX = 2 ** 31 - 1
EPS, MOMENTUM = float(np.float32(1e-3)), float(np.float32(0.1))   # as the kernel reads them (float fields)
MARGIN_ULPS = 256
DISTINCT = 4                                      # distinct points per pillar; the others repeat them
U = 2.0 ** -24


class Case:
    """One call of the training step.  Rows [s cap, s cap + clamp(n_dev[s], 0, cap)) are kept; the rest are
    garbage.  ties: (layer, pillar row, slots) exact ties built on purpose; dead: (layer, channel) with gamma = beta
    = 0 (pre-activation exactly 0 everywhere)."""

    def __init__(self, name, voxels, num_points, coords4, n_dev, segments, canvas, geom, params, grad_canvas,
                 ties=(), dead=()):
        self.name, self.voxels, self.num_points, self.coords4 = name, voxels, num_points, coords4
        self.n_dev, self.segments, self.canvas, self.geom = n_dev, segments, canvas, geom
        self.params, self.grad_canvas, self.ties, self.dead = params, grad_canvas, set(ties), set(dead)
        self._gold = None

    R = property(lambda self: self.voxels.shape[0])
    P = property(lambda self: self.voxels.shape[1])
    F = property(lambda self: self.voxels.shape[2])
    cap = property(lambda self: self.R // self.segments)
    canvas_shape = property(lambda self: (self.canvas[0], 64, self.canvas[1], self.canvas[2]))

    def keep(self):
        if self.n_dev is None:
            return np.arange(self.R)
        n = np.clip(np.asarray(self.n_dev, np.int64), 0, self.cap)
        return np.concatenate([np.arange(s * self.cap, s * self.cap + n[s]) for s in range(self.segments)])

    def slots(self):
        """N of the BN statistics: P * kept pillars"""
        return self.P * len(self.keep())

    def gold(self):
        """the float64 step on the kept rows (a dict of train_step)"""
        if self._gold is None:
            k = self.keep()
            self._gold = train_step(self.voxels[k], self.num_points[k], self.coords4[k], self.params, self.geom,
                                    self.canvas_shape, self.grad_canvas, eps=EPS, momentum=MOMENTUM)
        return self._gold


# ---- draws ---------------------------------------------------------------------------------------------------
def _f32(a):
    return np.asarray(a, np.float32).astype(np.float64)


def _dyadic(rng, shape, lim, step=1.0 / 64):
    return rng.integers(-int(lim / step), int(lim / step) + 1, size=shape) * step


def draw_params(rng, F, raw_xy=True):
    """W1 [32, F+5], W2 [64, 64], BN weights (a quarter negative), biases and running statistics, fp32 values"""
    def bn(u):
        return (np.where(rng.random(u) < 0.25, -1.0, 1.0) * (0.5 + rng.random(u)), rng.random(u) - 0.5,
                0.6 * rng.random(u) - 0.3, 0.5 + 1.5 * rng.random(u))
    W1 = rng.standard_normal((32, F + 5)) / math.sqrt(F + 5)
    if not raw_xy:
        W1[:, :2] = 0.0
    p = dict(W1=W1, W2=rng.standard_normal((64, 64)) / 8.0)
    for k, (g, b, rm, rv) in (("1", bn(32)), ("2", bn(64))):
        p.update({"g" + k: g, "b" + k: b, "rm" + k: rm, "rv" + k: rv})
    return {k: _f32(v) for k, v in p.items()}


def geometry(nx, ny):
    """(vx, vy, x_off, y_off): dyadic, vx != vy, and the centre of cell (nx // 2, ny // 2) exactly at the origin"""
    vx, vy = 1.0 / 32, 3.0 / 64
    return (vx, vy, -(nx // 2) * vx, -(ny // 2) * vy)


def pillar_rows(rng, n, P, F, distinct=DISTINCT):
    """[P, F] rows of one pillar relative to its centre: n dyadic points cycling over `distinct` drawn rows (so a
    32-point pillar adds no more decisions than a 4-point one), zero padding"""
    k = min(n, distinct)
    pool = np.zeros((k, F))
    pool[:, 0:2] = _dyadic(rng, (k, 2), 1.0)
    pool[:, 2] = _dyadic(rng, k, 2.0)
    pool[:, 3:] = _dyadic(rng, (k, F - 3), 1.0)
    rows = np.zeros((P, F))
    rows[:n] = pool[np.arange(n) % k]
    return rows


def place(rel, num, coords4, geom):
    """absolute voxels: each pillar's real rows moved to its centre (exact: dyadic values)"""
    vx, vy, xo, yo = geom
    v = rel.copy()
    real = np.arange(rel.shape[1])[None, :] < num[:, None]
    v[:, :, 0] += np.where(real, (coords4[:, 1] * vx + xo)[:, None], 0.0)
    v[:, :, 1] += np.where(real, (coords4[:, 2] * vy + yo)[:, None], 0.0)
    return v


def unique_cells(rng, M, B, nx, ny, avoid=()):
    """M distinct (b, x, y, 0) on the canvas, none in `avoid`"""
    bad = {(b * nx + x) * ny + y for b, x, y in avoid}
    pool = np.setdiff1d(np.arange(B * nx * ny), np.fromiter(bad, np.int64, len(bad)))
    flat = rng.choice(pool, M, replace=False)
    return np.stack([flat // (nx * ny), flat // ny % nx, flat % ny, np.zeros_like(flat)], 1)


def grad_canvas(rng, B, nx, ny):
    return _f32(rng.standard_normal((B, 64, nx, ny)))


def _pillars(rng, nums, P, F, templates=None):
    """(rel rows [M, P, F], num [M]); with templates, pillar i copies template i % K of the same n"""
    nums = np.asarray(nums, np.int64)
    if templates is None:
        return np.stack([pillar_rows(rng, n, P, F) for n in nums]) if len(nums) else np.zeros((0, P, F)), nums
    table = {}
    rel = np.zeros((len(nums), P, F))
    for i, n in enumerate(nums):
        key = (int(n), i % templates)
        if key not in table:
            table[key] = pillar_rows(rng, n, P, F)
        rel[i] = table[key]
    return rel, nums


# ---- margins ---------------------------------------------------------------------------------------------------
def margins(case):
    """-> (worst ReLU ratio, worst max-gap ratio, exact ties found, undeclared ties), ratios = margin / delta over
    every decision of the kept rows; the ties are {(layer, pillar row, slots)} of maxes > 0."""
    k = case.keep()
    x, num, c = case.voxels[k], case.num_points[k], case.coords4[k]
    p, gold, P, F = case.params, case.gold(), case.P, case.F
    h, pre1, y1, m1, pre2 = slot_values(x, num, c, p, case.geom, gold, eps=EPS)
    slot = np.arange(P)[None, :]
    cnt = np.minimum(num, P)[:, None]
    live = slot <= np.minimum(cnt, P - 1)            # real rows and kind A (one padding row stands for all)
    # magnitudes: |decorated| with the mean and the centre added to the columns they are subtracted from
    vx, vy, xo, yo = case.geom
    Mh = np.abs(h)
    mean = np.abs(x[:, :, :3].sum(axis=1) / num[:, None])
    Mh[:, :, F:F + 3] += mean[:, None, :]
    Mh[:, :, F + 3] += np.abs(c[:, 1] * vx + xo)[:, None]
    Mh[:, :, F + 4] += np.abs(c[:, 2] * vy + yo)[:, None]
    Mh *= slot[..., None] < cnt[..., None]
    sc1 = np.abs(p["g1"]) / np.sqrt(gold["var1"] + EPS)
    sc2 = np.abs(p["g2"]) / np.sqrt(gold["var2"] + EPS)
    S1 = sc1 * (Mh @ np.abs(p["W1"]).T + np.abs(gold["mu1"])) + np.abs(p["b1"])
    S1m = np.where(live[..., None], S1, 0).max(axis=1)
    S2 = sc2 * ((y1 + S1) @ np.abs(p["W2"][:, :32]).T + ((m1 + S1m) @ np.abs(p["W2"][:, 32:]).T)[:, None, :]
                + np.abs(gold["mu2"])) + np.abs(p["b2"])
    d1, d2 = MARGIN_ULPS * U * S1, MARGIN_ULPS * U * S2
    relu = []
    for layer, pre, d in ((1, pre1, d1), (2, pre2, d2)):
        with np.errstate(invalid="ignore"):          # 0 / 0 on dead channels, set below
            r = np.abs(pre) / d
        for (l, ch) in case.dead:
            if l == layer:
                assert not pre[..., ch][live].any(), "dead channel %d of layer %d is not exactly 0" % (ch, layer)
                r[..., ch] = np.inf
        relu.append(np.where(live[..., None], r, np.inf).min() if len(k) else np.inf)
    gaps, found = [], set()
    for layer, V, d in ((1, y1, d1), (2, pre2, d2)):
        V = np.where(live[..., None], V, -np.inf)
        D = np.where(live[..., None], d, 0).max(axis=1)
        top = V.max(axis=1) if len(k) else np.zeros((0, V.shape[2]))
        eq = V == top[:, None, :]
        runner = np.where(eq, -np.inf, V).max(axis=1) if len(k) else top
        active = top > 0
        gaps.append(np.where(active, (top - runner) / D, np.inf).min() if len(k) else np.inf)
        for v, ch in zip(*np.nonzero(active & (eq.sum(axis=1) > 1))):
            found.add((layer, int(k[v]), frozenset(np.nonzero(eq[v, :, ch])[0].tolist())))
    # rows with bit-equal decorated inputs tie in both precisions, and either one taking the gradient is the same
    same = {t for t in found if all(np.array_equal(h[np.searchsorted(k, t[1]), s], h[np.searchsorted(k, t[1]), min(t[2])])
                                    and s < num[np.searchsorted(k, t[1])] for s in t[2])}
    undeclared = {t for t in found if t not in case.ties and t not in same}
    return min(relu), min(gaps), found, undeclared


def landed(case, found):
    """every layer a declared tie names has one of them at a max > 0"""
    return all(any(t[0] == layer for t in found & case.ties) for layer in {t[0] for t in case.ties})


def settled(case):
    """the case meets every margin, has no tie it did not declare, and lands on its declared ties"""
    relu, gap, found, undeclared = margins(case)
    return relu >= 1.0 and gap >= 1.0 and not undeclared and landed(case, found)


def _settle(make, seed, tries=200):
    for t in range(tries):
        case = make(np.random.default_rng([seed, t]))
        if settled(case):
            return case
    raise AssertionError("no draw of %r meets its margins in %d tries" % (make, tries))


# ---- builders --------------------------------------------------------------------------------------------------
def _assemble(name, rng, rel, num, coords4, canvas, params, n_dev=None, segments=1, ties=(), dead=()):
    geom = geometry(canvas[1], canvas[2])
    vox = place(rel, num, coords4, geom)
    return Case(name, vox, num.astype(np.int32), coords4.astype(np.int32), n_dev, segments, canvas, geom, params,
                grad_canvas(rng, *canvas), ties, dead)


def pad_kinds(P):
    """pads P - n with n >= 1: 0 (no padding row), 1 (kind A only), 2 (kind B once), and > 2 (n = 1, and a middle
    one), as far as P allows"""
    pads = {0, 1, 2, P - 1, P // 2 + 1}
    return sorted(q for q in pads if 0 <= q <= P - 1)


def pf_case(P, F, seed=0, per_kind=2):
    """P x F: per_kind pillars at every pad kind P allows, on a 2 x 9 x 7 canvas"""
    kinds = pad_kinds(P)
    per_kind = max(per_kind, -(-6 // len(kinds)))

    def make(rng):
        nums = np.repeat([P - q for q in kinds], per_kind)
        rel, num = _pillars(rng, nums, P, F)
        canvas = (2, 9, 7)
        return _assemble("P%d F%d" % (P, F), rng, rel, num, unique_cells(rng, len(num), *canvas), canvas,
                         draw_params(rng, F))
    return _settle(make, seed)


FEW_ROWS = {"N1": (1, [1]), "N2-P1": (1, [1, 1]), "N2-P2": (2, [1])}   # name: (P, n of each pillar)


def few_rows_case(name, seed=0):
    P, nums = FEW_ROWS[name]

    def make(rng):
        rel, num = _pillars(rng, nums, P, 4)
        canvas = (1, 5, 6)
        return _assemble(name, rng, rel, num, unique_cells(rng, len(num), *canvas), canvas, draw_params(rng, 4))
    if P * len(nums) < 2:                            # nothing is computed: no margins to meet
        return make(np.random.default_rng(seed))
    return _settle(make, seed)


def _template_case(name, R, P, F, canvas, seed, K=4, segments=1, n_dev=None, tries=50):
    """R rows, row i a copy of template pillar i % (K P) (template t holds 1 + t % P points), moved to its own
    cell.  Rows not kept get NaN voxels, garbage counts and garbage coordinates (some on the canvas).  A draw is
    first settled on its K P templates alone when R is large (the same statistics up to each template's
    frequency), then checked at full size."""
    T = K * P
    for t in range(tries):
        rng = np.random.default_rng([seed, t])
        num = 1 + np.arange(T) % P
        rel, _ = _pillars(rng, num, P, F)
        params = draw_params(rng, F, raw_xy=False)
        if R > 4096 and not settled(_assemble(name, rng, rel, num, unique_cells(rng, T, *canvas), canvas, params)):
            continue
        idx = np.arange(R) % T
        case = _assemble(name, rng, rel[idx], num[idx], unique_cells(rng, R, *canvas), canvas, params,
                         n_dev=n_dev, segments=segments)
        drop = np.setdiff1d(np.arange(R), case.keep())
        case.voxels[drop] = np.nan
        case.num_points[drop] = rng.choice([-3, 0, 7, 1000, INT32_MAX], len(drop))
        case.coords4[drop] = rng.choice([-5, 0, 1, 3, 100000, INT32_MAX], (len(drop), 4))
        if settled(case):
            return case
    raise AssertionError("no draw of %s meets its margins in %d tries" % (name, tries))


def chunk_rows():
    """R at k * kPtChunk + {-1, 0, 1}, k = 1, 2"""
    return [k * CHUNK + d for k in (1, 2) for d in (-1, 0, 1)]


def grid_chunks():
    """chunk counts at the grid strides: kNumSMs * (B2/B3 multiplier, P1-P3/B1 multiplier) + {-1, 0, 1}"""
    return [NUM_SMS * m + d for m in (GRID_B23, GRID_P13) for d in (-1, 0, 1)]


def rows_case(R, seed=0, P=2, F=3):
    """R rows (the last chunk partial unless R is a multiple of kPtChunk), small P and F"""
    side = math.isqrt(max(R // 2, 1)) + 1
    return _template_case("R=%d (%d chunks)" % (R, -(-R // CHUNK)), R, P, F, (2, side, side + 1), seed)


def grid_case(chunks, seed=0):
    """chunks partials, the last one half full; one point per pillar keeps the float64 twin small"""
    return rows_case(chunks * CHUNK - CHUNK // 2, seed, P=1)


SEGMENTS = {                                          # name: (segments, cap, n_dev or None)
    "S1 null": (1, 40, None),
    "S1 INT32_MAX": (1, 40, [INT32_MAX]),
    "S3 cap+1 -1 mid": (3, 40, [41, -1, 17]),
    "S3 null": (3, 20, None),
    "S64 every count": (64, 4, [[-1, 0, 1, 4, 5, INT32_MAX, 2, 3][i % 8] for i in range(64)]),
}


def segment_case(name, seed=0):
    S, cap, n_dev = SEGMENTS[name]
    return _template_case(name, S * cap, 3, 4, (2, 17, 19), seed, segments=S,
                          n_dev=None if n_dev is None else np.asarray(n_dev, np.int64))


def canvas_case(nx, ny, seed=0, inner=12):
    """B = 2, nx x ny: pillars on the last batch / row / column and the corners, and pillars just off the canvas
    (x = nx, y = ny, y = -1, x = -1, b = B): those count in both BNs but write and receive nothing"""
    B = 2
    edge = [(B - 1, nx - 1, ny - 1), (0, 0, 0), (B - 1, 0, ny - 1), (0, nx - 1, 0), (B - 1, nx // 2, ny - 1)]
    off = [(0, nx, 3), (1, 2, ny), (0, 4, -1), (1, -1, 5), (B, 1, 1)]

    def make(rng):
        cells = np.concatenate([np.array([(*e, 0) for e in edge + off]),
                                unique_cells(rng, inner, B, nx, ny, avoid=edge)])
        nums = 1 + rng.integers(0, 4, len(cells))
        rel, num = _pillars(rng, nums, 4, 5)
        return _assemble("canvas %dx%d" % (nx, ny), rng, rel, num, cells, (B, nx, ny), draw_params(rng, 5))
    case = _settle(make, seed)
    ins = inside_canvas(case.coords4, case.canvas_shape)
    assert ins.sum() == len(ins) - len(off)
    return case


def tie_case(kind, seed=0):
    """(a) layer-1 tie of two real rows, (b) a real row tied with the padding row in both layers, (c) dead layer-2
    channels; 10 other random pillars around them (P = 6, F = 5)"""
    P, F, canvas, j = 6, 5, (2, 9, 11), 3

    def make(rng):
        nums = 1 + rng.integers(0, P, 10)
        p = draw_params(rng, F)
        ties, dead = [], []
        if kind == "a":                               # rows 1 and 3 of three pillars differ only in column j
            special = [4, 5, 6]
            p["W1"][0, j] = 0.0                       # channel 0 ignores it
            rel, num = _pillars(rng, np.concatenate([special, nums]), P, F)
            for i in range(len(special)):
                rel[i, 3] = rel[i, 1]
                rel[i, 1, j], rel[i, 3, j] = 1.0, -1.0
                ties.append((1, i, frozenset({1, 3})))
            cells = unique_cells(rng, len(num), *canvas)
        elif kind == "b":                             # row 1 of pillar 0 at the origin, centred cell, mean 0
            p["W1"][:, j] = 0.0
            p["b1"][::2] += 1.0                       # the padding row wins layer 1 on half the channels
            rel, num = _pillars(rng, np.concatenate([[3], nums]), P, F)
            rel[0, 1] = 0.0
            rel[0, 1, j] = 1.5
            rel[0, 2, :3] = -rel[0, 0, :3]
            cells = np.concatenate([[[0, canvas[1] // 2, canvas[2] // 2, 0]],
                                    unique_cells(rng, len(nums), *canvas, avoid=[(0, canvas[1] // 2, canvas[2] // 2)])])
            ties = [(1, 0, frozenset({1, 3})), (2, 0, frozenset({1, 3}))]
        else:                                         # channels 5, 40 below 0 everywhere; 17 exactly 0
            rel, num = _pillars(rng, nums, P, F)
            p["b2"][[5, 40]] -= 20.0
            p["g2"][17] = p["b2"][17] = 0.0
            dead = [(2, 17)]
            cells = unique_cells(rng, len(num), *canvas)
        return _assemble("tie %s" % kind, rng, rel, num, cells, canvas, p, ties=ties, dead=dead)

    return _settle(make, seed)
