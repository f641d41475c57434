"""Boundary cases of the detection-head kernels, derived from the kernels' own tiling and limit constants, and a
guard that carves every device allocation of a call out of a canary-filled buffer.

Every constant is read from the source that defines it (the C header's #defines, the kernels' constexprs), so a
retune of a tile, a block or a limit moves the cases with it:

    header_macro(name)          an integer #define of include/bevfusion_b200.h
    cu_const(file, name)        an integer constexpr of bevfusion_b200/csrc/<file>

Case builders (numpy, no device):

    factor_map(n, ...)          (C, H, W) with C * H * W == n: maps whose element count sits on a tile edge
    slot_case(M, ...)           CenterHead inds / masks whose duplicates straddle the slot passes of the backward
    tie_kinds(...)              hi / tie / lo cells for a threshold bin of an exact size in the top-K select
    grid_geometry(...)          BEVGridTransform scopes whose row block is forced to one row, or whose shared memory
                                is exactly the limit

DeviceGuard patches the `torch` of the wrapper modules for the duration of a block: every CUDA tensor they allocate
(outputs, gradients, workspaces of exactly the queried size) is placed GUARD bytes into a buffer GUARD bytes longer
on both sides, the whole buffer filled with a byte pattern, and check() verifies that no byte outside the tensors
changed."""
import math
import os
import re

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")
CSRC = os.path.join(ROOT, "bevfusion_b200", "csrc")
HEADER = os.path.join(ROOT, "include", "bevfusion_b200.h")


def _read(path):
    with open(path) as f:
        return f.read()


def _eval(expr, fname):
    def sub(m):
        tok = m.group(0)
        return str(header_macro(tok) if tok.startswith("BEVB200_") else cu_const(fname, tok))
    expr = re.sub(r"\b(BEVB200_\w+|k[A-Z]\w*)\b", sub, expr.strip())
    if not re.fullmatch(r"[\d\s()+\-*/<]+", expr):
        raise ValueError("not an integer constant expression: %r" % expr)
    return int(eval(expr.replace("/", "//"), {"__builtins__": {}}))   # noqa: S307  (digits and operators only)


def header_macro(name):
    m = re.search(r"^#define\s+%s\s+([^/\n]+)" % re.escape(name), _read(HEADER), re.M)
    if m is None:
        raise KeyError(name)
    return _eval(m.group(1), None)


def cu_const(fname, name):
    m = re.search(r"constexpr\s+(?:int|size_t)\s+%s\s*=\s*([^;]+);" % re.escape(name), _read(os.path.join(CSRC, fname)))
    if m is None:
        raise KeyError("%s in %s" % (name, fname))
    return _eval(m.group(1), fname)


# ---- the constants ----------------------------------------------------------------------------------------------
LOSS_TILE = cu_const("head_losses.cu", "kTile")                 # elements per CTA of a dense loss term
SLOT_THREADS = cu_const("head_losses.cu", "kSlotThreads")       # slots per compaction pass of the CenterHead backward
LOSS_MAX_TASKS = header_macro("BEVB200_LOSS_MAX_TASKS")
LOSS_MAX_OBJS = header_macro("BEVB200_LOSS_MAX_OBJS")
LOSS_MAX_LAYERS = header_macro("BEVB200_LOSS_MAX_LAYERS")
TOPK_TILE = cu_const("topk_select.cuh", "kTile")                # cells per candidate tile
BUF_CAP = cu_const("topk_select.cuh", "kBufCap")                # keys of the threshold bin held in shared memory
PROPOSALS_MAX_K = header_macro("BEVB200_PROPOSALS_MAX_K")
DECODE_MAX_K = header_macro("BEVB200_DECODE_MAX_K")
WIDE_COLUMNS = cu_const("transfusion_assign.cu", "kWideColumns")   # above: 8 warps per LSAP segment, else one
ASSIGN_MAX = header_macro("BEVB200_ASSIGN_MAX")
ASSIGN_THREADS = cu_const("head_targets.cu", "kAssignThreads")   # box stride of the head-target assign kernel
TARGETS_MAX_BOXES = header_macro("BEVB200_HEAD_TARGETS_MAX_BOXES")
TARGETS_MAX_TASKS = header_macro("BEVB200_HEAD_TARGETS_MAX_TASKS")
SEG_LOSS_TILE = cu_const("map_seg.cu", "kLossTile")
SEG_COUNT_TILE = cu_const("map_seg.cu", "kCountTile")
GRID_SMEM_LIMIT = cu_const("map_seg.cu", "kGridSmemLimit")
GRID_ROWS = (16, 8, 4, 2, 1)                                    # BEVGridTransform's rows-per-block candidates


# ---- map shapes -------------------------------------------------------------------------------------------------
def _pairs(n, min_side):
    """(H, W) with H * W == n and both >= min_side, the squarest first."""
    out = []
    for h in range(max(min_side, 1), int(math.isqrt(n)) + 1):
        if n % h == 0 and n // h >= min_side:
            out.append((h, n // h))
    return sorted(out, key=lambda p: p[1] - p[0])


def factor_map(n, min_side=1, max_c=64, want_c=None):
    """(C, H, W) with C * H * W == n, H and W >= min_side, C <= max_c (want_c first if it divides); None if none."""
    cs = ([want_c] if want_c else []) + list(range(1, max_c + 1))
    for c in cs:
        if c and n % c == 0 and c <= max_c:
            hw = _pairs(n // c, min_side)
            if hw:
                return (c,) + hw[0]
    return None


def tile_edges(tile, ks=(1, 3), extra=(1,)):
    """Element counts on the edges of `tile`: k * tile - 1, k * tile, k * tile + 1 for each k, and `extra`."""
    return sorted(set(list(extra) + [k * tile + d for k in ks for d in (-1, 0, 1)]))


# ---- CenterHead slots -------------------------------------------------------------------------------------------
SHARED_CELL = 17


def slot_case(M, B, HW, seed):
    """inds / masks [3 tasks][B, M] for the slot passes of SLOT_THREADS slots:
    task 0 -- sample 0 every slot masked in, sample 1 every slot masked out;
    task 1 -- masks with gaps (every 7th slot, a quarter-pass run) and duplicate cells whose first slot is in one
              pass and whose later slots are in the next ones: cell SHARED_CELL at slots 0, S - 1, S and M - 1;
    task 2 -- half the slots masked in, all of them on 8 cells."""
    S = SLOT_THREADS
    rng = np.random.default_rng(seed)
    inds, masks = [], []
    ind = rng.integers(0, HW, (B, M))
    mask = np.ones((B, M), np.uint8)
    mask[1:] = 0
    inds.append(ind)
    masks.append(mask)
    ind = rng.integers(0, HW, (B, M))
    mask = np.ones((B, M), np.uint8)
    mask[:, 3::7] = 0
    for m in range(5, M - S, 37):                  # a cell first at slot m and again one pass later
        ind[:, m + S] = ind[:, m]
        mask[:, [m, m + S]] = 1
    mask[:, S // 2:S // 2 + S // 4] = 0
    shared = [m for m in sorted({0, S - 1, S, M - 1}) if m < M]
    ind[:, shared] = SHARED_CELL
    mask[:, shared] = 1
    inds.append(ind)
    masks.append(mask)
    inds.append(rng.integers(0, 8, (B, M)))
    masks.append((rng.random((B, M)) < 0.5).astype(np.uint8))
    return inds, masks


# ---- top-K threshold bins ---------------------------------------------------------------------------------------
HI, TIE, LO = 0, 1, 2


def order_key_top_byte(v):
    """Top byte of topk_select.cuh's order-preserving key of fp32 values (NaN excluded)."""
    u = np.asarray(v, np.float32).view(np.uint32).astype(np.uint64)
    k = np.where(u & 0x80000000, ~u & 0xffffffff, u | 0x80000000)
    return (k >> 24).astype(np.int64)


def tie_kinds(cells, n_hi, n_tie, seed):
    """A random arrangement of n_hi HI, n_tie TIE and the rest LO over `cells` cells, the tied cells spread over every
    tile of the plane."""
    assert n_hi + n_tie <= cells
    kinds = np.full(cells, LO, np.int64)
    kinds[:n_hi] = HI
    kinds[n_hi:n_hi + n_tie] = TIE
    return np.random.default_rng(seed).permutation(kinds)


def tie_side(n_hi, n_tie, planes):
    """The side of a square map whose `planes` planes hold n_hi + n_tie cells and at least as many LO cells as HI."""
    return int(math.isqrt((n_tie + 2 * n_hi) // planes)) + 2


TIE_COUNTS = {"cap-1": BUF_CAP - 1, "cap": BUF_CAP, "cap+1": BUF_CAP + 1, "8cap": 8 * BUF_CAP}


# ---- grid transform geometry --------------------------------------------------------------------------------------
GRID_IN_ROWS = 32                                # a power of two: the row taps are exact, two per row


def grid_geometry(smem_bytes, direction, target_R, exact):
    """BEVGridTransform scopes of a GRID_IN_ROWS x W map to GRID_IN_ROWS x Wd whose `direction` ("fwd" or "bwd")
    picks target_R rows per block -- with exactly GRID_SMEM_LIMIT bytes of shared memory when `exact` -- every
    larger candidate over the limit, while the other direction fits.  The rows map to themselves; output column j
    sits a quarter cell right of input column j (two taps while both are inside).  smem_bytes:
    bevb200_map_grid_smem_bytes.  Returns (input_scope, output_scope, H, W, smem) for the narrowest such W, or
    None."""
    from bevfusion_b200 import map_seg as MS
    H = GRID_IN_ROWS
    isc_r = osc_r = [-H / 2, H / 2, 1.0]
    ry = MS.axis_taps(MS.axis_coords(isc_r, osc_r), H)
    n_f = {R: int(MS._blocks(ry, R)[1].max()) for R in GRID_ROWS}
    n_b = {R: int(MS._blocks(MS.transpose_taps(ry, H), R)[1].max()) for R in GRID_ROWS}
    n = (n_f if direction == "fwd" else n_b)[target_R]
    # smem < (20 + 8 n) max(W, Wd) + 32: nothing narrower reaches the limit
    for W in range(max((GRID_SMEM_LIMIT - 32) // (20 + 8 * n) - 64, 9), GRID_SMEM_LIMIT // (4 * n) + 2):
        for Wd in range(max(W - 64, 1), W + 65):
            nnz = 2 * Wd if Wd < W else 2 * W - 1
            fwd = [int(smem_bytes(W, Wd, nnz, n_f[R])) for R in GRID_ROWS]
            bwd = [int(smem_bytes(Wd, W, nnz, n_b[R])) for R in GRID_ROWS]
            mine, other = (fwd, bwd) if direction == "fwd" else (bwd, fwd)
            fits = [v <= GRID_SMEM_LIMIT for v in mine]
            if True not in fits or GRID_ROWS[fits.index(True)] != target_R or min(other) > GRID_SMEM_LIMIT:
                continue
            if exact and mine[fits.index(True)] != GRID_SMEM_LIMIT:
                continue
            geom = [isc_r, [-W / 2, W / 2, 1.0]], [osc_r, [-W / 2 + 0.25, -W / 2 + 0.25 + Wd, 1.0]]
            plans = [grid_plan_rows(smem_bytes, *geom, H, W, back) for back in (False, True)]
            R, got = plans[direction == "bwd"]
            if R == target_R and None not in plans[direction == "fwd"] and (not exact or got == GRID_SMEM_LIMIT):
                return geom[0], geom[1], H, W, got
    return None


def grid_plan_rows(smem_bytes, input_scope, output_scope, H, W, backward=False):
    """(rows per block, shared bytes) BEVGridTransform's forward or backward direction picks for these scopes, from
    the module's own tap tables (host only); (None, None) when nothing fits."""
    from bevfusion_b200 import map_seg as MS
    ry = MS.axis_taps(MS.axis_coords(input_scope[0], output_scope[0]), H)
    rx = MS.axis_taps(MS.axis_coords(input_scope[1], output_scope[1]), W)
    nnz = sum(len(t) for t in rx)
    src_w, dst_w = W, len(rx)
    if backward:
        ry, src_w, dst_w = MS.transpose_taps(ry, H), len(rx), W
    for R in GRID_ROWS:
        s = int(smem_bytes(src_w, dst_w, nnz, int(MS._blocks(ry, R)[1].max())))
        if s <= GRID_SMEM_LIMIT:
            return R, s
    return None, None


# ---- guarded allocations ------------------------------------------------------------------------------------------
GUARD = 4096


def pattern(n, device):
    return ((torch.arange(n, device=device) * 7 + 3) % 256).to(torch.uint8)


class DeviceGuard:
    """with DeviceGuard(module, ...) as g: ... g.check() -- see the module docstring."""

    _ALLOC = ("empty", "empty_like", "zeros", "zeros_like", "ones", "full", "full_like")

    def __init__(self, *modules):
        self.modules = modules
        self.blocks = []        # (buffer, first byte of the tensor, end byte of the tensor)
        self._saved = []

    def carve(self, real, fill):
        """A tensor shaped and typed as `real`, GUARD bytes into a canary-filled buffer (its contents `real`'s when
        fill, the canary otherwise)."""
        nbytes = real.numel() * real.element_size()
        buf = pattern(GUARD + nbytes + GUARD, real.device)
        t = torch.empty((0,), dtype=real.dtype, device=real.device)
        stride, acc = [], 1
        for s in reversed(real.shape):
            stride.insert(0, acc)
            acc *= s
        t.set_(buf.untyped_storage(), GUARD // real.element_size(), tuple(real.shape), tuple(stride))
        if fill:
            t.copy_(real)
        self.blocks.append((buf, GUARD, GUARD + nbytes))
        return t

    def _proxy(self):
        guard = self

        class _Torch:
            def __getattr__(self, name):
                fn = getattr(torch, name)
                if name not in DeviceGuard._ALLOC:
                    return fn

                def alloc(*args, **kwargs):
                    real = fn(*args, **kwargs)
                    if not real.is_cuda or real.layout != torch.strided:
                        return real
                    return guard.carve(real, fill=not name.startswith("empty"))
                return alloc
        return _Torch()

    def __enter__(self):
        proxy = self._proxy()
        for m in self.modules:
            self._saved.append((m, m.torch))
            m.torch = proxy
        return self

    def __exit__(self, *exc):
        for m, t in reversed(self._saved):
            m.torch = t
        self._saved = []
        return False

    def check(self, what=""):
        """Every byte before and after every carved tensor still holds the canary."""
        if any(b.is_cuda for b, _, _ in self.blocks):
            torch.cuda.synchronize()
        for i, (buf, lo, hi) in enumerate(self.blocks):
            want = pattern(buf.numel(), buf.device)
            for a, b in ((0, lo), (hi, buf.numel())):
                bad = torch.nonzero(buf[a:b] != want[a:b])
                assert bad.numel() == 0, "%s: allocation %d (%d bytes): %d bytes written outside it, first at byte " \
                    "%d of the tensor" % (what, i, hi - lo, bad.numel(), int(bad[0]) + a - lo)
        return len(self.blocks)
