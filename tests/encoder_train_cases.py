"""Boundary cases of the native SparseEncoder training step (csrc/encoder.cu, spconv_wgrad_tc.cu), derived from the
kernels' own chunk constants, and coordinate builders that put every level's row count exactly where a case asks.

    STAT_ROWS   kStatRows of encoder.cu: rows per partial of the BN sums (forward statistics and backward)
    WGT_ROWS    kWgtRows of spconv_wgrad_tc.cu: rows per tile of the filter gradient

Both are read from the source (head_boundaries.cu_const), so a retune moves the cases with it.

Coordinate builders (numpy, no device), each returning (coors [n, 4] int32 (b, x, y, z), rows per level):

    lattice_coors   n voxels on the lattice of spacing 2**levels.  A k3 s2 p1 (or k2 s2 p0) conv maps the input
                    site 2a to the output site a only, so each strided conv keeps every voxel in its own output
                    cell: every level holds exactly n rows.
    block_coors     the 8 voxels of one 2x2x2 block (plus optional lattice voxels elsewhere): a k2 s2 p0 conv maps
                    the whole block to one shared output cell.

Chains are lists of the conv(...) dicts of test_encoder_plan_gpu.py (one BatchNorm per conv in training)."""
import numpy as np

from head_boundaries import cu_const
from test_encoder_plan_gpu import RAW_CHAINS, conv

STAT_ROWS = cu_const("encoder.cu", "kStatRows")
WGT_ROWS = cu_const("spconv_wgrad_tc.cu", "kWgtRows")


def n_strided(convs):
    return sum(1 for c in convs if not c["subm"])


def level_shapes(shape, convs):
    """[level 0 shape, then the output shape of every strided conv] (ops.py:20-31)"""
    out = [list(shape)]
    for c in convs:
        if not c["subm"]:
            out.append([(out[-1][d] + 2 * c["pad"][d] - (c["ks"][d] - 1) - 1) // c["stride"][d] + 1 for d in range(3)])
    return out


def lattice_coors(shape, B, n, levels, seed, samples=None):
    """n distinct voxels of the given samples (default: all B) at coordinates that are multiples of 2**levels,
    shuffled -> (coors, [n] * (levels + 1))."""
    s = 2 ** levels
    X, Y, Z = [(v + s - 1) // s for v in shape]
    samples = list(range(B)) if samples is None else list(samples)
    sites = len(samples) * X * Y * Z
    assert n <= sites, "the lattice holds %d sites, %d asked" % (sites, n)
    rng = np.random.default_rng(seed)
    flat = rng.choice(sites, size=n, replace=False)
    z = flat % Z; y = (flat // Z) % Y; x = (flat // (Z * Y)) % X; b = np.asarray(samples)[flat // (Z * Y * X)]
    return np.stack([b, s * x, s * y, s * z], 1).astype(np.int32), [n] * (levels + 1)


def block_coors(shape, b=0, origin=(2, 2, 2), extra=0, seed=0):
    """the 8 voxels of the 2x2x2 block at `origin` (even) of sample b, then `extra` voxels of the spacing-2 lattice
    in other samples -> (coors, [8 + extra, 1 + extra]) for one k2 s2 p0 conv."""
    ox, oy, oz = origin
    assert ox % 2 == oy % 2 == oz % 2 == 0 and ox + 1 < shape[0] and oy + 1 < shape[1] and oz + 1 < shape[2]
    blk = np.array([[b, ox + i, oy + j, oz + k] for i in (0, 1) for j in (0, 1) for k in (0, 1)], np.int32)
    if extra:
        more, _ = lattice_coors(shape, b + 2, extra, 1, seed, samples=[b + 1])
        blk = np.concatenate([blk, more])
    return blk, [8 + extra, 1 + extra]


# ---- chains ----------------------------------------------------------------------------------------------------
# the strided raw chains of the eval-mode tests, now trained
TRAIN_RAW = {k: RAW_CHAINS[k] for k in ("residual-previous", "residual-two-back", "residual-on-last", "strided-first")}
TRAIN_RAW.update({
    # a SparseBasicBlock on every level of a two-strided-conv chain
    "residual-every-level": (5, [conv(5, 16), conv(16, 16), conv(16, 16, res=0), conv(16, 32, subm=False),
                                 conv(32, 32), conv(32, 32, res=3), conv(32, 64, subm=False), conv(64, 64),
                                 conv(64, 64, res=6)]),
    # c_out 16 on level 1 (strided and SubM): the 16-channel gradient image off level 0
    "strided-c16": (5, [conv(5, 16), conv(16, 16, subm=False), conv(16, 16), conv(16, 32, subm=False)]),
    # a 128-channel SubM, with no ReLU on the strided conv before it
    "subm-128": (5, [conv(5, 16), conv(16, 128, subm=False, relu=False), conv(128, 128)]),
    # first-conv widths: 7 (split to 16, widened to 32 for the filter gradient), 20 (32, no widen), 40 (64)
    "in-7": (7, [conv(7, 16, relu=False), conv(16, 32, subm=False), conv(32, 32)]),
    "in-20": (20, [conv(20, 32), conv(32, 32, subm=False), conv(32, 16, relu=False)]),
    "in-40": (40, [conv(40, 64), conv(64, 32, subm=False), conv(32, 32, res=1)]),
})


def stat_chain(c):
    """two strided convs of c channels (16: also a 16-channel SubM on level 1) on 4 input channels"""
    if c == 16:
        return 4, [conv(4, 16), conv(16, 16, subm=False), conv(16, 16), conv(16, 16, subm=False)]
    return 4, [conv(4, c), conv(c, c, subm=False), conv(c, c, subm=False, relu=False)]


# level 0 holds the 8 voxels of one block, level 1 the one cell they share
ONE_ROW_CHAIN = (5, [conv(5, 16), conv(16, 16, res=0), conv(16, 32, subm=False, ks=2, pad=0), conv(32, 32),
                     conv(32, 32, res=2)])

# one strided level for the filter-gradient tiles and the last-level-of-2 case
TILE_CHAIN = (6, [conv(6, 32), conv(32, 64, subm=False), conv(64, 64)])


def stat_counts():
    """k * STAT_ROWS - 1, k * STAT_ROWS, k * STAT_ROWS + 1 for k = 1, 2"""
    return [k * STAT_ROWS + d for k in (1, 2) for d in (-1, 0, 1)]


def tile_counts():
    """WGT_ROWS * m +- 1 and WGT_ROWS * m for m = 1, 3"""
    return [m * WGT_ROWS + d for m in (1, 3) for d in (-1, 0, 1)]


def stat_case(c, n, seed=0):
    """(in_channels, convs, shape, B, coors, rows): n rows on every one of three levels"""
    cin, convs = stat_chain(c)
    shape, B = [80, 76, 41], 2
    coors, rows = lattice_coors(shape, B, n, n_strided(convs), seed)
    return cin, convs, shape, B, coors, rows
