"""Edge cases of the SparseEncoder's INT8 plan (spconv_v6_forward_i8, include/bevfusion_b200.h, DESIGN.md 4.25), shared
by test_encoder_int8_edges_cpu.py (each case reaches its edge: an oracle stat > 0) and test_encoder_int8_edges_gpu.py
(dense() bit-equal to the oracle).

The dispatch constants are read from the source (head_boundaries.cu_const), so a retune moves the cases with it:

    WG_MIN_KBLOCKS  kWgMinKBlocks: Cout >= 64 with at least this many 32-unit K blocks takes spconv_wg_kernel
    V6_TILE_M       kV6TileM: rows per tile of spconv_v6_kernel (grid min(tiles, 2 kNumSMs))
    WG_TILE_M       WgShape::kTileM = 2 * 64 * kMT: rows per tile of spconv_wg_kernel (grid min(tiles, kNumSMs))

CASES maps a name to (edges, build): build(dev) -> (RawI8, rows per level or None); edges are (stat, conv indices,
minimum) of the oracle stats (encoder_int8_oracle.STAT_KEYS), the first the one the case is named for -- the CPU twin
asserts that each stat, summed over its convs, reaches its minimum.  TILE_CASES are the persistent-tile cases, whose
edge (a CTA that runs a second tile) follows from the row counts alone."""
import numpy as np
import torch

from encoder_train_cases import lattice_coors, n_strided
from head_boundaries import cu_const
from test_encoder_int8_gpu import INT8_RAW, RawI8, _grid
from test_encoder_plan_gpu import conv

WG_MIN_KBLOCKS = cu_const("spconv_v6.cu", "kWgMinKBlocks")
V6_TILE_M = cu_const("spconv_v6.cu", "kV6TileM")
NUM_SMS = cu_const("common.cuh", "kNumSMs")
WG_TILE_M = 2 * 64 * cu_const("spconv_v6.cu", "kMT")
V6_GRID, WG_GRID = 2 * NUM_SMS, NUM_SMS
T_MMA, T_WG = V6_GRID * V6_TILE_M, WG_GRID * WG_TILE_M      # rows past which some CTA runs a second tile

# the twelve INT8 instances: (mode, kernel, Cout); mode 5 is the chain's first conv (fp16 rows), mode 4 the others
INSTANCES = ({(m, "mma", c) for m in (4, 5) for c in (16, 32, 64, 128)}
             | {(m, "wg", c) for m in (4, 5) for c in (64, 128)})


def cin_eff(c_in):
    return next(e for e in (16, 32, 64, 128) if c_in <= e)


def int8_instance(conv_index, c_in, c_out, kvol):
    """(mode, kernel, Cout) that spconv_v6_forward_i8 launches: wgmma at Cout >= 64 and >= kWgMinKBlocks K blocks of
    32 four-byte units of the padded input channels (the BF16x3 rule, whatever the row width)"""
    nkb = (kvol * cin_eff(c_in) + 31) // 32
    return (5 if conv_index == 0 else 4, "wg" if c_out >= 64 and nkb >= WG_MIN_KBLOCKS else "mma", c_out)


def chain_instances(convs):
    return [int8_instance(i, c["cin"], c["cout"], int(np.prod(c["ks"]))) for i, c in enumerate(convs)]


def tiles_per_cta(n_rows, kernel):
    """most tiles one CTA of a persistent kernel runs at n_rows output rows"""
    tm, grid = (V6_TILE_M, V6_GRID) if kernel == "mma" else (WG_TILE_M, WG_GRID)
    tiles = -(-n_rows // tm)
    return -(-tiles // min(tiles, grid)) if tiles else 0


def k113(cin, cout):
    return dict(conv(cin, cout), ks=[1, 1, 3], pad=[0, 0, 1])


SHAPE, B = [40, 36, 20], 2


def _lattice(convs, n=700, seed=3):
    return lattice_coors(SHAPE, B, n, n_strided(convs), seed=seed)


def _raw(dev, cin, convs, seed=4, **kw):
    """the chain on 700 lattice voxels of each of B samples (every level holds 700 rows)"""
    coors, rows = _lattice(convs)
    return RawI8(dev, cin, SHAPE, B, convs, coors, seed=seed, **kw), rows


# ---- a. the instances no other INT8 test launches ----------------------------------------------------------------
INSTANCE_CHAINS = {
    "inst-5-64": (5, [conv(5, 64), k113(64, 64), conv(64, 32)]),           # mode 5 mma 64, mode 4 mma 64 (k(1,1,3))
    "inst-5-128": (5, [conv(5, 128), conv(128, 16)]),                      # mode 5 mma 128
    "inst-40-128": (40, [conv(40, 128), conv(128, 64), conv(64, 32, subm=False)]),   # mode 5 wgmma 128
    "inst-16-64": (5, [conv(5, 16), conv(16, 64), conv(64, 128, subm=False)]),       # mode 4 mma 64 (16 -> 64 k3)
    "inst-16-128": (5, [conv(5, 16), conv(16, 128), conv(128, 32)]),
}


def _instance_case(name):
    cin, convs = INSTANCE_CHAINS[name]
    return [("rows", [i], 1) for i in range(len(convs))], lambda dev: _raw(dev, cin, convs)


# ---- b. saturation ---------------------------------------------------------------------------------------------
SAT_CHAIN = INT8_RAW["in-40"]                  # mode 5 wgmma 64, a strided conv, a residual


def _sat_quarter(dev):
    raw, rows = _raw(dev, *SAT_CHAIN)
    raw.s_act = [s / 4 for s in raw.s_act]
    return raw, rows


def _sat_other_seed(dev):
    """the scales of the same chain on another seed's features and weights, as a deployed plan calibrated on other
    data runs"""
    cin, convs = INT8_RAW["residual-every-level"]
    other, _ = _raw(None, cin, convs, seed=31)
    return _raw(dev, cin, convs, seed=32, s_act=other.s_act)


TINY_CHAIN = (5, [conv(5, 32), conv(32, 32), conv(32, 16)])


def _sat_scale(s_out, shift=None):
    def build(dev):
        cin, convs = TINY_CHAIN
        base, rows = _raw(None, cin, convs, seed=5)
        s_act = list(base.s_act)
        s_act[1] = s_out
        return _raw(dev, cin, convs, seed=5, s_act=s_act, shifts=shift)
    return build


# ---- c. rounding ties ------------------------------------------------------------------------------------------
TIE_CHAIN = (5, [conv(5, 32, scale=False), conv(32, 32, scale=False), conv(32, 64, scale=False),
                 conv(64, 64, scale=False, res=2)])


def _tie_weights(g, kv, cin, cout, zero_col=None):
    """W = m 2^-8, m mostly small and odd (W / s_w = m / 2: a tie), one entry 254 per column: max |W| = 127 2^-7,
    so s_w = 2^-7 exactly"""
    m = torch.randint(-15, 16, (kv, cin, cout), generator=g) * 2 + 1
    m = torch.where(torch.rand(kv, cin, cout, generator=g) < 0.7, torch.zeros_like(m), m)
    k = torch.randint(0, kv * cin, (cout,), generator=g)
    m.view(-1, cout)[k, torch.arange(cout)] = 254 * torch.where(torch.rand(cout, generator=g) < 0.5, 1, -1)
    if zero_col is not None:
        m[:, :, zero_col] = 0
    return m.float() * 2.0 ** -8


def _pow2_up(s):
    return float(2.0 ** np.ceil(np.log2(s)))


def _ties(dev):
    """power-of-two scales, no BN scale, shifts on the 2^-1 grid: a = fl(s_in s_w) is a power of two, so fl(v r) of an
    integer acc lands on .5 whenever its low bits say so.  Conv-0 terms are on a 2^-6 grid (features 2^-1, weights
    2^-5), so its fl(v r) has .5 fractions too.  W / s_w ties: _tie_weights; conv 2 has an all-zero column."""
    cin, convs = TIE_CHAIN
    g = torch.Generator().manual_seed(41)
    n = 700
    coors, rows = _lattice(convs, n, seed=42)
    feats = _grid(torch.empty(n, cin), 2.0 ** -1, 2.0, g)
    w = {0: _grid(torch.empty(27, cin, 32), 2.0 ** -4, 0.5, g) * 0.5}
    for i, c in enumerate(convs[1:], 1):
        w[i] = _tie_weights(g, 27, c["cin"], c["cout"], zero_col=3 if i == 2 else None)
    t = {i: torch.randint(-2, 3, (c["cout"],), generator=g).float() * 0.5 for i, c in enumerate(convs)}
    probe = RawI8(None, cin, SHAPE, B, convs, coors, seed=43, feats=feats, weights=w, shifts=t,
                  s_act=[None] * len(convs))
    s_act = [_pow2_up(s) for s in probe.s_act]
    return RawI8(dev, cin, SHAPE, B, convs, coors, seed=43, feats=feats, weights=w, shifts=t, s_act=s_act), rows


# ---- d. accumulators past 2^24 ---------------------------------------------------------------------------------
CUBE = 6
ACC_CHAIN = (5, [conv(5, 128), conv(128, 128, scale=False), conv(128, 64, scale=False, shift=False)])


def _one_sign_weights(g, kv, cin, cout):
    """W = m 2^-7, m in [0, 127] with one in ten negated and one 127 per column: s_w = 2^-7, q = m"""
    m = torch.randint(0, 128, (kv, cin, cout), generator=g)
    m = torch.where(torch.rand(kv, cin, cout, generator=g) < 0.1, -m, m)
    m.view(-1, cout)[torch.randint(0, kv * cin, (cout,), generator=g), torch.arange(cout)] = 127
    return m


def _acc_past_2_24(dev):
    """One sample with a full 6x6x6 cube of voxels: its 64 interior rows see all 27 neighbours.  Conv 0's BN scale 0
    and shift 16 with s_0 = 2^-4 put 255 on every row (fl(16 * 16) = 256 saturates), so conv 1 (128 -> 128 k3, wgmma)
    sums acc = 255 sum_k,ci q over an interior row, past 2^24.  Its shift cancels all but 128 of fl(float(acc) a)
    (a = 2^-11, exact), so float(acc)'s rounding shows in the u8 image (r = 2^11): 128 when it rounds to nearest."""
    cin, convs = ACC_CHAIN
    g = torch.Generator().manual_seed(51)
    r = np.arange(1, CUBE + 1)
    xs, ys, zs = np.meshgrid(r, r, r, indexing="ij")
    coors = np.stack([np.zeros(CUBE ** 3, int), xs.ravel(), ys.ravel(), zs.ravel()], 1).astype(np.int32)
    m1 = _one_sign_weights(g, 27, 128, 128)
    f = (255 * m1.sum((0, 1)).numpy().astype(np.int64)).astype(np.float32)         # float32(acc) of interior rows
    shift1 = torch.from_numpy(-(f - np.float32(128)) * np.float32(2.0 ** -11))
    w = {1: m1.float() * 2.0 ** -7, 2: _one_sign_weights(g, 27, 128, 64).float() * 2.0 ** -7}
    raw = RawI8(dev, cin, [CUBE + 2] * 3, 1, convs, coors, seed=52, weights=w,
                bn_scales={0: torch.zeros(128)}, shifts={0: torch.full((128,), 16.0), 1: shift1},
                s_act=[2.0 ** -4, 2.0 ** -11, 1.0])
    return raw, [CUBE ** 3]


# ---- e. the last conv's half overflowing -----------------------------------------------------------------------
HALF_CHAIN = (5, [conv(5, 32), conv(32, 64)])


def _half_overflow(dev):
    """the last conv's v = acc a' + 65500 with a' spreading acc a' over [-24, 24]: half(v) is 65504 on
    [65488, 65520) and inf from 65520"""
    cin, convs = HALF_CHAIN
    base, rows = _raw(None, cin, convs, seed=61)
    d, _, _ = base.oracle()
    C = convs[-1]["cout"]
    t = base.t[-1].double()
    v = d.reshape(B, C, -1).transpose(0, 1).reshape(C, -1)
    span = torch.where(v > 0, (v - t[:, None]).abs(), torch.zeros_like(v)).amax(1).clamp_min(1e-3)
    scale = (base.s[-1].double() * 24 / span).float()
    return _raw(dev, cin, convs, seed=61, bn_scales={1: scale}, shifts={1: torch.full((C,), 65500.0)},
                s_act=base.s_act)


# ---- f. short chains -------------------------------------------------------------------------------------------
SHORT_CHAINS = {
    "one-conv-5-16": (5, [conv(5, 16)]),
    "one-conv-40-128": (40, [conv(40, 128)]),           # conv 0, fp16 in and out, through the INT8 epilogue (wgmma)
    "two-conv": (5, [conv(5, 32), conv(32, 16)]),       # mode 5 mma 32
}


def _short_case(name):
    cin, convs = SHORT_CHAINS[name]
    return [("f16_out", [len(convs) - 1], 1)], lambda dev: _raw(dev, cin, convs, seed=71)


# ---- g. NaN and +-inf features on valid rows ------------------------------------------------------------------
def _non_finite(dev):
    cin, convs = TINY_CHAIN
    coors, rows = _lattice(convs, seed=81)
    g = torch.Generator().manual_seed(82)
    f = _grid(torch.empty(coors.shape[0], cin), 2.0 ** -4, 8.0, g)
    finite = RawI8(None, cin, SHAPE, B, convs, coors, seed=83, feats=f)       # the scales of the finite features
    for k, v in enumerate((float("nan"), float("inf"), -float("inf"))):
        f[10 * k: 10 * k + 10, k] = v
    return RawI8(dev, cin, SHAPE, B, convs, coors, seed=83, feats=f, s_act=finite.s_act), rows


# ---- h. persistent tiles ---------------------------------------------------------------------------------------
# one level: conv 1 mode 4 mma.sync 64, conv 2 and conv 3 (the residual of conv 1) mode 4 wgmma 64
TILE_LEVEL_CHAIN = (5, [conv(5, 16), conv(16, 64), conv(64, 64), conv(64, 64, res=1)])
TILE_SHAPE, TILE_B = [64, 64, 41], 2


def tile_counts():
    return sorted({t + d for t in (T_MMA, T_WG) for d in (-1, 0, 1)} | {2 * T_MMA + 1, 2 * T_WG + 1})


def _tiles(n, n_rows=None):
    def build(dev):
        cin, convs = TILE_LEVEL_CHAIN
        coors, rows = lattice_coors(TILE_SHAPE, TILE_B, n, 0, seed=n)
        return RawI8(dev, cin, TILE_SHAPE, TILE_B, convs, coors, n_rows=n_rows, seed=n,
                     s_act=[None] * len(convs)), rows
    return build


# ---- the registry ----------------------------------------------------------------------------------------------
CASES = {}
for _name in INSTANCE_CHAINS:
    CASES[_name] = _instance_case(_name)
CASES.update({
    "sat-quarter": ([("sat", [0, 1], 1)], _sat_quarter),
    "sat-other-seed": ([("sat", list(range(8)), 1)], _sat_other_seed),
    # r_out = fl(1 / 2^-140) = +inf: v > 0 -> 255, v = 0 -> 0 inf = NaN -> 0; conv 2's a is subnormal
    "sat-rout-inf": ([("overflow", [1], 1), ("nan", [1], 1)], _sat_scale(2.0 ** -140)),
    # r_out = 2^126: fl(v r_out) = +inf from v >= 4 (shift 4 on half the channels)
    "sat-v-overflow": ([("overflow", [1], 1)], _sat_scale(2.0 ** -126, {1: torch.tensor([4.0, 0.0] * 16)})),
    "ties": ([("ties", [0, 1, 2], 1), ("w_ties", [1, 2, 3], 1), ("w_zero_cols", [2], 1)], _ties),
    "acc-2-24": ([("acc_inexact", [1], 1000), ("sat", [0], 1)], _acc_past_2_24),
    "half-overflow": ([("half_inf", [1], 1), ("half_max", [1], 1)], _half_overflow),
    "non-finite": ([("nan", [0], 1), ("sat", [0], 1)], _non_finite),
})
for _name in SHORT_CHAINS:
    CASES[_name] = _short_case(_name)

TILE_CASES = {"tiles-%d" % n: _tiles(n) for n in tile_counts()}
TILE_CASES["tiles-cap-%d-of-%d" % (T_MMA + 1, 2 * T_MMA + 1)] = _tiles(T_MMA + 1, n_rows=2 * T_MMA + 1)

# every chain the GPU edge tests run, for the instance map and the host acceptance
CHAINS = dict(INSTANCE_CHAINS, **SHORT_CHAINS)
CHAINS.update({"sat": SAT_CHAIN, "sat-other-seed": INT8_RAW["residual-every-level"], "tiny": TINY_CHAIN,
               "ties": TIE_CHAIN, "acc-2-24": ACC_CHAIN, "half-overflow": HALF_CHAIN, "tiles": TILE_LEVEL_CHAIN})
