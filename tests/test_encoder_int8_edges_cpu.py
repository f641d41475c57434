"""CPU twins of the INT8 plan's edge cases (encoder_int8_cases): the GPU cases together launch all twelve INT8 kernel
instances, the host accepts every chain they run, each case reaches the edge it is named for in the exact oracle
(saturation, rounding ties, accumulators past 2^24, the last conv's half overflowing, NaN / +-inf features, short
chains), the persistent-tile row counts put a second tile on some CTA of both kernels, and the oracle's stats leave
its results alone."""
import numpy as np
import pytest
import torch

from bevfusion_b200 import _C
from bevfusion_b200.spconv.ops import PREC_INT8
from encoder_int8_cases import (CASES, CHAINS, INSTANCES, T_MMA, T_WG, TILE_CASES, TILE_LEVEL_CHAIN, TILE_SHAPE,
                                chain_instances, int8_instance, tiles_per_cta, tile_counts)
from encoder_int8_oracle import STAT_KEYS
from test_encoder_int8_gpu import INT8_RAW
from test_encoder_plan_gpu import create


def test_gpu_cases_reach_all_twelve_instances():
    seen = {}
    for name, (_, convs) in CHAINS.items():
        for inst in chain_instances(convs):
            seen.setdefault(inst, name)
    print("\n".join("%s %s Cout %d: %s" % (m, k, c, seen.get((m, k, c))) for m, k, c in sorted(INSTANCES)))
    assert set(seen) == INSTANCES


def test_instance_map_of_the_four_new_ones():
    """the four instances the older INT8 chains never launch, each on the chain that adds it"""
    assert int8_instance(0, 5, 64, 27) == (5, "mma", 64)
    assert int8_instance(0, 5, 128, 27) == (5, "mma", 128)
    assert int8_instance(0, 40, 128, 27) == (5, "wg", 128)
    assert int8_instance(1, 16, 64, 27) == int8_instance(1, 64, 64, 3) == (4, "mma", 64)
    old = {inst for _, convs in INT8_RAW.values() for inst in chain_instances(convs)}
    assert not old & {(4, "mma", 64), (5, "mma", 64), (5, "mma", 128), (5, "wg", 128)}


@pytest.mark.parametrize("chain", list(CHAINS))
def test_chain_accepted_on_host(chain):
    cin, convs = CHAINS[chain]
    L = _C.lib()
    rc, h = create(cin, TILE_SHAPE, convs)
    assert rc == 0, L.bevb200_last_error()
    try:
        assert L.bevb200_encoder_set_precision(h, PREC_INT8) == 0, L.bevb200_last_error()
    finally:
        L.bevb200_encoder_destroy(h)


@pytest.mark.parametrize("case", list(CASES))
def test_case_reaches_its_edge(case):
    edges, build = CASES[case]
    raw, _ = build(None)
    stats = raw.stats()
    assert all(set(d) == set(STAT_KEYS) for d in stats)
    for i, d in enumerate(stats):
        print("conv %d: %s" % (i, " ".join("%s=%s" % (k, d[k]) for k in STAT_KEYS)))
    for stat, convs, least in edges:
        got = sum(stats[i][stat] for i in convs)
        assert got >= least, "%s: %s over convs %s is %s < %s" % (case, stat, convs, got, least)


def test_tile_counts_straddle_a_second_tile():
    counts = tile_counts()
    assert len(counts) >= 4 and set(TILE_CASES) >= {"tiles-%d" % n for n in counts}
    for n in counts:
        for kernel, t in (("mma", T_MMA), ("wg", T_WG)):
            assert (tiles_per_cta(n, kernel) >= 2) == (n > t)
    assert tiles_per_cta(T_MMA + 1, "mma") == 2 and tiles_per_cta(T_WG + 1, "wg") == 2
    assert tiles_per_cta(T_MMA, "mma") == 1 and tiles_per_cta(T_WG, "wg") == 1
    # the level holds a mode-4 mma.sync conv, a mode-4 wgmma conv and a residual
    _, convs = TILE_LEVEL_CHAIN
    inst = chain_instances(convs)
    assert (4, "mma", 64) in inst and (4, "wg", 64) in inst and any(c["res"] >= 0 for c in convs)
    assert all(c["subm"] for c in convs)


def test_stats_leave_results_alone():
    _, build = CASES["ties"]
    raw, _ = build(None)
    plain = raw.oracle(stats=None)
    st = []
    with_stats = raw.oracle(stats=st)
    assert len(st) == len(raw.convs)
    for a, b in zip(plain, with_stats):
        if isinstance(a, torch.Tensor):
            assert torch.equal(a, b)
        else:
            assert a == b
    assert [d["s_act"] for d in st] == raw.s_act
    assert np.isfinite([d["acc_max"] for d in st]).all()
