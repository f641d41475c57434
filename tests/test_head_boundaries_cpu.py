"""The boundary cases of test_head_boundaries_gpu on the CPU: the constants are read from the sources that define
them and agree with the Python modules' limits, and every case builder lands exactly on the boundary it names --
element counts on tile edges, duplicate slots across the backward's passes, threshold bins of kBufCap - 1, kBufCap
and kBufCap + 1 keys in their own key byte, grid geometries at one row per block and at exactly the shared-memory
limit; the allocation guard notices a byte written just outside a tensor and restores the modules."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
import head_boundaries as HB  # noqa: E402
from bevfusion_b200 import _C  # noqa: E402
from bevfusion_b200 import centerhead_decode as CD  # noqa: E402
from bevfusion_b200 import head_losses as HL  # noqa: E402
from bevfusion_b200 import head_targets as HT  # noqa: E402
from bevfusion_b200 import map_seg as MS  # noqa: E402
from bevfusion_b200 import transfusion_assign as TA  # noqa: E402
from bevfusion_b200 import transfusion_proposals as TP  # noqa: E402


def test_constants_match_the_modules():
    assert (HL.MAX_TASKS, HL.MAX_OBJS, HL.MAX_LAYERS) == (HB.LOSS_MAX_TASKS, HB.LOSS_MAX_OBJS, HB.LOSS_MAX_LAYERS)
    assert TP.MAX_PROPOSALS == HB.PROPOSALS_MAX_K and CD.MAX_NUM == HB.DECODE_MAX_K
    assert TA.MAX_SIZE == HB.ASSIGN_MAX
    assert (HT.MAX_BOXES, HT.MAX_TASKS) == (HB.TARGETS_MAX_BOXES, HB.TARGETS_MAX_TASKS)
    assert MS._SMEM_LIMIT == HB.GRID_SMEM_LIMIT
    assert HB.header_macro("BEVB200_PROPOSALS_MAX_CELLS") == TP.MAX_CELLS     # a parenthesised shift
    # the tile constants the cases straddle are multiples of their thread counts, as the kernels assume
    assert HB.TOPK_TILE % HB.cu_const("transfusion_proposals.cu", "kPeakThreads") == 0
    assert HB.LOSS_TILE % HB.cu_const("head_losses.cu", "kThreads") == 0
    assert HB.SEG_COUNT_TILE % HB.cu_const("map_seg.cu", "kThreads") == 0
    with pytest.raises(KeyError):
        HB.cu_const("head_losses.cu", "kNoSuchConstant")


def test_tile_edges_and_map_factors():
    for tile in (HB.LOSS_TILE, HB.TOPK_TILE, HB.SEG_COUNT_TILE):
        edges = HB.tile_edges(tile, ks=(1, 3))
        assert {tile - 1, tile, tile + 1, 3 * tile - 1, 3 * tile + 1} <= set(edges)
        for n in edges:
            c, h, w = HB.factor_map(n, max_c=8)
            assert c * h * w == n
    for n in HB.tile_edges(HB.TOPK_TILE, ks=(1, 2, 4), extra=()):
        chw = HB.factor_map(n, min_side=3, max_c=TP.MAX_CLASSES)
        assert chw is None or (np.prod(chw) == n and min(chw[1:]) >= 3)
    assert HB.factor_map(7, min_side=3) is None


@pytest.mark.parametrize("M", [HB.SLOT_THREADS - 1, HB.SLOT_THREADS + 1, 3 * HB.SLOT_THREADS + 1, HB.LOSS_MAX_OBJS])
def test_slot_case_straddles_the_passes(M):
    S = HB.SLOT_THREADS
    inds, masks = HB.slot_case(M, 2, 1440, seed=M)
    assert masks[0][0].all() and not masks[0][1].any()                     # a full sample next to an empty one
    ind, mask = inds[1], masks[1]
    shared = [m for m in (0, S - 1, S, M - 1) if m < M]
    assert (ind[:, shared] == HB.SHARED_CELL).all() and mask[:, shared].all()
    assert not mask[:, 3::7][:, 1:-1].all() and not mask[:, S // 2:S // 2 + S // 4].any()   # gaps
    if M > S + 5:
        # a duplicate whose first masked-in slot is in one pass and a later one in the next
        live = [(m // S, c) for m, c in enumerate(ind[0]) if mask[0, m]]
        passes = {}
        for p, c in live:
            passes.setdefault(c, set()).add(p)
        assert sum(len(v) > 1 for v in passes.values()) > 5
    assert len(np.unique(inds[2])) <= 8


def _sigmoid32(x):
    x = np.float32(x)
    return np.float32(1) / (np.float32(1) + np.exp(-x))


@pytest.mark.parametrize("ties", list(HB.TIE_COUNTS))
def test_tie_planes_put_the_threshold_bin_on_the_buffer_edge(ties):
    n_tie = HB.TIE_COUNTS[ties]
    n_hi = 100
    for planes, values in ((2, [_sigmoid32(3.0), _sigmoid32(-3.0), _sigmoid32(-8.0)]), (2, [0.9, 0.3, 0.01]),
                           (4, [0.9, 0.3, 0.01])):
        top = HB.order_key_top_byte(values)
        assert top[0] > top[1] > top[2]                                     # three separate first-digit bins
        side = HB.tie_side(n_hi, n_tie, planes)
        kinds = HB.tie_kinds(planes * side * side, n_hi, n_tie, seed=1)
        assert (kinds == HB.TIE).sum() == n_tie and (kinds == HB.HI).sum() == n_hi
        assert (kinds == HB.LO).sum() >= n_hi
        tiles = np.unique(np.nonzero(kinds == HB.TIE)[0] // HB.TOPK_TILE)
        assert len(tiles) == -(-kinds.size // HB.TOPK_TILE)                  # the tie reaches every tile
        K = min(n_hi + n_tie // 2, HB.PROPOSALS_MAX_K, side * side)
        assert n_hi < K < n_hi + n_tie                                      # the K-th key is a tied one
    assert {HB.TIE_COUNTS["cap-1"], HB.TIE_COUNTS["cap"], HB.TIE_COUNTS["cap+1"]} == \
        {HB.BUF_CAP - 1, HB.BUF_CAP, HB.BUF_CAP + 1}


@pytest.mark.parametrize("direction,R,exact", [("fwd", 1, False), ("fwd", 1, True), ("bwd", 1, True),
                                               ("fwd", HB.GRID_ROWS[0], True)])
def test_grid_geometries_at_the_shared_memory_limit(direction, R, exact):
    smem = _C.lib().bevb200_map_grid_smem_bytes
    geom = HB.grid_geometry(smem, direction, R, exact)
    assert geom is not None
    isc, osc, H, W, s = geom
    back = direction == "bwd"
    assert HB.grid_plan_rows(smem, isc, osc, H, W, back) == (R, s)
    assert HB.grid_plan_rows(smem, isc, osc, H, W, not back)[0] is not None      # the other direction fits too
    assert s <= HB.GRID_SMEM_LIMIT and (s == HB.GRID_SMEM_LIMIT) >= exact
    if R == 1:   # two rows per block would not fit
        ry = MS.axis_taps(MS.axis_coords(isc[0], osc[0]), H)
        rx = MS.axis_taps(MS.axis_coords(isc[1], osc[1]), W)
        nnz = sum(len(t) for t in rx)
        if back:
            n2 = int(MS._blocks(MS.transpose_taps(ry, H), 2)[1].max())
            assert smem(len(rx), W, nnz, n2) > HB.GRID_SMEM_LIMIT
        else:
            assert smem(W, len(rx), nnz, int(MS._blocks(ry, 2)[1].max())) > HB.GRID_SMEM_LIMIT


def test_guard_sees_a_byte_outside_the_tensor():
    import types
    mod = types.SimpleNamespace(torch=torch)
    with HB.DeviceGuard(mod) as g:
        assert mod.torch is not torch
        assert mod.torch.float32 is torch.float32
        cpu = mod.torch.zeros((3, 5))                  # host allocations are not carved
        assert len(g.blocks) == 0 and cpu.sum() == 0
        t = g.carve(torch.arange(15, dtype=torch.float32).view(3, 5), fill=True)
        assert torch.equal(t, torch.arange(15, dtype=torch.float32).view(3, 5)) and t.is_contiguous()
        t.fill_(7.0)
        g.check()
        buf, lo, hi = g.blocks[0]
        for pos in (lo - 1, hi):
            saved = int(buf[pos])
            buf[pos] = saved ^ 0xff
            with pytest.raises(AssertionError, match="written outside"):
                g.check()
            buf[pos] = saved
        g.check()
    assert mod.torch is torch
