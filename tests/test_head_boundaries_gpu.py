"""The detection-head kernels across their tile, block and limit boundaries against the float64 oracles, every
boundary read from the constant that sets it (head_boundaries): the CenterHead loss backward's slot passes, the
dense-loss tiles of both heads, the shared top-K select's threshold-bin buffer and candidate tiles for the TransFusion
proposals and the CenterHead decode, the LSAP solver's one-warp / eight-warp switch, the head-target assign stride and
limits, and the map-segmentation loss / count tiles and grid-transform shared memory.  Every call runs under a
DeviceGuard: its outputs, gradients and exactly-sized workspaces are carved from canary-filled buffers, and no byte
outside them may change."""
import os
import sys

import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
import centerhead_decode_oracle as CDO  # noqa: E402
import head_boundaries as HB  # noqa: E402
import head_losses_oracle as HLO  # noqa: E402
import head_targets_oracle as HTO  # noqa: E402
import map_seg_oracle as MSO  # noqa: E402
import transfusion_assign_oracle as TAO  # noqa: E402
import transfusion_proposals_oracle as TPO  # noqa: E402
from bevfusion_b200 import _C  # noqa: E402
from bevfusion_b200 import centerhead_decode as CD  # noqa: E402
from bevfusion_b200 import head_losses as HL  # noqa: E402
from bevfusion_b200 import head_targets as HT  # noqa: E402
from bevfusion_b200 import map_seg as MS  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200 import transfusion_assign as TA  # noqa: E402
from bevfusion_b200 import transfusion_proposals as TP  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
CW = [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.2, 0.2]
LOSS_RTOL, GRAD_TOL = 2e-6, 1e-5                  # test_head_losses_gpu's bounds
MAPS = (("reg", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2))
TF_MAPS = (("center", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2))


def guard(*modules):
    return HB.DeviceGuard(*modules)


def np64(t):
    return t.detach().double().cpu().numpy()


def dev_sigmoid(x):
    return torch.sigmoid(x.detach().float()).cpu().numpy()


def check_losses(got, want, rtol=LOSS_RTOL):
    assert list(got) == list(want)
    for k in want:
        g = float(got[k].detach())
        assert abs(g - want[k]) <= rtol * abs(want[k]) + 1e-30, (k, g, want[k])


def check_grad(got, want, name, tol=GRAD_TOL):
    """within tol of the largest |want|, zero exactly where want is"""
    got = np64(got)
    scale = max(np.abs(want).max(), 1e-30)
    assert np.abs(got - want).max() <= tol * scale, (name, np.abs(got - want).max(), scale)
    np.testing.assert_array_equal(got == 0, want == 0, err_msg=name + ": zero set")


def saved_avg(loss):
    """The avg factors the loss's forward saved for its backward (the last saved tensor of the autograd node)."""
    node = loss.grad_fn
    while not hasattr(node, "saved_tensors") or not node.saved_tensors:
        node = node.next_functions[0][0]
    return node.saved_tensors[-1].cpu().numpy()


# ---- 1, 2: CenterHead loss ----------------------------------------------------------------------------------------
def ch_inputs(rng, B, cats, H, W, M, code, inds, masks):
    preds, heat_t, annos = [], [], []
    for t, cat in enumerate(cats):
        p = {"heatmap": rng.standard_normal((B, cat, H, W)) * 2}
        for k, c in MAPS[:4 if code == 8 else 5]:
            p[k] = rng.standard_normal((B, c, H, W))
        preds.append([{k: torch.tensor(v, dtype=torch.float32, device=DEV).requires_grad_() for k, v in p.items()}])
        ht = rng.random((B, cat, H, W)) * 0.9
        ht.reshape(-1)[rng.integers(0, ht.size, max(1, ht.size // 50))] = 1.0
        heat_t.append(torch.tensor(ht, dtype=torch.float32, device=DEV))
        annos.append(torch.tensor(rng.standard_normal((B, M, code)), dtype=torch.float32, device=DEV))
    return preds, (heat_t, annos, [torch.tensor(i, dtype=torch.int64, device=DEV) for i in inds],
                   [torch.tensor(m, dtype=torch.uint8, device=DEV) for m in masks])


def run_ch(preds, targets, lw=(1.0, 0.25)):
    code = targets[1][0].shape[-1]
    with guard(HL) as g:
        losses, status = HL.centerhead_loss(preds, targets, dict(code_weights=CW[:code]),
                                            loss_cls=dict(type="GaussianFocalLoss", loss_weight=lw[0]),
                                            loss_bbox=dict(type="L1Loss", loss_weight=lw[1]), return_status=True)
        avg = saved_avg(losses["heatmap/task0"])
        sum(losses.values()).backward()
        g.check("centerhead_loss")
    assert int(status) == 0
    P = [{k: np64(v) for k, v in p[0].items()} for p in preds]
    T = tuple([np64(x) for x in lst] for lst in targets)
    want, wgrad = HLO.centerhead(P, T, CW[:code], cls=(lw[0], 2.0, 4.0), bbox_lw=lw[1],
                                 y32=[dev_sigmoid(p[0]["heatmap"]) for p in preds])
    check_losses(losses, want)
    for t in range(len(preds)):
        npos = np.float32(max(float((T[0][t] == 1).sum()), 1.0))
        num = np.float32(np.float32(T[3][t].astype(np.float32).sum()) + np.float32(1e-4))
        assert avg[2 * t] == npos and avg[2 * t + 1] == num, (t, avg[2 * t:2 * t + 2], npos, num)
        for k, v in preds[t][0].items():
            check_grad(v.grad, wgrad[t][k], "task%d %s" % (t, k))


S_ = HB.SLOT_THREADS
SLOT_M = {"S-1": S_ - 1, "S": S_, "S+1": S_ + 1, "2S": 2 * S_, "3S+1": 3 * S_ + 1, "MAX_OBJS": HB.LOSS_MAX_OBJS}


@pytest.mark.parametrize("name,code", [(n, 10) for n in SLOT_M] + [("S", 8), ("3S+1", 8)])
def test_centerhead_backward_slot_passes(name, code):
    """max_objs on both sides of each pass of kSlotThreads slots, duplicates straddling the passes, gaps in the
    masks, an all-masked-out sample next to a full one; loss, avg factors and every gradient with its zero set."""
    M = SLOT_M[name]
    B, H, W = 2, 40, 36
    inds, masks = HB.slot_case(M, B, H * W, seed=M)
    preds, targets = ch_inputs(np.random.default_rng(M + code), B, [1, 2, 2], H, W, M, code, inds, masks)
    run_ch(preds, targets)


def dense_cases(tile):
    """(id, B, cats, H, W): task 0's B * cat * H * W on each edge of `tile` (the vec and scalar paths), and MAX_TASKS
    tasks."""
    out = []
    for n in HB.tile_edges(tile, ks=(1, 3)):
        c, h, w = HB.factor_map(n, max_c=8)
        out.append(("n=%d" % n, 1, [c, 1], h, w))
    out.append(("MAX_TASKS", 2, [1 + t % 3 for t in range(HB.LOSS_MAX_TASKS)], 9, 7))
    return out


@pytest.mark.parametrize("case", dense_cases(HB.LOSS_TILE), ids=lambda c: c[0])
def test_centerhead_dense_tile_tails(case):
    _, B, cats, H, W = case
    M = 5
    rng = np.random.default_rng(B * H * W)
    inds = [rng.integers(0, H * W, (B, M)) for _ in cats]
    masks = [(rng.random((B, M)) < 0.7).astype(np.uint8) for _ in cats]
    preds, targets = ch_inputs(rng, B, cats, H, W, M, 10, inds, masks)
    run_ch(preds, targets, lw=(1.3, 0.4))


# ---- 2: TransFusion loss ----------------------------------------------------------------------------------------
def tf_case(rng, B, K, H, W, P, L, code=10):
    N = L * P
    pr = {"dense_heatmap": rng.standard_normal((B, K, H, W)) * 2, "heatmap": rng.standard_normal((B, K, N)) * 2}
    for k, c in TF_MAPS[:4 if code == 8 else 5]:
        pr[k] = rng.standard_normal((B, c, N))
    preds = {k: torch.tensor(v, dtype=torch.float32, device=DEV).requires_grad_() for k, v in pr.items()}
    heat = rng.random((B, K, H, W)) * 0.9
    heat.reshape(-1)[rng.integers(0, heat.size, max(1, heat.size // 40))] = 1.0
    labels = rng.integers(0, K + 1, (B, N))
    lweights = rng.integers(0, 2, (B, N))
    bt = rng.standard_normal((B, N, code)).astype(np.float32)
    bw = (rng.random((B, N, code)) < 0.6).astype(np.float32)
    num_pos = rng.integers(0, 4, B).astype(np.int32)
    mean_iou = rng.random(B).astype(np.float32)
    t = lambda a, dt: torch.tensor(a, dtype=dt, device=DEV)   # noqa: E731
    targets = (t(labels, torch.int64), t(lweights, torch.int64), t(bt, torch.float32), t(bw, torch.float32), None,
               t(num_pos, torch.int32), t(mean_iou, torch.float32), None, t(heat, torch.float32))
    oracle_t = (labels, lweights, bt, bw, int(num_pos.sum()), list(mean_iou), heat)
    return preds, targets, oracle_t


def tf_dense_cases(tile):
    """(id, B, K, H, W, P, L): the dense term B * K * H * W on each edge of `tile`, L 1 and MAX_LAYERS, P 1 and P
    with B * K * P past one tile"""
    out = []
    for i, n in enumerate(HB.tile_edges(tile, ks=(1, 3))):
        k, h, w = HB.factor_map(n, max_c=16)
        P, L = [(1, 1), (tile // k + 3, 1), (7, HB.LOSS_MAX_LAYERS), (1, HB.LOSS_MAX_LAYERS)][i % 4]
        out.append(("n=%d,P=%d,L=%d" % (n, P, L), 1, k, h, w, P, L))
    out.append(("B=2,P>tile,L=MAX", 2, 10, 13, 11, tile // 10 + 1, HB.LOSS_MAX_LAYERS))
    return out


@pytest.mark.parametrize("case", tf_dense_cases(HB.LOSS_TILE), ids=lambda c: c[0])
def test_transfusion_dense_tile_tails(case):
    _, B, K, H, W, P, L = case
    lw = (1.2, 0.8, 0.3)
    preds, targets, ot = tf_case(np.random.default_rng(K * H * W + P), B, K, H, W, P, L)
    with guard(HL) as g:
        losses = HL.transfusion_loss([[preds]], targets, P, L, True, dict(code_weights=CW),
                                     loss_cls=dict(type="FocalLoss", use_sigmoid=True, gamma=2.0, alpha=0.25,
                                                   loss_weight=lw[1]),
                                     loss_bbox=dict(type="L1Loss", loss_weight=lw[2]),
                                     loss_heatmap=dict(type="GaussianFocalLoss", loss_weight=lw[0]))
        avg = saved_avg(losses["loss_heatmap"])
        sum(v for k, v in losses.items() if k != "matched_ious").backward()
        g.check("transfusion_loss")
    pn = {k: np64(v) for k, v in preds.items()}
    want, wgrad = HLO.transfusion(pn, ot, P, L, True, CW, heat=(lw[0], 2.0, 4.0), cls=(lw[1], 0.25, 2.0),
                                  bbox_lw=lw[2], y32=dev_sigmoid(preds["dense_heatmap"]))
    check_losses(losses, want)
    assert avg[0] == np.float32(max(float((ot[6] == 1).sum()), 1.0)) and avg[1] == np.float32(max(ot[4], 1))
    for k, v in preds.items():
        check_grad(v.grad, wgrad[k], k)


# ---- 3: exact top-K ---------------------------------------------------------------------------------------------
def assert_same_proposals(got, want, what):
    for name, a, b in zip(("labels", "index"), got[:2], want[:2]):
        assert torch.equal(a, b), "%s %s: %d differ" % (what, name, int((a != b).sum()))
    gs, ws = got[2], want[2]
    assert torch.equal(torch.isnan(gs), torch.isnan(ws)) and bool(((gs.view(torch.int32) == ws.view(torch.int32))
                                                                    | torch.isnan(ws)).all()), what


def run_proposals(x, K, dataset):
    with guard(TP) as g:
        got = TP.transfusion_proposals(x, K, 3, dataset)
        g.check("transfusion_proposals")
    assert_same_proposals(got, TPO.torch_proposals(x, K, 3, dataset), (tuple(x.shape), K, dataset))


N_HI = 100


@pytest.mark.parametrize("ties", list(HB.TIE_COUNTS))
def test_proposals_threshold_bin_at_buffer_capacity(ties):
    """nuScenes' exempt classes 8 and 9 hold N_HI cells above, n_tie cells tied at the K-th key and the rest below,
    each group in its own top key byte: the select's threshold bin is exactly the tie (kBufCap - 1, kBufCap,
    kBufCap + 1 keys, or many times kBufCap spread over every tile).  The other classes are masked zeros."""
    n_tie = HB.TIE_COUNTS[ties]
    side = HB.tie_side(N_HI, n_tie, 2)
    kinds = HB.tie_kinds(2 * side * side, N_HI, n_tie, seed=n_tie).reshape(2, side, side)
    x = torch.full((1, 10, side, side), -200.0)
    x[0, 8:10] = torch.from_numpy(np.choose(kinds, [3.0, -3.0, -8.0]).astype(np.float32))
    x = x.to(DEV)
    K = min(N_HI + n_tie // 2, HB.PROPOSALS_MAX_K)       # the K-th key inside the tie
    for k in (K, 1, HB.PROPOSALS_MAX_K):
        run_proposals(x, k, "nuScenes")


def topk_shape_cases(tile, min_side, max_c):
    out = []
    for n in HB.tile_edges(tile, ks=(1, 2, 4), extra=()):
        chw = HB.factor_map(n, min_side=min_side, max_c=max_c)
        if chw is not None:
            out.append(("CHW=%d" % n,) + chw)
    return out


@pytest.mark.parametrize("case", topk_shape_cases(HB.TOPK_TILE, 3, TP.MAX_CLASSES), ids=lambda c: c[0])
def test_proposals_candidate_tile_edges(case):
    """C * H * W = k * kTile - 1, k * kTile, k * kTile + 1; K 1, MAX_K (when the plane has that many cells) and the
    whole plane (at least the candidate count: the rest are masked zeros by index)."""
    _, C, H, W = case
    gen = torch.Generator(device=DEV).manual_seed(C * H * W)
    x = torch.randn((2, C, H, W), generator=gen, device=DEV) * 2.5 - 2.0
    dataset = "Waymo" if C > 2 else "none"
    for K in sorted({1, min(HB.PROPOSALS_MAX_K, C * H * W)}):   # MAX_K, or every cell of a smaller plane
        run_proposals(x, K, dataset)


def ordered(x):
    i = x.contiguous().view(torch.int32).long()
    return torch.where(i < 0, -(i & 0x7fffffff), i)


def assert_bits(got, want, what, ulp=0):
    assert got.shape == want.shape and got.dtype == want.dtype, what
    if not got.is_floating_point():
        assert torch.equal(got, want), "%s: %d differ" % (what, int((got != want).sum()))
        return
    assert torch.equal(torch.isnan(got), torch.isnan(want)), what
    d = (ordered(got) - ordered(want)).abs().masked_fill(torch.isnan(want), 0)
    assert d.numel() == 0 or int(d.max()) <= ulp, (what, int(d.max()))


def decode_maps(gen, heat):
    B, _, H, W = heat.shape
    r = lambda c, s=1.0: torch.randn((B, c, H, W), generator=gen, device=DEV) * s   # noqa: E731
    return dict(heatmap=heat, reg=torch.rand((B, 2, H, W), generator=gen, device=DEV), height=r(1),
                dim=r(3, 0.7).exp(), rot=r(2), vel=r(2, 3.0))


def run_decode(tasks, cfg):
    """as test_centerhead_decode_gpu's check_decode: index, labels, counts, scores, centre, velocity bit for bit,
    sizes and yaw within 2 ulp, against the stable restatement"""
    with guard(CD) as g:
        boxes, scores, labels, counts, index = CD.centerhead_decode_batched(tasks, cfg, False, False, with_index=True)
        g.check("centerhead_decode")
    B = tasks[0]["heatmap"].shape[0]
    for t, task in enumerate(tasks):
        wb, ws, wl, wi, wc = CDO.compact(CDO.torch_decode(task, cfg, True))
        seg, w = slice(t * B, (t + 1) * B), (cfg["max_num"], cfg.get("score_threshold"), t)
        assert_bits(counts[seg], wc, (w, "counts"))
        assert_bits(index[seg], wi.int(), (w, "index"))
        assert_bits(labels[seg], wl, (w, "labels"))
        assert_bits(scores[seg], ws, (w, "scores"))
        assert_bits(boxes[seg][..., :3], wb[..., :3], (w, "centre"))
        assert_bits(boxes[seg][..., 3:7], wb[..., 3:7], (w, "size and yaw"), 2)
        assert_bits(boxes[seg][..., 7:], wb[..., 7:], (w, "velocity"))
    return counts


@pytest.mark.parametrize("ties", list(HB.TIE_COUNTS))
def test_decode_threshold_bin_at_buffer_capacity(ties):
    """The decode's scores taken as given: N_HI at 0.9, n_tie at 0.3 tied at the K-th key, the rest at 0.01 (three
    top key bytes) over two classes; K inside the tie, K = 1, and with a threshold of 0.5 K above the candidate
    count."""
    n_tie = HB.TIE_COUNTS[ties]
    cat = 2 if n_tie <= 2 * HB.BUF_CAP else 4
    side = HB.tie_side(N_HI, n_tie, cat)
    kinds = HB.tie_kinds(cat * side * side, N_HI, n_tie, seed=n_tie + 1).reshape(1, cat, side, side)
    heat = torch.from_numpy(np.choose(kinds, [0.9, 0.3, 0.01]).astype(np.float32)).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(n_tie)
    tasks = [decode_maps(gen, heat)]
    K = min(N_HI + n_tie // 2, HB.DECODE_MAX_K, side * side)
    for k, thr in ((K, None), (1, None), (K, 0.5)):
        counts = run_decode(tasks, S.centerhead_coder_cfg(side, side, max_num=k, score_threshold=thr))
        if thr:
            assert int(counts.max()) <= N_HI


@pytest.mark.parametrize("case", topk_shape_cases(HB.TOPK_TILE, 1, CD.MAX_CLASSES), ids=lambda c: c[0])
def test_decode_candidate_tile_edges(case):
    _, C, H, W = case
    gen = torch.Generator(device=DEV).manual_seed(C * H * W + 1)
    tasks = [decode_maps(gen, torch.rand((2, C, H, W), generator=gen, device=DEV)),
             decode_maps(gen, torch.rand((2, 1, H, W), generator=gen, device=DEV))]
    for K, thr in ((1, None), (min(H * W, HB.DECODE_MAX_K), None), (min(H * W, HB.DECODE_MAX_K), 0.999)):
        run_decode(tasks, S.centerhead_coder_cfg(H, W, max_num=K, score_threshold=thr))


# ---- 4: LSAP at the one-warp / eight-warp switch ------------------------------------------------------------------
def lsap_mats(width, seed):
    """At solver width `width`: a square, a transposed (rows > columns) and a tie-heavy integer case."""
    rng = np.random.default_rng(seed)
    return [rng.standard_normal((width, width)).astype(np.float32),
            rng.standard_normal((width, width - 300)).astype(np.float32),
            rng.integers(0, 3, (48, width)).astype(np.float32)]


def solve_and_check(mats, R, C):
    cost = np.full((len(mats), R, C), 7.0, np.float32)   # padding must not leak into a segment
    for s, m in enumerate(mats):
        cost[s, :m.shape[0], :m.shape[1]] = m
    rc = torch.tensor([m.shape[0] for m in mats], dtype=torch.int32, device=DEV)
    cc = torch.tensor([m.shape[1] for m in mats], dtype=torch.int32, device=DEV)
    with guard(TA) as g:
        c4r, r4c, st = TA.linear_sum_assignment_batched(torch.from_numpy(cost).to(DEV), rc, cc, return_status=True)
        g.check("lsap")
    c4r, r4c, st = c4r.cpu().numpy(), r4c.cpu().numpy(), st.cpu().numpy()
    for s, m in enumerate(mats):
        assert st[s] == 0
        rows = np.nonzero(c4r[s] >= 0)[0]
        cols = c4r[s][rows]
        # a valid matching of min(R, C) pairs inside the segment, row4col its inverse
        assert len(rows) == min(m.shape) and len(set(cols.tolist())) == len(cols) and cols.max() < m.shape[1]
        assert (c4r[s][m.shape[0]:] == -1).all() and (r4c[s][m.shape[1]:] == -1).all()
        assert np.array_equal(r4c[s][cols], rows) and (r4c[s] >= 0).sum() == len(rows)
        a, b = linear_sum_assignment(m)
        assert m[rows, cols].astype(np.float64).sum() == m[a, b].astype(np.float64).sum(), (s, m.shape)   # optimal
        assert np.array_equal(rows, a) and np.array_equal(cols, b), (s, m.shape)                          # scipy's


WIDTHS = {"wide-1": HB.WIDE_COLUMNS - 1, "wide": HB.WIDE_COLUMNS, "wide+1": HB.WIDE_COLUMNS + 1}


@pytest.mark.parametrize("name", list(WIDTHS))
def test_lsap_at_the_warp_switch(name):
    """One batched call padded to the width: its square, transposed and tie-heavy segments and, narrower segments
    through counts -- at width kWideColumns + 1 the eight-warp form solves segments of every width."""
    width = WIDTHS[name]
    mats = lsap_mats(width, width)
    mats += [mats[0][:w, :w] for w in WIDTHS.values() if w < width]
    solve_and_check(mats, width, width)


def test_lsap_at_assign_max():
    rng = np.random.default_rng(3)
    mats = [rng.standard_normal((HB.ASSIGN_MAX, 64)).astype(np.float32),
            rng.integers(0, 4, (HB.WIDE_COLUMNS + 1, 40)).astype(np.float32)]
    solve_and_check(mats, HB.ASSIGN_MAX, 64)


@pytest.mark.parametrize("name", list(WIDTHS))
def test_transfusion_assign_at_the_warp_switch(name):
    """num_proposals at the switch: the pipeline's matching is scipy's on its own cost, the cost and the targets
    the oracle's (test_transfusion_assign_gpu's bounds)."""
    P = WIDTHS[name]
    cfg, coder = S.TRANSFUSION_TRAIN_CFG, S.TRANSFUSION_CODER
    gb, gl = S.gt_boxes(seed=P, batch=1, min_boxes=60, max_boxes=90)
    pred = {k: v.to(DEV) for k, v in S.transfusion_predictions(P, 1, (gb, gl), num_proposals=P, num_classes=10,
                                                                 layers=1).items()}
    boxes, labels, counts = HT.pad_gt([b.to(DEV) for b in gb], [l.to(DEV) for l in gl])
    with guard(TA) as g:
        out, ex = TA.transfusion_assign_batched(pred, boxes, labels, counts, 10, P, cfg, coder, return_extras=True)
        g.check("transfusion_assign")
    G = len(gb[0])
    cost = ex["cost"][0, :, :G].cpu().numpy()
    r, c = linear_sum_assignment(cost)
    mine = np.zeros(P, np.int64)
    mine[r] = c + 1
    got_inds = ex["gt_inds"][0].cpu().numpy()
    assert np.array_equal(got_inds, mine)
    pn = {k: v.cpu().numpy() for k, v in pred.items()}
    want = TAO.targets(boxes.cpu().numpy(), labels.cpu().numpy(), counts.cpu().numpy(), pn, 10, P, cfg, coder)
    wc, _ = TAO.cost_matrix(TAO.decode(pn["center"][0], pn["height"][0], pn["dim"][0], pn["rot"][0], coder),
                            pn["heatmap"][0], gb[0].numpy(), gl[0].numpy(), cfg)
    assert np.abs(cost - wc).max() <= 1e-6
    if np.array_equal(got_inds, want["gt_inds"][0]):
        for i, k in enumerate(("labels", "label_weights")):
            assert np.array_equal(out[i].cpu().numpy(), want[k]), k
        assert out[5].cpu().tolist() == want["num_pos"].tolist()
        bt = out[2].cpu().numpy()
        d = np.abs(bt.view(np.int32).astype(np.int64) - want["bbox_targets"].view(np.int32).astype(np.int64))
        assert d.max() <= 2
    else:   # a different optimum of equal total cost
        c64 = wc.astype(np.float64)
        tot = lambda ind: sum(c64[p, g - 1] for p, g in enumerate(ind) if g > 0)   # noqa: E731
        assert abs(tot(got_inds) - tot(want["gt_inds"][0])) <= 1e-6 * G


# ---- 5: head targets --------------------------------------------------------------------------------------------
CFG_SIX = dict(point_cloud_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], grid_size=[1024, 1024, 40],
               voxel_size=[0.1, 0.1, 0.2], out_size_factor=8, dense_reg=1, gaussian_overlap=0.1, max_objs=500,
               min_radius=2)
SIX = [1, 2, 2, 1, 2, 2]


def random_boxes(rng, B, n, counts, labels_max, D=9):
    boxes = np.zeros((B, n, D), np.float32)
    boxes[..., :2] = rng.uniform(-50, 50, (B, n, 2))      # every centre on the map
    boxes[..., 2] = rng.uniform(-3, 1, (B, n))
    boxes[..., 3:6] = np.exp(rng.uniform(-0.7, 1.8, (B, n, 3)))
    boxes[..., 6] = rng.uniform(-np.pi, np.pi, (B, n))
    if D == 9:
        boxes[..., 7:] = rng.standard_normal((B, n, 2))
    labels = rng.integers(0, labels_max, (B, n)).astype(np.int32)
    return boxes, labels, np.asarray(counts, np.int32)


def ht_ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.where(np.isnan(a) & np.isnan(b), 0, np.abs(ia - ib))


def run_targets(mode, task_classes, cfg, boxes, labels, counts, max_objs=0):
    b, l, c = (torch.from_numpy(x).to(DEV) for x in (boxes, labels, counts))
    table = HT.centerhead_label_table(task_classes) if mode == "centerhead" else [(0, k) for k in range(10)]
    with guard(HT) as g:
        hm, anno, ind, mask, status, rec = HT._run(b, l, c, mode, task_classes, table, cfg, max_objs)
        g.check("head_targets")
    osf = cfg["out_size_factor"]
    hms = HT._split_heatmap(hm, b.shape[0], task_classes, cfg["grid_size"][1] // osf, cfg["grid_size"][0] // osf)
    want = HTO.targets(boxes, labels, counts, mode, task_classes, cfg, max_objs)
    # test_head_targets_gpu's rules: records, ind, mask exact; heatmaps within 1 ulp, anno_box within 2
    assert np.array_equal(rec.cpu().numpy(), want["records"]), "draw records"
    assert int(status.item()) == want["status"]
    for gh, wh in zip(hms, want["heatmaps"]):
        assert ht_ulps(gh.cpu().numpy(), wh).max(initial=0) <= 1
    if mode == "centerhead":
        assert np.array_equal(ind.cpu().numpy(), want["ind"]) and np.array_equal(mask.cpu().numpy(), want["mask"])
        assert ht_ulps(anno.cpu().numpy(), want["anno"]).max(initial=0) <= 2
        return want["mask"]


NMAX = {"T-1": HB.ASSIGN_THREADS - 1, "T": HB.ASSIGN_THREADS, "T+1": HB.ASSIGN_THREADS + 1,
        "MAX_BOXES": HB.TARGETS_MAX_BOXES}


@pytest.mark.parametrize("name", list(NMAX))
def test_head_targets_at_assign_stride(name):
    """nmax on the edges of the assign kernel's thread stride and at MAX_BOXES; max_objs below, equal to and above
    the largest per-task object count (the overflow drops what the reference drops); both modes."""
    nmax = NMAX[name]
    B = 1 if nmax == HB.TARGETS_MAX_BOXES else 2
    rng = np.random.default_rng(nmax)
    boxes, labels, counts = random_boxes(rng, B, nmax, [nmax, nmax - 2][:B], 10)
    table = HT.centerhead_label_table(SIX)
    per_task = max(int(np.sum([table[l][0] == t for l in labels[b, :counts[b]]])) for b in range(B) for t in range(6))
    for M in (per_task // 2, per_task, per_task + 1):
        mask = run_targets("centerhead", SIX, dict(CFG_SIX, max_objs=M), boxes, labels, counts, M)
        assert mask.sum(axis=-1).max() == min(M, per_task)
    run_targets("transfusion", [10], CFG_SIX, boxes, labels, counts)


def test_head_targets_max_tasks():
    T = HB.TARGETS_MAX_TASKS
    rng = np.random.default_rng(T)
    classes = [1 + t % 2 for t in range(T)]
    n_labels = sum(classes)
    boxes, labels, counts = random_boxes(rng, 2, 300, [300, 257], n_labels, D=7)
    mask = run_targets("centerhead", classes, dict(CFG_SIX, max_objs=9), boxes, labels, counts, 9)
    assert mask.shape[0] == T and (mask.sum(-1) == 9).any()


# ---- 6: map segmentation ----------------------------------------------------------------------------------------
def seg_shapes():
    out = []
    for n in sorted(set(HB.tile_edges(HB.SEG_LOSS_TILE, ks=(1, 3)) + HB.tile_edges(HB.SEG_COUNT_TILE, ks=(1, 2)))):
        _, h, w = HB.factor_map(n, max_c=1)
        out.append((n, h, w))
    return out


@pytest.mark.parametrize("n,H,W", seg_shapes(), ids=lambda v: str(v))
@pytest.mark.parametrize("loss", ["focal", "xent"])
def test_map_seg_loss_and_counts_at_tiles(loss, n, H, W):
    """H * W on the edges of the loss tile (kLossTile) and the count tile (kCountTile), test_map_seg_gpu's bounds."""
    gen = torch.Generator(device="cpu").manual_seed(n)
    B, K = 2, 3
    x = (torch.randn((B, K, H, W), generator=gen) * 4).to(DEV).requires_grad_(True)
    t = (torch.rand((B, K, H, W), generator=gen) < 0.35).to(DEV)
    w = torch.tensor([1.0, 0.5, -2.0], device=DEV)
    with guard(MS) as g:
        got = torch.stack(list(MS.map_seg_loss(x, t, loss, list("abc")).values()))
        (gx,) = torch.autograd.grad((got * w).sum(), x)
        pred = torch.rand((B, K, H, W), generator=gen).to(DEV)
        counts = MS.map_seg_counts(pred, t)
        g.check("map_seg")
    xn, tn = x.detach().double().cpu().numpy(), t.double().cpu().numpy()
    np.testing.assert_allclose(got.detach().cpu().numpy(), MSO.losses(xn, tn, loss), rtol=2e-6, atol=0)
    want = MSO.loss_grad(xn, tn, loss, w.cpu().numpy())
    assert np.abs(gx.double().cpu().numpy() - want).max() <= 1e-5 * np.abs(want).max()
    np.testing.assert_array_equal(counts.cpu().numpy(), MSO.counts(pred.cpu().numpy(), t.cpu().numpy(),
                                                                   MS.THRESHOLDS))


GRIDS = {"fwd-one-row": ("fwd", 1, False), "fwd-one-row-at-limit": ("fwd", 1, True),
         "bwd-one-row-at-limit": ("bwd", 1, True), "fwd-max-rows-at-limit": ("fwd", HB.GRID_ROWS[0], True)}


@pytest.mark.parametrize("name", list(GRIDS))
def test_grid_transform_at_shared_memory_limit(name):
    """Geometries that force a direction's rows per block down to one, and to exactly the shared-memory limit at one
    row and at the most rows; forward and backward against fwd64 / bwd64 (test_map_seg_gpu's bound)."""
    direction, R, exact = GRIDS[name]
    geom = HB.grid_geometry(_C.lib().bevb200_map_grid_smem_bytes, direction, R, exact)
    assert geom is not None
    isc, osc, H, W, smem = geom
    t = MS.BEVGridTransform(input_scope=isc, output_scope=osc)
    gen = torch.Generator(device="cpu").manual_seed(W)
    x = torch.randn((2, 3, H, W), generator=gen).to(DEV).requires_grad_(True)
    with guard(MS) as g:
        y = t(x)
        gy = torch.randn(y.shape, generator=gen).to(DEV)
        (gi,) = torch.autograd.grad(y, x, gy)
        g.check("grid transform")
    plan = t.plan(H, W, DEV)
    assert (plan.fwd if direction == "fwd" else plan.bwd).R == R
    Ay, Ax = (torch.from_numpy(a).to(DEV) for a in MSO.transform_matrices(isc, osc, H, W))
    eps = 2.0 ** -23
    want, scale = Ay @ x.detach().double() @ Ax.T, Ay.abs() @ x.detach().double().abs() @ Ax.abs().T
    assert bool(((y.double() - want).abs() <= 8 * eps * scale).all())
    want, scale = Ay.T @ gy.double() @ Ax, Ay.abs().T @ gy.double().abs() @ Ax.abs()
    assert bool(((gi.double() - want).abs() <= 8 * eps * scale).all())
