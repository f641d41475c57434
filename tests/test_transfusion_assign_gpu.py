"""TransFusion training-target assignment on the GPU (bevfusion_b200.transfusion_assign): the batched solver
against scipy, the cost against a torch-on-CUDA restatement of the reference's, the whole get_targets against
the reference's loop restated on CUDA tensors with scipy, the edge cases, reproducibility, CUDA-graph replay and
the launch count."""
import os
import sys

import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import lsap_oracle  # noqa: E402
import nms_oracle as O  # noqa: E402
from conftest import ref_module  # noqa: E402
from test_transfusion_assign_cpu import large_cases, lsap_cases  # noqa: E402

from bevfusion_b200 import _C, iou3d  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200 import transfusion_assign as TA  # noqa: E402
from bevfusion_b200.head_targets import pad_gt  # noqa: E402

pytestmark = pytest.mark.gpu
CFG, CODER = S.TRANSFUSION_TRAIN_CFG, S.TRANSFUSION_CODER
# Largest |native cost - restatement| allowed (costs are O(1)), and largest |ious - restatement|.  The
# restatement's IoU3D is float64, so both bound the kernel's fp32 overlap error (measured on an H100: 9e-8 and
# 4e-7 on these batches).
COST_TOL = 1e-6
IOU_TOL = 1e-6


def batch_solve(mats, dev, R=None, C=None):
    R = R or max(m.shape[0] for m in mats)
    C = C or max(m.shape[1] for m in mats)
    cost = np.full((len(mats), R, C), 7.0, np.float32)       # padding must not leak into a segment
    for s, m in enumerate(mats):
        cost[s, :m.shape[0], :m.shape[1]] = m
    rc = torch.tensor([m.shape[0] for m in mats], dtype=torch.int32, device=dev)
    cc = torch.tensor([m.shape[1] for m in mats], dtype=torch.int32, device=dev)
    c4r, r4c, st, steps = TA.linear_sum_assignment_batched(torch.from_numpy(cost).to(dev), rc, cc, True, True)
    return c4r.cpu().numpy(), r4c.cpu().numpy(), st.cpu().numpy(), steps.cpu().numpy()


def check_against_scipy(mats, c4r, r4c, st):
    for s, m in enumerate(mats):
        a, b = linear_sum_assignment(m)
        rows = np.nonzero(c4r[s] >= 0)[0]
        assert st[s] == 0
        assert np.array_equal(rows, a) and np.array_equal(c4r[s][rows], b), (s, m.shape)
        assert (c4r[s][m.shape[0]:] == -1).all() and (r4c[s][m.shape[1]:] == -1).all()
        cols = np.nonzero(r4c[s] >= 0)[0]
        assert len(cols) == len(rows) and np.array_equal(c4r[s][r4c[s][cols]], cols)


# ---- the solver ------------------------------------------------------------------------------------------------

def test_solver_equals_scipy_small(cuda):
    mats = list(lsap_cases(0, 3000))
    c4r, r4c, st, _ = batch_solve(mats, cuda)          # 3000 segments of 1..11 x 1..11 in one call
    check_against_scipy(mats, c4r, r4c, st)


def test_solver_equals_scipy_large_and_steps(cuda):
    mats = list(large_cases())
    c4r, r4c, st, steps = batch_solve(mats, cuda)
    check_against_scipy(mats, c4r, r4c, st)
    for s, m in enumerate(mats):
        assert steps[s] == lsap_oracle.solve_matching(m)[2]


def test_solver_mixed_sizes_and_wide(cuda):
    rng = np.random.default_rng(1)
    mats = [rng.standard_normal((8, 4096)).astype(np.float32), rng.integers(0, 3, (40, 4096)).astype(np.float32),
            rng.standard_normal((4096, 30)).astype(np.float32), rng.standard_normal((300, 1500)).astype(np.float32),
            rng.standard_normal((1, 1)).astype(np.float32), np.zeros((5, 0), np.float32)]
    for m in mats[:4]:                                          # one call each: the padding would be 4096^2
        c4r, r4c, st, _ = batch_solve([m], cuda)
        check_against_scipy([m], c4r, r4c, st)
    c4r, r4c, st, _ = batch_solve(mats[2:4], cuda)              # a CTA-wide segment next to another one
    check_against_scipy(mats[2:4], c4r, r4c, st)
    c4r, r4c, st, _ = batch_solve(mats[4:], cuda, R=8, C=8)     # an empty segment among others
    assert (c4r[1] == -1).all() and st[1] == 0


def test_solver_status(cuda):
    good = np.arange(6, dtype=np.float32).reshape(2, 3)
    nan, ninf, inf = good.copy(), good.copy(), np.array([[np.inf, np.inf], [1, 2]], np.float32)
    nan[1, 2] = np.nan
    ninf[0, 0] = -np.inf
    c4r, _, st, _ = batch_solve([good, nan, ninf, inf], cuda)
    assert st.tolist() == [0, TA.STATUS["invalid_cost"], TA.STATUS["invalid_cost"], TA.STATUS["infeasible"]]
    assert (c4r[1:] == -1).all() and (c4r[0][:2] >= 0).all()


# ---- the reference restated on CUDA tensors --------------------------------------------------------------------

def ref_decode(pred, b):
    c, h, d, r = (pred[k][b].clone() for k in ("center", "height", "dim", "rot"))
    c[0] = c[0] * CODER["out_size_factor"] * CODER["voxel_size"][0] + CODER["pc_range"][0]
    c[1] = c[1] * CODER["out_size_factor"] * CODER["voxel_size"][1] + CODER["pc_range"][1]
    d = d.exp()
    h = h - d[2:3] * 0.5
    return torch.cat([c, h, d, torch.atan2(r[0:1], r[1:2])], 0).T


def ref_overlaps(a, b, bev_fn=None):
    """BaseInstance3DBoxes.overlaps(a, b), mode iou.  By default in float64 (nms_oracle.iou3d_matrix, on the fp32
    boxes), so that an error of this package's overlap shows up on one side only; with bev_fn, a BEV overlap op on
    xyxyr boxes, in fp32 torch over that op, as the reference computes it."""
    if bev_fn is None:
        return torch.from_numpy(O.iou3d_matrix(a.detach().cpu().numpy(), b.detach().cpu().numpy())).to(a.device)
    bev = bev_fn(iou3d.xywhr2xyxyr(a[:, [0, 1, 3, 4, 6]]).contiguous(),
                 iou3d.xywhr2xyxyr(b[:, [0, 1, 3, 4, 6]]).contiguous())
    top = torch.min((a[:, 2] + a[:, 5]).view(-1, 1), (b[:, 2] + b[:, 5]).view(1, -1))
    bottom = torch.max(a[:, 2].view(-1, 1), b[:, 2].view(1, -1))
    ov = bev * torch.clamp(top - bottom, min=0)
    va, vb = (a[:, 3] * a[:, 4] * a[:, 5]).view(-1, 1), (b[:, 3] * b[:, 4] * b[:, 5]).view(1, -1)
    return ov / torch.clamp(va + vb - ov, min=1e-8)


def ref_cost(boxes, logits, gt, gl, bev_fn=None):
    """HungarianAssigner3D.assign's cost (hungarian_assigner.py:100-113, mmdet FocalLossCost) on CUDA tensors, the
    IoU3D term from ref_overlaps (float64 unless bev_fn is given) rounded to fp32.  Returns (cost, iou)."""
    p = logits.T.sigmoid()
    neg = -(1 - p + 1e-12).log() * (1 - 0.25) * p.pow(2.0)
    pos = -(p + 1e-12).log() * 0.25 * (1 - p).pow(2.0)
    cls = (pos[:, gl] - neg[:, gl]) * 0.15
    start = boxes.new(CFG["point_cloud_range"][0:2])
    span = boxes.new(CFG["point_cloud_range"][3:5]) - boxes.new(CFG["point_cloud_range"][0:2])
    reg = torch.cdist((boxes[:, :2] - start) / span, (gt[:, :2] - start) / span, p=1) * 0.25
    iou = ref_overlaps(boxes, gt, bev_fn)
    return cls + reg + (-iou.float()) * 0.25, iou


def ref_encode(g):
    t = torch.zeros([g.shape[0], 10], device=g.device)
    t[:, 0] = (g[:, 0] - CODER["pc_range"][0]) / (CODER["out_size_factor"] * CODER["voxel_size"][0])
    t[:, 1] = (g[:, 1] - CODER["pc_range"][1]) / (CODER["out_size_factor"] * CODER["voxel_size"][1])
    t[:, 3], t[:, 4], t[:, 5] = g[:, 3].log(), g[:, 4].log(), g[:, 5].log()
    t[:, 2] = g[:, 2] + g[:, 5] * 0.5
    t[:, 6], t[:, 7] = torch.sin(g[:, 6]), torch.cos(g[:, 6])
    t[:, 8:10] = g[:, 7:]
    return t


def ref_get_targets(gts, labels, pred, P):
    """transfusion.py:357-525 with HungarianAssigner3D and scipy, per sample, on CUDA tensors."""
    B, N = pred["heatmap"].shape[0], pred["heatmap"].shape[2]
    res = dict(labels=[], label_weights=[], bbox_targets=[], bbox_weights=[], ious=[], num_pos=[], mean_iou=[],
               gt_inds=[], cost=[])
    for b in range(B):
        boxes, gt, gl = ref_decode(pred, b), gts[b], labels[b]
        gt_inds = torch.zeros(N, dtype=torch.long, device=gt.device)
        ious = torch.zeros(N, device=gt.device)
        for layer in range(N // P):
            sl = slice(layer * P, (layer + 1) * P)
            if len(gt) == 0:
                res["cost"].append(None)
                continue
            cost, iou = ref_cost(boxes[sl], pred["heatmap"][b][:, sl], gt, gl)
            res["cost"].append(cost)
            r, c = linear_sum_assignment(cost.detach().cpu())
            r, c = torch.from_numpy(r).to(gt.device), torch.from_numpy(c).to(gt.device)
            gt_inds[r + layer * P] = c + 1
            ious[r + layer * P] = torch.clamp(iou[r, c], 0, 1).float()
        pos = torch.nonzero(gt_inds > 0).squeeze(1)
        lab = torch.full((N,), 10, dtype=torch.long, device=gt.device)
        bt = torch.zeros((N, 10), device=gt.device)
        bw = torch.zeros((N, 10), device=gt.device)
        if len(pos):
            bt[pos] = ref_encode(gt[gt_inds[pos] - 1])
            bw[pos] = 1.0
            lab[pos] = gl[gt_inds[pos] - 1]
        for k, v in (("labels", lab), ("label_weights", torch.ones(N, dtype=torch.long, device=gt.device)),
                     ("bbox_targets", bt), ("bbox_weights", bw), ("ious", ious), ("gt_inds", gt_inds)):
            res[k].append(v)
        res["num_pos"].append(len(pos))
        res["mean_iou"].append(float(ious[pos].sum() / max(len(pos), 1)))
    return res


def make_batch(seed, B, L, dev, P=200, min_boxes=40, max_boxes=120):
    gb, gl = S.gt_boxes(seed=seed, batch=B, min_boxes=min_boxes, max_boxes=max_boxes)
    pred = S.transfusion_predictions(seed + 100, B, (gb, gl), num_proposals=P, num_classes=10, layers=L)
    return [b.to(dev) for b in gb], [l.to(dev) for l in gl], {k: v.to(dev) for k, v in pred.items()}


def run_batched(gts, labels, pred, P, extras=True):
    boxes, lab, counts = pad_gt(gts, labels)
    return TA.transfusion_assign_batched(pred, boxes, lab, counts, 10, P, CFG, CODER, return_extras=extras)


def ulp_diff(a, b):
    a, b = a.cpu().numpy().astype(np.float32), b.cpu().numpy().astype(np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


# ---- cost, solver in the pipeline, end to end ----------------------------------------------------------------

@pytest.mark.parametrize("B,L", [(1, 1), (4, 1), (1, 2), (4, 2)])
def test_end_to_end_against_reference_loop(cuda, B, L):
    gts, labels, pred = make_batch(10 * B + L, B, L, cuda)
    out, ex = run_batched(gts, labels, pred, 200)
    ref = ref_get_targets(gts, labels, pred, 200)
    got_inds = ex["gt_inds"].cpu().numpy()
    want_inds = torch.stack(ref["gt_inds"]).cpu().numpy()
    differing, worst = 0, 0.0
    for s in range(B * L):
        b, layer = divmod(s, L)
        G = len(gts[b])
        cost = ex["cost"][s, :, :G]
        rc = ref["cost"][s]
        assert torch.isfinite(cost).all()
        worst = max(worst, (cost - rc).abs().max().item())
        # the solver in the pipeline: scipy on the call's own matrix gives the call's assignment
        r, c = linear_sum_assignment(cost.cpu().numpy())
        sl = slice(layer * 200, (layer + 1) * 200)
        mine = np.zeros(200, np.int64)
        mine[r] = c + 1
        assert np.array_equal(mine, got_inds[b, sl])
        if not np.array_equal(got_inds[b, sl], want_inds[b, sl]):   # allowed only at equal total cost
            differing += 1
            c64 = rc.double().cpu().numpy()
            tot = lambda ind: sum(c64[p, g - 1] for p, g in enumerate(ind) if g > 0)   # noqa: E731
            assert abs(tot(got_inds[b, sl]) - tot(want_inds[b, sl])) <= COST_TOL * G
    same = torch.from_numpy((got_inds == want_inds).all(1)).to(cuda)
    ious_err = (out[4][same] - torch.stack(ref["ious"])[same]).abs().max().item()
    print("segments whose assignment differs from the reference's at equal cost: %d of %d; largest |cost - "
          "restatement| %.3g, |ious - restatement| %.3g" % (differing, B * L, worst, ious_err))
    assert worst <= COST_TOL
    for k in ("labels", "label_weights", "bbox_weights"):
        assert torch.equal(out[["labels", "label_weights", "bbox_targets", "bbox_weights"].index(k)][same],
                           torch.stack(ref[k])[same]), k
    assert out[5].cpu().tolist() == ref["num_pos"]
    assert ulp_diff(out[2][same], torch.stack(ref["bbox_targets"])[same]).max() <= 2
    assert ious_err <= IOU_TOL
    assert np.abs(out[6].cpu().numpy() - np.array(ref["mean_iou"]))[same.cpu().numpy()].max(initial=0) <= IOU_TOL
    assert (out[7] == 0).all()


def test_cost_against_reference_iou3d_op(cuda):
    ref = ref_module("iou3d_cuda_ref")
    if ref is None:
        pytest.skip("oracle/_ref has no reference iou3d_cuda build")

    def ref_bev(a, b):
        out = torch.zeros((a.shape[0], b.shape[0]), device=a.device)
        ref.boxes_overlap_bev_gpu(a, b, out)
        return out

    gts, labels, pred = make_batch(77, 2, 1, cuda)
    _, ex = run_batched(gts, labels, pred, 200)
    worst = 0.0
    for b in range(2):
        rc, _ = ref_cost(ref_decode(pred, b), pred["heatmap"][b], gts[b], labels[b], ref_bev)
        worst = max(worst, (ex["cost"][b, :, :len(gts[b])] - rc).abs().max().item())
    print("largest |cost - cost with the reference's iou3d_cuda|: %.3g" % worst)
    assert worst <= 1e-3


def test_encode_division_is_torch_cuda_division(cuda):
    """Which division torch applies to (x - pc) / (osf * vs) on CUDA, and that the call matches it bit for bit."""
    gts, labels, pred = make_batch(5, 1, 1, cuda)
    out, ex = run_batched(gts, labels, pred, 200)
    g = gts[0]
    torch_div = (g[:, 0] - CODER["pc_range"][0]) / (CODER["out_size_factor"] * CODER["voxel_size"][0])
    inv = np.float32(1) / np.float32(CODER["out_size_factor"] * CODER["voxel_size"][0])
    recip = (g[:, 0] - CODER["pc_range"][0]) * float(inv)
    print("torch divides by a Python float on CUDA as a multiply by the fp32 reciprocal:",
          bool(torch.equal(torch_div, recip)))
    pos = ex["gt_inds"][0] > 0
    assert torch.equal(out[2][0][pos][:, 0], torch_div[ex["gt_inds"][0][pos] - 1])


# ---- edge cases ------------------------------------------------------------------------------------------------

def test_edges_empty_transposed_square_duplicates(cuda):
    gb, gl = S.gt_boxes(seed=3, batch=4, min_boxes=40, max_boxes=60)
    gb[1], gl[1] = gb[1][:0], gl[1][:0]                                 # empty sample
    g2, l2 = S.gt_boxes(seed=4, batch=2, min_boxes=64, max_boxes=80)
    gb[2], gl[2] = g2[0][:64], l2[0][:64]                               # G = P
    gb[3], gl[3] = g2[1][:80], l2[1][:80]                               # G > P
    P = 64
    pred = S.transfusion_predictions(9, 4, (gb, gl), num_proposals=P, num_classes=10, layers=2)
    gts, labels = [b.to(cuda) for b in gb], [l.to(cuda) for l in gl]
    pred = {k: v.to(cuda) for k, v in pred.items()}
    out, ex = run_batched(gts, labels, pred, P)
    assert out[5].cpu().tolist()[1] == 0 and (out[0][1] == 10).all() and (out[3][1] == 0).all()
    assert out[5].cpu().tolist()[2:] == [2 * P, 2 * P]
    assert (out[7] == 0).all()
    ref = ref_get_targets(gts, labels, pred, P)
    for s in range(8):
        b, layer = divmod(s, 2)
        if not len(gts[b]):
            continue
        r, c = linear_sum_assignment(ex["cost"][s, :, :len(gts[b])].cpu().numpy())
        mine = np.zeros(P, np.int64)
        mine[r] = c + 1
        assert np.array_equal(mine, ex["gt_inds"][b, layer * P:(layer + 1) * P].cpu().numpy())
        assert (ex["cost"][s, :, :len(gts[b])] - ref["cost"][s]).abs().max().item() <= COST_TOL


def test_nan_prediction_and_bad_label(cuda):
    gts, labels, pred = make_batch(21, 3, 1, cuda)
    pred["center"][1, 0, 17] = float("nan")
    labels[2] = labels[2].clone()
    labels[2][3] = 10
    out, _ = run_batched(gts, labels, pred, 200)
    st = out[7].cpu().tolist()
    assert st[0] == 0 and st[1] == TA.STATUS["invalid_cost"]
    assert st[2] & TA.STATUS["bad_label"]
    assert out[5].cpu().tolist()[1:] == [0, 0] and out[5].cpu().tolist()[0] > 0
    with pytest.raises(ValueError):
        TA.transfusion_targets(gts, labels, pred, 10, 200, CFG, CODER)


# ---- behaviour -------------------------------------------------------------------------------------------------

def test_reproducible_and_list_equals_batched(cuda):
    gts, labels, pred = make_batch(31, 4, 2, cuda)
    a = run_batched(gts, labels, pred, 200, extras=False)
    b = run_batched(gts, labels, pred, 200, extras=False)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    lst = TA.transfusion_targets([g.cpu() for g in gts], labels, [pred], 10, 200, CFG, CODER)
    for i in range(5):
        assert torch.equal(lst[i], a[i])
    assert lst[5] == int(a[5].sum())
    assert lst[6] == float(np.mean([float(v) for v in a[6].cpu()]))
    from bevfusion_b200.head_targets import transfusion_heatmap_targets
    assert torch.equal(lst[7], transfusion_heatmap_targets(gts, labels, 10, CFG))


def test_cuda_graph_replay_on_other_counts(cuda):
    B, P, nmax = 4, 200, 120
    shapes = [[40, 120, 77, 0], [120, 1, 60, 99], [55, 56, 57, 58], [90, 0, 0, 120]]
    batches = [make_batch(50 + i, B, 1, cuda, min_boxes=nmax, max_boxes=nmax) for i in range(4)]
    static_boxes = torch.zeros((B, nmax, 9), device=cuda)
    static_labels = torch.zeros((B, nmax), dtype=torch.int32, device=cuda)
    static_counts = torch.zeros((B,), dtype=torch.int32, device=cuda)
    static_pred = {k: v.clone() for k, v in batches[0][2].items()}

    def load(i):
        gts, labels, pred = batches[i]
        gts = [g[:n] for g, n in zip(gts, shapes[i])]
        labels = [l[:n] for l, n in zip(labels, shapes[i])]
        boxes, lab, counts = pad_gt(gts, labels)
        static_boxes.zero_()
        static_labels.zero_()
        static_boxes[:, :boxes.shape[1]] = boxes
        static_labels[:, :lab.shape[1]] = lab
        static_counts.copy_(counts)
        for k in static_pred:
            static_pred[k].copy_(pred[k])

    load(0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        TA.transfusion_assign_batched(static_pred, static_boxes, static_labels, static_counts, 10, P, CFG, CODER)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        static_out = TA.transfusion_assign_batched(static_pred, static_boxes, static_labels, static_counts, 10, P,
                                                   CFG, CODER)
    for i in (1, 2, 3):
        load(i)
        g.replay()
        eager = TA.transfusion_assign_batched(static_pred, static_boxes, static_labels, static_counts, 10, P, CFG,
                                              CODER)
        for x, y in zip(static_out, eager):
            assert torch.equal(x, y)
        assert static_out[5].cpu().tolist() == [min(n, P) for n in shapes[i]]


def test_launch_count_and_no_host_copy(cuda):
    gts, labels, pred = make_batch(61, 4, 1, cuda)
    boxes, lab, counts = pad_gt(gts, labels)
    pred = {k: v.contiguous() for k, v in pred.items()}
    TA.transfusion_assign_batched(pred, boxes, lab, counts, 10, 200, CFG, CODER)
    torch.cuda.synchronize()
    n0 = _C.launch_count()
    TA.transfusion_assign_batched(pred, boxes, lab, counts, 10, 200, CFG, CODER)
    assert _C.launch_count() - n0 == 3
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        TA.transfusion_assign_batched(pred, boxes, lab, counts, 10, 200, CFG, CODER)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert not any("DtoH" in n or "Device -> Host" in n for n in names)
    for k in ("tf_cost_kernel", "lsap_kernel", "tf_targets_kernel"):
        assert sum(k in n for n in names) >= 1, k


def test_hungarian_assigner_mirror(cuda):
    gts, labels, pred = make_batch(71, 1, 1, cuda)
    boxes = ref_decode(pred, 0)
    res = TA.HungarianAssigner3D(cls_cost=dict(type="FocalLossCost", gamma=2.0, alpha=0.25, weight=0.15),
                                 reg_cost=dict(type="BBoxBEVL1Cost", weight=0.25),
                                 iou_cost=dict(type="IoU3DCost", weight=0.25)).assign(
        boxes, gts[0], labels[0], pred["heatmap"][0:1], CFG)
    cost, iou = ref_cost(boxes, pred["heatmap"][0], gts[0], labels[0])
    r, c = linear_sum_assignment(cost.cpu().numpy())
    want = np.zeros(200, np.int64)
    want[r] = c + 1
    assert res.num_gts == len(gts[0])
    assert np.array_equal(res.gt_inds.cpu().numpy(), want)
    lab = np.full(200, -1)
    lab[r] = labels[0].cpu().numpy()[c]
    assert np.array_equal(res.labels.cpu().numpy(), lab)
    mo = np.zeros(200, np.float32)
    mo[r] = iou.cpu().numpy()[r, c]
    print("largest |max_overlaps - float64 restatement|: %.3g" % np.abs(res.max_overlaps.cpu().numpy() - mo).max())
    assert np.abs(res.max_overlaps.cpu().numpy() - mo).max() <= IOU_TOL
    empty = TA.HungarianAssigner3D().assign(boxes, gts[0][:0], labels[0][:0], pred["heatmap"][0:1], CFG)
    assert empty.max_overlaps is None and (empty.gt_inds == 0).all()
