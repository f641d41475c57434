"""The head losses on the H100: head_losses.centerhead_loss / transfusion_loss against the float64 restatement
(head_losses_oracle, clamp decisions taken from the device's fp32 sigmoid), against the fixture written by the
reference's own loss methods, and against the reference's lines restated on CUDA fp32 tensors under autograd;
edge cases, determinism, launch counts, the absence of synchronising calls and one CUDA graph of targets + loss +
backward."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "golden"))
import head_losses_oracle as O  # noqa: E402
from bevfusion_b200 import _C  # noqa: E402
from bevfusion_b200 import head_losses as HL  # noqa: E402
from bevfusion_b200 import head_targets as HT  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200.transfusion_assign import transfusion_assign_batched  # noqa: E402
from make_head_losses_golden import FocalLoss, GaussianFocalLoss, L1Loss  # noqa: E402  (the restated mmdet losses)
from test_head_losses_cpu import golden_centerhead, golden_transfusion, GOLDEN, CH_KEYS, TF_KEYS  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
CW = [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.2, 0.2]
LOSS_RTOL, GRAD_TOL = 2e-6, 1e-5
TASKS = [[n for n, _ in c] for c in S.CENTERHEAD_TASKS]


def ch_cfg(H):
    extent = 54.0
    return dict(point_cloud_range=[-extent, -extent, -5.0, extent, extent, 3.0], grid_size=[H * 8, H * 8, 1],
                voxel_size=[2 * extent / H / 8, 2 * extent / H / 8, 0.2], out_size_factor=8, dense_reg=1,
                gaussian_overlap=0.1, max_objs=500, min_radius=2, code_weights=CW)


def gt_padded(seed, B, code=10):
    boxes, labels = S.gt_boxes(seed=seed, batch=B)
    if code == 8:
        boxes = [b[:, :7].contiguous() for b in boxes]
    return HT.pad_gt([b.to(DEV) for b in boxes], [l.to(DEV) for l in labels])


def ch_inputs(seed, B, H, code=10, dtype=torch.float32):
    gt = S.gt_boxes(seed=seed, batch=B)
    outs = S.centerhead_head_outputs(seed, B, height=H, width=H, gt=gt)
    preds = [[{k: v.to(DEV, dtype).requires_grad_() for k, v in t.items() if code == 10 or k != "vel"}] for t in outs]
    targets = HT.centerhead_targets_batched(*gt_padded(seed, B, code), TASKS, ch_cfg(H))
    return preds, targets


def np64(t):
    return t.detach().double().cpu().numpy()


def dev_sigmoid(x):
    return torch.sigmoid(x.detach().float()).cpu().numpy()


def check_losses(got, want, rtol=LOSS_RTOL):
    assert list(got) == list(want)
    for k in want:
        g = float(got[k])
        if np.isnan(want[k]):
            assert np.isnan(g), k
        else:
            assert abs(g - want[k]) <= rtol * abs(want[k]) + 1e-30, (k, g, want[k])


def check_grad(got, want, tol=GRAD_TOL, name="", floor=0.0):
    """Within tol of the largest |want|, zero exactly where want is (|want| <= floor: the float64 fixture keeps
    gradients of 1e-87 at logits of -100 whose fp32 sigmoid, the reference's on CUDA, is exactly 0)."""
    got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else got
    scale = max(np.abs(want).max(), 1e-30)
    assert np.abs(got - want).max() <= tol * scale, (name, np.abs(got - want).max(), scale)
    np.testing.assert_array_equal(got == 0, np.abs(want) <= floor, err_msg=name + ": zero set")


def run_ch(preds, targets, lw=(1.0, 0.25), **kw):
    losses = HL.centerhead_loss(preds, targets, dict(code_weights=CW[:targets[1][0].shape[-1]]),
                                loss_cls=dict(type="GaussianFocalLoss", loss_weight=lw[0]),
                                loss_bbox=dict(type="L1Loss", loss_weight=lw[1]), **kw)
    return losses


def ch_oracle(preds, targets, lw=(1.0, 0.25)):
    P = [{k: np64(v) for k, v in p[0].items()} for p in preds]
    T = tuple([np64(x) for x in lst] for lst in targets)
    y32 = [dev_sigmoid(p[0]["heatmap"]) for p in preds]
    return O.centerhead(P, T, CW[:T[1][0].shape[-1]], cls=(lw[0], 2.0, 4.0), bbox_lw=lw[1], y32=y32)


@pytest.mark.parametrize("B,H,code,lw", [(1, 128, 10, (1.0, 0.25)), (4, 128, 8, (1.5, 0.4)),
                                         (1, 180, 10, (1.0, 0.25)), (4, 180, 10, (0.7, 0.25))])
def test_centerhead_matches_oracle(B, H, code, lw):
    preds, targets = ch_inputs(B * 7 + H, B, H, code)
    losses = run_ch(preds, targets, lw)
    sum(losses.values()).backward()
    want, wgrad = ch_oracle(preds, targets, lw)
    check_losses(losses, want)
    for t, p in enumerate(preds):
        for k, v in p[0].items():
            check_grad(v.grad, wgrad[t][k], name="task%d %s" % (t, k))


def reference_centerhead_lines(preds, targets, lw=(1.0, 0.25)):
    """centerpoint.py:596-634 on CUDA fp32 tensors, with the restated mmdet losses and the reference's .item()."""
    heatmaps, anno_boxes, inds, masks = targets
    loss_cls, loss_bbox = GaussianFocalLoss(loss_weight=lw[0]), L1Loss(loss_weight=lw[1])
    out = {}
    for task_id, pd in enumerate(preds):
        p = pd[0]
        hm = torch.clamp(p["heatmap"].sigmoid(), min=1e-4, max=1 - 1e-4)
        num_pos = heatmaps[task_id].eq(1).float().sum().item()
        out["heatmap/task%d" % task_id] = loss_cls(hm, heatmaps[task_id], avg_factor=max(num_pos, 1))
        target_box = anno_boxes[task_id]
        keys = ["reg", "height", "dim", "rot"] + (["vel"] if "vel" in p else [])
        pred = torch.cat([p[k] for k in keys], dim=1).permute(0, 2, 3, 1).contiguous()
        pred = pred.view(pred.size(0), -1, pred.size(3))
        ind = inds[task_id]
        pred = pred.gather(1, ind.unsqueeze(2).expand(ind.size(0), ind.size(1), pred.size(2)))
        num = masks[task_id].float().sum()
        mask = masks[task_id].unsqueeze(2).expand_as(target_box).float()
        mask *= (~torch.isnan(target_box)).float()
        bbox_weights = mask * mask.new_tensor(CW[:target_box.shape[-1]])
        out["bbox/task%d" % task_id] = loss_bbox(pred, target_box, bbox_weights, avg_factor=(num + 1e-4))
    return out


@pytest.mark.parametrize("B", [1, 4])
def test_centerhead_matches_reference_lines_on_cuda(B):
    preds, targets = ch_inputs(31 + B, B, 128)
    losses = run_ch(preds, targets)
    sum(losses.values()).backward()
    ref_preds = [[{k: v.detach().clone().requires_grad_() for k, v in p[0].items()}] for p in preds]
    ref = reference_centerhead_lines(ref_preds, targets)
    sum(ref.values()).backward()
    check_losses(losses, {k: float(v) for k, v in ref.items()}, 2e-6)
    for p, r in zip(preds, ref_preds):
        for k in p[0]:
            check_grad(p[0][k].grad, np64(r[0][k].grad), name=k)


def test_centerhead_matches_reference_fixture():
    g = np.load(GOLDEN)
    for name in ("ch", "chw"):
        preds, targets, grads, want = golden_centerhead(g, name)
        lw = tuple(g[name + "_lw"])
        P = [[{k: torch.tensor(v, device=DEV).requires_grad_() for k, v in p.items()}] for p in preds]
        T = ([torch.tensor(x, device=DEV) for x in targets[0]], [torch.tensor(x, device=DEV) for x in targets[1]],
             [torch.tensor(x, device=DEV) for x in targets[2]], [torch.tensor(x, device=DEV) for x in targets[3]])
        losses = run_ch(P, T, lw)
        sum(losses.values()).backward()
        # the fixture clamps at float64's 1e-4 / 1 - 1e-4, the device at their fp32 values: 2e-5 covers the saturated
        # cells (1 - fp32(1 - 1e-4) is 1.7e-4 relative away from 1e-4); against the oracle the tolerance is 2e-6
        check_losses(losses, want, 2e-5)
        for t in range(len(P)):
            for k in CH_KEYS:
                check_grad(P[t][0][k].grad, grads[t][k], name="%s task%d %s" % (name, t, k), floor=1e-38)


def test_centerhead_edges():
    B, H = 2, 128
    preds, targets = ch_inputs(5, B, H)
    heatmaps, annos, inds, masks = [list(x) for x in targets]
    # task 0: empty ground truth; task 1: duplicate inds, a NaN target on a masked-out slot, a target 1 ulp below 1;
    # task 2: logits at the clamp bounds and saturated
    heatmaps[0] = torch.zeros_like(heatmaps[0])
    masks[0] = torch.zeros_like(masks[0])
    inds[1] = inds[1].clone()
    masks[1] = masks[1].clone()
    inds[1][:, 1] = inds[1][:, 0]
    masks[1][:, :2] = 1
    annos[1] = annos[1].clone()
    annos[1][0, 499, 3] = float("nan")
    masks[1][0, 499] = 0
    heatmaps[1] = heatmaps[1].clone()
    heatmaps[1][0, 0, 0, :4] = torch.tensor([1.0, np.nextafter(np.float32(1), np.float32(0)), 1.0, 0.5])
    xs, ys = O.boundary_logits(lambda x: torch.sigmoid(torch.from_numpy(np.asarray(x, np.float32)).to(DEV)).cpu()
                               .numpy())
    assert (ys == np.float32(O.HI)).any() and (ys < np.float32(O.LO)).any() and (ys > np.float32(O.HI)).any()
    with torch.no_grad():
        h = preds[2][0]["heatmap"]
        h[0, 0, 0, :len(xs)] = torch.from_numpy(xs).to(DEV)
        h[0, 0, 1, :4] = torch.tensor([100.0, -100.0, 100.0, -100.0])
    targets = (heatmaps, annos, inds, masks)
    losses = run_ch(preds, targets)
    assert float(losses["bbox/task0"]) == 0.0 and np.isfinite(float(losses["heatmap/task0"]))
    assert np.isnan(float(losses["bbox/task1"]))
    finite = {k: v for k, v in losses.items() if k != "bbox/task1"}
    sum(finite.values()).backward()
    want, wgrad = ch_oracle(preds, targets)
    check_losses({k: v for k, v in losses.items() if k != "bbox/task1"},
                 {k: v for k, v in want.items() if k != "bbox/task1"})
    assert float(losses["heatmap/task0"]) == pytest.approx(want["heatmap/task0"], rel=2e-6)   # avg factor 1
    for t, p in enumerate(preds):
        for k, v in p[0].items():
            if t != 1 or k == "heatmap":
                check_grad(v.grad, wgrad[t][k], name="task%d %s" % (t, k))
    g = preds[2][0]["heatmap"].grad[0, 0, 0, :len(xs)].cpu().numpy()
    np.testing.assert_array_equal(g == 0, (ys < np.float32(O.LO)) | (ys > np.float32(O.HI)))
    # duplicate cells add: the bbox gradient of task 1 alone, against the oracle
    for p in preds:
        for v in p[0].values():
            v.grad = None
    losses = run_ch(preds, targets)
    losses["bbox/task1"].backward()
    for k in ("reg", "height", "dim", "rot", "vel"):
        check_grad(preds[1][0][k].grad, wgrad[1][k], name="dup " + k)


def test_centerhead_fp16_predictions():
    preds, targets = ch_inputs(11, 2, 128, dtype=torch.float16)
    losses = run_ch(preds, targets)
    sum(losses.values()).backward()
    want, wgrad = ch_oracle(preds, targets)
    check_losses(losses, want)
    for t, p in enumerate(preds):
        for k, v in p[0].items():
            assert v.grad.dtype == torch.float16
            w = wgrad[t][k]
            assert np.abs(v.grad.double().cpu().numpy() - w).max() <= 1e-3 * np.abs(w).max() + 1e-7


def test_centerhead_status_and_refusals():
    preds, targets = ch_inputs(3, 1, 128)
    inds = [i.clone() for i in targets[2]]
    masks = [m.clone() for m in targets[3]]
    inds[0][0, 0], masks[0][0, 0] = 128 * 128, 1
    inds[1][0, 1], masks[1][0, 1] = -5, 0
    _, status = run_ch(preds, (targets[0], targets[1], inds, masks), return_status=True)
    assert int(status) == HL.STATUS["bad_ind"]
    _, status = run_ch(preds, targets, return_status=True)
    assert int(status) == 0
    with pytest.raises(ValueError):
        run_ch(preds, (targets[0][:-1], targets[1], targets[2], targets[3]))
    with pytest.raises(ValueError):
        HL.centerhead_loss(preds, targets, dict(code_weights=CW[:9]))
    bad = [[dict(p[0], reg=p[0]["reg"][:, :1])] for p in preds]
    with pytest.raises(ValueError):
        run_ch(bad, targets)
    with pytest.raises(RuntimeError, match="CUDA"):
        run_ch([[{k: v.detach().cpu() for k, v in p[0].items()}] for p in preds], targets)


def test_centerhead_deterministic_launches_and_no_sync():
    preds, targets = ch_inputs(9, 4, 128)
    _C.reset_launch_count()
    a = run_ch(preds, targets)
    assert _C.launch_count() == 2
    with torch.autograd.set_multithreading_enabled(False):   # the launch counter is per host thread
        sum(a.values()).backward()
    assert _C.launch_count() == 4
    g1 = [v.grad.clone() for p in preds for v in p[0].values()]
    for p in preds:
        for v in p[0].values():
            v.grad = None
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = run_ch(preds, targets)
        sum(b.values()).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert all(torch.equal(a[k], b[k]) for k in a)
    g2 = [v.grad for p in preds for v in p[0].values()]
    assert all(torch.equal(x, y) for x, y in zip(g1, g2))


# ---- TransFusion --------------------------------------------------------------------------------------------
TF_CODER = dict(S.TRANSFUSION_CODER)


def tf_inputs(seed, B, H, L=2, code=10, dtype=torch.float32):
    gt = S.gt_boxes(seed=seed, batch=B)
    P = 200
    pr = S.transfusion_predictions(seed, B, gt, num_proposals=P, num_classes=10, layers=L)
    pr["dense_heatmap"] = S.transfusion_heatmap(seed, B, num_classes=10, height=H, width=H, gt=gt)
    preds = {k: v.to(DEV, dtype).requires_grad_() for k, v in pr.items() if code == 10 or k != "vel"}
    boxes, labels, counts = gt_padded(seed, B, code)
    cfg = dict(S.TRANSFUSION_TRAIN_CFG, grid_size=[H * 8, H * 8, 1], code_weights=CW[:code])
    coder = dict(TF_CODER, code_size=code)
    assign = transfusion_assign_batched({k: v.detach() for k, v in preds.items()}, boxes, labels, counts, 10, P,
                                        cfg, coder)
    heat = HT.transfusion_heatmap_targets_batched(boxes, labels, counts, 10, cfg)
    return preds, tuple(assign) + (heat,), cfg, P


def run_tf(preds, targets, P, L, aux, cfg, lw=(1.0, 1.0, 0.25), **kw):
    return HL.transfusion_loss([[preds]], targets, P, L, aux, cfg,
                               loss_cls=dict(type="FocalLoss", use_sigmoid=True, gamma=2.0, alpha=0.25,
                                             loss_weight=lw[1]),
                               loss_bbox=dict(type="L1Loss", loss_weight=lw[2]),
                               loss_heatmap=dict(type="GaussianFocalLoss", loss_weight=lw[0]), **kw)


def tf_oracle(preds, targets, P, L, aux, lw=(1.0, 1.0, 0.25)):
    labels, lweights, bt, bw, _, num_pos, mean_iou, _, heat = targets
    pn = {k: np64(v) for k, v in preds.items()}
    T = (np64(labels).astype(np.int64), np64(lweights), np64(bt), np64(bw), int(num_pos.sum()),
         list(np64(mean_iou)), np64(heat))
    return O.transfusion(pn, T, P, L, aux, CW[:bt.shape[-1]], heat=(lw[0], 2.0, 4.0), cls=(lw[1], 0.25, 2.0),
                         bbox_lw=lw[2], y32=dev_sigmoid(preds["dense_heatmap"]))


@pytest.mark.parametrize("B,H,code,aux,lw", [(1, 128, 10, True, (1.0, 1.0, 0.25)), (4, 180, 10, True, (1.0, 1.0, 0.25)),
                                             (4, 180, 8, False, (2.0, 0.5, 0.3)), (1, 180, 10, False, (1.0, 1.0, 0.25))])
def test_transfusion_matches_oracle(B, H, code, aux, lw):
    preds, targets, cfg, P = tf_inputs(B * 3 + H, B, H, code=code)
    losses = run_tf(preds, targets, P, 2, aux, cfg, lw)
    sum(v for k, v in losses.items() if k != "matched_ious").backward()
    want, wgrad = tf_oracle(preds, targets, P, 2, aux, lw)
    check_losses(losses, want)
    for k, v in preds.items():
        check_grad(v.grad, wgrad[k], name=k)


def test_transfusion_matches_reference_fixture():
    g = np.load(GOLDEN)
    for name in ("tf_aux", "tf_last"):
        preds, targets, grads, want, P, L, aux = golden_transfusion(g, name)
        pd = {k: torch.tensor(v, device=DEV).requires_grad_() for k, v in preds.items()}
        labels, lweights, bt, bw, num_pos, mious, hm = targets
        T = (torch.tensor(labels, device=DEV), torch.tensor(lweights, device=DEV),
             torch.tensor(bt, device=DEV, dtype=torch.float32), torch.tensor(bw, device=DEV, dtype=torch.float32),
             None, num_pos, mious[0], torch.tensor(hm, device=DEV))
        losses = run_tf(pd, T, P, L, aux, dict(code_weights=CW))
        sum(v for k, v in losses.items() if k != "matched_ious").backward()
        check_losses(losses, want, 2e-5)
        for k in TF_KEYS:
            check_grad(pd[k].grad, grads[k], name="%s %s" % (name, k), floor=1e-38)


def test_transfusion_background_weights_and_status():
    preds, targets, cfg, P = tf_inputs(17, 2, 128)
    labels, lweights = targets[0], targets[1]
    gen = torch.Generator(device="cpu").manual_seed(0)
    bg = (torch.full_like(labels, 10), torch.randint(0, 2, lweights.shape, generator=gen).to(DEV)) + targets[2:]
    losses = run_tf(preds, bg, P, 2, True, cfg)
    sum(v for k, v in losses.items() if k != "matched_ious").backward()
    want, wgrad = tf_oracle(preds, bg, P, 2, True)
    check_losses(losses, want)
    for k, v in preds.items():
        check_grad(v.grad, wgrad[k], name=k)
    bad = labels.clone()
    bad[0, 3] = 11
    _, status = run_tf(preds, (bad,) + targets[1:], P, 2, True, cfg, return_status=True)
    assert int(status) == HL.STATUS["bad_label"]
    with pytest.raises(ValueError):
        run_tf(preds, targets, 150, 2, True, cfg)
    with pytest.raises(ValueError):
        run_tf(dict(preds, rot=preds["rot"][:, :1]), targets, P, 2, True, cfg)


def test_transfusion_fp16_and_saturated():
    preds, targets, cfg, P = tf_inputs(23, 1, 128, dtype=torch.float16)
    with torch.no_grad():
        preds["heatmap"][0, :, :4] = torch.tensor([100.0, -100.0, 100.0, -100.0], dtype=torch.float16)
        preds["dense_heatmap"][0, 0, 0, :4] = torch.tensor([100.0, -100.0, 100.0, -100.0], dtype=torch.float16)
    losses = run_tf(preds, targets, P, 2, True, cfg)
    sum(v for k, v in losses.items() if k != "matched_ious").backward()
    want, wgrad = tf_oracle(preds, targets, P, 2, True)
    check_losses(losses, want)
    for k, v in preds.items():
        assert v.grad.dtype == torch.float16
        assert np.abs(v.grad.double().cpu().numpy() - wgrad[k]).max() <= 1e-3 * np.abs(wgrad[k]).max() + 1e-7


def test_transfusion_deterministic_launches_and_no_sync():
    preds, targets, cfg, P = tf_inputs(29, 4, 180)
    _C.reset_launch_count()
    a = run_tf(preds, targets, P, 2, True, cfg)
    assert _C.launch_count() == 2
    with torch.autograd.set_multithreading_enabled(False):   # the launch counter is per host thread
        sum(v for k, v in a.items() if k != "matched_ious").backward()
    assert _C.launch_count() == 3
    g1 = {k: v.grad.clone() for k, v in preds.items()}
    for v in preds.values():
        v.grad = None
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = run_tf(preds, targets, P, 2, True, cfg)
        sum(v for k, v in b.items() if k != "matched_ious").backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert all(torch.equal(a[k], b[k]) for k in a)
    assert all(torch.equal(g1[k], preds[k].grad) for k in preds)


def test_centerhead_graph_of_targets_loss_backward():
    """targets + loss + backward captured once, replayed on three ground-truth sets, bit-equal to eager calls."""
    B, H = 2, 128
    tasks = TASKS
    cfg = ch_cfg(H)
    outs = S.centerhead_head_outputs(0, B, height=H, width=H)
    leaves = [{k: v.to(DEV) for k, v in t.items()} for t in outs]
    sets = [gt_padded(s, B) for s in (1, 2, 3)]
    nmax = max(s[0].shape[1] for s in sets)
    pad = lambda s: (torch.nn.functional.pad(s[0], (0, 0, 0, nmax - s[0].shape[1])),
                     torch.nn.functional.pad(s[1], (0, nmax - s[1].shape[1])), s[2])
    sets = [pad(s) for s in sets]
    static = [x.clone() for x in sets[0]]

    def step():
        preds = [[{k: v.detach().requires_grad_() for k, v in t.items()}] for t in leaves]
        targets = HT.centerhead_targets_batched(*static, tasks, cfg)
        losses = run_ch(preds, targets)
        grads = torch.autograd.grad(sum(losses.values()), [v for p in preds for v in p[0].values()])
        return torch.stack(list(losses.values())), grads

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out_l, out_g = step()
    for gt in sets:
        for d, x in zip(static, gt):
            d.copy_(x)
        g.replay()
        torch.cuda.synchronize()
        want_l, want_g = step()
        assert torch.equal(out_l, want_l)
        assert all(torch.equal(a, b) for a, b in zip(out_g, want_g))
