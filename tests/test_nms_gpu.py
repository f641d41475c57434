"""GPU: rotated BEV IoU and NMS (bevfusion_b200.iou3d, csrc/box_nms.cu) against the float64 checker
(tests/nms_oracle.py), the reference fixture (tests/golden/nms_tiny.npz) and, when oracle/_ref holds it, the
reference's own iou3d_cuda op.

Two fp32 implementations of the rotated IoU differ in the last bits, so keep lists are compared exactly only
on lists drawn clear of the threshold (no pair with float64 IoU within 1e-3 of it); on unconstrained lists
the result must be a valid greedy NMS under a tolerance of 1e-4.  The batched forms are checked bit for bit
against the single-list ones."""
import math

import numpy as np
import pytest
import torch

import nms_oracle as O
from conftest import ref_module

pytestmark = pytest.mark.gpu

FIX = "nms_tiny.npz"
SIZES = [(0.3, 0.3), (0.6, 0.8), (0.8, 2.1), (1.95, 4.6), (2.5, 6.9), (2.9, 12.0)]
DELTA = 1e-4


@pytest.fixture(scope="module")
def fixture(golden_dir):
    import os
    return np.load(os.path.join(golden_dir, FIX))


@pytest.fixture(scope="module")
def iou3d():
    from bevfusion_b200 import iou3d as m
    return m


def rand_boxes(rng, n, span=61.0, cluster=True):
    """[n, 5] xyxyr boxes, clustered around n / 6 objects so that many pairs overlap."""
    objs = [(rng.uniform(-span, span), rng.uniform(-span, span), rng.uniform(-math.pi, math.pi),
             *SIZES[rng.integers(len(SIZES))]) for _ in range(max(1, n // 6 if cluster else n))]
    out = []
    for i in range(n):
        x, y, r, w, l = objs[rng.integers(len(objs))] if cluster else objs[i]
        w, l = w * rng.uniform(0.85, 1.15), l * rng.uniform(0.85, 1.15)
        x, y, r = x + rng.normal(0, 0.2 * w), y + rng.normal(0, 0.2 * l), r + rng.normal(0, 0.3)
        out.append([x - w / 2, y - l / 2, x + w / 2, y + l / 2, r])
    return np.array(out, np.float32).reshape(-1, 5)


def clear_boxes(rng, n, thresh, span=30.0):
    """Boxes drawn so that no pair has a float64 IoU within 1e-3 of thresh (pairs clearly apart excepted)."""
    boxes = []
    while len(boxes) < n:
        b = rand_boxes(rng, 1, span)[0] if not boxes or rng.uniform() < 0.25 else None
        if b is None:
            c = np.array(boxes[rng.integers(len(boxes))], np.float64)
            w, l = c[2] - c[0], c[3] - c[1]
            x, y = (c[0] + c[2]) / 2 + rng.normal(0, 0.25 * w), (c[1] + c[3]) / 2 + rng.normal(0, 0.25 * l)
            r = c[4] + rng.normal(0, 0.3)
            b = np.array([x - w / 2, y - l / 2, x + w / 2, y + l / 2, r], np.float32)
        b64 = b.astype(np.float64)
        if boxes:
            B = np.array(boxes, np.float64)
            iou = O.iou_matrix(b64[None], B)[0]
            near = np.abs(iou - thresh) < 1e-3
            if near.any():
                ra = 0.5 * np.hypot(b64[2] - b64[0], b64[3] - b64[1])
                rb = 0.5 * np.hypot(B[:, 2] - B[:, 0], B[:, 3] - B[:, 1])
                d = np.hypot((b64[0] + b64[2] - B[:, 0] - B[:, 2]) / 2, (b64[1] + b64[3] - B[:, 1] - B[:, 3]) / 2)
                if (near & ~((iou == 0) & (d > ra + rb + 1e-2))).any():
                    continue
        boxes.append(b)
    return np.array(boxes, np.float32).reshape(-1, 5)


def distinct_scores(rng, n):
    return ((rng.permutation(n) + rng.uniform(0.1, 0.9, n)) / max(n, 1)).astype(np.float32)


def ref_nms_sequence(mod, boxes, scores, thresh, pre_maxsize=None, post_max_size=None, normal=False):
    """iou3d_utils.py:24-68 restated, over any module with the iou3d_cuda interface."""
    order = scores.sort(0, descending=True)[1]
    if pre_maxsize is not None:
        order = order[:pre_maxsize]
    boxes = boxes[order].contiguous()
    keep = torch.zeros(boxes.size(0), dtype=torch.long)
    fn = mod.nms_normal_gpu if normal else mod.nms_gpu
    num_out = fn(boxes, keep, thresh, boxes.device.index)
    keep = order[keep[:num_out].cuda(boxes.device)].contiguous()
    if post_max_size is not None:
        keep = keep[:post_max_size]
    return keep


def normal_iou64(A, B):
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    w = np.maximum(np.minimum(A[:, None, 2], B[None, :, 2]) - np.maximum(A[:, None, 0], B[None, :, 0]), 0)
    h = np.maximum(np.minimum(A[:, None, 3], B[None, :, 3]) - np.maximum(A[:, None, 1], B[None, :, 1]), 0)
    inter = w * h
    sa, sb = (A[:, 2] - A[:, 0]) * (A[:, 3] - A[:, 1]), (B[:, 2] - B[:, 0]) * (B[:, 3] - B[:, 1])
    return inter / np.maximum(sa[:, None] + sb[None, :] - inter, 1e-8)


def cu(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


# ---- IoU values ----------------------------------------------------------------------------------------------

def test_iou_matches_float64_and_reference(cuda, iou3d, fixture):
    rng = np.random.default_rng(0)
    ref = ref_module("iou3d_cuda_ref")
    for boxes in (rand_boxes(rng, 500), rand_boxes(rng, 300, span=10.0)):
        b = cu(boxes, cuda)
        got = iou3d.boxes_iou_bev(b, b).cpu().numpy()
        gold = O.iou_matrix(boxes, boxes)
        assert np.abs(got - gold).max() <= 1e-4
        assert (gold > 0.05).sum() > 2 * len(boxes)               # plenty of overlapping pairs
        ov = iou3d.boxes_overlap_bev(b, b[:77]).cpu().numpy()
        ov64 = O.iou_matrix(boxes, boxes[:77], overlap=True)
        assert np.abs(ov - ov64).max() <= 1e-5 * ov64.max()
        if ref is not None:
            # off the diagonal: far from the origin the reference's fp32 misses corners of a box compared with
            # itself (IoU 1/3 instead of 1 for some boxes near 60 m), a fault of its arithmetic, not ours
            r = torch.zeros(len(boxes), len(boxes), device=cuda)
            ref.boxes_iou_bev_gpu(b, b, r)
            off = ~np.eye(len(boxes), dtype=bool)
            assert np.abs(got - r.cpu().numpy())[off].max() <= 1e-4
            assert np.abs(np.diagonal(got) - 1).max() <= 1e-5
    a, bb = cu(fixture["iou_a"], cuda), cu(fixture["iou_b"], cuda)
    pair = iou3d.boxes_iou_bev(a, bb).diagonal().cpu().numpy()
    assert np.abs(pair - fixture["iou_ref"]).max() <= 1e-4
    n = int(fixture["iou_named"])                                  # 1, 1/3, 0.7071, 0, 0, 1/16, 1/16, 0, 1
    assert np.abs(pair[:n] - fixture["iou_ref"][:n]).max() <= 1e-5


def test_iou_shapes_and_empty(cuda, iou3d):
    z = torch.zeros(0, 5, device=cuda)
    b = cu(rand_boxes(np.random.default_rng(1), 7), cuda)
    assert tuple(iou3d.boxes_iou_bev(z, b).shape) == (0, 7) and tuple(iou3d.boxes_iou_bev(b, z).shape) == (7, 0)
    assert iou3d.boxes_iou_bev(b, b).dtype == torch.float32
    with pytest.raises(ValueError):
        iou3d.boxes_iou_bev(b[:, :4].contiguous(), b)


# ---- keep lists against the reference ----------------------------------------------------------------------

def test_keep_lists_match_fixture(cuda, iou3d, fixture):
    for k in range(int(fixture["nms_cases"])):
        boxes, scores = cu(fixture["nms%d_boxes" % k], cuda), cu(fixture["nms%d_scores" % k], cuda)
        keep = iou3d.nms_gpu(boxes, scores, float(fixture["nms%d_thresh" % k]))
        assert keep.dtype == torch.int64 and keep.device == boxes.device
        assert np.array_equal(keep.cpu().numpy(), fixture["nms%d_keep" % k]), k


@pytest.mark.parametrize("n", [1, 63, 64, 65, 500, 1000])
@pytest.mark.parametrize("thresh", [0.2, 0.5])
def test_keep_lists_clear_of_threshold(cuda, iou3d, n, thresh):
    rng = np.random.default_rng(n * 10 + int(thresh * 10))
    boxes = clear_boxes(rng, n, thresh, span=30.0 if n < 1000 else 50.0)
    scores = distinct_scores(rng, n)
    b, s = cu(boxes, cuda), cu(scores, cuda)
    got = iou3d.nms_gpu(b, s, thresh).cpu().numpy()
    assert np.array_equal(got, O.nms(boxes, scores, thresh))
    ref = ref_module("iou3d_cuda_ref")
    if ref is not None:
        assert np.array_equal(got, ref_nms_sequence(ref, b, s, thresh).cpu().numpy())


@pytest.mark.parametrize("n", [1, 63, 64, 65, 500, 1000, 4096])
def test_keep_lists_valid_greedy_unconstrained(cuda, iou3d, n):
    rng = np.random.default_rng(100 + n)
    boxes, scores = rand_boxes(rng, n), distinct_scores(rng, n)
    got = iou3d.nms_gpu(cu(boxes, cuda), cu(scores, cuda), 0.2).cpu().numpy()
    order = O.sort_desc(scores)
    pos = np.empty(n, int)
    pos[order] = np.arange(n)
    iou = O.iou_matrix(boxes[order], boxes[order])
    assert O.check_greedy(iou, sorted(pos[got]), 0.2, DELTA) == []
    assert list(pos[got]) == sorted(pos[got])                       # kept in descending score order


def test_pre_and_post_max(cuda, iou3d):
    rng = np.random.default_rng(7)
    boxes = clear_boxes(rng, 500, 0.2)
    scores = distinct_scores(rng, 500)
    b, s = cu(boxes, cuda), cu(scores, cuda)
    full = O.nms(boxes, scores, 0.2)
    assert len(full) > 100
    for pre, post in [(None, None), (300, None), (None, 83), (300, 83), (1000, 5000), (64, 10), (0, 83)]:
        got = iou3d.nms_gpu(b, s, 0.2, pre_maxsize=pre, post_max_size=post).cpu().numpy()
        assert np.array_equal(got, O.nms(boxes, scores, 0.2, pre, post)), (pre, post)
    ref = ref_module("iou3d_cuda_ref")
    if ref is not None:
        got = iou3d.nms_gpu(b, s, 0.2, pre_maxsize=300, post_max_size=83)
        assert torch.equal(got, ref_nms_sequence(ref, b, s, 0.2, 300, 83))


def test_nms_normal(cuda, iou3d):
    rng = np.random.default_rng(3)
    for n, thresh in [(65, 0.2), (500, 0.5), (1000, 0.2)]:
        boxes = rand_boxes(rng, n, span=30.0)
        boxes[:, :4] = np.round(boxes[:, :4] * 8) / 8                # exact in fp32: the IoU is clear or exact
        scores = distinct_scores(rng, n)
        iou = normal_iou64(boxes, boxes)
        b, s = cu(boxes, cuda), cu(scores, cuda)
        got = iou3d.nms_normal_gpu(b, s, thresh).cpu().numpy()
        order = O.sort_desc(scores)
        gold = order[O.greedy(iou[order][:, order], thresh)]
        if not (np.abs(iou - thresh) < 1e-3).any():
            assert np.array_equal(got, gold)
        pos = np.empty(n, int)
        pos[order] = np.arange(n)
        assert O.check_greedy(iou[order][:, order], sorted(pos[got]), thresh, DELTA) == []
        ref = ref_module("iou3d_cuda_ref")
        if ref is not None and not (np.abs(iou - thresh) < 1e-3).any():
            assert np.array_equal(got, ref_nms_sequence(ref, b, s, thresh, normal=True).cpu().numpy())


# ---- NaN boxes and thresholds below 0 ----------------------------------------------------------------------

def test_nan_boxes_and_negative_threshold(cuda, iou3d):
    rng = np.random.default_rng(11)
    boxes = clear_boxes(rng, 65, 0.2, span=10.0)
    boxes[[3, 20, 64], 0] = np.nan                                  # NaN x1: IoU 0 with everything
    boxes[40, 4] = np.nan                                           # NaN yaw
    scores = distinct_scores(rng, 65)
    b, s = cu(boxes, cuda), cu(scores, cuda)
    iou = iou3d.boxes_iou_bev(b, b).cpu().numpy()
    assert (iou[[3, 20, 40, 64]] == 0).all() and (iou[:, [3, 20, 40, 64]] == 0).all()
    got = iou3d.nms_gpu(b, s, 0.2).cpu().numpy()
    assert {3, 20, 40, 64} <= set(got.tolist())                     # never suppressed, suppress nothing
    assert np.array_equal(got, O.nms(boxes, scores, 0.2))
    for thresh in (-0.1, -1e-6):                                    # IoU 0 > thresh: every later box goes
        assert np.array_equal(iou3d.nms_gpu(b, s, thresh).cpu().numpy(), [int(np.argmax(scores))])
    ref = ref_module("iou3d_cuda_ref")
    if ref is not None:
        for thresh in (0.2, -0.1):
            assert np.array_equal(iou3d.nms_gpu(b, s, thresh).cpu().numpy(),
                                  ref_nms_sequence(ref, b, s, thresh).cpu().numpy())


# ---- circle NMS ----------------------------------------------------------------------------------------------

def circle_points(rng, n, thresh, span):
    pts = []
    while len(pts) < n:
        p = rng.uniform(-span, span, 2).astype(np.float32)
        if pts and (np.abs(((np.array(pts, np.float64) - p) ** 2).sum(1) - thresh) < 1e-6 * thresh).any():
            continue
        pts.append(p)
    return np.array(pts, np.float32).reshape(-1, 2)


def test_circle_nms_matches_fixture_and_oracle(cuda, iou3d, fixture):
    for k in range(int(fixture["circle_cases"])):
        dets, thresh, post = fixture["circle%d_dets" % k], float(fixture["circle%d_thresh" % k]), int(fixture["circle%d_post" % k])
        got = iou3d.circle_nms(cu(dets, cuda), thresh, post_max_size=post)
        assert got.dtype == torch.int64 and got.is_cuda
        assert np.array_equal(got.cpu().numpy(), fixture["circle%d_keep" % k]), k
    rng = np.random.default_rng(5)
    for n, thresh, post in [(1, 4.0, 83), (63, 1.0, 83), (64, 0.175, 83), (65, 12.0, 10), (1000, 0.85, 83),
                            (4096, 4.0, 5000)]:
        pts = circle_points(rng, n, thresh, 4.0 if thresh < 2 else 40.0)
        dets = np.concatenate([pts, distinct_scores(rng, n)[:, None]], 1)
        got = iou3d.circle_nms(cu(dets, cuda), thresh, post_max_size=post).cpu().numpy()
        assert np.array_equal(got, O.circle_nms(dets, thresh, post)), (n, thresh)


# ---- batched forms -------------------------------------------------------------------------------------------

def padded(lists, dev, width=5):
    nmax = max([len(b) for b, _ in lists] + [1])
    B = np.zeros((len(lists), nmax, width), np.float32)
    S = np.zeros((len(lists), nmax), np.float32)
    for i, (b, s) in enumerate(lists):
        B[i, :len(b)], S[i, :len(s)] = b, s
        S[i, len(s):] = rng_pad_scores(nmax - len(s), i)           # pads may hold anything
    return cu(B, dev), cu(S, dev), torch.tensor([len(b) for b, _ in lists], dtype=torch.int32, device=dev)


def rng_pad_scores(n, seed):
    return np.random.default_rng(seed).uniform(2, 3, n).astype(np.float32)


@pytest.mark.parametrize("mode", ["rotate", "normal", "circle"])
def test_nms_batched_equals_per_list(cuda, iou3d, mode):
    rng = np.random.default_rng({"rotate": 1, "normal": 2, "circle": 3}[mode])
    sizes = [0, 1, 63, 64, 65, 500, 1000, 0, 37, 128, 129, 300] * 2                  # S = 24
    lists = [(rand_boxes(rng, n), distinct_scores(rng, n)) for n in sizes]
    B, Sc, counts = padded(lists, cuda)
    thresh = {"rotate": 0.2, "normal": 0.3, "circle": 1.0}[mode]
    for pre, post in [(None, None), (1000, 83), (300, 5000), (64, 500)]:
        keep, kc = iou3d.nms_batched(B, Sc, counts, mode, thresh, pre, post)
        P = post if post is not None else min(pre or B.shape[1], B.shape[1])
        assert tuple(keep.shape) == (24, P) and keep.dtype == torch.int64 and kc.dtype == torch.int32
        for i, (b, s) in enumerate(lists):
            bb, ss = cu(b, cuda), cu(s, cuda)
            if mode == "rotate":
                one = iou3d.nms_gpu(bb, ss, thresh, pre, post)
            elif mode == "normal" and pre is None and post is None:
                one = iou3d.nms_normal_gpu(bb, ss, thresh)
            else:                                                   # the same single-list path with the cuts
                one = iou3d._single(bb if mode == "normal" else bb[:, :2], ss, thresh, mode, pre, post)
            c = int(kc[i])
            assert c == len(one), (i, pre, post)
            assert torch.equal(keep[i, :c], one), (i, pre, post)
            assert bool((keep[i, c:] == -1).all())
        assert int(kc[0]) == 0 and int(kc[7]) == 0                                 # empty segments


def test_segment_limit(cuda, iou3d):
    # 65,536 boxes on a 1 m grid of 0.5 m boxes: nothing overlaps, everything is kept (1,024 bitmap words)
    n = 65536
    g = np.arange(n)
    xy = np.stack([g % 256, g // 256], 1).astype(np.float32)
    boxes = np.concatenate([xy, xy + 0.5, np.zeros((n, 1), np.float32)], 1)
    scores = np.random.default_rng(0).permutation(n).astype(np.float32)
    keep, kc = iou3d.nms_batched(cu(boxes[None], cuda), cu(scores[None], cuda),
                                 torch.tensor([n], device=cuda), "rotate", 0.0)
    assert int(kc[0]) == n
    assert np.array_equal(keep[0].cpu().numpy(), np.argsort(-scores, kind="stable"))
    with pytest.raises(ValueError):                                 # BEVB200_EUNSUPPORTED above 65,536
        iou3d.nms_batched(torch.zeros(1, n + 1, 5, device=cuda), torch.zeros(1, n + 1, device=cuda),
                          torch.tensor([1], device=cuda), "rotate", 0.2)
    from bevfusion_b200 import _C
    L = _C.lib()
    kcnt = torch.zeros(1, dtype=torch.int32, device=cuda)
    rc = L.bevb200_nms(_C.ptr(cu(boxes[None], cuda)), None, 1, n + 1, 0, 0.2, 10, None, None, _C.ptr(kcnt), None, 0,
                       _C.current_stream(cuda))
    assert rc == -4


def test_nms_batched_cuda_graph(cuda, iou3d):
    S, nmax = 24, 500
    boxes = torch.zeros(S, nmax, 5, device=cuda)
    scores = torch.zeros(S, nmax, device=cuda)
    counts = torch.zeros(S, dtype=torch.int32, device=cuda)

    def load(seed):
        r = np.random.default_rng(seed)
        cnt = r.integers(0, nmax + 1, S)
        cnt[seed % S] = 0
        boxes.copy_(cu(rand_boxes(r, S * nmax).reshape(S, nmax, 5), cuda))
        scores.copy_(cu(r.uniform(0, 1, (S, nmax)).astype(np.float32), cuda))
        counts.copy_(cu(cnt.astype(np.int32), cuda))

    load(0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            iou3d.nms_batched(boxes, scores, counts, "rotate", 0.2, 1000, 83)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        keep_g, kc_g = iou3d.nms_batched(boxes, scores, counts, "rotate", 0.2, 1000, 83)
    for seed in (1, 2, 3):
        load(seed)
        graph.replay()
        keep_e, kc_e = iou3d.nms_batched(boxes, scores, counts, "rotate", 0.2, 1000, 83)
        torch.cuda.synchronize()
        assert torch.equal(kc_g, kc_e) and torch.equal(keep_g, keep_e), seed
        assert int(kc_e.max()) > 10


# ---- CenterHead NMS step -------------------------------------------------------------------------------------

def reference_task(iou3d, decoded, task_id, nms_type, cfg, nms_scale):
    """CenterHead.get_bboxes (centerpoint.py:710-737) / get_task_detections (:768-884) for one task, restated
    with this package's single-list drop-ins in place of nms_gpu and the numba circle_nms."""
    out = []
    if nms_type == "circle":
        for d in decoded:
            boxes3d, scores, labels = d["bboxes"], d["scores"], d["labels"]
            boxes = torch.cat([boxes3d[:, [0, 1]], scores.view(-1, 1)], dim=1)
            keep = iou3d.circle_nms(boxes, cfg["min_radius"][task_id], post_max_size=cfg["post_max_size"])
            out.append(dict(bboxes=boxes3d[keep], scores=scores[keep], labels=labels[keep]))
        return out
    rng = torch.tensor(cfg["post_center_limit_range"], dtype=decoded[0]["bboxes"].dtype,
                       device=decoded[0]["bboxes"].device)
    for d in decoded:
        box_preds, top_scores = d["bboxes"], d["scores"]
        top_labels = d["labels"].long() if len(nms_scale) > 1 else torch.zeros_like(d["labels"], dtype=torch.long)
        if cfg["score_threshold"] > 0.0:
            keep_mask = top_scores >= torch.tensor([cfg["score_threshold"]], device=top_scores.device).type_as(top_scores)
            top_scores = top_scores.masked_select(keep_mask)
            box_preds, top_labels = box_preds[keep_mask], top_labels[keep_mask]
        if top_scores.shape[0] != 0:
            bev_box = box_preds[:, [0, 1, 3, 4, 6]]
            for cls, scale in enumerate(nms_scale):
                cur = bev_box[top_labels == cls]
                cur[:, [2, 3]] *= scale
                bev_box[top_labels == cls] = cur
            selected = iou3d.nms_gpu(iou3d.xywhr2xyxyr(bev_box), top_scores, thresh=cfg["nms_thr"],
                                     pre_maxsize=cfg["pre_max_size"], post_max_size=cfg["post_max_size"])
        else:
            selected = []
        sb, sl, ss = box_preds[selected], top_labels[selected], top_scores[selected]
        if sb.shape[0] != 0:
            mask = (sb[:, :3] >= rng[:3]).all(1) & (sb[:, :3] <= rng[3:]).all(1)
            out.append(dict(bboxes=sb[mask], scores=ss[mask], labels=sl[mask]))
        else:
            out.append(dict(bboxes=torch.zeros([0, sb.shape[1] if sb.dim() == 2 else 9], device=sb.device),
                            scores=torch.zeros([0], device=sb.device),
                            labels=torch.zeros([0], dtype=torch.long, device=sb.device)))
    return out


@pytest.mark.parametrize("batch", [1, 4])
def test_centerhead_nms_equals_restated_reference(cuda, iou3d, batch):
    from bevfusion_b200 import synthetic as S
    dets = S.centerhead_detections(seed=batch, batch=batch)
    cfg = dict(S.CENTERHEAD_TEST_CFG)
    dets[2][0]["bboxes"][:5, 0] = 61.5                                  # outside post_center_limit_range
    dets[4][-1] = {k: v[:0] for k, v in dets[4][-1].items()}           # an empty sample
    dets[1][0]["scores"][:] = 0.05                                      # every box below the score threshold
    for task_id, (nms_type, scale) in enumerate(zip(S.CENTERHEAD_RADAR_NMS_TYPE, S.CENTERHEAD_RADAR_NMS_SCALE)):
        decoded = [{k: v.to(cuda) for k, v in d.items()} for d in dets[task_id]]
        got = iou3d.centerhead_nms(decoded, task_id, nms_type, cfg, scale)
        want = reference_task(iou3d, decoded, task_id, nms_type, cfg, scale)
        assert len(got) == batch
        for g, w in zip(got, want):
            for key in ("bboxes", "scores", "labels"):
                assert g[key].dtype == w[key].dtype and g[key].device == w[key].device, key
                assert torch.equal(g[key], w[key]), (task_id, nms_type, key)
    # the default config: one rotate NMS for every task, with the default scale
    for task_id in range(6):
        decoded = [{k: v.to(cuda) for k, v in d.items()} for d in dets[task_id]]
        scale = [1.0] * len(S.CENTERHEAD_TASKS[task_id])
        got = iou3d.centerhead_nms(decoded, task_id, "rotate", cfg, scale)
        want = reference_task(iou3d, decoded, task_id, "rotate", cfg, scale)
        for g, w in zip(got, want):
            assert all(torch.equal(g[k], w[k]) for k in ("bboxes", "scores", "labels"))


def test_centerhead_detections_are_valid_greedy(cuda, iou3d):
    from bevfusion_b200 import synthetic as S
    dets = S.centerhead_detections(seed=3, batch=2)
    for task_id in (1, 2, 4, 5):
        scale = S.CENTERHEAD_RADAR_NMS_SCALE[task_id]
        for d in dets[task_id]:
            bev = d["bboxes"][:, [0, 1, 3, 4, 6]].clone()
            bev[:, 2:4] *= torch.tensor(scale)[d["labels"]][:, None]
            xyxyr = iou3d.xywhr2xyxyr(bev).numpy()
            s = d["scores"].numpy()
            got = iou3d.nms_gpu(cu(xyxyr, cuda), cu(s, cuda), 0.2).cpu().numpy()
            order = O.sort_desc(s)
            pos = np.empty(len(s), int)
            pos[order] = np.arange(len(s))
            assert O.check_greedy(O.iou_matrix(xyxyr[order], xyxyr[order]), sorted(pos[got]), 0.2, DELTA) == []


# ---- the drop-in iou3d_cuda module ----------------------------------------------------------------------------

def test_iou3d_cuda_shim(cuda, iou3d):
    from bevfusion_b200.shims import build as shim_build
    shim = shim_build.load_module("iou3d_cuda")
    rng = np.random.default_rng(13)
    boxes, scores = rand_boxes(rng, 500), distinct_scores(rng, 500)
    b, s = cu(boxes, cuda), cu(scores, cuda)
    for pre, post in [(None, None), (1000, 83), (200, 50)]:
        assert torch.equal(ref_nms_sequence(shim, b, s, 0.2, pre, post), iou3d.nms_gpu(b, s, 0.2, pre, post))
    assert torch.equal(ref_nms_sequence(shim, b, s, 0.3, normal=True), iou3d.nms_normal_gpu(b, s, 0.3))
    ans = b.new_zeros((500, 120))                                        # iou3d_utils.py:6-21
    assert shim.boxes_iou_bev_gpu(b, b[:120].contiguous(), ans) == 1
    assert torch.equal(ans, iou3d.boxes_iou_bev(b, b[:120]))
    ov = b.new_zeros((500, 120))
    shim.boxes_overlap_bev_gpu(b, b[:120].contiguous(), ov)
    assert torch.equal(ov, iou3d.boxes_overlap_bev(b, b[:120]))
    keep = torch.zeros(500, dtype=torch.long)                            # the raw call: boxes taken as sorted
    n = shim.nms_gpu(b, keep, 0.2, b.device.index)
    by_position = iou3d.nms_gpu(b, torch.arange(500, 0, -1, device=cuda, dtype=torch.float32), 0.2)
    assert not keep.is_cuda and torch.equal(keep[:n], by_position.cpu())
    with pytest.raises(RuntimeError):
        shim.nms_gpu(b.cpu(), keep, 0.2, 0)
