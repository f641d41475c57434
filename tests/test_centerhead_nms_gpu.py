"""GPU: bevfusion_b200.iou3d.centerhead_nms called the way CenterHead.get_bboxes calls its NMS step in each shipped
config, against a restatement of get_bboxes / get_task_detections (centerpoint.py:637-884) that takes the class
count from the task list, as the reference does (num_class_with_bg = self.num_classes[task_id], :670), and builds
nms_scales as get_bboxes does (:649-666).  Also: nms_batched orders tied scores stably, on lists shorter and longer
than 32 boxes."""
import numpy as np
import pytest
import torch

import nms_oracle as O
from test_nms_gpu import circle_points, clear_boxes, cu

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def iou3d():
    from bevfusion_b200 import iou3d as m
    return m


def nms_scales_of(test_cfg, num_classes):
    """get_bboxes (:649-666): a list per task from a list, a number, or nothing."""
    if "nms_scale" not in test_cfg:
        return [[1.0] * n for n in num_classes]
    if not isinstance(test_cfg["nms_scale"], list):
        return [[test_cfg["nms_scale"]] * n for n in num_classes]
    return test_cfg["nms_scale"]


def reference_task(iou3d, decoded, task_id, nms_type, cfg, nms_scale, num_class_with_bg):
    """One task of get_bboxes: the circle branch (:710-737) or get_task_detections (:768-884), with this
    package's single-list drop-ins in place of nms_gpu and the numba circle_nms."""
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
        box_preds, cls_preds, cls_labels = d["bboxes"], d["scores"], d["labels"]
        if num_class_with_bg == 1:
            top_scores = cls_preds.squeeze(-1)
            top_labels = torch.zeros(cls_preds.shape[0], device=cls_preds.device, dtype=torch.long)
        else:
            top_labels = cls_labels.long()
            top_scores = cls_preds.squeeze(-1)
        if cfg["score_threshold"] > 0.0:
            thresh = torch.tensor([cfg["score_threshold"]], device=cls_preds.device).type_as(cls_preds)
            top_scores_keep = top_scores >= thresh
            top_scores = top_scores.masked_select(top_scores_keep)
        if top_scores.shape[0] != 0:
            if cfg["score_threshold"] > 0.0:
                box_preds = box_preds[top_scores_keep]
                top_labels = top_labels[top_scores_keep]
            bev_box = box_preds[:, [0, 1, 3, 4, 6]]                    # LiDARInstance3DBoxes.bev
            for cls, scale in enumerate(nms_scale):
                cur_bev_box = bev_box[top_labels == cls]
                cur_bev_box[:, [2, 3]] *= scale
                bev_box[top_labels == cls] = cur_bev_box
            selected = iou3d.nms_gpu(iou3d.xywhr2xyxyr(bev_box), top_scores, thresh=cfg["nms_thr"],
                                     pre_maxsize=cfg["pre_max_size"], post_max_size=cfg["post_max_size"])
        else:
            selected = []
        selected_boxes, selected_labels = box_preds[selected], top_labels[selected]
        selected_scores = top_scores[selected]
        if selected_boxes.shape[0] != 0:
            mask = (selected_boxes[:, :3] >= rng[:3]).all(1) & (selected_boxes[:, :3] <= rng[3:]).all(1)
            out.append(dict(bboxes=selected_boxes[mask], scores=selected_scores[mask], labels=selected_labels[mask]))
        else:
            dev, dtype = box_preds.device, box_preds.dtype
            out.append(dict(bboxes=torch.zeros([0, 9], dtype=dtype, device=dev),
                            scores=torch.zeros([0], dtype=dtype, device=dev),
                            labels=torch.zeros([0], dtype=top_labels.dtype, device=dev)))
    return out


def detections(cuda, seed, batch):
    from bevfusion_b200 import synthetic as S
    dets = S.centerhead_detections(seed=seed, batch=batch)
    dets[2][0]["bboxes"][:5, 0] = 61.5                                  # outside post_center_limit_range
    dets[1][-1]["scores"][:] = 0.05                                     # every box below the score threshold
    return [[{k: v.to(cuda) for k, v in d.items()} for d in task] for task in dets]


def check(got, want, what):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        for key in ("bboxes", "scores", "labels"):
            assert g[key].dtype == w[key].dtype and g[key].shape == w[key].shape, (what, key)
            assert torch.equal(g[key], w[key]), (what, key)


@pytest.mark.parametrize("batch", [1, 4])
def test_default_config_without_nms_scale(cuda, iou3d, batch):
    """centerhead/default.yaml: nms_type rotate for every task, no nms_scale in test_cfg."""
    from bevfusion_b200 import synthetic as S
    cfg = dict(S.CENTERHEAD_TEST_CFG, nms_type="rotate")
    assert "nms_scale" not in cfg
    num_classes = [len(t) for t in S.CENTERHEAD_TASKS]
    scales = nms_scales_of(cfg, num_classes)
    dets = detections(cuda, 10 + batch, batch)
    for task_id, decoded in enumerate(dets):
        want = reference_task(iou3d, decoded, task_id, "rotate", cfg, scales[task_id], num_classes[task_id])
        check(iou3d.centerhead_nms(decoded, task_id, "rotate", cfg, None, num_classes[task_id]), want, task_id)
        check(iou3d.centerhead_nms(decoded, task_id, "rotate", cfg, scales[task_id], num_classes[task_id]), want,
              task_id)
        if num_classes[task_id] > 1 and any(len(w["labels"]) for w in want):   # the second class keeps its label
            assert any(bool((w["labels"] == 1).any()) for w in want), task_id


@pytest.mark.parametrize("batch", [1, 4])
def test_camera_radar_config(cuda, iou3d, batch):
    """lssfpn/camera+radar: per-task nms_type and per-class nms_scale, called as get_bboxes would."""
    from bevfusion_b200 import synthetic as S
    cfg = dict(S.CENTERHEAD_TEST_CFG, nms_type=S.CENTERHEAD_RADAR_NMS_TYPE, nms_scale=S.CENTERHEAD_RADAR_NMS_SCALE)
    num_classes = [len(t) for t in S.CENTERHEAD_TASKS]
    scales = nms_scales_of(cfg, num_classes)
    dets = detections(cuda, 20 + batch, batch)
    for task_id, decoded in enumerate(dets):
        nms_type = cfg["nms_type"][task_id]
        want = reference_task(iou3d, decoded, task_id, nms_type, cfg, scales[task_id], num_classes[task_id])
        check(iou3d.centerhead_nms(decoded, task_id, nms_type, cfg, scales[task_id], num_classes[task_id]), want,
              task_id)


def test_scalar_nms_scale(cuda, iou3d):
    """A number for nms_scale applies to every class, as get_bboxes expands it."""
    from bevfusion_b200 import synthetic as S
    cfg = dict(S.CENTERHEAD_TEST_CFG, nms_scale=1.5)
    num_classes = [len(t) for t in S.CENTERHEAD_TASKS]
    scales = nms_scales_of(cfg, num_classes)
    dets = detections(cuda, 31, 2)
    for task_id in (1, 5):
        want = reference_task(iou3d, dets[task_id], task_id, "rotate", cfg, scales[task_id], num_classes[task_id])
        check(iou3d.centerhead_nms(dets[task_id], task_id, "rotate", cfg, 1.5, num_classes[task_id]), want, task_id)


@pytest.mark.parametrize("mode", ["rotate", "circle"])
def test_nms_batched_orders_ties_stably(cuda, iou3d, mode):
    """Tied scores keep their row order, on a 20-box list and on 300-box lists, as a stable float64 sort does."""
    rng = np.random.default_rng(41)
    thresh = 0.2 if mode == "rotate" else 1.0
    sizes = [20, 300, 0, 300]
    lists = []
    for n in sizes:
        if mode == "rotate":
            boxes = clear_boxes(rng, n, thresh, span=12.0)
        else:                                                                   # centres in the first two columns
            boxes = np.zeros((n, 5), np.float32)
            boxes[:, :2] = circle_points(rng, n, thresh, 4.0)
        scores = rng.integers(0, 4, n).astype(np.float32) / 4                  # four score levels: many ties
        lists.append((boxes, scores))
    nmax = max(sizes)
    B = np.zeros((len(sizes), nmax, 5), np.float32)
    Sc = np.full((len(sizes), nmax), 2.0, np.float32)
    for i, (b, s) in enumerate(lists):
        B[i, :len(b)], Sc[i, :len(s)] = b, s
    counts = torch.tensor(sizes, dtype=torch.int32, device=cuda)
    keep, kc = iou3d.nms_batched(cu(B, cuda), cu(Sc, cuda), counts, mode, thresh, 1000, 83)
    for i, (b, s) in enumerate(lists):
        if mode == "rotate":
            gold = O.nms(b, s, thresh, 1000, 83)
        else:
            gold = O.circle_nms(np.concatenate([b[:, :2], s[:, None]], 1), thresh, 83)
        assert int(kc[i]) == len(gold), i
        assert np.array_equal(keep[i, :len(gold)].cpu().numpy(), gold), i

