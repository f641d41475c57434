"""CPU: argument checks of bevfusion_b200.iou3d.centerhead_nms that come before any device work.  The task's
class count decides whether labels are kept (get_task_detections, centerpoint.py:804-811), so a call that gives
neither num_classes nor a per-class nms_scale list is refused instead of guessing one class."""
import pytest
import torch


def decoded():
    return [dict(bboxes=torch.zeros(4, 9), scores=torch.arange(4.0), labels=torch.tensor([0, 1, 1, 0]))]


CFG = dict(post_max_size=83, score_threshold=0.1, nms_thr=0.2, pre_max_size=1000,
           post_center_limit_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0])


@pytest.mark.parametrize("nms_scale", [None, 1.0, 2.5])
def test_class_count_is_required_without_a_per_class_list(nms_scale):
    from bevfusion_b200 import iou3d
    with pytest.raises(ValueError):
        iou3d.centerhead_nms(decoded(), 1, "rotate", CFG, nms_scale)


def test_class_count_must_be_positive():
    from bevfusion_b200 import iou3d
    with pytest.raises(ValueError):
        iou3d.centerhead_nms(decoded(), 1, "rotate", CFG, None, 0)


@pytest.mark.parametrize("nms_scale, num_classes", [(None, 2), ([1.0, 1.0], None), (1.0, 2), ([2.5, 4.0], 2)])
def test_valid_class_counts_reach_the_device_check(nms_scale, num_classes):
    from bevfusion_b200 import iou3d
    with pytest.raises(RuntimeError):                 # CPU tensors: there is no CPU path
        iou3d.centerhead_nms(decoded(), 1, "rotate", CFG, nms_scale, num_classes)
