"""GPU: bevfusion_b200.head_targets against the fixture made from the reference's own code and against the numpy
restatement (tests/head_targets_oracle.py) on random synthetic.gt_boxes batches.  Draw records (plane, centre
cell, radius), ind and mask are compared bit for bit; the heatmap bit for bit on the fixture and within one fp32
ulp on random batches (a CUDA-versus-glibc double exp that crosses an fp32 rounding boundary), the number of
differing cells reported; anno_box within 2 fp32 ulp (log, sin, cos).  Also: the list form equals the batched
form, two runs are bitwise equal, one CUDA-graph capture replayed on three batches with other counts equals eager
calls, three launches per call, the status word, boxes on the CPU with labels on the device, and the
draw_heatmap_gaussian mirror against the reference's slicing and torch.max."""
import numpy as np
import pytest
import torch

import head_targets_oracle as O
from test_head_targets_cpu import TASK_CLASSES, case, fixture, oracle_case

pytestmark = pytest.mark.gpu

CFG_SIX = dict(point_cloud_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], grid_size=[1024, 1024, 40],
               voxel_size=[0.1, 0.1, 0.2], out_size_factor=8, dense_reg=1, gaussian_overlap=0.1, max_objs=500,
               min_radius=2)
CFG_TF = dict(point_cloud_range=[-54.0, -54.0, -5.0, 54.0, 54.0, 3.0], grid_size=[1440, 1440, 41],
              voxel_size=[0.075, 0.075, 0.2], out_size_factor=8, gaussian_overlap=0.1, min_radius=2)
TASKS = [dict(num_class=1, class_names=["car"]), dict(num_class=2, class_names=["truck", "construction_vehicle"]),
         dict(num_class=2, class_names=["bus", "trailer"]), dict(num_class=1, class_names=["barrier"]),
         dict(num_class=2, class_names=["motorcycle", "bicycle"]),
         dict(num_class=2, class_names=["pedestrian", "traffic_cone"])]


@pytest.fixture(scope="module")
def H():
    from bevfusion_b200 import head_targets as m
    return m


def ulps(a, b):
    """fp32 ulp distance per element (NaN equal to NaN)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    d = np.abs(ia - ib)
    return np.where(np.isnan(a) & np.isnan(b), 0, d)


def to_dev(dev, boxes, labels, counts):
    return (torch.from_numpy(np.ascontiguousarray(boxes)).to(dev), torch.from_numpy(labels.astype(np.int32)).to(dev),
            torch.from_numpy(counts.astype(np.int32)).to(dev))


def run(H, dev, mode, cfg, boxes, labels, counts, norm_bbox=True):
    """The native call -> numpy dict shaped as the oracle's result."""
    b, l, c = to_dev(dev, boxes, labels, counts)
    if mode == "centerhead":
        M = cfg["max_objs"] * cfg["dense_reg"]
        hm, anno, ind, mask, status, rec = H._run(b, l, c, "centerhead", TASK_CLASSES,
                                                  H.centerhead_label_table(TASK_CLASSES), cfg, M, norm_bbox)
        hms = H._split_heatmap(hm, b.shape[0], TASK_CLASSES, *O_fmap(cfg))
    else:
        hm, anno, ind, mask, status, rec = H._run(b, l, c, "transfusion", [10], [(0, k) for k in range(10)], cfg)
        hms = H._split_heatmap(hm, b.shape[0], [10], *O_fmap(cfg))
    torch.cuda.synchronize()
    out = dict(heatmaps=[h.cpu().numpy() for h in hms], records=rec.cpu().numpy(), status=int(status.item()))
    if anno is not None:
        out.update(anno=anno.cpu().numpy(), ind=ind.cpu().numpy(), mask=mask.cpu().numpy())
    return out


def O_fmap(cfg):
    osf = cfg["out_size_factor"]
    return cfg["grid_size"][1] // osf, cfg["grid_size"][0] // osf


def compare(got, want, heat_ulps, label):
    assert np.array_equal(got["records"], want["records"]), label + ": draw records"
    assert got["status"] == want["status"], label + ": status"
    diff = 0
    for g, w in zip(got["heatmaps"], want["heatmaps"]):
        u = ulps(g, w)
        diff += int((u > 0).sum())
        assert u.max(initial=0) <= heat_ulps, "%s: heatmap off by %d ulp" % (label, u.max())
    print("%s: %d heatmap cells differ" % (label, diff))
    if heat_ulps == 0:
        assert diff == 0
    if "anno" in got:
        assert np.array_equal(got["ind"], want["ind"]) and np.array_equal(got["mask"], want["mask"]), label
        assert ulps(got["anno"], want["anno"]).max(initial=0) <= 2, label + ": anno_box"
    return diff


@pytest.mark.parametrize("name", ["ch_six", "ch_small", "tf_ten", "tf_wide"])
def test_fixture_bit_exact(cuda, H, name):
    d = fixture()
    meta, boxes, labels, counts = case(d, name)
    got = run(H, cuda, meta["mode"], meta["cfg"], boxes, labels, counts, meta["norm_bbox"])
    _, want = oracle_case(d, name)
    if meta["mode"] == "centerhead":
        want["heatmaps"] = [d["%s_hm%d" % (name, t)] for t in range(6)]
        want["anno"], want["ind"], want["mask"] = d[name + "_anno"], d[name + "_ind"], d[name + "_mask"]
    else:
        want["heatmaps"] = [d[name + "_hm"]]
    compare(got, want, 0, name)


def synthetic_batch(seed, batch, D=9):
    from bevfusion_b200 import synthetic as S
    bl, ll = S.gt_boxes(seed=seed, batch=batch)
    n = max(b.shape[0] for b in bl)
    boxes = np.zeros((batch, n, D), np.float32)
    labels = np.zeros((batch, n), np.int32)
    counts = np.array([b.shape[0] for b in bl], np.int32)
    for i, (b, l) in enumerate(zip(bl, ll)):
        boxes[i, :len(b)] = b.numpy()[:, :D]
        labels[i, :len(b)] = l.numpy()
    return boxes, labels, counts


@pytest.mark.parametrize("seed,D,norm", [(0, 9, True), (1, 9, False), (2, 7, True), (3, 7, False)])
def test_centerhead_random_vs_oracle(cuda, H, seed, D, norm):
    boxes, labels, counts = synthetic_batch(seed, 4, D)
    got = run(H, cuda, "centerhead", CFG_SIX, boxes, labels, counts, norm)
    want = O.targets(boxes, labels, counts, "centerhead", TASK_CLASSES, CFG_SIX, 500, norm)
    compare(got, want, 1, "centerhead seed %d" % seed)
    assert got["mask"].sum() > 100


@pytest.mark.parametrize("seed,D", [(4, 9), (5, 7)])
def test_transfusion_random_vs_oracle(cuda, H, seed, D):
    boxes, labels, counts = synthetic_batch(seed, 4, D)
    got = run(H, cuda, "transfusion", CFG_TF, boxes, labels, counts)
    want = O.targets(boxes, labels, counts, "transfusion", [10], CFG_TF)
    compare(got, want, 1, "transfusion seed %d" % seed)
    assert (got["records"][..., 3] >= 0).sum() > 100


def test_small_max_objs_and_dense_reg(cuda, H):
    cfg = dict(CFG_SIX, max_objs=2, dense_reg=2)
    boxes, labels, counts = synthetic_batch(6, 3)
    got = run(H, cuda, "centerhead", cfg, boxes, labels, counts)
    want = O.targets(boxes, labels, counts, "centerhead", TASK_CLASSES, cfg, 4)
    compare(got, want, 1, "max_objs 2 x dense_reg 2")
    live = np.arange(labels.shape[1])[None, :] < counts[:, None]
    assert got["mask"].shape == (6, 3, 4) and ((labels == 0) & live).sum(1).max() > 4    # more cars than slots
    assert got["mask"][0].sum() > 4


def test_list_form_equals_batched(cuda, H):
    from bevfusion_b200 import synthetic as S
    bl, ll = S.gt_boxes(seed=7, batch=3)
    bl = [b.to(cuda) for b in bl]
    ll = [l.to(cuda) for l in ll]
    bl[1] = bl[1][:0]                                  # an empty sample
    ll[1] = ll[1][:0]

    class Boxes:
        def __init__(self, t):
            self.tensor = t
    a = H.centerhead_targets([Boxes(b) for b in bl], ll, TASKS, CFG_SIX)
    pb, pl, pc = H.pad_gt(bl, ll)
    b = H.centerhead_targets_batched(pb, pl, pc, TASKS, CFG_SIX)
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert torch.equal(u, v)
    assert [tuple(h.shape) for h in a[0]] == [(3, n, 128, 128) for n in TASK_CLASSES]
    assert all(h.is_contiguous() for h in a[0]) and tuple(a[1][0].shape) == (3, 500, 10)
    assert a[2][0].dtype == torch.int64 and a[3][0].dtype == torch.uint8
    assert not a[3][0][1].any() and not a[0][0][1].any()
    t1 = H.transfusion_heatmap_targets(bl, ll, 10, CFG_TF)
    t2 = H.transfusion_heatmap_targets_batched(pb, pl, pc, 10, CFG_TF)
    assert torch.equal(t1, t2) and tuple(t1.shape) == (3, 10, 180, 180)


def test_two_runs_bitwise_equal_and_three_launches(cuda, H):
    from bevfusion_b200 import _C
    pb, pl, pc = to_dev(cuda, *synthetic_batch(8, 4))
    a = H.centerhead_targets_batched(pb, pl, pc, TASKS, CFG_SIX)
    _C.reset_launch_count()
    b = H.centerhead_targets_batched(pb, pl, pc, TASKS, CFG_SIX)
    assert _C.launch_count() == 3
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert torch.equal(u.view(torch.uint8) if u.is_floating_point() else u,
                               v.view(torch.uint8) if v.is_floating_point() else v)
    _C.reset_launch_count()
    H.transfusion_heatmap_targets_batched(pb, pl, pc, 10, CFG_TF)
    assert _C.launch_count() == 3


def test_cuda_graph_replay_equals_eager(cuda, H):
    boxes, labels, counts = synthetic_batch(9, 4)
    sb, sl, sc = to_dev(cuda, boxes, labels, counts)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        H.centerhead_targets_batched(sb, sl, sc, TASKS, CFG_SIX)         # warm up outside the capture
        H.transfusion_heatmap_targets_batched(sb, sl, sc, 10, CFG_TF)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ch = H.centerhead_targets_batched(sb, sl, sc, TASKS, CFG_SIX)
        tf = H.transfusion_heatmap_targets_batched(sb, sl, sc, 10, CFG_TF)
    rng = np.random.default_rng(0)
    for k in range(3):
        nb, nl, _ = synthetic_batch(10 + k, 4)
        m = min(nb.shape[1], boxes.shape[1])
        new_counts = np.minimum(rng.integers(0, boxes.shape[1] + 1, 4), m).astype(np.int32)
        new_counts[k] = 0                                                  # one empty sample per batch
        sb.zero_()
        sb[:, :m].copy_(torch.from_numpy(nb[:, :m]))
        sl.zero_()
        sl[:, :m].copy_(torch.from_numpy(nl[:, :m]))
        sc.copy_(torch.from_numpy(new_counts))
        g.replay()
        eager = H.centerhead_targets_batched(sb, sl, sc, TASKS, CFG_SIX)
        eager_tf = H.transfusion_heatmap_targets_batched(sb, sl, sc, 10, CFG_TF)
        torch.cuda.synchronize()
        for x, y in zip(ch, eager):
            for u, v in zip(x, y):
                assert torch.equal(u, v), k
        assert torch.equal(tf, eager_tf), k
        want = O.targets(sb.cpu().numpy(), sl.cpu().numpy(), new_counts, "transfusion", [10], CFG_TF)
        assert ulps(tf.cpu().numpy(), want["heatmaps"][0]).max() <= 1


def test_status_counts_bad_labels_and_infinite_sizes(cuda, H):
    boxes, labels, counts = synthetic_batch(11, 2)
    counts[:] = [10, 10]
    boxes[0, 0, 3] = np.inf                      # infinite size: counted in both modes
    boxes[1, 1, 0] = np.nan                      # non-finite centre: skipped, not counted
    labels[0, 2], labels[1, 3], labels[1, 4] = 10, -1, 12
    pb, pl, pc = to_dev(cuda, boxes, labels, counts)
    hm, st = H.transfusion_heatmap_targets_batched(pb, pl, pc, 10, CFG_TF, return_status=True)
    assert int(st.item()) == 4
    out = H.centerhead_targets_batched(pb, pl, pc, TASKS, CFG_SIX, return_status=True)
    assert int(out[4].item()) == 1               # labels of no task are dropped silently, as in the reference
    want = O.targets(boxes, labels, counts, "transfusion", [10], CFG_TF)
    assert want["status"] == 4 and ulps(hm.cpu().numpy(), want["heatmaps"][0]).max() <= 1
    got = run(H, cuda, "centerhead", CFG_SIX, boxes, labels, counts)
    compare(got, O.targets(boxes, labels, counts, "centerhead", TASK_CLASSES, CFG_SIX, 500), 1, "status case")


def reference_draw(heatmap, center, radius, k=1):
    """gaussian.py:24-52 restated on a CPU torch tensor (the slicing and torch.max of the reference)."""
    x, y = int(center[0]), int(center[1])
    height, width = heatmap.shape[0:2]
    left, right = min(x, radius), min(width - x, radius + 1)
    top, bottom = min(y, radius), min(height - y, radius + 1)
    masked_heatmap = heatmap[y - top:y + bottom, x - left:x + right]
    masked_gaussian = torch.from_numpy(O.gaussian_2d(radius)[radius - top:radius + bottom,
                                                             radius - left:radius + right]).to(torch.float32)
    if min(masked_gaussian.shape) > 0 and min(masked_heatmap.shape) > 0:
        torch.max(masked_heatmap, masked_gaussian * k, out=masked_heatmap)
    return heatmap


@pytest.mark.parametrize("signed", [False, True])
def test_draw_heatmap_gaussian_mirror(cuda, H, signed):
    """Against the reference's slicing and torch.max: centres on and off the map, k = 1, 0, 2.5 and -1; with
    signed, the heatmap also holds negative values and a NaN, which cells where k * gaussian is 0 do not keep."""
    rng = np.random.default_rng(3)
    plane = rng.uniform(-0.5 if signed else 0.0, 0.5, (37, 53)).astype(np.float32)
    plane[::7, ::5] = 0.0
    if signed:
        plane[21, 11] = np.nan
    dev_plane = torch.from_numpy(plane.copy()).to(cuda)
    want = torch.from_numpy(plane.copy())
    draws = [(10, 20, 3, 1), (0, 0, 2, 1), (-3, 5, 3, 1), (-4, 5, 3, 1), (52, 36, 5, 1), (55, 10, 2, 1),
             (56, 10, 2, 1), (20, -2, 4, 1), (20, 40, 4, 1), (30, 18, 0, 1), (12, 22, 6, 0), (40, 8, 3, 2.5),
             (33, 30, 4, -1), (11, 21, 2, 1)]
    if not signed:
        draws.append((25, 25, 40, 1))                      # a window larger than the map
    for x, y, r, k in draws:
        H.draw_heatmap_gaussian(dev_plane, torch.tensor([x, y], dtype=torch.int32), r, k)
        reference_draw(want, (x, y), r, k)
    torch.cuda.synchronize()
    got, want = dev_plane.cpu().numpy(), want.numpy()
    assert ulps(got, want).max() <= 1
    assert np.array_equal(np.isnan(got), np.isnan(want))
    if signed:
        assert (want < 0).any() and np.isnan(want[21, 11])
        assert (want[22:29, 6:19] >= 0).all() and (got[22:29, 6:19] >= 0).all()   # k = 0 window, below the NaN
        assert (want[26:35, 29:38] < 0).any()              # k = -1 leaves negative cells negative


def test_cpu_boxes_with_cuda_labels(cuda, H):
    """The reference's data pipeline keeps gt_bboxes_3d on the CPU (formating.py:122-124) and the labels on the
    device; the list forms take that as it comes, equal to the all-CUDA call."""
    from bevfusion_b200 import synthetic as S

    class Boxes:
        def __init__(self, t):
            self.tensor = t
    bl, ll = S.gt_boxes(seed=12, batch=3)
    bl[2] = bl[2][:0]
    ll[2] = ll[2][:0]
    lab = [l.to(cuda) for l in ll]
    on_dev = H.centerhead_targets([b.to(cuda) for b in bl], lab, TASKS, CFG_SIX)
    on_cpu = H.centerhead_targets([Boxes(b) for b in bl], lab, TASKS, CFG_SIX)
    mixed = H.centerhead_targets([Boxes(bl[0]), Boxes(bl[1].to(cuda)), Boxes(bl[2].double())], lab, TASKS, CFG_SIX)
    for x, y, z in zip(on_dev, on_cpu, mixed):
        for u, v, w in zip(x, y, z):
            assert u.device == v.device == w.device == lab[0].device
            assert torch.equal(u, v) and torch.equal(u, w)
    t_dev = H.transfusion_heatmap_targets([b.to(cuda) for b in bl], lab, 10, CFG_TF)
    t_cpu = H.transfusion_heatmap_targets([Boxes(b) for b in bl], lab, 10, CFG_TF)
    assert torch.equal(t_dev, t_cpu) and t_cpu.is_cuda
    assert on_dev[3][0].sum() > 0
    with pytest.raises(RuntimeError):                          # the labels decide the device: CUDA only
        H.centerhead_targets([Boxes(b) for b in bl], ll, TASKS, CFG_SIX)
