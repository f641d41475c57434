"""centerhead_decode on the device against the reference's lines (centerpoint_bbox_coders.py:62-225,
centerpoint.py:637-757) restated with torch on the same GPU and stable sorts (centerhead_decode_oracle): cell index,
labels, counts, scores, x, y, z and velocity bit for bit, sizes and yaw within 2 ulp, over batch, task sets, map
shapes, max_num, the optional maps, the score threshold and both activation flags; edge planes; agreement with the
reference's unstable top-k where there is no tie; the whole get_bboxes against restatement -> centerhead_nms -> merge;
determinism, a CUDA-graph replay, the launch count and the absence of synchronising calls; refused calls."""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
import centerhead_decode_oracle as O  # noqa: E402
from bevfusion_b200 import _C, iou3d  # noqa: E402
from bevfusion_b200 import centerhead_decode as CD  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402

pytestmark = pytest.mark.gpu

SHAPES = [(128, 128), (180, 180), (7, 13), (200, 90)]
TASK_SETS = {"six": [1, 2, 2, 1, 2, 2], "one": [1], "ten": [10], "sixteen": [1, 2, 3] * 5 + [1]}
NUM_CLASSES = [len(c) for c in S.CENTERHEAD_TASKS]
MAX_ULP = 2        # sizes (expf) and yaw (atan2f) against torch's kernels


def ordered(x):
    i = x.contiguous().view(torch.int32).long()
    return torch.where(i < 0, -(i & 0x7fffffff), i)


def assert_bits(got, want, what, ulp=0):
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    if not got.is_floating_point():
        assert torch.equal(got, want), "%s: %d differ" % (what, int((got != want).sum()))
        return
    assert torch.equal(torch.isnan(got), torch.isnan(want)), "%s NaN positions" % what
    d = (ordered(got) - ordered(want)).abs().masked_fill(torch.isnan(want), 0)
    assert int(d.max()) <= ulp if d.numel() else True, "%s: up to %d ulp, %d differ" % (what, int(d.max()),
                                                                                         int((d > ulp).sum()))


def random_tasks(gen, cats, B, H, W, dev, reg=True, vel=True):
    def r(c, scale=1.0, shift=0.0):
        return torch.randn((B, c, H, W), generator=gen, device=dev) * scale + shift
    return [dict(heatmap=r(c, 2.5, -2.0), height=r(1), dim=r(3, 0.7, 0.5), rot=r(2),
                 **(dict(reg=torch.rand((B, 2, H, W), generator=gen, device=dev)) if reg else {}),
                 **(dict(vel=r(2, 3.0)) if vel else {})) for c in cats]


def activated(task, heat_is_logit, dim_is_log):
    return dict(heatmap=task["heatmap"].sigmoid() if heat_is_logit else task["heatmap"], reg=task.get("reg"),
                height=task["height"], dim=torch.exp(task["dim"]) if dim_is_log else task["dim"], rot=task["rot"],
                vel=task.get("vel"))


def check_decode(tasks, cfg, heat_is_logit=True, dim_is_log=True, what="", stable=True):
    """the native decode of `tasks` against the restatement, task by task; returns the native counts"""
    boxes, scores, labels, counts, index = CD.centerhead_decode_batched(tasks, cfg, heat_is_logit, dim_is_log,
                                                                        with_index=True)
    B = tasks[0]["heatmap"].shape[0]
    assert labels.dtype == torch.float32 and counts.dtype == torch.int32 and index.dtype == torch.int32
    for t, task in enumerate(tasks):
        wb, ws, wl, wi, wc = O.compact(O.torch_decode(activated(task, heat_is_logit, dim_is_log), cfg, stable))
        seg, w = slice(t * B, (t + 1) * B), (what, "task", t)
        assert_bits(counts[seg], wc, (w, "counts"))
        assert_bits(index[seg], wi.int(), (w, "index"))
        assert_bits(labels[seg], wl, (w, "labels"))
        assert_bits(scores[seg], ws, (w, "scores"))
        assert_bits(boxes[seg][..., :3], wb[..., :3], (w, "centre"))
        assert_bits(boxes[seg][..., 3:7], wb[..., 3:7], (w, "size and yaw"), MAX_ULP)
        assert_bits(boxes[seg][..., 7:], wb[..., 7:], (w, "velocity"))
    return counts


@pytest.mark.parametrize("maps", ["reg+vel", "reg", "vel", "none"])
@pytest.mark.parametrize("task_set", list(TASK_SETS))
def test_matches_stable_restatement_grid(cuda, task_set, maps):
    cats = TASK_SETS[task_set]
    gen = torch.Generator(device=cuda).manual_seed(100 * len(cats) + len(maps))
    thresholds, n, rejected = [None, 0.0, 0.1], 0, 0
    for B in (1, 2, 4):
        for H, W in SHAPES:
            if len(cats) * B * max(cats) * H * W > 6_000_000:      # the restatement's sorts, not the kernels, set this
                continue
            tasks = random_tasks(gen, cats, B, H, W, cuda, "reg" in maps, "vel" in maps)
            for K in (1, 83, 500, 4096, H * W):
                n += 1
                cfg = S.centerhead_coder_cfg(H, W, max_num=K, score_threshold=thresholds[n % 3])
                if K > min(H * W, CD.MAX_NUM):
                    with pytest.raises(ValueError):
                        CD.centerhead_decode_batched(tasks, cfg)
                    rejected += 1
                    continue
                logit = n % 2 == 0
                plain = [dict(t, heatmap=t["heatmap"].sigmoid(), dim=t["dim"].exp()) for t in tasks]
                check_decode(tasks if logit else plain, cfg, logit, logit, (task_set, maps, B, H, W, K))
    assert n > rejected > 0


@pytest.mark.parametrize("size", [(1, 128, 128), (4, 128, 128), (2, 180, 180)])
def test_matches_on_synthetic_head_outputs(cuda, size):
    B, H, W = size
    tasks = [{k: v.to(cuda) for k, v in t.items()} for t in S.centerhead_head_outputs(B + H, B, H, W)]
    for K in (83, 500, 4096):
        counts = check_decode(tasks, S.centerhead_coder_cfg(H, W, max_num=K), what=(size, K))
    assert bool((counts > 20).all()) and bool((counts < 4096).all())           # the threshold, not K, cuts


@pytest.mark.parametrize("size", [(1, 128, 128), (4, 128, 128)])
def test_agrees_with_unstable_topk_without_ties(cuda, size):
    B, H, W = size
    tasks = [{k: v.to(cuda) for k, v in t.items()} for t in S.centerhead_head_outputs(7 * B, B, H, W)]
    K = 100
    for t in tasks:
        top = t["heatmap"].sigmoid().flatten(1).sort(1, descending=True)[0][:, :K + 1]
        assert bool((top[:, :-1] > top[:, 1:]).all())                          # no tie in the top K + 1
    check_decode(tasks, S.centerhead_coder_cfg(H, W, max_num=K), stable=False)


def test_threshold_at_a_score_and_its_neighbours(cuda):
    tasks = [{k: v.to(cuda) for k, v in t.items()} for t in S.centerhead_head_outputs(3, 2)]
    v = tasks[1]["heatmap"].sigmoid().flatten(1).sort(1, descending=True)[0][0, 40]
    below, above = (torch.nextafter(v, torch.tensor(x, device=cuda)) for x in (0.0, 1.0))
    counts = [check_decode(tasks, S.centerhead_coder_cfg(max_num=500, score_threshold=float(th)), what=float(th))
              for th in (below, v, above)]
    B = 2
    assert int(counts[0][B]) == 41 and int(counts[1][B]) == 40 and int(counts[2][B]) <= 40   # strict >


def test_centres_on_the_range_limits_are_kept(cuda):
    gen = torch.Generator(device=cuda).manual_seed(5)
    H, W = 20, 24
    tasks = random_tasks(gen, [1], 2, H, W, cuda, reg=False)
    tasks[0]["height"].fill_(0.25)
    cfg = S.centerhead_coder_cfg(H, W, max_num=H * W, score_threshold=None)
    rows = (torch.arange(H, device=cuda).float() + 0.5) * cfg["out_size_factor"] * cfg["voxel_size"][0] \
        + cfg["pc_range"][0]
    cols = (torch.arange(W, device=cuda).float() + 0.5) * cfg["out_size_factor"] * cfg["voxel_size"][1] \
        + cfg["pc_range"][1]
    # the limits are centres of rows 3 and 15 and of columns 2 and 20, and the height itself
    cfg["post_center_range"] = [rows[3].item(), cols[2].item(), 0.25, rows[15].item(), cols[20].item(), 0.25]
    counts = check_decode(tasks, cfg)
    assert counts.tolist() == [13 * 19] * 2
    cfg["post_center_range"][2] = float(torch.nextafter(torch.tensor(0.25), torch.tensor(1.0)))
    assert check_decode(tasks, cfg).tolist() == [0, 0]


def edge_cases(dev):
    """(name, tasks, cfg, expected counts of the first task or None)"""
    gen = torch.Generator(device=dev).manual_seed(17)
    H, W = 64, 48
    cfg = S.centerhead_coder_cfg(H, W, max_num=500, score_threshold=0.1)
    wide = dict(cfg, post_center_range=[-1e30, -1e30, -1e30, 1e30, 1e30, 1e30])

    def base(cats=(2, 1), B=2):
        return random_tasks(gen, list(cats), B, H, W, dev)

    few = base()
    few[0]["heatmap"].fill_(-6.0)
    few[0]["heatmap"][0, 1, 5, 7] = few[0]["heatmap"][0, 0, 63, 47] = few[0]["heatmap"][1, 0, 0, 0] = 3.0
    yield "fewer_than_K_above", few, wide, [2, 1]
    none = base()
    none[0]["heatmap"].fill_(-6.0)
    yield "none_above", none, wide, [0, 0]
    allv = base()
    allv[0]["heatmap"].abs_()
    yield "all_above", allv, wide, [500, 500]
    equal = base()
    equal[0]["heatmap"].fill_(1.5)
    yield "all_equal", equal, wide, [500, 500]
    yield "all_equal_no_threshold", equal, dict(wide, score_threshold=None), [500, 500]
    sat = base()
    sat[0]["heatmap"].abs_().mul_(10).add_(17)                                 # sigmoid saturates at 1.0
    yield "saturated", sat, wide, [500, 500]
    nan = base()
    nan[0]["heatmap"][:, :, ::7, ::5] = float("nan")                           # 2 * 10 * 10 NaN cells per sample
    yield "nan_scores_take_places", nan, wide, None
    yield "nan_scores_no_threshold", nan, dict(wide, score_threshold=None), [500, 500]
    yield "all_nan_scores", [dict(nan[0], heatmap=torch.full_like(nan[0]["heatmap"], float("nan")))], wide, [0, 0]
    bad = base()
    for k, v in (("reg", float("nan")), ("height", float("inf")), ("dim", float("nan")), ("rot", float("inf")),
                 ("vel", -float("inf"))):
        bad[0][k][:, :, ::3, ::4] = v
        bad[1][k][:, :, 1::5, ::2] = v
    bad[0]["dim"][:, :, 1::3, ::4] = 200.0                                     # exp overflows
    yield "nan_inf_regression", bad, cfg, None
    yield "nan_inf_regression_wide", bad, dict(wide, score_threshold=0.0), None


EDGE_CASES = ["fewer_than_K_above", "none_above", "all_above", "all_equal", "all_equal_no_threshold", "saturated",
              "nan_scores_take_places", "nan_scores_no_threshold", "all_nan_scores", "nan_inf_regression",
              "nan_inf_regression_wide"]


@pytest.mark.parametrize("name", EDGE_CASES)
def test_edge_planes(cuda, name):
    _, tasks, cfg, want = next(c for c in edge_cases(cuda) if c[0] == name)
    counts = check_decode(tasks, cfg, what=name)
    if want is not None:
        assert counts[:2].tolist() == want
    if name == "nan_scores_take_places":
        # the 200 NaN cells of each sample hold 200 of the 500 places and are masked: 300 rows survive
        assert counts[:2].tolist() == [300, 300]


def test_padding_rows_are_zero(cuda):
    tasks = [{k: v.to(cuda) for k, v in t.items()} for t in S.centerhead_head_outputs(2, 2)]
    boxes, scores, labels, counts, index = CD.centerhead_decode_batched(tasks, S.centerhead_coder_cfg(),
                                                                        with_index=True)
    pad = torch.arange(500, device=cuda)[None, :] >= counts[:, None]
    assert bool(pad.any()) and bool((~pad).any())
    for v in (boxes, scores, labels, index):
        assert int(v[pad].count_nonzero()) == 0
    assert bool((scores[~pad] > 0.1).all())
    live = scores.masked_fill(pad, -float("inf"))
    assert bool((live[:, :-1] >= live[:, 1:]).all())                           # descending scores


@pytest.mark.parametrize("with_vel", [True, False])
def test_coder_decode_is_the_references(cuda, with_vel):
    B, H, W = 3, 40, 56
    raw = {k: v.to(cuda) for k, v in S.centerhead_head_outputs(4, B, H, W)[2].items()}
    cfg = S.centerhead_coder_cfg(H, W, max_num=83)
    maps = activated(raw, True, True)
    if not with_vel:
        maps["vel"] = None
    coder = CD.CenterPointBBoxCoder(**dict(cfg, code_size=9 if with_vel else 7))
    rot = raw["rot"]
    got = coder.decode(maps["heatmap"], rot[:, 0].unsqueeze(1), rot[:, 1].unsqueeze(1), maps["height"], maps["dim"],
                       maps["vel"], reg=maps["reg"], task_id=2)
    want = O.decode_lists(O.torch_decode(maps, cfg))
    assert len(got) == B
    for g, w in zip(got, want):
        assert g["labels"].dtype == torch.float32 and g["bboxes"].shape[1] == (9 if with_vel else 7)
        assert_bits(g["scores"], w["scores"], "scores")
        assert_bits(g["labels"], w["labels"], "labels")
        assert_bits(g["bboxes"], w["bboxes"], "bboxes", MAX_ULP)


def head_test_cfg(nms):
    cfg = dict(S.CENTERHEAD_TEST_CFG)
    if nms == "mixed":
        cfg.update(nms_type=list(S.CENTERHEAD_RADAR_NMS_TYPE), nms_scale=[list(s) for s in S.CENTERHEAD_RADAR_NMS_SCALE])
    else:
        cfg["nms_type"] = nms
    return cfg


@pytest.mark.parametrize("nms", ["circle", "rotate", "mixed"])
@pytest.mark.parametrize("batch", [1, 4])
def test_get_bboxes_equals_restatement_nms_merge(cuda, batch, nms):
    preds = [[{k: v.to(cuda) for k, v in t.items()}] for t in S.centerhead_head_outputs(10 + batch, batch)]
    coder, cfg = CD.CenterPointBBoxCoder(**S.centerhead_coder_cfg()), head_test_cfg(nms)
    got = CD.centerhead_get_bboxes(preds, coder, cfg, NUM_CLASSES)
    want = O.torch_get_bboxes(preds, S.centerhead_coder_cfg(), cfg, NUM_CLASSES, True, iou3d.centerhead_nms)
    assert len(got) == batch
    for (gb, gs, gl), (wb, ws, wl) in zip(got, want):
        assert gl.dtype == torch.int32 and 20 < len(gs) <= 6 * 83
        assert_bits(gl, wl, "labels")
        assert_bits(gs, ws, "scores")
        assert_bits(gb, wb, "bboxes", MAX_ULP)
        assert int(gl.max()) >= 8                                               # the last task's label offset
    bb, sc, lb, counts = CD.centerhead_get_bboxes_batched(preds, coder, cfg, NUM_CLASSES)
    assert bb.shape == (batch, 6 * 83, 9) and counts.dtype == torch.int32 and lb.dtype == torch.int32
    for i, (gb, gs, gl) in enumerate(got):
        n = int(counts[i])
        assert torch.equal(bb[i, :n], gb) and torch.equal(sc[i, :n], gs) and torch.equal(lb[i, :n], gl)
        assert int(bb[i, n:].count_nonzero()) == 0 and int(sc[i, n:].count_nonzero()) == 0
        assert int(lb[i, n:].count_nonzero()) == 0


def test_get_bboxes_without_norm_bbox_and_vel(cuda):
    preds = [[{k: v.to(cuda) for k, v in t.items() if k != "vel"}] for t in S.centerhead_head_outputs(8, 2, 64, 64)]
    for p in preds:
        p[0]["dim"] = p[0]["dim"].exp()
    ccfg, cfg = S.centerhead_coder_cfg(64, 64), head_test_cfg("mixed")
    got = CD.centerhead_get_bboxes(preds, ccfg, cfg, NUM_CLASSES, norm_bbox=False)
    want = O.torch_get_bboxes(preds, ccfg, cfg, NUM_CLASSES, False, iou3d.centerhead_nms)
    for g, w in zip(got, want):
        assert g[0].shape[1] == 7 and len(g[1]) > 0
        assert_bits(g[2], w[2], "labels")
        assert_bits(g[1], w[1], "scores")
        assert_bits(g[0], w[0], "bboxes", MAX_ULP)


def all_equal(a, b):
    return all(torch.equal(x.view(torch.int32) if x.is_floating_point() else x,
                           y.view(torch.int32) if y.is_floating_point() else y) for x, y in zip(a, b))


def test_repeated_calls_identical(cuda):
    gen = torch.Generator(device=cuda).manual_seed(23)
    tasks = random_tasks(gen, [1, 2, 2, 1, 2, 2], 4, 128, 128, cuda)
    for t in tasks:
        t["heatmap"] = (t["heatmap"] * 4).round() / 4                          # many ties
    cfg = S.centerhead_coder_cfg(max_num=500)
    first = CD.centerhead_decode_batched(tasks, cfg, with_index=True)
    for _ in range(5):
        assert all_equal(CD.centerhead_decode_batched(tasks, cfg, with_index=True), first)


def test_cuda_graph_replay(cuda):
    frames = [[[{k: v.to(cuda) for k, v in t.items()}] for t in S.centerhead_head_outputs(s, 2)] for s in (31, 32, 33)]
    static = [[{k: v.clone() for k, v in p[0].items()}] for p in frames[0]]
    coder, cfg = S.centerhead_coder_cfg(), head_test_cfg("mixed")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        CD.centerhead_get_bboxes_batched(static, coder, cfg, NUM_CLASSES)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = CD.centerhead_get_bboxes_batched(static, coder, cfg, NUM_CLASSES)
    for frame in frames[1:] + frames[:1]:
        for dst, src in zip(static, frame):
            for k in dst[0]:
                dst[0][k].copy_(src[0][k])
        g.replay()
        torch.cuda.synchronize()
        assert all_equal(out, CD.centerhead_get_bboxes_batched(frame, coder, cfg, NUM_CLASSES))
        assert int(out[3].min()) > 20


def test_launch_count_and_no_host_synchronisation(cuda):
    preds = [[{k: v.to(cuda) for k, v in t.items()}] for t in S.centerhead_head_outputs(41, 4)]
    tasks = [p[0] for p in preds]
    coder, cfg = S.centerhead_coder_cfg(), head_test_cfg("mixed")
    CD.centerhead_decode_batched(tasks, coder)
    want = CD.centerhead_get_bboxes_batched(preds, coder, cfg, NUM_CLASSES)
    torch.cuda.synchronize()
    n0 = _C.launch_count()
    CD.centerhead_decode_batched(tasks, coder)
    assert _C.launch_count() - n0 == 2                      # all six tasks and four samples
    # torch refuses every synchronising call in this mode: a device-to-host copy, .item(), a pageable upload
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = CD.centerhead_get_bboxes_batched(preds, coder, cfg, NUM_CLASSES)
        with pytest.raises(RuntimeError):                   # the list form reads the counts back once
            CD.centerhead_get_bboxes(preds, coder, cfg, NUM_CLASSES)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert all_equal(got, want)


def test_refused_calls_leave_outputs_untouched(cuda):
    tasks = random_tasks(torch.Generator(device=cuda).manual_seed(1), [2, 1], 2, 16, 16, cuda)
    T, B, H, W, K = 2, 2, 16, 16, 100
    outs = [torch.full((T * B, K, 9), 7.0, device=cuda), torch.full((T * B, K), 7.0, device=cuda),
            torch.full((T * B, K), 7.0, device=cuda), torch.full((T * B, K), 7, dtype=torch.int32, device=cuda),
            torch.full((T * B,), 7, dtype=torch.int32, device=cuda)]
    ws = torch.empty(CD.workspace_bytes([2, 1], B, H, W), dtype=torch.uint8, device=cuda)
    table = {k: _C.host_array(ctypes.c_void_p, [t[k].data_ptr() for t in tasks]) for k in tasks[0]}
    rng = _C.host_array(ctypes.c_double, [-60.0, -60.0, -10.0, 60.0, 60.0, 10.0])

    def call(cats=(2, 1), K=K, B=B, T=T, ws_bytes=ws.numel(), rng=rng, heat="heatmap"):
        return _C.lib().bevb200_centerhead_decode(
            table[heat] if heat else None, table["reg"], table["height"], table["dim"], table["rot"], table["vel"],
            _C.host_array(ctypes.c_int, cats), T, B, H, W, K, 1, 1, 8.0, 0.1, 0.1, -54.0, -54.0, rng, 1, 0.1,
            *[o.data_ptr() for o in outs], ws.data_ptr(), ws_bytes, _C.current_stream(cuda))

    for kw, rc in ((dict(K=0), -1), (dict(K=H * W + 1), -1), (dict(K=4097), -4), (dict(cats=(65, 1)), -4),
                   (dict(cats=(0, 1)), -1), (dict(B=0), -1), (dict(T=17, cats=(1,) * 17), -4), (dict(rng=None), -1),
                   (dict(heat=None), -1), (dict(ws_bytes=ws.numel() - 256), -3)):
        assert call(**kw) == rc, kw
    torch.cuda.synchronize()
    assert all(bool((o == 7).all()) for o in outs)
    assert call() == 0
    torch.cuda.synchronize()
    got = CD.centerhead_decode_batched(
        tasks, dict(S.centerhead_coder_cfg(H, W, max_num=K), voxel_size=[0.1, 0.1], pc_range=[-54.0, -54.0],
                    post_center_range=[-60.0, -60.0, -10.0, 60.0, 60.0, 10.0]), with_index=True)
    assert all_equal([outs[0], outs[1], outs[2], outs[4], outs[3]], got)
