"""The CenterHead box decode's specification on the CPU: the numpy restatement (centerhead_decode_oracle) against the
reference's own coder (the golden fixture) and against a torch-CPU restatement with stable sorts on tie-heavy planes;
the host-side validation of centerhead_decode and of the C entry point; the workspace query; the coder's signature."""
import ctypes
import inspect
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
import centerhead_decode_oracle as O  # noqa: E402
from bevfusion_b200 import _C  # noqa: E402
from bevfusion_b200 import centerhead_decode as CD  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "centerhead_decode_tiny.npz")
MAPS = ("heatmap", "reg", "height", "dim", "rot", "vel")


def golden_case(name):
    g = np.load(GOLDEN)
    maps = {k: g["%s_%s" % (name, k)] if "%s_%s" % (name, k) in g else None for k in MAPS}
    osf, K, thr = g[name + "_cfg"]
    cfg = dict(pc_range=list(g[name + "_pc_range"]), voxel_size=list(g[name + "_voxel_size"]),
               post_center_range=list(g[name + "_post_center_range"]), out_size_factor=int(osf), max_num=int(K),
               score_threshold=None if thr < 0 else float(thr))
    return maps, cfg, {k: g["%s_out_%s" % (name, k)] for k in ("bboxes", "scores", "labels", "counts")}


@pytest.mark.parametrize("case", ["two", "plain", "tight"])
def test_oracle_reproduces_reference_golden(case):
    maps, cfg, want = golden_case(case)
    d = O.decode(maps, cfg)
    np.testing.assert_array_equal(d["mask"].sum(1), want["counts"])
    m = d["mask"]
    np.testing.assert_array_equal(d["scores"][m].view(np.uint32), want["scores"].view(np.uint32))
    assert want["labels"].dtype == np.float32
    np.testing.assert_array_equal(d["labels"][m], want["labels"])
    got = d["boxes"][m]
    assert got.shape == want["bboxes"].shape
    other = [c for c in range(got.shape[1]) if c != 6]
    np.testing.assert_array_equal(got[:, other].view(np.uint32), want["bboxes"][:, other].view(np.uint32))
    np.testing.assert_allclose(got[:, 6], want["bboxes"][:, 6], rtol=3e-7, atol=0)   # numpy's atan2 against torch's


def tie_heavy_cases():
    """(name, maps of torch tensors, cfg): score planes whose top max_num is full of ties."""
    g = torch.Generator().manual_seed(9)

    def case(heat, K, thr, reg=True, vel=True):
        B, _, H, W = heat.shape
        r = lambda c, scale=1.0: torch.randn((B, c, H, W), generator=g) * scale       # noqa: E731
        maps = dict(heatmap=heat, reg=torch.rand((B, 2, H, W), generator=g) if reg else None, height=r(1),
                    dim=r(3).exp(), rot=r(2), vel=r(2, 3.0) if vel else None)
        return maps, S.centerhead_coder_cfg(H, W, extent=40.0, max_num=K, score_threshold=thr)

    yield ("constant",) + case(torch.full((2, 2, 9, 11), 0.3), 60, 0.1)
    yield ("saturated",) + case((torch.rand((2, 3, 10, 13), generator=g) * 30 + 20).sigmoid(), 90, None)
    yield ("underflow",) + case(torch.full((1, 10, 8, 8), -150.0).sigmoid(), 50, 0.0, reg=False)
    yield ("plateau",) + case(torch.randint(0, 4, (1, 4, 7, 13), generator=g).float() / 4, 91, 0.25, vel=False)
    odd = torch.randn((2, 2, 10, 12), generator=g).sigmoid()
    odd[0, 1, 4, 4] = odd[0, 0, 0, 5] = odd[1, 1, 9, 11] = float("nan")
    odd[1, 0, 6, 6] = odd[1, 0, 6, 7] = float("inf")
    odd[1, 1, 2, 2] = -float("inf")
    yield ("nan_inf",) + case(odd, 30, 0.4)
    yield ("nan_no_threshold",) + case(odd.clone(), 30, None)


@pytest.mark.parametrize("case", list(tie_heavy_cases()), ids=lambda c: c[0])
def test_oracle_matches_stable_torch_restatement(case):
    _, maps, cfg = case
    want = O.torch_decode(maps, cfg, stable=True)
    got = O.decode({k: None if v is None else v.numpy() for k, v in maps.items()}, cfg)
    np.testing.assert_array_equal(got["index"], want["index"].numpy())
    np.testing.assert_array_equal(got["labels"], want["labels"].numpy())
    np.testing.assert_array_equal(got["mask"], want["mask"].numpy())
    np.testing.assert_array_equal(got["scores"].view(np.uint32), want["scores"].numpy().view(np.uint32))
    other = [c for c in range(got["boxes"].shape[2]) if c != 6]
    np.testing.assert_array_equal(got["boxes"][..., other], want["boxes"].numpy()[..., other])
    np.testing.assert_allclose(got["boxes"][..., 6], want["boxes"].numpy()[..., 6], rtol=3e-7, atol=0)


def test_synthetic_head_outputs():
    tasks = S.centerhead_head_outputs(seed=0, batch=2)
    assert [t["heatmap"].shape[1] for t in tasks] == [len(c) for c in S.CENTERHEAD_TASKS]
    for t in tasks:
        assert all(t[k].shape == (2, c, 128, 128) and t[k].dtype == torch.float32
                   for k, c in (("reg", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2)))
        above = (t["heatmap"].sigmoid() > 0.1).flatten(1).sum(1)
        assert bool((above > 50).all()) and bool((above < 2000).all()), above


def _cpu(shape, dtype=torch.float32):
    return torch.zeros(1, dtype=dtype).expand(*shape)   # shape only: no storage behind it


def _task(B=1, cat=2, H=16, W=16, dtype=torch.float32, **over):
    t = dict(heatmap=_cpu((B, cat, H, W), dtype), reg=_cpu((B, 2, H, W), dtype), height=_cpu((B, 1, H, W), dtype),
             dim=_cpu((B, 3, H, W), dtype), rot=_cpu((B, 2, H, W), dtype), vel=_cpu((B, 2, H, W), dtype))
    t.update(over)
    return {k: v for k, v in t.items() if v is not None}


CFG = S.centerhead_coder_cfg(16, 16, max_num=100)


@pytest.mark.parametrize("tasks, cfg, match", [
    ([_task()], dict(CFG, max_num=0), "max_num"),
    ([_task()], dict(CFG, max_num=257), "max_num"),
    ([_task(H=80, W=80)], dict(CFG, max_num=4097), "at most"),
    ([_task(cat=65)], CFG, "at most"),
    ([_task(cat=2, H=4096, W=4096)], CFG, "at most"),
    ([_task()] * 17, CFG, "at most"),
    ([_task(B=65536 // 4)] * 4, CFG, "at most"),
    ([_task(), _task(H=8)], CFG, "in every task"),
    ([_task(), _task(B=2)], CFG, "in every task"),
    ([_task(rot=_cpu((1, 1, 16, 16)))], CFG, "in every task"),
    ([_task(), _task(reg=None)], CFG, "every task or in none"),
    ([_task(), _task(vel=None)], CFG, "every task or in none"),
    ([_task(dim=None)], CFG, "needs 'dim'"),
    ([_task(cat=0)], CFG, "empty"),
    ([], CFG, "non-empty"),
    ([_task(dtype=torch.float16)], CFG, "fp32"),
    ([_task(dtype=torch.float64)], CFG, "fp32"),
    ([_task()], dict(CFG, post_center_range=[0.0] * 5), "six"),
    ([_task()], CFG, "CUDA tensor"),
])
def test_rejected_inputs_raise(tasks, cfg, match):
    with pytest.raises(ValueError, match=match):
        CD.centerhead_decode_batched(tasks, cfg)


def test_missing_post_center_range_raises_as_the_reference():
    with pytest.raises(NotImplementedError):
        CD.centerhead_decode_batched([_task()], dict(CFG, post_center_range=None))
    coder = CD.CenterPointBBoxCoder([-54.0, -54.0], 8, [0.075, 0.075])
    z = torch.zeros(1, 1, 8, 8)
    with pytest.raises(NotImplementedError):
        coder.decode(z, z, z, z, torch.zeros(1, 3, 8, 8), None)


def test_cpu_tensors_raise():
    coder = CD.CenterPointBBoxCoder(**S.centerhead_coder_cfg(8, 8, max_num=10))
    z = torch.zeros(1, 1, 8, 8)
    with pytest.raises(ValueError, match="CUDA tensor"):
        coder.decode(z, z, z, z, torch.zeros(1, 3, 8, 8), torch.zeros(1, 2, 8, 8))
    preds = [[t] for t in S.centerhead_head_outputs(0, 1, 8, 8)]
    test_cfg = dict(S.CENTERHEAD_TEST_CFG, nms_type="rotate")
    for fn in (CD.centerhead_get_bboxes, CD.centerhead_get_bboxes_batched):
        with pytest.raises(ValueError, match="CUDA tensor"):
            fn(preds, coder, test_cfg, [1, 2, 2, 1, 2, 2])


def test_coder_signature_is_the_references():
    init = inspect.signature(CD.CenterPointBBoxCoder.__init__)
    assert [(p.name, p.default) for p in list(init.parameters.values())[1:]] == [
        ("pc_range", inspect.Parameter.empty), ("out_size_factor", inspect.Parameter.empty),
        ("voxel_size", inspect.Parameter.empty), ("post_center_range", None), ("max_num", 100),
        ("score_threshold", None), ("code_size", 9)]
    dec = inspect.signature(CD.CenterPointBBoxCoder.decode)
    assert [(p.name, p.default) for p in list(dec.parameters.values())[1:]] == [
        ("heat", inspect.Parameter.empty), ("rot_sine", inspect.Parameter.empty),
        ("rot_cosine", inspect.Parameter.empty), ("hei", inspect.Parameter.empty), ("dim", inspect.Parameter.empty),
        ("vel", inspect.Parameter.empty), ("reg", None), ("task_id", -1)]
    assert CD.CenterPointBBoxCoder([0, 0], 8, [0.1, 0.1]).encode() is None


def test_symbols_declared_and_exported():
    for name in ("bevb200_centerhead_decode_workspace_bytes", "bevb200_centerhead_decode"):
        assert name in _C.declared_symbols() and name in _C._SIGNATURES
        assert getattr(_C.lib(), name)
    header = open(_C.HEADER_PATH).read()
    for macro, value in (("MAX_TASKS", CD.MAX_TASKS), ("MAX_SEGMENTS", CD.MAX_SEGMENTS),
                         ("MAX_CLASSES", CD.MAX_CLASSES), ("MAX_K", CD.MAX_NUM)):
        assert "#define BEVB200_DECODE_%s %d" % (macro, value) in header
    assert "#define BEVB200_DECODE_MAX_CELLS (1 << 24)" in header and CD.MAX_CELLS == 1 << 24


@pytest.mark.parametrize("size", [([1, 2, 2, 1, 2, 2], 4, 128, 128), ([10], 1, 180, 180), ([1], 2, 7, 13),
                                  ([3] * 16, 3, 200, 90)])
def test_workspace_bytes_documented(size):
    cats, B, H, W = size
    tl = -(-max(cats) * H * W // 1024)
    align = lambda n: -(-n // 256) * 256                                     # noqa: E731
    assert CD.workspace_bytes(cats, B, H, W) == align(8 * len(cats) * B * tl * 1024) + align(4 * len(cats) * B * tl)


@pytest.mark.parametrize("size", [([1] * 17, 1, 8, 8), ([65], 1, 8, 8), ([1], 1, 4097, 4097), ([1, 0], 1, 8, 8),
                                  ([1], 0, 8, 8), ([1] * 16, 4096, 8, 8), ([1], 1, 0, 8)])
def test_workspace_bytes_zero_when_unsupported(size):
    assert CD.workspace_bytes(*size) == 0


def _c_call(cats=(1, 2), B=1, H=16, W=16, K=100, null=False, no_range=False, ws_bytes=1 << 30):
    L = _C.lib()
    T = len(cats)
    p = 256                        # never dereferenced: every case below is refused before any device work
    table = _C.host_array(ctypes.c_void_p, [None if null else p] * T)
    rng = None if no_range else _C.host_array(ctypes.c_double, [-1.0] * 3 + [1.0] * 3)
    return L.bevb200_centerhead_decode(table, table, table, table, table, table, _C.host_array(ctypes.c_int, cats),
                                       T, B, H, W, K, 1, 1, 8.0, 0.1, 0.1, -50.0, -50.0, rng, 1, 0.1, p, p, p, None,
                                       p, p, ws_bytes, None)


@pytest.mark.parametrize("kw, rc", [
    (dict(K=0), -1), (dict(K=257), -1), (dict(B=0), -1), (dict(H=0), -1), (dict(cats=(1, 0)), -1),
    (dict(null=True), -1), (dict(no_range=True), -1), (dict(K=4097, H=80, W=80), -4), (dict(cats=(65,)), -4),
    (dict(cats=(1,) * 17), -4), (dict(cats=(1,) * 16, B=4096), -4), (dict(cats=(2,), H=4096, W=4096), -4),
    (dict(ws_bytes=0), -3),
])
def test_c_entry_rejects(kw, rc):
    assert _c_call(**kw) == rc
    assert _C.lib().bevb200_last_error()
