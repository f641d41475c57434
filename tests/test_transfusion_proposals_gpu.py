"""transfusion_proposals on the device against the reference's lines (transfusion.py:238-274 and :322-325) restated
with torch on the same GPU and argsort(stable=True): labels, index and query_heatmap_score bit for bit (NaN where the
restatement has NaN), over batch, classes, map shape, kernel, dataset, num_proposals and dtype, on realistic and
tie-heavy planes; agreement with the reference's unstable argsort where its top K has no ties; determinism, a CUDA
graph replay and the launch count."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
import transfusion_proposals_oracle as O  # noqa: E402
from bevfusion_b200 import _C  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200.transfusion_proposals import MAX_PROPOSALS, transfusion_proposals  # noqa: E402
from test_transfusion_proposals_cpu import tie_heavy_cases  # noqa: E402

pytestmark = pytest.mark.gpu

SHAPES = [(128, 128), (180, 180), (7, 13), (200, 90)]
DATASETS = ["nuScenes", "Waymo", "none"]


def assert_same(got, want, what=""):
    gl, gi, gs = got
    wl, wi, ws = want
    assert gl.dtype == torch.int64 and gi.dtype == torch.int64 and gs.dtype == ws.dtype, what
    assert torch.equal(gl, wl), "%s labels: %d differ" % (what, int((gl != wl).sum()))
    assert torch.equal(gi, wi), "%s index: %d differ" % (what, int((gi != wi).sum()))
    assert torch.equal(torch.isnan(gs), torch.isnan(ws)), "%s score NaN positions" % what
    bits = torch.int16 if gs.dtype == torch.float16 else torch.int32
    same = (gs.view(bits) == ws.view(bits)) | torch.isnan(ws)
    assert bool(same.all()), "%s score: %d differ" % (what, int((~same).sum()))


def random_logits(gen, shape, dtype, dev):
    """Logits around the sigmoid's working range; fp16 rounding leaves ties on the plane."""
    x = torch.randn(shape, generator=gen, device=dev) * 2.5 - 2.0
    return x.to(dtype)


def valid(B, C, H, W, K, k, dataset):
    return (all(c < C for c in O.EXEMPT.get(dataset, ())) and H >= k and W >= k and 1 <= K <= C * H * W
            and K <= MAX_PROPOSALS)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("dataset", DATASETS)
@pytest.mark.parametrize("k", [3, 5, 7])
def test_matches_stable_restatement_grid(cuda, dtype, dataset, k):
    gen = torch.Generator(device=cuda).manual_seed(1000 * k + DATASETS.index(dataset) * 10 + (dtype == torch.half))
    checked = rejected = 0
    for B in (1, 2, 4):
        for C in (3, 10, 17):
            for H, W in SHAPES:
                x = random_logits(gen, (B, C, H, W), dtype, cuda)
                ref = None
                for K in (1, 200, 1000, C * H * W):
                    if not valid(B, C, H, W, K, k, dataset):
                        with pytest.raises(ValueError):
                            transfusion_proposals(x, K, k, dataset)
                        rejected += 1
                        continue
                    if ref is None:   # the stable order's prefix serves every K
                        ref = O.torch_proposals(x, C * H * W, k, dataset, stable=True)
                    want = (ref[0][:, :K], ref[1][:, :K], ref[2][:, :, :K].contiguous())
                    assert_same(transfusion_proposals(x, K, k, dataset), want, (B, C, H, W, K))
                    checked += 1
    assert checked > 0 and rejected > 0


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("size", [(1, 128, 128), (4, 128, 128), (1, 180, 180), (4, 180, 180)])
def test_matches_on_synthetic_heatmaps(cuda, dtype, size):
    B, H, W = size
    x = S.transfusion_heatmap(seed=B + H, batch=B, height=H, width=W, dtype=dtype).to(cuda)
    for K in (200, 1000, MAX_PROPOSALS):
        assert_same(transfusion_proposals(x, K), O.torch_proposals(x, K, 3, "nuScenes"), (size, K))


@pytest.mark.parametrize("case", list(tie_heavy_cases()), ids=lambda c: c[0])
def test_tie_heavy_edge_cases(cuda, case):
    _, x, K, k, dataset = case
    x = x.to(cuda)
    assert_same(transfusion_proposals(x, K, k, dataset), O.torch_proposals(x, K, k, dataset))


def edge_planes(dev):
    g = torch.Generator(device=dev).manual_seed(3)
    yield "constant", torch.full((2, 10, 128, 128), 1.5, device=dev), 200, "nuScenes"
    yield "underflow", torch.full((4, 10, 180, 180), -125.0, device=dev), 200, "nuScenes"
    few = torch.full((1, 10, 128, 128), -140.0, device=dev)
    few[0, 0, 10:13, 40:43] = 2.0                                            # a 3 x 3 plateau: nine peaks
    few[0, 3, 0, 17] = 3.0                                                   # border band: masked
    few[0, 8, 0, 0] = 1.0                                                    # exempt class: a peak
    few[0, 5, 64, 64] = float("nan")
    yield "few_peaks", few, 1000, "nuScenes"
    yield "saturated", torch.rand((2, 10, 128, 128), generator=g, device=dev) * 40 + 17, 4096, "Waymo"
    odd = torch.randn((4, 10, 180, 180), generator=g, device=dev) * 3
    odd[:, :, ::37, ::41] = float("nan")
    odd[:, :, 0, ::3] = float("nan")                                         # border band
    odd[:, :, 5::29, 7::31] = float("inf")
    odd[:, :, 11::23, 2::19] = -float("inf")
    yield "nan_inf", odd, 1000, "nuScenes"
    yield "all_nan", torch.full((1, 3, 9, 9), float("nan"), device=dev), 243, "none"


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("name", ["constant", "underflow", "few_peaks", "saturated", "nan_inf", "all_nan"])
def test_edge_planes(cuda, dtype, name):
    _, x, K, dataset = next(c for c in edge_planes(cuda) if c[0] == name)
    x = x.to(dtype)
    assert_same(transfusion_proposals(x, K, 3, dataset), O.torch_proposals(x, K, 3, dataset), name)


@pytest.mark.parametrize("size", [(1, 128, 128), (4, 128, 128), (2, 180, 180)])
def test_agrees_with_unstable_argsort_without_ties(cuda, size):
    B, H, W = size
    x = S.transfusion_heatmap(seed=7 * B + H, batch=B, height=H, width=W).to(cuda)
    K = 200
    want = O.torch_proposals(x, K + 1, 3, "nuScenes", stable=False)
    vals = torch.gather(want[2], 1, want[0][:, None, :]).squeeze(1)
    assert bool((vals[:, :-1] > vals[:, 1:]).all())                          # no tie in the top K + 1
    assert_same(transfusion_proposals(x, K), (want[0][:, :K], want[1][:, :K], want[2][:, :, :K].contiguous()))


def test_repeated_calls_identical(cuda):
    g = torch.Generator(device=cuda).manual_seed(11)
    x = (torch.randn((4, 10, 180, 180), generator=g, device=cuda) * 0.5).half()   # fp16: many ties
    first = transfusion_proposals(x, 1000)
    for _ in range(5):
        assert_same(transfusion_proposals(x, 1000), first)


def test_cuda_graph_replay(cuda):
    xs = [S.transfusion_heatmap(seed=s, batch=2).to(cuda) for s in (21, 22, 23)]
    static_x = xs[0].clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        transfusion_proposals(static_x, 200)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        static_out = transfusion_proposals(static_x, 200)
    for x in xs[1:] + xs[:1]:
        static_x.copy_(x)
        g.replay()
        torch.cuda.synchronize()
        assert_same(static_out, transfusion_proposals(x, 200))
        assert_same(static_out, O.torch_proposals(x, 200, 3, "nuScenes"))


def test_kernel_count(cuda):
    x = S.transfusion_heatmap(seed=31, batch=4).to(cuda)
    transfusion_proposals(x, 200)
    torch.cuda.synchronize()
    n0 = _C.launch_count()
    transfusion_proposals(x, 200)
    assert _C.launch_count() - n0 == 2
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        transfusion_proposals(x, 200)
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and "Memcpy" not in e.name and "Memset" not in e.name]
    assert 1 <= len(kernels) <= 3, [e.name for e in kernels]
    assert all("tf_peak_kernel" in e.name or "tf_select_kernel" in e.name for e in kernels), [e.name for e in kernels]
    names = [e.name for e in prof.events()]
    assert not any("DtoH" in n or "Device -> Host" in n for n in names)
