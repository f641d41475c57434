"""TransFusion query selection's specification on the CPU: the numpy restatement (transfusion_proposals_oracle)
against the reference's own lines (the golden fixture) and against a torch-CPU restatement with the stable argsort on
tie-heavy planes; the host-side validation of transfusion_proposals and of the C entry point; the workspace query."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
import transfusion_proposals_oracle as O  # noqa: E402
from bevfusion_b200 import _C  # noqa: E402
from bevfusion_b200 import synthetic as S  # noqa: E402
from bevfusion_b200 import transfusion_proposals as TP  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "transfusion_proposals_tiny.npz")
DATASETS = ["nuScenes", "Waymo", "none"]


@pytest.mark.parametrize("case", ["nus", "waymo", "none", "half"])
def test_oracle_reproduces_reference_golden(case):
    g = np.load(GOLDEN)
    k, K, ds = (int(v) for v in g[case + "_cfg"])
    labels, index, score = O.proposals(g[case + "_sigmoid"], K, k, O.EXEMPT.get(DATASETS[ds], ()))
    np.testing.assert_array_equal(labels, g[case + "_labels"])
    np.testing.assert_array_equal(index, g[case + "_index"])
    assert score.dtype == g[case + "_score"].dtype
    np.testing.assert_array_equal(score.view(np.uint8), g[case + "_score"].view(np.uint8))


def tie_heavy_cases():
    """(name, logits [B, C, H, W], K, k, dataset): planes whose top K is full of ties."""
    g = torch.Generator().manual_seed(5)
    yield "constant", torch.full((2, 4, 9, 11), 0.3), 120, 3, "Waymo"
    yield "underflow", torch.full((1, 10, 8, 8), -150.0), 50, 3, "nuScenes"
    few = torch.full((1, 10, 12, 12), -130.0)
    few[0, 2, 5, 5], few[0, 9, 0, 0], few[0, 4, 0, 3] = 1.0, -1.0, 2.0      # three peaks (one in the border band)
    yield "few_peaks", few, 40, 3, "nuScenes"
    yield "saturated", torch.rand((2, 3, 10, 13), generator=g) * 30 + 20, 90, 5, "none"
    plateau = (torch.randint(-3, 3, (1, 10, 16, 16), generator=g).float() * 0.5).half()
    yield "fp16_plateau", plateau, 300, 3, "nuScenes"
    yield "fp16_near_one", (torch.rand((1, 3, 12, 12), generator=g) * 4 + 6).half(), 60, 3, "Waymo"
    odd = torch.randn((2, 10, 10, 12), generator=g)
    odd[0, 1, 4, 4] = float("nan")
    odd[0, 3, 0, 5] = float("nan")                                            # border band
    odd[0, 8, 3, 3] = float("nan")                                            # exempt class
    odd[1, 2, 6, 6] = float("inf")
    odd[1, 2, 6, 7] = float("inf")
    odd[1, 5, 2, 2] = -float("inf")
    yield "nan_inf", odd, 80, 3, "nuScenes"
    yield "k7_all", torch.randn((1, 3, 7, 9), generator=g), 189, 7, "Waymo"


@pytest.mark.parametrize("case", list(tie_heavy_cases()), ids=lambda c: c[0])
def test_oracle_matches_stable_torch_restatement(case):
    _, x, K, k, dataset = case
    want = O.torch_proposals(x, K, k, dataset, stable=True)
    got = O.proposals(x.sigmoid().numpy(), K, k, O.EXEMPT.get(dataset, ()))
    np.testing.assert_array_equal(got[0], want[0].numpy())
    np.testing.assert_array_equal(got[1], want[1].numpy())
    np.testing.assert_array_equal(np.isnan(got[2]), np.isnan(want[2].numpy()))
    np.testing.assert_array_equal(np.nan_to_num(got[2]), np.nan_to_num(want[2].numpy()))


def test_synthetic_heatmap_has_sparse_peaks():
    x = S.transfusion_heatmap(seed=0, batch=2)
    assert tuple(x.shape) == (2, 10, 128, 128) and x.dtype == torch.float32
    s = x.sigmoid().numpy()
    m = O.masked_plane(s, 3, ())
    frac = (m > 0).mean()
    assert 0.005 < frac < 0.1, frac                     # peaks, not a plateau nor iid noise (1 / 9)
    assert (m > 0.5).sum() > 40                         # the objects' blobs
    assert S.transfusion_heatmap(seed=0, batch=1, dtype=torch.float16).dtype == torch.float16


def _cpu(shape, dtype=torch.float32):
    return torch.zeros(1, dtype=dtype).expand(*shape)   # shape only: no storage behind it


@pytest.mark.parametrize("args, match", [
    (((1, 10, 16, 16), 200, 4, "nuScenes"), "odd"),
    (((1, 10, 16, 16), 200, 1, "nuScenes"), "odd"),
    (((1, 10, 16, 16), 200, 0, "nuScenes"), "odd"),
    (((1, 10, 4, 16), 10, 5, "nuScenes"), "smaller"),
    (((1, 10, 16, 4), 10, 5, "nuScenes"), "smaller"),
    (((1, 9, 16, 16), 10, 3, "nuScenes"), "exempt"),
    (((1, 2, 16, 16), 10, 3, "Waymo"), "exempt"),
    (((1, 3, 4, 4), 49, 3, "none"), "num_proposals"),
    (((1, 3, 4, 4), 0, 3, "none"), "num_proposals"),
    (((1, 3, 64, 64), 4097, 3, "none"), "at most"),
    (((1, 65, 8, 8), 10, 3, "none"), "at most"),
    (((1, 1, 4097, 4097), 10, 3, "none"), "at most"),
    (((1, 3, 32, 32), 10, 17, "none"), "at most"),
    (((65536, 1, 3, 3), 1, 3, "none"), "at most"),
    (((1, 0, 8, 8), 1, 3, "none"), "empty"),
    (((10, 16, 16), 10, 3, "none"), r"\[B, C, H, W\]"),
])
def test_rejected_inputs_raise(args, match):
    shape, K, k, dataset = args
    with pytest.raises(ValueError, match=match):
        TP.transfusion_proposals(_cpu(shape), K, k, dataset)


@pytest.mark.parametrize("dtype", [torch.float64, torch.bfloat16, torch.int32])
def test_other_dtypes_raise(dtype):
    with pytest.raises(ValueError, match="fp32 or fp16"):
        TP.transfusion_proposals(_cpu((1, 10, 16, 16), dtype), 200)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_cpu_tensors_raise(dtype):
    with pytest.raises(ValueError, match="CUDA tensor"):
        TP.transfusion_proposals(torch.zeros((1, 10, 16, 16), dtype=dtype), 200)


def test_exempt_classes():
    assert TP.exempt_classes("nuScenes") == (8, 9)
    assert TP.exempt_classes("Waymo") == (1, 2)
    assert TP.exempt_classes("Lyft") == () and TP.exempt_classes(None) == ()


@pytest.mark.parametrize("size", [(1, 10, 128, 128), (4, 10, 180, 180), (2, 3, 7, 13), (3, 17, 200, 90),
                                  (1, 64, 512, 512)])
def test_workspace_bytes_documented(size):
    B, C, H, W = size
    T = -(-C * H * W // 1024)
    align = lambda n: -(-n // 256) * 256                                     # noqa: E731
    assert TP.workspace_bytes(B, C, H, W) == align(8 * B * T * 1024) + align(4 * B * T)


@pytest.mark.parametrize("size", [(0, 10, 8, 8), (1, 0, 8, 8), (1, 10, 0, 8), (65536, 1, 8, 8), (1, 65, 8, 8),
                                  (1, 1, 4097, 4097), (-1, 10, 8, 8)])
def test_workspace_bytes_zero_when_unsupported(size):
    assert TP.workspace_bytes(*size) == 0


def _c_call(B=1, C=10, H=16, W=16, K=200, k=3, ex=(8, 9), dtype=0, null=False, ws_bytes=1 << 30):
    L = _C.lib()
    p = None if null else 256      # never dereferenced: every case below is refused before any device work
    return L.bevb200_transfusion_proposals(p, dtype, B, C, H, W, K, k, ex[0], ex[1], p, p, p, p, ws_bytes, None)


@pytest.mark.parametrize("kw, rc", [
    (dict(k=4), -1), (dict(k=1), -1), (dict(H=2), -1), (dict(W=2), -1), (dict(ex=(8, 10)), -1),
    (dict(ex=(-2, 1)), -1), (dict(K=0), -1), (dict(C=1, H=3, W=3, K=10, ex=(-1, -1)), -1), (dict(B=0), -1),
    (dict(null=True), -1), (dict(dtype=2), -4), (dict(K=4097, H=64, W=64), -4), (dict(C=65), -4),
    (dict(k=17, H=32, W=32), -4), (dict(ws_bytes=0), -3),
])
def test_c_entry_rejects(kw, rc):
    assert _c_call(**kw) == rc
    assert _C.lib().bevb200_last_error()
