"""GPU: the camera augmentation (image_aug_batched) bit-equal to the numpy restatement of Pillow + torchvision at
every tiling, tap-capacity and limit boundary of image_aug.cu (tests/data_pipeline_cases.py): crop widths on the
edges of the pass blocks, bands on the edges of the horizontal pass's row blocks, 1 x 1 frames, draws exactly at and
one step over the filter tables' width, 1 x 1 resizes of 1600 x 900 and large upscales, kMaxFrame-wide and -tall
frames through every rotate path, crops at the draw check's bound, the tallest input (more row blocks than grid.y
holds) and 65535 cameras.  Every call runs under head_boundaries.DeviceGuard: outputs and the workspace of exactly
the queried size sit in canary-filled buffers, and nothing outside them may change."""
import numpy as np
import pytest
import torch

import data_pipeline_cases as C
import image_aug_oracle as O
from head_boundaries import DeviceGuard

pytestmark = pytest.mark.gpu

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
CALLS = C.image_calls()


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def run(cuda, name, call):
    """one call of image_aug_batched on the case's cameras, checked camera by camera"""
    from bevfusion_b200 import image_aug as IA
    imgs = C.call_images(name, call)
    fH, fW = call["fH"], call["fW"]
    images = torch.from_numpy(imgs[None]).to(cuda)
    draws = torch.from_numpy(C.pack(call["draws"])[None]).to(cuda)
    with DeviceGuard(IA) as g:
        out, mat, status = IA.image_aug_batched(images, draws, (fH, fW), MEAN, STD, call["min_resize"],
                                                return_status=True)
        assert g.check(name) == 4                      # out, matrix, status, workspace
    want_status = 0
    for s in call["expect"]:
        want_status |= s
    assert int(status) == want_status, name
    out, mat = out[0].cpu().numpy(), mat[0].cpu()
    for n, ((resize, dims, xy, flip, rot), st) in enumerate(zip(call["draws"], call["expect"])):
        if st:
            assert np.isnan(out[n]).all() and bool(torch.isnan(mat[n]).all()), (name, n)
            continue
        want = O.augment(imgs[n], dims, xy, (fH, fW), flip, rot, MEAN, STD)
        assert bits_equal(out[n], want), (name, n, call["draws"][n])
        box = (xy[0], xy[1], xy[0] + fW, xy[1] + fH)
        assert torch.equal(mat[n], IA.img_aug_matrix(resize, box, flip, rot)), (name, n)


@pytest.mark.parametrize("name", [n for n in CALLS if n != "tall"])
def test_bit_equal_at_the_boundary(cuda, name):
    run(cuda, name, CALLS[name])


def test_tall_image_resamples_past_the_grid_limit(cuda):
    """in_h = kMaxSource - 1 needs more than kMaxGridY row blocks of kHpassRows.  Resized to kMaxFrame rows and
    cropped whole, every source row is in the band, and the last output rows depend on the rows past
    kMaxGridY * kHpassRows (the CPU twin checks that they change with them), which only the horizontal pass's second
    stride over the row blocks resamples"""
    run(cuda, "tall", CALLS["tall"])


def test_65535_cameras(cuda):
    """the grid.z limit: tiny images and draws repeating with coprime periods, every camera checked, the last
    included"""
    from bevfusion_b200 import image_aug as IA
    N = C.MAX_GRID
    base = np.stack([C.camera_image(100 + i, 3, 3) for i in range(C.CAM_IMAGES)])
    draws = C.many_camera_draws()
    cam = np.arange(N)
    images = torch.from_numpy(base[cam % C.CAM_IMAGES][None]).to(cuda)
    packed = torch.from_numpy(C.pack(draws)[cam % C.CAM_DRAWS][None]).to(cuda)
    with DeviceGuard(IA) as g:
        out, mat, status = IA.image_aug_batched(images, packed, (2, 2), MEAN, STD, (1, 1), return_status=True)
        g.check("65535 cameras")
    assert int(status) == 0
    want = np.empty((C.CAM_IMAGES, C.CAM_DRAWS, 3, 2, 2), np.float32)
    for i in range(C.CAM_IMAGES):
        for k, (_, dims, xy, flip, rot) in enumerate(draws):
            want[i, k] = O.augment(base[i], dims, xy, (2, 2), flip, rot, MEAN, STD)
    assert bits_equal(out[0].cpu().numpy(), want[cam % C.CAM_IMAGES, cam % C.CAM_DRAWS])
    mats = torch.stack([IA.img_aug_matrix(r, (xy[0], xy[1], xy[0] + 2, xy[1] + 2), f, a) for r, _, xy, f, a in draws])
    assert torch.equal(mat[0].cpu(), mats[torch.from_numpy(cam % C.CAM_DRAWS)])


def test_65536_cameras_are_refused_before_any_device_work(cuda):
    from bevfusion_b200 import _C
    from bevfusion_b200 import image_aug as IA
    N = C.MAX_GRID + 1
    L = _C.lib()
    assert L.bevb200_image_aug_workspace_bytes(N, 3, 3, 2, 2, 1, 1) == 0
    images = torch.zeros((1, N, 3, 3, 3), dtype=torch.uint8, device=cuda)
    draws = torch.from_numpy(C.pack(C.many_camera_draws())[np.arange(N) % C.CAM_DRAWS][None]).to(cuda)
    with DeviceGuard(IA) as g:
        with pytest.raises(ValueError, match="unsupported sizes"):
            IA.image_aug_batched(images, draws, (2, 2), MEAN, STD, (1, 1))
        assert g.check() == 0                         # refused before anything was allocated
    # the C entry itself: nothing it was handed changes
    g = DeviceGuard()
    out = g.carve(torch.empty((N * 12,), dtype=torch.float32, device=cuda), fill=False)
    mat = g.carve(torch.empty((N * 16,), dtype=torch.float32, device=cuda), fill=False)
    status = g.carve(torch.empty((1,), dtype=torch.int32, device=cuda), fill=False)
    ws = g.carve(torch.empty((1 << 20,), dtype=torch.uint8, device=cuda), fill=False)
    before = [t.clone() for t in (out, mat, status, ws)]
    rc = L.bevb200_image_aug(_C.ptr(images), N, 3, 3, _C.ptr(draws), 2, 2, 1, 1, *MEAN, *STD, _C.ptr(out),
                             _C.ptr(mat), _C.ptr(status), _C.ptr(ws), ws.numel(), _C.current_stream(cuda))
    assert rc == C.EINVAL and "cams" in L.bevb200_last_error().decode()
    g.check("refused call")
    assert all(torch.equal(a, b) for a, b in zip(before, (out, mat, status, ws)))
