"""CPU: the numpy restatement of the camera augmentation (tests/image_aug_oracle.py) against the installed Pillow +
torchvision, bit for bit: seeded train-mode draws and the test-mode draw at 1600x900, odd sizes, crops past the
resized image and the rotation cases Image.rotate treats apart.  Also ImageAug3D's RNG sequence, img_aug_matrix
against the reference's torch fp32 matmuls, the C declarations and the workspace query."""
import math
import re

import numpy as np
import pytest
import torch

import image_aug_oracle as O

PIL = pytest.importorskip("PIL.Image")
TF = pytest.importorskip("torchvision.transforms.functional")

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
NUSC_TRAIN = dict(final_dim=(256, 704), resize_lim=(0.38, 0.55), bot_pct_lim=(0.0, 0.0), rot_lim=(-5.4, 5.4),
                  rand_flip=True, is_train=True)
NUSC_TEST = dict(NUSC_TRAIN, is_train=False)


def pillow(img, dims, crop, flip, rotate):
    """The reference's ImageAug3D.img_transform pixel steps followed by ImageNormalize's ToTensor + Normalize."""
    im = PIL.fromarray(img).resize(dims).crop(crop)
    if flip:
        im = im.transpose(PIL.FLIP_LEFT_RIGHT)
    return TF.normalize(TF.to_tensor(im.rotate(rotate)), MEAN, STD).numpy()


def bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.int32),
                                                 np.ascontiguousarray(b).view(np.int32))


def camera_image(seed, H=900, W=1600):
    """Noise over smooth gradients: hits the clip to 0 / 255 after each pass as well as mid-range values."""
    rng = np.random.RandomState(seed)
    y, x = np.mgrid[0:H, 0:W]
    base = np.stack([x * 255.0 / W, y * 255.0 / H, (x + y) % 256], -1)
    return np.clip(base + rng.randint(-90, 91, (H, W, 3)), 0, 255).astype(np.uint8)


def oracle(img, draw, final_dim):
    resize, dims, crop, flip, rotate = draw
    return O.augment(img, dims, crop[:2], final_dim, flip, rotate, MEAN, STD)


def test_oracle_equals_pillow_on_200_train_draws():
    from bevfusion_b200.image_aug import ImageAug3D
    aug = ImageAug3D(**NUSC_TRAIN, rng=np.random.RandomState(2024))
    imgs = [camera_image(s) for s in range(3)]
    for i in range(200):
        d = aug.sample_augmentation({"ori_shape": (1600, 900)})
        img = imgs[i % 3]
        assert bits_equal(oracle(img, d, (256, 704)), pillow(img, d[1], d[2], d[3], d[4])), d


def test_oracle_equals_pillow_on_the_test_draw():
    from bevfusion_b200.image_aug import ImageAug3D
    d = ImageAug3D(**NUSC_TEST).sample_augmentation({"ori_shape": (1600, 900)})
    assert d[3] is False and d[4] == 0
    img = camera_image(7)
    assert bits_equal(oracle(img, d, (256, 704)), pillow(img, d[1], d[2], d[3], d[4]))


@pytest.mark.parametrize("H,W,dims,crop,flip,rotate", [
    (37, 53, (131, 97), (5, 9, 105, 60), False, 3.0),            # upscale
    (37, 53, (131, 97), (40, -7, 140, 90), True, -2.5),           # crop past right and top
    (900, 1600, (123, 77), (-20, -11, 101, 70), False, 5.4),      # strong downscale, crop past every side
    (61, 99, (99, 61), (0, 0, 99, 61), False, 0.0),              # no resize: a copy
    (61, 99, (98, 61), (1, 2, 60, 41), True, 1.0),                # horizontal only, odd crop
    (61, 99, (99, 60), (3, 0, 48, 59), False, -1.0),              # vertical only
    (47, 83, (1, 1), (0, 0, 17, 13), False, 4.0),                  # one-pixel resize
    (47, 83, (200, 3), (150, 1, 211, 9), True, 0.5),               # extreme aspect
    (900, 1600, (608, 342), (0, 86, 704, 342), True, -5.4),       # resize narrower than the crop: right part is 0
])
def test_oracle_equals_pillow_on_odd_sizes(H, W, dims, crop, flip, rotate):
    img = camera_image(H * W, H, W)
    got = O.augment(img, dims, crop[:2], (crop[3] - crop[1], crop[2] - crop[0]), flip, rotate, MEAN, STD)
    assert bits_equal(got, pillow(img, dims, crop, flip, rotate))


@pytest.mark.parametrize("rotate", [0, 0.0, -0.0, 360.0, -360.0, 5.4, -5.4, 1e-9, -1e-9, 3e-14, -1e-20, 1e-300,
                                    90, -90, 180, -180, 270, 180 + 1e-13, 179.99999999, 45.0, 33.3, 359.9])
@pytest.mark.parametrize("shape", [(40, 64), (41, 41), (40, 40)])
def test_rotate_rule_equals_pillow(rotate, shape):
    h, w = shape
    img = camera_image(h + w, h, w)
    got = O.rotate(img, rotate)
    assert np.array_equal(got, np.asarray(PIL.fromarray(img).rotate(rotate)))


def test_rotate_rule_takes_every_path():
    assert O.rotate_rule(0, 5, 7)[0] == "copy" and O.rotate_rule(-360.0, 5, 7)[0] == "copy"
    assert O.rotate_rule(180, 5, 7)[0] == "rot180" and O.rotate_rule(-180, 5, 7)[0] == "rot180"
    assert O.rotate_rule(90, 6, 6)[0] == "rot90" and O.rotate_rule(270, 6, 6)[0] == "rot270"
    assert O.rotate_rule(90, 6, 7)[0] == "affine"
    assert O.rotate_rule(-1e-20, 6, 7)[0] == "scale"        # -1e-20 % 360 == 360.0: sin rounds to 0
    assert O.rotate_rule(1e-9, 6, 7)[0] == "affine"


def test_normalize_equals_torchvision():
    img = camera_image(3, 33, 71)
    want = TF.normalize(TF.to_tensor(PIL.fromarray(img)), MEAN, STD).numpy()
    assert bits_equal(O.normalize(img, MEAN, STD), want)


@pytest.mark.parametrize("cfg", [NUSC_TRAIN, dict(NUSC_TRAIN, bot_pct_lim=(0.0, 0.22), rand_flip=False), NUSC_TEST])
def test_draw_follows_the_reference_rng_sequence(cfg):
    """sample_augmentation draws, per image: resize ~ U(resize_lim), bottom share ~ U(bot_pct_lim), horizontal crop
    ~ U(0, max(0, newW - fW)), flip = choice([0, 1]) only when rand_flip, rotation ~ U(rot_lim); test mode draws
    nothing and takes the means, a centred crop, no flip and no rotation."""
    from bevfusion_b200.image_aug import ImageAug3D
    np.random.seed(11)
    got = ImageAug3D(**cfg).draws((1600, 900), 6)
    after = np.random.uniform()
    r = np.random.RandomState(11)
    fH, fW = cfg["final_dim"]
    for d in got:
        if cfg["is_train"]:
            s = r.uniform(*cfg["resize_lim"])
            nw, nh = int(1600 * s), int(900 * s)
            ch = int((1 - r.uniform(*cfg["bot_pct_lim"])) * nh) - fH
            cw = int(r.uniform(0, max(0, nw - fW)))
            fl = bool(cfg["rand_flip"] and r.choice([0, 1]))
            rot = r.uniform(*cfg["rot_lim"])
        else:
            s = np.mean(cfg["resize_lim"])
            nw, nh = int(1600 * s), int(900 * s)
            ch = int((1 - np.mean(cfg["bot_pct_lim"])) * nh) - fH
            cw = int(max(0, nw - fW) / 2)
            fl, rot = False, 0
        assert d == (s, (nw, nh), (cw, ch, cw + fW, ch + fH), fl, rot)
    assert after == r.uniform()      # the same number of RNG calls


def reference_matrix(resize, crop, flip, rotate):
    """ImageAug3D.img_transform's post-homography as the reference composes it: torch fp32 2x2 matmuls."""
    rotation, translation = torch.eye(2) * resize, torch.zeros(2) - torch.Tensor(crop[:2])
    if flip:
        A = torch.Tensor([[-1, 0], [0, 1]])
        rotation, translation = A.matmul(rotation), A.matmul(translation) + torch.Tensor([crop[2] - crop[0], 0])
    theta = rotate / 180 * np.pi
    A = torch.Tensor([[np.cos(theta), np.sin(theta)], [-np.sin(theta), np.cos(theta)]])
    half = torch.Tensor([crop[2] - crop[0], crop[3] - crop[1]]) / 2
    out = torch.eye(4)
    out[:2, :2] = A.matmul(rotation)
    b = A.matmul(-half) + half
    out[:2, 3] = A.matmul(translation) + b
    return out


def test_img_aug_matrix_equals_the_reference_torch_code():
    from bevfusion_b200.image_aug import ImageAug3D, img_aug_matrix
    aug = ImageAug3D(**NUSC_TRAIN, rng=np.random.RandomState(5))
    draws = [aug.sample_augmentation({"ori_shape": (1600, 900)}) for _ in range(300)]
    draws.append(ImageAug3D(**NUSC_TEST).sample_augmentation({"ori_shape": (1600, 900)}))
    for resize, _, crop, flip, rotate in draws:
        assert torch.equal(img_aug_matrix(resize, crop, flip, rotate), reference_matrix(resize, crop, flip, rotate))


def test_post_transforms_split_the_matrix():
    from bevfusion_b200.image_aug import img_aug_matrix, post_transforms
    M = torch.stack([img_aug_matrix(0.48, (40, 176, 744, 432), True, 2.0)] * 2)
    rots, trans = post_transforms(M)
    assert rots.shape == (2, 3, 3) and trans.shape == (2, 3) and rots.is_contiguous() and trans.is_contiguous()
    assert torch.equal(rots[0], M[0, :3, :3]) and torch.equal(trans[1], M[1, :3, 3])


def test_c_symbols_are_declared_and_bound():
    from bevfusion_b200 import _C
    declared = _C.declared_symbols()
    with open(_C.HEADER_PATH) as f:
        header = f.read()
    for name in ("bevb200_image_aug_workspace_bytes", "bevb200_image_aug"):
        assert name in declared and name in _C._SIGNATURES
        assert hasattr(_C.lib(), name)
        params = re.search(r"\b%s\(([^)]*)\)" % name, header).group(1).split(",")
        assert len(params) == len(_C._SIGNATURES[name][1]), name


def test_workspace_query():
    from bevfusion_b200 import _C
    L = _C.lib()
    q = L.bevb200_image_aug_workspace_bytes
    one = q(1, 900, 1600, 256, 704, 608, 342)
    # staging rows (in_h x out_w RGBx) and the coefficient tables dominate, one set per camera
    assert one >= 900 * 704 * 4 + 704 * 4 * (2 * math.ceil(2 * 1600 / 608) + 1)
    assert q(6, 900, 1600, 256, 704, 608, 342) >= 6 * 900 * 704 * 4
    assert q(6, 900, 1600, 256, 704, 300, 342) > q(6, 900, 1600, 256, 704, 608, 342)    # wider filter, more taps
    assert q(0, 900, 1600, 256, 704, 608, 342) >= 0
    for bad in [(1, 900, 1600, 0, 704, 608, 342), (1, 900, 1600, 256, 16385, 608, 342), (1, 0, 1600, 256, 704, 1, 1),
                (1, 900, 1600, 256, 704, 0, 342), (-1, 900, 1600, 256, 704, 608, 342), (1, 1 << 19, 16, 8, 8, 1, 1)]:
        assert q(*bad) == 0, bad


def test_refusals_before_any_device_work():
    from bevfusion_b200.image_aug import image_aug, image_aug_batched
    draw = [[(0.48, (768, 432), (32, 176, 736, 432), False, 0.0)]]
    with pytest.raises(ValueError, match="uint8"):
        image_aug(torch.zeros(1, 1, 900, 1600, 3, dtype=torch.float32), draw, MEAN, STD)
    with pytest.raises(ValueError, match="RGB"):
        image_aug(torch.zeros(1, 1, 900, 1600, 4, dtype=torch.uint8), draw, MEAN, STD)
    with pytest.raises(ValueError, match="resize_dims"):
        image_aug(torch.zeros(1, 1, 900, 1600, 3, dtype=torch.uint8),
                  [[(0.0, (0, 0), (32, 176, 736, 432), False, 0.0)]], MEAN, STD)
    with pytest.raises(ValueError, match="CUDA"):
        image_aug(torch.zeros(1, 1, 900, 1600, 3, dtype=torch.uint8), draw, MEAN, STD)
    with pytest.raises(ValueError, match="CUDA"):
        image_aug_batched(torch.zeros(1, 1, 900, 1600, 3, dtype=torch.uint8), torch.zeros(1, 1, 7, dtype=torch.float64),
                          (256, 704), MEAN, STD, (608, 342))
