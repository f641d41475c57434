"""GPU: the device camera augmentation (image_aug / image_aug_batched) bit-equal to the numpy restatement of Pillow +
torchvision and to the stored Pillow outputs, at B = 1 and 4 with six 1600x900 cameras in train and test mode; the
device img_aug_matrix against the reference's torch fp32 code; a CUDA-graph replay with new draws against eager
calls; BEVPoolPlan.rebuild_ fed from the device matrix against a plan built from the host matrices; and the status
word for draws the call refuses."""
import numpy as np
import pytest
import torch

import image_aug_oracle as O

pytestmark = pytest.mark.gpu

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
NUSC = dict(final_dim=(256, 704), resize_lim=(0.38, 0.55), bot_pct_lim=(0.0, 0.0), rot_lim=(-5.4, 5.4),
            rand_flip=True)


def camera_images(seed, B, N, H=900, W=1600):
    """Noise over smooth gradients, one image per camera: hits the clips to 0 / 255 as well as mid-range values."""
    rng = np.random.RandomState(seed)
    y, x = np.mgrid[0:H, 0:W]
    base = np.stack([x * 255 // W, y * 255 // H, (x + y) % 256], -1).astype(np.int16)
    out = np.empty((B, N, H, W, 3), np.uint8)
    for b in range(B):
        for n in range(N):
            out[b, n] = np.clip(base + rng.randint(-90, 91, (H, W, 3)).astype(np.int16), 0, 255)
    return out


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def draws_for(B, N, is_train, seed):
    from bevfusion_b200.image_aug import ImageAug3D
    aug = ImageAug3D(**NUSC, is_train=is_train, rng=np.random.RandomState(seed))
    return [aug.draws((1600, 900), N) for _ in range(B)]


def check_against_oracle(imgs, draws, out, mat):
    from bevfusion_b200.image_aug import img_aug_matrix
    out, mat = out.cpu().numpy(), mat.cpu()
    for b, sample in enumerate(draws):
        for n, (resize, dims, crop, flip, rotate) in enumerate(sample):
            want = O.augment(imgs[b, n], dims, crop[:2], (256, 704), flip, rotate, MEAN, STD)
            assert bits_equal(out[b, n], want), (b, n, sample[n])
            assert torch.equal(mat[b, n], img_aug_matrix(resize, crop, flip, rotate)), (b, n, sample[n])


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("is_train", [True, False])
def test_bit_equal_to_the_oracle(cuda, B, is_train):
    from bevfusion_b200.image_aug import image_aug
    imgs = camera_images(B * 10 + is_train, B, 6)
    draws = draws_for(B, 6, is_train, seed=B)
    out, mat = image_aug(torch.from_numpy(imgs).to(cuda), draws, MEAN, STD)
    assert out.shape == (B, 6, 3, 256, 704) and mat.shape == (B, 6, 4, 4)
    check_against_oracle(imgs, draws, out, mat)


def test_bit_equal_to_the_pillow_golden(cuda, golden_dir):
    import os
    from bevfusion_b200.image_aug import image_aug, image_aug_batched
    z = np.load(os.path.join(golden_dir, "image_aug_tiny.npz"))
    images = torch.from_numpy(z["images"]).to(cuda)
    fd = tuple(int(v) for v in z["final_dim"])
    out, _ = image_aug(images, z["draws"], z["mean"], z["std"], final_dim=fd)
    assert bits_equal(out.cpu().numpy(), z["out"])
    out2, _, status = image_aug_batched(images, torch.from_numpy(z["draws"]).to(cuda), fd, z["mean"], z["std"],
                                        (1, 1), return_status=True)
    assert int(status) == 0 and bits_equal(out2.cpu().numpy(), z["out"])


def test_cuda_graph_replays_new_draws(cuda):
    from bevfusion_b200.image_aug import image_aug_batched, pack_draw
    B, N = 2, 6
    images = torch.from_numpy(camera_images(3, B, N)).to(cuda)
    static_draws = torch.zeros((B, N, 7), dtype=torch.float64, device=cuda)

    def packed(seed):
        return torch.tensor([[pack_draw(*d) for d in s] for s in draws_for(B, N, True, seed)], dtype=torch.float64)

    static_draws.copy_(packed(100))
    min_resize = (int(1600 * 0.38), int(900 * 0.38))
    s = torch.cuda.Stream(cuda)
    s.wait_stream(torch.cuda.current_stream(cuda))
    with torch.cuda.stream(s):
        image_aug_batched(images, static_draws, (256, 704), MEAN, STD, min_resize)   # warm-up outside capture
    torch.cuda.current_stream(cuda).wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gout, gmat, gstatus = image_aug_batched(images, static_draws, (256, 704), MEAN, STD, min_resize,
                                                return_status=True)
    for seed in (101, 102, 103):
        d = packed(seed)
        static_draws.copy_(d)
        g.replay()
        eout, emat = image_aug_batched(images, d.to(cuda), (256, 704), MEAN, STD, min_resize)
        torch.cuda.synchronize()
        assert int(gstatus) == 0
        assert torch.equal(gout.view(torch.int32), eout.view(torch.int32)) and torch.equal(gmat, emat)


def test_rebuild_from_the_device_matrix(cuda):
    from bevfusion_b200 import synthetic as S
    from bevfusion_b200.bev_pool import BEVPoolPlan
    from bevfusion_b200.image_aug import image_aug, img_aug_matrix, post_transforms
    from bevfusion_b200.vtransform import create_frustum
    cfg = S.CONFIGS["C2"]
    B, N = 2, 6
    rig = {k: v.to(cuda) for k, v in S.camera_rig(N, cfg["image_size"], B).items()}
    fr = create_frustum(cfg["image_size"], cfg["feature_size"], cfg["dbound"]).to(cuda)
    bounds = (cfg["xbound"], cfg["ybound"], cfg["zbound"])
    base = [rig[k] for k in ("camera2lidar_rots", "camera2lidar_trans", "intrins", "post_rots", "post_trans")]
    plan = BEVPoolPlan.from_cameras(fr, *base, *bounds, sync=False)
    draws = draws_for(B, N, True, seed=9)
    _, mat = image_aug(torch.from_numpy(camera_images(4, B, N)).to(cuda), draws, MEAN, STD)
    post_rots, post_trans = post_transforms(mat)
    plan.rebuild_(*base[:3], post_rots, post_trans)
    host_mat = torch.stack([torch.stack([img_aug_matrix(d[0], d[2], d[3], d[4]) for d in s]) for s in draws])
    hr, ht = post_transforms(host_mat.to(cuda))
    host = BEVPoolPlan.from_cameras(fr, *base[:3], hr, ht, *bounds)
    h, d = host.tables, plan.tables
    n_kept, n_int = int(d.n_kept), int(d.n_intervals)
    assert (n_kept, n_int) == (h.n_kept, h.n_intervals)
    assert torch.equal(d.perm, h.perm) and torch.equal(d.ranks, h.ranks)
    assert torch.equal(d.geom[:n_kept], h.geom)
    assert torch.equal(d.starts[:n_int], h.starts) and torch.equal(d.lengths[:n_int], h.lengths)


def test_refused_draws_set_the_status_and_give_nan(cuda):
    from bevfusion_b200.image_aug import BAD_DRAW, OVER_CAPACITY, image_aug_batched, pack_draw
    images = torch.from_numpy(camera_images(5, 1, 4, 90, 160)).to(cuda)
    good = pack_draw(0.5, (80, 45), (10, 5, 74, 37), True, 2.0)
    rows = [good, pack_draw(0.2, (32, 18), (0, 0, 64, 32), False, 0.0),        # below min_resize: over capacity
            good[:5] + [0.5] + good[6:], good[:6] + [float("nan")]]           # flip 0.5, rotate NaN: bad draw
    draws = torch.tensor([rows], dtype=torch.float64, device=cuda)
    out, mat, status = image_aug_batched(images, draws, (32, 64), MEAN, STD, (64, 36), return_status=True)
    assert int(status) == BAD_DRAW | OVER_CAPACITY
    assert bool(torch.isfinite(out[0, 0]).all()) and bool(torch.isfinite(mat[0, 0]).all())
    for n in (1, 2, 3):
        assert bool(torch.isnan(out[0, n]).all()) and bool(torch.isnan(mat[0, n]).all())
    want = O.augment(images[0, 0].cpu().numpy(), (80, 45), (10, 5), (32, 64), True, 2.0, MEAN, STD)
    assert bits_equal(out[0, 0].cpu().numpy(), want)


def test_many_rotations_and_odd_shapes(cuda):
    """Every rotate path and crops past each side, on odd sizes, against the oracle."""
    from bevfusion_b200.image_aug import image_aug
    H, W, fH, fW = 61, 99, 37, 53
    rots = [0.0, -0.0, 360.0, 5.4, -5.4, 1e-9, -1e-20, 90.0, -90.0, 180.0, 180 + 1e-13, 33.3, 359.9, 270.0]
    rng = np.random.RandomState(12)
    draws = []
    for r in rots:
        w, h = int(rng.randint(20, 240)), int(rng.randint(15, 130))
        x0, y0 = int(rng.randint(-10, w)), int(rng.randint(-10, h))
        draws.append((w / W, (w, h), (x0, y0, x0 + fW, y0 + fH), bool(rng.randint(2)), r))
    imgs = camera_images(6, 1, len(draws), H, W)
    out, _ = image_aug(torch.from_numpy(imgs).to(cuda), [draws], MEAN, STD)
    out = out.cpu().numpy()
    for n, (_, dims, crop, flip, r) in enumerate(draws):
        assert bits_equal(out[0, n], O.augment(imgs[0, n], dims, crop[:2], (fH, fW), flip, r, MEAN, STD)), draws[n]
    # square crops take the 90 / 270 transposes
    sq = [(0.5, (50, 30), (3, 1, 32, 30), False, r) for r in (90.0, 270.0, -90.0, 180.0)]
    imgs = camera_images(7, 1, len(sq), H, W)
    out, _ = image_aug(torch.from_numpy(imgs).to(cuda), [sq], MEAN, STD)
    out = out.cpu().numpy()
    for n, (_, dims, crop, flip, r) in enumerate(sq):
        assert bits_equal(out[0, n], O.augment(imgs[0, n], dims, crop[:2], (29, 29), flip, r, MEAN, STD)), sq[n]
