"""image_aug -- ImageAug3D and ImageNormalize of the camera pipeline (transforms_3d.py:98-192, 992-1006) on the device
(csrc/image_aug.cu), bit-exact to Pillow + torchvision.

    ImageAug3D(final_dim, resize_lim, bot_pct_lim, rot_lim, rand_flip, is_train)
        the reference's constructor and sample_augmentation: the same numpy RNG calls in the same order, so with the
        same seed it draws what the reference draws, in train and test mode.  draws(ori_shape, n_cam) stacks one draw
        per camera as the reference's __call__ does (one sample_augmentation per image).
    image_aug(images_u8, draws, mean, std) -> (images [B, N, 3, fH, fW] fp32, img_aug_matrix [B, N, 4, 4] fp32)
        images_u8 [B, N, H, W, 3] uint8 on the device; draws a list over samples of per-camera draws (the tuples
        sample_augmentation returns) or an array [B, N, 7] of pack_draw rows.  The draws go over in one pinned,
        asynchronous copy.
    image_aug_batched(images_u8, draws, final_dim, mean, std, min_resize)
        the same with the draws already a float64 device tensor [B, N, 7]: no host work, CUDA-graph capturable.
    img_aug_matrix(resize, crop, flip, rotate)
        ImageAug3D's post-homography in the reference's fp32 arithmetic, on the host ([4, 4]).
    post_transforms(img_aug_matrix) -> (post_rots [.., 3, 3], post_trans [.., 3]) for BEVPoolPlan.rebuild_.

Each output value equals TF.normalize(TF.to_tensor(img.resize(dims).crop(box)[.transpose(FLIP_LEFT_RIGHT)]
.rotate(deg)), mean, std) bit for bit, and the matrix equals the reference's torch fp32 result.  GPU only: CPU
tensors raise ValueError, as do a dtype other than uint8, a channel count other than 3 and an empty resize."""

import numpy as np
import torch

from . import _C

__all__ = ["ImageAug3D", "image_aug", "image_aug_batched", "img_aug_matrix", "pack_draw", "post_transforms",
           "DRAW_FIELDS", "BAD_DRAW", "OVER_CAPACITY"]

DRAW_FIELDS = 7        # BEVB200_IMAGE_AUG_DRAW_FIELDS: resize, resize_w, resize_h, crop_x, crop_y, flip, rotate
BAD_DRAW = 1           # BEVB200_IMAGE_AUG_BAD_DRAW
OVER_CAPACITY = 2      # BEVB200_IMAGE_AUG_OVER_CAPACITY
MAX_FRAME = 16384      # output sides the kernel accepts


class ImageAug3D:
    """The reference's ImageAug3D draw.  Random numbers come from numpy's global RandomState, as in the reference,
    or from `rng` (a numpy RandomState) when one is given."""

    def __init__(self, final_dim, resize_lim, bot_pct_lim, rot_lim, rand_flip, is_train, rng=None):
        self.final_dim = final_dim
        self.resize_lim = resize_lim
        self.bot_pct_lim = bot_pct_lim
        self.rand_flip = rand_flip
        self.rot_lim = rot_lim
        self.is_train = is_train
        self.rng = rng

    def sample_augmentation(self, results):
        """(resize, resize_dims, crop, flip, rotate) for one image of results["ori_shape"] = (W, H)."""
        r = np.random if self.rng is None else self.rng
        W, H = results["ori_shape"]
        fH, fW = self.final_dim
        if self.is_train:
            resize = r.uniform(*self.resize_lim)
            newW, newH = int(W * resize), int(H * resize)
            crop_h = int((1 - r.uniform(*self.bot_pct_lim)) * newH) - fH
            crop_w = int(r.uniform(0, max(0, newW - fW)))
            flip = bool(self.rand_flip and r.choice([0, 1]))
            rotate = r.uniform(*self.rot_lim)
        else:
            resize = np.mean(self.resize_lim)
            newW, newH = int(W * resize), int(H * resize)
            crop_h = int((1 - np.mean(self.bot_pct_lim)) * newH) - fH
            crop_w = int(max(0, newW - fW) / 2)
            flip = False
            rotate = 0
        return resize, (newW, newH), (crop_w, crop_h, crop_w + fW, crop_h + fH), flip, rotate

    def draws(self, ori_shape, n_cam):
        """One draw per camera, in camera order: a list of sample_augmentation tuples."""
        return [self.sample_augmentation({"ori_shape": ori_shape}) for _ in range(n_cam)]

    def min_resize(self, ori_shape):
        """The smallest resized (w, h) this augmentation draws for ori_shape = (W, H): the capacity image_aug_batched
        needs for every draw of this pipeline."""
        W, H = ori_shape
        s = min(self.resize_lim) if self.is_train else np.mean(self.resize_lim)
        return max(int(W * s), 1), max(int(H * s), 1)


def pack_draw(resize, resize_dims, crop, flip, rotate):
    """One draw as the kernel reads it: float64 [7] = resize, resize_w, resize_h, crop_x, crop_y, flip, rotate."""
    return [float(resize), float(resize_dims[0]), float(resize_dims[1]), float(crop[0]), float(crop[1]),
            1.0 if flip else 0.0, float(rotate)]


def img_aug_matrix(resize, crop, flip, rotate):
    """ImageAug3D's img_aug_matrix of one draw ([4, 4] fp32 on the host): scale by resize, shift by -crop, the
    optional left-right flip about the crop width, then the rotation about the crop centre, composed in torch fp32
    with each 2-term product summed as two rounded products and one rounded add, as the reference's matmuls are."""
    f = torch.float32
    fw, fh = float(crop[2] - crop[0]), float(crop[3] - crop[1])
    rot = torch.eye(2, dtype=f) * torch.tensor(float(resize), dtype=f)
    tran = torch.zeros(2, dtype=f) - torch.tensor([float(crop[0]), float(crop[1])], dtype=f)
    if flip:
        A = torch.tensor([[-1.0, 0.0], [0.0, 1.0]], dtype=f)
        rot = A[:, :1] * rot[:1, :] + A[:, 1:] * rot[1:, :]
        tran = A[:, 0] * tran[0] + A[:, 1] * tran[1] + torch.tensor([fw, 0.0], dtype=f)
    theta = rotate / 180 * np.pi
    A = torch.tensor([[np.cos(theta), np.sin(theta)], [-np.sin(theta), np.cos(theta)]], dtype=f)
    half = torch.tensor([fw, fh], dtype=f) / 2
    b = A[:, 0] * -half[0] + A[:, 1] * -half[1] + half
    out = torch.eye(4, dtype=f)
    out[:2, :2] = A[:, :1] * rot[:1, :] + A[:, 1:] * rot[1:, :]
    out[:2, 3] = A[:, 0] * tran[0] + A[:, 1] * tran[1] + b
    return out


def post_transforms(matrix):
    """(post_rots [..., 3, 3], post_trans [..., 3]) of img_aug_matrix [..., 4, 4], contiguous, for
    BEVPoolPlan.rebuild_ and the view transforms."""
    return matrix[..., :3, :3].contiguous(), matrix[..., :3, 3].contiguous()


def _check_images(images, device=True):
    if not isinstance(images, torch.Tensor):
        raise ValueError("images must be a torch.Tensor")
    if images.dtype != torch.uint8:
        raise ValueError("images must be uint8, got %s" % images.dtype)
    if images.dim() != 5 or images.shape[-1] != 3:
        raise ValueError("images must be [B, N, H, W, 3] (RGB), got %s" % (tuple(images.shape),))
    if images.shape[2] < 1 or images.shape[3] < 1:
        raise ValueError("empty images %s" % (tuple(images.shape),))
    if device and not images.is_cuda:
        raise ValueError("images must be a CUDA tensor: bevfusion_b200 has no CPU implementation")


def _norm(v, name):
    v = [float(x) for x in v]
    if len(v) != 3:
        raise ValueError("%s needs three values (RGB)" % name)
    return [float(np.float32(x)) for x in v]


def image_aug_batched(images, draws, final_dim, mean, std, min_resize, return_status=False):
    """images [B, N, H, W, 3] uint8 and draws [B, N, 7] float64 (pack_draw rows), both on one CUDA device ->
    (images [B, N, 3, fH, fW] fp32, img_aug_matrix [B, N, 4, 4] fp32) for final_dim = (fH, fW).  min_resize (w, h)
    sizes the filter tables: a draw that resizes below it (or is malformed) sets the status word and gives NaN for
    its camera; with return_status the int32 [1] status word is returned as a third value.  No host
    synchronisation: capturable in a CUDA graph with the draws as a static input."""
    _check_images(images)
    if not isinstance(draws, torch.Tensor) or not draws.is_cuda:
        raise ValueError("draws must be a CUDA tensor")
    B, N, H, W, _ = images.shape
    if draws.dtype != torch.float64 or tuple(draws.shape) != (B, N, DRAW_FIELDS):
        raise ValueError("draws must be float64 [%d, %d, %d], got %s %s" % (B, N, DRAW_FIELDS, draws.dtype,
                                                                            tuple(draws.shape)))
    if draws.device != images.device:
        raise ValueError("draws and images must be on one device")
    fH, fW = (int(v) for v in final_dim)
    if not (1 <= fH <= MAX_FRAME and 1 <= fW <= MAX_FRAME):
        raise ValueError("final_dim sides must be in 1..%d, got %s" % (MAX_FRAME, (fH, fW)))
    mw, mh = (int(v) for v in min_resize)
    if mw < 1 or mh < 1:
        raise ValueError("min_resize must be positive, got %s" % ((mw, mh),))
    m, s = _norm(mean, "mean"), _norm(std, "std")
    images = images.contiguous()
    draws = draws.contiguous()
    dev = images.device
    cams = B * N
    L = _C.lib()
    ws_bytes = L.bevb200_image_aug_workspace_bytes(cams, H, W, fH, fW, mw, mh)
    if ws_bytes == 0 and cams > 0:
        raise ValueError("unsupported sizes: images %s, final_dim %s, min_resize %s"
                         % (tuple(images.shape), (fH, fW), (mw, mh)))
    out = torch.empty((B, N, 3, fH, fW), dtype=torch.float32, device=dev)
    mat = torch.empty((B, N, 4, 4), dtype=torch.float32, device=dev)
    status = torch.empty((1,), dtype=torch.int32, device=dev)
    ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _C.check(L.bevb200_image_aug(_C.ptr(images), cams, H, W, _C.ptr(draws), fH, fW, mw, mh, *m, *s, _C.ptr(out),
                                     _C.ptr(mat), _C.ptr(status), _C.ptr(ws), ws_bytes, _C.current_stream(dev)),
                 "image_aug")
    return (out, mat, status) if return_status else (out, mat)


def _pack_host(draws, B, N):
    if isinstance(draws, np.ndarray):
        rows = np.asarray(draws, np.float64)
        if rows.shape != (B, N, DRAW_FIELDS):
            raise ValueError("draws must be [%d, %d, %d], got %s" % (B, N, DRAW_FIELDS, rows.shape))
        return rows
    if len(draws) != B or any(len(d) != N for d in draws):
        raise ValueError("draws must hold %d samples of %d camera draws" % (B, N))
    return np.array([[pack_draw(*d) for d in sample] for sample in draws], np.float64).reshape(B, N, DRAW_FIELDS)


def image_aug(images, draws, mean, std, final_dim=None):
    """images [B, N, H, W, 3] uint8 on the device and host draws (a list over samples of lists of
    sample_augmentation tuples, or a float64 array [B, N, 7] of pack_draw rows) -> (images [B, N, 3, fH, fW] fp32,
    img_aug_matrix [B, N, 4, 4] fp32) on the device.  final_dim defaults to the crop boxes' size.  The draws are
    staged in one pinned buffer and copied asynchronously; the resize capacity is the smallest drawn size."""
    _check_images(images, device=False)
    B, N = images.shape[0], images.shape[1]
    if final_dim is None:
        if isinstance(draws, np.ndarray) or B * N == 0:
            raise ValueError("final_dim is needed with packed or empty draws")
        boxes = {(c[3] - c[1], c[2] - c[0]) for sample in draws for (_, _, c, _, _) in sample}
        if len(boxes) != 1:
            raise ValueError("every crop box must have one size, got %s" % sorted(boxes))
        final_dim = boxes.pop()
    rows = _pack_host(draws, B, N)
    if B * N and (not np.isfinite(rows).all() or rows[..., 1:3].min() < 1):
        raise ValueError("every draw needs finite fields and a non-empty resize_dims")
    min_resize = (int(rows[..., 1].min()), int(rows[..., 2].min())) if B * N else (1, 1)
    _check_images(images)
    staged = torch.from_numpy(rows).pin_memory()
    dev_draws = staged.to(images.device, non_blocking=True)
    return image_aug_batched(images, dev_draws, final_dim, mean, std, min_resize)
