"""lidar_aug -- GlobalRotScaleTrans + RandomFlip3D on the LiDAR and radar clouds and the GT boxes, with
ObjectRangeFilter and ObjectNameFilter (transforms_3d.py:195-232, 323-353, 534-636) on the device, bit-exact to the
reference's torch CPU lines.

    GlobalRotScaleTrans(resize_lim, rot_lim, trans_lim, is_train, rng=None).draw()  -> (scale, theta, translation)
    RandomFlip3D(rng=None).draw()                                                    -> (horizontal, vertical)
        the reference's draws: uniform, uniform, three normal(0, trans_lim), then choice([0, 1]) twice, on numpy's
        global RNG or on `rng`.  With is_train=False GlobalRotScaleTrans draws nothing (scale, theta, translation
        are None).  Reproducing a reference sample means calling every draw of its pipeline in pipeline order: the
        sweep choice of LoadPointsFromMultiSweeps, ImageAug3D per camera, these two, and even GridMask at prob 0.0,
        which still consumes one np.random.rand().
    draw_sample(global_rot_scale_trans, random_flip) -> LidarAugDraw   both draws of one sample, in pipeline order
    lidar_aug_matrix(draw) -> the reference's lidar_aug_matrix [4, 4] float32 (host)
    LidarAug(max_batch, device)
        one device block: the per-sample records the kernels read (bevb200_lidar_aug_t), matrix [B, 4, 4],
        extra_rots [B, 3, 3] and extra_trans [B, 3] (for BEVPoolPlan.rebuild_ and the depth images) and the flip
        flags.  write(draws) refreshes all of it with one pinned asynchronous copy, so a CUDA graph that reads the
        block replays with new draws.  Passed as aug= to SweepStore / RadarSweepStore .assemble / .launch, where the
        sweep kernels augment each row before their range test.
        boxes(boxes, labels, counts, point_cloud_range, classes) -> the padded boxes after the transforms,
        ObjectRangeFilter (with limit_yaw) and ObjectNameFilter, on the device (csrc/box_aug.cu)
        flip_masks(masks) -> gt_masks_bev [B, C, H, W] flipped as RandomFlip3D flips it, from the device flags

The device evaluates no sine or cosine: they are computed here with torch on the CPU, as the reference computes
them (CUDA's and glibc's differ in the last ulp).  GPU only: a CPU device raises."""
import collections

import numpy as np
import torch

from . import _C

__all__ = ["GlobalRotScaleTrans", "RandomFlip3D", "LidarAugDraw", "draw_sample", "lidar_aug_matrix", "LidarAug",
           "AUG_DTYPE", "BAD_COUNT"]

BAD_COUNT = 1                                     # BEVB200_BOX_AUG_BAD_COUNT
MAX_BOXES = 4096                                  # BEVB200_HEAD_TARGETS_MAX_BOXES

# bevb200_lidar_aug_t, C layout
AUG_DTYPE = np.dtype([("enabled", "<i4"), ("rot_scale_trans", "<i4"), ("flip_horizontal", "<i4"),
                      ("flip_vertical", "<i4"), ("translation", "<f4", (3,)), ("scale", "<f4"), ("yaw_inc", "<f4"),
                      ("point_rot", "<f4", (9,)), ("box_rot", "<f4", (9,))], align=True)

LidarAugDraw = collections.namedtuple("LidarAugDraw", "scale theta translation flip_horizontal flip_vertical")
LidarAugDraw.__doc__ = """One sample's draws: GlobalRotScaleTrans' (scale, theta, translation [3]), all None when it
does not train, and RandomFlip3D's two flags."""


class GlobalRotScaleTrans:
    """The reference's GlobalRotScaleTrans draw (transforms_3d.py:196-232)."""

    def __init__(self, resize_lim, rot_lim, trans_lim, is_train, rng=None):
        self.resize_lim = resize_lim
        self.rot_lim = rot_lim
        self.trans_lim = trans_lim
        self.is_train = is_train
        self.rng = rng

    def draw(self):
        """(scale, theta, translation float64 [3]), or (None, None, None) when not training"""
        if not self.is_train:
            return None, None, None
        r = np.random if self.rng is None else self.rng
        scale = r.uniform(*self.resize_lim)
        theta = r.uniform(*self.rot_lim)
        translation = np.array([r.normal(0, self.trans_lim) for i in range(3)])
        return scale, theta, translation


class RandomFlip3D:
    """The reference's RandomFlip3D draw (transforms_3d.py:323-353)."""

    def __init__(self, rng=None):
        self.rng = rng

    def draw(self):
        r = np.random if self.rng is None else self.rng
        flip_horizontal = r.choice([0, 1])
        flip_vertical = r.choice([0, 1])
        return bool(flip_horizontal), bool(flip_vertical)


def draw_sample(global_rot_scale_trans, random_flip=None):
    """One sample's LidarAugDraw: GlobalRotScaleTrans' draw, then RandomFlip3D's (no flips without one)."""
    scale, theta, translation = global_rot_scale_trans.draw()
    fh, fv = random_flip.draw() if random_flip is not None else (False, False)
    return LidarAugDraw(scale, theta, translation, fh, fv)


def cuda_device(device):
    """torch.device("cuda") as the indexed device it names (the current one), so it compares equal to tensors'"""
    device = torch.device(device)
    return torch.device("cuda", torch.cuda.current_device()) if device.index is None else device


def _rot_mats(theta):
    """(rot_mat_T of BasePoints.rotate(-theta), rot_mat_T of LiDARInstance3DBoxes.rotate(theta), fl32(theta)) with
    the reference's own torch CPU calls (base_points.py:145-171, lidar_box3d.py:157-167)"""
    a = torch.tensor(-theta, dtype=torch.float32)
    s, c = torch.sin(a), torch.cos(a)
    point_rot = a.new_tensor([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T
    b = torch.tensor(theta, dtype=torch.float32)
    s, c = torch.sin(b), torch.cos(b)
    box_rot = b.new_tensor([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    return point_rot.numpy(), box_rot.numpy(), b.numpy()


def lidar_aug_matrix(draw):
    """The reference's data["lidar_aug_matrix"] ([4, 4] float32): GlobalRotScaleTrans' rotation.T * scale and
    translation * scale in float64 stored to fp32 (rotation = eye(3) @ the boxes' fp32 rot_mat_T), then RandomFlip3D's
    rotation @ m[:3, :] in float64 stored to fp32."""
    transform = np.eye(4).astype(np.float32)
    if draw.scale is not None:
        rotation = np.eye(3) @ _rot_mats(draw.theta)[1]
        transform[:3, :3] = rotation.T * draw.scale
        transform[:3, 3] = np.asarray(draw.translation) * draw.scale
    rotation = np.eye(3)
    if draw.flip_horizontal:
        rotation = np.array([[1, 0, 0], [0, -1, 0], [0, 0, 1]]) @ rotation
    if draw.flip_vertical:
        rotation = np.array([[-1, 0, 0], [0, 1, 0], [0, 0, 1]]) @ rotation
    transform[:3, :] = rotation @ transform[:3, :]
    return transform


def pack_record(draw):
    """bevb200_lidar_aug_t of one draw (a numpy record)"""
    rec = np.zeros((), AUG_DTYPE)
    rec["enabled"] = 1
    rec["flip_horizontal"], rec["flip_vertical"] = int(bool(draw.flip_horizontal)), int(bool(draw.flip_vertical))
    if draw.scale is not None:
        translation = np.asarray(draw.translation, np.float64)
        if translation.shape != (3,):
            raise ValueError("translation needs 3 values")
        point_rot, box_rot, yaw = _rot_mats(draw.theta)
        rec["rot_scale_trans"] = 1
        rec["translation"] = torch.tensor(translation, dtype=torch.float32).numpy()   # new_tensor(translation)
        rec["scale"] = np.float32(draw.scale)                                          # t *= scale in fp32
        rec["yaw_inc"] = yaw
        rec["point_rot"], rec["box_rot"] = point_rot.reshape(9), box_rot.reshape(9)
    return rec


class LidarAug:
    """The per-sample augmentation block on the device (see the module docstring).  Views into the block:
    records (for the kernels), matrix [max_batch, 4, 4], extra_rots [max_batch, 3, 3], extra_trans [max_batch, 3],
    flip_horizontal / flip_vertical [max_batch] bool.  `batch` is the number of samples the last write() was given:
    launches and boxes() over more samples than that raise, so a sample cannot go unaugmented by accident (a sample
    that should stay untouched is written as None)."""

    def __init__(self, max_batch, device="cuda"):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError("LidarAug lives on a CUDA device: bevfusion_b200 has no CPU implementation")
        self.device = cuda_device(self.device)
        if max_batch < 1:
            raise ValueError("max_batch must be positive")
        B = self.max_batch = int(max_batch)
        sizes = [("records", B * AUG_DTYPE.itemsize), ("matrix", B * 64), ("extra_rots", B * 36),
                 ("extra_trans", B * 12), ("flips", B * 2)]
        self._at, off = {}, 0
        for name, n in sizes:
            self._at[name] = (off, n)
            off += (n + 15) // 16 * 16
        self.block = torch.zeros((off,), dtype=torch.uint8, device=self.device)
        view = lambda name, dtype: self.block[slice(self._at[name][0], sum(self._at[name]))].view(dtype)
        self.records = view("records", torch.uint8)
        self.matrix = view("matrix", torch.float32).view(B, 4, 4)
        self.extra_rots = view("extra_rots", torch.float32).view(B, 3, 3)
        self.extra_trans = view("extra_trans", torch.float32).view(B, 3)
        flips = view("flips", torch.bool).view(2, B)
        self.flip_horizontal, self.flip_vertical = flips[0], flips[1]
        self.batch = 0
        self.write([])

    def ptr(self):
        return self.records.data_ptr()

    def write(self, draws):
        """Refresh the whole block from one LidarAugDraw per sample (at most max_batch), in one pinned asynchronous
        copy on the current stream.  A None entry writes a disabled record: that sample is left exactly as it is
        (identity matrix, no flips)."""
        draws = list(draws)
        B = len(draws)
        if B > self.max_batch:
            raise ValueError("%d draws, the block was made for %d" % (B, self.max_batch))
        host = np.zeros(self.block.numel(), np.uint8)
        rec = np.zeros(self.max_batch, AUG_DTYPE)
        mat = np.tile(np.eye(4, dtype=np.float32), (self.max_batch, 1, 1))
        flips = np.zeros((2, self.max_batch), np.bool_)
        for b, d in enumerate(draws):
            if d is None:
                continue
            d = LidarAugDraw(*d)
            rec[b] = pack_record(d)
            mat[b] = lidar_aug_matrix(d)
            flips[:, b] = bool(d.flip_horizontal), bool(d.flip_vertical)
        for name, arr in (("records", rec), ("matrix", mat), ("extra_rots", np.ascontiguousarray(mat[:, :3, :3])),
                          ("extra_trans", np.ascontiguousarray(mat[:, :3, 3])), ("flips", flips)):
            off, n = self._at[name]
            host[off:off + n] = np.frombuffer(arr.tobytes(), np.uint8)
        with torch.cuda.device(self.device):
            self.block.copy_(torch.from_numpy(host).pin_memory(), non_blocking=True)
        self.batch = B

    def check_batch(self, batch):
        """Raise unless the last write() covered `batch` samples."""
        if batch > self.batch:
            raise ValueError("%d samples, but the last LidarAug.write() had %d draws" % (batch, self.batch))

    def boxes(self, boxes, labels, counts, point_cloud_range, classes, augment=True):
        """GlobalRotScaleTrans + RandomFlip3D on padded GT boxes, then ObjectRangeFilter (in_range_bev on
        point_cloud_range[[0, 1, 3, 4]] as fp32, then limit_yaw(0.5, 2 pi)) and ObjectNameFilter (labels in
        [0, len(classes)), or [0, classes) for an int).

        boxes [B, Nmax, 7 | 9] fp32, labels [B, Nmax] int32, counts [B] int32 on this device (head_targets.pad_gt's
        layout), B <= the last write()'s batch -> (boxes, labels, counts, status [1] int32) in the same layout, survivors in input
        order, the rest zeroed; no host synchronisation, CUDA-graph capturable.  augment=False applies only the
        filters."""
        for t, name, dt in ((boxes, "boxes", torch.float32), (labels, "labels", torch.int32),
                            (counts, "counts", torch.int32)):
            _C.require_cuda(t, name, dt)
            if t.device != self.device:
                raise ValueError("%s is on %s, the block on %s" % (name, t.device, self.device))
        if boxes.dim() != 3 or boxes.shape[2] not in (7, 9):
            raise ValueError("boxes must be [B, Nmax, 7 | 9], got %s" % (tuple(boxes.shape),))
        B, nmax, D = boxes.shape
        if labels.shape != (B, nmax) or counts.shape != (B,):
            raise ValueError("labels must be [B, Nmax] and counts [B]")
        if augment:
            self.check_batch(B)
        if nmax > MAX_BOXES:
            raise ValueError("at most %d boxes per sample (got %d)" % (MAX_BOXES, nmax))
        rng = np.asarray(point_cloud_range, np.float32)
        if rng.shape != (6,):
            raise ValueError("point_cloud_range needs 6 values")
        num_classes = classes if isinstance(classes, int) else len(classes)
        out_boxes = torch.empty_like(boxes)
        out_labels = torch.empty_like(labels)
        out_counts = torch.empty_like(counts)
        status = torch.empty((1,), dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _C.check(_C.lib().bevb200_box_aug(
                _C.ptr(boxes), _C.ptr(labels), _C.ptr(counts), B, nmax, D, self.ptr() if augment else 0,
                float(rng[0]), float(rng[1]), float(rng[3]), float(rng[4]), num_classes, _C.ptr(out_boxes),
                _C.ptr(out_labels), _C.ptr(out_counts), _C.ptr(status), _C.current_stream(self.device)), "box_aug")
        return out_boxes, out_labels, out_counts, status

    def flip_masks(self, masks):
        """gt_masks_bev [B, C, H, W] as RandomFlip3D leaves it: [:, :, ::-1] with the horizontal flag, then
        [:, ::-1, :] with the vertical one, per sample, selected on the device."""
        B = masks.shape[0]
        if masks.dim() != 4 or B > self.max_batch:
            raise ValueError("masks must be [B, C, H, W] with B <= %d" % self.max_batch)
        self.check_batch(B)
        fh = self.flip_horizontal[:B].view(B, 1, 1, 1)
        fv = self.flip_vertical[:B].view(B, 1, 1, 1)
        masks = torch.where(fh, masks.flip(-1), masks)
        return torch.where(fv, masks.flip(-2), masks)
