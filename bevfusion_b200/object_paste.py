"""object_paste -- ObjectPaste (GT-database sampling) of the LiDAR training pipeline (transforms_3d.py:357-449,
dbsampler.py, box_np_ops.py:430-451, 692-775, pipelines/utils.py:31-111), bit-exact to the reference.

The draw and the collision test run here, on the host: their inputs are annotations (tens of boxes), and their result
decides which objects' rows have to reach the device at all.  The removal of the points inside the kept boxes and the
paste of the objects' rows run inside the sweep assemble kernels (csrc/lidar_sweeps.cu), with paste= on
SweepStore.write_frame / launch / assemble.

    DataBaseSampler(db_infos, rate, prepare, sample_groups, classes, rng=None)
        the reference's sampler over a loaded dbinfos dict: filter_by_difficulty / filter_by_min_points in the order of
        `prepare`, then one shuffled class sampler per database key, in dict order (each consumes the RNG).
    ObjectPaste(sampler, stop_epoch=None)
        set_epoch(epoch); draw(gt_bboxes [N, 9] f32, gt_labels) -> PasteDraw or None (nothing pasted, nothing drawn
        once epoch >= stop_epoch); merge(gt_bboxes, gt_labels, draw) -> the reference's gt_bboxes_3d / gt_labels_3d.
    box_collision_test(boxes, qboxes)   the reference's numba collision test, vectorised, bit for bit
    box_planes(boxes) -> (normal [S, 6, 3], d [S, 6]) fp32, points_in_rbbox's face planes
    load_object_points(path, load_dim)  an object's raw rows as LoadPointsFromFile reads them (before use_dim)
    ObjectStore(max_rows, load_dim, max_objects, object_cap, device)
        packed raw object rows [max_rows, load_dim] fp32 and an (offset, rows) table on the device: put(index, rows),
        clear().  Holds the whole filtered database (index = PasteDraw.indices) or each frame's drawn objects.
    PasteBlock(store, max_batch, max_paste, device)
        the per-frame device block the kernels read: write(draws, use_dim, indices=None) in one pinned asynchronous
        copy, so a CUDA graph replays with new draws and new objects.

Every draw is made on numpy's global RNG (or `rng`), as the reference makes it, so a caller reproducing a reference
sample calls draw() after the sweep choice and before ImageAug3D's draws (INTEGRATION.md).  GPU only for the device
classes: a CPU device raises."""
import collections

import numpy as np
import torch

from . import _C

__all__ = ["DataBaseSampler", "ObjectPaste", "PasteDraw", "box_collision_test", "center_to_corner_box2d",
           "box_planes", "load_object_points", "ObjectStore", "PasteBlock", "BAD_PASTE", "MAX_PASTE"]

BAD_PASTE = 8                                  # BEVB200_SWEEPS_BAD_PASTE
MAX_PASTE = 256                                # BEVB200_PASTE_MAX_OBJECTS
MAX_DIM = 8                                    # BEVB200_SWEEP_MAX_DIM

# bevb200_paste_sample_t / bevb200_paste_object_t, C layout
SAMPLE_DTYPE = np.dtype([("count", "<i4"), ("cols", "<i4", (MAX_DIM,)), ("reserved", "<i4", (3,))], align=True)
OBJECT_DTYPE = np.dtype([("index", "<i4"), ("translation", "<f4", (3,)), ("planes", "<f4", (6, 4))], align=True)

PasteDraw = collections.namedtuple("PasteDraw", "infos indices boxes labels")
PasteDraw.__doc__ = """One sample's kept objects in the reference's order: their db infos, their indices in
DataBaseSampler.infos, boxes [S, 9] (their box3d_lidar) and labels [S] int64."""


class _ClassSampler:
    """The reference's BatchSampler over one class: a shuffled index order consumed in runs; a run that reaches the
    end (idx + num >= n, equality included) returns the remainder, then reshuffles and restarts."""

    def __init__(self, n, rng):
        self.rng = rng
        self.order = np.arange(n)
        self._r().shuffle(self.order)
        self.idx = 0

    def _r(self):
        return np.random if self.rng is None else self.rng

    def sample(self, num):
        if self.idx + num >= len(self.order):
            ret = self.order[self.idx:].copy()
            self._r().shuffle(self.order)
            self.idx = 0
        else:
            ret = self.order[self.idx:self.idx + num].copy()
            self.idx += num
        return ret


class DataBaseSampler:
    """The reference's DataBaseSampler on an already loaded dbinfos dict ({class: [info, ...]}, each info with
    "name", "path", "box3d_lidar" (float32, as the GT-database builder stores it), "difficulty" and
    "num_points_in_gt").  infos is the filtered database flattened in key order; PasteDraw.indices index it."""

    def __init__(self, db_infos, rate, prepare, sample_groups, classes, rng=None):
        self.rate = rate
        self.classes = list(classes)
        self.cat2label = {name: i for i, name in enumerate(self.classes)}
        for prep, val in prepare.items():
            if prep == "filter_by_difficulty":
                db_infos = {k: [i for i in v if i["difficulty"] not in val] for k, v in db_infos.items()}
            elif prep == "filter_by_min_points":
                db_infos = dict(db_infos)
                for name, min_num in val.items():
                    if int(min_num) > 0:
                        db_infos[name] = [i for i in db_infos[name] if i["num_points_in_gt"] >= int(min_num)]
            else:
                raise ValueError("unknown prepare function %r" % prep)
        self.db_infos = db_infos
        for k, v in db_infos.items():
            for info in v:
                if np.asarray(info["box3d_lidar"]).dtype != np.float32:
                    raise ValueError("db info boxes must be float32 (class %s)" % k)
        self.sample_groups = [(name, int(num)) for name, num in sample_groups.items()]
        self.infos, self.first = [], {}
        for k, v in db_infos.items():
            self.first[k] = len(self.infos)
            self.infos += v
        self.samplers = {k: _ClassSampler(len(v), rng) for k, v in db_infos.items()}

    def sample_all(self, gt_bboxes, gt_labels):
        """The reference's sample_all without the file loads: (infos, indices, boxes [S, 9], labels [S]) or None"""
        nums = []
        for name, max_num in self.sample_groups:
            label = self.cat2label[name]
            n = int(max_num - np.sum([g == label for g in gt_labels]))
            nums.append(np.round(self.rate * n).astype(np.int64))
        infos, indices, boxes = [], [], []
        avoid = gt_bboxes
        for (name, _), num in zip(self.sample_groups, nums):
            if num <= 0:
                continue
            kept = self._sample_class(name, num, avoid)
            if kept:
                infos += [self.db_infos[name][i] for i in kept]
                indices += [self.first[name] + i for i in kept]
                b = np.stack([self.db_infos[name][i]["box3d_lidar"] for i in kept], axis=0)
                boxes.append(b)
                avoid = np.concatenate([avoid, b], axis=0)
        if not infos:
            return None
        labels = np.array([self.cat2label[i["name"]] for i in infos], dtype=np.int64)
        return infos, indices, np.concatenate(boxes, axis=0), labels

    def _sample_class(self, name, num, gt_bboxes):
        """sample_class_v2: the drawn candidates' positions in db_infos[name] that pass the collision loop"""
        drawn = self.samplers[name].sample(num)
        if len(drawn) == 0:
            raise ValueError("need at least one array to stack (class %s has no database objects)" % name)
        sp = np.stack([self.db_infos[name][i]["box3d_lidar"] for i in drawn], axis=0)
        # the avoid-set's and the candidates' corners in two calls, as the reference makes them
        sp = np.concatenate([gt_bboxes, sp], axis=0)[gt_bboxes.shape[0]:]
        total = np.concatenate([center_to_corner_box2d(b[:, 0:2], b[:, 3:5], b[:, 6]) for b in (gt_bboxes, sp)])
        num_gt = gt_bboxes.shape[0]
        coll = box_collision_test(total[num_gt:], total)        # the candidates' rows of the full matrix
        coll[np.arange(len(drawn)), num_gt + np.arange(len(drawn))] = False
        kept = []
        for k in range(len(drawn)):
            if coll[k].any():
                coll[k] = False
                coll[:, num_gt + k] = False
            else:
                kept.append(int(drawn[k]))
        return kept


def _corners(dims, norm):
    # corners_nd: dims * (corner pattern - origin) in dims' dtype
    return dims.reshape(-1, 1, dims.shape[1]) * (np.asarray(norm, dims.dtype)).reshape(1, *np.shape(norm))


def center_to_corner_box2d(centers, dims, angles):
    """BEV corners [N, 4, 2] (clockwise from the minimum corner, origin 0.5) with box_np_ops' numpy calls, in the
    boxes' dtype"""
    corners = _corners(dims, np.array([[0, 0], [0, 1], [1, 1], [1, 0]], dims.dtype) - np.array(0.5, dims.dtype))
    s, c = np.sin(angles), np.cos(angles)
    corners = np.einsum("aij,jka->aik", corners, np.stack([[c, -s], [s, c]]))
    corners += centers.reshape([-1, 1, 2])
    return corners


_CORNERS_3D = [[0, 0, 0], [0, 0, 1], [0, 1, 1], [0, 1, 0], [1, 0, 0], [1, 0, 1], [1, 1, 1], [1, 1, 0]]
_FACES = [[0, 1, 2, 3], [7, 6, 5, 4], [0, 3, 7, 4], [1, 5, 6, 2], [0, 4, 5, 1], [3, 2, 6, 7]]


def box_planes(boxes):
    """points_in_rbbox's face planes of boxes [S, >= 7] (origin (0.5, 0.5, 0), z axis): (normal [S, 6, 3], d [S, 6])
    with the reference's numpy calls in its order (corners, np.cross, np.einsum), in the boxes' dtype.  A point is
    inside a box unless ((x n0 + y n1) + z n2) + d >= 0 for one face."""
    dims = boxes[:, 3:6]
    corners = _corners(dims, np.array(_CORNERS_3D, dims.dtype) - np.array([0.5, 0.5, 0], dtype=dims.dtype))
    s, c = np.sin(boxes[:, 6]), np.cos(boxes[:, 6])
    zeros, ones = np.zeros_like(c), np.ones_like(c)
    rot = np.stack([[c, -s, zeros], [s, c, zeros], [zeros, zeros, ones]])
    corners = np.einsum("aij,jka->aik", corners, rot)
    corners += boxes[:, :3].reshape([-1, 1, 3])
    surfaces = corners[:, _FACES][:, :, :3, :]
    vec = surfaces[:, :, :2, :] - surfaces[:, :, 1:3, :]
    normal = np.cross(vec[:, :, 0, :], vec[:, :, 1, :])
    d = np.einsum("aij, aij->ai", normal, surfaces[:, :, 0, :])
    return normal, -d


def box_collision_test(boxes, qboxes):
    """The reference's box_collision_test(boxes [N, 4, 2], qboxes [K, 4, 2], clockwise=True) -> [N, K] bool, with the
    same operations in the same dtype, evaluated for every pair at once: the strict standup overlap (iw > 0, ih > 0),
    then a proper segment crossing of any edge pair, then containment of one box's corners in the other."""
    N, K = boxes.shape[0], qboxes.shape[0]
    if N == 0 or K == 0:
        return np.zeros((N, K), np.bool_)
    lo, hi, qlo, qhi = boxes.min(1), boxes.max(1), qboxes.min(1), qboxes.max(1)
    iw = np.minimum(hi[:, None, 0], qhi[None, :, 0]) - np.maximum(lo[:, None, 0], qlo[None, :, 0])
    ih = np.minimum(hi[:, None, 1], qhi[None, :, 1]) - np.maximum(lo[:, None, 1], qlo[None, :, 1])
    standup = (iw > 0) & (ih > 0)
    nxt = [1, 2, 3, 0]
    A = boxes[:, None, :, None, :]                    # [N, 1, 4 (k), 1, 2]
    B = boxes[:, nxt][:, None, :, None, :]
    C = qboxes[None, :, None, :, :]                   # [1, K, 1, 4 (l), 2]
    D = qboxes[:, nxt][None, :, None, :, :]

    def ccw(P, Q, R):   # (R1 - P1) * (Q0 - P0) > (Q1 - P1) * (R0 - P0)
        return (R[..., 1] - P[..., 1]) * (Q[..., 0] - P[..., 0]) > (Q[..., 1] - P[..., 1]) * (R[..., 0] - P[..., 0])

    acd, bcd = ccw(A, C, D), ccw(B, C, D)
    abc, abd = ccw(A, B, C), ccw(A, B, D)
    cross_edges = ((acd != bcd) & (abc != abd)).any(axis=(2, 3))

    def contains(P, Q):
        # [n, k]: every corner l of Q strictly inside P: no edge k of P has cross >= 0 (NaN counts as inside)
        vec = -(P - P[:, nxt])                                          # [n, 4, 2]
        Pk = P[:, None, :, None, :]
        v = vec[:, None, :, None, :]
        Ql = Q[None, :, None, :, :]
        cross = v[..., 1] * (Pk[..., 0] - Ql[..., 0])
        cross = cross - v[..., 0] * (Pk[..., 1] - Ql[..., 1])
        return ~(cross >= 0).any(axis=(2, 3))

    return standup & (cross_edges | contains(boxes, qboxes) | contains(qboxes, boxes).T)


def load_object_points(path, load_dim):
    """One object's raw rows [n, load_dim] fp32 as LoadPointsFromFile reads them (np.fromfile, then reshape); the
    loader's use_dim is applied on the device by the paste block's column map."""
    return np.fromfile(path, dtype=np.float32).reshape(-1, load_dim)


class ObjectPaste:
    """The reference's ObjectPaste without sample_2d: the draw on the host, the removal and the paste on the device."""

    def __init__(self, sampler, stop_epoch=None, sample_2d=False):
        if sample_2d:
            raise ValueError("sample_2d (pasting image patches) is not supported")
        self.sampler = sampler
        self.stop_epoch = stop_epoch
        self.epoch = -1

    def set_epoch(self, epoch):
        self.epoch = epoch

    def draw(self, gt_bboxes, gt_labels):
        """One sample's draw from its GT boxes [N, 9] f32 and labels [N] (-1 never counts): a PasteDraw, or None when
        nothing is kept or the epoch gate is closed (then nothing is drawn)."""
        if self.stop_epoch is not None and self.epoch >= self.stop_epoch:
            return None
        gt_bboxes = np.asarray(gt_bboxes)
        if gt_bboxes.dtype != np.float32 or gt_bboxes.ndim != 2 or gt_bboxes.shape[1] < 7:
            raise ValueError("gt_bboxes must be float32 [N, >= 7], got %s %s" % (gt_bboxes.dtype, gt_bboxes.shape))
        got = self.sampler.sample_all(gt_bboxes, np.asarray(gt_labels))
        return None if got is None else PasteDraw(*got)

    @staticmethod
    def merge(gt_bboxes, gt_labels, draw):
        """The reference's gt_bboxes_3d tensor [N + S, D] float32 and gt_labels_3d [N + S] int64 after the paste"""
        gt_bboxes = np.asarray(gt_bboxes, np.float32)
        gt_labels = np.asarray(gt_labels)
        if draw is None:
            return gt_bboxes, gt_labels.astype(np.int64)
        return (np.concatenate([gt_bboxes, draw.boxes]).astype(np.float32),
                np.concatenate([gt_labels, draw.labels]).astype(np.int64))


def _cuda(device, what):
    from .lidar_aug import cuda_device
    device = torch.device(device)
    if device.type != "cuda":
        raise ValueError("%s lives on a CUDA device: bevfusion_b200 has no CPU implementation" % what)
    return cuda_device(device)


class ObjectStore:
    """Raw object rows packed on the device ([max_rows, load_dim] fp32) with a device table [max_objects, 2] int32 of
    (first row, rows) per object index.  put() appends; clear() empties the store and the table."""

    def __init__(self, max_rows, load_dim=5, max_objects=1, object_cap=16384, device="cuda"):
        self.device = _cuda(device, "ObjectStore")
        if max_rows < 0 or max_objects < 1 or object_cap < 1 or not 1 <= load_dim <= 64:
            raise ValueError("need max_rows >= 0, max_objects >= 1, object_cap >= 1 and 1 <= load_dim <= 64")
        self.max_rows, self.load_dim, self.max_objects, self.object_cap = (int(max_rows), int(load_dim),
                                                                           int(max_objects), int(object_cap))
        self.rows = torch.zeros((max(self.max_rows, 1), self.load_dim), dtype=torch.float32, device=self.device)
        self.table = torch.zeros((self.max_objects, 2), dtype=torch.int32, device=self.device)
        self.host_rows = np.zeros(self.max_objects, np.int64)
        self.used = 0

    def clear(self):
        with torch.cuda.device(self.device):
            self.table.zero_()
        self.host_rows[:] = 0
        self.used = 0

    def put(self, index, rows):
        """Store object `index`'s raw rows [n, load_dim] fp32 (numpy, pinned host or CUDA) after the rows stored so
        far; the copy and the table entry are enqueued on the current stream."""
        if not 0 <= index < self.max_objects:
            raise ValueError("object %d outside [0, %d)" % (index, self.max_objects))
        if isinstance(rows, np.ndarray):
            rows = torch.from_numpy(np.ascontiguousarray(rows, np.float32))
        if rows.dtype != torch.float32 or rows.dim() != 2 or rows.shape[1] != self.load_dim:
            raise ValueError("rows must be float32 [n, %d], got %s %s" % (self.load_dim, rows.dtype,
                                                                          tuple(rows.shape)))
        n = rows.shape[0]
        if n > self.object_cap or self.used + n > self.max_rows:
            raise ValueError("%d rows do not fit (object_cap %d, %d of %d rows used)" % (n, self.object_cap,
                                                                                        self.used, self.max_rows))
        entry = torch.tensor([self.used, n], dtype=torch.int32).pin_memory()
        with torch.cuda.device(self.device):
            if n:
                self.rows[self.used:self.used + n].copy_(rows, non_blocking=True)
            self.table[index].copy_(entry, non_blocking=True)
        self.host_rows[index] = n
        self.used += n


class PasteBlock:
    """The per-frame paste block on the device: per sample the kept-object count and the column map
    (bevb200_paste_sample_t), then [max_batch, max_paste] kept objects (store index, fl32 translation, 6 face
    planes).  `batch` is the number of samples the last write() was given: a launch over more raises."""

    def __init__(self, store, max_batch, max_paste=64, device=None):
        if not isinstance(store, ObjectStore):
            raise TypeError("store must be an ObjectStore")
        self.store = store
        self.device = store.device if device is None else _cuda(device, "PasteBlock")
        if self.device != store.device:
            raise ValueError("the block and its store must share a device")
        if max_batch < 1 or not 1 <= max_paste <= MAX_PASTE:
            raise ValueError("need max_batch >= 1 and 1 <= max_paste <= %d" % MAX_PASTE)
        self.max_batch, self.max_paste = int(max_batch), int(max_paste)
        self._objects_at = (self.max_batch * SAMPLE_DTYPE.itemsize + 15) // 16 * 16
        self.block = torch.zeros((self._objects_at + self.max_batch * self.max_paste * OBJECT_DTYPE.itemsize,),
                                 dtype=torch.uint8, device=self.device)
        self.batch = 0
        self.rows = [0] * self.max_batch       # pasted rows per sample, for the default cap
        self.out_dim = None

    def samples_ptr(self):
        return self.block.data_ptr()

    def objects_ptr(self):
        return self.block.data_ptr() + self._objects_at

    def write(self, draws, use_dim=5, indices=None):
        """Refresh the block from one PasteDraw (or None: nothing pasted or removed) per sample, in one pinned
        asynchronous copy on the current stream.  use_dim is the database points_loader's use_dim (an int n for
        range(n)); indices[b] gives sample b's objects' store indices (default: draw.indices, for a store holding the
        whole database)."""
        draws = list(draws)
        B = len(draws)
        if B > self.max_batch:
            raise ValueError("%d draws, the block was made for %d" % (B, self.max_batch))
        cols = list(range(use_dim)) if isinstance(use_dim, int) else [int(c) for c in use_dim]
        if not 1 <= len(cols) <= MAX_DIM or any(c < 0 or c >= self.store.load_dim for c in cols):
            raise ValueError("use_dim %s must name 1..%d columns in [0, %d)" % (cols, MAX_DIM, self.store.load_dim))
        smp = np.zeros(self.max_batch, SAMPLE_DTYPE)
        obj = np.zeros((self.max_batch, self.max_paste), OBJECT_DTYPE)
        smp["cols"][:, :len(cols)] = cols
        rows = [0] * self.max_batch
        for b, d in enumerate(draws):
            if d is None:
                continue
            S = len(d.boxes)
            if S > self.max_paste:
                raise ValueError("sample %d keeps %d objects, the block was made for %d" % (b, S, self.max_paste))
            idx = list(d.indices if indices is None else indices[b])
            if len(idx) != S or any(not 0 <= i < self.store.max_objects for i in idx):
                raise ValueError("sample %d needs %d store indices in [0, %d)" % (b, S, self.store.max_objects))
            boxes = np.asarray(d.boxes)
            normal, dd = box_planes(boxes)
            smp["count"][b] = S
            obj["index"][b, :S] = idx
            # BasePoints.translate: tensor.new_tensor(box[:3]), fp32
            obj["translation"][b, :S] = torch.tensor(boxes[:, :3]).to(torch.float32).numpy()
            obj["planes"][b, :S, :, :3] = normal
            obj["planes"][b, :S, :, 3] = dd
            rows[b] = int(self.store.host_rows[idx].sum())
        host = np.zeros(self.block.numel(), np.uint8)
        host[:smp.nbytes] = np.frombuffer(smp.tobytes(), np.uint8)
        host[self._objects_at:] = np.frombuffer(obj.tobytes(), np.uint8)
        with torch.cuda.device(self.device):
            self.block.copy_(torch.from_numpy(host).pin_memory(), non_blocking=True)
        self.batch, self.rows, self.out_dim = B, rows, len(cols)

    def check_batch(self, batch, out_dim):
        """Raise unless the last write() covered `batch` samples with `out_dim` columns."""
        if batch > self.batch:
            raise ValueError("%d samples, but the last PasteBlock.write() had %d draws" % (batch, self.batch))
        if batch and out_dim != self.out_dim:
            raise ValueError("the cloud has %d columns, the pasted objects %s" % (out_dim, self.out_dim))
