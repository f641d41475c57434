"""lidar_sweeps -- LoadPointsFromMultiSweeps + PointsRangeFilter of the LiDAR pipeline (loading.py:87-235,
transforms_3d.py:585-614, base_points.py:208-232) on the device (csrc/lidar_sweeps.cu), bit-exact to the reference.

    SweepStore(slots, slot_cap, load_dim, device)
        raw point rows [slots, slot_cap, load_dim] fp32 on the device plus a device row count per slot.
        put(slot, points) uploads one raw sweep (or key) asynchronously; a frame names its entries by slot, so a
        caller running at the sweep rate uploads one new sweep per frame.
        assemble(samples, use_dim, ...) -> per sample the reference's results["points"].tensor
        write_frame(samples, use_dim, ...) + launch(batch, out_dim, cap): the same split in two, for CUDA graphs: the
        frame's parameters go to a device block at a fixed address in one copy, and launch() reads them from there.
        aug= (a lidar_aug.LidarAug) applies GlobalRotScaleTrans + RandomFlip3D to every row before the range filter,
        as the reference's training pipeline orders them.
        paste= (an object_paste.PasteBlock) applies ObjectPaste first: the rows inside each sample's kept boxes are
        removed and the kept objects' rows come first, then every row is augmented and range-filtered.
    assemble_sweeps(key, sweeps, rotations, translations, lags, use_dim, ...)   one sample from host or device arrays
    choose_sweeps(n_sweeps, sweeps_num, test_mode)   the reference's sweep draw, on numpy's global RNG
    time_lag(timestamp, sweep_timestamp)             the reference's ts - sweep_ts (float64)

A sample is (key_slot, sweeps) with sweeps the chosen sweeps in the order of `choices`, each (slot, rotation [3, 3],
translation [3], lag).  With pad_empty_sweeps and no sweeps, the key is repeated sweeps_num times, through
remove_close, with time 0.  The key's slot holds the raw row LoadPointsFromFile reads; key_use_dim is that
loader's use_dim (default: every column), and the sweep loader's use_dim is applied on top, as in the reference.
GPU only: CPU stores raise."""
import numpy as np
import torch

from . import _C

__all__ = ["SlotStore", "SweepStore", "assemble_sweeps", "choose_sweeps", "time_lag", "OVERFLOW", "BAD_ENTRY",
           "BAD_PARAMS", "BAD_PASTE"]

NONE, KEY, SWEEP, PAD = 0, 1, 2, 3            # BEVB200_SWEEP_*
MAX_DIM = 8                                   # BEVB200_SWEEP_MAX_DIM: F <= 8, as the fused voxelizer takes
OVERFLOW, BAD_ENTRY, BAD_PARAMS, BAD_PASTE = 1, 2, 4, 8    # BEVB200_SWEEPS_*: status bits

# bevb200_sweep_entry_t / bevb200_sweep_params_t, C layout (align=True)
ENTRY_DTYPE = np.dtype([("kind", "<i4"), ("slot", "<i4"), ("rotation", "<f8", (9,)), ("translation", "<f8", (3,)),
                        ("lag", "<f8")], align=True)
PARAMS_DTYPE = np.dtype([("key_cols", "<i4", (MAX_DIM,)), ("sweep_cols", "<i4", (MAX_DIM,)), ("remove_close", "<i4"),
                         ("has_range", "<i4"), ("radius", "<f4"), ("range", "<f4", (6,))], align=True)
_ENTRIES_AT = 128                             # byte offset of the entries in the parameter block


def choose_sweeps(n_sweeps, sweeps_num, test_mode=False):
    """Indices of the sweeps LoadPointsFromMultiSweeps loads (loading.py:196-210), drawn as the reference draws
    them: all of them when there are at most sweeps_num, the first sweeps_num in test_mode, otherwise
    np.random.choice(n_sweeps, sweeps_num, replace=False) on numpy's global RNG (so sweeps_num = 0 still consumes
    it, and a pipeline that leaves test_mode unset draws at test time too)."""
    if n_sweeps <= sweeps_num:
        return np.arange(n_sweeps)
    if test_mode:
        return np.arange(sweeps_num)
    return np.random.choice(n_sweeps, sweeps_num, replace=False)


def time_lag(timestamp, sweep_timestamp):
    """Column 4 of a sweep before its fp32 store: results["timestamp"] / 1e6 - sweep["timestamp"] / 1e6."""
    return timestamp / 1e6 - sweep_timestamp / 1e6


def _dims(use_dim, n, name):
    if isinstance(use_dim, int):
        use_dim = list(range(use_dim))
    use_dim = [int(c) for c in use_dim]
    if any(c < 0 or c >= n for c in use_dim):
        raise ValueError("%s %s names a column outside [0, %d)" % (name, use_dim, n))
    return use_dim


def _check_loader_options(reduce_beams, load_augmented):
    # loading.py:148-149, 216-217: only these values leave the points as they are
    if reduce_beams and reduce_beams < 32:
        raise ValueError("reduce_beams=%r is not supported (None or >= 32 leave the beams as they are)" % reduce_beams)
    if load_augmented:
        raise ValueError("load_augmented=%r is not supported" % load_augmented)


class SlotStore:
    """Raw sweep rows on the device, one sweep per slot ([slots, slot_cap, load_dim] fp32 plus a device row count per
    slot), and a device block of block_bytes for the parameters of the frame being assembled.  SweepStore and
    radar_sweeps.RadarSweepStore build on it."""

    def __init__(self, slots, slot_cap, load_dim, device, block_bytes):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError("%s lives on a CUDA device: bevfusion_b200 has no CPU implementation"
                             % type(self).__name__)
        self.slots, self.slot_cap, self.load_dim = int(slots), int(slot_cap), int(load_dim)
        self.rows = torch.zeros((slots, slot_cap, load_dim), dtype=torch.float32, device=self.device)
        self.slot_rows = torch.zeros((slots,), dtype=torch.int32, device=self.device)
        self.host_rows = [0] * slots          # what put() stored, for the default cap
        self.block = torch.empty((block_bytes,), dtype=torch.uint8, device=self.device)

    def put(self, slot, points):
        """Store `points` [n, load_dim] fp32 (pinned host or CUDA; other host memory is copied synchronously) in
        `slot`.  The copy and the row count are enqueued on the current stream."""
        if not 0 <= slot < self.slots:
            raise ValueError("slot %d outside [0, %d)" % (slot, self.slots))
        if isinstance(points, np.ndarray):
            points = torch.from_numpy(np.ascontiguousarray(points, np.float32))
        if points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] != self.load_dim:
            raise ValueError("points must be float32 [n, %d], got %s %s" % (self.load_dim, points.dtype,
                                                                            tuple(points.shape)))
        n = points.shape[0]
        if n > self.slot_cap:
            raise ValueError("%d rows do not fit a slot of %d" % (n, self.slot_cap))
        with torch.cuda.device(self.device):
            if n:
                self.rows[slot, :n].copy_(points, non_blocking=True)
            self.slot_rows[slot:slot + 1].fill_(n)
        self.host_rows[slot] = n

    def _write_block(self, host):
        # one pinned asynchronous copy into the block the assemble launches read
        with torch.cuda.device(self.device):
            self.block[:host.size].copy_(torch.from_numpy(host).pin_memory(), non_blocking=True)


class SweepStore(SlotStore):
    """Raw LiDAR rows on the device, one sweep (or key) per slot, and the parameter block of the frame being
    assembled.  max_batch and max_entries size the block: a sample has at most max_entries entries (its key and its
    sweeps or pad copies)."""

    def __init__(self, slots, slot_cap, load_dim=5, device="cuda", max_batch=4, max_entries=11):
        if slots < 1 or slot_cap < 1 or max_batch < 1 or max_entries < 1:
            raise ValueError("slots, slot_cap, max_batch and max_entries must be positive")
        if not 3 <= load_dim <= 64:
            raise ValueError("load_dim must be in 3..64, got %d" % load_dim)
        if max_entries * slot_cap >= 2 ** 31:
            raise ValueError("max_entries * slot_cap must be below 2^31")
        self.max_batch, self.max_entries = int(max_batch), int(max_entries)
        super().__init__(slots, slot_cap, load_dim, device,
                         _ENTRIES_AT + max_batch * max_entries * ENTRY_DTYPE.itemsize)

    def _pack(self, samples, use_dim, key_use_dim, sweeps_num, pad_empty_sweeps, remove_close, point_cloud_range,
              radius):
        sweep_cols = _dims(use_dim, self.load_dim, "use_dim")
        F = len(sweep_cols)
        if not 5 <= F <= MAX_DIM:
            raise ValueError("len(use_dim) must be in 5..8 (column 4 is the time lag), got %d" % F)
        file_cols = _dims(range(self.load_dim) if key_use_dim is None else key_use_dim, self.load_dim, "key_use_dim")
        key_cols = [file_cols[c] for c in _dims(sweep_cols, len(file_cols), "use_dim (on the key)")]
        B = len(samples)
        if B > self.max_batch:
            raise ValueError("%d samples, the store was made for %d" % (B, self.max_batch))
        p = np.zeros((), PARAMS_DTYPE)
        p["key_cols"][:F], p["sweep_cols"][:F] = key_cols, sweep_cols
        p["remove_close"] = int(bool(remove_close))
        p["radius"] = np.float32(radius)
        if point_cloud_range is not None:
            rng = np.asarray(point_cloud_range, np.float32)     # PointsRangeFilter keeps the range as np.float32
            if rng.shape != (6,):
                raise ValueError("point_cloud_range needs 6 values")
            p["has_range"], p["range"] = 1, rng
        e = np.zeros((B, self.max_entries), ENTRY_DTYPE)
        bound = 0
        for b, (key_slot, sweeps) in enumerate(samples):
            ents = [(KEY, key_slot, None)]
            if pad_empty_sweeps and len(sweeps) == 0:
                ents += [(PAD, key_slot, None)] * sweeps_num
            else:
                ents += [(SWEEP, s[0], s) for s in sweeps]
            if len(ents) > self.max_entries:
                raise ValueError("sample %d has %d entries, the store was made for %d" % (b, len(ents),
                                                                                       self.max_entries))
            for j, (kind, slot, s) in enumerate(ents):
                if not 0 <= slot < self.slots:
                    raise ValueError("sample %d names slot %d outside [0, %d)" % (b, slot, self.slots))
                e["kind"][b, j], e["slot"][b, j] = kind, slot
                if s is not None:
                    R, t = np.asarray(s[1], np.float64), np.asarray(s[2], np.float64)
                    if R.shape != (3, 3) or t.shape != (3,):
                        raise ValueError("a sweep needs rotation [3, 3] and translation [3]")
                    e["rotation"][b, j], e["translation"][b, j], e["lag"][b, j] = R.reshape(9), t, float(s[3])
            bound = max(bound, sum(self.host_rows[slot] for _, slot, _ in ents))
        host = np.zeros(_ENTRIES_AT + e.nbytes, np.uint8)
        host[:PARAMS_DTYPE.itemsize] = np.frombuffer(p.tobytes(), np.uint8)
        host[_ENTRIES_AT:] = np.frombuffer(e.tobytes(), np.uint8)
        return host, F, bound

    def write_frame(self, samples, use_dim, key_use_dim=None, sweeps_num=9, pad_empty_sweeps=True, remove_close=True,
                    point_cloud_range=None, radius=1.0, reduce_beams=None, load_augmented=None, paste=None):
        """Pack the frame's parameters and copy them, in one pinned asynchronous copy, into the device block that
        launch() reads.  Returns (batch, out_dim, bound): bound is the most rows a sample can keep, from the row
        counts put() stored, plus the rows paste's last write() pastes into a sample."""
        _check_loader_options(reduce_beams, load_augmented)
        host, F, bound = self._pack(samples, use_dim, key_use_dim, sweeps_num, pad_empty_sweeps, remove_close,
                                    point_cloud_range, radius)
        if paste is not None:
            _check_paste(paste, len(samples), F, self.device)
            bound += max(paste.rows[:len(samples)], default=0)
        self._write_block(host)
        return len(samples), F, bound

    def launch(self, batch, out_dim, cap, aug=None, paste=None):
        """Assemble the frame the block holds: (points [batch, cap, out_dim], counts [batch] int32, status [1]
        int32), all on the device, no host synchronisation; CUDA-graph capturable.  With aug (a LidarAug whose
        records write() refreshed) each row is augmented before the range test.  With paste (a PasteBlock whose
        write() covered the batch) each sample's kept objects are pasted and the rows in their boxes removed first."""
        if not 0 <= batch <= self.max_batch or not 5 <= out_dim <= MAX_DIM or cap < 1:
            raise ValueError("batch %d, out_dim %d or cap %d out of range" % (batch, out_dim, cap))
        _check_aug(aug, batch, self.device)
        dev = self.device
        L = _C.lib()
        if paste is not None:
            _check_paste(paste, batch, out_dim, dev)
            return self._launch_paste(batch, out_dim, cap, aug, paste)
        ws_bytes = L.bevb200_lidar_sweeps_workspace_bytes(batch, self.max_entries, self.slot_cap)
        out = torch.empty((batch, cap, out_dim), dtype=torch.float32, device=dev)
        counts = torch.empty((batch,), dtype=torch.int32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
        base = self.block.data_ptr()
        with torch.cuda.device(dev):
            if aug is None:
                _C.check(L.bevb200_lidar_sweeps_assemble(
                    _C.ptr(self.rows), self.slots, self.slot_cap, self.load_dim, _C.ptr(self.slot_rows), base,
                    base + _ENTRIES_AT, batch, self.max_entries, out_dim, cap, _C.ptr(out), _C.ptr(counts),
                    _C.ptr(status), _C.ptr(ws), ws.numel(), _C.current_stream(dev)), "lidar_sweeps_assemble")
            else:
                _C.check(L.bevb200_lidar_sweeps_assemble_aug(
                    _C.ptr(self.rows), self.slots, self.slot_cap, self.load_dim, _C.ptr(self.slot_rows), base,
                    base + _ENTRIES_AT, aug.ptr(), batch, self.max_entries, out_dim, cap, _C.ptr(out), _C.ptr(counts),
                    _C.ptr(status), _C.ptr(ws), ws.numel(), _C.current_stream(dev)), "lidar_sweeps_assemble_aug")
        return out, counts, status

    def _launch_paste(self, batch, out_dim, cap, aug, paste):
        dev, ps = self.device, paste.store
        L = _C.lib()
        ws_bytes = L.bevb200_lidar_sweeps_paste_workspace_bytes(batch, self.max_entries, self.slot_cap,
                                                                paste.max_paste, ps.object_cap)
        if ws_bytes == 0 and batch:
            raise ValueError("max_entries + max_paste or the object cap out of range")
        out = torch.empty((batch, cap, out_dim), dtype=torch.float32, device=dev)
        counts = torch.empty((batch,), dtype=torch.int32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
        base = self.block.data_ptr()
        with torch.cuda.device(dev):
            _C.check(L.bevb200_lidar_sweeps_assemble_paste(
                _C.ptr(self.rows), self.slots, self.slot_cap, self.load_dim, _C.ptr(self.slot_rows), base,
                base + _ENTRIES_AT, 0 if aug is None else aug.ptr(), _C.ptr(ps.rows), ps.max_rows, ps.load_dim,
                _C.ptr(ps.table), ps.max_objects, ps.object_cap, paste.samples_ptr(), paste.objects_ptr(),
                paste.max_paste, batch, self.max_entries, out_dim, cap, _C.ptr(out), _C.ptr(counts), _C.ptr(status),
                _C.ptr(ws), ws.numel(), _C.current_stream(dev)), "lidar_sweeps_assemble_paste")
        return out, counts, status

    def assemble(self, samples, use_dim, key_use_dim=None, sweeps_num=9, pad_empty_sweeps=True, remove_close=True,
                 point_cloud_range=None, cap=None, sync=True, radius=1.0, reduce_beams=None, load_augmented=None,
                 aug=None, paste=None):
        """LoadPointsFromMultiSweeps (+ ObjectPaste with paste, a PasteBlock holding one draw per sample)
        (+ GlobalRotScaleTrans and RandomFlip3D with aug, a LidarAug holding one draw per sample)
        (+ PointsRangeFilter with point_cloud_range) for each sample.

        sync=True: a list of [n_k, len(use_dim)] tensors, the reference's results["points"].tensor; raises when a
        sample keeps more than cap rows.  sync=False: (points [B, cap, F], counts [B] int32, status [1] int32) on
        the device, with no host synchronisation; rows past counts[k] are unspecified.  cap defaults to the most
        rows a sample can keep, so no sample overflows it."""
        batch, F, bound = self.write_frame(samples, use_dim, key_use_dim, sweeps_num, pad_empty_sweeps, remove_close,
                                           point_cloud_range, radius, reduce_beams, load_augmented, paste)
        out, counts, status = self.launch(batch, F, max(bound, 1) if cap is None else int(cap), aug, paste)
        if not sync:
            return out, counts, status
        st = int(status.item())
        if st:
            raise ValueError("lidar_sweeps_assemble status %d: %s" % (st, ", ".join(
                name for bit, name in ((OVERFLOW, "a sample keeps more than cap rows"), (BAD_ENTRY, "a bad entry"),
                                       (BAD_PARAMS, "bad column maps"), (BAD_PASTE, "a bad paste block"))
                if st & bit)))
        return [out[k, :n] for k, n in enumerate(counts.tolist())]


def _check_aug(aug, batch, device):
    if aug is None:
        return
    if not hasattr(aug, "ptr") or not hasattr(aug, "check_batch"):
        raise TypeError("aug must be a lidar_aug.LidarAug")
    from .lidar_aug import cuda_device
    if aug.device != cuda_device(device):
        raise ValueError("aug is on %s, the store on %s" % (aug.device, device))
    aug.check_batch(batch)


def _check_paste(paste, batch, out_dim, device):
    from .lidar_aug import cuda_device
    from .object_paste import PasteBlock
    if not isinstance(paste, PasteBlock):
        raise TypeError("paste must be an object_paste.PasteBlock")
    if paste.device != cuda_device(device):
        raise ValueError("paste is on %s, the store on %s" % (paste.device, device))
    paste.check_batch(batch, out_dim)


def assemble_sweeps(key, sweeps, rotations, translations, lags, use_dim, key_use_dim=None, sweeps_num=9,
                    pad_empty_sweeps=True, remove_close=True, point_cloud_range=None, device="cuda", radius=1.0):
    """One sample: key [n0, load_dim] and the chosen sweeps [n_i, load_dim] (raw rows, numpy or torch, in the
    order of `choices`) with their rotations [3, 3], translations [3] and time lags -> [n, len(use_dim)] fp32 on
    the device, the reference's results["points"].tensor."""
    if not (len(sweeps) == len(rotations) == len(translations) == len(lags)):
        raise ValueError("sweeps, rotations, translations and lags must have one entry per sweep")
    rows = [key] + list(sweeps)
    load_dim = rows[0].shape[1]
    cap = max(max(r.shape[0] for r in rows), 1)
    entries = 1 + (sweeps_num if pad_empty_sweeps and not sweeps else len(sweeps))
    store = SweepStore(len(rows), cap, load_dim, device, max_batch=1, max_entries=entries)
    for s, r in enumerate(rows):
        store.put(s, r)
    sample = (0, [(i + 1, rotations[i], translations[i], lags[i]) for i in range(len(sweeps))])
    return store.assemble([sample], use_dim, key_use_dim, sweeps_num, pad_empty_sweeps, remove_close,
                          point_cloud_range, radius=radius)[0]
