"""radar_sweeps -- LoadRadarPointsMultiSweeps + the radar face of PointsRangeFilter (loading.py:717-790,
transforms_3d.py:607-612, radar_points.py:92-107) on the device (csrc/radar_sweeps.cu), bit-exact to the reference.

    RadarSweepStore(slots, slot_cap, device)
        raw radar rows [slots, slot_cap, 18] fp32 on the device plus a device row count per slot (a SlotStore).
        put(slot, points) uploads one raw sweep asynchronously; each radar sweep appears in sweeps_num consecutive
        frames, so a caller at the sweep rate uploads one new sweep per radar and frame.
        assemble(samples, use_dim, ...) -> per sample the reference's results["radar"].tensor after PointsRangeFilter
        write_frame(samples, use_dim, ...) + launch(batch, out_dim, cap): the same split in two, for CUDA graphs: the
        frame's parameters go to a device block at a fixed address in one copy, and launch() reads them from there.
        aug= (a lidar_aug.LidarAug) applies GlobalRotScaleTrans + RandomFlip3D to output columns 0..4 of every row
        (RadarPoints' rotate, scale and flip) before the range filter; it needs len(use_dim) >= 5.
    radar_entries(radars_dict, sweeps_num, slot_of)   one sample's entries: the reference's sweep choice and time lags
    assemble_radar_sweeps(radars_dict, points_of, sweeps_num, use_dim, ...)   one sample, in one call

A sample is a list of entries (slot, sensor2lidar_rotation [3, 3], sensor2lidar_translation [3], time_diff) in the
reference's concatenation order: radars in the iteration order of results['radar'], within each radar its first
min(len(sweeps), sweeps_num) sweeps.  Quirks of the reference that are kept:
  - max_num is accepted and ignored: __call__ never calls _pad_or_drop, so there is no pad, drop or permutation.
  - time_diff is sweeps[0]['timestamp'] * 1e-6 - sweep['timestamp'] * 1e-6 (a product, not LiDAR's / 1e6).
  - a radar with no sweeps raises IndexError at sweeps[0], in radar_entries as in the reference.
  - a one-hot source (columns 3, 11, 14) that is NaN or rounds outside [-w, w) makes the reference raise
    IndexError in perform_encodings; the device leaves that block zero and sets BAD_CATEGORY (assemble(sync=True)
    raises).  Negative values in [-w, -1] wrap as numpy indexing does.
  - `filtering` acts inside the nuScenes devkit's file reader, before the rows reach the store; the device does not
    depend on it.
GPU only: CPU stores raise."""
import numpy as np
import torch

from . import _C
from .lidar_sweeps import SlotStore, SWEEP, _check_aug

__all__ = ["RadarSweepStore", "radar_entries", "assemble_radar_sweeps", "column_ops", "OVERFLOW",
           "BAD_ENTRY", "BAD_PARAMS", "BAD_CATEGORY"]

LOAD_DIM = 18                                           # BEVB200_RADAR_LOAD_DIM
VIRTUAL_DIM = 58                                        # the row after perform_encodings
MAX_DIM = 64                                            # BEVB200_RADAR_SWEEP_MAX_DIM
OVERFLOW, BAD_ENTRY, BAD_PARAMS, BAD_CATEGORY = 1, 2, 4, 8
OP_RAW, OP_XYZ, OP_VELO, OP_VELO_COMP, OP_LAG, OP_ONE_HOT, OP_ORDINAL, OP_NUSC = range(8)   # BEVB200_RADAR_OP_*
OP_NORMALIZE = 1 << 24
NORMALIZE_DIMS = [(3, 0, 50), (4, -100, 100), (5, -100, 100)]     # LoadRadarPointsMultiSweeps' default
BEV_RANGE = (-55.0, -55.0, 55.0, 55.0)                  # PointsRangeFilter's radar face (transforms_3d.py:610)
SHIPPED_USE_DIM = [0, 1, 2, 5, 8, 9] + list(range(18, 57))   # configs/nuscenes/det/default.yaml radar_use_dims

# bevb200_radar_sweep_entry_t / bevb200_radar_sweep_params_t, C layout (align=True)
ENTRY_DTYPE = np.dtype([("kind", "<i4"), ("slot", "<i4"), ("rotation", "<f8", (9,)), ("translation", "<f8", (3,)),
                        ("time_diff", "<f8")], align=True)
PARAMS_DTYPE = np.dtype([("norm_min", "<f8", (MAX_DIM,)), ("norm_span", "<f8", (MAX_DIM,)),
                         ("ops", "<i4", (MAX_DIM,)), ("compensate_velocity", "<i4"), ("has_range", "<i4"),
                         ("range", "<f4", (4,))], align=True)
_ENTRIES_AT = 1536                                      # byte offset of the entries in the parameter block


def _op(kind, arg=0, block=0):
    return kind | arg << 8 | block << 16


def _virtual_op(col):
    """op code of column `col` of the 58-column row (loading.py:769-772 and perform_encodings)"""
    if col < 3:
        return _op(OP_XYZ, col)
    if col < 6 or 10 <= col < 18:
        return _op(OP_RAW, col)
    if col < 8:
        return _op(OP_VELO, col - 6)
    if col < 10:
        return _op(OP_VELO_COMP, col - 8)
    if col == 18:
        return _op(OP_LAG)
    for block, (first, width) in enumerate(((19, 8), (27, 5), (32, 18))):
        if first <= col < first + width:
            return _op(OP_ONE_HOT, col - first, block)
    if col < 57:
        return _op(OP_ORDINAL, col - 50)
    return _op(OP_NUSC)


def column_ops(use_dim, normalize=False, normalize_dims=NORMALIZE_DIMS):
    """(ops int32 [F], norm_min float64 [F], norm_span float64 [F]): use_dim composed into one op code per output
    column, with normalize_feats' (v - min) / (max - min) on the columns normalize_dims names (max - min computed as
    Python computes it).  use_dim may repeat columns and index from the end as numpy does."""
    cols = []
    for c in use_dim:
        c = int(c)
        if not -VIRTUAL_DIM <= c < VIRTUAL_DIM:
            raise ValueError("use_dim names column %d outside the %d-column row" % (c, VIRTUAL_DIM))
        cols.append(c % VIRTUAL_DIM)
    F = len(cols)
    if not 3 <= F <= MAX_DIM:
        raise ValueError("len(use_dim) must be in 3..%d, got %d" % (MAX_DIM, F))
    ops = np.array([_virtual_op(c) for c in cols], np.int32)
    lo, span = np.zeros(F, np.float64), np.ones(F, np.float64)
    if normalize:
        seen = set()
        for dim, mn, mx in normalize_dims:
            dim = int(dim)
            if not -F <= dim < F:
                raise ValueError("normalize_dims names column %d of a %d-column output" % (dim, F))
            dim %= F
            if dim in seen:
                raise ValueError("normalize_dims lists output column %d twice" % dim)
            seen.add(dim)
            ops[dim] |= OP_NORMALIZE
            lo[dim], span[dim] = float(mn), float(mx - mn)
    return ops, lo, span


def radar_entries(radars_dict, sweeps_num, slot_of):
    """One sample's entries from its info dict results['radar'] (radar name -> list of sweep dicts with
    'timestamp', 'sensor2lidar_rotation', 'sensor2lidar_translation'): the reference's sweep choice and time lags
    (loading.py:731-745).  slot_of(sweep) names the store slot holding that sweep's raw rows."""
    entries = []
    for sweeps in radars_dict.values():
        n = len(sweeps) if len(sweeps) < sweeps_num else sweeps_num
        ts = sweeps[0]["timestamp"] * 1e-6     # a radar with no sweeps raises IndexError here, as in the reference
        for idx in range(n):
            sweep = sweeps[idx]
            entries.append((slot_of(sweep), sweep["sensor2lidar_rotation"], sweep["sensor2lidar_translation"],
                            ts - sweep["timestamp"] * 1e-6))
    return entries


class RadarSweepStore(SlotStore):
    """Raw radar rows on the device, one sweep per slot, and the parameter block of the frame being assembled.
    max_batch and max_entries size the block: a sample has at most max_entries sweeps (5 radars x 6 sweeps in the
    shipped config)."""

    def __init__(self, slots, slot_cap, device="cuda", max_batch=4, max_entries=30):
        if slots < 1 or slot_cap < 1 or max_batch < 1 or max_entries < 1:
            raise ValueError("slots, slot_cap, max_batch and max_entries must be positive")
        if max_entries * slot_cap >= 2 ** 31:
            raise ValueError("max_entries * slot_cap must be below 2^31")
        self.max_batch, self.max_entries = int(max_batch), int(max_entries)
        super().__init__(slots, slot_cap, LOAD_DIM, device,
                         _ENTRIES_AT + max_batch * max_entries * ENTRY_DTYPE.itemsize)

    def _pack(self, samples, use_dim, compensate_velocity, normalize, normalize_dims, bev_range):
        ops, lo, span = column_ops(use_dim, normalize, normalize_dims)
        F = len(ops)
        B = len(samples)
        if B > self.max_batch:
            raise ValueError("%d samples, the store was made for %d" % (B, self.max_batch))
        p = np.zeros((), PARAMS_DTYPE)
        p["ops"][:F], p["norm_min"][:F], p["norm_span"][:F] = ops, lo, span
        p["compensate_velocity"] = int(bool(compensate_velocity))
        if bev_range is not None:
            rng = np.asarray(bev_range, np.float64)
            if rng.shape != (4,):
                raise ValueError("bev_range needs 4 values (x_min, y_min, x_max, y_max)")
            p["has_range"], p["range"] = 1, rng.astype(np.float32)   # torch compares fp32 with the fp32 bound
        e = np.zeros((B, self.max_entries), ENTRY_DTYPE)
        bound = 0
        for b, entries in enumerate(samples):
            if len(entries) > self.max_entries:
                raise ValueError("sample %d has %d sweeps, the store was made for %d" % (b, len(entries),
                                                                                      self.max_entries))
            for j, (slot, R, t, td) in enumerate(entries):
                if not 0 <= slot < self.slots:
                    raise ValueError("sample %d names slot %d outside [0, %d)" % (b, slot, self.slots))
                R, t = np.asarray(R, np.float64), np.asarray(t, np.float64)
                if R.shape != (3, 3) or t.shape != (3,):
                    raise ValueError("a sweep needs rotation [3, 3] and translation [3]")
                e["kind"][b, j], e["slot"][b, j] = SWEEP, slot
                e["rotation"][b, j], e["translation"][b, j], e["time_diff"][b, j] = R.reshape(9), t, float(td)
            bound = max(bound, sum(self.host_rows[s[0]] for s in entries))
        host = np.zeros(_ENTRIES_AT + e.nbytes, np.uint8)
        host[:PARAMS_DTYPE.itemsize] = np.frombuffer(p.tobytes(), np.uint8)
        host[_ENTRIES_AT:] = np.frombuffer(e.tobytes(), np.uint8)
        return host, F, bound

    def write_frame(self, samples, use_dim, compensate_velocity=False, normalize=False,
                    normalize_dims=NORMALIZE_DIMS, bev_range=BEV_RANGE, max_num=None):
        """Pack the frame's parameters and copy them, in one pinned asynchronous copy, into the device block that
        launch() reads.  Returns (batch, out_dim, bound): bound is the most rows a sample can keep, from the row
        counts put() stored.  max_num is ignored, as the reference ignores it."""
        host, F, bound = self._pack(samples, use_dim, compensate_velocity, normalize, normalize_dims, bev_range)
        self._write_block(host)
        return len(samples), F, bound

    def launch(self, batch, out_dim, cap, aug=None):
        """Assemble the frame the block holds: (points [batch, cap, out_dim], counts [batch] int32, status [1]
        int32), all on the device, no host synchronisation; CUDA-graph capturable.  With aug (a LidarAug whose
        records write() refreshed) output columns 0..4 are augmented before the range test."""
        if not 0 <= batch <= self.max_batch or not 3 <= out_dim <= MAX_DIM or cap < 1:
            raise ValueError("batch %d, out_dim %d or cap %d out of range" % (batch, out_dim, cap))
        _check_aug(aug, batch, self.device)
        if aug is not None and out_dim < 5:
            raise ValueError("the augmentation reads columns 3 and 4 (RadarPoints.rotate): out_dim must be >= 5")
        dev = self.device
        L = _C.lib()
        ws_bytes = L.bevb200_radar_sweeps_workspace_bytes(batch, self.max_entries, self.slot_cap)
        out = torch.empty((batch, cap, out_dim), dtype=torch.float32, device=dev)
        counts = torch.empty((batch,), dtype=torch.int32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
        base = self.block.data_ptr()
        with torch.cuda.device(dev):
            if aug is None:
                _C.check(L.bevb200_radar_sweeps_assemble(
                    _C.ptr(self.rows), self.slots, self.slot_cap, _C.ptr(self.slot_rows), base, base + _ENTRIES_AT,
                    batch, self.max_entries, out_dim, cap, _C.ptr(out), _C.ptr(counts), _C.ptr(status), _C.ptr(ws),
                    ws.numel(), _C.current_stream(dev)), "radar_sweeps_assemble")
            else:
                _C.check(L.bevb200_radar_sweeps_assemble_aug(
                    _C.ptr(self.rows), self.slots, self.slot_cap, _C.ptr(self.slot_rows), base, base + _ENTRIES_AT,
                    aug.ptr(), batch, self.max_entries, out_dim, cap, _C.ptr(out), _C.ptr(counts), _C.ptr(status),
                    _C.ptr(ws), ws.numel(), _C.current_stream(dev)), "radar_sweeps_assemble_aug")
        return out, counts, status

    def assemble(self, samples, use_dim, compensate_velocity=False, normalize=False, normalize_dims=NORMALIZE_DIMS,
                 bev_range=BEV_RANGE, cap=None, sync=True, max_num=None, aug=None):
        """LoadRadarPointsMultiSweeps (+ GlobalRotScaleTrans and RandomFlip3D with aug, a LidarAug holding one draw
        per sample) (+ PointsRangeFilter's radar face with bev_range; None gives the cloud before any filter) for
        each sample.

        sync=True: a list of [n_k, len(use_dim)] tensors, the reference's results["radar"].tensor; raises when a
        sample keeps more than cap rows or the reference would raise.  sync=False: (points [B, cap, F], counts [B]
        int32, status [1] int32) on the device, with no host synchronisation; rows past counts[k] are unspecified.
        cap defaults to the most rows a sample can keep, so no sample overflows it."""
        batch, F, bound = self.write_frame(samples, use_dim, compensate_velocity, normalize, normalize_dims,
                                           bev_range, max_num)
        out, counts, status = self.launch(batch, F, max(bound, 1) if cap is None else int(cap), aug)
        if not sync:
            return out, counts, status
        st = int(status.item())
        if st:
            raise ValueError("radar_sweeps_assemble status %d: %s" % (st, ", ".join(
                name for bit, name in ((OVERFLOW, "a sample keeps more than cap rows"), (BAD_ENTRY, "a bad entry"),
                                       (BAD_PARAMS, "bad column ops"),
                                       (BAD_CATEGORY, "a one-hot category outside its encoding")) if st & bit)))
        return [out[k, :n] for k, n in enumerate(counts.tolist())]


def assemble_radar_sweeps(radars_dict, points_of, sweeps_num, use_dim, compensate_velocity=False, normalize=False,
                          normalize_dims=NORMALIZE_DIMS, bev_range=BEV_RANGE, device="cuda", max_num=None):
    """One sample, as LoadRadarPointsMultiSweeps.__call__ + PointsRangeFilter build it: results['radar'] as
    radars_dict and points_of(sweep) -> the raw [n, 18] fp32 rows of that sweep (numpy or torch) ->
    [n, len(use_dim)] fp32 on the device."""
    sweeps, slots = [], {}

    def slot_of(sweep):
        slots[id(sweep)] = len(sweeps)
        sweeps.append(sweep)
        return slots[id(sweep)]

    entries = radar_entries(radars_dict, sweeps_num, slot_of)
    raws = [points_of(s) for s in sweeps]
    cap = max([int(r.shape[0]) for r in raws] + [1])
    store = RadarSweepStore(max(len(raws), 1), cap, device, max_batch=1, max_entries=max(len(entries), 1))
    for s, r in enumerate(raws):
        store.put(s, r)
    return store.assemble([entries], use_dim, compensate_velocity, normalize, normalize_dims, bev_range,
                          max_num=max_num)[0]
