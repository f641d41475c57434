"""GPU: the multi-sweep assembly (SweepStore, bevb200_lidar_sweeps_assemble) against the reference restatement at its
boundaries (tests/data_pipeline_cases.py): remove_close on the raw columns of a sweep row and on the selected columns
of a pad copy, rows transformed exactly onto a range face and one fp32 ulp either side, non-finite coordinates and
lags, signed zeros, out_dim 5..8 with load_dim 3 and 64, caps on the write kernel's tile offsets, device row counts
outside [0, slot_cap], NONE entries between real ones, bad column maps, 64 samples of 64 entries, and quarter turns,
half turns, arbitrary rotations and far translations.

Transformed rows are held to the exact FMA chain (lidar_sweeps_oracle exact=True); a sweep with non-finite
coordinates, which the exact chain cannot take, to numpy's `@`, which equals the chain on every finite pose the CPU
tests draw.  Their coordinates and lag compare NaN positions (CUDA makes the canonical NaN, numpy keeps the
payload); everything else compares bits, NaN payloads and -0.0 included.  Every call runs under
head_boundaries.DeviceGuard."""
import numpy as np
import pytest
import torch

import data_pipeline_cases as C
import lidar_sweeps_oracle as O
from head_boundaries import DeviceGuard

pytestmark = pytest.mark.gpu

USE5 = [0, 1, 2, 3, 4]


def cloud(out, counts):
    return [out[k, :n].cpu().numpy() for k, n in enumerate(counts.tolist())]


class Frame:
    """raw rows by slot, a pose and lag per sweep slot, and a guarded store holding them"""

    def __init__(self, cuda, raws, poses=None, lags=None, max_batch=1, max_entries=11, slot_cap=None):
        from bevfusion_b200 import lidar_sweeps as LS
        self.raws = raws
        rng = np.random.default_rng(len(raws))
        self.poses = poses or [O.nuscenes_pose(rng, k) for k in range(len(raws))]
        self.lags = lags or [0.05 * k + 0.01 for k in range(len(raws))]
        self.guard = DeviceGuard(LS)
        with self.guard:
            self.store = LS.SweepStore(len(raws), slot_cap or max(max(len(r) for r in raws), 1), raws[0].shape[1],
                                       cuda, max_batch=max_batch, max_entries=max_entries)
            for s, r in enumerate(raws):
                self.store.put(s, r)

    def sample(self, key, chosen, lags=None):
        return key, [(s, self.poses[s][0], self.poses[s][1], self.lags[s] if lags is None else lags[i])
                     for i, s in enumerate(chosen)]

    def parts(self, key, chosen, use_dim, lags=None, **kw):
        return C.expected_parts(self.raws[key], [self.raws[s] for s in chosen], [self.poses[s] for s in chosen],
                                [self.lags[s] for s in chosen] if lags is None else lags, use_dim, **kw)

    def assemble(self, samples, use_dim, **kw):
        with self.guard:
            out, counts, status = self.store.assemble(samples, use_dim, sync=False, **kw)
        self.guard.check()
        return out, counts, int(status.item())


def check(frame, cases, use_dim, **kw):
    """assemble the samples of `cases` [(key, chosen, lags or None)] in one call and hold each to its parts"""
    okw = {k: v for k, v in kw.items() if k != "cap"}
    samples = [frame.sample(k, ch, lg) for k, ch, lg in cases]
    out, counts, status = frame.assemble(samples, use_dim, **kw)
    assert status == 0
    for (k, ch, lg), got in zip(cases, cloud(out, counts)):
        parts = frame.parts(k, ch, use_dim, lags=lg, **okw)
        assert C.rows_equal(got, parts), (k, ch, kw)
    return out, counts


@pytest.mark.parametrize("pcr", [None, C.PCR])
def test_remove_close_on_raw_and_selected_columns(cuda, pcr):
    """sweep rows are tested on raw columns 0 and 1, pad copies on the key's selected columns (here 5 and 6): |v|
    exactly 1, one ulp below and above, +-0.0, NaN and +-inf on each"""
    raws = [C.boundary_rows(5, seed=s) for s in range(3)]
    f = Frame(cuda, raws, max_batch=3)
    use = [5, 6, 2, 3, 4]
    check(f, [(0, [1, 2], None), (1, [], None), (2, [0], None)], use, sweeps_num=3, point_cloud_range=pcr)
    check(f, [(0, [1, 2], None), (1, [], None)], use, sweeps_num=2, remove_close=False, point_cloud_range=pcr)


@pytest.mark.parametrize("pose", C.FACE_POSES)
def test_transformed_rows_on_the_range_faces(cuda, pose):
    R, t = C.wide_poses()[pose]
    rows = C.face_rows(R, t, C.PCR)
    rng = np.random.default_rng(len(pose))
    sweep = O.nuscenes_sweep(rng, len(rows) + 40)
    sweep[:len(rows), :3] = np.stack([r for r, _, _ in rows])
    key = np.zeros((len(rows), 5), np.float32)            # the faces untransformed: the key's own comparisons
    lo, hi = np.float32(C.PCR[:3]), np.float32(C.PCR[3:])
    for i, (_, j, where) in enumerate(rows):
        key[i, :3] = (lo + hi) / 2
        face = (lo[j], hi[j])[i % 2]
        key[i, j] = {"on": face, "in": np.nextafter(face, np.float32(0)),
                     "out": np.nextafter(face, np.float32(np.inf) if face > 0 else np.float32(-np.inf))}[where]
        key[i, 3] = i
    f = Frame(cuda, [key, sweep], poses=[(np.eye(3), np.zeros(3)), (R, t)])
    out, counts = check(f, [(0, [1], None)], USE5, point_cloud_range=C.PCR, remove_close=False)
    got = cloud(out, counts)[0]
    want_in = C.face_truth(O.transform_exact(sweep[:len(rows), :3], R, t), C.PCR)
    assert want_in.sum() == sum(w == "in" for _, _, w in rows)
    assert int(counts[0]) == C.face_truth(key[:, :3], C.PCR).sum() + \
        C.face_truth(O.transform_exact(sweep[:, :3], R, t), C.PCR).sum()
    assert got.shape[0] == int(counts[0])


def test_non_finite_rows_lags_and_signed_zeros(cuda):
    """inf / NaN coordinates and NaN payloads in sweep rows, key rows and pad copies; lags that round to +-inf, to
    subnormals and to zero in fp32, and a NaN lag; zero rows (+0.0 and -0.0) under a rotation row of three negative
    entries and a -0.0 translation, which the reference sums to +0.0"""
    rng = np.random.default_rng(8)
    nan = C.NAN_PAYLOADS
    key = O.nuscenes_sweep(rng, 64)
    key[:8, 0] = np.concatenate([nan, np.array([np.inf, -np.inf, -0.0, 0.0], np.float32)])
    key[8:16, 1] = key[:8, 0]
    key[16:24, 3] = key[:8, 0]
    key[:24:3, 2] = -0.0
    odd = O.nuscenes_sweep(rng, 48)
    odd[:8, 0] = key[:8, 0]
    odd[8:16, 2] = key[:8, 0]
    odd[16:24, 3] = key[:8, 0]
    zeros = np.zeros((16, 5), np.float32)
    zeros[8:, :3] = -0.0
    zeros[4:8, 0] = 3.0                                       # outside the remove_close square
    zeros[12:16, 1] = -3.0
    zeros[:, 3] = nan[np.arange(16) % 4]
    R, j = C.all_negative_row_pose()
    poses = [(np.eye(3), np.zeros(3)), O.nuscenes_pose(rng, 1), (R, np.array([-0.0, -0.0, -0.0]))]
    f = Frame(cuda, [key, odd, zeros], poses=poses, max_batch=3, max_entries=len(C.LAGS) + 2)
    lags = list(C.LAGS.values())
    with np.errstate(over="ignore"):
        check(f, [(0, [1] * len(lags), lags), (0, [], None), (1, [2, 1], [0.25, -1e39])], USE5, sweeps_num=4)
        out, counts = check(f, [(2, [2], [0.5])], USE5, remove_close=False)
    got = cloud(out, counts)[0][len(zeros):]
    assert len(got) == len(zeros)
    z = got[(zeros[:, :3] == 0).all(1)]
    assert len(z) and not np.signbit(z[:, j]).any() and (z[:, :3] == 0).all()


@pytest.mark.parametrize("load_dim,use_dim,key_use_dim", [
    (3, [0, 1, 2, 2, 0], None),                              # columns repeated to make five
    (3, [2, 1, 0, 0, 1, 2, 1], None),                        # out_dim 7
    (8, [0, 1, 2, 3, 4, 5, 6, 7], None),                     # out_dim 8
    (9, [1, 0, 2, 8, 4, 6, 3, 7], [8, 1, 0, 2, 4, 5, 3, 6, 7]),
    (C.MAX_LOAD_DIM, [C.MAX_LOAD_DIM - 1, 0, 1, 62, 4, 40, 2, 33], list(range(C.MAX_LOAD_DIM))[::-1]),
])
def test_row_widths(cuda, load_dim, use_dim, key_use_dim):
    rng = np.random.default_rng(load_dim + len(use_dim))
    raws = []
    for n in (1500, 1100, 0, 1300):
        r = O.nuscenes_sweep(rng, n, max(load_dim, 5))[:, :load_dim]
        raws.append(np.ascontiguousarray(r))
    f = Frame(cuda, raws, max_batch=2)
    check(f, [(0, [1, 2, 3], None), (3, [0], None)], use_dim, key_use_dim=key_use_dim, point_cloud_range=C.PCR)
    check(f, [(2, [], None)], use_dim, key_use_dim=key_use_dim, sweeps_num=2)


def _assemble_raw(store, guard, batch, out_dim, cap):
    """bevb200_lidar_sweeps_assemble on the store's block, outputs and the workspace carved by the guard"""
    from bevfusion_b200 import _C
    L = _C.lib()
    dev = store.device
    ws_bytes = L.bevb200_lidar_sweeps_workspace_bytes(batch, store.max_entries, store.slot_cap)
    out = guard.carve(torch.empty((batch, cap, out_dim), dtype=torch.float32, device=dev), fill=False)
    counts = guard.carve(torch.empty((batch,), dtype=torch.int32, device=dev), fill=False)
    status = guard.carve(torch.empty((1,), dtype=torch.int32, device=dev), fill=False)
    ws = guard.carve(torch.empty((ws_bytes,), dtype=torch.uint8, device=dev), fill=False)
    base = store.block.data_ptr()
    _C.check(L.bevb200_lidar_sweeps_assemble(
        _C.ptr(store.rows), store.slots, store.slot_cap, store.load_dim, _C.ptr(store.slot_rows), base, base + 128,
        batch, store.max_entries, out_dim, cap, _C.ptr(out), _C.ptr(counts), _C.ptr(status), _C.ptr(ws), ws_bytes,
        _C.current_stream(dev)), "lidar_sweeps_assemble")
    guard.check("assemble")
    return out, counts, int(status.item())


def _cut(parts, n):
    out = []
    for rows, tr in parts:
        out.append((rows[:max(n, 0)], tr))
        n -= len(rows)
    return out


def test_caps_on_the_tile_offsets(cuda):
    """a key and two sweeps spanning several kTile-row tiles, every row kept, so the tile offsets carry across
    entries; caps at 1, at each tile's offset (the write kernel's early return), one either side, and around the
    total; a second sample whose first sweep remove_close thins to two rows in three, so its tile counts are
    uneven"""
    rng = np.random.default_rng(9)
    raws = []
    for n in C.TILE_ROWS + (C.TILE_ROWS[0],):
        r = O.nuscenes_sweep(rng, n)
        r[:, 0] = np.where(r[:, 0] < 0, r[:, 0] - 2, r[:, 0] + 2)
        raws.append(r)
    thin = raws[3]
    thin[::3, :2] = 0.25                                    # inside the remove_close square
    f = Frame(cuda, raws, max_batch=2)
    samples = [f.sample(0, [1, 2]), f.sample(2, [3, 1])]
    parts = [f.parts(0, [1, 2], USE5), f.parts(2, [3, 1], USE5)]
    assert len(parts[1][1][0]) == len(thin) - len(thin[::3])
    totals = [sum(len(p) for p, _ in ps) for ps in parts]
    caps, _, total = C.tile_caps(C.TILE_ROWS)
    assert totals[0] == total
    for cap in caps:
        with f.guard as g:
            f.store.write_frame(samples, USE5)
            out, counts, status = _assemble_raw(f.store, g, 2, 5, cap)
        assert status == (C.OVERFLOW if max(totals) > cap else 0), cap
        assert counts.tolist() == [min(t, cap) for t in totals], cap
        for k in range(2):
            n = min(totals[k], cap)
            assert C.rows_equal(out[k, :n].cpu().numpy(), _cut(parts[k], n)), (cap, k)


def test_device_row_counts_outside_the_slot(cuda):
    """a negative device row count gives no rows; one above slot_cap is clamped to slot_cap (the slot's rows past
    what put() stored are the store's zeros)"""
    rng = np.random.default_rng(10)
    raws = [O.nuscenes_sweep(rng, n) for n in (900, 700, 500)]
    f = Frame(cuda, raws, slot_cap=1000)
    f.store.slot_rows[1] = -7
    f.store.slot_rows[2] = f.store.slot_cap + 1000
    full = f.store.rows[2].cpu().numpy()
    with f.guard as g:
        f.store.write_frame([f.sample(0, [1, 2])], USE5, point_cloud_range=C.PCR)
        out, counts, status = _assemble_raw(f.store, g, 1, 5, 4000)
    assert status == 0
    f.raws[1] = raws[1][:0]
    f.raws[2] = full
    assert C.rows_equal(cloud(out, counts)[0], f.parts(0, [1, 2], USE5, point_cloud_range=C.PCR))


def test_none_entries_between_real_ones(cuda):
    from bevfusion_b200.lidar_sweeps import ENTRY_DTYPE
    rng = np.random.default_rng(11)
    raws = [O.nuscenes_sweep(rng, n) for n in (800, 600, 700, 500)]
    f = Frame(cuda, raws, max_batch=2, max_entries=7)
    f.store.write_frame([f.sample(0, [1]), f.sample(1, [2])], USE5, point_cloud_range=C.PCR)
    e = np.zeros((2, 7), ENTRY_DTYPE)
    layout = [[(C.SWEEP_KEY, 0), (C.SWEEP_NONE, 3), (C.SWEEP_SWEEP, 1), (C.SWEEP_NONE, 0), (C.SWEEP_SWEEP, 3)],
              [(C.SWEEP_NONE, 2), (C.SWEEP_KEY, 1), (C.SWEEP_SWEEP, 2), (C.SWEEP_NONE, 1), (C.SWEEP_NONE, 1),
               (C.SWEEP_SWEEP, 0), (C.SWEEP_NONE, 0)]]
    for b, ents in enumerate(layout):
        for i, (kind, slot) in enumerate(ents):
            R, t = f.poses[slot]
            e[b, i] = (kind, slot, R.reshape(9), t, f.lags[slot])
    f.store.block[128:128 + e.nbytes] = torch.from_numpy(np.frombuffer(e.tobytes(), np.uint8).copy()).to(cuda)
    with f.guard as g:
        out, counts, status = _assemble_raw(f.store, g, 2, 5, 5000)
    assert status == 0
    got = cloud(out, counts)
    assert C.rows_equal(got[0], f.parts(0, [1, 3], USE5, point_cloud_range=C.PCR))
    assert C.rows_equal(got[1], f.parts(1, [2, 0], USE5, point_cloud_range=C.PCR))


def test_bad_column_maps(cuda):
    """a key or sweep column outside [0, load_dim) sets BAD_PARAMS and no sample gets rows; a column past out_dim is
    never read"""
    from bevfusion_b200.lidar_sweeps import PARAMS_DTYPE
    rng = np.random.default_rng(12)
    raws = [O.nuscenes_sweep(rng, n) for n in (800, 600)]
    f = Frame(cuda, raws, max_batch=2)
    samples = [f.sample(0, [1]), f.sample(1, [0])]
    off = {k: PARAMS_DTYPE.fields[k][1] for k in ("key_cols", "sweep_cols")}
    for field, col, value, bad in [("key_cols", 0, 5, True), ("sweep_cols", 1, -1, True),
                                   ("key_cols", 4, 1 << 20, True), ("sweep_cols", 5, 99, False),
                                   ("key_cols", 7, -3, False)]:
        f.store.write_frame(samples, USE5)
        at = off[field] + 4 * col
        f.store.block[at:at + 4] = torch.tensor([value], dtype=torch.int32).view(torch.uint8).to(cuda)
        with f.guard as g:
            out, counts, status = _assemble_raw(f.store, g, 2, 5, 3000)
        if bad:
            assert status == C.BAD_PARAMS and counts.tolist() == [0, 0], (field, col)
        else:
            assert status == 0
            got = cloud(out, counts)
            assert C.rows_equal(got[0], f.parts(0, [1], USE5)) and C.rows_equal(got[1], f.parts(1, [0], USE5))


def test_64_samples_of_64_entries(cuda):
    rng = np.random.default_rng(13)
    S, B, E = 16, 64, 64
    raws = [O.nuscenes_sweep(rng, int(rng.integers(0, 300))) for _ in range(S)]
    f = Frame(cuda, raws, max_batch=B, max_entries=E, slot_cap=300)
    chosen = [[int(s) for s in rng.integers(0, S, E - 1)] for _ in range(B)]
    sweep_parts = C.expected_parts(raws[0], raws, f.poses, f.lags, USE5, point_cloud_range=C.PCR)[1:]
    key_parts = [C.expected_parts(raws[s], [], [], [], USE5, sweeps_num=0, point_cloud_range=C.PCR)[0]
                 for s in range(S)]
    out, counts, status = f.assemble([f.sample(b % S, chosen[b]) for b in range(B)], USE5, point_cloud_range=C.PCR)
    assert status == 0
    for b, got in enumerate(cloud(out, counts)):
        assert C.rows_equal(got, [key_parts[b % S]] + [sweep_parts[s] for s in chosen[b]]), b


def test_wide_poses_follow_the_fma_chain(cuda):
    """quarter and half turns about each axis, arbitrary rotations and translations up to 10 km: the kernel equals
    the exact FMA chain on every row (numpy's `@` equals it too: no pinned double-rounding case)"""
    poses = C.wide_poses()
    names = sorted(poses)
    raws = [np.zeros((0, 5), np.float32)]
    for k, name in enumerate(names):
        r = np.zeros((1500, 5), np.float32)
        r[:, :3] = C.wide_points(k)
        r[:, 3] = k
        raws.append(r)
    f = Frame(cuda, raws, poses=[(np.eye(3), np.zeros(3))] + [poses[n] for n in names],
              max_entries=len(names) + 1)
    # held to the chain on every row, so at a pinned case (C.DOUBLE_ROUNDING) too, where numpy's `@` differs
    check(f, [(0, list(range(1, len(raws))), None)], USE5, remove_close=False)
