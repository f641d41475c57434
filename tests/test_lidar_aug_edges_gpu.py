"""GPU: the augmentation kernels at their edges, against the exact form of tests/lidar_aug_oracle.py, with no
tolerance (NaN equal to NaN, signed zeros distinct).

- Rows transformed exactly onto each range face and one ulp either side of it (found by scanning inputs through
  the oracle), with the oracle's torch form agreeing on every one of them; boxes centred on those inputs.
- Box yaws at +-pi, at limit_yaw's wrap and around them; signed zeros, NaN and +-inf coordinates in rows and boxes.
- Radar rows whose augmented x or y is exactly on a face of the radar range (+-55) or one ulp off it, with columns
  3 and 4 carried through the rotation and flips; caps that truncate augmented radar tiles.
- Caps and overflow with the augmentation on; B = max_batch; box counts at the box kernel's block size +-1 and at
  BEVB200_HEAD_TARGETS_MAX_BOXES; counts outside [0, nmax] (BAD_COUNT); 7- and 9-column boxes.
Boundaries are read from the kernel sources' constants."""
import os
import re

import numpy as np
import pytest
import torch

import lidar_aug_oracle as O

pytestmark = pytest.mark.gpu

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "bevfusion_b200", "csrc")


def const(fname, name):
    with open(os.path.join(CSRC, fname)) as f:
        return int(re.search(r"constexpr int %s = (\d+);" % name, f.read()).group(1))


BOX_BLOCK = const("box_aug.cu", "kThreads")
SWEEP_TILE = const("lidar_sweeps.cu", "kThreads") * const("lidar_sweeps.cu", "kRounds")
DRAWS = [(1.0734, 0.61, np.array([0.31, -0.27, 0.12]), 1, 0), (0.9123, -0.7712, np.array([-0.4, 0.05, -0.2]), 0, 1),
         (1.05, 0.0, np.array([0.0, 0.0, 0.0]), 1, 1)]


def same(a, b):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return O.count_diff(a, b) == 0


def block(cuda, draws, max_batch=None):
    from bevfusion_b200.lidar_aug import LidarAug, LidarAugDraw
    aug = LidarAug(max_batch or len(draws), cuda)
    aug.write([LidarAugDraw(*d) for d in draws])
    return aug


def face_rows(draw, seed=0):
    """[k, 5] LiDAR rows whose augmented x, y or z is exactly on a face of POINT_CLOUD_RANGE or one ulp off it"""
    rng = np.random.default_rng(seed)
    r = np.asarray(O.POINT_CLOUD_RANGE, np.float32)
    scale, theta, trans, fh, fv = draw
    R = O.rot_mats(theta)[0].astype(np.float64)
    rows = []
    for axis in range(3):
        for face in (r[axis], r[axis + 3]):
            targets = [face, np.nextafter(face, np.float32(np.inf)), np.nextafter(face, np.float32(-np.inf))]
            want = np.zeros(3)
            want[axis] = face if not ((axis == 1 and fh) or (axis == 0 and fv)) else -face
            for j in range(3):
                if j != axis:
                    want[j] = rng.uniform(-0.5, 0.5) * (r[j + 3] - r[j])
            p0 = (want / scale - trans) @ np.linalg.inv(R)       # the real preimage
            k = int(np.abs(R[:, axis]).argmax())                  # the input that moves this output most
            cand = np.tile(p0.astype(np.float32), (8193, 1))
            cand[:, k] = p0[k].astype(np.float32) + np.arange(-4096, 4097) * np.spacing(np.float32(p0[k]))
            pts = np.zeros((len(cand), 5), np.float32)
            pts[:, :3] = cand
            out = O.augment_points(pts, draw, exact=True)
            for t in targets:
                hit = np.nonzero(out[:, axis] == t)[0]
                if len(hit):
                    rows.append(pts[hit[0]])
    return np.array(rows, np.float32)


@pytest.mark.parametrize("d", range(len(DRAWS)))
def test_rows_on_the_range_faces(cuda, d):
    from bevfusion_b200.lidar_sweeps import SweepStore
    draw = DRAWS[d]
    rows = face_rows(draw, d)
    assert len(rows) >= 12      # most faces hit exactly and on both sides
    special = np.array([[0.0, -0.0, -0.0, 1, 0], [-0.0, -0.0, 0.0, 2, 0], [np.nan, 1.0, 0.0, 3, 0],
                        [np.inf, 0.0, 0.0, 4, 0], [-np.inf, 1.0, 1.0, 5, 0], [1.0, np.inf, -np.inf, 6, 0],
                        [1e-40, -1e-40, 0.5, 7, 0], [3e38, 1.0, 0.0, 8, 0]], np.float32)
    rows = np.concatenate([rows, special])
    want = O.augment_points(rows, draw, exact=True)
    assert O.count_diff(want, O.augment_points(rows, draw)) == 0
    aug = block(cuda, [draw])
    store = SweepStore(1, len(rows), 5, cuda, max_batch=1, max_entries=1)
    store.put(0, rows)
    for rng in (O.POINT_CLOUD_RANGE, None):
        got = store.assemble([(0, [])], 5, pad_empty_sweeps=False, point_cloud_range=rng, aug=aug)[0]
        assert same(got, want if rng is None else want[O.in_range_3d(want, rng)])


def test_caps_overflow_and_full_batch(cuda):
    from bevfusion_b200.lidar_sweeps import OVERFLOW, SweepStore
    rng = np.random.default_rng(3)
    B = 4
    clouds = []
    for b in range(B):
        n = [SWEEP_TILE - 1, SWEEP_TILE, SWEEP_TILE + 1, 3 * SWEEP_TILE + 5][b]
        p = np.zeros((n, 5), np.float32)
        p[:, :3] = rng.uniform(-60, 60, (n, 3)) * [1, 1, 0.1]
        clouds.append(p)
    draws = [DRAWS[b % len(DRAWS)] for b in range(B)]
    aug = block(cuda, draws, max_batch=B)
    store = SweepStore(B, max(len(c) for c in clouds), 5, cuda, max_batch=B, max_entries=1)
    for b, c in enumerate(clouds):
        store.put(b, c)
    want = []
    for c, d in zip(clouds, draws):
        w = O.augment_points(c, d, exact=True)
        want.append(w[O.in_range_3d(w, O.POINT_CLOUD_RANGE)])
    kept = [len(w) for w in want]
    for cap in (min(kept) - 1, SWEEP_TILE // 2, max(kept), max(kept) + 1):
        out, counts, status = store.assemble([(b, []) for b in range(B)], 5, pad_empty_sweeps=False,
                                             point_cloud_range=O.POINT_CLOUD_RANGE, cap=cap, sync=False, aug=aug)
        assert counts.tolist() == [min(k, cap) for k in kept]
        assert int(status[0]) == (OVERFLOW if max(kept) > cap else 0)
        for b in range(B):
            assert same(out[b, :min(kept[b], cap)], want[b][:cap])


RADAR_TILE = const("radar_sweeps.cu", "kThreads")
RADAR_USE_DIM = [0, 1, 2, 5, 8]    # x, y, z, rcs, vx_comp: under an identity pose the raw values, as fp32


def radar_store(cuda, raws):
    from bevfusion_b200.radar_sweeps import RadarSweepStore
    store = RadarSweepStore(len(raws), max(len(r) for r in raws), cuda, max_batch=len(raws), max_entries=1)
    for k, r in enumerate(raws):
        store.put(k, r)
    return store, [[(k, np.eye(3), np.zeros(3), 0.0)] for k in range(len(raws))]


def radar_face_rows(draw, seed):
    """raw [k, 18] radar rows whose augmented output x or y (use_dim RADAR_USE_DIM, identity pose) is exactly on a
    face of the radar range or one ulp off it"""
    import radar_sweeps_oracle as RO
    rng = np.random.default_rng(seed)
    r = np.asarray(O.RADAR_BEV_RANGE, np.float32)
    scale, theta, trans, fh, fv = draw
    R = O.rot_mats(theta)[0].astype(np.float64)
    rows = []
    for axis in range(2):
        for face in (r[axis], r[axis + 2]):
            targets = [face, np.nextafter(face, np.float32(np.inf)), np.nextafter(face, np.float32(-np.inf))]
            want = np.array([rng.uniform(-40, 40), rng.uniform(-40, 40), rng.uniform(-1, 2)])
            want[axis] = face if not ((axis == 1 and fh) or (axis == 0 and fv)) else -face
            p0 = (want / scale - trans) @ np.linalg.inv(R)
            k = int(np.abs(R[:2, axis]).argmax())
            cand = RO.radar_sweep(rng, 8193)
            cand[:, :3] = p0.astype(np.float32)
            cand[:, k] = p0[k].astype(np.float32) + np.arange(-4096, 4097) * np.spacing(np.float32(p0[k]))
            out = O.augment_radar(cand[:, RADAR_USE_DIM], draw, exact=True)
            for t in targets:
                hit = np.nonzero(out[:, axis] == t)[0]
                if len(hit):
                    rows.append(cand[hit[0]])
    return np.array(rows, np.float32)


@pytest.mark.parametrize("d", range(len(DRAWS)))
def test_radar_rows_on_the_range_faces(cuda, d):
    import radar_sweeps_oracle as RO
    draw = DRAWS[d]
    rows = radar_face_rows(draw, d)
    assert len(rows) >= 8      # most faces hit exactly and on both sides
    special = RO.radar_sweep(np.random.default_rng(d), 6)
    special[:, [0, 1, 2, 5, 8]] = [[0.0, -0.0, -0.0, -0.0, 0.0], [np.nan, 1, 0, 2, 3], [np.inf, 0, 0, 1, -1],
                                   [1, -np.inf, 0, np.inf, 0], [1, 2, 3, np.nan, -np.inf], [1e-40, -1e-40, 0, 1e-40, 3e38]]
    rows = np.concatenate([rows, special])
    store, samples = radar_store(cuda, [rows])
    plain = store.assemble(samples, RADAR_USE_DIM, bev_range=None)[0].cpu().numpy()
    want = O.augment_radar(plain, draw, exact=True)
    assert O.count_diff(want, O.augment_radar(plain, draw)) == 0
    on_face = np.isin(np.abs(want[:len(rows) - 6, :2]), np.float32(55.0)).any(1).sum()
    assert on_face >= 3
    got = store.assemble(samples, RADAR_USE_DIM, aug=block(cuda, [draw]))[0]
    assert same(got, want[O.in_range_bev(want[:, :2], O.RADAR_BEV_RANGE)])


def test_radar_caps_truncate_augmented_tiles(cuda):
    import radar_sweeps_oracle as RO
    from bevfusion_b200.radar_sweeps import OVERFLOW
    rng = np.random.default_rng(5)
    B = 3
    raws = []
    for b in range(B):
        r = RO.radar_sweep(rng, [RADAR_TILE - 1, 2 * RADAR_TILE + 1, 4 * RADAR_TILE + 7][b])
        r[:, :2] = rng.uniform(-70, 70, (len(r), 2))
        raws.append(r)
    store, samples = radar_store(cuda, raws)
    draws = [DRAWS[b % len(DRAWS)] for b in range(B)]
    aug = block(cuda, draws)
    use_dim = RO.SHIPPED_USE_DIM
    plain = store.assemble(samples, use_dim, bev_range=None)
    want = []
    for p, d in zip(plain, draws):
        w = O.augment_radar(p.cpu().numpy(), d, exact=True)
        want.append(w[O.in_range_bev(w[:, :2], O.RADAR_BEV_RANGE)])
    kept = [len(w) for w in want]
    for cap in (min(kept) - 1, RADAR_TILE - 1, RADAR_TILE + 1, max(kept) - 1, max(kept)):
        out, counts, status = store.assemble(samples, use_dim, cap=cap, sync=False, aug=aug)
        assert counts.tolist() == [min(k, cap) for k in kept]
        assert int(status[0]) == (OVERFLOW if max(kept) > cap else 0)
        for b in range(B):
            assert same(out[b, :min(kept[b], cap)], want[b][:cap])


def boxes_case(rng, n, D):
    b = np.zeros((n, D), np.float32)
    b[:, :2] = rng.uniform(-60, 60, (n, 2))
    b[:, 2] = rng.uniform(-3, 1, n)
    b[:, 3:6] = rng.uniform(0.3, 12, (n, 3))
    b[:, 6] = rng.uniform(-4, 4, n)
    if D == 9:
        b[:, 7:9] = rng.normal(0, 5, (n, 2))
    return b, rng.integers(-1, 11, n).astype(np.int32)


def yaw_edges(draw):
    """yaws that the draw takes to +-fl32(pi), to limit_yaw's wrap points and next to them"""
    _, _, yaw = O.rot_mats(draw[1])
    pi = O.PI32
    out = []
    for v in (pi, -pi, 3 * pi, -3 * pi, np.float32(0.0)):
        for k in range(-2, 3):
            t = np.float32(v)
            for _ in range(abs(k)):
                t = np.nextafter(t, np.float32(np.inf) if k > 0 else np.float32(-np.inf))
            out += [t, np.float32(t - yaw), np.float32(-t + pi - yaw)]
    return np.array(out, np.float32)


@pytest.mark.parametrize("D", [7, 9])
def test_boxes_at_the_edges(cuda, D):
    from bevfusion_b200.lidar_aug import BAD_COUNT, MAX_BOXES
    rng = np.random.default_rng(D)
    B = len(DRAWS) + 1
    draws = DRAWS + [(None, None, None, 1, 1)]
    sizes = [BOX_BLOCK - 1, BOX_BLOCK, BOX_BLOCK + 1, MAX_BOXES]
    nmax = MAX_BOXES
    pb = np.zeros((B, nmax, D), np.float32)
    pl = np.zeros((B, nmax), np.int32)
    cases = []
    for b in range(B):
        boxes, labels = boxes_case(rng, sizes[b], D)
        ye = yaw_edges(draws[b] if draws[b][0] is not None else DRAWS[0])
        boxes[:len(ye), 6] = ye
        boxes[len(ye):len(ye) + 6, :3] = [[0.0, -0.0, -0.0], [np.nan, 1, 1], [np.inf, 0, 0], [1, -np.inf, 0],
                                          [-0.0, -0.0, np.nan], [1e-40, 3e38, 0]]
        labels[len(ye):len(ye) + 6] = 0
        faces = face_rows(draws[b] if draws[b][0] is not None else DRAWS[2], b)[:, :3]
        boxes[-len(faces):, :3] = faces
        pb[b, :len(boxes)], pl[b, :len(boxes)] = boxes, labels
        cases.append((boxes, labels))
    aug = block(cuda, draws)
    tb, tl = torch.from_numpy(pb).to(cuda), torch.from_numpy(pl).to(cuda)
    tc = torch.tensor(sizes[:B], dtype=torch.int32, device=cuda)
    ob, ol, oc, st = aug.boxes(tb, tl, tc, O.POINT_CLOUD_RANGE, O.OBJECT_CLASSES)
    assert int(st[0]) == 0
    for b, (boxes, labels) in enumerate(cases):
        wb, wl = O.boxes_filtered(boxes, labels, draws[b], exact=True)
        tb_, tl_ = O.boxes_filtered(boxes, labels, draws[b])
        assert O.count_diff(wb, tb_) == 0
        n = int(oc[b])
        assert n == len(wb) and same(ob[b, :n], wb) and np.array_equal(ol[b, :n].cpu().numpy(), wl)
        assert not ob[b, n:].any() and not ol[b, n:].any()
    # counts outside [0, nmax] are read as clamped and flagged
    bad = torch.tensor([-1, nmax + 1, 0, 5], dtype=torch.int32, device=cuda)
    ob, ol, oc, st = aug.boxes(tb, tl, bad, O.POINT_CLOUD_RANGE, 10)
    assert int(st[0]) == BAD_COUNT and int(oc[0]) == 0 and int(oc[2]) == 0
    full = O.boxes_filtered(pb[1], pl[1], draws[1], exact=True)[0]
    assert int(oc[1]) == len(full)
