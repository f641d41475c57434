"""Boundary cases of the data-pipeline kernels, image_aug.cu (ImageAug3D + ImageNormalize) and lidar_sweeps.cu
(LoadPointsFromMultiSweeps + PointsRangeFilter), shared by test_image_aug_edges_{cpu,gpu}.py and
test_lidar_sweeps_edges_{cpu,gpu}.py.  numpy only: no device.

Every boundary is read from the constant that sets it (head_boundaries.cu_const / header_macro), so a retune of a
block, a tile or a limit moves the cases with it:

    HPASS_COLS, HPASS_ROWS  kHpassCols x kHpassRows: crop columns x band rows per CTA of the horizontal pass
    VPASS_COLS              kVpassCols: output columns per CTA of the vertical pass
    MAX_FRAME, MAX_SOURCE   kMaxFrame (output sides), kMaxSource (input and resized sides are below it)
    MAX_GRID                kMaxGridY: CUDA's grid.y / grid.z limit (horizontal-pass row blocks, cameras)
    CROP_LIMIT              the |crop_x|, |crop_y| bound of the setup kernel's draw check
    SWEEP_TILE              kTile: rows per CTA of the sweep count and write kernels
    MAX_LOAD_DIM, MAX_DIM   kMaxLoadDim, BEVB200_SWEEP_MAX_DIM

Camera cases are calls: dict(H, W, fH, fW, min_resize, draws, expect), one draw per camera (resize, (w, h), (x0, y0),
flip, rotate) and its expected status (0, OVER_CAPACITY or BAD_DRAW).  Sweep cases are (raw rows, poses, lags)
with the expected cloud split into parts (expected_parts), so a check knows which rows went through the transform."""
import math
import re

import numpy as np

import lidar_sweeps_oracle as LO
from head_boundaries import CSRC, cu_const, header_macro

# ---- camera augmentation ------------------------------------------------------------------------------------------
HPASS_COLS = cu_const("image_aug.cu", "kHpassCols")
HPASS_ROWS = cu_const("image_aug.cu", "kHpassRows")
VPASS_COLS = cu_const("image_aug.cu", "kVpassCols")
MAX_FRAME = cu_const("image_aug.cu", "kMaxFrame")
MAX_SOURCE = cu_const("image_aug.cu", "kMaxSource")
MAX_GRID = cu_const("image_aug.cu", "kMaxGridY")
BAD_DRAW = header_macro("BEVB200_IMAGE_AUG_BAD_DRAW")
OVER_CAPACITY = header_macro("BEVB200_IMAGE_AUG_OVER_CAPACITY")
EINVAL = header_macro("BEVB200_EINVAL")


def _crop_limit():
    with open("%s/image_aug.cu" % CSRC) as f:
        m = re.search(r"is_int_in\(cxd, -(\d+)\.0, (\d+)\.0\)", f.read())
    assert m and m.group(1) == m.group(2), "the crop bound of image_aug_setup_kernel"
    return int(m.group(1))


CROP_LIMIT = _crop_limit()


def ksize(in_size, out_size):
    """Pillow's BICUBIC taps for in_size -> out_size (filter_geom / ksize_for: the float box, support 2 scaled)"""
    scale = float(np.float32(in_size)) / out_size
    return int(math.ceil(2.0 * max(scale, 1.0))) * 2 + 1


def cap_sizes(in_size, min_resize):
    """(smallest out size whose filter still has ksize == kcap, the table width min_resize sets; the next smaller
    one, the first whose filter is over capacity)"""
    kcap = ksize(in_size, min_resize)
    w = min_resize
    while w > 1 and ksize(in_size, w - 1) <= kcap:
        w -= 1
    return w, w - 1


def bounds(in_size, out_size, xx):
    """(xmin, count) of Pillow's precompute_coeffs for output index xx, without the weights"""
    scale = float(in_size) / out_size
    support = 2.0 * max(scale, 1.0)
    center = (xx + 0.5) * scale
    xmin = max(int(center - support + 0.5), 0)
    return xmin, min(int(center + support + 0.5), in_size) - xmin


def band_rows(H, h, y0, fH):
    """source rows the vertical pass reads for crop rows [y0, y0 + fH) of an H -> h resize (the setup kernel's band)"""
    rows = [bounds(H, h, y) for y in range(max(y0, 0), min(y0 + fH, h))]
    if not rows:
        return 0
    return max(a + n for a, n in rows) - min(a for a, _ in rows)


def _call(H, W, fH, fW, draws, min_resize=None, expect=None):
    min_resize = min_resize or (min(d[1][0] for d in draws), min(d[1][1] for d in draws))
    return dict(H=H, W=W, fH=fH, fW=fW, min_resize=min_resize, draws=draws, expect=expect or [0] * len(draws))


def _draw(W, dims, xy, flip=False, rotate=0.0):
    return (dims[0] / W, tuple(dims), tuple(xy), flip, rotate)


def frame_width_edges():
    """fW on the edges of kHpassCols and kVpassCols: k * cols - 1, k * cols, k * cols + 1 for k = 1, 2, and 1"""
    return sorted({1} | {k * c + d for c in (HPASS_COLS, VPASS_COLS) for k in (1, 2) for d in (-1, 0, 1)})


def band_row_edges():
    """band rows on the edges of kHpassRows: k * rows - 1, k * rows, k * rows + 1 for k = 1, 2, 3, and 1"""
    return sorted({1} | {k * HPASS_ROWS + d for k in (1, 2, 3) for d in (-1, 0, 1)})


# the band cases: (name, H -> h) -- an upscale cropped at the top edge, a downscale cropped inside the image
BAND_KINDS = (("top", ((1, 3), (61, 90)), (0,)), ("inside", ((200, 97),), tuple(range(5, 40))))


def band_cases(target):
    """{kind: (H, h, y0, fH)} whose crop rows make a band of exactly `target` source rows, for each of BAND_KINDS that
    reaches it (a downscale reads at least a few rows per output row: it has no one-row band)"""
    out = {}
    for kind, sizes, y0s in BAND_KINDS:
        found = [(H, h, y0, fH) for H, h in sizes for y0 in y0s for fH in range(1, 2 * target + 8)
                 if band_rows(H, h, y0, fH) == target]
        if found:
            out[kind] = found[0]
    return out


def image_calls():
    """name -> call; every camera case of the kernel's tiling, capacity and limit boundaries"""
    calls = {}
    for fW in frame_width_edges():
        w = 3 * fW // 2 + 7
        calls["fW=%d" % fW] = _call(61, 99, 5, fW, [_draw(99, (w, 80), (-3, 2)),
                                                    _draw(99, (w, 80), (w - fW + 2, 70), True, 2.0)])
    for n in band_row_edges():
        for kind, (H, h, y0, fH) in band_cases(n).items():
            calls["band=%d/%s" % (n, kind)] = _call(H, 23, fH, 17, [_draw(23, (30, h), (-2, y0)),
                                                                   _draw(23, (30, h), (1, y0), True, -3.0)])
    calls["frame=1x1"] = _call(3, 4, 1, 1, [_draw(4, (4, 3), (1, 1)), _draw(4, (9, 7), (4, 3), True, 90.0),
                                            _draw(4, (2, 2), (1, 0), False, 180.0),
                                            _draw(4, (5, 5), (2, 2), True, 33.3),
                                            _draw(4, (1, 1), (0, 0), False, -1e-20)])
    # tap capacity: the table is ksize(in, min_resize) taps wide
    (we, wo), (he, ho) = cap_sizes(1600, 608), cap_sizes(900, 342)
    calls["kcap"] = _call(900, 1600, 32, 64, [
        _draw(1600, (608, 342), (100, 50)),                       # ksize == kcap at min_resize
        _draw(1600, (we, 342), (we - 40, 300), True, 1.5),         # the smallest width with ksize == kcap
        _draw(1600, (wo, 342), (0, 0)),                            # one below: over capacity
        _draw(1600, (608, he), (7, he - 20), False, -2.0),         # the smallest height with ksize == kcap
        _draw(1600, (608, ho), (0, 0)),                            # one below: over capacity
        _draw(1600, (4000, 2250), (1900, 1000), True, 4.0)],      # far above: most of each table row unused
        min_resize=(608, 342), expect=[0, 0, OVER_CAPACITY, 0, OVER_CAPACITY, 0])
    # extreme resamples: 1600 x 900 -> 1 x 1 (6401 x 3601 taps), one axis to 1, and a 5 x 7 image blown up
    calls["to-1x1"] = _call(900, 1600, 4, 5, [_draw(1600, (1, 1), (0, 0)), _draw(1600, (1, 1), (-2, -1), True, 3.0),
                                              _draw(1600, (1, 900), (-1, 400)), _draw(1600, (1600, 1), (700, -3))],
                            min_resize=(1, 1))
    calls["upscale"] = _call(5, 7, 64, 96, [_draw(7, (5000, 3000), (2400, 1400)),
                                            _draw(7, (7000, 4000), (0, 3950), True, -4.5)], min_resize=(7, 5))
    # frame sides at kMaxFrame through every rotate path (90 / 270 of a non-square frame take the affine one)
    rots = [33.3, -1e-20, 90.0, 270.0, 180.0]
    calls["fW=max"] = _call(40, 2000, 16, MAX_FRAME, [_draw(2000, (MAX_FRAME + 116, 60), (50, 10), i % 2 == 1, r)
                                                      for i, r in enumerate(rots)])
    calls["fH=max"] = _call(2000, 40, MAX_FRAME, 16, [_draw(40, (60, MAX_FRAME + 116), (10, 50), i % 2 == 1, r)
                                                      for i, r in enumerate(rots)])
    # crop offsets at the +-CROP_LIMIT bounds (the crop lies outside the resized image: all fill) and one past them
    L = CROP_LIMIT
    crops = [(L, 0), (-L, 3), (0, L), (2, -L), (-L, -L), (L, L), (L + 1, 0), (0, -L - 1)]
    calls["crop=limit"] = _call(90, 160, 20, 30, [_draw(160, (120, 70), xy, i % 2 == 1, 7.0 * i)
                                                  for i, xy in enumerate(crops)],
                                expect=[0] * 6 + [BAD_DRAW] * 2)
    # the tallest input: ceil(H / kHpassRows) > MAX_GRID row blocks.  Resized to kMaxFrame rows and cropped whole,
    # every source row is in the band, and the last output rows weigh the rows past MAX_GRID * kHpassRows heavily
    H = MAX_SOURCE - 1
    calls["tall"] = _call(H, 1, MAX_FRAME, 1, [_draw(1, (1, MAX_FRAME), (0, 0))])
    return calls


# the calls the CPU file holds against Pillow (the shapes nothing else checks there)
PILLOW_CALLS = ("tall", "fW=max", "fH=max", "to-1x1", "upscale", "crop=limit", "frame=1x1")


def camera_image(seed, H, W):
    """noise over smooth gradients, uint8 [H, W, 3]: hits the clips to 0 / 255 as well as mid-range values"""
    rng = np.random.RandomState(seed % (1 << 31))
    y, x = np.mgrid[0:H, 0:W]
    base = np.stack([x * 255 // max(W, 1), y * 255 // max(H, 1), (x + y) % 256], -1).astype(np.int16)
    return np.clip(base + rng.randint(-90, 91, (H, W, 3)).astype(np.int16), 0, 255).astype(np.uint8)


def tall_tail_matters(call, img):
    """whether the tall case's expected output changes when the source rows past MAX_GRID * kHpassRows (the rows only
    a second pass over the row blocks resamples) are inverted"""
    import image_aug_oracle as IO
    (_, dims, xy, flip, rot), = call["draws"]
    frame = (call["fH"], call["fW"])
    other = img.copy()
    other[MAX_GRID * HPASS_ROWS:] = 255 - other[MAX_GRID * HPASS_ROWS:]
    a = IO.augment_u8(img, dims, xy, frame, flip, rot)
    b = IO.augment_u8(other, dims, xy, frame, flip, rot)
    return int((a != b).any(axis=-1).sum())


def call_images(name, call):
    return np.stack([camera_image(len(name) * 1000 + i, call["H"], call["W"]) for i in range(len(call["draws"]))])


def pack(draws):
    return np.array([[float(r), float(d[0]), float(d[1]), float(xy[0]), float(xy[1]), 1.0 if f else 0.0, float(a)]
                     for r, d, xy, f, a in draws], np.float64)


# many cameras: tiny images and draws repeating with coprime periods
CAM_IMAGES, CAM_DRAWS = 7, 16


def many_camera_draws():
    """CAM_DRAWS draws of a 3 x 3 image into a 2 x 2 frame: every rotate path, flips, crops past each side"""
    rots = (0.0, 90.0, 180.0, 270.0, 33.3, -1e-20, -7.5, 200.0)
    return [_draw(3, (1 + k % 6, 1 + (k * 5) % 6), (k % 5 - 1, (k * 3) % 5 - 1), k % 3 == 0, rots[k % len(rots)])
            for k in range(CAM_DRAWS)]


# ---- multi-sweep assembly -------------------------------------------------------------------------------------------
SWEEP_TILE = cu_const("lidar_sweeps.cu", "kTile")
MAX_LOAD_DIM = cu_const("lidar_sweeps.cu", "kMaxLoadDim")
MAX_DIM = header_macro("BEVB200_SWEEP_MAX_DIM")
SWEEP_NONE, SWEEP_KEY, SWEEP_SWEEP, SWEEP_PAD = (header_macro("BEVB200_SWEEP_" + k)
                                                 for k in ("NONE", "KEY", "SWEEP", "PAD"))
OVERFLOW = header_macro("BEVB200_SWEEPS_OVERFLOW")
BAD_ENTRY = header_macro("BEVB200_SWEEPS_BAD_ENTRY")
BAD_PARAMS = header_macro("BEVB200_SWEEPS_BAD_PARAMS")
PCR = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]        # 51.2 is not a float32: the faces are fl32(51.2)

F32 = np.float32
ONE_BELOW = np.nextafter(F32(1), F32(0))
ONE_ABOVE = np.nextafter(F32(1), F32(2))
NAN_PAYLOADS = np.array([0x7fc00000, 0x7fa00001, 0xffc12345, 0x7f800001], np.uint32).view(np.float32)


def rotation(yaw, pitch=0.0, roll=0.0):
    cz, sz, cy, sy, cx, sx = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch), np.cos(roll), np.sin(roll)
    return np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) \
        @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])


def random_rotation(rng):
    """a uniformly random rotation (unit quaternion)"""
    q = rng.standard_normal(4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def wide_poses():
    """name -> (R, t): quarter and half turns about each axis, arbitrary rotations, and translations up to 10 km"""
    rng = np.random.default_rng(2027)
    poses = {}
    for deg in (90, 180, 270, -90):
        a = np.deg2rad(deg)
        poses["yaw%d" % deg] = (rotation(a), np.array([0.5 * deg / 90, -1.25, 0.125]))
        poses["pitch%d" % deg] = (rotation(0.0, a), np.array([3.0, 0.0, -2.0]))
        poses["roll%d" % deg] = (rotation(0.0, 0.0, a), np.array([-7.0, 1.0, 0.0]))
    for k in range(6):
        poses["random%d" % k] = (random_rotation(rng), rng.uniform(-30, 30, 3))
    for k, s in enumerate((1e3, 1e4)):
        poses["far%d" % k] = (random_rotation(rng), rng.uniform(-s, s, 3))
        poses["far-yaw180-%d" % k] = (rotation(np.pi), np.array([s, -s, 0.5]))
    return poses


def wide_points(seed, n=1500):
    """fp32 xyz for the wide poses: a 70 m spin, large coordinates and small ones"""
    rng = np.random.default_rng(seed)
    pts = LO.nuscenes_sweep(rng, n)[:, :3]
    pts[: n // 4] *= F32(100)
    pts[n // 4: n // 2] *= F32(1e-3)
    return np.ascontiguousarray(pts)


def double_rounding_cases():
    """[(pose name, row, column)] where numpy's `@` and the exact FMA chain disagree after the fp32 store, over
    wide_poses() x wide_points()"""
    out = []
    for k, (name, (R, t)) in enumerate(sorted(wide_poses().items())):
        _, _, diff = LO.transform_both(wide_points(k), R, t)
        out += [(name, int(i), int(j)) for i, j in zip(*diff)]
    return out


# numpy's OpenBLAS dgemm agrees with the FMA chain on every wide pose: no double-rounding case to pin
DOUBLE_ROUNDING = []


def expected_parts(key, sweeps, poses, lags, use_dim, key_use_dim=None, sweeps_num=9, pad_empty_sweeps=True,
                   remove_close=True, point_cloud_range=None, radius=1.0):
    """The reference cloud split into its parts: [(rows, transformed)], the key, then each sweep (transformed, by the
    exact FMA chain when its coordinates are finite, else by numpy's `@`) or each pad copy.  Concatenated they are
    lidar_sweeps_oracle.multi_sweeps."""
    empty = np.zeros((0, key.shape[1]), np.float32)
    kw = dict(point_cloud_range=point_cloud_range, remove_close_on=remove_close)
    head = LO.multi_sweeps(key, [], [], [], [], use_dim, key_use_dim, sweeps_num=0, **kw)
    parts = [(head, False)]
    if pad_empty_sweeps and len(sweeps) == 0:
        pad = LO.multi_sweeps(key, [], [], [], [], use_dim, key_use_dim, sweeps_num=sweeps_num, **kw)[len(head):]
        step = len(pad) // max(sweeps_num, 1)
        parts += [(pad[k * step:(k + 1) * step], False) for k in range(sweeps_num)]
    else:
        for raw, (R, t), lag in zip(sweeps, poses, lags):
            exact = bool(np.isfinite(raw[:, use_dim[:3]]).all())
            with np.errstate(all="ignore"):
                rows = LO.multi_sweeps(empty, [raw], [R], [t], [lag], use_dim, key_use_dim, exact=exact, **kw)
            parts.append((rows, True))
    if radius != 1.0:
        raise ValueError("the oracle's remove_close radius is 1.0")
    return parts


TRANSFORMED_COLS = (0, 1, 2, 4)


def rows_equal(got, parts):
    """got [n, F] against expected_parts: bits everywhere, except that a transformed row's coordinates and lag
    compare NaN positions (CUDA makes the canonical NaN, numpy keeps the payload)"""
    want = np.concatenate([p for p, _ in parts], 0) if parts else np.zeros((0, got.shape[1]), np.float32)
    if got.shape != want.shape:
        return False
    gi, wi = got.view(np.int32).copy(), want.view(np.int32).copy()
    at = 0
    for rows, transformed in parts:
        if transformed:
            for c in TRANSFORMED_COLS:
                g, w = got[at:at + len(rows), c], want[at:at + len(rows), c]
                if not np.array_equal(np.isnan(g), np.isnan(w)):
                    return False
                gi[at:at + len(rows), c][np.isnan(g)] = 0
                wi[at:at + len(rows), c][np.isnan(w)] = 0
        at += len(rows)
    return np.array_equal(gi, wi)


def boundary_rows(n_extra_cols, seed):
    """raw rows [n, 2 + n_extra_cols] whose columns 0, 1 take every pair of the remove_close boundary values (1.0
    and +-nextafter(1, 0) and nextafter(1, 2), +-0.0, NaN, +-inf, 0.5, 2.0 with signs), and whose other columns are a
    shuffled copy of the same pairs -- the pad copies are filtered on those"""
    vals = np.array([1.0, -1.0, ONE_BELOW, -ONE_BELOW, ONE_ABOVE, 0.0, -0.0, np.nan, np.inf, -np.inf, 0.5, -2.0],
                    np.float32)
    xy = np.array([(a, b) for a in vals for b in vals], np.float32)
    rng = np.random.default_rng(seed)
    out = np.zeros((len(xy), 2 + n_extra_cols), np.float32)
    out[:, :2] = xy
    for c in range(2, 2 + n_extra_cols):
        out[:, c] = xy[rng.permutation(len(xy)), c % 2]
    return out


def _ulps(v, steps):
    """v (fp32) moved by each of `steps` fp32 ulps"""
    out = np.empty(len(steps), np.float32)
    for i, s in enumerate(steps):
        x = F32(v)
        for _ in range(abs(int(s))):
            x = np.nextafter(x, F32(np.inf) if s > 0 else F32(-np.inf))
        out[i] = x
    return out


def face_rows(R, t, rng_bounds, budget=48):
    """sweep rows xyz (fp32) whose exact FMA-chain transform under (R, t) lands on each face of the fp32 range box,
    one fp32 ulp inside and one outside it, with the other two coordinates at the box centre: [(xyz, axis, where)]
    with where in ("on", "in", "out"); a target no row within `budget` ulps of the first guess reaches is left out"""
    lo, hi = F32(rng_bounds[:3]), F32(rng_bounds[3:])
    centre = (lo.astype(np.float64) + hi) / 2
    Ri = np.linalg.inv(np.asarray(R, np.float64))
    out = []
    for j in range(3):
        k = int(np.argmax(np.abs(np.asarray(R)[j])))
        for face, inward, outward in ((lo[j], np.inf, -np.inf), (hi[j], -np.inf, np.inf)):
            for where, target in (("on", face), ("in", np.nextafter(face, F32(inward))),
                                  ("out", np.nextafter(face, F32(outward)))):
                goal = centre.copy()
                goal[j] = float(target)
                p = (Ri @ (goal - np.asarray(t, np.float64))).astype(np.float32)
                for lo_s in range(0, budget, 8):
                    steps = [s for a in range(lo_s, lo_s + 8) for s in ((a, -a) if a else (0,))]
                    cand = np.repeat(p[None], len(steps), 0)
                    cand[:, k] = _ulps(p[k], steps)
                    got = LO.transform_exact(cand, R, t)
                    hit = np.nonzero(got[:, j].view(np.int32) == np.float32(target).view(np.int32))[0]
                    if len(hit):
                        out.append((cand[hit[0]], j, where))
                        break
    return out


# the poses of the face cases: every face, one ulp in and one out, is reached from an fp32 input
FACE_POSES = ("yaw90", "yaw180", "yaw-90", "roll90", "roll270")


def face_truth(xyz_out, rng_bounds):
    """in_range_3d of transformed fp32 rows"""
    lo, hi = F32(rng_bounds[:3]), F32(rng_bounds[3:])
    return np.all((xyz_out > lo) & (xyz_out < hi), axis=1)


def all_negative_row_pose():
    """(R, row j) of a rotation whose row j has three negative entries: a zero point's dot product with it is three
    -0.0 terms, which the dgemm sums from +0.0 to +0.0"""
    for yaw in np.linspace(0.2, 3.0, 15):
        for pitch in (-0.4, 0.4):
            for roll in (-0.3, 0.3):
                R = rotation(yaw, pitch, roll)
                for j in range(3):
                    if (R[j] < 0).all():
                        return R, j
    return None


LAGS = {"inf": 1e39, "-inf": -1e39, "subnormal": 1e-40, "-subnormal": -3e-42, "to-zero": 5e-324,
        "nan": float("nan"), "tiny": 1.5e-38}


def tile_caps(n_kept_per_entry):
    """caps on the edges of the write kernel's tile offsets, with every row of every entry kept: 1, each offset at
    which a kTile-row tile starts (the early return off >= cap) and one either side, and the total and one either
    side"""
    offs, at = [], 0
    for n in n_kept_per_entry:
        offs += [at + t * SWEEP_TILE for t in range(-(-n // SWEEP_TILE))]
        at += n
    caps = {1, at - 1, at, at + 1}
    for o in offs:
        caps |= {o - 1, o, o + 1}
    return sorted(c for c in caps if c >= 1), offs, at


# entries of the tile case: rows of the key and two sweeps, each spanning tiles
TILE_ROWS = (2 * SWEEP_TILE + 5, 3 * SWEEP_TILE - 1, SWEEP_TILE + 1)
