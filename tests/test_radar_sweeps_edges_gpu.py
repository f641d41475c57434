"""GPU: RadarSweepStore.assemble at the edges of its numerical contract, bit-equal (int32 view) to the numpy
restatement of the reference: rows transformed exactly onto the +-55 range faces and one fp32 ulp either side; NaN
and inf coordinates, velocities and lags; signed zeros through the rotation chains; one-hot sources at .5 ties, in
[-w, -1] and outside [-w, w) (the reference raises there; the device zeroes the block and sets BAD_CATEGORY); the
ordinal and nusc-filter columns at their thresholds."""
import numpy as np
import pytest

import radar_sweeps_oracle as O

pytestmark = pytest.mark.gpu

ALL = list(range(58))


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def run(cuda, raws, poses, lags, use_dim=ALL, compensate=True, bev_range=O.BEV_RANGE, bad_category="raise"):
    """device output, counts and status of one sample against the oracle"""
    from bevfusion_b200.radar_sweeps import RadarSweepStore
    store = RadarSweepStore(len(raws), max(max(len(r) for r in raws), 1), cuda, max_batch=1,
                            max_entries=len(raws))
    for k, r in enumerate(raws):
        store.put(k, r)
    sample = [(k, poses[k][0], poses[k][1], lags[k]) for k in range(len(raws))]
    out, counts, status = store.assemble([sample], use_dim, compensate, bev_range=bev_range, sync=False)
    got = out[0, :int(counts[0])].cpu().numpy()
    with np.errstate(all="ignore"):
        want = O.multi_sweeps(raws, [p[0] for p in poses], [p[1] for p in poses], lags, use_dim, compensate,
                              bev_range=bev_range, bad_category=bad_category)
    return got, want, int(status.item())


def plain_rows(n, rng=None):
    rng = rng or np.random.default_rng(n)
    r = O.radar_sweep(rng, n)
    r[:, 6:10] = 0.0
    return r


IDENTITY = (np.eye(3), np.zeros(3))


@pytest.mark.parametrize("translate", [False, True])
def test_range_faces_and_one_ulp_either_side(cuda, translate):
    # identity rotation: x = fl32(fl32(r0) + t0), so raw values land exactly where chosen
    f32 = np.float32
    vals = []
    for face in (f32(-55.0), f32(55.0)):
        vals += [face, np.nextafter(face, f32(0)), np.nextafter(face, f32(np.copysign(np.inf, face)))]
    vals += [f32(0.0), f32(-0.0), f32(np.nan), f32(np.inf), f32(-np.inf)]
    xs, ys = np.meshgrid(np.array(vals, f32), np.array(vals, f32))
    raw = plain_rows(xs.size)
    t = np.array([5.0, -3.0, 0.25]) if translate else np.zeros(3)
    raw[:, 0], raw[:, 1] = xs.ravel() - f32(t[0]), ys.ravel() - f32(t[1])   # x - 5 + 5, y + 3 - 3: exact here
    got, want, st = run(cuda, [raw], [(np.eye(3), t)], [0.0], compensate=False)
    assert st == 0 and bits_equal(got, want)
    assert want.shape[0] == 16          # both coordinates one ulp inside a face, or +-0


def test_nan_inf_coordinates_velocities_and_lags(cuda):
    rng = np.random.default_rng(3)
    raws, poses, lags = [], [], []
    for k, lag in enumerate([0.0, np.nan, np.inf, -np.inf, 1e308, -0.0, 5e-324]):
        r = O.radar_sweep(rng, 40)
        r[0, 0], r[1, 1], r[2, 2] = np.nan, np.inf, -np.inf
        r[3, 6], r[4, 7], r[5, 8], r[6, 9] = np.nan, np.inf, -np.inf, np.nan
        r[7, 8:10] = np.float32(3e38)
        raws.append(r)
        poses.append(O.radar_pose(rng, k % 5))
        lags.append(lag)
    for bev_range in (O.BEV_RANGE, None):
        for compensate in (True, False):
            got, want, st = run(cuda, raws, poses, lags, compensate=compensate, bev_range=bev_range)
            assert st == 0 and bits_equal(got, want), (bev_range, compensate)


def test_signed_zeros_through_the_chains(cuda):
    # zero points and velocities, with and without -0.0, under rotations whose rows have negative entries and a
    # -0.0 translation: the +0 start of the chain and the +0 column of the velocity rows decide each sign
    z, nz = np.float32(0.0), np.float32(-0.0)
    combos = np.array(np.meshgrid([z, nz], [z, nz], [z, nz])).reshape(3, -1).T.astype(np.float32)
    raw = plain_rows(len(combos))
    raw[:, 0:3] = combos
    raw[:, 6:8] = combos[:, :2]
    raw[:, 8:10] = combos[:, 1:]
    rots = [-np.eye(3), np.array([[-1.0, -0.0, -0.0], [-0.0, -1.0, -0.0], [0.0, 0.0, 1.0]]),
            np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, -1.0]])]
    for R in rots:
        for t in (np.array([-0.0, -0.0, -0.0]), np.zeros(3)):
            for lag in (0.0, -0.0, 0.5):
                got, want, st = run(cuda, [raw], [(R, t)], [lag], bev_range=None)
                assert st == 0 and bits_equal(got, want), (R.tolist(), t.tolist(), lag)


def test_one_hot_ties_and_wrapped_indices(cuda):
    halves = np.arange(-8.5, 7.5, 0.5, dtype=np.float32)       # every value rounds into [-8, 7]
    raw = plain_rows(len(halves))
    raw[:, 3] = halves
    raw[:, 11] = np.clip(halves, -5.0, 4.5)
    raw[:, 14] = halves
    raw[:, 15] = halves
    got, want, st = run(cuda, [raw], [IDENTITY], [0.0], bev_range=None)
    assert st == 0 and bits_equal(got, want)
    assert want[:, 19:27].sum() == len(halves) and want[0, 19] == 1.0   # rint(-8.5) = -8 wraps to index 0


@pytest.mark.parametrize("col,bad", [(3, 7.5), (3, -9.0), (11, 5.0), (11, -5.5), (14, 18.0), (14, np.nan),
                                     (3, np.inf), (14, -np.inf), (11, 3e9)])
def test_one_hot_outside_the_encoding(cuda, col, bad):
    from bevfusion_b200.radar_sweeps import BAD_CATEGORY
    raw = plain_rows(50)
    raw[[3, 17, 49], col] = np.float32(bad)
    with pytest.raises(IndexError):                       # the reference raises on this frame
        O.multi_sweeps([raw], [np.eye(3)], [np.zeros(3)], [0.0], ALL, bev_range=None)
    got, want, st = run(cuda, [raw], [IDENTITY], [0.0], bev_range=None, bad_category="zero")
    assert st == BAD_CATEGORY and bits_equal(got, want)
    # not selected by use_dim: the reference still raises, so the status still says so
    got, want, st = run(cuda, [raw], [IDENTITY], [0.0], use_dim=[0, 1, 2], bev_range=None, bad_category="zero")
    assert st == BAD_CATEGORY and bits_equal(got, want)


def test_ordinal_and_nusc_filter_thresholds(cuda):
    f32 = np.float32
    pdh = np.array([-0.5, 0.0, 0.5, 0.5000001, 1.5, 2.5, 6.4999995, 6.5, 7.5, np.nan, np.inf, -np.inf], f32)
    raw = plain_rows(len(pdh) * 4)
    raw[:, 15] = np.tile(pdh, 4)
    raw[:, 14] = np.repeat(np.array([0.0, -0.0, 0.0, 1.0], f32), len(pdh))
    raw[:, 3] = np.tile(np.array([6.0, 7.0, 6.4999995, 6.0], f32), len(pdh))
    raw[:, 11] = np.repeat(np.array([3.0, 3.0, 3.0, 3.0], f32), len(pdh))
    raw[::5, 11] = f32(2.9999998)
    got, want, st = run(cuda, [raw], [IDENTITY], [0.0], bev_range=None)
    assert st == 0 and bits_equal(got, want)
    assert 0 < want[:, 57].sum() < len(raw)
