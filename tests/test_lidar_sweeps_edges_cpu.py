"""CPU: the multi-sweep assembly's boundary cases (tests/data_pipeline_cases.py) -- numpy's `@` against the exact FMA
chain over quarter and half turns, arbitrary rotations and translations up to 10 km (the double-rounding cases are
pinned), and that each case builder lands on the boundary it names: rows transformed exactly onto the range faces,
remove_close boundaries that tell the raw columns from the selected ones, the all-negative rotation row of the
signed-zero case, and the caps on the write kernel's tile offsets."""
import numpy as np

import data_pipeline_cases as C
import lidar_sweeps_oracle as O


def test_double_rounding_cases_are_pinned():
    """numpy's dgemm and the FMA chain agree on every wide pose; a BLAS that disagreed would show up here first"""
    found = C.double_rounding_cases()
    assert found == C.DOUBLE_ROUNDING, found[:20]
    assert len(C.wide_poses()) >= 20


def test_face_rows_land_on_the_faces():
    poses = C.wide_poses()
    for name in C.FACE_POSES:
        R, t = poses[name]
        rows = C.face_rows(R, t, C.PCR)
        assert sorted((j, w) for _, j, w in rows) == sorted((j, w) for j in range(3) for w in ("on", "in", "out")
                                                             for _ in range(2)), name
        xyz = np.stack([r for r, _, _ in rows])
        out = O.transform_exact(xyz, R, t)
        lo, hi = np.float32(C.PCR[:3]), np.float32(C.PCR[3:])
        for (_, j, where), o in zip(rows, out):
            faces = (lo[j], hi[j])
            if where == "on":
                assert o[j] in faces
            else:
                assert any(o[j] == np.nextafter(f, np.float32(s)) for f in faces for s in (-np.inf, np.inf))
        assert list(C.face_truth(out, C.PCR)) == [w == "in" for _, _, w in rows], name


def test_boundary_rows_tell_raw_from_selected_columns():
    raw = C.boundary_rows(5, seed=1)
    sel = raw[:, [5, 6, 2, 3, 4]]
    kept_raw, kept_sel = len(O.remove_close(raw)), len(O.remove_close(sel))
    assert kept_raw != kept_sel and 0 < kept_raw < len(raw) and 0 < kept_sel < len(raw)
    close = lambda r: (np.abs(r[:, 0]) < 1) & (np.abs(r[:, 1]) < 1)
    assert (close(raw) != close(sel)).sum() > 10
    v = raw[:, 0]
    assert (v == 1.0).any() and (v == C.ONE_BELOW).any() and (v == C.ONE_ABOVE).any() and np.isnan(v).any()
    assert (np.signbit(v) & (v == 0)).any() and np.isinf(v).any()


def test_signed_zero_pose_and_the_reference_sum():
    """a zero row under a rotation row of three negative entries and a -0.0 translation: the reference (numpy's
    dgemm, then += t) gives +0.0, while a chain started from the product p0 * R[j][0] would give -0.0"""
    R, j = C.all_negative_row_pose()
    assert (R[j] < 0).all()
    zero = np.zeros((3, 3), np.float32)
    zero[1] = -0.0
    zero[2, 1] = -0.0
    t = np.array([-0.0, -0.0, -0.0])
    ref = O.transform_numpy(zero, R, t)
    assert not np.signbit(ref[0]).any() and (ref == 0).all()
    from_product = [[((p[0] * R[jj][0] + p[1] * R[jj][1]) + p[2] * R[jj][2]) + t[jj] for jj in range(3)]
                    for p in zero.astype(np.float64)]
    assert np.signbit(from_product[0][j])
    assert np.array_equal(O.transform_exact(zero, R, t).view(np.int32), ref.view(np.int32))


def test_tile_caps_sit_on_the_offsets():
    caps, offs, total = C.tile_caps(C.TILE_ROWS)
    assert total == sum(C.TILE_ROWS) and all(n > C.SWEEP_TILE for n in C.TILE_ROWS)
    starts = np.cumsum((0,) + C.TILE_ROWS[:-1])
    want = sorted(int(s) + t * C.SWEEP_TILE for s, n in zip(starts, C.TILE_ROWS)
                  for t in range(-(-n // C.SWEEP_TILE)))
    assert offs == want and len(offs) == sum(-(-n // C.SWEEP_TILE) for n in C.TILE_ROWS)
    for o in offs:
        assert {c for c in (o - 1, o, o + 1) if c >= 1} <= set(caps)
    assert {1, total - 1, total, total + 1} <= set(caps)


def test_expected_parts_concatenate_to_the_oracle():
    rng = np.random.default_rng(4)
    key = O.nuscenes_sweep(rng, 300, 6)
    sweeps = [O.nuscenes_sweep(rng, 200 + 10 * k, 6) for k in range(3)]
    poses = [O.nuscenes_pose(rng, k + 1) for k in range(3)]
    lags = [0.05, 0.1, 0.15]
    use = [0, 1, 2, 5, 4]
    parts = C.expected_parts(key, sweeps, poses, lags, use, point_cloud_range=C.PCR)
    want = O.multi_sweeps(key, sweeps, [p[0] for p in poses], [p[1] for p in poses], lags, use,
                          point_cloud_range=C.PCR)
    assert [tr for _, tr in parts] == [False, True, True, True]
    assert C.rows_equal(want, parts)
    pads = C.expected_parts(key, [], [], [], use, sweeps_num=4)
    assert len(pads) == 5 and not any(tr for _, tr in pads)
    assert C.rows_equal(O.multi_sweeps(key, [], [], [], [], use, sweeps_num=4), pads)


def test_constants_and_shapes():
    assert C.SWEEP_TILE % 32 == 0 and 8 <= C.MAX_LOAD_DIM and C.MAX_DIM == 8
    assert (C.SWEEP_NONE, C.SWEEP_KEY, C.SWEEP_SWEEP, C.SWEEP_PAD) == (0, 1, 2, 3)
    with np.errstate(over="ignore"):
        lags = np.array(list(C.LAGS.values()), np.float64).astype(np.float32)
    assert np.isinf(lags[0]) and np.isinf(lags[1]) and np.isnan(lags[5])
    assert 0 < abs(lags[2]) < np.finfo(np.float32).tiny and 0 < abs(lags[3]) < np.finfo(np.float32).tiny
    assert lags[4] == 0
