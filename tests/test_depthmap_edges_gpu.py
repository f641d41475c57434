"""The LiDAR depth rasteriser against a float64 projection written from the reference's formulas
(not from the oracle's operation order), on pixel and bin edges where fp32 is exact, on collisions,
and on the inputs it must refuse."""
import numpy as np
import pytest
import torch

import oracle

pytestmark = pytest.mark.gpu

U = 2.0 ** -23     # twice the fp32 unit roundoff: every first-order bound below keeps a factor 2 in hand


def _affine(M, x, e):
    """y = M[:3, :3] x + M[:3, 3] in float64 for rows x [N, 3] with absolute error e [N, 3] on x:
    returns (y, error bound of the fp32 evaluation of the same expression).  Each of the four terms
    of a row is rounded once and added with at most three more roundings, so the rounding part is
    below 4 * 2^-24 * (|M| |x| + |t|) to first order (U doubles it); the incoming error is
    carried through by |M|."""
    R, t = M[:3, :3].astype(np.float64), M[:3, 3].astype(np.float64)
    return x @ R.T + t, e @ np.abs(R).T + 4 * U * (np.abs(x) @ np.abs(R).T + np.abs(t))


def project_f64(points, lidar2image, img_aug, lidar_aug):
    """BaseDepthTransform.forward's projection (base.py:289-305) for one sample in float64 matrix
    algebra: x = inv(R_aug) (p - t_aug); y = L x; z = clamp(y_z, 1e-5, 1e5); (u, v) = A (y_x / z,
    y_y / z, z).  Returns per camera u, v, z [ncam, N] and eu, ev, ez, bounds on how far the fp32
    pipeline can be from them: every fp32 operation adds 2^-24 of its result (the _affine bound per
    matrix step, one rounding per subtract / divide), each matrix step carries the previous step's
    error through |M|, and the divide is bounded as an interval.  The fp32 3x3 inverse (adjugate: 2 products, one
    subtract, one divide by a 5-operation determinant) is within 16 * 2^-24 * max|inv| of the
    float64 one for the rotation-times-scale matrices used here."""
    p = np.asarray(points, np.float64)[:, :3]
    la = np.asarray(lidar_aug, np.float64)
    x1 = p - la[:3, 3]
    e1 = U * np.abs(x1)
    inv = np.linalg.inv(la[:3, :3])
    x2 = x1 @ inv.T
    e2 = e1 @ np.abs(inv).T + 3 * U * (np.abs(x1) @ np.abs(inv).T) + 16 * U * np.abs(inv).max() * np.abs(x1).sum(1, keepdims=True)
    lo, hi = np.float64(np.float32(1e-5)), np.float64(np.float32(1e5))
    us, vs, zs, eus, evs, ezs = [], [], [], [], [], []
    for L, A in zip(np.asarray(lidar2image, np.float64), np.asarray(img_aug, np.float64)):
        y, ey = _affine(L, x2, e2)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            z = np.clip(y[:, 2], lo, hi)                     # the clamp is 1-Lipschitz ...
            ez = np.where((y[:, 2] + ey[:, 2] < lo) | (y[:, 2] - ey[:, 2] > hi), 0.0, ey[:, 2])   # ... and exact once it binds
            # the fp32 z lies in [zmin, zmax] (never outside the clamp) and the numerators in y +- ey:
            # the quotient's interval comes from its four corners, plus the divide's own rounding
            zmin, zmax = np.maximum(z - ez, lo)[:, None], np.minimum(z + ez, hi)[:, None]
            q = y[:, :2] / z[:, None]
            corners = np.stack([(y[:, :2] - ey[:, :2]) / zmin, (y[:, :2] - ey[:, :2]) / zmax,
                                (y[:, :2] + ey[:, :2]) / zmin, (y[:, :2] + ey[:, :2]) / zmax])
            eq = np.maximum(corners.max(0) - q, q - corners.min(0)) * (1 + U) + U * np.abs(q)
            w, ew = _affine(A, np.concatenate([q, z[:, None]], 1), np.concatenate([eq, ez[:, None]], 1))
        us.append(w[:, 0]); vs.append(w[:, 1]); zs.append(z)
        eus.append(ew[:, 0]); evs.append(ew[:, 1]); ezs.append(ez)
    return tuple(np.stack(a) for a in (us, vs, zs, eus, evs, ezs))


def expected_depth_f64(points, lidar2image, img_aug, lidar_aug, image_size):
    """-> (winner [ncam, H, W] point index or -1, z [ncam, N], ez [ncam, N], skip [ncam, H, W]).
    A point is decided for a camera when, with its error bound on either side, u and v stay in
    one pixel or stay off the image; the winner of a pixel is the largest decided index landing on
    it (sequential index_put, base.py:321).  Pixels an undecided point could touch are in `skip`."""
    H, W = int(image_size[0]), int(image_size[1])
    u, v, z, eu, ev, ez = project_f64(points, lidar2image, img_aug, lidar_aug)
    ncam, n = u.shape
    winner = np.full((ncam, H, W), -1, np.int64)
    skip = np.zeros((ncam, H, W), bool)
    with np.errstate(invalid="ignore"):
        for c in range(ncam):
            fin = np.isfinite(u[c]) & np.isfinite(v[c]) & np.isfinite(eu[c]) & np.isfinite(ev[c])
            ulo, uhi, vlo, vhi = u[c] - eu[c], u[c] + eu[c], v[c] - ev[c], v[c] + ev[c]
            off = (uhi < 0) | (ulo >= W) | (vhi < 0) | (vlo >= H)
            one = (np.floor(ulo) == np.floor(uhi)) & (np.floor(vlo) == np.floor(vhi)) & (ulo >= 0) & (uhi < W) \
                & (vlo >= 0) & (vhi < H)
            # non-finite projections (NaN / inf points, or the error blown up by z ~ 0) that are far
            # off the image in float64 stay off it in fp32: |u| beyond 1e6 pixels cannot round back
            far = ~fin & ~(np.abs(u[c]) < 1e6) | ~fin & ~(np.abs(v[c]) < 1e6)
            on = fin & one
            idx = np.nonzero(on)[0]
            np.maximum.at(winner[c], (np.floor(v[c][idx]).astype(np.int64), np.floor(u[c][idx]).astype(np.int64)), idx)
            und = np.nonzero(~(on | (fin & off) | far))[0]
            for i in und:
                if not fin[i]:
                    skip[c] = True
                    continue
                r0, r1 = int(max(np.floor(vlo[i]), 0)), int(min(np.floor(vhi[i]), H - 1))
                c0, c1 = int(max(np.floor(ulo[i]), 0)), int(min(np.floor(uhi[i]), W - 1))
                skip[c, r0:r1 + 1, c0:c1 + 1] = True
    return winner, z, ez, skip


def assert_scalar_matches_f64(depth, feats_planes, points, expected, what=""):
    """depth [ncam, H, W] (and feature planes [ncam, F, H, W] or None) against expected_depth_f64:
    on every pixel not skipped, the winner's float64 depth to 8 fp32 ulp plus the bound of its own
    rounding, zero where no point lands; feature planes carry the winner's row.  Returns
    the share of skipped pixels."""
    winner, z, ez, skip = expected
    ncam = winner.shape[0]
    for c in range(ncam):
        w = winner[c]
        has = (w >= 0) & ~skip[c]
        none = (w < 0) & ~skip[c]
        assert not depth[c][none].any(), what + ": depth written where no point projects"
        zz, tol = z[c][w[has]], 8 * 2.0 ** -23 * z[c][w[has]] + ez[c][w[has]]
        assert (np.abs(depth[c][has] - zz) <= tol).all(), what + ": depth differs from the float64 projection"
        assert (depth[c][has] > 0).all()
        if feats_planes is not None:
            assert np.array_equal(feats_planes[c][:, has], points[w[has]].T), what + ": feature planes"
            assert not feats_planes[c][:, none].any()
    return skip.mean()


def rig(ncam, image_size, aug, batch):
    """lidar2image / img_aug / lidar_aug for `ncam` cameras: the six synthetic cameras repeated with
    a different crop each; aug = none | rot_scale_trans | reflection (negative determinant)."""
    from bevfusion_b200 import synthetic as S
    M = S.lidar_camera_matrices(min(ncam, 6), image_size, batch=batch, augment=aug != "none")
    idx = torch.arange(ncam) % min(ncam, 6)
    l2i, ia, la = M["lidar2image"][:, idx].clone(), M["img_aug_matrix"][:, idx].clone(), M["lidar_aug_matrix"].clone()
    for k in range(6, ncam):
        ia[:, k, 0, 3] += 0.37 * k
        ia[:, k, 1, 3] -= 0.21 * k
    if aug == "reflection":
        la[:, :3, :3] = la[:, :3, :3] @ torch.diag(torch.tensor([1.0, -1.0, 1.0]))
        assert float(torch.det(la[0, :3, :3])) < 0
    return dict(lidar2image=l2i.contiguous(), img_aug_matrix=ia.contiguous(), lidar_aug_matrix=la.contiguous())


def cloud(nf, seed, n=None):
    from bevfusion_b200 import synthetic as S
    c = S.lidar_cloud(seed=seed, sweeps=1)
    if n is not None:
        c = c[:n]
    rng = np.random.default_rng(seed)
    if nf <= 5:
        return np.ascontiguousarray(c[:, :nf])
    return np.ascontiguousarray(np.concatenate([c, rng.standard_normal((len(c), nf - 5)).astype(np.float32)], 1))


def run_ours(cuda, clouds, M, image_size, **kw):
    from bevfusion_b200.vtransform import points_to_depth
    pts = [torch.from_numpy(c).to(cuda) for c in clouds]
    d = points_to_depth(pts, M["lidar2image"].to(cuda), M["img_aug_matrix"].to(cuda),
                        M["lidar_aug_matrix"].to(cuda), image_size, **kw)
    return d.cpu().numpy()


NCAMS = [1, 6, 16]
IMAGE_SIZES = [(256, 704), (64, 176), (1, 1), (37, 53)]
AUGS = ["none", "rot_scale_trans", "reflection"]
WIDTHS = [3, 5, 45]


def projection_cases():
    out = []
    for i, ncam in enumerate(NCAMS):
        for j, size in enumerate(IMAGE_SIZES):
            for k, aug in enumerate(AUGS):
                out.append((ncam, size, aug, WIDTHS[(i + j + k) % 3]))
    return out


@pytest.mark.parametrize("ncam,image_size,aug,nf", projection_cases())
def test_scalar_depth_vs_float64_projection(cuda, ncam, image_size, aug, nf):
    """A batch of three samples (one empty) with different point counts; scalar depth plus feature
    planes; every decided pixel matches the float64 projection."""
    clouds = [cloud(nf, 1), cloud(nf, 2)[:0], cloud(nf, 3, n=5000)]
    M = rig(ncam, image_size, aug, batch=3)
    d = run_ours(cuda, clouds, M, image_size, add_depth_features=True)
    assert d.shape == (3, ncam, 1 + nf) + tuple(image_size)
    assert not d[1].any()
    shares, hits = [], 0
    for b in (0, 2):
        la = M["lidar_aug_matrix"][b].numpy()
        exp = expected_depth_f64(clouds[b], M["lidar2image"][b].numpy(), M["img_aug_matrix"][b].numpy(), la, image_size)
        shifted = clouds[b].copy()
        shifted[:, :3] -= la[:3, 3]                          # the feature planes carry xyz - t_aug (base.py:290)
        shares.append(assert_scalar_matches_f64(d[b, :, 0], d[b, :, 1:], shifted, exp, "sample %d" % b))
        hits += int((exp[0] >= 0).sum())
    if image_size[0] * image_size[1] >= 1000:
        assert max(shares) < 0.01 and hits > 50
    else:
        assert min(shares) < 1.0 or image_size == (1, 1)


# ---- exact cases: identity augmentations, power-of-two focal length and depths -> no fp32 rounding
EXACT_SIZE = (8, 16)


def exact_rig():
    """cam 0: f = 4, principal point (8, 4).  cam 1: f = 4, principal point (0, 4) and every zero of
    its matrices that meets the u row written as -0.0, so that a point with X = -0.0 reaches
    u = -0.0 without a single +0.0 being added on the way."""
    K0 = np.array([[4, 0, 8, 0], [0, 4, 4, 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float32)
    K1 = np.array([[4, -0.0, -0.0, -0.0], [0, 4, 4, 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float32)
    A0 = np.eye(4, dtype=np.float32)
    A1 = np.eye(4, dtype=np.float32)
    A1[0, 1:] = -0.0
    return dict(lidar2image=torch.from_numpy(np.stack([K0, K1])[None]),
                img_aug_matrix=torch.from_numpy(np.stack([A0, A1])[None]),
                lidar_aug_matrix=torch.eye(4)[None])


def exact_all_ways(cuda, pts, **kw):
    """kernel == oracle, bit for bit, on the exact rig; returns the [2, C, 8, 16] image."""
    M = exact_rig()
    d = run_ours(cuda, [pts], M, EXACT_SIZE, **kw)[0]
    gold = oracle.points_to_depth(pts, M["lidar2image"][0].numpy(), M["img_aug_matrix"][0].numpy(),
                                  M["lidar_aug_matrix"][0].numpy(), EXACT_SIZE,
                                  **{k: v for k, v in kw.items() if k != "height_expand"})
    assert np.array_equal(d.view(np.int32), gold.view(np.int32))
    return d


def test_exact_pixel_edges(cuda):
    """u = 0 and u = W - 1 are kept, u = W and v = H are dropped, pixel corners belong to the pixel
    they open, z beyond 1e5 is clamped: kernel, oracle and float64 agree exactly."""
    pts = np.array([
        [-4, 0, 2],          # u = 0,  v = 4, z = 2
        [7, 0, 4],           # u = 15 = W - 1
        [8, 0, 4],           # u = 16 = W: dropped
        [0, 4, 4],           # v = 8 = H: dropped
        [-5, -2, 4],         # corner (u, v) = (3, 2)
        [-8, -4, 4],         # corner (0, 0)
        [7, 3, 4],           # corner (15, 7)
        [-8.5, 0, 4],        # u = -0.5: dropped
        [0, 0, 131072],      # z = 2^17 > 1e5: depth 1e5, u = 8 * 2^17 / 1e5 = 10.48
    ], np.float32)
    d = exact_all_ways(cuda, pts)[0, 0]
    want = np.zeros(EXACT_SIZE, np.float32)
    want[4, 0], want[4, 15], want[2, 3], want[0, 0], want[7, 15], want[5, 10] = 2, 4, 4, 4, 4, 1e5
    assert np.array_equal(d, want)
    M = exact_rig()
    winner, z, ez, skip = expected_depth_f64(pts, M["lidar2image"][0, :1].numpy(), M["img_aug_matrix"][0, :1].numpy(),
                                             np.eye(4), EXACT_SIZE)
    # float64 sees the same pixels wherever its own (conservative) rounding margin lets it decide;
    # the points placed exactly on an edge are the ones it must leave open
    assert np.array_equal(np.where(winner[0] >= 0, z[0][winner[0]], 0).astype(np.float32)[~skip[0]], want[~skip[0]])
    assert winner[0, 5, 10] == 8


def test_pin_u_of_minus_zero_is_column_zero(cuda):
    """u = -0.0 passes `u >= 0` and truncates to column 0, in the kernel and in the oracle."""
    pts = np.array([[-0.0, 0.5, 1]], np.float32)             # camera 1: u = -0.0, v = 4 * 0.5 + 4 = 6
    d = exact_all_ways(cuda, pts)
    assert d[1, 0, 6, 0] == 1.0 and np.count_nonzero(d[1]) == 1
    M = exact_rig()
    u = np.float32(M["lidar2image"][0, 1, 0, 0]) * pts[0, 0]
    assert u == 0 and np.signbit(u)


def test_pin_behind_camera_points_are_clamped_to_depth_1e_5(cuda):
    """z <= 0 is clamped to 1e-5 BEFORE the perspective divide (base.py:299-300), so a point at or
    behind the camera is not dropped: it is drawn wherever (x, y) / 1e-5 lands.  A point in the
    camera centre, or behind the camera with x = y = 0 in image space, writes depth 1e-5 at pixel
    (0, 0); an on-axis point behind the camera is thrown far off the image."""
    eps = np.float32(1e-5)
    d = exact_all_ways(cuda, np.array([[0, 0, 0]], np.float32))
    assert d[0, 0, 0, 0] == eps and np.count_nonzero(d[0]) == 1
    d = exact_all_ways(cuda, np.array([[2, 1, -1]], np.float32))          # 4 * 2 + 8 * -1 = 0, 4 * 1 + 4 * -1 = 0
    assert d[0, 0, 0, 0] == eps and np.count_nonzero(d[0]) == 1
    d = exact_all_ways(cuda, np.array([[0, 0, -1]], np.float32))          # u = -8 / 1e-5
    assert np.count_nonzero(d[0]) == 0


@pytest.mark.parametrize("D", [1, 2, 118])
@pytest.mark.parametrize("features", [False, True])
def test_one_hot_bin_edges(cuda, D, features):
    """On-axis points (all on pixel (4, 8) of camera 0) with depths on integers, just under them,
    below 1 and at or beyond D - 1: bin = int(min(z, D - 1)); every bin hit is set, and the feature
    planes follow the largest index."""
    below = lambda x: np.nextafter(np.float32(x), np.float32(0))
    zs = np.array([0.5, below(1), 1, below(2), 2, 3, 116, below(117), 117, 117.5, 118, 5000, 2.5], np.float32)
    pts = np.zeros((len(zs), 4), np.float32)
    pts[:, 2] = zs
    pts[:, 3] = np.arange(len(zs)) + 100
    d = exact_all_ways(cuda, pts, depth_input="one-hot", depth_bins=D, add_depth_features=features)
    bins = sorted({int(min(float(z), D - 1)) for z in zs})
    planes = d[0, :D]
    assert np.nonzero(planes[:, 4, 8])[0].tolist() == bins and (planes[bins, 4, 8] == 1).all()
    assert np.count_nonzero(planes) == len(bins)
    if D == 118:
        assert bins == [0, 1, 2, 3, 116, 117]
    if features:
        assert np.array_equal(d[0, D:, 4, 8], pts[-1]) and np.count_nonzero(d[0, D:]) == 2


def test_collisions_last_index_wins(cuda):
    """10 000 points on one pixel: the largest index wins the scalar and the feature planes, and
    does so again on a second run."""
    n = 10000
    pts = np.zeros((n, 5), np.float32)
    pts[:, 2] = 1 + np.random.default_rng(0).permutation(n) / 1024.0        # exact in fp32, all distinct
    pts[:, 3] = np.arange(n)
    pts[:, 4] = -1.5
    d = exact_all_ways(cuda, pts, add_depth_features=True)
    assert d[0, 0, 4, 8] == pts[-1, 2] and np.array_equal(d[0, 1:, 4, 8], pts[-1])
    assert np.count_nonzero(d[0, 0]) == 1
    assert np.array_equal(exact_all_ways(cuda, pts, add_depth_features=True), d)


def test_height_expand_on_exact_points(cuda):
    """height_expand == the reference's repeat_interleave(8) with z = 0.25 .. 2.0 (base.py:269-273)."""
    from bevfusion_b200.vtransform import points_to_depth
    pts = np.array([[-1, 0, 9, 5], [0.5, 0.25, 9, 6], [0, -0.5, 9, 7]], np.float32)
    M = exact_rig()
    d = run_ours(cuda, [pts], M, EXACT_SIZE, height_expand=True, add_depth_features=True)[0]
    rep = np.repeat(pts, 8, axis=0)
    rep[:, 2] = np.tile(np.arange(0.25, 2.25, 0.25, dtype=np.float32), len(pts))
    gold = oracle.points_to_depth(rep, M["lidar2image"][0].numpy(), M["img_aug_matrix"][0].numpy(), np.eye(4),
                                  EXACT_SIZE, add_depth_features=True)
    assert np.array_equal(d, gold) and np.count_nonzero(d[0, 0]) > 3


def test_refused_inputs(cuda):
    from bevfusion_b200 import _C
    from bevfusion_b200.vtransform import points_to_depth
    pts = torch.rand(10, 5, device=cuda)
    eye = torch.eye(4, device=cuda)
    with pytest.raises(_C.BevB200Error, match="bad camera / image size"):
        points_to_depth([pts], eye.repeat(1, 17, 1, 1), eye.repeat(1, 17, 1, 1), eye[None], (8, 16))
    with pytest.raises(ValueError, match="depth_bins"):
        points_to_depth([pts], eye.repeat(1, 2, 1, 1), eye.repeat(1, 2, 1, 1), eye[None], (8, 16),
                        depth_input="one-hot", depth_bins=0)
    before = _C.launch_count()
    with pytest.raises(ValueError, match="same number of point features"):
        points_to_depth([pts, pts[:, :4].contiguous()], eye.repeat(2, 2, 1, 1), eye.repeat(2, 2, 1, 1),
                        eye.repeat(2, 1, 1), (8, 16))
    assert _C.launch_count() == before                       # refused before the first sample is rasterised
