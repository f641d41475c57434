"""Voxelization on cell faces: hard, dynamic, the fused mean and voxelize_batch on clouds whose
coordinates sit on range_min / range_max, on cell faces and one ulp either side of them, for every
row width and cap the entry points accept.  Integer work is bit-equal to the oracle; the cell index
is also checked against float64 wherever float64 can decide it."""
import numpy as np
import pytest
import torch

import oracle
from conftest import ref_module

pytestmark = pytest.mark.gpu

# name -> (voxel_size, range, exact): `exact` = lo is 0 and every voxel size a power of two, so
# (p - lo) / vs has no rounding and float64 must agree on every finite point
GEOMS = {
    "exact": ([0.5, 0.25, 0.5], [0.0, 0.0, 0.0, 8.0, 4.0, 2.0], True),
    "c3": ([0.075, 0.075, 0.2], [-54.0, -54.0, -5.0, 54.0, 54.0, 3.0], False),
    "c5": ([0.05, 0.05, 0.2], [-54.0, -54.0, -5.0, 54.0, 54.0, 3.0], False),
    "pillar": ([0.2, 0.2, 8.0], [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], False),
    "nondividing": ([0.3, 0.3, 0.3], [0.0, 0.0, 0.0, 10.0, 10.0, 10.0], False),   # grid 33: [9.9, 10) is cut off
    "single": ([4.0, 4.0, 4.0], [-2.0, -2.0, -2.0, 2.0, 2.0, 2.0], False),        # 1 x 1 x 1
}
WIDTHS = [3, 4, 5, 8, 9, 45]
CAPS = ["p1_v7", "p10_binding", "p64_free"]


def grid_of(vs, cr):
    """round((hi - lo) / vs) in fp32, as every implementation computes it."""
    vs, cr = np.asarray(vs, np.float32), np.asarray(cr, np.float32)
    return np.round((cr[3:] - cr[:3]) / vs).astype(np.int64)


def face_values(vs, lo, hi, grid):
    """The coordinates one axis is probed with."""
    f32 = np.float32
    vs, lo, hi = f32(vs), f32(lo), f32(hi)
    out = []
    for k in sorted({0, 1, int(grid) // 2, max(int(grid) - 2, 0), int(grid) - 1, int(grid)}):
        face = f32(np.float64(lo) + k * np.float64(vs))
        out += [face, np.nextafter(face, f32(-np.inf)), np.nextafter(face, f32(np.inf))]
    tiny = f32(1e-45)
    out += [lo, hi, np.nextafter(hi, f32(-np.inf)), f32(0.0), f32(-0.0), tiny, -tiny, f32(3e38), f32(-3e38),
            f32(np.nan), f32(np.inf), f32(-np.inf)]
    return np.asarray(out, f32)


def boundary_cloud(vs, cr, nf, seed, background=1500):
    """Background (half uniform with a margin outside the range, half in tight clusters so that
    max_points binds) with, shuffled into it, points that have ONE coordinate from face_values()
    and the other two random inside the range.  Returns (points [N, nf] fp32, is_probe [N])."""
    rng = np.random.default_rng(seed)
    vs32, cr32 = np.asarray(vs, np.float32), np.asarray(cr, np.float32)
    grid = grid_of(vs, cr)
    lo = cr32[:3].astype(np.float64)
    span = grid * vs32.astype(np.float64)
    half = background // 2
    uni = lo - 0.1 * span + rng.random((half, 3)) * 1.2 * span
    centres = lo + (rng.integers(0, grid, (12, 3)) + 0.5) * vs32
    clu = centres[rng.integers(0, 12, background - half)] + (rng.random((background - half, 3)) - 0.5) * 0.8 * vs32
    probes = []
    for axis in range(3):
        vals = face_values(vs32[axis], cr32[axis], cr32[3 + axis], grid[axis])
        p = (lo + rng.random((2 * len(vals), 3)) * span).astype(np.float32)
        p[:, axis] = np.repeat(vals, 2)
        probes.append(p)
    probes = np.concatenate(probes)
    xyz = np.concatenate([uni.astype(np.float32), clu.astype(np.float32), probes])
    is_probe = np.zeros(len(xyz), bool)
    is_probe[-len(probes):] = True
    pts = np.concatenate([xyz, rng.standard_normal((len(xyz), nf - 3)).astype(np.float32)], axis=1)
    order = rng.permutation(len(pts))
    return np.ascontiguousarray(pts[order]), is_probe[order]


def cells_f64(pts, vs, cr):
    """floor((float64(p) - float64(lo)) / float64(vs)) with lo, vs the fp32 values ->
    (coords [N, 3] int64 with -1 rows for points outside, decided [N] bool).  A point is decided
    when no axis' float64 quotient q lies within 4 * 2^-24 * max(1, |q|) of an integer.  The fp32
    subtract and the fp32 divide each add a relative error of at most 2^-24, so the fp32 quotient
    is within about 2 * 2^-24 * |q| of q (one denormal when it underflows); twice that is the
    margin, and anything closer to a face is left to the bit-exact oracle.  Non-finite
    coordinates are decided: outside."""
    vs32, cr32 = np.asarray(vs, np.float32), np.asarray(cr, np.float32)
    grid = grid_of(vs, cr)
    with np.errstate(invalid="ignore", over="ignore"):
        q = (pts[:, :3].astype(np.float64) - cr32[:3].astype(np.float64)) / vs32.astype(np.float64)
        fin = np.isfinite(q)
        cell = np.floor(np.where(fin, q, -1.0))
        inside = fin & (cell >= 0) & (cell < grid)
        near = fin & (np.abs(q - np.round(q)) <= 4 * 2.0 ** -24 * np.maximum(1.0, np.abs(q)))
        # far outside the grid no rounding can bring a point back in
        near &= (q > -1.5) & (q < grid + 1.5)
    coords = np.where(inside.all(1)[:, None], np.clip(cell, -1, 2 ** 31 - 1), -1).astype(np.int64)
    return coords, ~near.any(1)


def caps_for(case, pts, vs, cr):
    """(max_points, max_voxels, distinct occupied cells) of a CAPS case for this cloud."""
    dyn = oracle.dynamic_voxelize(pts, vs, cr)
    distinct = len(np.unique(dyn[dyn[:, 0] >= 0], axis=0))
    if case == "p1_v7":
        return 1, 7, distinct
    if case == "p10_binding":
        return 10, max(distinct // 2, 1), distinct
    return 64, distinct + 5, distinct


def run_hard(cuda, pts, vs, cr, mp, mv):
    from bevfusion_b200.voxelize import voxelization
    v, c, n = voxelization(torch.from_numpy(pts).to(cuda), list(vs), list(cr), mp, mv, True)
    return v, c, n


@pytest.mark.parametrize("caps", CAPS)
@pytest.mark.parametrize("nf", WIDTHS)
@pytest.mark.parametrize("geom", list(GEOMS))
def test_hard_and_fused_mean_on_cell_faces(cuda, geom, nf, caps):
    from bevfusion_b200 import _C
    from bevfusion_b200.voxelize import voxelize_mean, voxelize_mean_fused
    vs, cr, _ = GEOMS[geom]
    pts, _ = boundary_cloud(vs, cr, nf, seed=len(geom) * 100 + nf)
    mp, mv, distinct = caps_for(caps, pts, vs, cr)
    gv, gc, gn, gm = oracle.hard_voxelize(pts, vs, cr, mp, mv)
    assert gm == min(mv, distinct)
    if caps == "p10_binding" and geom != "single":
        assert mv < distinct and (gn == mp).any()            # both caps bind
    v, c, n = run_hard(cuda, pts, vs, cr, mp, mv)
    assert c.shape[0] == gm
    assert np.array_equal(c.cpu().numpy(), gc), "voxel coords / order differ"
    assert np.array_equal(n.cpu().numpy(), gn), "points-per-voxel differ"
    assert np.array_equal(v.cpu().numpy().view(np.int32), gv.view(np.int32)), "payload bits differ"
    slots = torch.arange(mp, device=cuda).view(1, mp, 1) >= n.view(-1, 1, 1)
    assert not bool((v.view(torch.int32) != 0)[slots.expand_as(v)].any()), "slots past the count are not zero"

    p = torch.from_numpy(pts).to(cuda)
    if nf > 8:
        with pytest.raises(_C.BevB200Error, match="bad point tensor shape"):
            voxelize_mean_fused(p, vs, cr, mp, mv)
        return
    feats, coords4 = voxelize_mean(v, c, n, batch_idx=2)
    f2, c2, n2 = voxelize_mean_fused(p, vs, cr, mp, mv, batch_idx=2)
    assert torch.equal(c2, coords4) and torch.equal(n2, n)
    assert torch.equal(c2[:, 1:], c) and bool((c2[:, 0] == 2).all())
    assert torch.equal(f2.view(torch.int32), feats.view(torch.int32)), "fused mean != voxel_mean of the hard output"
    rows = gv.astype(np.float64)                             # unused slots are zero
    ref = rows.sum(1) / gn[:, None]
    oracle.assert_within(f2.cpu().numpy(), ref, oracle.fp32_sum_bound(np.abs(rows).sum(1), gn[:, None], mean_of=ref),
                         "fused mean")
    f3, c3, n3, count = voxelize_mean_fused(p, vs, cr, mp, mv, batch_idx=2, sync=False)
    assert f3.shape[0] == mv and int(count.item()) == gm
    assert torch.equal(f3[:gm].view(torch.int32), f2.view(torch.int32))
    assert torch.equal(c3[:gm], c2) and torch.equal(n3[:gm], n2)


@pytest.mark.parametrize("nf", [3, 5, 45])
@pytest.mark.parametrize("geom", list(GEOMS))
def test_dynamic_on_cell_faces_vs_oracle_and_float64(cuda, geom, nf):
    from bevfusion_b200.voxelize import voxelization
    vs, cr, exact = GEOMS[geom]
    pts, is_probe = boundary_cloud(vs, cr, nf, seed=7 + nf)
    coors = voxelization(torch.from_numpy(pts).to(cuda), vs, cr, -1, -1, True).cpu().numpy()
    assert np.array_equal(coors, oracle.dynamic_voxelize(pts, vs, cr))
    assert ((coors < 0).all(1) | (coors >= 0).all(1)).all()                # a dropped point is -1 in every column
    ref, decided = cells_f64(pts, vs, cr)
    if exact:
        decided[:] = True
    else:
        assert 0 < (~decided).sum() <= is_probe.sum()        # the faces were reached, and only by the probes
    assert np.array_equal(coors[decided], ref[decided]), "cell index differs from float64 away from every face"
    # hard voxelization without a binding cap sees exactly the valid dynamic cells
    valid = np.unique(coors[coors[:, 0] >= 0], axis=0)
    c = run_hard(cuda, pts, vs, cr, 3, len(valid) + 1)[1].cpu().numpy()
    assert np.array_equal(np.unique(c, axis=0), valid) and len(c) == len(valid)


def test_range_faces_exact_geometry(cuda):
    """p == lo is kept in cell 0, p == hi is dropped, the last ulp below hi is in cell grid - 1,
    -0.0 is cell 0 and the first denormal below lo is dropped."""
    from bevfusion_b200.voxelize import voxelization
    vs, cr, _ = GEOMS["exact"]
    below = np.nextafter(np.float32(8.0), np.float32(0))
    tiny = np.float32(1e-45)
    xs = np.array([0.0, -0.0, tiny, -tiny, 8.0, below, 0.5, np.nextafter(np.float32(0.5), np.float32(0))], np.float32)
    pts = np.full((len(xs), 4), 0.1, np.float32)
    pts[:, 0] = xs
    coors = voxelization(torch.from_numpy(pts).to(cuda), vs, cr, -1, -1, True).cpu().numpy()
    assert coors[:, 0].tolist() == [0, 0, 0, -1, -1, 15, 1, 0]
    assert np.array_equal(coors, oracle.dynamic_voxelize(pts, vs, cr))


def test_pin_negative_quotient_rounding_to_minus_zero_is_cell_zero(cuda):
    """A point a denormal below range_min whose fp32 quotient rounds to -0.0 is kept, in cell 0:
    floor(-0.0) = -0.0 and -0.0 >= 0.  The reference's `int c = floor(..); c < 0` reads it the same
    way.  (float64 would call it cell -1; fp32 is the definition.)"""
    from bevfusion_b200.voxelize import voxelization
    vs, cr = [4.0, 4.0, 4.0], [0.0, 0.0, 0.0, 8.0, 8.0, 8.0]
    tiny = np.float32(1e-45)
    pts = np.array([[-tiny, 1.0, 1.0, 0.0], [1.0, -tiny, 5.0, 0.0], [np.float32(-4e-45), 1.0, 1.0, 0.0]], np.float32)
    with np.errstate(under="ignore"):
        assert np.signbit(pts[0, 0] / np.float32(4.0)) and pts[0, 0] / np.float32(4.0) == 0.0
        assert pts[2, 0] / np.float32(4.0) < 0                                  # -1 denormal: still negative
    coors = voxelization(torch.from_numpy(pts).to(cuda), vs, cr, -1, -1, True).cpu().numpy()
    assert coors.tolist() == [[0, 0, 0], [0, 0, 1], [-1, -1, -1]]
    assert np.array_equal(coors, oracle.dynamic_voxelize(pts, vs, cr))
    v, c, n = run_hard(cuda, pts, vs, cr, 2, 4)
    assert c.tolist() == [[0, 0, 0], [0, 0, 1]] and n.tolist() == [1, 1]


def _reference_glue(pts, vox, reduce):
    """BEVFusion.voxelize (bevfusion.py:169-197) restated in torch on top of the module."""
    import torch.nn.functional as F
    feats, coords, sizes = [], [], []
    for k, p in enumerate(pts):
        ret = vox(p)
        if isinstance(ret, tuple):
            f, c, n = ret
            sizes.append(n)
        else:
            f, c = p, ret
        feats.append(f)
        coords.append(F.pad(c, (1, 0), mode="constant", value=k))
    feats, coords = torch.cat(feats), torch.cat(coords)
    if sizes:
        sizes = torch.cat(sizes)
        if reduce:
            feats = feats.sum(dim=1) / sizes.type_as(feats).view(-1, 1)
    return feats, coords, sizes


@pytest.mark.parametrize("nf", [5, 45])
@pytest.mark.parametrize("kind", ["hard", "dynamic"])
@pytest.mark.parametrize("reduce", [True, False])
@pytest.mark.parametrize("training", [False, True])
def test_voxelize_batch_branches(cuda, training, reduce, kind, nf):
    """Every branch of voxelize_batch on a batch [cloud, empty, 3-point cloud, cloud]: the fused
    mean (rows of <= 8 columns), Voxelization + voxel_mean (wider rows), no reduce, and a dynamic
    module, in eval and training mode (different caps, both binding)."""
    from bevfusion_b200.voxelize import Voxelization, voxelize_batch
    vs, cr, _ = GEOMS["c3"]
    clouds = [boundary_cloud(vs, cr, nf, seed=s)[0] for s in (1, 2)]
    inside = clouds[1][(oracle.dynamic_voxelize(clouds[1], vs, cr) >= 0).all(1)]
    clouds = [clouds[0], clouds[0][:0], inside[:3].copy(), clouds[1]]
    three = oracle.hard_voxelize(clouds[2], vs, cr, 10, 10)[3]
    pts = [torch.from_numpy(c).to(cuda) for c in clouds]
    train_cap, eval_cap = 200, 400
    vox = Voxelization(vs, cr, 10 if kind == "hard" else -1, (train_cap, eval_cap)).train(training)
    feats, coords, sizes = voxelize_batch(pts, vox, voxelize_reduce=reduce)
    rf, rc, rs = _reference_glue(pts, vox, reduce)
    assert torch.equal(coords, rc) and coords.dtype == torch.int32
    assert sorted(set(coords[:, 0].tolist())) == [0, 2, 3]
    if kind == "dynamic":
        assert sizes == [] and torch.equal(feats.view(torch.int32), torch.cat(pts).view(torch.int32))
        return
    cap = train_cap if training else eval_cap
    assert torch.equal(sizes, rs) and coords.shape[0] == 2 * cap + three       # both clouds hit the cap
    if not reduce:
        assert torch.equal(feats, rf) and feats.shape[1:] == (10, nf)
        return
    # torch's sum(dim=1) adds the 10 slots in its own order: compare both with float64
    rows = torch.cat([vox(p)[0] for p in pts]).double().cpu().numpy()
    n = rs.cpu().numpy()[:, None]
    ref = rows.sum(1) / n
    bound = oracle.fp32_sum_bound(np.abs(rows).sum(1), n, mean_of=ref)
    oracle.assert_within(feats.cpu().numpy(), ref, bound, "voxelize_batch mean")
    oracle.assert_within(rf.cpu().numpy(), ref, bound, "torch glue mean")


@pytest.mark.parametrize("vs,cr", [
    ([0.0, 0.5, 0.5], [0, 0, 0, 4, 4, 2]),
    ([0.5, -0.5, 0.5], [0, 0, 0, 4, 4, 2]),
    ([0.5, 0.5, float("nan")], [0, 0, 0, 4, 4, 2]),
    ([0.5, 0.5, 0.5], [0, 0, 0, 4, 0, 2]),               # hi == lo
    ([0.5, 0.5, 0.5], [0, 0, 0, -4, 4, 2]),              # hi < lo
])
def test_bad_grids_are_refused_on_the_host(cuda, vs, cr):
    from bevfusion_b200 import _C
    from bevfusion_b200.voxelize import voxelization, voxelize_mean_fused
    pts = torch.rand(64, 4, device=cuda)
    with pytest.raises(_C.BevB200Error, match="bad voxel grid"):
        voxelization(pts, vs, cr, 5, 10, True)
    with pytest.raises(_C.BevB200Error, match="bad voxel grid"):
        voxelization(pts, vs, cr, -1, -1, True)
    with pytest.raises(_C.BevB200Error, match="bad voxel grid"):
        voxelize_mean_fused(pts, vs, cr, 5, 10)


def test_boundary_cloud_vs_reference_cuda_kernel(cuda):
    """The C3 boundary cloud through the reference's own deterministic CUDA voxelizer.  Rows with a
    NaN coordinate are left out: the reference's CUDA kernel converts floor(NaN) to int 0 and files
    them in cell 0, its CPU kernel drops them; this library drops them (test_voxelize_gpu.py,
    test_edge_cases)."""
    ref = ref_module("voxel_layer_ref")
    if ref is None:
        pytest.skip("oracle/_ref not built")
    vs, cr, _ = GEOMS["c3"]
    pts, _ = boundary_cloud(vs, cr, 5, seed=11, background=20000)
    pts = np.ascontiguousarray(pts[~np.isnan(pts[:, :3]).any(1)])
    p = torch.from_numpy(pts).to(cuda)
    mp, mv = 10, 8000
    voxels = torch.zeros(mv, mp, 5, device=cuda)
    coors = torch.zeros(mv, 3, dtype=torch.int32, device=cuda)
    num = torch.zeros(mv, dtype=torch.int32, device=cuda)
    m = ref.hard_voxelize(p, voxels, coors, num, vs, cr, mp, mv, 3, True)
    v, c, n = run_hard(cuda, pts, vs, cr, mp, mv)
    assert c.shape[0] == m
    assert torch.equal(c, coors[:m]) and torch.equal(n, num[:m]) and torch.equal(v, voxels[:m])
