"""GPU: the rotated BEV overlap (csrc/rot_overlap.cuh) on the box families where polygon clipping goes wrong
(tests/box_families.py): touching and nested boxes, collinear edges at any yaw, yaw + pi, a square turned by
pi / 2, yaws one ulp apart, zero-width boxes.  boxes_iou_bev and boxes_overlap_bev against the float64 checker on
the same fp32 boxes, in both argument orders; NMS keep lists on lists of these pairs; the TransFusion assignment's
cost and max_overlaps on proposals equal to, slid from, touching or stacked on their gt, against a float64
restatement; and, printed only, the reference's iou3d_cuda on the same pairs."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import box_families as F  # noqa: E402
import nms_oracle as O  # noqa: E402
from conftest import ref_module  # noqa: E402
from test_transfusion_assign_gpu import CFG, ref_cost  # noqa: E402

pytestmark = pytest.mark.gpu
N = 2000          # pairs per family
TOL = 1e-4        # largest |IoU - float64 IoU|; the overlap may be off by TOL times the larger box's area


@pytest.fixture(scope="module")
def fams():
    out = {}
    for name, (A, B, _, _) in F.families(np.random.default_rng(2024), N).items():
        A32, B32 = A.astype(np.float32), B.astype(np.float32)
        a64, b64 = A32.astype(np.float64), B32.astype(np.float64)
        out[name] = (A32, B32, np.array([O.iou_bev(p, q) for p, q in zip(a64, b64)]),
                     np.array([O.overlap_bev(p, q) for p, q in zip(a64, b64)]))
    return out


def pairs(fn, A, B, dev):
    """fn on the pairs (A[i], B[i]) -> [n] numpy."""
    a, b = torch.from_numpy(A).to(dev), torch.from_numpy(B).to(dev)
    return fn(a, b).diagonal().cpu().numpy()


def area(X):
    return (X[:, 2].astype(np.float64) - X[:, 0]) * (X[:, 3].astype(np.float64) - X[:, 1])


def test_iou_and_overlap_on_families(cuda, fams):
    from bevfusion_b200 import iou3d
    bad = {}
    for name, (A, B, iou64, ov64) in fams.items():
        scale = np.maximum(area(A), area(B))
        for X, Y in ((A, B), (B, A)):
            ei = np.abs(pairs(iou3d.boxes_iou_bev, X, Y, cuda) - iou64)
            eo = np.abs(pairs(iou3d.boxes_overlap_bev, X, Y, cuda) - ov64)
            n = int(((ei > TOL) | (eo > TOL * scale)).sum())
            bad[name] = bad.get(name, 0) + n
            print("%-15s %s  pairs off: %4d of %d  largest IoU error %.3g" % (name, "ab" if X is A else "ba", n,
                                                                              len(A), ei.max()))
    assert not any(bad.values()), bad


def test_families_cover_the_geometry(fams):
    """The families hold what they are named for: overlapping slides, touching pairs, yaws beyond pi."""
    for name in ("touch_end", "touch_side", "touch_corner", "zero_width"):
        assert fams[name][2].max() <= 1e-4, name
    for name in ("slide", "yaw_pi", "square_half_pi", "nested"):
        assert np.median(fams[name][2]) > 0.2, name
    assert np.median(fams["yaw_ulp"][2]) > 0.999
    yaw = np.concatenate([f[0][:, 4] for f in fams.values()])
    assert (np.abs(yaw) > np.pi).any() and (np.abs(yaw) == np.float32(np.pi / 2)).any()


# ---- NMS on lists of these pairs ---------------------------------------------------------------------------------

NMS_PAIRS = 500


@pytest.fixture(scope="module")
def nms_lists(fams):
    """Per family: its first NMS_PAIRS pairs as one list and the list's float64 IoU matrix."""
    out = {}
    for name, (A, B, _, _) in fams.items():
        boxes = np.concatenate([A[:NMS_PAIRS], B[:NMS_PAIRS]])
        out[name] = (boxes, O.iou_matrix(boxes, boxes))
    return out


def clear_list(boxes, iou, thresh, rng):
    """The list less one box of every pair whose float64 IoU is within 1e-3 of thresh, distinct scores, and the
    float64 checker's keep list."""
    keep = np.ones(len(boxes), bool)
    for i, j in zip(*np.nonzero(np.triu(np.abs(iou - thresh) < 1e-3, 1))):
        if keep[i] and keep[j]:
            keep[j] = False
    boxes, iou = boxes[keep], iou[keep][:, keep]
    n = len(boxes)
    scores = ((rng.permutation(n) + rng.uniform(0.1, 0.9, n)) / n).astype(np.float32)
    order = O.sort_desc(scores)
    return boxes, scores, order[O.greedy(iou[order][:, order], thresh)]


@pytest.mark.parametrize("thresh", [0.01, 0.2, 0.5])
def test_nms_on_families(cuda, nms_lists, thresh):
    from bevfusion_b200 import iou3d
    rng = np.random.default_rng(int(thresh * 100))
    lists = [clear_list(boxes, iou, thresh, rng) for boxes, iou in nms_lists.values()]
    for (boxes, scores, want), name in zip(lists, nms_lists):
        got = iou3d.nms_gpu(torch.from_numpy(boxes).to(cuda), torch.from_numpy(scores).to(cuda), thresh)
        assert np.array_equal(got.cpu().numpy(), want), (name, thresh)
    nmax = max(len(b) for b, _, _ in lists)
    Bx = np.zeros((len(lists), nmax, 5), np.float32)
    Sc = np.full((len(lists), nmax), 5.0, np.float32)              # pads past each count may hold anything
    for i, (b, s, _) in enumerate(lists):
        Bx[i, :len(b)], Sc[i, :len(s)] = b, s
    counts = torch.tensor([len(b) for b, _, _ in lists], dtype=torch.int32, device=cuda)
    keep, kc = iou3d.nms_batched(torch.from_numpy(Bx).to(cuda), torch.from_numpy(Sc).to(cuda), counts, "rotate",
                                 thresh)
    for i, (_, _, want) in enumerate(lists):
        assert int(kc[i]) == len(want) and np.array_equal(keep[i, :len(want)].cpu().numpy(), want), i


# ---- the TransFusion assignment ----------------------------------------------------------------------------------

P_PER_GT = 5


def assignment_case(rng, G):
    """G gt boxes (x, y, z, dx, dy, dz, yaw) and P_PER_GT proposals for each: equal to it, slid along one of its
    axes, touching it end to end or side by side, stacked on it or under it touching, and stacked overlapping it
    in z (slid in half the cases)."""
    cx, cy = F.centres(rng, G)
    w, l = F.sizes(rng, G)
    r = F.yaws(rng, G)
    z, dz = rng.uniform(-3, 1, G), rng.uniform(0.5, 3, G)
    gt = np.stack([cx, cy, z, w, l, dz, r], 1)

    def box(px, py, zz, dd):
        c, s = np.cos(r), np.sin(r)
        return np.stack([cx + px * c + py * s, cy - px * s + py * c, zz, w, l, dd, r], 1)

    px, py, _, _ = F.slide_offset(rng, G, w, l)
    along_x = rng.uniform(size=G) < 0.5
    sign = rng.choice([-1.0, 1.0], G)
    dz2 = rng.uniform(0.5, 3, G)
    above = rng.uniform(size=G) < 0.5
    half = rng.uniform(size=G) < 0.5
    props = [
        gt.copy(),
        box(px, py, z, dz),
        box(np.where(along_x, sign * w, 0.0), np.where(along_x, 0.0, sign * l), z, dz),
        box(0.0, 0.0, np.where(above, z + dz, z - dz2), np.where(above, dz, dz2)),
        box(np.where(half, px, 0.0), np.where(half, py, 0.0), z + rng.uniform(-0.9, 0.9, G) * dz, dz),
    ]
    return gt.astype(np.float32), np.stack(props, 1).reshape(-1, 7).astype(np.float32)


def test_assignment_on_families(cuda):
    from bevfusion_b200 import transfusion_assign as TA
    rng = np.random.default_rng(5)
    G, K = 40, 10
    P = G * P_PER_GT
    worst_cost = worst_iou = 0.0
    for sample in range(4):
        gt, dec = assignment_case(rng, G)
        gl = torch.from_numpy(rng.integers(0, K, G).astype(np.int64)).to(cuda)
        heat = torch.from_numpy(rng.normal(0, 2, (1, K, P)).astype(np.float32)).to(cuda)
        g, d = torch.from_numpy(gt).to(cuda), torch.from_numpy(dec).to(cuda)
        coder = dict(pc_range=[0.0, 0.0], voxel_size=[1.0, 1.0], out_size_factor=1, code_size=8)
        _, ex = TA._run(heat, None, None, None, None, d[None], g[None], gl[None].int(),
                        torch.tensor([G], dtype=torch.int32, device=cuda), K, P, CFG, coder, extras=True)
        want_cost, iou64 = ref_cost(d, heat[0], g, gl)
        iou64 = iou64.cpu().numpy()
        designed = iou64.reshape(G, P_PER_GT, G)[np.arange(G), :, np.arange(G)]   # each proposal with its gt
        # equal boxes: 1 up to the fp32 rounding of x -+ dx / 2 against dx; stacked touching: 0 up to that of z + dz
        assert np.abs(designed[:, 0] - 1).max() < 1e-3 and designed[:, 3].max() < 1e-6
        worst_cost = max(worst_cost, (ex["cost"][0] - want_cost).abs().max().item())
        res = TA.HungarianAssigner3D(cls_cost=dict(type="FocalLossCost", gamma=2.0, alpha=0.25, weight=0.15),
                                     reg_cost=dict(type="BBoxBEVL1Cost", weight=0.25),
                                     iou_cost=dict(type="IoU3DCost", weight=0.25)).assign(d, g, gl, heat, CFG)
        inds = res.gt_inds.cpu().numpy()
        assert np.array_equal(inds, ex["gt_inds"][0].cpu().numpy())
        matched = np.nonzero(inds > 0)[0]
        assert len(matched) == G
        mo = np.zeros(P)
        mo[matched] = iou64[matched, inds[matched] - 1]
        for got in (res.max_overlaps, ex["max_overlaps"][0]):
            worst_iou = max(worst_iou, np.abs(got.cpu().numpy() - mo).max())
    print("largest |cost - float64 restatement| %.3g, |max_overlaps - float64| %.3g" % (worst_cost, worst_iou))
    assert worst_iou <= TOL and worst_cost <= 0.25 * TOL + 1e-6


# ---- the reference's iou3d_cuda, for comparison --------------------------------------------------------------------

def test_reference_iou3d_on_families(cuda, fams):
    ref = ref_module("iou3d_cuda_ref")
    if ref is None:
        pytest.skip("oracle/_ref has no reference iou3d_cuda build")

    def ref_iou(a, b):
        out = torch.zeros((a.shape[0], b.shape[0]), device=a.device)
        ref.boxes_iou_bev_gpu(a, b, out)
        return out

    for name, (A, B, iou64, _) in fams.items():
        e = np.abs(pairs(ref_iou, A, B, cuda) - iou64)
        print("reference iou3d_cuda  %-15s pairs with IoU error above %g: %4d of %d  largest %.3g" %
              (name, TOL, int((e > TOL).sum()), len(A), e.max()))
