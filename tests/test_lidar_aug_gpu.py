"""GPU: GlobalRotScaleTrans + RandomFlip3D + the range and name filters on the device, with no tolerance.

- LiDAR: SweepStore.assemble(aug=) on the reference's own pipeline cases (golden/lidar_aug_tiny.npz: every flip pair,
  rot_lim [0, 0], is_train False), bit-equal to its points; the boxes (LidarAug.boxes), masks (flip_masks) and the
  block's matrix / extra_rots / extra_trans bit-equal to its outputs.
- Radar: RadarSweepStore.assemble(aug=) on seeded frames equal to the oracle applied to the unaugmented cloud.
- assemble(aug=None) and a block of disabled records equal the plain path; a graph of write_frame-free launches
  replayed after new write() calls equals the eager calls.
- centerhead_targets_batched on the device-augmented boxes equals the targets of the host-augmented ones; rebuild_
  with LidarAug.extra_* equals from_cameras with the reference's matrix."""
import numpy as np
import pytest
import torch

import lidar_aug_oracle as O
import radar_sweeps_oracle as RO

pytestmark = pytest.mark.gpu

CASES = ["flip00", "flip01", "flip10", "flip11", "rot0", "test", "empty"]


@pytest.fixture(scope="module")
def z(golden_dir):
    import os
    return np.load(os.path.join(golden_dir, "lidar_aug_tiny.npz"))


def same(a, b):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return O.count_diff(a, b) == 0


def draw_of(z, case):
    from bevfusion_b200.lidar_aug import LidarAugDraw
    scale, theta, trans, fh, fv = O.draw_tuple(z[case + "_draw"])
    if scale is None:
        theta = trans = None
    return LidarAugDraw(scale, theta, trans, bool(fh), bool(fv))


def lidar_store(cuda, clouds, max_batch=4):
    from bevfusion_b200.lidar_sweeps import SweepStore
    store = SweepStore(len(clouds), max(max(len(c) for c in clouds), 1), 5, cuda, max_batch=max_batch, max_entries=1)
    for k, c in enumerate(clouds):
        store.put(k, c)
    return store


def lidar_assemble(store, slots, aug=None, **kw):
    return store.assemble([(s, []) for s in slots], 5, pad_empty_sweeps=False,
                          point_cloud_range=O.POINT_CLOUD_RANGE, aug=aug, **kw)


def padded(boxes, labels, cuda):
    from bevfusion_b200.head_targets import pad_gt
    return pad_gt([torch.from_numpy(np.ascontiguousarray(b)) for b in boxes],
                  [torch.from_numpy(np.asarray(l, np.int32)).to(cuda) for l in labels])


@pytest.mark.parametrize("case", CASES)
def test_bit_equal_to_the_reference_pipeline(cuda, z, case):
    from bevfusion_b200.lidar_aug import LidarAug
    d = draw_of(z, case)
    aug = LidarAug(1, cuda)
    aug.write([d])
    pts = lidar_assemble(lidar_store(cuda, [z[case + "_points_in"]]), [0], aug)[0]
    assert same(pts, z[case + "_points"])
    boxes_in = z[case + "_boxes_in"]
    pb, pl, pc = padded([boxes_in], [z[case + "_labels_in"]], cuda)
    ob, ol, oc, st = aug.boxes(pb, pl, pc, O.POINT_CLOUD_RANGE, O.OBJECT_CLASSES)
    n = int(oc[0])
    assert int(st[0]) == 0 and n == len(z[case + "_boxes"])
    assert same(ob[0, :n], z[case + "_boxes"]) and np.array_equal(ol[0, :n].cpu().numpy(), z[case + "_labels"])
    assert not ob[0, n:].any() and not ol[0, n:].any()
    masks = torch.from_numpy(z[case + "_masks_in"]).to(cuda)[None]
    assert np.array_equal(aug.flip_masks(masks)[0].cpu().numpy(), z[case + "_masks"])
    m = z[case + "_matrix"]
    assert same(aug.matrix[0], m) and same(aug.extra_rots[0], m[:3, :3]) and same(aug.extra_trans[0], m[:3, 3])


def radar_frame(cuda, seed, B, rows=(40, 125)):
    from bevfusion_b200.radar_sweeps import RadarSweepStore
    rng = np.random.default_rng(seed)
    raws = [RO.radar_sweep(rng, int(rng.integers(*rows))) for _ in range(3 * B)]
    poses = [RO.radar_pose(rng, k % 5) for k in range(3 * B)]
    store = RadarSweepStore(len(raws), max(len(r) for r in raws), cuda, max_batch=4, max_entries=3)
    for k, r in enumerate(raws):
        store.put(k, r)
    samples = [[(3 * b + j, poses[3 * b + j][0], poses[3 * b + j][1], 0.05 * j) for j in range(3)] for b in range(B)]
    return store, samples


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("use_dim", [RO.SHIPPED_USE_DIM, [0, 1, 2, 8, 9], [0, 1, 2, 5, 8, 9, 18, 3]])
def test_radar_equals_the_oracle(cuda, B, use_dim):
    from bevfusion_b200.lidar_aug import LidarAug, GlobalRotScaleTrans, RandomFlip3D, draw_sample
    store, samples = radar_frame(cuda, 7 + B, B)
    plain = store.assemble(samples, use_dim, compensate_velocity=True, bev_range=None)
    rng = np.random.RandomState(B)
    draws = [draw_sample(GlobalRotScaleTrans(O.SHIPPED_SCALE, O.SHIPPED_ROTATE, O.SHIPPED_TRANSLATE, True, rng=rng),
                         RandomFlip3D(rng=rng)) for _ in range(B)]
    aug = LidarAug(4, cuda)
    aug.write(draws)
    got = store.assemble(samples, use_dim, compensate_velocity=True, aug=aug)
    for b in range(B):
        r = O.augment_radar(plain[b].cpu().numpy(), tuple(draws[b]))
        assert same(got[b], r[O.in_range_bev(r[:, :2], O.RADAR_BEV_RANGE)])


def test_no_aug_and_disabled_records_equal_the_plain_path(cuda, z):
    from bevfusion_b200.lidar_aug import LidarAug
    clouds = [z[c + "_points_in"] for c in CASES[:4]]
    store = lidar_store(cuda, clouds)
    plain = lidar_assemble(store, range(4))
    off = LidarAug(4, cuda)
    off.write([None] * 4)            # every record disabled
    for got in (lidar_assemble(store, range(4), None), lidar_assemble(store, range(4), off)):
        assert all(same(g, p.cpu().numpy()) for g, p in zip(got, plain))
    rstore, samples = radar_frame(cuda, 3, 4)
    rplain = rstore.assemble(samples, RO.SHIPPED_USE_DIM, compensate_velocity=True)
    rgot = rstore.assemble(samples, RO.SHIPPED_USE_DIM, compensate_velocity=True, aug=off)
    assert all(same(g, p.cpu().numpy()) for g, p in zip(rgot, rplain))
    # boxes with a NULL record (augment=False) and with disabled records: the filters only
    b, l = z["flip00_boxes_in"], z["flip00_labels_in"]
    pb, pl, pc = padded([b], [l], cuda)
    want_b, want_l = O.boxes_filtered(b, l, (None, None, None, 0, 0))
    for ob, ol, oc, st in (off.boxes(pb, pl, pc, O.POINT_CLOUD_RANGE, 10, augment=False),
                           off.boxes(pb, pl, pc, O.POINT_CLOUD_RANGE, 10)):
        n = int(oc[0])
        assert n == len(want_b) and same(ob[0, :n], want_b) and np.array_equal(ol[0, :n].cpu().numpy(), want_l)


def test_graph_replay_with_new_draws_equals_eager_calls(cuda, z):
    from bevfusion_b200.lidar_aug import LidarAug, GlobalRotScaleTrans, RandomFlip3D, draw_sample
    clouds = [z[c + "_points_in"] for c in CASES[:4]]
    store = lidar_store(cuda, clouds)
    batch, F, bound = store.write_frame([(s, []) for s in range(4)], 5, pad_empty_sweeps=False,
                                        point_cloud_range=O.POINT_CLOUD_RANGE)
    pb, pl, pc = padded([z[c + "_boxes_in"] for c in CASES[:4]], [z[c + "_labels_in"] for c in CASES[:4]], cuda)
    aug = LidarAug(4, cuda)
    rng = np.random.RandomState(5)
    new_draws = lambda: [draw_sample(GlobalRotScaleTrans(O.SHIPPED_SCALE, O.SHIPPED_ROTATE, O.SHIPPED_TRANSLATE,
                                                         True, rng=rng), RandomFlip3D(rng=rng)) for _ in range(4)]
    aug.write(new_draws())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm up outside the capture
        store.launch(batch, F, bound, aug)
        aug.boxes(pb, pl, pc, O.POINT_CLOUD_RANGE, 10)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pts, counts, status = store.launch(batch, F, bound, aug)
        ob, ol, oc, bst = aug.boxes(pb, pl, pc, O.POINT_CLOUD_RANGE, 10)
    for _ in range(3):
        draws = new_draws()
        aug.write(draws)
        g.replay()
        torch.cuda.synchronize()
        e_pts, e_counts, _ = store.launch(batch, F, bound, aug)
        e_b, e_l, e_c, _ = aug.boxes(pb, pl, pc, O.POINT_CLOUD_RANGE, 10)
        assert torch.equal(counts, e_counts) and int(status[0]) == 0 and torch.equal(oc, e_c)
        for b in range(4):
            n = int(counts[b])
            assert torch.equal(pts[b, :n].view(torch.int32), e_pts[b, :n].view(torch.int32))
            p = O.augment_points(clouds[b], tuple(draws[b]), exact=True)
            assert same(pts[b, :n], p[O.in_range_3d(p, O.POINT_CLOUD_RANGE)])
        assert torch.equal(ob.view(torch.int32), e_b.view(torch.int32)) and torch.equal(ol, e_l)


def test_centerhead_targets_from_device_augmented_boxes(cuda, z):
    from bevfusion_b200 import head_targets as H
    from bevfusion_b200.lidar_aug import LidarAug
    tasks = [dict(num_class=1, class_names=["car"]), dict(num_class=2, class_names=["truck", "construction_vehicle"]),
             dict(num_class=2, class_names=["bus", "trailer"]), dict(num_class=1, class_names=["barrier"]),
             dict(num_class=2, class_names=["motorcycle", "bicycle"]),
             dict(num_class=2, class_names=["pedestrian", "traffic_cone"])]
    cfg = dict(point_cloud_range=O.POINT_CLOUD_RANGE, grid_size=[1440, 1440, 41], voxel_size=[0.075, 0.075, 0.2],
               out_size_factor=8, dense_reg=1, gaussian_overlap=0.1, max_objs=500, min_radius=2)
    cases = CASES[:4]
    aug = LidarAug(4, cuda)
    aug.write([draw_of(z, c) for c in cases])
    pb, pl, pc = padded([z[c + "_boxes_in"] for c in cases], [z[c + "_labels_in"] for c in cases], cuda)
    ob, ol, oc, _ = aug.boxes(pb, pl, pc, O.POINT_CLOUD_RANGE, O.OBJECT_CLASSES)
    host = [O.boxes_filtered(z[c + "_boxes_in"], z[c + "_labels_in"], O.draw_tuple(z[c + "_draw"])) for c in cases]
    hb, hl, hc = padded([h[0] for h in host], [h[1] for h in host], cuda)
    dev_t = H.centerhead_targets_batched(ob, ol, oc, tasks, cfg)
    host_t = H.centerhead_targets_batched(hb, hl, hc, tasks, cfg)
    for a_list, b_list in zip(dev_t, host_t):
        for a, b in zip(a_list, b_list):
            assert torch.equal(a, b)


def test_rebuild_with_the_block_equals_from_cameras_with_the_reference_matrix(cuda, z):
    from bevfusion_b200 import synthetic as S
    from bevfusion_b200.bev_pool import BEVPoolPlan
    from bevfusion_b200.lidar_aug import LidarAug
    from test_bev_pool_sync_free_gpu import assert_tables_equal, calib, frustum, rig
    cfg = S.CONFIGS["tiny"]
    fr = frustum(cuda, cfg)
    B = 2
    r = rig(cuda, cfg, B, seed=11)
    c = calib(r)
    dev = BEVPoolPlan.from_cameras(fr, *c[:5], cfg["xbound"], cfg["ybound"], cfg["zbound"], c[5], c[6], sync=False)
    aug = LidarAug(B, cuda)
    for cases in (["flip01", "flip10"], ["rot0", "flip11"]):
        aug.write([draw_of(z, k) for k in cases])
        dev.rebuild_(*c[:5], aug.extra_rots, aug.extra_trans)
        m = torch.from_numpy(np.stack([z[k + "_matrix"] for k in cases])).to(cuda)
        host = BEVPoolPlan.from_cameras(fr, *c[:5], cfg["xbound"], cfg["ybound"], cfg["zbound"],
                                        m[:, :3, :3].contiguous(), m[:, :3, 3].contiguous())
        assert_tables_equal(host, dev)


def test_an_unindexed_device_matches_its_tensors(cuda):
    from bevfusion_b200.lidar_aug import LidarAug
    from bevfusion_b200.lidar_sweeps import SweepStore
    aug = LidarAug(1, "cuda")
    aug.write([None])
    assert aug.device == torch.device("cuda", torch.cuda.current_device())
    b = torch.zeros((1, 2, 7), device=cuda)
    l = torch.zeros((1, 2), dtype=torch.int32, device=cuda)
    c = torch.ones((1,), dtype=torch.int32, device=cuda)
    assert int(aug.boxes(b, l, c, O.POINT_CLOUD_RANGE, 10)[2][0]) == 1
    store = SweepStore(1, 4, 5, "cuda", max_batch=1, max_entries=1)
    store.put(0, np.zeros((2, 5), np.float32))
    assert store.assemble([(0, [])], 5, pad_empty_sweeps=False, aug=aug)[0].shape == (2, 5)


def test_a_batch_past_the_last_write_raises(cuda, z):
    from bevfusion_b200.lidar_aug import LidarAug
    clouds = [z[c + "_points_in"] for c in CASES[:2]]
    store = lidar_store(cuda, clouds)
    aug = LidarAug(2, cuda)
    aug.write([draw_of(z, "flip01")])
    with pytest.raises(ValueError, match="write"):
        lidar_assemble(store, range(2), aug)
    pb, pl, pc = padded([z["flip00_boxes_in"]] * 2, [z["flip00_labels_in"]] * 2, cuda)
    with pytest.raises(ValueError, match="write"):
        aug.boxes(pb, pl, pc, O.POINT_CLOUD_RANGE, 10)
    with pytest.raises(ValueError, match="write"):
        aug.flip_masks(torch.zeros((2, 1, 4, 4), dtype=torch.bool, device=cuda))
    aug.boxes(pb, pl, pc, O.POINT_CLOUD_RANGE, 10, augment=False)     # the filters alone read no record
    aug.write([draw_of(z, "flip01"), None])
    got = lidar_assemble(store, range(2), aug)
    assert same(got[1], lidar_assemble(store, [1])[0].cpu().numpy())
