"""GPU: ObjectPaste in the sweep assemble kernels, with no tolerance.

- The reference's own cases (golden/object_paste_tiny.npz): paste only, paste + aug and paste + aug + range filter,
  bit-equal to the reference's cloud (and to the lidar_aug oracle applied to it).
- Rows exactly on a face and one ulp either side, +-0, +-inf and NaN rows (NaN removed when S >= 1, kept when S = 0),
  yaw at +-pi, caps that cut the pasted rows mid-tile, S = 0 beside S = max_paste with B = max_batch.
- A block of None draws and no block at all equal the plain aug launch; malformed blocks set BAD_PASTE and paste
  nothing; a graph replayed after new draws and new objects equals the eager calls; CenterHead targets from the
  merged, device-augmented boxes equal those of the host-augmented ones."""
import os

import numpy as np
import pytest
import torch

import lidar_aug_oracle as LA
import object_paste_oracle as O

pytestmark = pytest.mark.gpu

FRAMES = [("shipped", 0), ("exhaust", 0), ("exhaust", 1), ("exhaust", 2), ("many_gt", 0), ("empty_gt", 0),
          ("all_collide", 0), ("contains_gt", 0), ("pending", 0), ("epoch_gate", 0)]
f32 = np.float32


@pytest.fixture(scope="module")
def z(golden_dir):
    return O.load_fixture(os.path.join(golden_dir, "object_paste_tiny.npz"))


def same(a, b):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return O.count_diff(a, b) == 0


def db_store(cuda, z, case):
    from bevfusion_b200.object_paste import ObjectStore
    off = z[case + "_db_offsets"]
    store = ObjectStore(int(off[-1]), 5, len(off) - 1, 64, cuda)
    for i in range(len(off) - 1):
        store.put(i, z[case + "_db_rows"][off[i]:off[i + 1]])
    return store


def fixture_draw(z, case, j):
    from bevfusion_b200.object_paste import PasteDraw
    p = "%s_f%d_" % (case, j)
    kept = z[p + "kept"].tolist()
    if not kept:
        return None
    n = len(z[p + "gt_boxes"])
    return PasteDraw([None] * len(kept), kept, z[p + "boxes"][n:], z[p + "labels"][n:])


def cloud_store(cuda, clouds, max_batch=4, cap=None):
    from bevfusion_b200.lidar_sweeps import SweepStore
    store = SweepStore(len(clouds), cap or max(max(len(c) for c in clouds), 1), 5, cuda, max_batch=max_batch,
                       max_entries=1)
    for k, c in enumerate(clouds):
        store.put(k, c)
    return store


def assemble(store, n, **kw):
    return store.assemble([(s, []) for s in range(n)], 5, pad_empty_sweeps=False, **kw)


def aug_draws(n, seed):
    from bevfusion_b200.lidar_aug import GlobalRotScaleTrans, RandomFlip3D, draw_sample
    rng = np.random.RandomState(seed)
    return [draw_sample(GlobalRotScaleTrans(LA.SHIPPED_SCALE, LA.SHIPPED_ROTATE, LA.SHIPPED_TRANSLATE, True, rng=rng),
                        RandomFlip3D(rng=rng)) for _ in range(n)]


@pytest.mark.parametrize("mode", ["paste", "aug", "aug_range"])
def test_reference_cases(cuda, z, mode):
    from bevfusion_b200.lidar_aug import LidarAug
    from bevfusion_b200.object_paste import PasteBlock
    for case, j in FRAMES:
        p = "%s_f%d_" % (case, j)
        block = PasteBlock(db_store(cuda, z, case), 1, 64)
        block.write([fixture_draw(z, case, j)], 5)
        want = z[p + "points"]
        kw = {}
        if mode != "paste":
            d = aug_draws(1, len(want))[0]
            aug = LidarAug(1, cuda)
            aug.write([d])
            kw["aug"] = aug
            want = LA.augment_points(want, tuple(d), exact=True)
            if mode == "aug_range":
                kw["point_cloud_range"] = LA.POINT_CLOUD_RANGE
                want = want[LA.in_range_3d(want, LA.POINT_CLOUD_RANGE)]
        got = assemble(cloud_store(cuda, [z[p + "cloud"]]), 1, paste=block, **kw)[0]
        assert same(got, want), (case, j, mode)


def box(x, y, z0, l, w, h, yaw):
    return np.array([x, y, z0, l, w, h, yaw, 0, 0], f32)


def face_cloud(boxes):
    """rows on every face centre of each box, one ulp either side along x, y and z, plus +-0, +-inf and NaN rows"""
    from bevfusion_b200.object_paste import box_planes
    rows = []
    for b in boxes:
        c, s = np.cos(b[6]), np.sin(b[6])
        for lx, ly, lz in ((0.5, 0, 0.5), (-0.5, 0, 0.5), (0, 0.5, 0.5), (0, -0.5, 0.5), (0, 0, 0), (0, 0, 1)):
            px, py = lx * b[3], ly * b[4]
            p = np.array([b[0] + px * c - py * s, b[1] + px * s + py * c, b[2] + lz * b[5]], f32)
            for axis in range(3):
                for toward in (-np.inf, np.inf):
                    q = p.copy()
                    q[axis] = np.nextafter(q[axis], f32(toward))
                    rows.append(q)
            rows.append(p)
    rows += [[0, 0, 0], [-0.0, -0.0, -0.0], [np.inf, 0, 0], [-np.inf, 0, 0], [np.nan, 0, 0], [0, np.nan, 1],
             [0, 0, np.nan]]
    xyz = np.array(rows, f32)
    return np.c_[xyz, np.arange(len(xyz), dtype=f32) / 7, np.zeros(len(xyz), f32)].astype(f32)


def key_cloud(rng, n, half):
    """[n, 5] key rows in [-half, half]^2 x [-2, 1]: column 4 is 0, as LoadPointsFromMultiSweeps leaves it"""
    return np.c_[rng.uniform(-half, half, (n, 2)), rng.uniform(-2, 1, (n, 1)), rng.uniform(0, 1, (n, 1)),
                 np.zeros((n, 1))].astype(f32)


def small_store(cuda, objects):
    from bevfusion_b200.object_paste import ObjectStore
    store = ObjectStore(sum(len(o) for o in objects), 5, len(objects), 4096, cuda)
    for i, o in enumerate(objects):
        store.put(i, o)
    return store


def draw_of(boxes, indices):
    from bevfusion_b200.object_paste import PasteDraw
    boxes = np.asarray(boxes, f32).reshape(-1, 9)
    return PasteDraw([None] * len(boxes), list(indices), boxes, np.zeros(len(boxes), np.int64))


def oracle(cloud, objects, d):
    if d is None:
        return cloud
    n, dd = O.planes(d.boxes)
    return O.paste(cloud, [objects[i] for i in d.indices], d.boxes, n, dd)


def test_faces_ulps_nonfinite_and_yaw_pi(cuda):
    from bevfusion_b200.object_paste import PasteBlock
    boxes = [box(0, 0, -1, 4, 2, 2, 0), box(10, 0, -1, 3, 3, 2, np.pi), box(-10, 5, -1, 5, 2, 2, -np.pi),
             box(0, 12, -1, 4, 4, 3, np.pi / 2), box(5, -9, -1, 3.3, 1.7, 1.1, 0.7)]
    cloud = face_cloud(boxes)
    rng = np.random.default_rng(5)
    objects = [np.c_[rng.uniform(-1, 1, (n, 3)), rng.uniform(0, 1, (n, 2))].astype(f32) for n in (3, 700, 1500, 0, 9)]
    store = small_store(cuda, objects)
    block = PasteBlock(store, 2, 8)
    d = draw_of(boxes, range(5))
    block.write([d, None], 5)
    got = assemble(cloud_store(cuda, [cloud, cloud]), 2, paste=block)
    want = oracle(cloud, objects, d)
    inside = O.inside_any(cloud[:, :3], *O.planes(d.boxes))
    # the first box is axis-aligned with exact planes: its face centres give sign == 0 (kept), one ulp inward is in
    assert inside.any() and (~inside).any() and not inside[6:42:7].any()
    assert same(got[0], want) and not np.isnan(got[0][:, :3].cpu().numpy()).any()
    assert same(got[1], cloud) and np.isnan(got[1][:, :3].cpu().numpy()).any(1).sum() == 3


def test_overflow_mid_paste_and_full_batch(cuda):
    from bevfusion_b200.object_paste import PasteBlock
    from bevfusion_b200.lidar_sweeps import OVERFLOW
    rng = np.random.default_rng(9)
    objects = [np.c_[rng.uniform(-1, 1, (n, 3)), rng.uniform(0, 1, (n, 2))].astype(f32) for n in (1500, 300, 2100)]
    boxes = [box(-20 + 8 * k, 3 * k, -1, 2 + k, 2, 2, 0.3 * k) for k in range(8)]
    cloud = key_cloud(rng, 5000, 30)
    block = PasteBlock(small_store(cuda, objects), 4, 8)
    draws = [draw_of(boxes, [k % 3 for k in range(8)]), None, draw_of(boxes[:3], [2, 0, 1]), draw_of(boxes[:1], [1])]
    block.write(draws, 5)
    store = cloud_store(cuda, [cloud] * 4)
    got = assemble(store, 4, paste=block)
    wants = [oracle(cloud, objects, d) for d in draws]
    assert all(same(g, w) for g, w in zip(got, wants))
    for cap in (700, 1024, 1500 + 299, 2000):           # cut inside the pasted rows, at a tile edge, mid-object
        out, counts, status = assemble(store, 4, paste=block, cap=cap, sync=False)
        assert int(status[0]) & OVERFLOW
        for b in range(4):
            n = min(cap, len(wants[b]))
            assert int(counts[b]) == n and same(out[b, :n], wants[b][:n])


def test_none_block_equals_the_plain_aug_launch(cuda, z):
    from bevfusion_b200.lidar_aug import LidarAug
    from bevfusion_b200.object_paste import PasteBlock
    clouds = [z["shipped_f0_cloud"], z["empty_gt_f0_cloud"], z["pending_f0_cloud"]]
    store = cloud_store(cuda, clouds)
    aug = LidarAug(4, cuda)
    aug.write(aug_draws(3, 1))
    block = PasteBlock(db_store(cuda, z, "shipped"), 4, 16)
    block.write([None] * 3, 5)
    kw = dict(point_cloud_range=LA.POINT_CLOUD_RANGE, aug=aug, sync=False)
    ref = assemble(store, 3, **kw)
    got = assemble(store, 3, paste=block, **kw)
    n = ref[1].tolist()
    assert n == got[1].tolist() and int(got[2][0]) == 0
    assert all(same(got[0][k, :n[k]], ref[0][k, :n[k]].cpu().numpy()) for k in range(3))


def test_malformed_blocks_set_bad_paste(cuda):
    from bevfusion_b200.lidar_sweeps import BAD_PASTE
    from bevfusion_b200.object_paste import PasteBlock, SAMPLE_DTYPE, OBJECT_DTYPE
    rng = np.random.default_rng(3)
    objects = [np.c_[rng.uniform(-1, 1, (50, 3)), rng.uniform(0, 1, (50, 2))].astype(f32) for _ in range(2)]
    cloud = key_cloud(rng, 800, 5)
    store = small_store(cuda, objects)
    block = PasteBlock(store, 2, 4)
    good = draw_of([box(0, 0, -1, 3, 3, 3, 0)], [1])
    cs = cloud_store(cuda, [cloud, cloud])
    for field, value in (("count", 5), ("count", -1), ("cols", 5), ("index", 2), ("index", -1)):
        block.write([good, good], 5)
        host = block.block.cpu().numpy()
        smp = host[:SAMPLE_DTYPE.itemsize * 2].view(SAMPLE_DTYPE)
        obj = host[block._objects_at:].view(OBJECT_DTYPE)
        if field == "count":
            smp["count"][1] = value
        elif field == "cols":
            smp["cols"][1, 4] = value
        else:
            obj["index"][4] = value          # sample 1's first object
        block.block.copy_(torch.from_numpy(host))
        out, counts, status = assemble(cs, 2, paste=block, cap=2000, sync=False)
        assert int(status[0]) == BAD_PASTE, field
        want = oracle(cloud, objects, good)
        assert int(counts[0]) == len(want) and same(out[0, :len(want)], want)
        assert int(counts[1]) == len(cloud) and same(out[1, :len(cloud)], cloud)   # nothing pasted or removed
    with pytest.raises(ValueError):
        block.write([good], 5)
        assemble(cs, 2, paste=block)                  # past the last write()


def test_graph_replay_with_new_draws_and_new_objects(cuda):
    from bevfusion_b200.lidar_aug import LidarAug
    from bevfusion_b200.object_paste import ObjectStore, PasteBlock
    rng = np.random.default_rng(21)
    cloud = key_cloud(rng, 6000, 30)
    store = cloud_store(cuda, [cloud, cloud[::2]], max_batch=2)
    objs = ObjectStore(20000, 5, 16, 4096, cuda)
    block = PasteBlock(objs, 2, 16)
    aug = LidarAug(2, cuda)

    def frame(seed):
        r = np.random.default_rng(seed)
        objects = [np.c_[r.uniform(-1, 1, (n, 3)), r.uniform(0, 1, (n, 2))].astype(f32)
                   for n in r.integers(0, 1800, 6)]
        objs.clear()
        for i, o in enumerate(objects):
            objs.put(i, o)
        draws = [draw_of([box(*r.uniform(-25, 25, 2), -1, *r.uniform(1, 6, 3), r.uniform(-np.pi, np.pi))
                          for _ in range(k)], list(r.permutation(6)[:k])) for k in (int(r.integers(1, 7)), 3)]
        block.write(draws, 5)
        aug.write(aug_draws(2, seed))
        return objects, draws

    samples = [(0, []), (1, [])]
    frame(0)
    batch, F, bound = store.write_frame(samples, 5, pad_empty_sweeps=False, point_cloud_range=LA.POINT_CLOUD_RANGE,
                                        paste=block)
    assert bound <= 20000
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        store.launch(2, F, 20000, aug=aug, paste=block)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out, counts, status = store.launch(2, F, 20000, aug=aug, paste=block)
    for seed in (1, 2, 3):
        frame(seed)
        g.replay()
        eo, ec, es = store.launch(2, F, 20000, aug=aug, paste=block)
        torch.cuda.synchronize()
        assert counts.tolist() == ec.tolist() and int(status[0]) == int(es[0]) == 0
        for b in range(2):
            assert same(out[b, :int(counts[b])], eo[b, :int(ec[b])].cpu().numpy())


def test_centerhead_targets_from_merged_device_augmented_boxes(cuda, z):
    from bevfusion_b200 import head_targets as H
    from bevfusion_b200.lidar_aug import LidarAug
    from bevfusion_b200.object_paste import ObjectPaste
    tasks = [dict(num_class=1, class_names=["car"]), dict(num_class=2, class_names=["truck", "construction_vehicle"]),
             dict(num_class=2, class_names=["bus", "trailer"]), dict(num_class=1, class_names=["barrier"]),
             dict(num_class=2, class_names=["motorcycle", "bicycle"]),
             dict(num_class=2, class_names=["pedestrian", "traffic_cone"])]
    cfg = dict(point_cloud_range=LA.POINT_CLOUD_RANGE, grid_size=[1440, 1440, 41], voxel_size=[0.075, 0.075, 0.2],
               out_size_factor=8, dense_reg=1, gaussian_overlap=0.1, max_objs=500, min_radius=2)
    frames = [("shipped", 0), ("exhaust", 1), ("many_gt", 0), ("epoch_gate", 0)]
    merged = [ObjectPaste.merge(z["%s_f%d_gt_boxes" % f], z["%s_f%d_gt_labels" % f], fixture_draw(z, *f))
              for f in frames]
    for (c, j), (b, l) in zip(frames, merged):
        assert same(b, z["%s_f%d_boxes" % (c, j)])
    draws = aug_draws(4, 11)
    aug = LidarAug(4, cuda)
    aug.write(draws)
    from bevfusion_b200.head_targets import pad_gt
    pb, pl, pc = pad_gt([torch.from_numpy(b) for b, _ in merged],
                        [torch.from_numpy(l.astype(np.int32)).to(cuda) for _, l in merged])
    ob, ol, oc, _ = aug.boxes(pb, pl, pc, LA.POINT_CLOUD_RANGE, LA.OBJECT_CLASSES)
    host = [LA.boxes_filtered(b, l, tuple(d)) for (b, l), d in zip(merged, draws)]
    hb, hl, hc = pad_gt([torch.from_numpy(np.ascontiguousarray(h[0])) for h in host],
                        [torch.from_numpy(np.asarray(h[1], np.int32)).to(cuda) for h in host])
    for a_list, b_list in zip(H.centerhead_targets_batched(ob, ol, oc, tasks, cfg),
                              H.centerhead_targets_batched(hb, hl, hc, tasks, cfg)):
        for a, b in zip(a_list, b_list):
            assert torch.equal(a, b)
