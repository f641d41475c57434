"""Numpy restatement of ObjectPaste (transforms_3d.py:357-449, dbsampler.py, box_np_ops.py:430-451, 692-775,
pipelines/utils.py:31-111): the sampler, the collision loop pair by pair, the face planes and the removal, plus the
synthetic databases and clouds the golden file and the tests share.

Everything is float32 with one rounding per operation, as the reference's numba functions evaluate it."""
import hashlib
import os

import numpy as np

import lidar_aug_oracle as LA

CLASSES = LA.OBJECT_CLASSES
SHIPPED_GROUPS = {"car": 2, "truck": 3, "construction_vehicle": 7, "bus": 4, "trailer": 6, "barrier": 2,
                  "motorcycle": 6, "bicycle": 6, "pedestrian": 2, "traffic_cone": 2}
SHIPPED_PREPARE = {"filter_by_difficulty": [-1], "filter_by_min_points": {c: 5 for c in CLASSES}}
LOAD_DIM = 5
f32 = np.float32


# ---- the sampler ---------------------------------------------------------------------------------------------------
class Sampler:
    """DataBaseSampler + BatchSampler on numpy's global RNG: db is {class: [info, ...]}"""

    def __init__(self, db, rate, prepare, groups):
        for prep, val in prepare.items():
            if prep == "filter_by_difficulty":
                db = {k: [i for i in v if i["difficulty"] not in val] for k, v in db.items()}
            else:
                db = {k: [i for i in v if k not in val or int(val[k]) <= 0 or i["num_points_in_gt"] >= int(val[k])]
                      for k, v in db.items()}
        self.db, self.rate, self.groups = db, rate, list(groups.items())
        self.state = {}
        for k, v in db.items():
            order = np.arange(len(v))
            np.random.shuffle(order)
            self.state[k] = [order, 0]

    def take(self, name, num):
        order, idx = self.state[name]
        if idx + num >= len(order):
            out = order[idx:].copy()
            np.random.shuffle(order)
            self.state[name][1] = 0
        else:
            out = order[idx:idx + num].copy()
            self.state[name][1] = idx + num
        return [self.db[name][i] for i in out]

    def sample_all(self, gt_boxes, gt_labels):
        """-> list of kept infos in order"""
        nums = [np.round(self.rate * int(m - sum(int(l) == CLASSES.index(c) for l in gt_labels))).astype(np.int64)
                for c, m in self.groups]
        kept, avoid = [], gt_boxes
        for (c, _), num in zip(self.groups, nums):
            if num <= 0:
                continue
            cand = self.take(c, num)
            boxes = np.concatenate([avoid, np.stack([i["box3d_lidar"] for i in cand])])
            keep = collision_loop(boxes, avoid.shape[0])
            mine = [i for i, k in zip(cand, keep) if k]
            kept += mine
            if mine:
                avoid = np.concatenate([avoid, np.stack([i["box3d_lidar"] for i in mine])])
        return kept


# ---- the collision test ----------------------------------------------------------------------------------------------
def bev_corners(boxes):
    """center_to_corner_box2d in float32: clockwise corners [N, 4, 2] from the minimum one"""
    norm = np.array([[-0.5, -0.5], [-0.5, 0.5], [0.5, 0.5], [0.5, -0.5]], f32)
    c = boxes[:, 3:5, None].transpose(0, 2, 1) * norm[None]
    s, co = np.sin(boxes[:, 6]), np.cos(boxes[:, 6])
    x = c[..., 0] * co[:, None] + c[..., 1] * s[:, None]
    y = c[..., 0] * -s[:, None] + c[..., 1] * co[:, None]
    return np.stack([x, y], -1) + boxes[:, None, 0:2]


def collide(b, q):
    """box_collision_test for one pair of corner sets [4, 2], scalar by scalar"""
    if not (min(b[:, 0].max(), q[:, 0].max()) - max(b[:, 0].min(), q[:, 0].min()) > 0):
        return False
    if not (min(b[:, 1].max(), q[:, 1].max()) - max(b[:, 1].min(), q[:, 1].min()) > 0):
        return False

    def ccw(P, Q, R):
        return (R[1] - P[1]) * (Q[0] - P[0]) > (Q[1] - P[1]) * (R[0] - P[0])

    for k in range(4):
        A, B = b[k], b[(k + 1) % 4]
        for l in range(4):
            C, D = q[l], q[(l + 1) % 4]
            if ccw(A, C, D) != ccw(B, C, D) and ccw(A, B, C) != ccw(A, B, D):
                return True

    def inside(P, Q):
        for l in range(4):
            for k in range(4):
                v = -(P[k] - P[(k + 1) % 4])
                cross = v[1] * (P[k, 0] - Q[l, 0])
                cross = cross - v[0] * (P[k, 1] - Q[l, 1])
                if cross >= 0:
                    return False
        return True

    return inside(b, q) or inside(q, b)


def collision_loop(boxes, num_gt, corners=None):
    """sample_class_v2's loop: keep flags of the candidates boxes[num_gt:]"""
    cs = bev_corners(boxes) if corners is None else corners
    n = len(boxes)
    m = np.array([[i != j and collide(cs[i], cs[j]) for j in range(n)] for i in range(num_gt, n)], bool).reshape(-1, n)
    keep = []
    for k in range(n - num_gt):
        if m[k].any():
            m[k] = False
            m[:, num_gt + k] = False
            keep.append(False)
        else:
            keep.append(True)
    return keep


# ---- the removal and the paste -------------------------------------------------------------------------------------
def inside_any(xyz, normal, d):
    """[n] bool: points_in_rbbox(...).any(-1): ((x n0 + y n1) + z n2) + d < 0 on all 6 faces of some box (a NaN
    comparison counts as < 0), in float32"""
    xyz = np.asarray(xyz, f32)
    if len(normal) == 0:
        return np.zeros(len(xyz), bool)
    x, y, z = (xyz[:, None, None, k] for k in range(3))
    with np.errstate(invalid="ignore"):
        s = ((x * normal[None, ..., 0] + y * normal[None, ..., 1]) + z * normal[None, ..., 2]) + d[None]
    return (~(s >= 0)).all(-1).any(-1)


def paste(cloud, objects, boxes, normal, d, use_dim=LOAD_DIM):
    """cat([object rows[:, use_dim] translated by fl32(box[:3]), ...], the cloud's rows outside every box)"""
    cols = list(range(use_dim)) if isinstance(use_dim, int) else list(use_dim)
    rows = []
    for o, b in zip(objects, boxes):
        r = np.asarray(o, f32)[:, cols].copy()
        r[:, :3] += np.asarray(b[:3], f32)
        rows.append(r)
    keep = ~inside_any(cloud[:, :3], normal, d) if len(boxes) else np.ones(len(cloud), bool)
    return np.concatenate(rows + [cloud[keep]]).astype(f32) if rows else cloud.copy()


def planes(boxes):
    """points_in_rbbox's face planes, with the package's numpy calls (bevfusion_b200.object_paste.box_planes)"""
    from bevfusion_b200.object_paste import box_planes
    return box_planes(np.asarray(boxes, f32))


# ---- synthetic databases and clouds ----------------------------------------------------------------------------------
def make_db(rng, per_class, spot=None, big=False, extra_key=True, rows=(5, 40)):
    """{class: [info]} with float32 boxes; each info has an "id" and its raw rows under "rows" (local coordinates,
    as the GT database stores them).  spot: place every box at that (x, y); big: boxes of 30-40 m."""
    db, k = {}, 0
    keys = list(CLASSES) + (["ignored"] if extra_key else [])
    for c in keys:
        infos = []
        for _ in range(per_class.get(c, 6) if isinstance(per_class, dict) else per_class):
            xy = rng.uniform(-45, 45, 2) if spot is None else np.asarray(spot) + rng.uniform(-0.3, 0.3, 2)
            size = rng.uniform(30, 40, 3) if big else rng.uniform([0.5, 0.5, 1.0], [10.0, 3.0, 3.5])
            box = np.array([xy[0], xy[1], rng.uniform(-2, 0), size[0], size[1], size[2],
                            rng.uniform(-np.pi, np.pi), rng.normal(0, 2), rng.normal(0, 2)], f32)
            n = int(rng.integers(*rows))
            pts = np.concatenate([rng.uniform(-0.5, 0.5, (n, 3)) * size[None, :3] * 0.9, rng.uniform(0, 1, (n, 2))],
                                 1).astype(f32)
            pts[:, 2] += size[2] / 2
            infos.append({"name": c, "path": "obj_%04d.bin" % k, "id": k, "box3d_lidar": box,
                          "difficulty": int(rng.choice([0, 0, 0, -1])), "num_points_in_gt": int(rng.integers(2, 60)),
                          "rows": pts})
            k += 1
        db[c] = infos
    return db


def write_db(db, root):
    """the .bin files of db under root; returns the infos without their rows, as the pickled dbinfos hold them"""
    out = {}
    for c, infos in db.items():
        out[c] = []
        for i in infos:
            i["rows"].astype(f32).tofile(os.path.join(root, i["path"]))
            out[c].append({k: v for k, v in i.items() if k != "rows"})
    return out


def make_cloud(rng, n, db, gt_boxes, special=True):
    """[n, 5] float32 key rows (column 4, the time lag, is 0 as LoadPointsFromMultiSweeps leaves it on the key):
    uniform rows, rows around every database box and GT box, and (special) non-finite rows"""
    centers = [i["box3d_lidar"] for v in db.values() for i in v] + list(gt_boxes)
    parts = [np.c_[rng.uniform(-55, 55, (n, 2)), rng.uniform(-4, 3, (n, 1)), rng.uniform(0, 1, (n, 2))]]
    for b in centers:
        m = 12
        parts.append(np.c_[b[0] + rng.uniform(-1, 1, (m, 1)) * b[3], b[1] + rng.uniform(-1, 1, (m, 1)) * b[4],
                           b[2] + rng.uniform(-0.2, 1.2, (m, 1)) * b[5], rng.uniform(0, 1, (m, 2))])
    cloud = np.concatenate(parts).astype(f32)
    cloud[:, 4] = 0
    if special:
        cloud = np.concatenate([cloud, np.array([[np.nan, 0, 0, 0.5, 0], [0, np.inf, 0, 0.5, 0],
                                                 [-np.inf, 0, 1, 0.5, 0], [0.0, -0.0, 0, 0.5, 0]], f32)])
    return cloud


def gt_set(rng, n, labels=None):
    """n float32 GT boxes [n, 9] and labels (some -1)"""
    b = np.c_[rng.uniform(-48, 48, (n, 2)), rng.uniform(-2, 0, (n, 1)), rng.uniform(0.5, 8, (n, 1)),
              rng.uniform(0.5, 3, (n, 1)), rng.uniform(1, 3, (n, 1)), rng.uniform(-np.pi, np.pi, (n, 1)),
              rng.normal(0, 2, (n, 2))].astype(f32)
    if labels is None:
        labels = rng.integers(-1, len(CLASSES), n)
    return b.reshape(-1, 9), np.asarray(labels, np.int64)


def collision_pairs(rng, n):
    """n adversarial box pairs [n, 2, 9] float32: touching, collinear, shared corners, nested, near-miss by one ulp,
    yaw at 0, +-pi/2 and +-pi"""
    a = np.zeros((n, 9), f32)
    a[:, 0:2] = rng.integers(-4, 5, (n, 2))
    a[:, 3:5] = rng.integers(1, 5, (n, 2))
    a[:, 5] = 1
    yaws = np.array([0, np.pi / 2, -np.pi / 2, np.pi, -np.pi, np.pi / 4], f32)
    a[:, 6] = yaws[rng.integers(0, len(yaws), n)] * (rng.random(n) < 0.7) + rng.uniform(-np.pi, np.pi, n) * (
        rng.random(n) >= 0.7)
    b = a.copy()
    kind = rng.integers(0, 5, n)
    off = rng.integers(-6, 7, (n, 2)).astype(f32) * 0.5                # touching / collinear on a half grid
    b[:, 0:2] = np.where(kind[:, None] <= 1, a[:, 0:2] + off, b[:, 0:2])
    b[:, 3:5] = np.where(kind[:, None] == 1, rng.integers(1, 5, (n, 2)), b[:, 3:5])
    b[:, 3:5] = np.where(kind[:, None] == 2, a[:, 3:5] * rng.uniform(0.1, 0.9, (n, 1)), b[:, 3:5])   # nested
    b[:, 0:2] = np.where(kind[:, None] == 3, a[:, 0:2] + rng.normal(0, 3, (n, 2)), b[:, 0:2])
    b[:, 3:5] = np.where(kind[:, None] == 3, rng.uniform(0.2, 6, (n, 2)), b[:, 3:5])
    b[:, 0:2] = np.where(kind[:, None] == 4, np.nextafter(a[:, 0:2] + off, np.where(rng.random((n, 2)) < 0.5, -99, 99)
                                                          .astype(f32)), b[:, 0:2])
    b[:, 6] = np.where(rng.random(n) < 0.5, a[:, 6], yaws[rng.integers(0, len(yaws), n)])
    return np.stack([a, b], 1).astype(f32)


def _case_setup(case, rng):
    """(db, sample_groups, prepare, frames [(gt_boxes, gt_labels)], epoch, stop_epoch) of a golden case"""
    groups, prepare, epoch, stop = SHIPPED_GROUPS, SHIPPED_PREPARE, -1, None
    if case == "shipped":
        db = make_db(rng, 8)
        frames = [gt_set(rng, 20)]
    elif case == "exhaust":
        db = make_db(rng, {"bus": 4, "trailer": 5})
        groups, prepare = {"bus": 2, "trailer": 3}, {}
        frames = [gt_set(rng, 0) for _ in range(3)]
    elif case == "many_gt":
        db = make_db(rng, 8)
        frames = [gt_set(rng, 60, np.repeat(np.arange(10), 6))]
    elif case == "empty_gt":
        db = make_db(rng, 8)
        frames = [gt_set(rng, 0)]
    elif case == "all_collide":
        db = make_db(rng, 6)
        gt, labels = gt_set(rng, 1, [-1])
        gt[0, :7] = [0, 0, -1, 300, 300, 10, 0.1]
        frames = [(gt, labels)]
    elif case == "contains_gt":
        db = make_db(rng, 4, spot=(3.0, -2.0), big=True)
        gt, labels = gt_set(rng, 1, [0])
        gt[0, :7] = [3, -2, -1, 1.0, 1.0, 1.5, 0.3]
        frames = [(gt, labels)]
    elif case == "pending":
        db = make_db(rng, {c: 6 for c in CLASSES}, spot=(10.0, 10.0))
        groups, prepare = {"truck": 3, "bus": 2}, {}
        frames = [gt_set(rng, 0)]
    elif case == "epoch_gate":
        db = make_db(rng, 8)
        epoch, stop = 15, 15
        frames = [gt_set(rng, 20)]
    return db, groups, prepare, frames, epoch, stop


CASES = ["shipped", "exhaust", "many_gt", "empty_gt", "all_collide", "contains_gt", "pending", "epoch_gate"]


CASES = ["shipped", "exhaust", "many_gt", "empty_gt", "all_collide", "contains_gt", "pending", "epoch_gate"]


def case_inputs(case, seed):
    """(db, sample_groups, prepare, frames [(gt_boxes, gt_labels, cloud)], epoch, stop_epoch) of golden case `case`,
    regenerated from its seed"""
    rng = np.random.default_rng(seed)
    db, groups, prepare, frames, epoch, stop = _case_setup(case, rng)
    frames = [(gt, labels, make_cloud(rng, 1500, db, gt)) for gt, labels in frames]
    return db, groups, prepare, frames, epoch, stop


def digest(*arrays):
    """SHA-256 of the arrays' bytes, as uint8 [32]"""
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return np.frombuffer(h.digest(), np.uint8)


def inputs_digest(db, frames):
    flat = [i for v in db.values() for i in v]
    arrays = [np.stack([i["box3d_lidar"] for i in flat])] + [i["rows"] for i in flat]
    arrays += [np.array([[i["id"], i["difficulty"], i["num_points_in_gt"]] for i in flat], np.int64)]
    return digest(*(arrays + [a for f in frames for a in f]))


def load_fixture(path):
    """golden/object_paste_tiny.npz with its regenerated inputs: a dict holding the stored arrays plus, per case, the
    database (<case>_db_keys / _db_class / _db_boxes / _db_difficulty / _db_npts / _db_offsets / _db_rows) and, per
    frame, the input cloud (<case>_f<j>_cloud) and the reference's output (<case>_f<j>_points).  Raises when a
    regenerated input or a rebuilt output differs from what the reference saw or produced."""
    z = dict(np.load(path))
    for case in CASES:
        db, _, _, frames, _, _ = case_inputs(case, int(z[case + "_seed"]))
        if not np.array_equal(inputs_digest(db, frames), z[case + "_inputs_sha256"]):
            raise ValueError("the regenerated inputs of case %s differ from the reference's" % case)
        keys = list(db)
        flat = [i for v in db.values() for i in v]
        z[case + "_db_keys"] = np.array(keys)
        z[case + "_db_class"] = np.array([keys.index(i["name"]) for i in flat], np.int32)
        z[case + "_db_boxes"] = np.stack([i["box3d_lidar"] for i in flat]).astype(f32)
        z[case + "_db_difficulty"] = np.array([i["difficulty"] for i in flat], np.int32)
        z[case + "_db_npts"] = np.array([i["num_points_in_gt"] for i in flat], np.int32)
        z[case + "_db_offsets"] = np.cumsum([0] + [len(i["rows"]) for i in flat]).astype(np.int64)
        z[case + "_db_rows"] = np.concatenate([i["rows"] for i in flat]).astype(f32)
        for j, (gt, labels, cloud) in enumerate(frames):
            p = "%s_f%d_" % (case, j)
            keep = np.unpackbits(z[p + "keep"])[:len(cloud)].astype(bool)
            rows = []
            for k, b in zip(z[p + "kept"], z[p + "boxes"][len(gt):]):
                r = flat[int(k)]["rows"].astype(f32).copy()
                r[:, :3] += b[:3]
                rows.append(r)
            points = np.concatenate(rows + [cloud[keep]]).astype(f32)
            if not np.array_equal(digest(points), z[p + "points_sha256"]):
                raise ValueError("the rebuilt output of %s frame %d differs from the reference's" % (case, j))
            z[p + "cloud"], z[p + "points"] = cloud, points
    return z


count_diff = LA.count_diff          # elements that differ bit for bit, NaN payloads aside
