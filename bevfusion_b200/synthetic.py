"""Deterministic synthetic inputs with the shapes / statistics of the reference's nuScenes
configs (SURVEY.md section 8d).  numpy / torch on the host; no dataset, no network."""
import math

import numpy as np
import torch

from .vtransform import create_frustum, get_geometry

# BASELINE.json configs, made concrete (BASELINE.md section 3)
CONFIGS = {
    # C1: bev_pool correctness case (1 cam, 64x176 features, D=60, 128x128 grid, C=64)
    "C1": dict(n_cam=1, image_size=(512, 1408), feature_size=(64, 176), dbound=(1.0, 61.0, 1.0),
               xbound=(-51.2, 51.2, 0.8), ybound=(-51.2, 51.2, 0.8), zbound=(-10.0, 10.0, 20.0), C=64),
    # C2: camera+lidar/swint_v0p075 view transform (6 cam, 256x704 -> 32x88, D=118, 360x360, C=80)
    "C2": dict(n_cam=6, image_size=(256, 704), feature_size=(32, 88), dbound=(1.0, 60.0, 0.5),
               xbound=(-54.0, 54.0, 0.3), ybound=(-54.0, 54.0, 0.3), zbound=(-10.0, 10.0, 20.0), C=80),
    # C2 literal: 180x180 BEV grid as BASELINE.json words it
    "C2_180": dict(n_cam=6, image_size=(256, 704), feature_size=(32, 88), dbound=(1.0, 60.0, 0.5),
                   xbound=(-54.0, 54.0, 0.6), ybound=(-54.0, 54.0, 0.6), zbound=(-10.0, 10.0, 20.0), C=80),
    # C5: stress (6 cam 512x1408 -> 64x176, D=200, 256x256, C=80)
    "C5": dict(n_cam=6, image_size=(512, 1408), feature_size=(64, 176), dbound=(1.0, 61.0, 0.3),
               xbound=(-51.2, 51.2, 0.4), ybound=(-51.2, 51.2, 0.4), zbound=(-10.0, 10.0, 20.0), C=80),
    # tiny case for smoke / fast tests
    "tiny": dict(n_cam=2, image_size=(64, 176), feature_size=(8, 22), dbound=(1.0, 21.0, 1.0),
                 xbound=(-16.0, 16.0, 0.5), ybound=(-16.0, 16.0, 0.5), zbound=(-10.0, 10.0, 20.0), C=80),
}

LIDAR_C3 = dict(voxel_size=[0.075, 0.075, 0.2], point_cloud_range=[-54.0, -54.0, -5.0, 54.0, 54.0, 3.0],
                max_num_points=10, max_voxels=(120000, 160000), sparse_shape=[1440, 1440, 41])


def camera_rig(n_cam=6, image_size=(256, 704), batch=1):
    """nuScenes-shaped 6-camera rig (SURVEY.md section 8d): yaw {0,-55,+55,180,+110,-110} deg,
    fx=fy=1266 (rear 809), cx=816, cy=491 on 1600x900, image aug = resize then crop to
    image_size (0.48 / (32,176) for 704x256).  Returns a dict of [B, N, ...] fp32 tensors."""
    yaws = [0.0, -55.0, 55.0, 180.0, 110.0, -110.0][:n_cam]
    iH, iW = image_size
    scale = 0.48 * iW / 704.0
    crop_w = (1600 * scale - iW) / 2.0
    crop_h = 900 * scale - iH
    rots, trans, intr, prot, ptr = [], [], [], [], []
    R0 = torch.tensor([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])
    for i, yaw in enumerate(yaws):
        t = math.radians(yaw)
        Rz = torch.tensor([[math.cos(t), -math.sin(t), 0.0], [math.sin(t), math.cos(t), 0.0],
                           [0.0, 0.0, 1.0]])
        rots.append(Rz @ R0)
        trans.append(Rz @ torch.tensor([0.6, 0.0, 0.0]) + torch.tensor([0.0, 0.0, -0.3]))
        f = 809.0 if abs(yaw) == 180.0 else 1266.0
        intr.append(torch.tensor([[f, 0.0, 816.0], [0.0, f, 491.0], [0.0, 0.0, 1.0]]))
        prot.append(torch.diag(torch.tensor([scale, scale, 1.0])))
        ptr.append(torch.tensor([-crop_w, -crop_h, 0.0]))

    def st(v):
        return torch.stack(v).unsqueeze(0).repeat(batch, *([1] * (v[0].dim() + 1))).float().contiguous()

    return dict(camera2lidar_rots=st(rots), camera2lidar_trans=st(trans), intrins=st(intr),
                post_rots=st(prot), post_trans=st(ptr))


def lidar_camera_matrices(n_cam=6, image_size=(256, 704), batch=1, augment=True):
    """4x4 matrices the depth-aware lift consumes (base.py:237-262), consistent with camera_rig:
    lidar2image = K @ inverse(camera2lidar), img_aug_matrix from the resize / crop, and a
    per-sample lidar augmentation (z rotation, scale, translation).  [B, N, 4, 4] / [B, 4, 4] fp32."""
    rig = camera_rig(n_cam, image_size, batch)
    B, N = batch, n_cam
    eye = torch.eye(4).view(1, 1, 4, 4).repeat(B, N, 1, 1)
    cam2lidar = eye.clone()
    cam2lidar[..., :3, :3] = rig["camera2lidar_rots"]
    cam2lidar[..., :3, 3] = rig["camera2lidar_trans"]
    lidar2cam = torch.inverse(cam2lidar)
    K = eye.clone()
    K[..., :3, :3] = rig["intrins"]
    lidar2image = K.matmul(lidar2cam)
    img_aug = eye.clone()
    img_aug[..., :3, :3] = rig["post_rots"]
    img_aug[..., :3, 3] = rig["post_trans"]
    lidar_aug = torch.eye(4).view(1, 4, 4).repeat(B, 1, 1)
    if augment:
        for b in range(B):
            a = 0.1 - 0.17 * b
            sc = 1.0 + 0.05 * (b + 1)
            lidar_aug[b, :3, :3] = sc * torch.tensor([[math.cos(a), -math.sin(a), 0.0],
                                                      [math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]])
            lidar_aug[b, :3, 3] = torch.tensor([0.5 - b, -0.25 + 0.5 * b, 0.1 * b])
    out = dict(rig)
    out.update(lidar2image=lidar2image.float().contiguous(), img_aug_matrix=img_aug.float().contiguous(),
               lidar_aug_matrix=lidar_aug.float().contiguous(), camera2lidar=cam2lidar.float().contiguous(),
               lidar2camera=lidar2cam.float().contiguous(), cam_intrinsic=K.float().contiguous())
    return out


def camera_geometry(cfg_name="C2", batch=1, device="cpu"):
    """(geom [B, N, D, fH, fW, 3] fp32, cfg dict) for one of CONFIGS."""
    cfg = CONFIGS[cfg_name]
    rig = camera_rig(cfg["n_cam"], cfg["image_size"], batch)
    frustum = create_frustum(cfg["image_size"], cfg["feature_size"], cfg["dbound"])
    geom = get_geometry(frustum, rig["camera2lidar_rots"], rig["camera2lidar_trans"],
                        rig["intrins"], rig["post_rots"], rig["post_trans"])
    return geom.contiguous().to(device), cfg


def lifted_features(cfg_name, batch=1, device="cpu", seed=0, dtype=torch.float32):
    """x [B, N, D, fH, fW, C] standard-normal lifted camera features."""
    cfg = CONFIGS[cfg_name]
    D = len(np.arange(*cfg["dbound"]))
    fH, fW = cfg["feature_size"]
    g = torch.Generator(device="cpu").manual_seed(seed)
    shape = (batch, cfg["n_cam"], D, fH, fW, cfg["C"])
    if device == "cpu":
        return torch.randn(shape, generator=g, dtype=dtype)
    gd = torch.Generator(device=device).manual_seed(seed)
    return torch.randn(shape, generator=gd, dtype=dtype, device=device)


def lidar_cloud(seed=0, sweeps=10, beams=32, az_steps=1090, shuffle=True):
    """10-sweep, 32-beam synthetic LiDAR cloud (SURVEY.md section 8d): ground plane at z=-1.84 plus
    per-sweep random walls, ~295 k points of (x, y, z, intensity, dt) fp32."""
    rng = np.random.default_rng(seed)
    elev = np.deg2rad(np.linspace(-30.67, 10.67, beams))
    az = np.linspace(-np.pi, np.pi, az_steps, endpoint=False)
    pts = []
    for s in range(sweeps):
        ox = 0.5 * s  # ego motion between sweeps
        sector_r = rng.uniform(6.0, 60.0, size=64)
        E, A = np.meshgrid(elev, az, indexing="ij")
        sec = ((A + np.pi) / (2 * np.pi) * 64).astype(int) % 64
        wall_r = sector_r[sec] * (1.0 + 0.02 * rng.standard_normal(E.shape))
        with np.errstate(divide="ignore", invalid="ignore"):
            ground_r = np.where(E < 0, 1.84 / np.sin(-E), np.inf)
        hits_wall = (wall_r * np.sin(E) + 1.84) < 4.0
        r = np.minimum(ground_r, np.where(hits_wall, wall_r / np.maximum(np.cos(E), 1e-3), np.inf))
        r = r * (1.0 + 0.003 * rng.standard_normal(E.shape))
        ok = np.isfinite(r) & (r > 1.0) & (r < 75.0)
        r, E_, A_ = r[ok], E[ok], A[ok]
        x = r * np.cos(E_) * np.cos(A_) - ox
        y = r * np.cos(E_) * np.sin(A_)
        z = r * np.sin(E_)
        inten = rng.uniform(0.0, 1.0, size=x.shape)
        dt = np.full(x.shape, 0.05 * s)
        pts.append(np.stack([x, y, z, inten, dt], axis=1))
    pts = np.concatenate(pts, axis=0).astype(np.float32)
    if shuffle:
        pts = pts[rng.permutation(pts.shape[0])]
    return pts


def uniform_cloud(n, seed=0, margin=2.0, rng_range=(-54.0, -54.0, -5.0, 54.0, 54.0, 3.0), nf=5):
    """uniform-random cloud, some points outside the range on every side."""
    rng = np.random.default_rng(seed)
    lo = np.array(rng_range[:3]) - margin
    hi = np.array(rng_range[3:]) + margin
    xyz = rng.uniform(lo, hi, size=(n, 3))
    extra = rng.uniform(0, 1, size=(n, nf - 3))
    return np.concatenate([xyz, extra], axis=1).astype(np.float32)


def radar_cloud(seed=0, radars=5, sweeps=6, per_sweep=110, clusters=4, cluster_points=60, out_of_range=0.03):
    """Synthetic nuScenes-style radar cloud [N, 45] fp32 laid out like `radar_use_dims` (loading.py:618-652):
    x, y, z, rcs, vx_comp, vy_comp, time_diff, dynprop one-hot x8, ambig_state one-hot x5, invalid_state
    one-hot x18, pdh0 ordinal x7.  `radars` sensors around the ego x `sweeps` sweeps of about `per_sweep`
    returns each (a few thousand points in all), a fraction `out_of_range` outside +-51.2 m, and `clusters`
    dense groups of `cluster_points` returns in one 0.8 m pillar each, so that some pillars exceed P = 20."""
    rng = np.random.default_rng(seed)
    yaws = np.deg2rad([0.0, 50.0, -50.0, 130.0, -130.0])[:radars]
    rows = []
    for s in range(sweeps):
        for yaw in yaws:
            k = rng.poisson(per_sweep)
            az = yaw + rng.uniform(-0.6, 0.6, k)
            r = rng.gamma(2.0, 12.0, k) + 1.0
            rows.append(np.stack([r * np.cos(az), r * np.sin(az), rng.normal(0.5, 0.6, k),
                                  np.full(k, 0.05 * s)], 1))
    for c in range(clusters):
        centre = (rng.integers(-60, 60, 2) + 0.5) * 0.8
        off = rng.uniform(-0.35, 0.35, (cluster_points, 2))
        rows.append(np.stack([centre[0] + off[:, 0], centre[1] + off[:, 1], rng.normal(0.5, 0.3, cluster_points),
                              np.full(cluster_points, 0.05 * (c % sweeps))], 1))
    base = np.concatenate(rows, 0)
    n = base.shape[0]
    far = rng.uniform(size=n) < out_of_range
    base[far, :2] *= rng.uniform(1.6, 3.0, (int(far.sum()), 1))
    rcs = rng.uniform(-10.0, 40.0, n)
    vel = rng.normal(0.0, 3.0, (n, 2))
    def one_hot(k, width):
        out = np.zeros((n, width))
        out[np.arange(n), k] = 1.0
        return out
    pdh = rng.integers(0, 8, n)
    pts = np.concatenate([base[:, :3], rcs[:, None], vel, base[:, 3:4],
                          one_hot(rng.integers(0, 8, n), 8), one_hot(rng.integers(0, 5, n), 5),
                          one_hot(rng.integers(0, 18, n), 18),
                          (pdh[:, None] > np.arange(7)[None, :]).astype(np.float64)], 1).astype(np.float32)
    return pts[rng.permutation(n)]


# CenterHead tasks of the nuScenes configs (centerhead/default.yaml: tasks) with typical (w, l, h) in metres
CENTERHEAD_TASKS = [
    [("car", (1.95, 4.6, 1.7))],
    [("truck", (2.5, 6.9, 2.8)), ("construction_vehicle", (2.9, 6.4, 3.2))],
    [("bus", (2.9, 11.5, 3.5)), ("trailer", (2.9, 12.0, 3.9))],
    [("barrier", (2.5, 0.5, 1.0))],
    [("motorcycle", (0.8, 2.1, 1.5)), ("bicycle", (0.6, 1.8, 1.3))],
    [("pedestrian", (0.7, 0.7, 1.8)), ("traffic_cone", (0.3, 0.3, 1.1))],
]
# the box post-processing part of test_cfg (centerhead/default.yaml, lssfpn/camera+radar/default.yaml)
CENTERHEAD_TEST_CFG = dict(post_center_limit_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0], max_per_img=500,
                           min_radius=[4, 12, 10, 1, 0.85, 0.175], score_threshold=0.1, pre_max_size=1000,
                           post_max_size=83, nms_thr=0.2)
CENTERHEAD_RADAR_NMS_TYPE = ["circle", "rotate", "rotate", "circle", "rotate", "rotate"]
CENTERHEAD_RADAR_NMS_SCALE = [[1.0], [1.0, 1.0], [1.0, 1.0], [1.0], [1.0, 1.0], [2.5, 4.0]]


def gt_boxes(seed=0, batch=1, min_boxes=40, max_boxes=120, extent=54.0):
    """nuScenes-shaped ground truth for the head training targets: (boxes, labels), lists over samples of
    [n, 9] fp32 LiDARInstance3DBoxes tensors (x, y, z_bottom, dx, dy, dz, yaw, vx, vy) and [n] int64 labels
    0..9 (the classes of CENTERHEAD_TASKS in task order), n in [min_boxes, max_boxes].  Sizes are the class's
    (w, l, h) jittered by +-15 %, centres uniform over +-extent m (so some lie off a +-51.2 m map), yaw in
    [-pi, pi), velocities N(0, 3) m/s (0 for barriers and cones)."""
    rng = np.random.default_rng(seed)
    sizes = [s for classes in CENTERHEAD_TASKS for _, s in classes]
    static = {5, 9}                                      # barrier, traffic_cone
    boxes, labels = [], []
    for _ in range(batch):
        n = int(rng.integers(min_boxes, max_boxes + 1))
        lab = rng.integers(0, len(sizes), n)
        whl = np.array([sizes[l] for l in lab]) * rng.uniform(0.85, 1.15, (n, 3))
        vel = rng.normal(0.0, 3.0, (n, 2)) * (~np.isin(lab, list(static)))[:, None]
        b = np.concatenate([rng.uniform(-extent, extent, (n, 2)), rng.uniform(-2.5, 0.5, (n, 1)), whl,
                            rng.uniform(-math.pi, math.pi, (n, 1)), vel], 1)
        boxes.append(torch.from_numpy(b.astype(np.float32)))
        labels.append(torch.from_numpy(lab.astype(np.int64)))
    return boxes, labels


TRANSFUSION_CODER = dict(pc_range=[-51.2, -51.2], voxel_size=[0.1, 0.1], out_size_factor=8, code_size=10)
TRANSFUSION_TRAIN_CFG = dict(point_cloud_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], grid_size=[1024, 1024, 1],
                             voxel_size=[0.1, 0.1, 0.2], out_size_factor=8, gaussian_overlap=0.1, min_radius=2,
                             pos_weight=-1,
                             assigner=dict(type="HungarianAssigner3D",
                                           iou_calculator=dict(type="BboxOverlaps3D", coordinate="lidar"),
                                           cls_cost=dict(type="FocalLossCost", gamma=2.0, alpha=0.25, weight=0.15),
                                           reg_cost=dict(type="BBoxBEVL1Cost", weight=0.25),
                                           iou_cost=dict(type="IoU3DCost", weight=0.25)))


def transfusion_predictions(seed, batch, gt, num_proposals=200, num_classes=10, layers=1):
    """Raw TransFusionHead predictions for the training-target assignment, shaped as the head emits them (the
    transfusion/default.yaml coder: pc_range -51.2, voxel 0.1, out_size_factor 8): dict(heatmap [B, K, N] logits,
    center [B, 2, N] feature cells, height [B, 1, N] gravity-centre z, dim [B, 3, N] log sizes, rot [B, 2, N]
    (sin, cos), vel [B, 2, N]) fp32 CPU tensors, N = layers * num_proposals.  gt = (boxes, labels) as gt_boxes
    gives them.  In each layer about half the proposals are jittered copies of gts (their logit raised at the
    gt's label) and the rest random; a few proposals are exact copies of others, so the cost has ties."""
    rng = np.random.default_rng(seed)
    boxes, labels = gt
    P, K, N = num_proposals, num_classes, layers * num_proposals
    cell = TRANSFUSION_CODER["out_size_factor"] * TRANSFUSION_CODER["voxel_size"][0]
    out = {k: np.zeros((batch, r, N), np.float32) for k, r in
           (("heatmap", K), ("center", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2))}
    for b in range(batch):
        g = boxes[b].numpy().astype(np.float64) if len(boxes[b]) else np.zeros((0, 9))
        lab = labels[b].numpy()
        for l in range(layers):
            cols = slice(l * P, (l + 1) * P)
            heat = rng.normal(-2.0, 1.0, (K, P))
            xy = rng.uniform(-51.2, 51.2, (P, 2))
            z = rng.uniform(-2.0, 1.0, P)
            d = np.log(rng.uniform(0.3, 6.0, (P, 3)))
            yaw = rng.uniform(-np.pi, np.pi, P)
            vel = rng.normal(0.0, 2.0, (P, 2))
            n_copy = min(len(g), P // 2)
            if n_copy:
                pick = rng.choice(len(g), n_copy, replace=False)
                dst = rng.choice(P, n_copy, replace=False)
                src = g[pick]
                xy[dst] = src[:, :2] + rng.normal(0.0, 0.3, (n_copy, 2))
                z[dst] = src[:, 2] + src[:, 5] * 0.5 + rng.normal(0.0, 0.1, n_copy)
                d[dst] = np.log(src[:, 3:6]) + rng.normal(0.0, 0.08, (n_copy, 3))
                yaw[dst] = src[:, 6] + rng.normal(0.0, 0.15, n_copy)
                vel[dst] = src[:, 7:9] + rng.normal(0.0, 0.3, (n_copy, 2))
                heat[lab[pick], dst] += rng.uniform(1.0, 4.0, n_copy)
            out["heatmap"][b, :, cols] = heat
            out["center"][b, :, cols] = ((xy - np.array(TRANSFUSION_CODER["pc_range"])) / cell).T
            out["height"][b, 0, cols] = z
            out["dim"][b, :, cols] = d.T
            out["rot"][b, :, cols] = np.stack([np.sin(yaw), np.cos(yaw)]) * rng.uniform(0.8, 1.2, P)
            out["vel"][b, :, cols] = vel.T
            dup = rng.choice(P, 8, replace=False) + l * P            # exact duplicate proposals: cost ties
            for key in out:
                out[key][b, :, dup[4:]] = out[key][b, :, dup[:4]]
    return {k: torch.from_numpy(v) for k, v in out.items()}


def centerhead_detections(seed=0, batch=1, max_num=500):
    """What CenterPointBBoxCoder.decode hands to the NMS step, per task and sample: a list over the six
    tasks of a list over samples of dict(bboxes [n, 9] fp32 (x, y, z, w, l, h, yaw, vx, vy), scores [n]
    fp32, labels [n] int64).  30-80 objects per (task, sample), each seen as 4-10 jittered candidates
    (n capped at max_num, the coder's max_num), centres within +-61 m, yaw in [-pi, pi), scores distinct,
    in random order and spread over (0.02, 0.97), so that some fall below the 0.1 score threshold."""
    rng = np.random.default_rng(seed)
    out = []
    for classes in CENTERHEAD_TASKS:
        task = []
        for _ in range(batch):
            rows, labels = [], []
            for _ in range(int(rng.integers(30, 81))):
                lab = int(rng.integers(len(classes)))
                w, l, h = np.array(classes[lab][1]) * rng.uniform(0.85, 1.15, 3)
                x, y = rng.uniform(-61.0, 61.0, 2)
                z, yaw = rng.uniform(-2.0, 1.0), rng.uniform(-math.pi, math.pi)
                vx, vy = rng.normal(0, 3, 2)
                for _ in range(int(rng.integers(4, 11))):
                    jit = rng.normal(0, 1, 9) * [0.15 * w, 0.15 * l, 0.1, 0.05 * w, 0.05 * l, 0.05 * h, 0.15,
                                                 0.3, 0.3]
                    rows.append(np.array([x, y, z, w, l, h, yaw, vx, vy]) + jit)
                    labels.append(lab)
            n = min(len(rows), max_num)
            pick = rng.permutation(len(rows))[:n]
            b = np.array(rows)[pick]
            b[:, :2] = b[:, :2].clip(-61.0, 61.0)
            b[:, 6] = (b[:, 6] + math.pi) % (2 * math.pi) - math.pi
            scores = (rng.permutation(n) + rng.uniform(0.05, 0.95, n)) / n * 0.95 + 0.02
            task.append(dict(bboxes=torch.from_numpy(b.astype(np.float32)),
                             scores=torch.from_numpy(scores.astype(np.float32)),
                             labels=torch.from_numpy(np.array(labels)[pick].astype(np.int64))))
        out.append(task)
    return out
