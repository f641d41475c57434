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


def augmented_rig(n_cam=6, image_size=(256, 704), batch=1, seed=0):
    """camera_rig under one seeded draw of the reference's training augmentation (configs/nuscenes/default.yaml):
    ImageAug3D per image (resize 0.38-0.55 of 1600x900 -- scaled with the image width, as camera_rig's 0.48 is --,
    bottom crop, random horizontal crop, flip with p = 0.5, rotation +-5.4 deg about the image centre) and, per sample,
    GlobalRotScaleTrans (scale 0.9-1.1, z rotation +-45 deg, translation N(0, 0.5 m)) followed by RandomFlip3D (x and
    y flips, p = 0.5 each).  Returns camera_rig's dict with post_rots / post_trans replaced and extra_rots [B, 3, 3] /
    extra_trans [B, 3] (the lidar augmentation) added; fp32 on the host."""
    rig = camera_rig(n_cam, image_size, batch)
    rng = np.random.RandomState(seed)
    fH, fW = image_size
    width_scale = fW / 704.0
    post_rots = torch.eye(3).repeat(batch, n_cam, 1, 1)
    post_trans = torch.zeros(batch, n_cam, 3)
    for b in range(batch):
        for n in range(n_cam):
            resize = rng.uniform(0.38, 0.55) * width_scale
            new_w, new_h = int(1600 * resize), int(900 * resize)
            crop_h = new_h - fH
            crop_w = int(rng.uniform(0, max(0, new_w - fW)))
            flip = bool(rng.choice([0, 1]))
            theta = math.radians(rng.uniform(-5.4, 5.4))
            rot = resize * np.eye(2)
            tran = -np.array([crop_w, crop_h], dtype=np.float64)
            if flip:
                A = np.array([[-1.0, 0.0], [0.0, 1.0]])
                rot, tran = A @ rot, A @ tran + np.array([fW, 0.0])
            A = np.array([[math.cos(theta), math.sin(theta)], [-math.sin(theta), math.cos(theta)]])
            centre = np.array([fW, fH], dtype=np.float64) / 2.0
            rot, tran = A @ rot, A @ tran + (A @ -centre + centre)
            post_rots[b, n, :2, :2] = torch.from_numpy(rot).float()
            post_trans[b, n, :2] = torch.from_numpy(tran).float()
    extra_rots = torch.zeros(batch, 3, 3)
    extra_trans = torch.zeros(batch, 3)
    for b in range(batch):
        scale = rng.uniform(0.9, 1.1)
        theta = rng.uniform(-0.78539816, 0.78539816)
        t = rng.normal(0.0, 0.5, 3)
        R = np.array([[math.cos(theta), -math.sin(theta), 0.0], [math.sin(theta), math.cos(theta), 0.0],
                      [0.0, 0.0, 1.0]])
        M = np.concatenate([R.T * scale, (t * scale)[:, None]], 1)
        if rng.choice([0, 1]):
            M = np.diag([1.0, -1.0, 1.0]) @ M
        if rng.choice([0, 1]):
            M = np.diag([-1.0, 1.0, 1.0]) @ M
        extra_rots[b] = torch.from_numpy(M[:, :3]).float()
        extra_trans[b] = torch.from_numpy(M[:, 3]).float()
    rig.update(post_rots=post_rots.contiguous(), post_trans=post_trans.contiguous(),
               extra_rots=extra_rots.contiguous(), extra_trans=extra_trans.contiguous())
    return rig


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


def transfusion_heatmap(seed, batch, num_classes=10, height=128, width=128, dtype=torch.float32, gt=None,
                        extent=54.0):
    """Dense TransFusion heatmap logits [B, C, H, W] on the CPU, shaped like a trained head's output: a smooth
    background near logit -5 (sigmoid about 0.007; iid N(0, 1) noise blurred over 3 x 3 cells, so that a few per cent
    of the cells are local maxima) plus one Gaussian blob per object at its label's channel, centred on the object's
    cell, with a peak logit raise of 3 to 9 and a sigma of half the object's footprint in cells (at least 0.7).
    gt = (boxes, labels) as gt_boxes gives them (default gt_boxes(seed, batch)); a centre maps to
    column (x + extent) / (2 extent) * W and row (y + extent) / (2 extent) * H, and objects off the map are skipped.
    Labels at or above num_classes are skipped.  Computed in float64, returned in `dtype`."""
    rng = np.random.default_rng(seed)
    boxes, labels = gt if gt is not None else gt_boxes(seed=seed, batch=batch)
    noise = rng.standard_normal((batch, num_classes, height + 2, width + 2))
    base = sum(noise[:, :, dy:dy + height, dx:dx + width] for dy in range(3) for dx in range(3)) / 3.0
    heat = base * 0.5 - 5.0
    rows, cols = np.arange(height)[:, None], np.arange(width)[None, :]
    for b in range(batch):
        g = boxes[b].numpy().astype(np.float64)
        lab = labels[b].numpy()
        for i in range(len(g)):
            if lab[i] >= num_classes:
                continue
            cx = (g[i, 0] + extent) / (2 * extent) * width
            cy = (g[i, 1] + extent) / (2 * extent) * height
            if not (0 <= cx < width and 0 <= cy < height):
                continue
            sigma = max(0.7, 0.5 * max(g[i, 3] / (2 * extent) * width, g[i, 4] / (2 * extent) * height))
            amp = rng.uniform(3.0, 9.0)
            heat[b, lab[i]] += amp * np.exp(-((cols - cx) ** 2 + (rows - cy) ** 2) / (2 * sigma * sigma))
    return torch.from_numpy(heat).to(dtype).contiguous()


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


def centerhead_coder_cfg(height=128, width=128, extent=54.0, max_num=500, score_threshold=0.1):
    """The CenterPointBBoxCoder fields that put a +-extent m scene on a height x width map at out_size_factor 8 (the
    nuScenes configs: extent 54, 180 x 180, voxel 0.075).  The coder's x runs along the map's rows."""
    return dict(pc_range=[-extent, -extent], out_size_factor=8,
                voxel_size=[2 * extent / height / 8, 2 * extent / width / 8],
                post_center_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0], max_num=max_num,
                score_threshold=score_threshold, code_size=9)


def centerhead_head_outputs(seed, batch, height=128, width=128, gt=None, extent=54.0):
    """Raw CenterHead outputs for the six nuScenes tasks (CENTERHEAD_TASKS), shaped like a trained head's: a list
    over tasks of dict(heatmap [B, cat, H, W] logits, reg [B, 2, H, W], height [B, 1, H, W], dim [B, 3, H, W] log
    sizes, rot [B, 2, H, W] (sine, cosine), vel [B, 2, H, W]) fp32 CPU tensors for centerhead_coder_cfg(height,
    width, extent).  The heatmap is built like transfusion_heatmap: a smooth background around logit -3.5 (the
    head's bias initialisation, -2.19, is sigmoid 0.1; a trained background lies below it) plus one Gaussian blob
    per object of gt = (boxes, labels) (default gt_boxes(seed, batch)) in its class's channel, of a sigma of a quarter
    of the object's footprint in cells (0.7 to 2), so that a few hundred
    cells per task and sample exceed a 0.1 score threshold.  The regression maps hold the object's values (centre
    offset, gravity-centre z, log size, yaw, velocity, lightly jittered) within two cells of its centre and noise
    elsewhere.  The box x axis runs along the rows, as the coder decodes it."""
    rng = np.random.default_rng(seed)
    boxes, labels = gt if gt is not None else gt_boxes(seed=seed, batch=batch)
    first = np.cumsum([0] + [len(c) for c in CENTERHEAD_TASKS])
    rows, cols = np.arange(height)[:, None], np.arange(width)[None, :]
    out = []
    for t, classes in enumerate(CENTERHEAD_TASKS):
        cat = len(classes)
        noise = rng.standard_normal((batch, cat, height + 2, width + 2))
        heat = sum(noise[:, :, dy:dy + height, dx:dx + width] for dy in range(3) for dx in range(3)) / 6.0 - 3.5
        reg = rng.uniform(0.0, 1.0, (batch, 2, height, width))
        hei = rng.normal(-0.5, 1.0, (batch, 1, height, width))
        dim = np.log(rng.uniform(0.3, 8.0, (batch, 3, height, width)))
        rot = rng.normal(0.0, 0.6, (batch, 2, height, width))
        vel = rng.normal(0.0, 1.0, (batch, 2, height, width))
        for b in range(batch):
            g = boxes[b].numpy().astype(np.float64)
            lab = labels[b].numpy()
            for i in np.nonzero((lab >= first[t]) & (lab < first[t + 1]))[0]:
                cx = (g[i, 0] + extent) / (2 * extent) * height          # x along the rows
                cy = (g[i, 1] + extent) / (2 * extent) * width
                if not (0 <= cx < height and 0 <= cy < width):
                    continue
                sigma = min(2.0, max(0.7, 0.25 * max(g[i, 3] / (2 * extent) * height, g[i, 4] / (2 * extent) * width)))
                heat[b, lab[i] - first[t]] += rng.uniform(2.0, 7.0) * np.exp(
                    -((rows - cx) ** 2 + (cols - cy) ** 2) / (2 * sigma * sigma))
                r0, r1 = max(int(cx) - 2, 0), min(int(cx) + 3, height)
                c0, c1 = max(int(cy) - 2, 0), min(int(cy) + 3, width)
                n = (r1 - r0, c1 - c0)
                reg[b, 0, r0:r1, c0:c1] = cx - np.arange(r0, r1)[:, None] + rng.normal(0, 0.05, n)
                reg[b, 1, r0:r1, c0:c1] = cy - np.arange(c0, c1)[None, :] + rng.normal(0, 0.05, n)
                hei[b, 0, r0:r1, c0:c1] = g[i, 2] + 0.5 * g[i, 5] + rng.normal(0, 0.05, n)
                for d in range(3):
                    dim[b, d, r0:r1, c0:c1] = np.log(g[i, 3 + d]) + rng.normal(0, 0.03, n)
                yaw = g[i, 6] + rng.normal(0, 0.05, n)
                rot[b, 0, r0:r1, c0:c1], rot[b, 1, r0:r1, c0:c1] = np.sin(yaw), np.cos(yaw)
                for d in range(2):
                    vel[b, d, r0:r1, c0:c1] = g[i, 7 + d] + rng.normal(0, 0.1, n)
        out.append({k: torch.from_numpy(v.astype(np.float32)).contiguous() for k, v in
                    dict(heatmap=heat, reg=reg, height=hei, dim=dim, rot=rot, vel=vel).items()})
    return out


# ---- BEV map segmentation ------------------------------------------------------------------------------------------
MAP_CLASSES = ("drivable_area", "ped_crossing", "walkway", "stop_line", "carpark_area", "divider")
MAP_SEG_CFG = dict(input_scope=[[-51.2, 51.2, 0.8], [-51.2, 51.2, 0.8]],
                   output_scope=[[-50, 50, 0.5], [-50, 50, 0.5]])   # configs/nuscenes/seg/default.yaml


def map_seg_features(seed=0, batch=1, channels=512, height=128, width=128, dtype=torch.float32):
    """Seeded BEV features [B, C, H, W]: smooth fields (a few low-frequency sinusoids per channel) plus noise, the
    value range of a decoder neck's ReLU output."""
    g = torch.Generator().manual_seed(seed)
    yy = torch.linspace(0, 1, height)[:, None]
    xx = torch.linspace(0, 1, width)[None, :]
    f = torch.rand((batch, channels, 3, 3), generator=g) * 6.0
    ph = torch.rand((batch, channels, 3), generator=g) * 6.3
    x = torch.zeros((batch, channels, height, width))
    for k in range(3):
        x += torch.sin(f[:, :, k, 0, None, None] * xx + f[:, :, k, 1, None, None] * yy + ph[:, :, k, None, None])
    x = torch.relu(x + 0.3 * torch.randn((batch, channels, height, width), generator=g))
    return x.to(dtype).contiguous()


def map_seg_masks(seed=0, batch=1, height=200, width=200, classes=MAP_CLASSES, dtype=torch.int64):
    """Seeded BEV map masks [B, K, H, W] with plausible shapes: drivable area as the union of a few straight roads
    (axis-aligned or slanted bands) and a roundabout disc; pedestrian crossings as striped patches where roads meet
    the edge of an intersection; walkways as bands along the road borders; stop lines as thin bars across a road;
    car parks as rectangles off the road; dividers as thin lines along road centres.  Classes beyond these six get
    random blobs.  dtype int64 is the loader's np.long."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:height, 0:width].astype(np.float64)
    out = np.zeros((batch, len(classes), height, width), np.uint8)
    for b in range(batch):
        road = np.zeros((height, width), bool)
        centre = np.zeros((height, width), bool)
        walk = np.zeros((height, width), bool)
        cross = np.zeros((height, width), bool)
        stop = np.zeros((height, width), bool)
        for _ in range(rng.integers(2, 5)):
            ang = rng.choice([0.0, np.pi / 2, rng.uniform(0, np.pi)])
            off = rng.uniform(-0.35, 0.35) * min(height, width)
            half = rng.uniform(6, 14)
            d = (xx - width / 2) * np.sin(ang) - (yy - height / 2) * np.cos(ang) - off
            along = (xx - width / 2) * np.cos(ang) + (yy - height / 2) * np.sin(ang)
            road |= np.abs(d) <= half
            centre |= np.abs(d) <= 0.6
            walk |= (np.abs(d) > half) & (np.abs(d) <= half + 4)
            a0 = rng.uniform(-0.3, 0.3) * min(height, width)
            cross |= (np.abs(d) <= half) & (np.abs(along - a0) <= 4) & ((np.floor(d / 2) % 2) == 0)
            stop |= (np.abs(d) <= half) & (np.abs(along - a0 - 6) <= 0.75) & (d > 0)
        cy, cx, r = rng.uniform(0.3, 0.7) * height, rng.uniform(0.3, 0.7) * width, rng.uniform(8, 20)
        road |= (yy - cy) ** 2 + (xx - cx) ** 2 <= r * r
        park = np.zeros((height, width), bool)
        for _ in range(rng.integers(1, 4)):
            y0, x0 = rng.integers(0, height - 20), rng.integers(0, width - 20)
            park[y0:y0 + rng.integers(8, 20), x0:x0 + rng.integers(8, 20)] = True
        park &= ~road
        shapes = {"drivable_area": road, "ped_crossing": cross, "walkway": walk & ~road, "stop_line": stop,
                  "carpark_area": park, "divider": centre & road}
        for k, name in enumerate(classes):
            m = shapes.get(name)
            if m is None:
                y0, x0 = rng.uniform(0, height), rng.uniform(0, width)
                m = (yy - y0) ** 2 + (xx - x0) ** 2 <= rng.uniform(5, 25) ** 2
            out[b, k] = m
    return torch.from_numpy(out).to(dtype)
