"""GlobalRotScaleTrans + RandomFlip3D + the range and name filters of a training frame, on the device and on the host.
Each sample is the key and nine sweeps of 34,720 five-float rows (tools/lidar_sweeps_bench.py's spin) and 60 GT boxes.

    python tools/lidar_aug_bench.py OUT_DIR [--rounds 5] [--frames 20]

For B = 1 and 4:
  assemble_plain   SweepStore.launch with the range filter, as a CUDA graph replay
  assemble_aug     the same launch with a LidarAug (the augmentation fused into the sweep kernels), graph replay
  box_aug          LidarAug.boxes on the padded boxes, graph replay
  write_and_aug    LidarAug.write of new draws + the two graphs above: the per-frame device cost of the stages
  host_lines       the reference's lines for the same stages on the host, on each sample's merged cloud and boxes
                   (torch CPU rotate / translate / scale / flip, in_range_3d, the box transforms, in_range_bev,
                   limit_yaw and the name filter), without the copy of the result to the device
Every time is per frame, from a host clock around the work that ends in a device synchronise, the median of --rounds
rounds of --frames frames; kernel times of assemble with and without aug come from a torch.profiler run of their own.
The card name and power limit are read in the same run.  Writes OUT_DIR/lidar_aug_bench.json.  Needs a CUDA device."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bevfusion_b200.head_targets import pad_gt  # noqa: E402
from bevfusion_b200.lidar_aug import GlobalRotScaleTrans, LidarAug, RandomFlip3D, draw_sample  # noqa: E402
from bevfusion_b200.lidar_sweeps import SweepStore  # noqa: E402
from encoder_fp16_bench import card_info, graph_of, kernel_us  # noqa: E402
from lidar_sweeps_bench import LOAD_DIM, PCR, ROWS, SWEEPS, USE_DIM, per_frame_ms, pose, sweep  # noqa: E402

CAP = SWEEPS * ROWS
N_BOXES = 60
CLASSES = 10


def boxes_of(rng):
    b = np.zeros((N_BOXES, 9), np.float32)
    b[:, :2] = rng.uniform(-60, 60, (N_BOXES, 2))
    b[:, 2] = rng.uniform(-3, 1, N_BOXES)
    b[:, 3:6] = rng.uniform(0.3, 12, (N_BOXES, 3))
    b[:, 6] = rng.uniform(-np.pi, np.pi, N_BOXES)
    b[:, 7:9] = rng.normal(0, 5, (N_BOXES, 2))
    return b, rng.integers(-1, CLASSES, N_BOXES)


def host_lines(points, boxes, labels, d):
    """transforms_3d.py:203-232, 325-353, 594-606, 544-575, 628-635 with the point and box classes' methods inlined"""
    pts, bx = points.clone(), boxes.clone()
    if d.scale is not None:
        a = pts.new_tensor(-d.theta)
        s, c = torch.sin(a), torch.cos(a)
        pts[:, :3] = pts[:, :3] @ a.new_tensor([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T
        pts[:, :3] += pts.new_tensor(d.translation)
        pts[:, :3] *= d.scale
        a = bx.new_tensor(d.theta)
        s, c = torch.sin(a), torch.cos(a)
        R = bx.new_tensor([[c, -s, 0], [s, c, 0], [0, 0, 1]])
        bx[:, :3] = bx[:, :3] @ R
        bx[:, 6] += a
        bx[:, 7:9] = bx[:, 7:9] @ R[:2, :2]
        bx[:, :3] += bx.new_tensor(d.translation)
        bx[:, :6] *= d.scale
        bx[:, 7:] *= d.scale
    if d.flip_horizontal:
        pts[:, 1] = -pts[:, 1]
        bx[:, 1::7] = -bx[:, 1::7]
        bx[:, 6] = -bx[:, 6] + np.pi
    if d.flip_vertical:
        pts[:, 0] = -pts[:, 0]
        bx[:, 0::7] = -bx[:, 0::7]
        bx[:, 6] = -bx[:, 6]
    r = np.array(PCR, np.float32)
    keep = ((pts[:, 0] > r[0]) & (pts[:, 1] > r[1]) & (pts[:, 2] > r[2]) & (pts[:, 0] < r[3]) & (pts[:, 1] < r[4])
            & (pts[:, 2] < r[5]))
    pts = pts[keep]
    m = (bx[:, 0] > r[0]) & (bx[:, 1] > r[1]) & (bx[:, 0] < r[3]) & (bx[:, 1] < r[4])
    bx, lab = bx[m], labels[m.numpy()]
    bx[:, 6] = bx[:, 6] - torch.floor(bx[:, 6] / (2 * np.pi) + 0.5) * (2 * np.pi)
    named = np.array([n in range(CLASSES) for n in lab], dtype=np.bool_)
    return pts, bx[named], lab[named]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=20)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    dev = torch.device("cuda")
    rng = np.random.default_rng(0)
    raw = [sweep(rng) for _ in range(SWEEPS + 1)]
    poses = [pose(rng, k) for k in range(SWEEPS + 1)]
    store = SweepStore(SWEEPS + 1, ROWS, LOAD_DIM, dev, max_batch=4)
    for k in range(SWEEPS + 1):
        store.put(k, torch.from_numpy(raw[k]).pin_memory())
    sample = (0, [(s, poses[s][0], poses[s][1], 0.05 * s) for s in range(1, SWEEPS)])
    draw_rng = np.random.RandomState(0)
    grst = GlobalRotScaleTrans([0.9, 1.1], [-0.78539816, 0.78539816], 0.5, True, rng=draw_rng)
    flip = RandomFlip3D(rng=draw_rng)
    result = {"card": card_info(), "torch_threads": torch.get_num_threads(), "rows_in_per_sample": SWEEPS * ROWS,
              "boxes_per_sample": N_BOXES, "ms_per_frame": {}, "kernels": {}}
    for B in (1, 4):
        # the merged clouds for the host lines first: assemble() rewrites the frame's parameter block, and every
        # launch below must read the block with the range filter on
        merged_host = [m.cpu() for m in store.assemble([sample] * B, USE_DIM, point_cloud_range=None)]
        store.write_frame([sample] * B, USE_DIM, point_cloud_range=PCR)
        aug = LidarAug(B, dev)
        draws = [draw_sample(grst, flip) for _ in range(B)]
        aug.write(draws)
        boxes = [boxes_of(rng) for _ in range(B)]
        pb, pl, pc = pad_gt([torch.from_numpy(b) for b, _ in boxes],
                            [torch.from_numpy(l.astype(np.int32)).to(dev) for _, l in boxes])
        # the timed launches filter: check that their kept rows are the host lines' for the block's draws
        out, counts, _ = store.launch(B, 5, CAP, aug)
        first = host_lines(merged_host[0], torch.from_numpy(boxes[0][0]), boxes[0][1], draws[0])[0]
        assert torch.equal(out[0, :int(counts[0])].cpu().view(torch.int32), first.view(torch.int32))
        result["rows_kept_B%d" % B] = [int(c) for c in counts.tolist()]
        g_plain, _ = graph_of(lambda: store.launch(B, 5, CAP))
        g_aug, _ = graph_of(lambda: store.launch(B, 5, CAP, aug))
        g_box, _ = graph_of(lambda: aug.boxes(pb, pl, pc, PCR, CLASSES))

        def write_and_aug():
            aug.write([draw_sample(grst, flip) for _ in range(B)])
            g_aug.replay()
            g_box.replay()

        def host():
            for b in range(B):
                host_lines(merged_host[b], torch.from_numpy(boxes[b][0]), boxes[b][1], draw_sample(grst, flip))

        for name, fn in (("assemble_plain", g_plain.replay), ("assemble_aug", g_aug.replay),
                         ("box_aug", g_box.replay), ("write_and_aug", write_and_aug), ("host_lines", host)):
            result["ms_per_frame"]["%s_B%d" % (name, B)] = per_frame_ms(fn, args.frames, args.rounds)[0]
        result["kernels"]["assemble_plain_B%d" % B] = kernel_us(lambda: store.launch(B, 5, CAP))
        result["kernels"]["assemble_aug_B%d" % B] = kernel_us(lambda: store.launch(B, 5, CAP, aug))
    print(json.dumps(result, indent=1), flush=True)
    with open(os.path.join(args.out_dir, "lidar_aug_bench.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
