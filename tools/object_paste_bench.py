"""ObjectPaste (GT-database sampling) of a training frame, on the device and on the host.  Each sample is the key and
nine sweeps of 34,720 five-float rows (tools/lidar_sweeps_bench.py's spin) and 60 GT boxes; the database is synthetic
(10 classes x 200 objects of 50-800 rows, written as .bin files to a temporary directory) and drawn with the shipped
sample_groups.

    python tools/object_paste_bench.py OUT_DIR [--rounds 5] [--frames 20]

For B = 1 and 4:
  kernels              assemble with aug + range filter, without and with a paste block (torch.profiler, own run)
  assemble_aug         graph replay of the assemble with aug, no paste
  assemble_paste_aug   graph replay of the same assemble with the paste block
  device_frame         per sample ObjectPaste.draw (sampler + collision test), then PasteBlock.write and
                       LidarAug.write, then the paste + aug graph: the per-frame cost of the device path
  host_lines           per sample the reference's host lines on the merged cloud: the same draw, the objects' file
                       loads and translations, remove_points_in_boxes (points_in_rbbox through numba when it is
                       installed, else numpy) and the cat, without the augmentation or the copy to the device
Before timing, the device cloud of sample 0 is checked against the host lines followed by the augmentation and the
range filter.  Times are per frame, from a host clock around work that ends in a device synchronise, the median of
--rounds rounds of --frames frames.  The card name and power limit are read in the same run.  Writes
OUT_DIR/object_paste_bench.json.  Needs a CUDA device."""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

from bevfusion_b200 import object_paste as OP  # noqa: E402
from bevfusion_b200.lidar_aug import GlobalRotScaleTrans, LidarAug, RandomFlip3D, draw_sample  # noqa: E402
from bevfusion_b200.lidar_sweeps import SweepStore  # noqa: E402
from encoder_fp16_bench import card_info, graph_of, kernel_us  # noqa: E402
from lidar_aug_bench import boxes_of, host_lines  # noqa: E402
from lidar_sweeps_bench import LOAD_DIM, PCR, ROWS, SWEEPS, USE_DIM, per_frame_ms, pose, sweep  # noqa: E402

CLASSES = ["car", "truck", "construction_vehicle", "bus", "trailer", "barrier", "motorcycle", "bicycle", "pedestrian",
           "traffic_cone"]
GROUPS = {"car": 2, "truck": 3, "construction_vehicle": 7, "bus": 4, "trailer": 6, "barrier": 2, "motorcycle": 6,
          "bicycle": 6, "pedestrian": 2, "traffic_cone": 2}
PREPARE = {"filter_by_difficulty": [-1], "filter_by_min_points": {c: 5 for c in CLASSES}}
PER_CLASS = 200


def database(rng, root):
    db, k = {}, 0
    for c in CLASSES:
        db[c] = []
        for _ in range(PER_CLASS):
            size = rng.uniform([0.5, 0.5, 1.0], [10.0, 3.0, 3.5])
            box = np.array([*rng.uniform(-50, 50, 2), rng.uniform(-2, 0), *size, rng.uniform(-np.pi, np.pi), 0, 0],
                           np.float32)
            n = int(rng.integers(50, 800))
            pts = np.c_[rng.uniform(-0.45, 0.45, (n, 3)) * size, rng.uniform(0, 1, (n, 2))].astype(np.float32)
            path = os.path.join(root, "obj_%05d.bin" % k)
            pts.tofile(path)
            db[c].append({"name": c, "path": path, "box3d_lidar": box, "difficulty": 0, "num_points_in_gt": n})
            k += 1
    return db


def removal():
    """points_in_rbbox(...).any(-1) on the host: the reference's numba loop when numba is installed"""
    try:
        import numba
    except ImportError:
        import object_paste_oracle
        return "numpy", object_paste_oracle.inside_any

    @numba.njit
    def inside(points, normal, d):
        out = np.zeros(points.shape[0], np.bool_)
        for i in range(points.shape[0]):
            for j in range(normal.shape[0]):
                ok = True
                for k in range(6):
                    s = points[i, 0] * normal[j, k, 0] + points[i, 1] * normal[j, k, 1] + points[i, 2] * normal[j, k, 2] \
                        + d[j, k]
                    if s >= 0:
                        ok = False
                        break
                if ok:
                    out[i] = True
                    break
        return out

    return "numba", lambda xyz, n, d: inside(np.ascontiguousarray(xyz), n, d)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=20)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    sys.path.insert(0, os.path.join(HERE, "..", "tests"))
    dev = torch.device("cuda")
    rng = np.random.default_rng(0)
    raw = [sweep(rng) for _ in range(SWEEPS + 1)]
    poses = [pose(rng, k) for k in range(SWEEPS + 1)]
    store = SweepStore(SWEEPS + 1, ROWS, LOAD_DIM, dev, max_batch=4)
    for k in range(SWEEPS + 1):
        store.put(k, torch.from_numpy(raw[k]).pin_memory())
    sample = (0, [(s, poses[s][0], poses[s][1], 0.05 * s) for s in range(1, SWEEPS)])
    remove_name, inside = removal()
    with tempfile.TemporaryDirectory() as root:
        sampler = OP.DataBaseSampler(database(rng, root), 1.0, PREPARE, GROUPS, CLASSES,
                                     rng=np.random.RandomState(0))
        paste = OP.ObjectPaste(sampler)
        objects = OP.ObjectStore(sum(int(i["num_points_in_gt"]) for i in sampler.infos), LOAD_DIM, len(sampler.infos),
                                 1024, dev)
        for k, info in enumerate(sampler.infos):
            objects.put(k, OP.load_object_points(info["path"], LOAD_DIM))
        draw_rng = np.random.RandomState(0)
        grst = GlobalRotScaleTrans([0.9, 1.1], [-0.78539816, 0.78539816], 0.5, True, rng=draw_rng)
        flip = RandomFlip3D(rng=draw_rng)
        result = {"card": card_info(), "torch_threads": torch.get_num_threads(), "rows_in_per_sample": SWEEPS * ROWS,
                  "boxes_per_sample": 60, "database_objects": len(sampler.infos), "database_rows": objects.used,
                  "host_removal": remove_name, "ms_per_frame": {}, "kernels": {}}

        def host_paste(cloud, boxes, labels):
            d = paste.draw(boxes, labels)
            if d is None:
                return cloud
            pts = [OP.load_object_points(i["path"], LOAD_DIM)[:, :5].copy() for i in d.infos]
            for p, b in zip(pts, d.boxes):
                p[:, :3] += b[:3]
            keep = ~inside(cloud[:, :3], *OP.box_planes(d.boxes))
            return np.concatenate(pts + [cloud[keep]])

        for B in (1, 4):
            merged = [m.cpu().numpy() for m in store.assemble([sample] * B, USE_DIM, point_cloud_range=None)]
            gts = [boxes_of(rng) for _ in range(B)]
            block = OP.PasteBlock(objects, B, 64)
            aug = LidarAug(B, dev)
            sampler_state = {k: (s.order.copy(), s.idx) for k, s in sampler.samplers.items()}
            draws = [paste.draw(*g) for g in gts]
            block.write(draws, USE_DIM)
            adraws = [draw_sample(grst, flip) for _ in range(B)]
            aug.write(adraws)
            store.write_frame([sample] * B, USE_DIM, point_cloud_range=PCR, paste=block)
            cap = SWEEPS * ROWS + max(block.rows)
            out, counts, status = store.launch(B, 5, cap, aug, block)
            # the host lines from the same sampler state must give the same cloud
            for k, (o, i) in sampler_state.items():
                sampler.samplers[k].order[:], sampler.samplers[k].idx = o, i
            want = host_paste(merged[0], *gts[0])
            want = host_lines(torch.from_numpy(want), torch.from_numpy(gts[0][0]), gts[0][1], adraws[0])[0]
            assert int(status[0]) == 0 and torch.equal(out[0, :int(counts[0])].cpu().view(torch.int32),
                                                       want.view(torch.int32)), "device cloud != host lines"
            result["rows_kept_B%d" % B] = [int(c) for c in counts.tolist()]
            result["objects_kept_B%d" % B] = [0 if d is None else len(d.boxes) for d in draws]
            g_aug, _ = graph_of(lambda: store.launch(B, 5, cap, aug))
            g_paste, _ = graph_of(lambda: store.launch(B, 5, cap, aug, block))

            def device_frame():
                block.write([paste.draw(*g) for g in gts], USE_DIM)
                aug.write([draw_sample(grst, flip) for _ in range(B)])
                g_paste.replay()

            def host():
                for b in range(B):
                    host_paste(merged[b], *gts[b])

            for name, fn in (("assemble_aug", g_aug.replay), ("assemble_paste_aug", g_paste.replay),
                             ("device_frame", device_frame), ("host_lines", host)):
                result["ms_per_frame"]["%s_B%d" % (name, B)] = per_frame_ms(fn, args.frames, args.rounds)[0]
            block.write(draws, USE_DIM)
            result["kernels"]["assemble_aug_B%d" % B] = kernel_us(lambda: store.launch(B, 5, cap, aug))
            result["kernels"]["assemble_paste_aug_B%d" % B] = kernel_us(lambda: store.launch(B, 5, cap, aug, block))
    print(json.dumps(result, indent=1), flush=True)
    with open(os.path.join(args.out_dir, "object_paste_bench.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
