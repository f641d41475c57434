"""The multi-sweep radar cloud of a nuScenes-shaped frame: five radars x six sweeps of raw 18-column rows through
LoadRadarPointsMultiSweeps (the shipped config: radar_use_dims, compensate_velocity) and PointsRangeFilter's radar
face, into the radar encoder (RadarFeatureNet [128, 128, 128, 64] + scatter on the 128 x 128 grid).

    python tools/radar_sweeps_bench.py OUT_DIR [--rounds 5] [--frames 50] [--rows 125]

Per frame, at B = 1 and B = 4:
  a_host    the reference's lines restated on the host from preloaded raw arrays (tests/radar_sweeps_oracle.py: three
            float64 matmuls, the 58-column encodings, use_dim, torch in_range_bev), the H2D copy of each sample's
            [N, 45] cloud and forward_points on the list
  b_device  one new sweep per radar through put (pinned H2D), the frame's parameter block, and one CUDA graph of
            assemble + forward_points(num_points=)
Every time is per frame, from a host clock around the work that ends in a device synchronise, the median of --rounds
rounds of --frames frames.  Also the kernel time of assemble alone from a torch.profiler run of its own.  The card
name and power limit are read in the same run.  Writes OUT_DIR/radar_sweeps_bench.json.  Needs a CUDA device."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", "tests"))
sys.path.insert(0, HERE)

import radar_sweeps_oracle as O  # noqa: E402
from bevfusion_b200.radar_encoder import RadarEncoder  # noqa: E402
from bevfusion_b200.radar_sweeps import RadarSweepStore  # noqa: E402
from bevfusion_b200.voxelize import Voxelization  # noqa: E402
from encoder_fp16_bench import card_info, graph_of, kernel_us  # noqa: E402

RADARS, SWEEPS = 5, 6
RVS, RPCR = [0.8, 0.8, 8.0], [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]


def per_frame_ms(fn, frames, rounds):
    fn()
    torch.cuda.synchronize()
    res = []
    for _ in range(rounds):
        t = time.perf_counter()
        for _ in range(frames):
            fn()
        torch.cuda.synchronize()
        res.append((time.perf_counter() - t) * 1e3 / frames)
    return statistics.median(res), res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--rows", type=int, default=125, help="raw rows per radar sweep (nuScenes: up to 125)")
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    dev = torch.device("cuda")
    torch.manual_seed(0)
    enc = RadarEncoder(dict(type="RadarFeatureNet", in_channels=45, feat_channels=[128, 128, 128, 64],
                            voxel_size=RVS, point_cloud_range=RPCR, norm_cfg=dict(type="BN1d", eps=1e-3,
                                                                                  momentum=0.01)),
                       dict(type="PointPillarsScatter", in_channels=64, output_shape=[128, 128])).to(dev).eval()
    vox = Voxelization(RVS, RPCR, 10, (30000, 60000)).eval()
    result = {"card": card_info(), "torch_threads": torch.get_num_threads(), "cpu_count": os.cpu_count(),
              "rows_per_sweep": args.rows, "ms_per_frame": {}, "rounds_ms": {}, "rows_kept": {}, "equal": {}}
    for B in (1, 4):
        rng = np.random.default_rng(B)
        # per sample, per radar, a ring of SWEEPS + 1 slots: the frame uses the newest SWEEPS, a new sweep replaces
        # the oldest
        ring = SWEEPS + 1
        n_slots = B * RADARS * ring
        raw = [O.radar_sweep(rng, args.rows) for _ in range(n_slots)]
        poses = [O.radar_pose(rng, (s // ring) % RADARS) for s in range(n_slots)]
        pinned = [torch.from_numpy(r).pin_memory() for r in raw]
        store = RadarSweepStore(n_slots, args.rows, dev, max_batch=B, max_entries=RADARS * SWEEPS)
        for s in range(n_slots):
            store.put(s, pinned[s])
        step = [0]

        def slots_of(b, t):
            return [(b * RADARS + r) * ring + (t - k) % ring for r in range(RADARS) for k in range(SWEEPS)]

        def samples(t):
            return [[(s, poses[s][0], poses[s][1], 0.075 * k) for k, s in enumerate(slots_of(b, t))]
                    for b in range(B)]

        def host_clouds(t):
            out = []
            for b in range(B):
                sl = slots_of(b, t)
                out.append(O.multi_sweeps([raw[s] for s in sl], [poses[s][0] for s in sl], [poses[s][1] for s in sl],
                                          [0.075 * k for k in range(len(sl))], O.SHIPPED_USE_DIM))
            return out

        cap = RADARS * SWEEPS * args.rows
        store.write_frame(samples(0), O.SHIPPED_USE_DIM, True)

        def device_frame():
            out, counts, _ = store.launch(B, 45, cap)
            with torch.no_grad():
                return enc.forward_points(out, vox, num_points=counts)

        g, static_canvas = graph_of(device_frame)

        def a_host():
            step[0] += 1
            clouds = [torch.from_numpy(c).pin_memory().to(dev, non_blocking=True) for c in host_clouds(step[0])]
            with torch.no_grad():
                return enc.forward_points(clouds, vox)

        def b_device():
            step[0] += 1
            t = step[0]
            for b in range(B):
                for r in range(RADARS):
                    s = (b * RADARS + r) * ring + t % ring
                    store.put(s, pinned[s])
            store.write_frame(samples(t), O.SHIPPED_USE_DIM, True)
            g.replay()

        # the two paths give the same canvas on the same frame
        step[0] = 0
        b_device()
        torch.cuda.synchronize()
        dev_canvas = static_canvas.clone()
        step[0] = 0
        host_canvas = a_host()
        result["equal"]["B%d" % B] = bool(torch.equal(dev_canvas, host_canvas))
        result["rows_kept"]["B%d" % B] = [int(c.shape[0]) for c in host_clouds(1)]
        for name, fn in (("a_host", a_host), ("b_device", b_device)):
            med, rounds = per_frame_ms(fn, args.frames, args.rounds)
            result["ms_per_frame"]["%s_B%d" % (name, B)] = med
            result["rounds_ms"]["%s_B%d" % (name, B)] = rounds
        result["kernels_assemble_B%d" % B] = kernel_us(lambda: store.launch(B, 45, cap))
    print(json.dumps({k: v for k, v in result.items() if k != "rounds_ms"}, indent=1), flush=True)
    with open(os.path.join(args.out_dir, "radar_sweeps_bench.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
