"""The multi-sweep LiDAR cloud of one nuScenes sample: the key and nine earlier sweeps of 34,720 five-float rows through
LoadPointsFromMultiSweeps (remove_close, pose transform, time lag) and PointsRangeFilter (voxelnet 0.075 range).

    python tools/lidar_sweeps_bench.py OUT_DIR [--rounds 5] [--frames 20]

  a_host_merge      the reference's lines restated on the host (numpy remove_close, float64 transform, concatenation,
                    torch in_range_3d) plus the H2D copy of the merged cloud
  b_raw_upload      H2D of the ten raw sweeps (pinned) into a SweepStore + assemble(sync=False)
  c_one_sweep_graph H2D of one new sweep + the frame's parameter block + assemble as a CUDA graph replay
  d_device_frame    (c) + voxelize_mean_fused(num_points=) + the eval SparseEncoder, one graph
  d_host_frame      the same frame from a host-merged cloud: (a) + voxelize + encoder, one graph
Every time is per frame, from a host clock around the work that ends in a device synchronise, the median of --rounds
rounds of --frames frames.  Also: kernel times from a torch.profiler run of its own, and the HBM floor of assemble
(every raw row read once, every kept row written once, at the data sheet's 3.35 TB/s).  The card name and power limit
are read in the same run.  Writes OUT_DIR/lidar_sweeps_bench.json.  Needs a CUDA device."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bevfusion_b200.lidar_sweeps import SweepStore  # noqa: E402
from bevfusion_b200.sparse_encoder import voxelnet_0p075_encoder  # noqa: E402
from bevfusion_b200.voxelize import voxelize_mean_fused  # noqa: E402
from encoder_fp16_bench import card_info, graph_of, kernel_us  # noqa: E402

ROWS, SWEEPS, LOAD_DIM, USE_DIM = 34720, 10, 5, [0, 1, 2, 3, 4]
PCR = [-54.0, -54.0, -5.0, 54.0, 54.0, 3.0]
VS, MAX_POINTS, MAX_VOXELS = [0.075, 0.075, 0.2], 10, 160000
CAP = SWEEPS * ROWS
HBM_BYTES_PER_S = 3.35e12


def sweep(rng, n=ROWS):
    """a 32-beam spin out to 70 m: (x, y, z, intensity, ring) float32"""
    r, az = rng.uniform(0.3, 70.0, n), rng.uniform(-np.pi, np.pi, n)
    return np.stack([r * np.cos(az), r * np.sin(az), rng.uniform(-6.0, 4.0, n), rng.uniform(0, 255, n).round(),
                     rng.integers(0, 32, n)], 1).astype(np.float32)


def pose(rng, k):
    yaw = rng.uniform(-0.1, 0.1)
    R = np.array([[np.cos(yaw), -np.sin(yaw), 0.0], [np.sin(yaw), np.cos(yaw), 0.0], [0.0, 0.0, 1.0]])
    return R, np.array([-0.5 * k, rng.uniform(-0.2, 0.2), rng.uniform(-0.02, 0.02)])


def host_merge(key, sweeps, poses, lags):
    """loading.py:186-233 and transforms_3d.py:604-606 as the reference writes them"""
    points = key[:, USE_DIM].copy()
    points[:, 4] = 0
    parts = [points]
    for raw, (R, t), lag in zip(sweeps, poses, lags):
        ps = np.copy(raw).reshape(-1, LOAD_DIM)
        close = np.logical_and(np.abs(ps[:, 0]) < 1.0, np.abs(ps[:, 1]) < 1.0)
        ps = ps[np.logical_not(close)][:, USE_DIM]
        ps[:, :3] = ps[:, :3] @ R.T
        ps[:, :3] += t
        ps[:, 4] = lag
        parts.append(ps)
    out = torch.from_numpy(np.concatenate(parts, 0))
    rng = np.array(PCR, dtype=np.float32)
    mask = ((out[:, 0] > rng[0]) & (out[:, 1] > rng[1]) & (out[:, 2] > rng[2]) & (out[:, 0] < rng[3])
            & (out[:, 1] < rng[4]) & (out[:, 2] < rng[5]))
    return out[mask]


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
    ap.add_argument("--frames", type=int, default=20)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    dev = torch.device("cuda")
    rng = np.random.default_rng(0)
    raw = [sweep(rng) for _ in range(SWEEPS + 1)]          # slot 0 the key, slots 1..10 the sweeps
    poses = [pose(rng, k) for k in range(SWEEPS + 1)]
    lags = [0.05 * k for k in range(SWEEPS + 1)]
    pinned = [torch.from_numpy(r).pin_memory() for r in raw]
    chosen = list(range(1, SWEEPS))                         # key + 9 sweeps = ten sweeps of ROWS rows
    sample = (0, [(s, poses[s][0], poses[s][1], lags[s]) for s in chosen])
    store = SweepStore(SWEEPS + 1, ROWS, LOAD_DIM, dev, max_batch=1)
    for k in range(SWEEPS + 1):
        store.put(k, pinned[k])
    torch.manual_seed(0)
    enc = voxelnet_0p075_encoder().to(dev).eval()

    def merged_on_host():
        return host_merge(raw[0], [raw[s] for s in chosen], [poses[s] for s in chosen], [lags[s] for s in chosen])

    kept = merged_on_host()
    n_kept = kept.shape[0]
    check = store.assemble([sample], USE_DIM, point_cloud_range=PCR)[0]
    assert torch.equal(check.cpu().view(torch.int32), kept.view(torch.int32)), "device cloud differs from the host's"
    rows_in = sum(raw[s].shape[0] for s in [0] + chosen)
    floor_us = (rows_in * LOAD_DIM * 4 + n_kept * 5 * 4) / HBM_BYTES_PER_S * 1e6

    def a_host_merge():
        return merged_on_host().to(dev)

    def b_raw_upload():
        for k in [0] + chosen:
            store.put(k, pinned[k])
        return store.assemble([sample], USE_DIM, point_cloud_range=PCR, cap=CAP, sync=False)

    g_asm, _ = graph_of(lambda: store.launch(1, 5, CAP))
    step = [0]

    def refresh():
        """the newest sweep into its slot (one pinned H2D copy) and the frame's parameter block"""
        step[0] += 1
        store.put(chosen[0], pinned[step[0] % (SWEEPS + 1)])
        store.write_frame([sample], USE_DIM, point_cloud_range=PCR)

    def c_one_sweep_graph():
        refresh()
        g_asm.replay()

    def device_frame():
        out, counts, _ = store.launch(1, 5, CAP)
        f, c, _, nv = voxelize_mean_fused(out[0], VS, PCR, MAX_POINTS, MAX_VOXELS, 0, sync=False, num_points=counts)
        with torch.no_grad():
            return enc(f, c, 1, num_voxels=nv)

    static_pts = torch.zeros((CAP, 5), dtype=torch.float32, device=dev)
    static_n = torch.zeros((1,), dtype=torch.int32, device=dev)

    def host_frame_graph():
        f, c, _, nv = voxelize_mean_fused(static_pts, VS, PCR, MAX_POINTS, MAX_VOXELS, 0, sync=False,
                                          num_points=static_n)
        with torch.no_grad():
            return enc(f, c, 1, num_voxels=nv)

    store.write_frame([sample], USE_DIM, point_cloud_range=PCR)
    g_dev, out_dev = graph_of(device_frame)
    static_pts[:n_kept].copy_(kept.to(dev))
    static_n.fill_(n_kept)
    g_host, out_host = graph_of(host_frame_graph)
    g_dev.replay()
    g_host.replay()
    torch.cuda.synchronize()
    same_frame = bool(torch.equal(out_dev, out_host))

    def d_device_frame():
        refresh()
        g_dev.replay()

    def d_host_frame():
        m = merged_on_host()
        static_pts[:m.shape[0]].copy_(m.pin_memory(), non_blocking=True)
        static_n.fill_(m.shape[0])
        g_host.replay()

    fns = {"a_host_merge": a_host_merge, "b_raw_upload": b_raw_upload, "c_one_sweep_graph": c_one_sweep_graph,
           "d_device_frame": d_device_frame, "d_host_frame": d_host_frame}
    result = {"card": card_info(), "torch_threads": torch.get_num_threads(), "cpu_count": os.cpu_count(),
              "rows_in": rows_in, "rows_kept": n_kept, "hbm_floor_us": floor_us, "device_equals_host_frame": same_frame,
              "ms_per_frame": {}, "rounds_ms": {}}
    for k, fn in fns.items():
        med, rounds = per_frame_ms(fn, args.frames, args.rounds)
        result["ms_per_frame"][k] = med
        result["rounds_ms"][k] = rounds
    result["kernels_assemble"] = kernel_us(lambda: store.launch(1, 5, CAP))
    result["assemble_kernels_share_of_hbm_floor"] = floor_us / result["kernels_assemble"]["device_us_per_call"]
    print(json.dumps({k: v for k, v in result.items() if k not in ("rounds_ms",)}, indent=1), flush=True)
    with open(os.path.join(args.out_dir, "lidar_sweeps_bench.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
