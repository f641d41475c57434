"""GPU: SweepStore.assemble (LoadPointsFromMultiSweeps + PointsRangeFilter on the device) bit-equal to the numpy
restatement of the reference on seeded nuScenes-like sweeps at B = 1 and 4, load_dim 5 and a wider permuted row; empty
keys, empty sweeps, pad copies and clouds the filters empty; kept counts around the ballot and tile sizes; overflow
of cap; voxelize_mean_fused with a device point count against the host-compacted cloud; a CUDA graph of assemble +
voxelize + the eval SparseEncoder replayed over new frames; and a store reused across frames."""
import numpy as np
import pytest
import torch

import lidar_sweeps_oracle as O

pytestmark = pytest.mark.gpu

PCR = [-54.0, -54.0, -5.0, 54.0, 54.0, 3.0]     # voxelnet 0.075
VS = [0.075, 0.075, 0.2]
ROWS = 34720


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


class Scene:
    """ten raw sweeps (slot k holds sweep k; slot 0 is the key) with poses and lags, and the store holding them"""

    def __init__(self, cuda, seed, load_dim=5, n_sweeps=10, rows=None, slot_cap=36000, max_batch=4):
        from bevfusion_b200.lidar_sweeps import SweepStore
        rng = np.random.default_rng(seed)
        rows = rows or [int(rng.integers(ROWS - 3000, ROWS + 1)) for _ in range(n_sweeps + 1)]
        self.raw = [O.nuscenes_sweep(rng, n, load_dim) for n in rows]
        self.poses = [O.nuscenes_pose(rng, k) for k in range(len(rows))]
        self.lags = [0.05 * k + 1e-3 * rng.uniform() for k in range(len(rows))]
        self.store = SweepStore(len(rows), slot_cap, load_dim, cuda, max_batch=max_batch)
        for k, r in enumerate(self.raw):
            self.store.put(k, torch.from_numpy(r).pin_memory() if k % 2 else torch.from_numpy(r).to(cuda))

    def sample(self, key, chosen):
        return key, [(s, self.poses[s][0], self.poses[s][1], self.lags[s]) for s in chosen]

    def oracle(self, key, chosen, use_dim, key_use_dim=None, **kw):
        return O.multi_sweeps(self.raw[key], [self.raw[s] for s in chosen], [self.poses[s][0] for s in chosen],
                              [self.poses[s][1] for s in chosen], [self.lags[s] for s in chosen], use_dim,
                              key_use_dim, **kw)


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("load_dim,use_dim,key_use_dim", [(5, [0, 1, 2, 3, 4], None),
                                                          (7, [1, 0, 2, 6, 4, 3], [6, 1, 0, 2, 4, 5, 3])])
def test_bit_equal_to_the_reference(cuda, B, load_dim, use_dim, key_use_dim):
    from bevfusion_b200.lidar_sweeps import choose_sweeps
    sc = Scene(cuda, seed=B * 10 + load_dim, load_dim=load_dim)
    np.random.seed(B)
    picks = [(b, [1 + int(c) for c in choose_sweeps(10, 9)]) for b in range(B)]   # 9 of 10, as at test time
    samples = [sc.sample(0 if b == 0 else b, ch) for b, ch in picks]
    for pcr in (PCR, None):
        got = sc.store.assemble(samples, use_dim, key_use_dim, point_cloud_range=pcr)
        for (key, ch), g in zip(samples, got):
            want = sc.oracle(key, [s for s, *_ in ch], use_dim, key_use_dim, point_cloud_range=pcr)
            assert bits_equal(g.cpu().numpy(), want), (key, pcr)


def test_pad_empty_and_filtered_entries(cuda):
    rows = [3000, 0, 2500, 1800]
    sc = Scene(cuda, seed=3, rows=rows, slot_cap=4096)
    far = [-200.0, -200.0, -200.0, -100.0, -100.0, -100.0]       # nothing lies inside
    cases = [((0, []), dict()),                                  # pad: nine copies of the key through remove_close
             ((0, []), dict(sweeps_num=0)),
             ((1, []), dict()),                                  # empty key, padded
             ((1, [2, 3]), dict()),                              # empty key, two sweeps
             ((0, [1, 1, 2]), dict()),                           # an empty sweep between others, a slot twice
             ((2, [3]), dict(point_cloud_range=far)),            # all rows filtered
             ((2, [3, 0]), dict(remove_close=False, point_cloud_range=PCR)),
             ((3, []), dict(pad_empty_sweeps=False))]
    for (key, chosen), kw in cases:
        got = sc.store.assemble([sc.sample(key, chosen)], [0, 1, 2, 3, 4], **kw)[0].cpu().numpy()
        okw = {("remove_close_on" if k == "remove_close" else k): v for k, v in kw.items()}
        want = sc.oracle(key, chosen, [0, 1, 2, 3, 4], **okw)
        assert bits_equal(got, want), (key, chosen, kw)


@pytest.mark.parametrize("layout", ["front", "scattered"])
@pytest.mark.parametrize("kept", [0, 1, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025, 2047, 2049, 5000])
def test_kept_counts_around_ballot_and_tile_sizes(cuda, kept, layout):
    """one sweep of 6000 rows of which `kept` survive, the first ones (so a warp, 256-row round or 1024-row tile
    ends exactly at or next to the last) or scattered; the key keeps 300 of 1100"""
    from bevfusion_b200.lidar_sweeps import SweepStore
    rng = np.random.default_rng(kept)
    key = O.nuscenes_sweep(rng, 1100)
    key[:, 0] = np.where(np.arange(1100) % 11 < 3, 10.0, 80.0)     # 300 inside, 800 outside x
    key[:, 1], key[:, 2] = rng.uniform(-40, 40, 1100), rng.uniform(-4, 2, 1100)
    sweep = O.nuscenes_sweep(rng, 6000)
    sweep[:, :3] = [90.0, 0.0, 0.0]
    inside = np.arange(kept) if layout == "front" else rng.choice(6000, kept, replace=False)
    sweep[inside, 0], sweep[inside, 1] = rng.uniform(2, 40, kept), rng.uniform(-40, 40, kept)
    sweep[inside, 2] = rng.uniform(-4, 2, kept)
    R, t = np.eye(3), np.zeros(3)
    store = SweepStore(2, 6000, 5, cuda, max_batch=1)
    store.put(0, torch.from_numpy(key).to(cuda))
    store.put(1, torch.from_numpy(sweep).to(cuda))
    got = store.assemble([(0, [(1, R, t, 0.25)])], [0, 1, 2, 3, 4], point_cloud_range=PCR)[0].cpu().numpy()
    want = O.multi_sweeps(key, [sweep], [R], [t], [0.25], [0, 1, 2, 3, 4], point_cloud_range=PCR)
    assert want.shape[0] == 300 + kept
    assert bits_equal(got, want)


def test_overflow_writes_cap_rows_and_nothing_past_them(cuda):
    from bevfusion_b200 import _C
    from bevfusion_b200.lidar_sweeps import OVERFLOW
    sc = Scene(cuda, seed=11, rows=[4000, 3000, 2000], slot_cap=4096, max_batch=1)
    sample = sc.sample(0, [2, 1])
    want = sc.oracle(0, [2, 1], [0, 1, 2, 3, 4], point_cloud_range=PCR)
    cap = want.shape[0] - 1
    batch, F, bound = sc.store.write_frame([sample], [0, 1, 2, 3, 4], point_cloud_range=PCR)
    assert (batch, F) == (1, 5) and bound == 9000
    guard = 4096
    buf = torch.full((cap * F + guard,), float("nan"), device=cuda)
    buf.view(torch.int32)[cap * F:] = 0x7f812345                      # a signalling pattern the kernel never makes
    counts = torch.full((1,), -1, dtype=torch.int32, device=cuda)
    status = torch.full((1,), -1, dtype=torch.int32, device=cuda)
    L = _C.lib()
    st = sc.store
    ws = torch.empty(L.bevb200_lidar_sweeps_workspace_bytes(1, st.max_entries, st.slot_cap), dtype=torch.uint8,
                     device=cuda)
    base = st.block.data_ptr()
    _C.check(L.bevb200_lidar_sweeps_assemble(_C.ptr(st.rows), st.slots, st.slot_cap, st.load_dim,
                                             _C.ptr(st.slot_rows), base, base + 128, 1, st.max_entries, F, cap,
                                             _C.ptr(buf), _C.ptr(counts), _C.ptr(status), _C.ptr(ws), ws.numel(),
                                             _C.current_stream(cuda)), "assemble")
    assert int(counts.item()) == cap and int(status.item()) == OVERFLOW
    assert bits_equal(buf[:cap * F].view(cap, F).cpu().numpy(), want[:cap])
    assert bool((buf.view(torch.int32)[cap * F:] == 0x7f812345).all())
    with pytest.raises(ValueError, match="more than cap"):
        sc.store.assemble([sample], [0, 1, 2, 3, 4], point_cloud_range=PCR, cap=cap)
    out, counts, status = sc.store.assemble([sample], [0, 1, 2, 3, 4], point_cloud_range=PCR, cap=cap + 1,
                                            sync=False)
    assert int(status.item()) == 0 and int(counts.item()) == cap + 1
    assert bits_equal(out[0].cpu().numpy(), want)


def test_bad_entries_set_the_status(cuda):
    from bevfusion_b200.lidar_sweeps import BAD_ENTRY, ENTRY_DTYPE
    sc = Scene(cuda, seed=12, rows=[500, 400], slot_cap=512, max_batch=2)
    sc.store.write_frame([sc.sample(0, [1]), sc.sample(1, [0])], [0, 1, 2, 3, 4])
    # sample 1's first entry names a slot the store does not have
    at = 128 + sc.store.max_entries * ENTRY_DTYPE.itemsize + ENTRY_DTYPE.fields["slot"][1]
    sc.store.block[at:at + 4] = torch.tensor([7], dtype=torch.int32).view(torch.uint8).to(cuda)
    out, counts, status = sc.store.launch(2, 5, 2000)
    assert int(status.item()) == BAD_ENTRY
    want = sc.oracle(0, [1], [0, 1, 2, 3, 4])
    assert int(counts[0]) == want.shape[0] and bits_equal(out[0, :want.shape[0]].cpu().numpy(), want)
    assert int(counts[1]) == sc.oracle(1, [0], [0, 1, 2, 3, 4]).shape[0] - 400   # the key's rows are gone


@pytest.mark.parametrize("max_voxels", [120000, 160000])
def test_voxelizer_with_a_device_count(cuda, max_voxels):
    from bevfusion_b200.voxelize import voxelize_mean_fused
    sc = Scene(cuda, seed=21)
    samples = [sc.sample(0, range(1, 10)), sc.sample(10, [9, 3, 5])]
    out, counts, _ = sc.store.assemble(samples, [0, 1, 2, 3, 4], point_cloud_range=PCR, sync=False)
    host = sc.store.assemble(samples, [0, 1, 2, 3, 4], point_cloud_range=PCR)
    for k in range(2):
        got = voxelize_mean_fused(out[k], VS, PCR, 10, max_voxels, k, num_points=counts[k:k + 1])
        want = voxelize_mean_fused(host[k].clone(), VS, PCR, 10, max_voxels, k)
        assert got[0].shape == want[0].shape
        for g, w in zip(got, want):
            assert bits_equal(g.cpu().numpy(), w.cpu().numpy())
        f, c, n, nv = voxelize_mean_fused(out[k], VS, PCR, 10, max_voxels, k, sync=False,
                                          num_points=counts[k:k + 1])
        assert int(nv.item()) == want[0].shape[0]
    # a count of 0 and a count above the rows given (clamped to them)
    zero = torch.zeros(1, dtype=torch.int32, device=cuda)
    assert voxelize_mean_fused(out[0], VS, PCR, 10, max_voxels, num_points=zero)[0].shape[0] == 0
    big = torch.full((1,), out.shape[1] + 5, dtype=torch.int32, device=cuda)
    got = voxelize_mean_fused(out[0], VS, PCR, 10, max_voxels, num_points=big)
    want = voxelize_mean_fused(out[0].clone(), VS, PCR, 10, max_voxels)
    assert all(bits_equal(g.cpu().numpy(), w.cpu().numpy()) for g, w in zip(got, want))


def test_graph_replay_of_assemble_voxelize_encoder(cuda):
    """one graph: assemble (parameters read from the store's block) + voxelize with the device count + the eval
    SparseEncoder with num_voxels; frames with other slots, counts and poses replayed against eager calls"""
    from bevfusion_b200.sparse_encoder import voxelnet_0p075_encoder
    from bevfusion_b200.voxelize import voxelize_mean_fused
    torch.manual_seed(0)
    enc = voxelnet_0p075_encoder().to(cuda).eval()
    sc = Scene(cuda, seed=31, max_batch=1)
    cap = 400000

    def frame():
        out, counts, _ = sc.store.launch(1, 5, cap)
        f, c, _, nv = voxelize_mean_fused(out[0], VS, PCR, 10, 160000, 0, sync=False, num_points=counts[0:1])
        with torch.no_grad():
            return enc(f, c, 1, num_voxels=nv)

    frames = [(0, list(range(1, 10))), (5, [4, 3, 2, 1]), (10, [9, 8, 7, 6, 5, 4, 3, 2, 1, 0]), (3, [])]
    sc.store.write_frame([sc.sample(*frames[0])], [0, 1, 2, 3, 4], point_cloud_range=PCR)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        frame()
        frame()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:                                                    # the sync-free path: no device-to-host wait
        out, counts, status = sc.store.assemble([sc.sample(*frames[1])], [0, 1, 2, 3, 4], point_cloud_range=PCR,
                                                cap=cap, sync=False)
        f, c, _, nv = voxelize_mean_fused(out[0], VS, PCR, 10, 160000, 0, sync=False, num_points=counts[0:1])
        with torch.no_grad():
            enc(f, c, 1, num_voxels=nv)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_out = frame()
    rng = np.random.default_rng(5)
    for k, (key, chosen) in enumerate(frames):
        if k == 2:                                          # a new sweep and a new pose between replays
            sc.raw[7] = O.nuscenes_sweep(rng, 20000)
            sc.store.put(7, torch.from_numpy(sc.raw[7]).pin_memory())
            sc.poses[8] = O.nuscenes_pose(rng, 3)
        sc.store.write_frame([sc.sample(key, chosen)], [0, 1, 2, 3, 4], point_cloud_range=PCR)
        graph.replay()
        got = static_out.clone()
        want = frame()
        assert bits_equal(got.cpu().numpy(), want.cpu().numpy()), k
        cloud = sc.store.assemble([sc.sample(key, chosen)], [0, 1, 2, 3, 4], point_cloud_range=PCR)[0]
        assert bits_equal(cloud.cpu().numpy(), sc.oracle(key, chosen, [0, 1, 2, 3, 4], point_cloud_range=PCR)), k


def test_store_reused_across_frames(cuda):
    """slots overwritten between frames: every frame gets its own result (sync=False, nothing read in between)"""
    from bevfusion_b200.lidar_sweeps import SweepStore
    rng = np.random.default_rng(41)
    store = SweepStore(4, 36000, 5, cuda, max_batch=2)
    results, wants = [], []
    raw = [None] * 4
    for frame in range(6):
        for s in ([0, 1, 2, 3] if frame == 0 else [frame % 4]):     # one new sweep per frame
            raw[s] = O.nuscenes_sweep(rng, int(rng.integers(1000, 36001)))
            store.put(s, torch.from_numpy(raw[s]).pin_memory())
        poses = [O.nuscenes_pose(rng, k) for k in range(4)]
        key = frame % 4
        chosen = [(key + d) % 4 for d in (1, 2, 3)]
        samples = [(key, [(s, *poses[s], 0.05 * s) for s in chosen]), (chosen[0], [(key, *poses[key], 0.3)])]
        results.append(store.assemble(samples, [0, 1, 2, 3, 4], point_cloud_range=PCR, cap=150000, sync=False))
        wants.append([O.multi_sweeps(raw[key], [raw[s] for s in chosen], [poses[s][0] for s in chosen],
                                     [poses[s][1] for s in chosen], [0.05 * s for s in chosen], [0, 1, 2, 3, 4],
                                     point_cloud_range=PCR),
                      O.multi_sweeps(raw[chosen[0]], [raw[key]], [poses[key][0]], [poses[key][1]], [0.3],
                                     [0, 1, 2, 3, 4], point_cloud_range=PCR)])
    for (out, counts, status), want in zip(results, wants):
        assert int(status.item()) == 0
        for k in range(2):
            n = int(counts[k])
            assert bits_equal(out[k, :n].cpu().numpy(), want[k])


def test_assemble_sweeps_one_shot(cuda):
    from bevfusion_b200.lidar_sweeps import assemble_sweeps
    rng = np.random.default_rng(51)
    key = O.nuscenes_sweep(rng, 5000)
    sweeps = [O.nuscenes_sweep(rng, 4000 + 100 * k) for k in range(3)]
    poses = [O.nuscenes_pose(rng, k + 1) for k in range(3)]
    lags = [0.05, 0.1, 0.15]
    got = assemble_sweeps(key, sweeps, [p[0] for p in poses], [p[1] for p in poses], lags, [0, 1, 2, 3, 4],
                          point_cloud_range=PCR, device=cuda)
    want = O.multi_sweeps(key, sweeps, [p[0] for p in poses], [p[1] for p in poses], lags, [0, 1, 2, 3, 4],
                          point_cloud_range=PCR)
    assert bits_equal(got.cpu().numpy(), want)
    got = assemble_sweeps(torch.from_numpy(key).to(cuda), [], [], [], [], [0, 1, 2, 3, 4], device=cuda)
    assert bits_equal(got.cpu().numpy(), O.multi_sweeps(key, [], [], [], [], [0, 1, 2, 3, 4]))
