"""GPU: RadarSweepStore.assemble (LoadRadarPointsMultiSweeps + PointsRangeFilter's radar face on the device) bit-equal
to the reference's stored outputs and to the numpy restatement on seeded nuScenes-like frames at B = 1..4 and use_dim
sets of 3 to 64 columns (repeats included); kept counts around the tile and ballot sizes; cap overflow writing
exactly cap rows; bad slots and bad op codes; a store reused across frames; RadarEncoder.forward_points with device
counts against per-sample calls on the synced lists; and one CUDA graph of assemble + fused voxelize + radar net +
canvas replayed over new frames against eager calls."""
import numpy as np
import pytest
import torch

import radar_sweeps_oracle as O

pytestmark = pytest.mark.gpu

RVS = [0.8, 0.8, 8.0]
RPCR = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


class Scene:
    """raw radar sweeps in slots 0..n-1 with poses and time lags, and the store holding them"""

    def __init__(self, cuda, seed, n_slots=40, rows=None, slot_cap=300, max_batch=4, max_entries=30):
        from bevfusion_b200.radar_sweeps import RadarSweepStore
        rng = np.random.default_rng(seed)
        rows = rows or [int(rng.integers(30, 125)) for _ in range(n_slots)]
        self.rng = rng
        self.raw = [O.radar_sweep(rng, n) for n in rows]
        self.poses = [O.radar_pose(rng, k % 5) for k in range(len(rows))]
        self.lags = [0.075 * (k % 6) + 1e-3 * rng.uniform() for k in range(len(rows))]
        self.store = RadarSweepStore(len(rows), slot_cap, cuda, max_batch=max_batch, max_entries=max_entries)
        for k, r in enumerate(self.raw):
            self.store.put(k, torch.from_numpy(r).pin_memory() if k % 2 else torch.from_numpy(r).to(cuda))

    def put(self, slot, raw):
        self.raw[slot] = raw
        self.store.put(slot, torch.from_numpy(raw).to(self.store.device))

    def sample(self, slots):
        return [(s, self.poses[s][0], self.poses[s][1], self.lags[s]) for s in slots]

    def oracle(self, slots, use_dim, **kw):
        return O.multi_sweeps([self.raw[s] for s in slots], [self.poses[s][0] for s in slots],
                              [self.poses[s][1] for s in slots], [self.lags[s] for s in slots], use_dim, **kw)


@pytest.mark.parametrize("case", O.GOLDEN_CASES)
def test_bit_equal_to_the_reference_outputs(cuda, case):
    from bevfusion_b200.radar_sweeps import RadarSweepStore
    z = np.load(O.GOLDEN)
    g = O.golden_case(z, case)
    raws = g["raws"]
    store = RadarSweepStore(len(raws), max(len(r) for r in raws), cuda, max_batch=1, max_entries=len(raws))
    for k, r in enumerate(raws):
        store.put(k, r)
    sample = [(k, g["rotations"][k], g["translations"][k], g["time_diffs"][k]) for k in range(len(raws))]
    for bev_range, key in ((O.BEV_RANGE, "_after"), (None, "_before")):
        got = store.assemble([sample], g["use_dim"], g["compensate_velocity"], g["normalize"], bev_range=bev_range)
        assert bits_equal(got[0].cpu().numpy(), z[case + key]), (case, key)


@pytest.mark.parametrize("B", [1, 2, 3, 4])
@pytest.mark.parametrize("compensate", [True, False])
def test_bit_equal_to_the_oracle_shipped_config(cuda, B, compensate):
    sc = Scene(cuda, seed=B * 7 + compensate)
    samples = [list(range(6 * b, 6 * b + 30)) if b < 2 else list(range(b, 40, 3))[:30] for b in range(B)]
    got = sc.store.assemble([sc.sample(s) for s in samples], O.SHIPPED_USE_DIM, compensate, max_num=2500)
    for s, g in zip(samples, got):
        assert bits_equal(g.cpu().numpy(), sc.oracle(s, O.SHIPPED_USE_DIM, compensate_velocity=compensate))


USE_DIMS = [[0, 1, 2], [1, 0, 18], [0, 1, 2, 3, 4], [0, 1, 2, 57, 57, 6, 7, 8, 9, 18, 50, 56],
            list(range(58)), list(range(58)) + [0, 1, 2, 18, 25, 57], [5] + [0] * 63, list(range(57, -1, -1))[:33]]


@pytest.mark.parametrize("use_dim", USE_DIMS, ids=lambda u: "F%d_%d" % (len(u), u[0]))
def test_use_dim_sets(cuda, use_dim):
    sc = Scene(cuda, seed=len(use_dim))
    samples = [list(range(0, 30)), list(range(10, 40))]
    norm = [(0, -60, 60), (1, 0.5, 2.5), (len(use_dim) - 1, -3, 7)]
    for normalize in (False, True):
        for bev_range in (O.BEV_RANGE, None):
            got = sc.store.assemble([sc.sample(s) for s in samples], use_dim, True, normalize, norm,
                                    bev_range=bev_range)
            for s, g in zip(samples, got):
                want = sc.oracle(s, use_dim, normalize=normalize, normalize_dims=norm, bev_range=bev_range)
                assert bits_equal(g.cpu().numpy(), want), (normalize, bev_range)


@pytest.mark.parametrize("rows", [[1], [31, 32, 33], [127], [128], [129], [255, 256, 257], [300, 128, 1, 127]])
def test_kept_counts_around_tile_and_ballot_sizes(cuda, rows):
    # every row inside the range: the kept count is the row count, on each side of the 32-row ballot and 128-row tile
    sc = Scene(cuda, seed=sum(rows), rows=rows)
    for k in range(len(rows)):
        r = sc.raw[k].copy()
        r[:, 0], r[:, 1] = np.float32(5.0), np.float32(-3.0)
        sc.put(k, r)
    got = sc.store.assemble([sc.sample(range(len(rows)))], O.SHIPPED_USE_DIM, True)[0]
    want = sc.oracle(range(len(rows)), O.SHIPPED_USE_DIM)
    assert want.shape[0] == sum(rows) and bits_equal(got.cpu().numpy(), want)


@pytest.mark.parametrize("short", [1, 31, 128, 129])
def test_cap_overflow_writes_exactly_cap_rows(cuda, short):
    from bevfusion_b200.radar_sweeps import OVERFLOW
    sc = Scene(cuda, seed=short, rows=[300] * 4)
    samples = [[0, 1, 2], [3, 2]]
    want = [sc.oracle(s, O.SHIPPED_USE_DIM) for s in samples]
    cap = want[0].shape[0] - short
    assert want[1].shape[0] <= cap
    out, counts, status = sc.store.assemble([sc.sample(s) for s in samples], O.SHIPPED_USE_DIM, True, cap=cap,
                                            sync=False)
    assert int(status.item()) == OVERFLOW and counts.tolist() == [cap, want[1].shape[0]]
    assert bits_equal(out[0].cpu().numpy(), want[0][:cap])          # the first cap rows, nothing past them
    assert bits_equal(out[1, :want[1].shape[0]].cpu().numpy(), want[1])
    with pytest.raises(ValueError, match="cap"):
        sc.store.assemble([sc.sample(s) for s in samples], O.SHIPPED_USE_DIM, True, cap=cap)


def test_bad_slots_and_bad_ops(cuda):
    from bevfusion_b200 import radar_sweeps as RS
    sc = Scene(cuda, seed=3)
    samples = [[0, 1, 2, 3], [4, 5]]
    batch, F, bound = sc.store.write_frame([sc.sample(s) for s in samples], O.SHIPPED_USE_DIM, True)
    e = RS.ENTRY_DTYPE.itemsize
    slot_at = RS._ENTRIES_AT + 1 * e + 4                           # sample 0, entry 1
    for bad_slot in (-1, sc.store.slots, 1 << 30):
        sc.store.block[slot_at:slot_at + 4].copy_(torch.tensor([bad_slot], dtype=torch.int32).view(torch.uint8))
        out, counts, status = sc.store.launch(batch, F, bound)
        assert int(status.item()) == RS.BAD_ENTRY
        want = [sc.oracle([0, 2, 3], O.SHIPPED_USE_DIM), sc.oracle([4, 5], O.SHIPPED_USE_DIM)]
        for k in range(2):                                         # the bad entry contributes no rows
            assert bits_equal(out[k, :int(counts[k])].cpu().numpy(), want[k])
    kind_at = RS._ENTRIES_AT + 1 * e
    sc.store.write_frame([sc.sample(s) for s in samples], O.SHIPPED_USE_DIM, True)
    sc.store.block[kind_at:kind_at + 4].copy_(torch.tensor([1], dtype=torch.int32).view(torch.uint8))   # a KEY
    _, _, status = sc.store.launch(batch, F, bound)
    assert int(status.item()) == RS.BAD_ENTRY
    for c, op in ((0, 0xff), (5, RS.OP_XYZ | 3 << 8), (44, RS.OP_ONE_HOT | 5 << 8 | 1 << 16), (7, 1 << 25)):
        sc.store.write_frame([sc.sample(s) for s in samples], O.SHIPPED_USE_DIM, True)
        at = RS.PARAMS_DTYPE.fields["ops"][1] + 4 * c
        sc.store.block[at:at + 4].copy_(torch.tensor([op], dtype=torch.int32).view(torch.uint8))
        _, counts, status = sc.store.launch(batch, F, bound)
        assert int(status.item()) == RS.BAD_PARAMS and counts.tolist() == [0, 0], c
    # an op past out_dim is never read
    sc.store.write_frame([sc.sample(s) for s in samples], [0, 1, 2, 5], True)
    at = RS.PARAMS_DTYPE.fields["ops"][1] + 4 * 4
    sc.store.block[at:at + 4].copy_(torch.tensor([0xff], dtype=torch.int32).view(torch.uint8))
    out, counts, status = sc.store.launch(batch, 4, bound)
    assert int(status.item()) == 0
    assert bits_equal(out[1, :int(counts[1])].cpu().numpy(), sc.oracle([4, 5], [0, 1, 2, 5]))


def test_store_reused_across_frames(cuda):
    """slots overwritten between frames, one new sweep per radar per frame: every frame gets its own result"""
    sc = Scene(cuda, seed=11, n_slots=30)
    results, wants = [], []
    for frame in range(4):
        for radar in range(5):                                     # the oldest sweep of each radar is replaced
            slot = radar * 6 + (frame % 6)
            sc.put(slot, O.radar_sweep(sc.rng, int(sc.rng.integers(20, 125))))
        slots = [r * 6 + (frame - k) % 6 for r in range(5) for k in range(6)]
        results.append(sc.store.assemble([sc.sample(slots)], O.SHIPPED_USE_DIM, True, sync=False))
        wants.append(sc.oracle(slots, O.SHIPPED_USE_DIM))
    for (out, counts, status), want in zip(results, wants):
        assert int(status.item()) == 0
        assert bits_equal(out[0, :int(counts[0])].cpu().numpy(), want)


def radar_encoder(cuda):
    from bevfusion_b200.radar_encoder import RadarEncoder
    torch.manual_seed(0)
    cfg = dict(type="RadarFeatureNet", in_channels=45, feat_channels=[128, 128, 128, 64], voxel_size=RVS,
               point_cloud_range=RPCR, norm_cfg=dict(type="BN1d", eps=1e-3, momentum=0.01))
    enc = RadarEncoder(cfg, dict(type="PointPillarsScatter", in_channels=64, output_shape=[128, 128])).to(cuda).eval()
    for layer in enc.pts_voxel_encoder.rfn_layers:
        layer.norm.running_mean.uniform_(-0.3, 0.3)
        layer.norm.bias.data.uniform_(-0.5, 0.5)
        layer.norm.weight.data.uniform_(-1.5, 1.5)
    return enc


@pytest.mark.parametrize("B", [1, 4])
def test_forward_points_with_device_counts(cuda, B):
    from bevfusion_b200.voxelize import Voxelization
    enc = radar_encoder(cuda)
    vox = Voxelization(RVS, RPCR, 10, (30000, 60000)).eval()
    sc = Scene(cuda, seed=50 + B)
    samples = [list(range(b, 40, 2))[:30] for b in range(B)]
    if B == 4:                                      # an empty sample: the device count is 0
        sc.put(39, O.radar_sweep(sc.rng, 0))
        samples[3] = [39]
    with torch.no_grad():
        enc.forward_points([torch.zeros(10, 45, device=cuda)], vox)   # packs the weights
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:                                                   # the sync-free path: no device-to-host wait
        out, counts, _ = sc.store.assemble([sc.sample(s) for s in samples], O.SHIPPED_USE_DIM, True, cap=3000,
                                           sync=False)
        with torch.no_grad():
            got, gn = enc.forward_points(out, vox, return_voxel_num=True, num_points=counts)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    lists = [out[k, :n] for k, n in enumerate(counts.tolist())]
    with torch.no_grad():
        want, wn = enc.forward_points(lists, vox, return_voxel_num=True)
    assert torch.equal(gn, wn) and (B < 4 or int(gn[3]) == 0)
    assert bits_equal(got.cpu().numpy(), want.cpu().numpy())


def test_graph_replay_of_assemble_voxelize_radar_net(cuda):
    """one graph: assemble (parameters read from the store's block) + fused voxelize with the device counts + the
    radar net + the canvas; frames with other slots, counts and poses replayed against eager calls"""
    from bevfusion_b200.voxelize import Voxelization
    enc = radar_encoder(cuda)
    vox = Voxelization(RVS, RPCR, 10, (30000, 60000)).eval()
    sc = Scene(cuda, seed=77)
    cap = 4000

    def frame():
        out, counts, _ = sc.store.launch(2, 45, cap)
        with torch.no_grad():
            return enc.forward_points(out, vox, num_points=counts)

    frames = [[list(range(30)), list(range(10, 40))], [list(range(0, 40, 2)), [3, 1]], [[5], list(range(39, 9, -1))]]
    sc.store.write_frame([sc.sample(s) for s in frames[0]], O.SHIPPED_USE_DIM, True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        frame()
        frame()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_out = frame()
    for k, samples in enumerate(frames):
        if k == 2:                                         # a new sweep and a new pose between replays
            sc.put(7, O.radar_sweep(sc.rng, 110))
            sc.poses[8] = O.radar_pose(sc.rng, 3)
        sc.store.write_frame([sc.sample(s) for s in samples], O.SHIPPED_USE_DIM, True)
        graph.replay()
        got = static_out.clone()
        want = frame()
        assert bits_equal(got.cpu().numpy(), want.cpu().numpy()), k
        clouds = sc.store.assemble([sc.sample(s) for s in samples], O.SHIPPED_USE_DIM, True)
        for s, c in zip(samples, clouds):
            assert bits_equal(c.cpu().numpy(), sc.oracle(s, O.SHIPPED_USE_DIM)), k
        with torch.no_grad():
            assert bits_equal(enc.forward_points(clouds, vox).cpu().numpy(), got.cpu().numpy()), k
