"""GPU tests of the native SparseEncoder training step (bevb200_encoder_forward_train / _backward) on every chain
the plan accepts and across its chunk, row-count and stride boundaries, against a float64 CPU twin
(encoder_train_oracle.raw_train_forward / twin_forward, the backward from float64 autograd) that applies the
native run's ReLU masks.

  * Raw C-ABI chains: the strided chains of the eval-mode tests (residual from the previous conv, from two back,
    on the last conv, a strided first conv), a residual block on every level, c_out 16 on level 1, a 128-channel
    SubM, first-conv widths 7 / 20 / 40, convs without ReLU; an all-SubM chain trains forward only and its backward
    is refused without a write.
  * Module chains (voxelnet, the default SparseEncoder, a basicblock chain on 4 channels) at B = 3 on odd grids
    with voxels on every border face, in the very last site and an empty middle sample.
  * Level counts at k * kStatRows + {-1, 0, 1} (the BN sum chunks) on every level, 2 rows and 1 row on the last
    level (the unbiased variance, and BEVB200_ENCODER_FEW_ROWS with its exactly-zero gradients), kWgtRows * m +-1
    and a count below one filter-gradient tile under a cap of hundreds of tiles.
  * The ABI contracts: out_batch_stride in both calls (canaries between samples), level caps at and one below a
    level's count, every output overwritten (NaN-filled, then re-run over garbage: bit-equal), state and workspace
    at exactly their queried sizes inside canary-filled buffers.

Bounds are those of test_encoder_train_gpu.BOUNDS; status counts, num_batches_tracked, inactive cells and gradient
rows past the count are checked exactly."""
import ctypes

import numpy as np
import pytest
import torch

from bevfusion_b200 import _C
from bevfusion_b200.encoder_plan import _BNDesc
from encoder_train_cases import (ONE_ROW_CHAIN, STAT_ROWS, TILE_CHAIN, TRAIN_RAW, WGT_ROWS, block_coors,
                                 lattice_coors, level_shapes, stat_case, stat_counts, tile_counts)
from encoder_train_oracle import raw_train_forward, rel
from test_encoder_plan_gpu import RAW_CHAINS, create, default_encoder, odd_coors, random_coors, voxelnet
from test_encoder_train_gpu import BOUNDS, _native_masks, _stats, _step

pytestmark = pytest.mark.gpu

GUARD = 4096                   # canary bytes on each side of the state and the workspace
CANARY = 0xA5
EPS, MOMENTUM = 1e-3, 0.1
BEVB200_EINVAL = -1
TRUNCATED, FEW_ROWS = 1, 2


def _guarded(nbytes, dev):
    """(buffer, tensor of exactly nbytes GUARD bytes into it), the whole buffer canary-filled"""
    buf = torch.full((nbytes + 2 * GUARD,), CANARY, dtype=torch.uint8, device=dev)
    return buf, buf[GUARD:GUARD + nbytes]


def _guard_intact(buf, nbytes):
    b = buf.cpu()
    return bool((b[:GUARD] == CANARY).all()) and bool((b[GUARD + nbytes:] == CANARY).all())


def _arr(ts):
    return (ctypes.c_void_p * len(ts))(*[_C.ptr(t) for t in ts])


class RawTrain:
    """One raw conv chain through the C ABI: create, forward_train, backward, on exactly-sized state / workspace.
    Rows past n_valid (up to n_rows) are NaN features at coordinates outside the grid."""

    def __init__(self, dev, in_channels, shape, B, convs, coors, n_rows=None, caps=None, stride=0, seed=0):
        self.dev, self.cin, self.shape, self.B, self.convs = dev, in_channels, list(shape), B, convs
        self.coors = np.ascontiguousarray(coors, dtype=np.int32)
        self.n_valid = self.coors.shape[0]
        self.n_rows = n_rows or self.n_valid
        self.caps = None if caps is None else (ctypes.c_int32 * len(caps))(*caps)
        self.stride = stride
        L = self.L = _C.lib()
        g = torch.Generator().manual_seed(seed)
        feats = torch.randn(self.n_valid, in_channels, generator=g)
        self.feats = torch.cat([feats, torch.full((self.n_rows - self.n_valid, in_channels), float("nan"))]).to(dev)
        pad = np.full((self.n_rows - self.n_valid, 4), 100000, np.int32)
        self.coors_dev = torch.from_numpy(np.concatenate([self.coors, pad])).to(dev)
        self.n_dev = torch.tensor([self.n_valid], dtype=torch.int32, device=dev)
        self.w, self.gamma, self.beta, self.rm, self.rv = [], [], [], [], []
        for c in convs:
            kv = int(np.prod(c["ks"]))
            self.w.append((torch.randn(kv, c["cin"], c["cout"], generator=g) / (kv * c["cin"]) ** 0.5).to(dev))
            self.gamma.append((torch.rand(c["cout"], generator=g) * 0.4 + 0.8).to(dev))
            self.beta.append((torch.randn(c["cout"], generator=g) * 0.1).to(dev))
            self.rm.append((torch.randn(c["cout"], generator=g) * 0.1).to(dev))
            self.rv.append((torch.rand(c["cout"], generator=g) + 0.5).to(dev))
        self.nbt = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in convs]
        self.before = [(m.clone(), v.clone()) for m, v in zip(self.rm, self.rv)]
        rc, self.h = create(in_channels, shape, convs)
        assert rc == 0, L.bevb200_last_error()
        self.n_levels = L.bevb200_encoder_num_levels(self.h)
        oshape, oc = (ctypes.c_int32 * 3)(), ctypes.c_int32()
        _C.check(L.bevb200_encoder_output_shape(self.h, oshape, ctypes.byref(oc)), "encoder_output_shape")
        X, Y, Z = list(oshape)
        self.out_shape = (B, oc.value * Z, X, Y)
        self.per = oc.value * Z * X * Y
        assert stride == 0 or stride >= self.per
        caps_out = (ctypes.c_int32 * self.n_levels)()
        _C.check(L.bevb200_encoder_level_caps(self.h, self.n_rows, B, self.caps, caps_out), "encoder_level_caps")
        self.level_caps = list(caps_out)
        self.state_bytes = L.bevb200_encoder_train_state_bytes(self.h, self.n_rows, B, self.caps)
        self.state_buf, self.state = _guarded(self.state_bytes, dev)
        self.ws_bytes = L.bevb200_encoder_backward_workspace_bytes(self.h, self.n_rows, B, self.caps)
        self.ws_buf, self.ws = _guarded(self.ws_bytes, dev)

    def close(self):
        if self.h is not None:
            self.L.bevb200_encoder_destroy(self.h)
            self.h = None

    def _bn(self):
        descs = (_BNDesc * len(self.convs))()
        for i, d in enumerate(descs):
            d.weight, d.bias = _C.ptr(self.gamma[i]), _C.ptr(self.beta[i])
            d.running_mean, d.running_var = _C.ptr(self.rm[i]), _C.ptr(self.rv[i])
            d.num_batches_tracked = _C.ptr(self.nbt[i])
            d.eps, d.momentum = EPS, MOMENTUM
        return descs

    def canvas(self, fill):
        if self.stride:
            return torch.full((self.B, self.stride), fill, device=self.dev)
        return torch.full(self.out_shape, fill, device=self.dev)

    def forward(self):
        """-> status list; self.out is the output (the [B, stride] canvas when stride != 0)"""
        self.out = self.canvas(-7.25 if self.stride else float("nan"))
        self.status = torch.full((1 + self.n_levels,), -1, dtype=torch.int32, device=self.dev)
        rc = self.L.bevb200_encoder_forward_train(
            self.h, _arr(self.w), self._bn(), _C.ptr(self.feats), _C.ptr(self.coors_dev), self.n_rows,
            _C.ptr(self.n_dev), self.B, self.caps, _C.ptr(self.out), self.stride, _C.ptr(self.status),
            _C.ptr(self.state), self.state_bytes, _C.current_stream(self.dev), None)
        _C.check(rc, "encoder_forward_train")
        torch.cuda.synchronize()
        return self.status.cpu().tolist()

    def dense_out(self):
        return self.out[:, :self.per].reshape(self.out_shape) if self.stride else self.out

    def masks(self):
        """the ReLU mask of every conv, decoded from the split images the forward saved"""
        st = self.status.cpu().tolist()
        out, level = [], 0
        for i, c in enumerate(self.convs):
            level += 0 if c["subm"] else 1
            zo, yo = ctypes.c_size_t(), ctypes.c_size_t()
            _C.check(self.L.bevb200_encoder_train_saved(self.h, self.n_rows, self.B, self.caps, i, ctypes.byref(zo),
                                                        ctypes.byref(yo)), "encoder_train_saved")
            n, cc = st[1 + level], c["cout"]
            img = self.state[yo.value:yo.value + n * cc * 4].view(torch.bfloat16).view(n, cc // 16, 2, 16).float()
            out.append(((img[:, :, 0] + img[:, :, 1]).reshape(n, cc) > 0).cpu())
        return out

    def grad_canvas(self, R):
        """R [B, C*Z, X, Y] as the backward's input; with a stride, NaN between the samples"""
        if not self.stride:
            return R.to(self.dev)
        g = self.canvas(float("nan"))
        g[:, :self.per] = R.reshape(self.B, -1).to(self.dev)
        return g

    def backward(self, R, fill=float("nan")):
        """-> (return code, dict of gradients: features [n_rows, c_in], w, gamma, beta lists), outputs prefilled"""
        gf = torch.full((self.n_rows, self.cin), fill, device=self.dev)
        gw = [torch.full_like(w, fill) for w in self.w]
        gg = [torch.full_like(v, fill) for v in self.gamma]
        gb = [torch.full_like(v, fill) for v in self.beta]
        rc = self.L.bevb200_encoder_backward(
            self.h, _arr(self.w), _C.ptr(self.state), self.state_bytes, self.n_rows, self.B, self.caps,
            _C.ptr(self.grad_canvas(R)), self.stride, _C.ptr(gf), _arr(gw), _arr(gg), _arr(gb), _C.ptr(self.ws),
            self.ws_bytes, _C.current_stream(self.dev))
        torch.cuda.synchronize()
        return rc, {"features": gf.cpu(), "w": [t.cpu() for t in gw], "gamma": [t.cpu() for t in gg],
                    "beta": [t.cpu() for t in gb]}

    def guards_intact(self):
        return _guard_intact(self.state_buf, self.state_bytes) and _guard_intact(self.ws_buf, self.ws_bytes)


def float64_step(run, masks, R):
    """the float64 twin of run's step -> (dense output, rows per level, gradients, running stats, counts)"""
    x = run.feats[:run.n_valid].double().cpu().requires_grad_(True)
    ws = [w.double().cpu().requires_grad_(True) for w in run.w]
    gs = [v.double().cpu().requires_grad_(True) for v in run.gamma]
    bs = [v.double().cpu().requires_grad_(True) for v in run.beta]
    bufs = [[m.double().cpu(), v.double().cpu(), 0] for m, v in run.before]
    out, rows = raw_train_forward(run.convs, x, run.coors, run.B, run.shape, ws, list(zip(gs, bs)), bufs, masks,
                                  EPS, MOMENTUM, run.stride)
    if run.stride:
        out = out[:, :run.per].reshape(run.out_shape)
    (out * R.double()).sum().backward()
    grads = {"features": x.grad, "w": [w.grad for w in ws], "gamma": [v.grad for v in gs],
             "beta": [v.grad for v in bs]}
    return out.detach(), rows, grads, bufs


def check_step(run, what, seed=1, flags=0):
    """forward + backward of run against float64: bounds on every gradient and statistics move, exact status,
    counts and zeros, untouched canaries.  -> (status, native gradients, float64 gradients)"""
    st = run.forward()
    masks = run.masks()
    R = torch.randn(run.out_shape, generator=torch.Generator().manual_seed(seed))
    rc, got = run.backward(R)
    assert rc == 0, run.L.bevb200_last_error()
    want_out, rows, want, bufs = float64_step(run, masks, R)
    assert st == [flags] + rows, "%s: status %s, float64 rows %s" % (what, st, rows)
    out = run.dense_out().cpu()
    assert rel(out, want_out)[1] <= 1e-4, what
    assert not bool(out[want_out == 0].any()), "%s: an inactive cell is not 0" % what
    if run.stride:
        tail = run.out[:, run.per:].cpu()
        assert bool((tail == -7.25).all()), "%s: the canvas between samples changed" % what
    n = run.n_valid
    assert bool((got["features"][n:] == 0).all()), "%s: gradient rows past the count are not 0" % what
    table = [("input", "features", rel(got["features"][:n], want["features"])[0])]
    for i in range(len(run.convs)):
        table.append(("conv", "w%d" % i, rel(got["w"][i], want["w"][i])[0]))
        table.append(("bn", "gamma%d" % i, rel(got["gamma"][i], want["gamma"][i])[0]))
        table.append(("bn", "beta%d" % i, rel(got["beta"][i], want["beta"][i])[0]))
        m0, v0 = run.before[i]
        table.append(("stats", "mean%d" % i, rel((run.rm[i] - m0).cpu(), bufs[i][0] - m0.double().cpu())[0]))
        table.append(("stats", "var%d" % i, rel((run.rv[i] - v0).cpu(), bufs[i][1] - v0.double().cpu())[0]))
        assert int(run.nbt[i]) == bufs[i][2], "%s: num_batches_tracked of conv %d" % (what, i)
    print("%-30s rows %s  worst rel L2: %s" % (what, rows, "  ".join(
        "%s %.2e" % (k, max(l2 for kk, _, l2 in table if kk == k)) for k in BOUNDS)))
    bad = [(k, name, l2) for k, name, l2 in table if not l2 <= BOUNDS[k]]
    assert not bad, (what, bad)
    assert run.guards_intact(), "%s: a byte outside the state or the workspace changed" % what
    return st, got, want


def _run(cuda, cin, convs, shape, B, coors, what, **kw):
    run = RawTrain(cuda, cin, shape, B, convs, coors, **kw)
    try:
        return run, check_step(run, what)
    finally:
        run.close()


# ---------------------------------------------------------------------------------------------------- raw chains
@pytest.mark.parametrize("chain", list(TRAIN_RAW))
def test_raw_chain_train(cuda, chain):
    cin, convs = TRAIN_RAW[chain]
    shape, B = [40, 36, 15], 2
    _run(cuda, cin, convs, shape, B, random_coors(shape, B, 3000, seed=len(chain)), chain, seed=len(chain))


def test_all_subm_forward_only(cuda):
    """one level: the forward trains against float64, the backward is refused and writes nothing"""
    cin, convs = RAW_CHAINS["all-subm"]
    shape, B = [40, 36, 15], 2
    run = RawTrain(cuda, cin, shape, B, convs, random_coors(shape, B, 3000, seed=8))
    try:
        st = run.forward()
        R = torch.randn(run.out_shape, generator=torch.Generator().manual_seed(2))
        want_out, rows, _, bufs = float64_step(run, run.masks(), R)
        assert st == [0] + rows
        assert rel(run.dense_out().cpu(), want_out)[1] <= 1e-4
        for i in range(len(convs)):
            m0, v0 = run.before[i]
            assert rel((run.rm[i] - m0).cpu(), bufs[i][0] - m0.double().cpu())[0] <= BOUNDS["stats"]
            assert rel((run.rv[i] - v0).cpu(), bufs[i][1] - v0.double().cpu())[0] <= BOUNDS["stats"]
        state = run.state_buf.clone()
        rc, got = run.backward(R, fill=3.5)
        assert rc == BEVB200_EINVAL
        assert torch.equal(run.state_buf, state)
        assert bool((run.ws_buf == CANARY).all())
        for t in [got["features"]] + got["w"] + got["gamma"] + got["beta"]:
            assert bool((t == 3.5).all())
    finally:
        run.close()


# ---------------------------------------------------------------------------------------------------- module chains
def _basic4(shape, seed=0):
    """a three-stage basicblock chain on 4 input channels"""
    from bevfusion_b200.sparse_encoder import SparseEncoder
    torch.manual_seed(seed)
    return SparseEncoder(in_channels=4, sparse_shape=shape, output_channels=128,
                         encoder_channels=((16, 16, 32), (32, 32, 64), (64, 64)),
                         encoder_paddings=((0, 0, 1), (0, 0, 1), (0, 0)), block_type="basicblock")


MODULES = {"voxelnet": (voxelnet, [57, 43, 41]), "default": (default_encoder, [57, 43, 23]),
           "basic-4": (_basic4, [57, 43, 23])}


@pytest.mark.parametrize("chain", list(MODULES))
def test_module_chain_train_odd_grid(cuda, chain):
    import copy

    from bevfusion_b200 import encoder_plan
    from encoder_train_oracle import twin_forward
    make, shape = MODULES[chain]
    m = make(shape, seed=3).to(cuda).train()
    for mod in m.modules():                                      # BN parameters away from (1, 0)
        if isinstance(mod, torch.nn.BatchNorm1d):
            mod.weight.data.uniform_(0.8, 1.2); mod.bias.data.normal_(0, 0.1)
    B = 3
    coors = torch.from_numpy(odd_coors(shape, B, 5000, seed=4, empty=1)).to(cuda)
    feats = torch.randn(coors.shape[0], m.in_channels, device=cuda, generator=torch.Generator(device=cuda).manual_seed(5))
    n_dev = torch.tensor([coors.shape[0]], dtype=torch.int32, device=cuda)
    masks = _native_masks(m, feats, coors, B, n_dev)
    twin = copy.deepcopy(m).double()
    before = _stats(m)
    X, Y, Z = m.plan().out_shape
    R = torch.randn((B, m.plan().out_channels * Z, X, Y), device=cuda, generator=torch.Generator(device=cuda).manual_seed(6))
    out, gx = _step(m, feats, coors, B, n_dev, R)
    chain64 = encoder_plan._chain_of(twin)
    x64 = feats.detach().double().requires_grad_(True)
    out64 = twin_forward(chain64, x64, coors, B, shape, masks, [(bn.weight, bn.bias) for _, bn, _, _ in chain64],
                         [(bn.running_mean, bn.running_var, bn.num_batches_tracked) for _, bn, _, _ in chain64])
    (out64 * R.double()).sum().backward()
    out64 = out64.detach()
    assert rel(out, out64)[1] <= 1e-4
    assert not bool(out[out64 == 0].any()) and not bool(out[1].any())
    table = [("input", "features", rel(gx, x64.grad)[0])]
    p64 = dict(twin.named_parameters())
    table += [("bn" if p.dim() == 1 else "conv", k, rel(p.grad, p64[k].grad)[0]) for k, p in m.named_parameters()]
    b64 = dict(twin.named_buffers())
    for k, b in m.named_buffers():
        if k.endswith(("running_mean", "running_var")):
            table.append(("stats", k, rel(b - before[k], b64[k] - before[k].double())[0]))
        elif k.endswith("num_batches_tracked"):
            assert int(b) == int(b64[k]) == int(before[k]) + 1, k
    print("%-30s worst rel L2: %s" % (chain + " odd B=3", "  ".join(
        "%s %.2e" % (k, max(l2 for kk, _, l2 in table if kk == k)) for k in BOUNDS)))
    bad = [(k, name, l2) for k, name, l2 in table if not l2 <= BOUNDS[k]]
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------- row counts
@pytest.mark.parametrize("c", [16, 128])
@pytest.mark.parametrize("n", stat_counts())
def test_stat_chunk_counts(cuda, c, n):
    """every level holds n rows, n on a kStatRows chunk edge"""
    cin, convs, shape, B, coors, rows = stat_case(c, n)
    assert rows == [n] * 3
    _run(cuda, cin, convs, shape, B, coors, "stats c%d n=%d (chunk %d)" % (c, n, STAT_ROWS))


def test_two_rows_on_the_last_level(cuda):
    """n = 2 on every level: the unbiased running variance at its largest factor n / (n - 1)"""
    cin, convs = TILE_CHAIN
    shape, B = [20, 18, 9], 1
    coors, rows = lattice_coors(shape, B, 2, 1, seed=3)
    (run, (st, _, _)) = _run(cuda, cin, convs, shape, B, coors, "two rows")
    assert st[1:] == [2, 2]


def test_one_row_on_the_last_level(cuda):
    """8 voxels of one 2x2x2 block, a k2 s2 p0 conv: level 0 holds 8 rows, level 1 one.  The flag is set, only
    level 1's running statistics stay, and every gradient that reaches level 0 through level 1's BN is exactly 0."""
    cin, convs = ONE_ROW_CHAIN
    shape, B = [12, 10, 8], 1
    coors, rows = block_coors(shape)
    assert rows == [8, 1]
    run = RawTrain(cuda, cin, shape, B, convs, coors, seed=4)
    try:
        st, got, want = check_step(run, "one row on level 1", flags=FEW_ROWS)
        for i, lv in enumerate([0, 0, 1, 1, 1]):
            m0, v0 = run.before[i]
            assert (torch.equal(run.rm[i], m0) and torch.equal(run.rv[i], v0)) == (lv == 1), i
            assert int(run.nbt[i]) == 1 - lv, i
            assert bool((got["w"][i] == 0).all()) and bool((got["gamma"][i] == 0).all()), i
            if lv == 0:                                          # reached only through level 1's BN
                assert bool((got["beta"][i] == 0).all()), i
        assert bool((got["features"] == 0).all())
        assert bool((got["beta"][4] != 0).any())                 # the last BN's beta still sees its gradient
        for t in [want["features"]] + want["w"][:2]:
            assert bool((t == 0).all())
    finally:
        run.close()


@pytest.mark.parametrize("n", tile_counts())
def test_wgrad_tile_counts(cuda, n):
    """level 1 holds n rows, n on a kWgtRows tile edge"""
    cin, convs = TILE_CHAIN
    shape, B = [40, 36, 15], 2
    coors, rows = lattice_coors(shape, B, n, 1, seed=n)
    _run(cuda, cin, convs, shape, B, coors, "wgrad tiles n=%d (tile %d)" % (n, WGT_ROWS))


def test_wgrad_count_below_one_tile_under_a_large_cap(cuda):
    """5 valid rows of 4096: level 1's cap spans hundreds of tiles, its count fills part of one, so all but one
    filter-gradient chunk is empty"""
    cin, convs = TILE_CHAIN
    shape, B = [80, 72, 31], 2
    coors, _ = lattice_coors(shape, B, 5, 1, seed=5)
    run, _ = _run(cuda, cin, convs, shape, B, coors, "5 rows under cap", n_rows=4096)
    assert run.level_caps[1] // WGT_ROWS >= 200, run.level_caps


# ---------------------------------------------------------------------------------------------------- ABI contracts
def test_out_batch_stride(cuda):
    """the encoder writes into, and reads its gradient from, a canvas wider than its output"""
    cin, convs = TRAIN_RAW["residual-every-level"]
    shape, B = [41, 37, 15], 3
    X, Y, Z = level_shapes(shape, convs)[-1]
    per = convs[-1]["cout"] * X * Y * Z
    _run(cuda, cin, convs, shape, B, odd_coors(shape, B, 2500, seed=9, empty=1), "out_batch_stride",
         stride=per + 1000 + 3)


@pytest.mark.parametrize("delta", [0, -1])
def test_level_cap_at_count(cuda, delta):
    """level 1 capped at exactly its count (no truncation: float64 bounds) and one below (flagged, finite)"""
    cin, convs = TILE_CHAIN
    shape, B = [40, 36, 15], 2
    n = 300
    coors, _ = lattice_coors(shape, B, n, 1, seed=6)
    caps = [0, n + delta]
    if delta == 0:
        run, _ = _run(cuda, cin, convs, shape, B, coors, "cap = count", caps=caps)
        assert run.level_caps[1] == n
        return
    run = RawTrain(cuda, cin, shape, B, convs, coors, caps=caps)
    try:
        st = run.forward()
        assert st[0] & TRUNCATED and st[1:] == [n, n - 1]
        rc, got = run.backward(torch.randn(run.out_shape, generator=torch.Generator().manual_seed(7)))
        assert rc == 0
        assert bool(torch.isfinite(run.out).all())
        for t in [got["features"]] + got["w"] + got["gamma"] + got["beta"]:
            assert bool(torch.isfinite(t).all())
        assert run.guards_intact()
    finally:
        run.close()


def test_outputs_overwritten_and_state_reusable(cuda):
    """a second backward on the same state, over outputs filled with large garbage, is bit-equal to the first
    (over NaN); the state is unchanged by either"""
    cin, convs = TRAIN_RAW["residual-two-back"]
    shape, B = [40, 36, 15], 2
    run = RawTrain(cuda, cin, shape, B, convs, random_coors(shape, B, 3000, seed=10), n_rows=3100)
    try:
        run.forward()
        state = run.state_buf.clone()
        R = torch.randn(run.out_shape, generator=torch.Generator().manual_seed(8))
        rc1, g1 = run.backward(R)
        rc2, g2 = run.backward(R, fill=1e30)
        assert rc1 == rc2 == 0
        assert torch.equal(run.state_buf, state)
        for a, b in zip([g1["features"]] + g1["w"] + g1["gamma"] + g1["beta"],
                        [g2["features"]] + g2["w"] + g2["gamma"] + g2["beta"]):
            assert bool(torch.isfinite(a).all()) and torch.equal(a, b)
        assert run.guards_intact()
    finally:
        run.close()
