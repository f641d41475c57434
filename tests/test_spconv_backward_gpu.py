"""GPU tests of the sparse-conv backward (bevb200_spconv_backward) against a float64 reference built from the
neighbour table directly, on every kernel the dispatch can pick:

  * input gradient: the SIMT forward on the transposed table, the mma.sync / wgmma forward on the out-grad image the
    filter gradient already split ("shared image"), the BF16x3 forward with its own temporaries, 3xTF32 and TF32;
  * filter gradient: spconv_wgrad2_kernel, the generic spconv_wgrad_kernel <1,1> / <2,2> / <4,4> with channel tails
    and for misaligned pointers, and the tensor-core kernel for every operand-image shape (ci_eff, co_eff).

Every call fills both outputs with NaN first and puts a canary behind the queried workspace; every case runs twice and
must be bit-identical.  The full-size C3 layer rulebooks and a SparseEncoder training step against a float64 twin
(rulebooks from the CPU oracle) close the file."""
import copy

import numpy as np
import pytest
import torch

import oracle
from bevfusion_b200 import _C

pytestmark = pytest.mark.gpu

EWORKSPACE = -3
CANARY = 4096


# ---------------------------------------------------------------------------------------------------- helpers
def _canary_bytes(device):
    return (torch.arange(CANARY, device=device) * 37 + 11).remainder(256).to(torch.uint8)


def backward_cabi(f, w, g, nbr, nbr_t, prec, ws_bytes=None):
    """bevb200_spconv_backward at an explicit precision -> (input_grad, weight_grad).  Outputs start as NaN (so a
    row or offset the call leaves alone, or accumulates into, shows); the workspace is the queried size plus a
    canary tail that must come back untouched."""
    lib = _C.lib()
    n_in, c_in = f.shape
    kv, n_out = nbr.shape
    c_out = w.shape[-1]
    din = torch.full((n_in, c_in), float("nan"), device=f.device)
    dw = torch.full((kv, c_in, c_out), float("nan"), device=f.device)
    need = lib.bevb200_spconv_backward_workspace_bytes(n_in, n_out, c_in, c_out, kv)
    assert need > 0
    ws = torch.empty(need + CANARY, dtype=torch.uint8, device=f.device)
    canary = _canary_bytes(f.device)
    ws[need:] = canary
    _C.check(lib.bevb200_spconv_backward(_C.ptr(f), _C.ptr(w), _C.ptr(g), _C.ptr(nbr), _C.ptr(nbr_t), n_in, n_out,
                                         c_in, c_out, kv, int(prec), _C.ptr(din), _C.ptr(dw), _C.ptr(ws),
                                         need if ws_bytes is None else ws_bytes, _C.current_stream(f.device)),
             "spconv_backward")
    torch.cuda.synchronize()
    assert torch.equal(ws[need:], canary), "the backward wrote past the workspace size it asked for"
    assert not bool(torch.isnan(din).any()), "input_grad has rows the backward did not write"
    assert not bool(torch.isnan(dw).any()), "weight_grad has elements the backward did not write"
    return din, dw


def reference(f, w, g, nbr):
    """float64 gradients from nbr itself (not nbr_t): dW[k] = F[nbr[k, v]]^T G[v] and dIn += G[v] W[k]^T over the
    valid v (0 <= nbr[k, v] < n_in).  Also returns the mask of input rows some valid entry refers to."""
    n_in = f.shape[0]
    f64, w64, g64 = f.double(), w.double(), g.double()
    din = torch.zeros(n_in, f.shape[1], dtype=torch.float64, device=f.device)
    dw = torch.zeros(w.shape, dtype=torch.float64, device=f.device)
    fed = torch.zeros(n_in, dtype=torch.bool, device=f.device)
    for k in range(nbr.shape[0]):
        m = (nbr[k] >= 0) & (nbr[k] < n_in)
        rows = nbr[k][m].long()
        dw[k] = f64[rows].t() @ g64[m]
        din.index_add_(0, rows, g64[m] @ w64[k].t())
        fed[rows] = True
    return din, dw, fed


def check(din, dw, ref_din, ref_dw, fed, prec, what=""):
    """dW per offset <= 1e-4 of that offset's max|ref| (empty offsets exactly 0); dIn <= 1e-4 of max|ref| (3e-3 for
    single-pass TF32), rows nothing feeds exactly 0.  Returns (dIn error, worst dW error), both relative."""
    err_k = (dw.double() - ref_dw).abs().flatten(1).amax(1)
    scale_k = ref_dw.abs().flatten(1).amax(1)
    bad = (err_k > 1e-4 * scale_k).nonzero().flatten().tolist()
    assert not bad, "%s weight grad: offsets %s, rel err %s" % (what, bad, (err_k[bad] / scale_k[bad]).tolist())
    dw_err = float((err_k / scale_k.clamp_min(1e-300)).max()) if dw.numel() else 0.0
    assert bool((din[~fed] == 0).all()), "%s input grad: a row no output is fed by is not 0" % what
    din_err = 0.0
    if din.numel():
        den = float(ref_din.abs().max())
        din_err = float((din.double() - ref_din).abs().max()) / max(den, 1e-300)
        tol = 3e-3 if prec == 2 else 1e-4
        assert din_err <= tol, "%s input grad: rel err %.3e > %.0e" % (what, din_err, tol)
    return din_err, dw_err


def random_table(kv, n_in, n_out, gen, miss=0.4, junk=True):
    """nbr [kv, n_out]: each offset injective (a random permutation slice of the live input rows), a fraction `miss`
    of the entries -1, 1/16 of the input rows referenced by no offset, one offset with no pair at all, and (junk) a
    few entries >= n_in or < -1 that the backward must treat as missing."""
    dev = gen.device
    n_dead = n_in // 16
    live = torch.randperm(n_in, generator=gen, device=dev)[n_dead:]
    assert live.numel() >= n_out
    nbr = torch.stack([live[torch.randperm(live.numel(), generator=gen, device=dev)[:n_out]] for _ in range(kv)])
    nbr = nbr.to(torch.int32)
    nbr[torch.rand(kv, n_out, generator=gen, device=dev) < miss] = -1
    if junk:
        vals = torch.tensor([n_in, n_in + 7, 2 ** 31 - 1, -2, -1000, -2 ** 31], dtype=torch.int32, device=dev)
        pos = torch.rand(kv, n_out, generator=gen, device=dev) < 0.01
        pick = torch.randint(0, vals.numel(), (kv, n_out), generator=gen, device=dev)
        nbr[pos] = vals[pick[pos]]
    if kv > 1:
        nbr[kv // 3] = -1
    return nbr


GEOMS = {"subm_k3": ([3, 3, 3], [1, 1, 1], [1, 1, 1], True),
         "conv_k3s2p1": ([3, 3, 3], [2, 2, 2], [1, 1, 1], False)}


def geometric_table(geom, seed, cuda):
    """nbr of a real conv on random voxels at about 20 % occupancy (6000 of 2 x 40 x 36 x 11 sites)."""
    from bevfusion_b200.spconv import ops
    ks, st, pd, subm = GEOMS[geom]
    shape, B, n = [40, 36, 11], 2, 6000
    rng = np.random.default_rng(seed)
    flat = rng.choice(B * shape[0] * shape[1] * shape[2], size=n, replace=False)
    z = flat % shape[2]; y = (flat // shape[2]) % shape[1]
    x = (flat // (shape[2] * shape[1])) % shape[0]; b = flat // (shape[2] * shape[1] * shape[0])
    idx = torch.from_numpy(np.stack([b, x, y, z], 1).astype(np.int32)).to(cuda)
    rb, _ = ops.get_rulebook(idx, B, shape, ks, st, pd, 1, 0, subm)
    return rb.nbr, n


def run_case(cuda, prec, cin, cout, kv, n_out, seed, geom=None, misalign=False):
    from bevfusion_b200.spconv import ops
    gen = torch.Generator(device=cuda).manual_seed(seed)
    if geom is not None:
        nbr, n_in = geometric_table(geom, seed, cuda)
        n_out = nbr.shape[1]
    else:
        n_in = n_out + n_out // 8 + 16
        nbr = random_table(kv, n_in, n_out, gen)
    f = torch.randn(n_in, cin, device=cuda, generator=gen)
    if misalign:                                   # 4 bytes past a 256-byte aligned allocation
        buf = torch.empty(n_in * cin + 1, device=cuda)
        buf[1:] = f.flatten()
        f = buf[1:].view(n_in, cin)
        assert f.data_ptr() % 16 == 4
    w = torch.randn(kv, cin, cout, device=cuda, generator=gen) / (cin * kv) ** 0.5
    g = torch.randn(n_out, cout, device=cuda, generator=gen)
    nbr_t = ops.transpose_nbr(nbr, n_in)
    din, dw = backward_cabi(f, w, g, nbr, nbr_t, prec)
    din2, dw2 = backward_cabi(f, w, g, nbr, nbr_t, prec)
    assert torch.equal(din, din2) and torch.equal(dw, dw2), "not bit-reproducible"
    # the Python binding (own transposed table, own workspace) runs the same kernels
    pdin, pdw = ops.sparse_conv_backward(f, w, g, nbr, precision=prec)
    assert torch.equal(pdin, din) and torch.equal(pdw, dw), "ops.sparse_conv_backward differs from the C ABI"
    ref_din, ref_dw, fed = reference(f, w, g, nbr)
    errs = check(din, dw, ref_din, ref_dw, fed, prec, "prec %d (%d,%d) kvol %d n_out %d" % (prec, cin, cout, kv, n_out))
    print("prec %d  %3d -> %3d  kvol %2d  n_out %5d  dIn %.2e  dW %.2e" % (prec, cin, cout, kv, n_out, *errs))
    return errs


# ---------------------------------------------------------------------------------------------------- dispatch
def case(prec, cin, cout, kv, n_out=3000, geom=None, misalign=False):
    tag = "p%d-%dx%d-k%d-n%d%s%s" % (prec, cin, cout, kv, n_out, "-" + geom if geom else "", "-misaligned" if misalign else "")
    return pytest.param(prec, cin, cout, kv, n_out, geom, misalign, id=tag)


DISPATCH = [
    # precision 0: dIn = SIMT forward on nbr_t; dW = spconv_wgrad2_kernel<Cin/16, Cout/16>
    case(0, 16, 16, 27, geom="subm_k3"),        # wgrad2<1,1>: the stage-1 SubM shape
    case(0, 32, 16, 27),                        # wgrad2<2,1>
    case(0, 64, 32, 27),                        # wgrad2<4,2>
    case(0, 128, 64, 27),                       # wgrad2<8,4>
    # precision 0: dW = generic spconv_wgrad_kernel
    case(0, 16, 64, 27),                        # power-of-16 pair outside the wgrad2 switch -> generic <2,2>
    case(0, 128, 16, 27),                       # ditto -> generic <2,2>
    case(0, 64, 100, 27),                       # generic <4,4>, Cout tail
    case(0, 48, 40, 27),                        # generic <2,2>, Cin and Cout tails
    case(0, 24, 8, 27),                         # generic <1,1>, tails
    # features 4 bytes off 16-byte alignment: no float4 loads, no tensor-core dW
    case(0, 32, 32, 27, misalign=True),         # dIn SIMT; dW generic <2,2> (misaligned fallback)
    case(3, 32, 32, 27, misalign=True),         # dIn BF16x3 forward on its own split (not shared); dW generic <2,2>
    # precision 3, Cout in {32, 64, 128}: tensor-core dW, then dIn gathers from dW's out-grad image (shared image)
    case(3, 16, 32, 27),                        # dIn mma.sync (Cout' = 16); dW images (32, 32)
    case(3, 64, 32, 27),                        # dIn wgmma fed by a 32-channel image (27 K blocks); dW images (64, 32)
    case(3, 128, 64, 27),                       # dIn wgmma, Cout' = 128; dW images (128, 64)
    case(3, 32, 128, 27),                       # dIn mma.sync (Cout' = 32); dW images (32, 128)
    case(3, 64, 64, 8),                         # dIn wgmma at exactly 16 K blocks (the threshold); dW images (64, 64)
    case(3, 64, 32, 8),                         # dIn mma.sync at 8 K blocks; dW images (64, 32)
    case(3, 32, 64, 27, geom="conv_k3s2p1"),    # shared image on a strided rulebook (n_out < n_in)
    # precision 3, Cout = 16: tensor-core dW with co_eff 32 (padded); dIn = BF16x3 forward with its own temporaries
    case(3, 16, 16, 27, geom="subm_k3"),        # the stage-1 SubM
    case(3, 64, 16, 27),
    # precision 3, Cin not a tensor-core output width: dIn SIMT; dW tensor cores with padded ci_eff
    case(3, 48, 64, 27),                        # ci_eff 64
    case(3, 100, 32, 27),                       # ci_eff 128
    case(3, 5, 32, 27),                         # ci_eff 32 (conv_input's Cin)
    # precision 3, Cout with no tensor-core dW form: dIn BF16x3 forward with temporaries (Cin' 48 -> 64); dW SIMT <2,2>
    case(3, 32, 48, 27),
    # precision 1 (3xTF32): dIn on mma.sync; dW SIMT
    case(1, 64, 48, 27),                        # out-grad rows padded 48 -> 64; dW generic <2,2>
    case(1, 16, 16, 27),                        # dW wgrad2<1,1>
    # precision 2 (TF32): dIn single-pass TF32; dW still on the BF16x3-class tensor-core kernel
    case(2, 32, 64, 27, geom="conv_k3s2p1"),
    case(2, 64, 16, 3),                         # co_eff 32; chunk count clamped to the tile count
    # kernel volume 1
    case(3, 32, 64, 1),                         # shared image, dIn mma.sync; dW tensor cores
    case(0, 32, 64, 1),                         # SIMT dIn; dW wgrad2<2,4>
]


@pytest.mark.parametrize("prec,cin,cout,kv,n_out,geom,misalign", DISPATCH)
def test_backward_dispatch(cuda, prec, cin, cout, kv, n_out, geom, misalign):
    run_case(cuda, prec, cin, cout, kv, n_out, seed=1000 * cin + 10 * cout + kv + prec, geom=geom, misalign=misalign)


# row counts around the 32-row tensor-core tile and the 2048-row SIMT chunk
@pytest.mark.parametrize("n_out", [1, 31, 32, 33, 2047, 2048, 2049, 4097])
@pytest.mark.parametrize("prec,cin,cout", [(0, 32, 64), (3, 32, 64), (0, 16, 16), (3, 16, 16)])
def test_backward_row_counts(cuda, prec, cin, cout, n_out):
    run_case(cuda, prec, cin, cout, 27, n_out, seed=n_out + 7 * cin + prec)


@pytest.mark.parametrize("prec", [0, 3])
def test_backward_chunk_count_clamped_to_tiles(cuda, prec):
    # kvol 3 asks for 132 chunks; 200 rows are 7 tiles of 32
    run_case(cuda, prec, 32, 64, 3, 200, seed=31 + prec)


# ---------------------------------------------------------------------------------------------------- edges
@pytest.mark.parametrize("prec", [0, 3])
def test_backward_no_output_rows(cuda, prec):
    n_in, cin, cout, kv = 300, 32, 64, 27
    f = torch.randn(n_in, cin, device=cuda)
    w = torch.randn(kv, cin, cout, device=cuda)
    nbr = torch.empty(kv, 0, dtype=torch.int32, device=cuda)
    nbr_t = torch.full((kv, n_in), -1, dtype=torch.int32, device=cuda)
    din, dw = backward_cabi(f, w, torch.empty(0, cout, device=cuda), nbr, nbr_t, prec)
    assert bool((din == 0).all()) and bool((dw == 0).all())


@pytest.mark.parametrize("prec", [0, 3])
def test_backward_no_input_rows(cuda, prec):
    n_out, cin, cout, kv = 100, 32, 64, 27
    nbr = torch.randint(-3, 5, (kv, n_out), dtype=torch.int32, device=cuda)   # nothing is < n_in = 0
    f = torch.empty(0, cin, device=cuda)
    w = torch.randn(kv, cin, cout, device=cuda)
    g = torch.randn(n_out, cout, device=cuda)
    din, dw = backward_cabi(f, w, g, nbr, torch.empty(kv, 0, dtype=torch.int32, device=cuda), prec)
    assert din.shape == (0, cin) and bool((dw == 0).all())


@pytest.mark.parametrize("prec", [0, 3])
def test_backward_workspace_too_small(cuda, prec):
    from bevfusion_b200.spconv import ops
    lib = _C.lib()
    n_in, n_out, cin, cout, kv = 500, 400, 32, 64, 27
    gen = torch.Generator(device=cuda).manual_seed(5)
    nbr = random_table(kv, n_in, n_out, gen)
    f = torch.randn(n_in, cin, device=cuda)
    w = torch.randn(kv, cin, cout, device=cuda)
    g = torch.randn(n_out, cout, device=cuda)
    nbr_t = ops.transpose_nbr(nbr, n_in)
    need = lib.bevb200_spconv_backward_workspace_bytes(n_in, n_out, cin, cout, kv)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda)
    din = torch.empty(n_in, cin, device=cuda)
    dw = torch.empty(kv, cin, cout, device=cuda)
    stream = _C.current_stream(cuda)
    for ptr, size in ((_C.ptr(ws), need - 1), (0, need)):
        rc = lib.bevb200_spconv_backward(_C.ptr(f), _C.ptr(w), _C.ptr(g), _C.ptr(nbr), _C.ptr(nbr_t), n_in, n_out,
                                         cin, cout, kv, prec, _C.ptr(din), _C.ptr(dw), ptr, size, stream)
        assert rc == EWORKSPACE
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------- C3 layers
C3_LAYERS = [("in", 5, 16, True, 3, 1, 1), ("s1 subm", 16, 16, True, 3, 1, 1), ("s1 down", 16, 32, False, 3, 2, 1),
             ("s2 subm", 32, 32, True, 3, 1, 1), ("s2 down", 32, 64, False, 3, 2, 1),
             ("s3 subm", 64, 64, True, 3, 1, 1), ("s3 down", 64, 128, False, 3, 2, [1, 1, 0]),
             ("s4 subm", 128, 128, True, 3, 1, 1), ("out", 128, 128, False, [1, 1, 3], [1, 1, 2], 0)]


@pytest.fixture(scope="module")
def c3_rulebooks(cuda):
    """(name, cin, cout, n_in, nbr) of the nine distinct conv layers of the C3 encoder on the seed-0 cloud."""
    from bevfusion_b200 import synthetic as S
    from bevfusion_b200.spconv import ops
    from bevfusion_b200.voxelize import Voxelization, voxelize_mean
    L = S.LIDAR_C3
    pts = torch.from_numpy(S.lidar_cloud(seed=0)).to(cuda)
    vox = Voxelization(L["voxel_size"], L["point_cloud_range"], L["max_num_points"], L["max_voxels"]).eval()
    _, idx = voxelize_mean(*vox(pts), 0)
    shape = L["sparse_shape"]
    out = []
    for name, cin, cout, subm, ks, st, pd in C3_LAYERS:
        rb, oshape = ops.get_rulebook(idx, 1, shape, ks, st, pd, 1, 0, subm)
        out.append((name, cin, cout, idx.shape[0], rb.nbr))
        if not subm:
            idx, shape = rb.outids, oshape
    return out


@pytest.mark.parametrize("prec", [3, 0])
def test_backward_c3_layers(cuda, c3_rulebooks, prec):
    from bevfusion_b200.spconv import ops
    gen = torch.Generator(device=cuda).manual_seed(prec)
    for name, cin, cout, n_in, nbr in c3_rulebooks:
        kv, n_out = nbr.shape
        f = torch.randn(n_in, cin, device=cuda, generator=gen)
        w = torch.randn(kv, cin, cout, device=cuda, generator=gen) / (cin * kv) ** 0.5
        g = torch.randn(n_out, cout, device=cuda, generator=gen)
        din, dw = backward_cabi(f, w, g, nbr, ops.transpose_nbr(nbr, n_in), prec)
        ref_din, ref_dw, fed = reference(f, w, g, nbr)
        errs = check(din, dw, ref_din, ref_dw, fed, prec, name)
        print("C3 %-8s prec %d  n_in %6d n_out %6d  %3d -> %3d  dIn %.2e  dW %.2e" % (name, prec, n_in, n_out, cin, cout,
                                                                                   *errs))


# ---------------------------------------------------------------------------------------------------- training step
def _twin_forward(m, feats, coors, batch_size, sparse_shape, masks, flips):
    """SparseEncoder.forward in whatever dtype `m` has, with rulebooks from the CPU oracle (strided outputs put in
    ascending flat-index order, the order of ours), convs as gather / matmul / index_add_, torch BN, dense() as
    index_put.  Each ReLU applies the next of `masks` (the run under test's ReLU masks, in execution order): a
    pre-activation within rounding of 0 may fall on the other side of the kink in fp32, and one flipped element
    moves a gradient by far more than any kernel error.  `flips` collects, per ReLU, (elements whose sign differs
    from the mask, max |pre-activation| among them / max |pre-activation|)."""
    from bevfusion_b200.sparse_block import SparseBasicBlock
    dev = feats.device
    books = {}
    masks = iter(masks)

    def conv(mod, f, idx, shape):
        key = (id(idx), tuple(mod.kernel_size), tuple(mod.stride), tuple(mod.padding), mod.subm)
        if key not in books:
            outids, pairs, num, oshape = oracle.get_indice_pairs(idx, batch_size, shape, mod.kernel_size, mod.stride,
                                                                 mod.padding, mod.dilation, mod.subm)
            inv = np.arange(outids.shape[0])
            if not mod.subm:
                order = np.argsort(oracle.flat_index(outids, oshape), kind="stable")
                inv[order] = np.arange(order.size)
                outids = outids[order]
            pl = [(torch.from_numpy(pairs[k, 0, :num[k]]).long().to(dev),
                   torch.from_numpy(inv[pairs[k, 1, :num[k]]]).long().to(dev)) for k in range(num.shape[0])]
            books[key] = (idx if mod.subm else outids, pl, list(oshape))
        oidx, pl, oshape = books[key]
        w = mod.weight.reshape(-1, mod.in_channels, mod.out_channels)
        out = f.new_zeros(oidx.shape[0], mod.out_channels)
        for k, (i, o) in enumerate(pl):
            if i.numel():
                out.index_add_(0, o, f[i] @ w[k])
        return out, oidx, oshape

    def relu(pre):
        mask = next(masks)
        flip = (pre.detach() > 0) != mask
        top = float(pre.detach().abs().max())
        flips.append((int(flip.sum()), float(pre.detach()[flip].abs().max()) / top if flip.any() else 0.0))
        return pre * mask

    def seq(s, f, idx, shape):
        f, idx, shape = conv(s[0], f, idx, shape)
        return relu(s[1](f)), idx, shape

    idx, shape = coors.cpu().numpy(), list(sparse_shape)
    f, idx, shape = seq(m.conv_input, feats, idx, shape)
    for stage in m.encoder_layers:
        for block in stage:
            if isinstance(block, SparseBasicBlock):
                o, _, _ = conv(block.conv1, f, idx, shape)
                o = relu(block.norm1(o))
                o, _, _ = conv(block.conv2, o, idx, shape)
                f = relu(block.norm2(o) + f)
            else:
                f, idx, shape = seq(block, f, idx, shape)
    f, idx, shape = seq(m.conv_out, f, idx, shape)
    assert next(masks, None) is None, "the twin ran fewer ReLUs than the model"
    li = torch.from_numpy(idx).long().to(dev)
    dense = f.new_zeros(batch_size, *shape, f.shape[1]).index_put((li[:, 0], li[:, 1], li[:, 2], li[:, 3]), f)
    dense = dense.permute(0, 4, 3, 1, 2)                                   # [B, C, Z, X, Y]
    N, C, D, H, W = dense.shape
    return dense.reshape(N, C * D, H, W)


def _rel(got, want):
    d = (got.double() - want).flatten()
    return float(d.norm() / want.norm().clamp_min(1e-300)), float(d.abs().max() / want.abs().max().clamp_min(1e-300))


# Relative L2 bounds of the training step per gradient kind: the worst tensor measured on an H100 80GB HBM3 (400 W)
# with 10x headroom, never looser than 1e-4.  fp32: input 2.1e-6, conv weights 2.7e-6, BN weight / bias 3.6e-6,
# running-statistics update 5.5e-6.  bf16x3 (forward and input gradient in BF16x3, about 1e-5 per layer, over 21
# convs): input 2.0e-5, conv 3.6e-5, BN 4.4e-5, statistics 5.5e-6 -- the 1e-4 cap leaves it 2.2x to 5x headroom.
TRAIN_BOUNDS = {"fp32": {"input": 2e-5, "conv": 3e-5, "bn": 4e-5, "stats": 6e-5},
                "bf16x3": {"input": 1e-4, "conv": 1e-4, "bn": 1e-4, "stats": 6e-5}}


@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
def test_encoder_training_step_vs_float64(cuda, monkeypatch, mode):
    from bevfusion_b200 import synthetic as S
    from bevfusion_b200.sparse_encoder import SparseEncoder
    from bevfusion_b200.voxelize import Voxelization, voxelize_mean
    if mode == "fp32":
        monkeypatch.setenv("BEVB200_SPCONV_PRECISION", "fp32")
    else:
        monkeypatch.delenv("BEVB200_SPCONV_PRECISION", raising=False)      # the default
    L = S.LIDAR_C3
    pts = torch.from_numpy(S.lidar_cloud(seed=0)).to(cuda)
    vox = Voxelization(L["voxel_size"], [-12.0, -12.0, -5.0, 12.0, 12.0, 3.0], L["max_num_points"], L["max_voxels"])
    feats, coors = voxelize_mean(*vox.eval()(pts), 0)
    sparse_shape = [320, 320, 41]
    torch.manual_seed(0)
    m = SparseEncoder(in_channels=5, sparse_shape=sparse_shape, output_channels=128,
                      encoder_channels=((16, 16, 32), (32, 32, 64), (64, 64, 128), (128, 128)),
                      encoder_paddings=((0, 0, 1), (0, 0, 1), (0, 0, (1, 1, 0)), (0, 0)),
                      block_type="basicblock").to(cuda)
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm1d):
            mod.running_mean.normal_(0, 0.1); mod.running_var.uniform_(0.5, 1.5)
            mod.weight.data.uniform_(0.8, 1.2); mod.bias.data.normal_(0, 0.1)
    twin = copy.deepcopy(m).double()
    before = {k: v.clone() for k, v in m.named_buffers()}
    m.train(); twin.train()

    masks = []
    hooks = [mod.register_forward_hook(lambda mod, inp, out: masks.append(out.detach() > 0))
             for mod in m.modules() if isinstance(mod, torch.nn.ReLU)]
    x = feats.detach().clone().requires_grad_(True)
    try:
        out = m(x, coors, 1)
    finally:
        for h in hooks:
            h.remove()
    assert len(masks) == 21                             # conv_input, 2 in each of 7 blocks, 3 strided convs, conv_out
    R = torch.randn(out.shape, device=cuda, generator=torch.Generator(device=cuda).manual_seed(1))
    (out * R).sum().backward()
    x64 = feats.detach().double().requires_grad_(True)
    flips = []
    out64 = _twin_forward(twin, x64, coors, 1, sparse_shape, masks, flips)
    assert out64.shape == out.shape
    (out64 * R.double()).sum().backward()

    out_err = _rel(out.detach(), out64.detach())
    n_flip = sum(n for n, _ in flips)
    print("training step (%s), %d voxels: output rel L2 %.2e, max-abs/max %.2e; %d ReLU elements of %d on the other "
          "side of the kink, all within %.1e of max |pre-activation|" % (
              mode, feats.shape[0], *out_err, n_flip, sum(mk.numel() for mk in masks), max(t for _, t in flips)))
    assert out_err[1] <= 1e-4
    # only elements within the forward's 1e-4 parity bar of 0 may sit on the other side of a ReLU kink
    assert max(t for _, t in flips) <= 1e-4 and n_flip <= 1e-4 * sum(mk.numel() for mk in masks)
    bounds = TRAIN_BOUNDS[mode]
    rows = [("input", "features", *_rel(x.grad, x64.grad))]
    p64 = dict(twin.named_parameters())
    for name, p in m.named_parameters():
        rows.append(("bn" if p.dim() == 1 else "conv", name, *_rel(p.grad, p64[name].grad)))
    b64 = dict(twin.named_buffers())
    for name, b in m.named_buffers():
        if name.endswith(("running_mean", "running_var")):       # the step's update of the statistics
            rows.append(("stats", name, *_rel(b - before[name], b64[name].detach() - before[name].double())))
    for kind, name, l2, mx in rows:
        print("  %-5s %-48s rel L2 %.2e  max-abs/max %.2e" % (kind, name, l2, mx))
    for kind in bounds:
        print("  worst %-5s rel L2 %.2e" % (kind, max(l2 for k, _, l2, _ in rows if k == kind)))
    bad = [(name, l2) for kind, name, l2, _ in rows if not l2 <= bounds[kind]]
    assert not bad, bad
