"""GPU tests of the BF16x3 sparse-conv forward through its C entry point bevb200_spconv_forward_split, on random
neighbour tables.  Cout >= 64 with >= 16 K blocks runs the warpgroup-MMA kernel, the rest the mma.sync kernel.
Covered: row counts that are not a multiple of the tile, a device-side row count below the host one, a neighbour
table wider than the row count, each output alone, every Cout with Cin up to 128, the float64 oracle, and
bit-reproducibility."""
import pytest
import torch

from bevfusion_b200 import _C

pytestmark = pytest.mark.gpu


def _split_rows(f):
    lib = _C.lib()
    n, c = f.shape
    ce = lib.bevb200_spconv_split_channels(c)
    out = torch.empty((n, ce * 4), dtype=torch.uint8, device=f.device)
    _C.check(lib.bevb200_spconv_split_rows(_C.ptr(f), n, 0, c, _C.ptr(out), _C.current_stream(f.device)), "split_rows")
    return out, ce


def _pack(w):
    lib = _C.lib()
    kv, cin, cout = w.shape
    pk = torch.empty(lib.bevb200_spconv_split_weight_bytes(cin, cout, kv), dtype=torch.uint8, device=w.device)
    _C.check(lib.bevb200_spconv_pack_split_weights(_C.ptr(w), cin, cout, kv, _C.ptr(pk), _C.current_stream(w.device)),
             "pack")
    return pk


def _forward(fs, ce, pk, nbr, n_in, cout, scale, shift, residual, relu, n_dev=None, want_out=True, want_split=True,
             n_out=None):
    """-> (fp32 rows or None, split image or None); rows not produced keep the NaN / 0xff fill.  nbr is
    [kv, nbr_stride]; n_out (default nbr_stride) may be smaller, as in the encoder's cap-wide tables."""
    kv, stride = nbr.shape
    n_out = stride if n_out is None else n_out
    out = torch.full((n_out, cout), float("nan"), device=fs.device) if want_out else None
    osp = torch.full((n_out, cout * 4), 255, dtype=torch.uint8, device=fs.device) if want_split else None
    _C.check(_C.lib().bevb200_spconv_forward_split(
        _C.ptr(fs), _C.ptr(pk), _C.ptr(nbr), stride, n_in, n_out, _C.ptr(n_dev), ce, cout, kv, _C.ptr(scale),
        _C.ptr(shift), _C.ptr(residual), int(relu), _C.ptr(out), _C.ptr(osp), _C.current_stream(fs.device)),
        "forward_split")
    return out, osp


def _decode_split(osp, c):
    n = osp.shape[0]
    w = osp.view(torch.int16).view(n, c // 16, 2, 16)          # [row, group, hi | lo, 16 bf16]
    f = (w.to(torch.int32) << 16).view(torch.float32)
    return (f[:, :, 0, :] + f[:, :, 1, :]).reshape(n, c)


def _oracle(f, w, nbr, scale, shift, residual, relu):
    f64, w64 = f.double(), w.double()
    out = torch.zeros(nbr.shape[1], w.shape[2], dtype=torch.float64, device=f.device)
    for k in range(nbr.shape[0]):
        m = nbr[k] >= 0
        out[m] += f64[nbr[k][m].long()] @ w64[k]
    out = out * scale.double() + shift.double() + residual.double()
    return out.clamp_min(0) if relu else out


def _case(cin, cout, n_in, n_out, kv, seed, cuda):
    g = torch.Generator(device=cuda).manual_seed(seed)
    f = torch.randn(n_in, cin, device=cuda, generator=g)
    w = torch.randn(kv, cin, cout, device=cuda, generator=g) / (cin * kv) ** 0.5
    nbr = torch.randint(0, n_in, (kv, n_out), device=cuda, generator=g, dtype=torch.int32)
    nbr[torch.rand(kv, n_out, device=cuda, generator=g) < 0.5] = -1       # missing neighbours
    scale = torch.rand(cout, device=cuda, generator=g) + 0.5
    shift = torch.randn(cout, device=cuda, generator=g) * 0.1
    res = torch.randn(n_out, cout, device=cuda, generator=g) * 0.1
    return f, w, nbr, scale, shift, res


@pytest.mark.parametrize("cout", [16, 32, 64, 128])
@pytest.mark.parametrize("cin", [5, 16, 32, 64, 128])
def test_forward_vs_float64_with_device_row_count(cin, cout, cuda):
    # 1000 rows: neither 128- nor 256-row tiles divide it; the device count stops 131 rows short of it
    n_in, n_out, n_dev_val, kv = 1500, 1000, 869, 27
    f, w, nbr, scale, shift, res = _case(cin, cout, n_in, n_out, kv, cin * 1000 + cout, cuda)
    fs, ce = _split_rows(f)
    pk = _pack(w)
    n_dev = torch.tensor([n_dev_val], dtype=torch.int32, device=cuda)
    out, osp = _forward(fs, ce, pk, nbr, n_in, cout, scale, shift, res, True, n_dev=n_dev)
    gold = _oracle(f, w, nbr, scale, shift, res, True)
    torch.cuda.synchronize()
    den = gold[:n_dev_val].abs().max().item()
    err = (out[:n_dev_val].double() - gold[:n_dev_val]).abs().max().item() / den
    print(f"cin {cin} cout {cout}: max rel err vs float64 {err:.2e}")
    assert err <= 1e-4
    # the split image is the split of the fp32 rows (hi + lo exact to 2^-17 |x|)
    dec = _decode_split(osp[:n_dev_val], cout)
    assert ((dec - out[:n_dev_val]).abs() <= out[:n_dev_val].abs() * 2.0 ** -16).all()
    # rows at or past the device count are not written
    assert torch.isnan(out[n_dev_val:]).all() and (osp[n_dev_val:] == 255).all()


@pytest.mark.parametrize("cout", [16, 128])
def test_each_output_alone_and_bit_reproducible(cout, cuda):
    n_in, n_out, kv, cin = 3000, 2 * 256 * 132 + 77, 27, 64          # more tiles than SMs: the persistent loop
    f, w, nbr, scale, shift, res = _case(cin, cout, n_in, n_out, kv, 7 + cout, cuda)
    fs, ce = _split_rows(f)
    pk = _pack(w)
    both_out, both_split = _forward(fs, ce, pk, nbr, n_in, cout, scale, shift, res, False)
    again_out, again_split = _forward(fs, ce, pk, nbr, n_in, cout, scale, shift, res, False)
    only_out, none_split = _forward(fs, ce, pk, nbr, n_in, cout, scale, shift, res, False, want_split=False)
    none_out, only_split = _forward(fs, ce, pk, nbr, n_in, cout, scale, shift, res, False, want_out=False)
    torch.cuda.synchronize()
    assert none_split is None and none_out is None
    assert torch.equal(both_out, again_out) and torch.equal(both_split, again_split)
    assert torch.equal(only_out, both_out) and torch.equal(only_split, both_split)
    gold = _oracle(f, w, nbr, scale, shift, res, False)
    err = (both_out.double() - gold).abs().max().item() / gold.abs().max().item()
    assert err <= 1e-4


# a neighbour table wider than n_out (nbr_stride = the level's row cap, as bevb200_encoder_forward lays it out): the
# columns past n_out hold in-range rows that must not be read
@pytest.mark.parametrize("cin,cout,kv", [(16, 16, 27), (32, 32, 27), (16, 64, 27), (64, 64, 27), (32, 128, 27),
                                         (128, 128, 3)])
def test_forward_nbr_stride_wider_than_rows(cin, cout, kv, cuda):
    n_in, n_out, stride = 1500, 1000, 1337
    f, w, nbr, scale, shift, res = _case(cin, cout, n_in, n_out, kv, 31 * cin + cout, cuda)
    wide = torch.randint(0, n_in, (kv, stride), device=cuda, dtype=torch.int32,
                         generator=torch.Generator(device=cuda).manual_seed(cout))
    wide[:, :n_out] = nbr
    fs, ce = _split_rows(f)
    pk = _pack(w)
    out, osp = _forward(fs, ce, pk, wide, n_in, cout, scale, shift, res, True, n_out=n_out)
    gold = _oracle(f, w, nbr, scale, shift, res, True)
    torch.cuda.synchronize()
    err = (out.double() - gold).abs().max().item() / gold.abs().max().item()
    print(f"cin {cin} cout {cout} kvol {kv}: nbr_stride {stride} > n_out {n_out}, max rel err vs float64 {err:.2e}")
    assert err <= 1e-4
    dec = _decode_split(osp, cout)
    assert ((dec - out).abs() <= out.abs() * 2.0 ** -16).all()
