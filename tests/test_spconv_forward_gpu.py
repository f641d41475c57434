"""GPU tests of the sparse-conv forward (bevb200_spconv_forward / bevb200_spconv_forward_packed) against a float64
reference built from the neighbour table directly, on every kernel the dispatch can pick:

  * precision 0: the exact-fp32 SIMT kernel spconv_simt_kernel<16,4> / <32,4> / <64,4> / <128,8>, with channel
    tails and with the float4 loads off (features or weights 4 bytes off 16-byte alignment);
  * precision 3 (BF16x3): the split pass into stream-ordered temporaries, then spconv_v6_kernel (mma.sync) or, at
    Cout >= 64 with >= 16 K blocks, spconv_wg_kernel (warpgroup MMAs); Cin padded to 16 / 32 / 64 / 128;
  * precision 3 falling back to SIMT: Cout with no tensor-core form, `out` or `residual` not 16-byte aligned;
  * precision 1 (3xTF32) and 2 (single-pass TF32): spconv_v6_kernel on fp32 rows, zero-padded to a power of two in
    a temporary when Cin is not one; misaligned unpadded features fall back to SIMT.

Every call fills `out` with NaN, runs twice and must be bit-identical, and ops.sparse_conv (with and without
pre-packed weights) must give exactly the same rows.  Output rows with no valid neighbour must be exactly the fp32
epilogue of 0.  Each case prints its family and relative error."""
import pytest
import torch

from bevfusion_b200 import _C
from encoder_oracle import conv_nbr, epilogue

pytestmark = pytest.mark.gpu

EINVAL, EUNSUPPORTED = -1, -4


# ---------------------------------------------------------------------------------------------------- helpers
def misalign(t):
    """The same values 4 bytes past a 16-byte boundary (a fresh allocation is 256-byte aligned)."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    buf[1:] = t.flatten()
    v = buf[1:].view(t.shape)
    assert v.data_ptr() % 16 == 4
    return v


def forward_cabi(f, w, nbr, prec, scale=None, shift=None, residual=None, relu=False, packed=None, out=None):
    """bevb200_spconv_forward (or _forward_packed when `packed` is given) at an explicit precision into `out`
    (default: a fresh [n_out, Cout] tensor), which is NaN-filled first.  -> (return code, out)."""
    lib = _C.lib()
    n_in, c_in = f.shape
    kv, n_out = nbr.shape
    c_out = w.shape[-1]
    if out is None:
        out = torch.empty(n_out, c_out, device=f.device)
    out.fill_(float("nan"))
    args = (_C.ptr(nbr), n_in, n_out, c_in, c_out, kv, _C.ptr(scale), _C.ptr(shift), _C.ptr(residual), int(relu),
            int(prec), _C.ptr(out), _C.current_stream(f.device))
    if packed is None:
        rc = lib.bevb200_spconv_forward(_C.ptr(f), _C.ptr(w), *args)
    else:
        rc = lib.bevb200_spconv_forward_packed(_C.ptr(f), _C.ptr(packed), *args)
    torch.cuda.synchronize()
    return rc, out


def random_table(kv, n_in, n_out, gen, miss=0.4):
    """nbr [kv, n_out]: random input rows, a fraction `miss` of the entries -1, a few entries >= n_in or < -1 (missing
    too), one offset with no pair at all and every 13th output row from row 6 on with no valid neighbour."""
    dev = gen.device
    nbr = torch.randint(0, n_in, (kv, n_out), generator=gen, device=dev, dtype=torch.int32)
    nbr[torch.rand(kv, n_out, generator=gen, device=dev) < miss] = -1
    vals = torch.tensor([n_in, n_in + 7, 2 ** 31 - 1, -2, -1000, -2 ** 31], dtype=torch.int32, device=dev)
    pos = torch.rand(kv, n_out, generator=gen, device=dev) < 0.01
    pick = torch.randint(0, vals.numel(), (kv, n_out), generator=gen, device=dev)
    nbr[pos] = vals[pick[pos]]
    if kv > 1:
        nbr[kv // 3] = -1
    empty = nbr[:, 6::13]
    nbr[:, 6::13] = torch.where(torch.rand(empty.shape, generator=gen, device=dev) < 0.8, -1, vals[pick[:, 6::13]])
    return nbr


def empty_rows(nbr, n_in):
    return ~((nbr >= 0) & (nbr < n_in)).any(0)


EPILOGUES = {"none": (False, False, False, False), "scale": (True, False, False, False),
             "shift": (False, True, False, False), "relu": (False, False, False, True),
             "full": (True, True, True, True)}


def run_case(cuda, prec, cin, cout, kv, n_out, seed, family, mis="", epi="full"):
    """One forward at `prec` against float64.  mis: which pointers sit 4 bytes off alignment -- f(eatures),
    w(eights), r(esidual), o(ut).  Returns the relative error."""
    from bevfusion_b200.spconv import ops
    gen = torch.Generator(device=cuda).manual_seed(seed)
    n_in = n_out + n_out // 8 + 16
    nbr = random_table(kv, n_in, n_out, gen)
    f = torch.randn(n_in, cin, device=cuda, generator=gen)
    w = torch.randn(kv, cin, cout, device=cuda, generator=gen) / (cin * kv) ** 0.5
    use_scale, use_shift, use_res, relu = EPILOGUES[epi]
    scale = torch.rand(cout, device=cuda, generator=gen) + 0.5 if use_scale else None
    shift = torch.randn(cout, device=cuda, generator=gen) * 0.5 if use_shift else None
    res = torch.randn(n_out, cout, device=cuda, generator=gen) * 0.5 if use_res else None
    if "f" in mis:
        f = misalign(f)
    if "w" in mis:
        w = misalign(w)
    if "r" in mis:
        res = misalign(res)
    out = misalign(torch.empty(n_out, cout, device=cuda)) if "o" in mis else None
    rc, got = forward_cabi(f, w, nbr, prec, scale, shift, res, relu, out=out)
    assert rc == 0, _C.lib().bevb200_last_error()
    assert not bool(torch.isnan(got).any()), "the forward left rows unwritten"
    got = got.clone()
    rc, again = forward_cabi(f, w, nbr, prec, scale, shift, res, relu, out=out)
    assert rc == 0 and torch.equal(got, again), "not bit-reproducible"

    # the Python binding runs the same kernel (its `out` is aligned, so not for a misaligned-out case)
    py = ops.sparse_conv(f, w, nbr, n_out, scale, shift, res, relu, prec)
    if "o" not in mis:
        assert torch.equal(py, got), "ops.sparse_conv differs from the C ABI"
    packed = ops.pack_weights(w, prec) if prec != 0 else None
    if packed is not None:
        # pre-packed weights: the same kernel, unless the call would need the SIMT fallback, which has no packed form
        needs_simt = "r" in mis or ("f" in mis and prec in (1, 2) and cin in (8, 16, 32, 64, 128))
        if needs_simt:
            with pytest.raises(_C.BevB200Error):
                ops.sparse_conv(f, w, nbr, n_out, scale, shift, res, relu, prec, packed=packed)
        else:
            pk = ops.sparse_conv(f, w, nbr, n_out, scale, shift, res, relu, prec, packed=packed)
            assert torch.equal(pk, py), "pre-packed weights give a different result"

    ref = epilogue(conv_nbr(f, w, nbr), scale, shift, res, relu)
    den = float(ref.abs().max())
    err = float((got.double() - ref).abs().max()) / max(den, 1e-300)
    tol = 3e-3 if prec == 2 else 1e-4
    what = "%s prec %d %d->%d kvol %d n_out %d mis '%s' epi %s" % (family, prec, cin, cout, kv, n_out, mis, epi)
    print("%-14s prec %d  %3d -> %3d  kvol %2d  n_out %6d  mis %-2s epi %-5s  rel err %.2e" % (
        family, prec, cin, cout, kv, n_out, mis, epi, err))
    assert err <= tol, "%s: rel err %.3e > %.0e" % (what, err, tol)
    # rows with no valid neighbour: exactly the fp32 epilogue of 0
    e = empty_rows(nbr, n_in)
    assert bool(e.any()) or n_out <= 6
    want = epilogue(torch.zeros(int(e.sum()), cout, device=cuda), scale, shift, None if res is None else res[e], relu)
    assert torch.equal(got[e], want), "%s: a row with no neighbour is not the epilogue of 0" % what
    return err


# ---------------------------------------------------------------------------------------------------- dispatch
def case(prec, cin, cout, kv, family, mis="", n_out=2000):
    tag = "p%d-%dx%d-k%d-%s%s" % (prec, cin, cout, kv, family, "-mis" + mis if mis else "")
    return pytest.param(prec, cin, cout, kv, family, mis, n_out, id=tag)


DISPATCH = [
    # precision 0: spconv_simt_kernel<BN, TN>, BN the smallest of 16 / 32 / 64 / 128 >= Cout
    case(0, 5, 8, 27, "simt<16,4>"),            # Cin and Cout tails
    case(0, 16, 16, 27, "simt<16,4>"),
    case(0, 24, 24, 27, "simt<32,4>"),          # tails
    case(0, 32, 32, 27, "simt<32,4>"),
    case(0, 48, 48, 27, "simt<64,4>"),          # tails
    case(0, 64, 64, 27, "simt<64,4>"),
    case(0, 100, 100, 27, "simt<128,8>"),       # tails
    case(0, 128, 128, 27, "simt<128,8>"),
    case(0, 32, 64, 27, "simt<64,4>", mis="fw"),     # no float4 loads of features or weights
    case(0, 5, 100, 27, "simt<128,8>", mis="fw"),    # ditto, with tails
    case(0, 16, 32, 1, "simt<32,4>"),           # kernel volume 1
    # precision 3 (BF16x3), split temporaries: spconv_v6_kernel (mma.sync) below Cout 64 or 16 K blocks
    case(3, 16, 16, 27, "mma.sync"),            # 14 K blocks (one block spans two offsets)
    case(3, 32, 32, 27, "mma.sync"),
    case(3, 16, 64, 27, "mma.sync"),            # Cout 64 at 14 K blocks
    case(3, 64, 32, 8, "mma.sync"),
    case(3, 128, 128, 3, "mma.sync"),           # conv_out's k(1,1,3): 12 K blocks at Cout 128
    case(3, 32, 64, 1, "mma.sync"),             # kernel volume 1: one K block
    case(3, 16, 16, 1, "mma.sync"),             # kernel volume 1: half a K block
    case(3, 5, 16, 27, "mma.sync"),             # Cin 5 -> 16
    case(3, 24, 32, 27, "mma.sync"),            # Cin 24 -> 32
    # precision 3, spconv_wg_kernel (warpgroup MMAs): Cout 64 / 128 with >= 16 K blocks
    case(3, 64, 64, 8, "wgmma"),                # exactly 16 K blocks
    case(3, 64, 64, 27, "wgmma"),
    case(3, 32, 128, 27, "wgmma"),
    case(3, 128, 128, 27, "wgmma"),
    case(3, 48, 64, 27, "wgmma"),               # Cin 48 -> 64
    case(3, 100, 128, 27, "wgmma"),             # Cin 100 -> 128
    case(3, 32, 64, 27, "wgmma", mis="f"),      # the split pass reads misaligned features
    # precision 3 falling back to the SIMT kernel
    case(3, 32, 48, 27, "bf16x3->simt"),        # Cout 48 has no tensor-core form
    case(3, 32, 64, 27, "bf16x3->simt", mis="o"),
    case(3, 16, 32, 27, "bf16x3->simt", mis="r"),
    # precision 1 (3xTF32): spconv_v6_kernel<2, Cout> on fp32 rows
    case(1, 5, 16, 27, "tf32x3"),               # Cin 5 -> 8 in a padded temporary
    case(1, 24, 32, 27, "tf32x3"),              # 24 -> 32
    case(1, 100, 128, 27, "tf32x3"),            # 100 -> 128
    case(1, 32, 64, 27, "tf32x3"),              # unpadded
    case(1, 5, 16, 27, "tf32x3", mis="f"),      # the pad kernel reads misaligned features
    case(1, 32, 32, 27, "tf32x3->simt", mis="f"),    # unpadded misaligned rows: SIMT
    case(1, 16, 48, 27, "tf32x3->simt"),        # Cout 48
    # precision 2 (single-pass TF32): spconv_v6_kernel<1, Cout>
    case(2, 32, 64, 27, "tf32"),
    case(2, 5, 16, 27, "tf32"),                 # Cin 5 -> 8
]


@pytest.mark.parametrize("prec,cin,cout,kv,family,mis,n_out", DISPATCH)
def test_forward_dispatch(cuda, prec, cin, cout, kv, family, mis, n_out):
    run_case(cuda, prec, cin, cout, kv, n_out, 1000 * cin + 10 * cout + kv + prec, family, mis)


# the fused epilogue in every combination the encoder uses, on each kernel family
FAMILIES = {"simt": (0, 32, 32, 27), "mma.sync": (3, 32, 32, 27), "wgmma": (3, 64, 64, 27),
            "tf32x3": (1, 32, 32, 27), "tf32": (2, 32, 32, 27)}


@pytest.mark.parametrize("epi", list(EPILOGUES))
@pytest.mark.parametrize("family", list(FAMILIES))
def test_forward_epilogue(cuda, family, epi):
    prec, cin, cout, kv = FAMILIES[family]
    run_case(cuda, prec, cin, cout, kv, 1500, 17 + prec + len(epi), family, epi=epi)


# row counts around the 128-row tiles (SIMT <32,4>, mma.sync), the 256-row wgmma tile, and past the persistent
# loop's first wave (2 CTAs x 132 SMs x 256 rows)
@pytest.mark.parametrize("n_out", [1, 127, 128, 129, 255, 256, 257, 2 * 132 * 256 + 1])
@pytest.mark.parametrize("family", ["simt", "mma.sync", "wgmma"])
def test_forward_row_counts(cuda, family, n_out):
    prec, cin, cout, kv = FAMILIES[family]
    run_case(cuda, prec, cin, cout, kv, n_out, n_out + prec, family)


# ---------------------------------------------------------------------------------------------------- edges
@pytest.mark.parametrize("prec", [0, 1, 3])
def test_forward_no_output_rows(cuda, prec):
    """n_out = 0: success, and nothing is written (also through the packed entry point)."""
    from bevfusion_b200.spconv import ops
    f = torch.randn(300, 32, device=cuda)
    w = torch.randn(27, 32, 64, device=cuda)
    nbr = torch.empty(27, 0, dtype=torch.int32, device=cuda)
    canary = torch.full((8, 64), float("nan"), device=cuda)
    lib = _C.lib()
    stream = _C.current_stream(cuda)
    assert lib.bevb200_spconv_forward(_C.ptr(f), _C.ptr(w), _C.ptr(nbr), 300, 0, 32, 64, 27, 0, 0, 0, 1, prec,
                                      _C.ptr(canary), stream) == 0
    if prec:
        pk = ops.pack_weights(w, prec)
        assert lib.bevb200_spconv_forward_packed(_C.ptr(f), _C.ptr(pk), _C.ptr(nbr), 300, 0, 32, 64, 27, 0, 0, 0, 1,
                                                 prec, _C.ptr(canary), stream) == 0
    torch.cuda.synchronize()
    assert bool(torch.isnan(canary).all())
    assert ops.sparse_conv(f, w, nbr, 0, precision=prec).shape == (0, 64)


@pytest.mark.parametrize("cin", [5, 32])
@pytest.mark.parametrize("prec", [0, 1, 2, 3])
def test_forward_no_input_rows(cuda, prec, cin):
    """n_in = 0: every entry is missing, so every row is exactly the epilogue of 0."""
    from bevfusion_b200.spconv import ops
    n_out, cout, kv = 300, 64, 27
    gen = torch.Generator(device=cuda).manual_seed(prec)
    f = torch.empty(0, cin, device=cuda)
    w = torch.randn(kv, cin, cout, device=cuda, generator=gen)
    nbr = torch.randint(-3, 5, (kv, n_out), dtype=torch.int32, device=cuda, generator=gen)   # nothing is < n_in
    scale = torch.rand(cout, device=cuda, generator=gen) + 0.5
    shift = torch.randn(cout, device=cuda, generator=gen)
    res = torch.randn(n_out, cout, device=cuda, generator=gen)
    want = epilogue(torch.zeros(n_out, cout, device=cuda), scale, shift, res, True)
    rc, got = forward_cabi(f, w, nbr, prec, scale, shift, res, True)
    assert rc == 0 and torch.equal(got, want)
    assert torch.equal(ops.sparse_conv(f, w, nbr, n_out, scale, shift, res, True, prec), want)


@pytest.mark.parametrize("cout", [129, 256])
@pytest.mark.parametrize("prec", [0, 3])
def test_forward_cout_above_128_is_unsupported(cuda, prec, cout):
    f = torch.randn(100, 32, device=cuda)
    w = torch.randn(27, 32, cout, device=cuda)
    nbr = torch.randint(-1, 100, (27, 80), dtype=torch.int32, device=cuda)
    rc, out = forward_cabi(f, w, nbr, prec)
    assert rc == EUNSUPPORTED
    assert bool(torch.isnan(out).all())


@pytest.mark.parametrize("prec", [1, 3])
def test_forward_packed_misaligned_out_is_an_error(cuda, prec):
    """Pre-packed weights have no SIMT form, so an `out` the tensor cores cannot store to is refused, and nothing is
    written."""
    from bevfusion_b200.spconv import ops
    f = torch.randn(400, 32, device=cuda)
    w = torch.randn(27, 32, 64, device=cuda)
    nbr = torch.randint(-1, 400, (27, 300), dtype=torch.int32, device=cuda)
    out = misalign(torch.empty(300, 64, device=cuda))
    rc, out = forward_cabi(f, w, nbr, prec, packed=ops.pack_weights(w, prec), out=out)
    assert rc == EINVAL
    assert bool(torch.isnan(out).all())
