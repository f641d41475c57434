"""spconv.ops -- host-side mirror of mmdet3d/ops/spconv/ops.py and of the pybind module
`sparse_conv_ext` (src/all.cc:22-50), backed by libbevfusion_b200.so.

Reference-compatible entry points (same names / argument order / return layouts):
    get_conv_output_size, get_deconv_output_size
    get_indice_pairs(...) -> (outids, indice_pairs[K,2,N], indice_pair_num[K])
    indice_conv(features, filters, indice_pairs, indice_pair_num, num_activate_out, inverse, subm)
    sparse_conv_ext.get_indice_pairs_3d / indice_conv_fp32
native entry points:
    get_rulebook(...) -> Rulebook   (neighbour table nbr[K, n_out]; legacy pairs built lazily)
    sparse_conv(features, weight, rulebook, scale, shift, residual, relu, precision)
"""
import ctypes
import os

import torch

from .. import _C

PREC_FP32, PREC_TF32X3, PREC_TF32, PREC_BF16X3 = 0, 1, 2, 3
_PREC_NAMES = {"fp32": PREC_FP32, "tf32x3": PREC_TF32X3, "tf32": PREC_TF32, "bf16x3": PREC_BF16X3}


def default_precision():
    """Precision of the sparse-conv GEMMs: env BEVB200_SPCONV_PRECISION in {fp32, tf32x3, tf32,
    bf16x3}.  Default bf16x3: features and weights split into two bf16 parts, three kind::f16 MMAs
    with fp32 accumulation -- 5e-6 .. 8e-6 of max|out| against the float64 oracle (3xTF32: 1e-6 ..
    1e-5), half the operand bytes and half the MMA instructions of 3xTF32."""
    return _PREC_NAMES[os.environ.get("BEVB200_SPCONV_PRECISION", "bf16x3").lower()]


def get_conv_output_size(input_size, kernel_size, stride, padding, dilation):
    # ops.py:20-31
    ndim = len(input_size)
    output_size = []
    for i in range(ndim):
        size = (input_size[i] + 2 * padding[i] - dilation[i] * (kernel_size[i] - 1) - 1) // stride[i] + 1
        output_size.append(1 if kernel_size[i] == -1 else size)
    return output_size


def get_deconv_output_size(input_size, kernel_size, stride, padding, dilation, output_padding):
    # ops.py:34-42
    ndim = len(input_size)
    output_size = []
    for i in range(ndim):
        if kernel_size[i] == -1:
            raise ValueError("deconv don't support kernel_size < 0")
        output_size.append((input_size[i] - 1) * stride[i] - 2 * padding[i] + kernel_size[i]
                           + output_padding[i])
    return output_size


def _i32(vals):
    return _C.host_array(ctypes.c_int32, [int(v) for v in vals])


def _vp(arr):
    return ctypes.cast(arr, ctypes.c_void_p)


class Rulebook:
    """Neighbour-table rulebook of one sparse conv: nbr[k, o] = input row or -1."""

    def __init__(self, outids, nbr, n_in, n_out, kernel_volume, site_state=None):
        self.outids, self.nbr = outids, nbr
        self.n_in, self.n_out, self.kernel_volume = n_in, n_out, kernel_volume
        self._pairs = None
        # strided convs keep (workspace, batch, out_shape): the site bitmap + ranks of their OUTPUT
        # grid are exactly what a SubM rulebook over those outputs needs
        self.site_state = site_state

    def pairs(self):
        """(indice_pairs [K, 2, n_in] int32 (-1 padded), indice_pair_num [K] int32): the
        reference layout (spconv_ops.h:53-57)."""
        if self._pairs is None:
            dev = self.nbr.device
            with torch.cuda.device(dev):
                pairs = torch.empty((self.kernel_volume, 2, self.n_in), dtype=torch.int32, device=dev)
                num = torch.empty((self.kernel_volume,), dtype=torch.int32, device=dev)
                rc = _C.lib().bevb200_rulebook_to_pairs(_C.ptr(self.nbr), self.kernel_volume,
                                                        self.n_out, self.n_in, _C.ptr(pairs),
                                                        _C.ptr(num), _C.current_stream(dev))
            _C.check(rc, "rulebook_to_pairs")
            self._pairs = (pairs, num)
        return self._pairs


def _listify(v, ndim):
    return list(v) if isinstance(v, (list, tuple)) else [v] * ndim


def get_rulebook(indices, batch_size, spatial_shape, ksize=3, stride=1, padding=0, dilation=1,
                 out_padding=0, subm=False, transpose=False):
    """Build the rulebook of one conv on the device (replaces getIndicePair<3>,
    spconv_ops.h:27-141).  One host sync for strided convs (the number of outputs)."""
    _C.require_cuda(indices, "indices", torch.int32)
    ndim = indices.shape[1] - 1
    if ndim != 3:
        raise NotImplementedError("only 3-D sparse convolution is implemented")
    if transpose:
        raise NotImplementedError("transposed sparse convolution is outside the hot path")
    ksize, stride, padding = _listify(ksize, 3), _listify(stride, 3), _listify(padding, 3)
    dilation = _listify(dilation, 3)
    for d, s in zip(dilation, stride):
        assert any([s == 1, d == 1]), "don't support this."
    spatial_shape = [int(v) for v in spatial_shape]
    if subm:
        out_shape = spatial_shape
    else:
        out_shape = get_conv_output_size(spatial_shape, ksize, stride, padding, dilation)
    batch_size = int(batch_size)
    n_in = indices.shape[0]
    kvol = ksize[0] * ksize[1] * ksize[2]
    dev = indices.device
    L = _C.lib()
    hs, ho, hk, hst, hp, hd = (_i32(spatial_shape), _i32(out_shape), _i32(ksize), _i32(stride),
                               _i32(padding), _i32(dilation))
    if subm:
        # (workspace, batch, out_shape, ready event) left on the tensor by the strided conv that made it
        st = getattr(indices, "_b200_site_state", None)
        if st is not None and st[1] == batch_size and st[2] == spatial_shape and n_in > 0:
            if st[3] is not None:          # built on another stream: order this stream after it
                torch.cuda.current_stream(dev).wait_event(st[3])
            # rows are the outputs of a strided conv built moments ago: reuse its bitmap + ranks
            with torch.cuda.device(dev):
                nbr = torch.empty((kvol, n_in), dtype=torch.int32, device=dev)
                rc = L.bevb200_rulebook_fill_subm_sorted(_C.ptr(indices), n_in, batch_size, _vp(hs), _vp(hk),
                                                         _vp(hd), _C.ptr(nbr), _C.ptr(st[0]), st[0].numel(),
                                                         _C.current_stream(dev))
            _C.check(rc, "rulebook_fill_subm_sorted")
            return Rulebook(indices, nbr, n_in, n_in, kvol), out_shape
    with torch.cuda.device(dev):
        stream = _C.current_stream(dev)
        ws = torch.empty(max(L.bevb200_rulebook_workspace_bytes(n_in, batch_size, _vp(ho)), 256),
                         dtype=torch.uint8, device=dev)
        n_out_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        rc = L.bevb200_rulebook_prepare(_C.ptr(indices), n_in, batch_size, _vp(hs), _vp(ho), _vp(hk),
                                        _vp(hst), _vp(hp), _vp(hd), int(bool(subm)),
                                        _C.ptr(n_out_dev), _C.ptr(ws), ws.numel(), stream)
        _C.check(rc, "rulebook_prepare")
        if subm:
            n_out, outids = n_in, indices
        else:
            n_out = int(n_out_dev.item())
            outids = torch.empty((n_out, 4), dtype=torch.int32, device=dev)
        nbr = torch.empty((kvol, n_out), dtype=torch.int32, device=dev)
        rc = L.bevb200_rulebook_fill(_C.ptr(indices), n_in, batch_size, _vp(hs), _vp(ho), _vp(hk),
                                     _vp(hst), _vp(hp), _vp(hd), int(bool(subm)), n_out,
                                     _C.ptr(outids), _C.ptr(nbr), _C.ptr(ws), ws.numel(), stream)
        _C.check(rc, "rulebook_fill")
    rb = Rulebook(outids, nbr, n_in, n_out, kvol)
    if not subm and n_out > 0:
        # the output-site bitmap + ranks live exactly as long as `outids` does: they ride on the tensor
        # object (no module-level cache), with the event a consumer on another stream must wait for
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream(dev))
        outids._b200_site_state = (ws, batch_size, list(out_shape), ready)
    return rb, out_shape


def get_indice_pairs(indices, batch_size, spatial_shape, ksize=3, stride=1, padding=0, dilation=1,
                     out_padding=0, subm=False, transpose=False, grid=None):
    """Drop-in for ops.get_indice_pairs (ops.py:45-125): returns
    (outids [M, 4], indice_pairs [K, 2, N], indice_pair_num [K])."""
    rb, _ = get_rulebook(indices, batch_size, spatial_shape, ksize, stride, padding, dilation,
                         out_padding, subm, transpose)
    pairs, num = rb.pairs()
    return rb.outids, pairs, num


def nbr_from_pairs(indice_pairs, indice_pair_num, num_activate_out, inverse=False):
    _C.require_cuda(indice_pairs, "indice_pairs", torch.int32)
    _C.require_cuda(indice_pair_num, "indice_pair_num", torch.int32)
    kvol, _, pdim = indice_pairs.shape
    dev = indice_pairs.device
    with torch.cuda.device(dev):
        nbr = torch.empty((kvol, int(num_activate_out)), dtype=torch.int32, device=dev)
        rc = _C.lib().bevb200_pairs_to_nbr(_C.ptr(indice_pairs), _C.ptr(indice_pair_num), kvol, pdim,
                                           int(num_activate_out), int(bool(inverse)), _C.ptr(nbr),
                                           _C.current_stream(dev))
    _C.check(rc, "pairs_to_nbr")
    return nbr


def pack_weights(weight, precision=None):
    """Pre-pack conv weights [k..., Cin, Cout] for the tensor-core kernel (None when the shape /
    precision has no tensor-core form).  Do this once for static weights."""
    _C.require_cuda(weight, "weight", torch.float32)
    if precision is None:
        precision = default_precision()
    c_in, c_out = weight.shape[-2], weight.shape[-1]
    kvol = weight.numel() // (c_in * c_out)
    nbytes = _C.lib().bevb200_spconv_packed_weight_bytes(c_in, c_out, kvol, int(precision))
    if nbytes == 0:
        return None
    dev = weight.device
    with torch.cuda.device(dev):
        packed = torch.empty(nbytes // 4, dtype=torch.float32, device=dev)
        rc = _C.lib().bevb200_spconv_pack_weights(_C.ptr(weight), c_in, c_out, kvol, int(precision),
                                                  _C.ptr(packed), _C.current_stream(dev))
    _C.check(rc, "spconv_pack_weights")
    return packed


def sparse_conv(features, weight, nbr, n_out, scale=None, shift=None, residual=None, relu=False,
                precision=None, packed=None):
    """out[o] = epilogue(sum_k features[nbr[k, o]] @ weight[k]) -- one implicit-GEMM launch.
    `packed` = pack_weights(weight, precision) skips the per-call weight packing."""
    _C.require_cuda(features, "features", torch.float32)
    _C.require_cuda(weight, "weight", torch.float32)
    _C.require_cuda(nbr, "nbr", torch.int32)
    n_in, c_in = features.shape
    c_out = weight.shape[-1]
    kvol = nbr.shape[0]
    assert weight.numel() == kvol * c_in * c_out, "weight must be [k..., Cin, Cout]"
    assert nbr.shape[1] == n_out
    for t, name in ((scale, "scale"), (shift, "shift")):
        if t is not None:
            _C.require_cuda(t, name, torch.float32)
            assert t.numel() == c_out
    if residual is not None:
        _C.require_cuda(residual, "residual", torch.float32)
        assert tuple(residual.shape) == (n_out, c_out)
    if precision is None:
        precision = default_precision()
    dev = features.device
    with torch.cuda.device(dev):
        out = torch.empty((n_out, c_out), dtype=torch.float32, device=dev)
        if packed is not None and precision != PREC_FP32:
            # narrow inputs (conv_input: 5 channels) run zero-padded; pad here with the caching
            # allocator instead of letting the library take a stream-ordered temporary per call
            c_pad = _C.lib().bevb200_spconv_padded_channels(c_in, int(precision))
            if c_pad != c_in:
                features = torch.nn.functional.pad(features, (0, c_pad - c_in))
                c_in = c_pad
            rc = _C.lib().bevb200_spconv_forward_packed(
                _C.ptr(features), _C.ptr(packed), _C.ptr(nbr), n_in, int(n_out), c_in, c_out, kvol,
                _C.ptr(scale), _C.ptr(shift), _C.ptr(residual), int(bool(relu)), int(precision),
                _C.ptr(out), _C.current_stream(dev))
        else:
            rc = _C.lib().bevb200_spconv_forward(
                _C.ptr(features), _C.ptr(weight), _C.ptr(nbr), n_in, int(n_out), c_in, c_out, kvol,
                _C.ptr(scale), _C.ptr(shift), _C.ptr(residual), int(bool(relu)), int(precision),
                _C.ptr(out), _C.current_stream(dev))
    _C.check(rc, "spconv_forward")
    return out


def indice_conv(features, filters, indice_pairs, indice_pair_num, num_activate_out, inverse=False,
                subm=False, precision=None, bias=None):
    """Drop-in for ops.indice_conv (ops.py:128-152).  `indice_pairs` may be the reference
    [K, 2, N] tensor (converted to a neighbour table first) or a Rulebook.  `bias` [Cout] is added
    in the conv epilogue (fused_indice_conv, ops.py:155-174)."""
    if filters.dtype not in (torch.float32, torch.half):
        raise NotImplementedError("filters must be fp32 or fp16")
    if isinstance(indice_pairs, Rulebook):
        assert not inverse
        nbr = indice_pairs.nbr
    else:
        nbr = nbr_from_pairs(indice_pairs, indice_pair_num, num_activate_out, inverse)
    if filters.dtype == torch.half or features.dtype == torch.half:
        # indice_conv_half (ops.py:141-150): the reference runs HGEMMs; here half tensors are
        # widened, the conv accumulates in fp32 on the tensor cores, and the result is narrowed
        # once -- at least as accurate as the reference's fp16 path
        out = sparse_conv(features.float().contiguous(), filters.float().contiguous(), nbr,
                          int(num_activate_out), shift=None if bias is None else bias.float().contiguous(),
                          precision=precision)
        return out.half()
    return sparse_conv(features.contiguous(), filters.contiguous(), nbr, int(num_activate_out),
                       shift=None if bias is None else bias.contiguous(), precision=precision)


def fused_indice_conv(features, filters, bias, indice_pairs, indice_pair_num, num_activate_out, inverse,
                      subm, precision=None):
    """Drop-in for ops.fused_indice_conv (ops.py:155-174; fusedIndiceConvBatchNorm,
    fused_spconv_ops.h:28-131): the output starts from the bias instead of zero."""
    return indice_conv(features, filters, indice_pairs, indice_pair_num, num_activate_out, bool(inverse),
                       bool(subm), precision=precision, bias=bias)


def transpose_nbr(nbr, n_in):
    """nbr [K, n_out] -> nbr_t [K, n_in]: nbr_t[k, j] = output row fed by input row j through k."""
    _C.require_cuda(nbr, "nbr", torch.int32)
    kvol, n_out = nbr.shape
    dev = nbr.device
    with torch.cuda.device(dev):
        nbr_t = torch.empty((kvol, int(n_in)), dtype=torch.int32, device=dev)
        rc = _C.lib().bevb200_rulebook_transpose(_C.ptr(nbr), kvol, n_out, int(n_in), _C.ptr(nbr_t),
                                                 _C.current_stream(dev))
    _C.check(rc, "rulebook_transpose")
    return nbr_t


def sparse_conv_backward(features, weight, out_grad, nbr, nbr_t=None, precision=None):
    """(input_grad [n_in, Cin], weight_grad like `weight`) of out = sparse_conv(features, weight, nbr)."""
    _C.require_cuda(features, "features", torch.float32)
    _C.require_cuda(weight, "weight", torch.float32)
    _C.require_cuda(out_grad, "out_grad", torch.float32)
    n_in, c_in = features.shape
    c_out = weight.shape[-1]
    kvol, n_out = nbr.shape
    assert tuple(out_grad.shape) == (n_out, c_out)
    if nbr_t is None:
        nbr_t = transpose_nbr(nbr, n_in)
    if precision is None:
        precision = default_precision()
    dev = features.device
    L = _C.lib()
    with torch.cuda.device(dev):
        din = torch.empty((n_in, c_in), dtype=torch.float32, device=dev)
        dw = torch.empty_like(weight)
        ws = torch.empty(max(L.bevb200_spconv_backward_workspace_bytes(int(n_in), int(n_out), c_in, c_out, kvol), 256),
                         dtype=torch.uint8, device=dev)
        rc = L.bevb200_spconv_backward(_C.ptr(features), _C.ptr(weight), _C.ptr(out_grad), _C.ptr(nbr),
                                       _C.ptr(nbr_t), n_in, n_out, c_in, c_out, kvol, int(precision),
                                       _C.ptr(din), _C.ptr(dw), _C.ptr(ws), ws.numel(),
                                       _C.current_stream(dev))
    _C.check(rc, "spconv_backward")
    return din, dw


def indice_conv_backward(features, filters, out_bp, indice_pairs, indice_pair_num, inverse=False,
                         subm=False, precision=None):
    """Drop-in for ops.indice_conv_backward (ops.py:177-189): returns [input_grad, filters_grad].
    `indice_pairs` may be the reference [K, 2, N] tensor or a Rulebook."""
    if torch.half in (filters.dtype, features.dtype, out_bp.dtype):
        # indice_conv_backward_half (ops.py:183-186): widened, computed with fp32 accumulation, narrowed
        # once -- each gradient to the dtype of the tensor it belongs to, so fp32 weights next to half
        # features get an fp32 filter gradient (no fp16 rounding, no overflow the weights cannot have)
        din, dw = indice_conv_backward(features.float(), filters.float(), out_bp.float(), indice_pairs,
                                       indice_pair_num, inverse, subm, precision)
        return [din.to(features.dtype), dw.to(filters.dtype)]
    if filters.dtype != torch.float32:
        raise NotImplementedError("filters must be fp32 or fp16")
    if isinstance(indice_pairs, Rulebook):
        assert not inverse
        nbr = indice_pairs.nbr
    else:
        nbr = nbr_from_pairs(indice_pairs, indice_pair_num, out_bp.shape[0], inverse)
    din, dw = sparse_conv_backward(features.contiguous(), filters.contiguous(), out_bp.contiguous(), nbr,
                                   precision=precision)
    return [din, dw]


class _SparseConvExt:
    """Stand-in for the reference pybind module `sparse_conv_ext` (src/all.cc)."""

    @staticmethod
    def get_indice_pairs_3d(indices, batch_size, out_shape, spatial_shape, ksize, stride, padding,
                            dilation, out_padding, subm, transpose):
        outids, pairs, num = get_indice_pairs(indices, batch_size, spatial_shape, ksize, stride,
                                              padding, dilation, out_padding, bool(subm),
                                              bool(transpose))
        return [outids, pairs, num]

    @staticmethod
    def indice_conv_fp32(features, filters, indice_pairs, indice_pair_num, num_activate_out,
                         inverse, subm):
        return indice_conv(features, filters, indice_pairs, indice_pair_num, num_activate_out,
                           bool(inverse), bool(subm))

    @staticmethod
    def indice_conv_half(features, filters, indice_pairs, indice_pair_num, num_activate_out,
                         inverse, subm):
        return indice_conv(features, filters, indice_pairs, indice_pair_num, num_activate_out,
                           bool(inverse), bool(subm))

    @staticmethod
    def indice_conv_backward_fp32(features, filters, out_bp, indice_pairs, indice_pair_num, inverse, subm):
        return indice_conv_backward(features, filters, out_bp, indice_pairs, indice_pair_num,
                                    bool(inverse), bool(subm))

    indice_conv_backward_half = indice_conv_backward_fp32      # half tensors are widened by the callee

    @staticmethod
    def fused_indice_conv_fp32(features, filters, bias, indice_pairs, indice_pair_num, num_activate_out,
                               inverse, subm):
        return fused_indice_conv(features, filters, bias, indice_pairs, indice_pair_num, num_activate_out,
                                 inverse, subm)

    fused_indice_conv_half = fused_indice_conv_fp32

    def __getattr__(self, name):
        # 2-D / 4-D rulebooks, grid rulebooks, sparse max-pool: not used by any shipped config.
        # AttributeError (not NotImplementedError) so that hasattr() / copy / pickle probing works.
        raise AttributeError("sparse_conv_ext.%s is outside the hot path (not implemented)" % name)


sparse_conv_ext = _SparseConvExt()


def _batch_stride_of(out, shape):
    """`out` must be a [B, C, ...] view that is dense inside each batch item (a channel slice
    of a wider channels-first buffer qualifies); returns its batch stride in elements."""
    if tuple(out.shape) != tuple(shape) or out.dtype != torch.float32:
        raise ValueError(f"out must be float32 of shape {tuple(shape)}")
    inner = 1
    for size, stride in zip(reversed(out.shape[1:]), reversed(out.stride()[1:])):
        if size != 1 and stride != inner:
            raise ValueError("out must be contiguous inside each batch item")
        inner *= size
    return int(out.stride(0)) if out.shape[0] > 1 else inner


def sparse_to_dense(features, indices, batch_size, spatial_shape, z_major=False, out=None):
    """dense() of a sparse tensor, channels first (structure.py:49-59); z_major=True gives the
    SparseEncoder output layout [B, C*Z, X, Y] directly (sparse_encoder.py:126-130).  `out`
    may be a channel slice of the fuser's concatenated input (fusers/conv.py:16)."""
    _C.require_cuda(features, "features", torch.float32)
    _C.require_cuda(indices, "indices", torch.int32)
    n, c = features.shape
    X, Y, Z = (int(v) for v in spatial_shape)
    dev = features.device
    with torch.cuda.device(dev):
        shape = (batch_size, c * Z, X, Y) if z_major else (batch_size, c, X, Y, Z)
        if out is None:
            out = torch.empty(shape, dtype=torch.float32, device=dev)
        stride = _batch_stride_of(out, shape)
        rc = _C.lib().bevb200_sparse_to_dense(_C.ptr(features), _C.ptr(indices), n, c, int(batch_size),
                                              _vp(_i32([X, Y, Z])), int(bool(z_major)), stride,
                                              _C.ptr(out), _C.current_stream(dev))
    _C.check(rc, "sparse_to_dense")
    return out
