"""Float64 restatements of the sparse-conv forward and of an eval-mode SparseEncoder, for the GPU tests.

  * conv_nbr / epilogue: out[o] = relu(sum_k f[nbr[k, o]] @ W[k] * scale + shift + residual) straight from a
    neighbour table; entries outside [0, n_in) are missing neighbours, as in every forward kernel.
  * encoder_forward: SparseEncoder.forward of an eval-mode float64 copy of the module, with rulebooks from the CPU
    oracle (oracle.get_indice_pairs), convs as gather / matmul / index_add_, torch BatchNorm1d and dense() as
    index_put.  It also returns the mask of active output cells and the rows of every level."""
import numpy as np
import torch

import oracle


def conv_nbr(f, w, nbr):
    """sum_k f[nbr[k, o]] @ w[k] in float64 -> [n_out, Cout]; w is [k..., Cin, Cout]."""
    n_in = f.shape[0]
    kv, n_out = nbr.shape
    w64 = w.double().reshape(kv, -1, w.shape[-1])
    f64 = f.double()
    out = torch.zeros(n_out, w.shape[-1], dtype=torch.float64, device=f.device)
    for k in range(kv):
        m = (nbr[k] >= 0) & (nbr[k] < n_in)
        out[m] += f64[nbr[k][m].long()] @ w64[k]
    return out


def epilogue(acc, scale=None, shift=None, residual=None, relu=False):
    """acc * scale + shift + residual, then ReLU, in acc's dtype; None terms are left out."""
    y = acc
    if scale is not None:
        y = y * scale.to(acc.dtype)
    if shift is not None:
        y = y + shift.to(acc.dtype)
    if residual is not None:
        y = y + residual.to(acc.dtype)
    return y.clamp_min(0) if relu else y


def dense_zmajor(f, idx, batch_size, shape):
    """SparseEncoder's dense(): rows f at idx (b, x, y, z) -> [B, C*Z, X, Y], zero elsewhere."""
    li = idx.long().to(f.device)
    dense = f.new_zeros(batch_size, *shape, f.shape[1]).index_put((li[:, 0], li[:, 1], li[:, 2], li[:, 3]), f)
    dense = dense.permute(0, 4, 3, 1, 2)                                   # [B, C, Z, X, Y]
    N, C, D, H, W = dense.shape
    return dense.reshape(N, C * D, H, W)


def encoder_forward(m, feats, coors, batch_size):
    """SparseEncoder.forward of `m`, an eval-mode float64 copy of the module, on float64 `feats`.
    -> (dense [B, C*Z, X, Y], active-cell mask of the same shape, rows per level: [n, then one per strided conv])."""
    from bevfusion_b200.sparse_block import SparseBasicBlock
    assert not m.training
    dev = feats.device
    books = {}
    rows = [int(coors.shape[0])]

    def conv(mod, f, idx, shape):
        key = (id(idx), tuple(mod.kernel_size), tuple(mod.stride), tuple(mod.padding), mod.subm)
        if key not in books:
            outids, pairs, num, oshape = oracle.get_indice_pairs(idx, batch_size, shape, mod.kernel_size, mod.stride,
                                                                 mod.padding, mod.dilation, mod.subm)
            pl = [(torch.from_numpy(pairs[k, 0, :num[k]]).long().to(dev),
                   torch.from_numpy(pairs[k, 1, :num[k]]).long().to(dev)) for k in range(num.shape[0])]
            books[key] = (idx if mod.subm else outids, pl, list(oshape))
        oidx, pl, oshape = books[key]
        w = mod.weight.reshape(-1, mod.in_channels, mod.out_channels)
        out = f.new_zeros(oidx.shape[0], mod.out_channels)
        for k, (i, o) in enumerate(pl):
            if i.numel():
                out.index_add_(0, o, f[i] @ w[k])
        if mod.bias is not None:
            out = out + mod.bias
        if not mod.subm:
            rows.append(int(oidx.shape[0]))
        return out, oidx, oshape

    def seq(s, f, idx, shape):
        f, idx, shape = conv(s[0], f, idx, shape)
        return torch.relu(s[1](f)), idx, shape

    with torch.no_grad():
        idx, shape = coors.cpu().numpy(), list(m.sparse_shape)
        f, idx, shape = seq(m.conv_input, feats, idx, shape)
        for stage in m.encoder_layers:
            for block in stage:
                if isinstance(block, SparseBasicBlock):
                    o, _, _ = conv(block.conv1, f, idx, shape)
                    o = torch.relu(block.norm1(o))
                    o, _, _ = conv(block.conv2, o, idx, shape)
                    f = torch.relu(block.norm2(o) + f)
                else:
                    f, idx, shape = seq(block, f, idx, shape)
        f, idx, shape = seq(m.conv_out, f, idx, shape)
        idx = torch.from_numpy(np.ascontiguousarray(idx))
        dense = dense_zmajor(f, idx, batch_size, shape)
        active = dense_zmajor(torch.ones_like(f), idx, batch_size, shape) != 0
    return dense, active, rows
