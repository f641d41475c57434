"""float64 oracle of one SparseEncoder training step: rulebooks from the CPU oracle, convs as gather / matmul /
index_add_, BatchNorm1d in train mode written out (biased batch variance for the normalisation, the running
statistics updated with the unbiased one), ReLU masks supplied by the run under test, dense() as index_put."""
import numpy as np
import torch

import oracle


def bn_train(x, weight, bias, running_mean, running_var, eps, momentum):
    """torch.nn.BatchNorm1d(x) in train mode on [n, c] rows; updates running_mean / running_var in place."""
    n = x.shape[0]
    mean = x.mean(0)
    var = ((x - mean) ** 2).mean(0)
    y = (x - mean) / torch.sqrt(var + eps) * weight + bias
    with torch.no_grad():
        running_mean.mul_(1 - momentum).add_(momentum * mean.detach())
        running_var.mul_(1 - momentum).add_(momentum * var.detach() * n / (n - 1))
    return y


def twin_forward(chain, feats, coors, batch_size, sparse_shape, masks, bn_params, bn_buffers, train=True):
    """The encoder `chain` (EncoderPlan.chain of the float64 twin: (conv, bn, relu, residual_from) per conv) on
    float64 `feats`.  masks[i] (bool [rows, c_out]) is the ReLU mask of conv i (None: relu itself);
    bn_params[i] = (weight, bias), bn_buffers[i] = (running_mean, running_var, num_batches_tracked), updated in
    place in train mode; train=False normalises with the running statistics.  Returns [B, C*Z, X, Y]."""
    dev = feats.device
    books = {}

    def conv(mod, f, idx, shape):
        key = (id(idx), tuple(mod.kernel_size), tuple(mod.stride), tuple(mod.padding), mod.subm)
        if key not in books:
            outids, pairs, num, oshape = oracle.get_indice_pairs(idx, batch_size, shape, mod.kernel_size, mod.stride,
                                                                 mod.padding, mod.dilation, mod.subm)
            inv = np.arange(outids.shape[0])
            if not mod.subm:      # strided outputs in ascending flat-index order, the order of the native plan
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

    idx, shape = coors.cpu().numpy(), list(sparse_shape)
    outs = []
    f = feats
    for i, (cv, bn, relu, res) in enumerate(chain):
        z, idx, shape = conv(cv, f, idx, shape)
        g, b = bn_params[i]
        rm, rv, nbt = bn_buffers[i]
        if train:
            y = bn_train(z, g, b, rm, rv, bn.eps, bn.momentum)
            nbt += 1
        else:
            y = (z - rm) / torch.sqrt(rv + bn.eps) * g + b
        if res >= 0:
            y = y + outs[res]
        if relu:
            y = y.clamp_min(0) if masks is None else y * masks[i][:y.shape[0]]
        outs.append(y)
        f = y
    li = torch.from_numpy(idx).long().to(dev)
    dense = f.new_zeros(batch_size, *shape, f.shape[1]).index_put((li[:, 0], li[:, 1], li[:, 2], li[:, 3]), f)
    dense = dense.permute(0, 4, 3, 1, 2)                                   # [B, C, Z, X, Y]
    N, C, D, H, W = dense.shape
    return dense.reshape(N, C * D, H, W)


def rel(got, want):
    """(relative L2, max-abs / max) of got against the float64 want."""
    d = (got.double() - want.double()).flatten()
    want = want.double()
    return float(d.norm() / want.norm().clamp_min(1e-300)), float(d.abs().max() / want.abs().max().clamp_min(1e-300))
