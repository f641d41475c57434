"""float64 oracle of one SparseEncoder training step: rulebooks from the CPU oracle, convs as gather / matmul /
index_add_, BatchNorm1d in train mode written out (biased batch variance for the normalisation, the running
statistics updated with the unbiased one), ReLU masks supplied by the run under test, dense() as index_put.

twin_forward runs a module chain (EncoderPlan.chain); raw_train_forward runs a raw C-ABI conv list, with the native
rule for levels of fewer than 2 rows (bn_train_rows) and an optional wider output canvas."""
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


def bn_train_rows(x, weight, bias, running_mean, running_var, eps, momentum):
    """bn_train with the native rule for fewer than 2 rows, where torch's BatchNorm1d raises: normalise with the rows
    there are (one row: mean = x, variance 0; none: nothing) and leave the running statistics alone.
    -> (y, whether the running statistics moved)"""
    n = x.shape[0]
    if n >= 2:
        return bn_train(x, weight, bias, running_mean, running_var, eps, momentum), True
    if n == 0:
        return x, False
    mean = x.mean(0)
    return (x - mean) / torch.sqrt(((x - mean) ** 2).mean(0) + eps) * weight + bias, False


def raw_rulebook(idx, batch_size, shape, c):
    """(output coordinates, [(input rows, output rows)] per offset, output shape) of the conv dict c on the
    coordinates idx (numpy), from the CPU oracle; strided outputs in ascending flat-index order (the native plan's)"""
    outids, pairs, num, oshape = oracle.get_indice_pairs(idx, batch_size, shape, c["ks"], c["stride"], c["pad"],
                                                         [1, 1, 1], c["subm"])
    inv = np.arange(outids.shape[0])
    if not c["subm"]:
        order = np.argsort(oracle.flat_index(outids, oshape), kind="stable")
        inv[order] = np.arange(order.size)
        outids = outids[order]
    pl = [(torch.from_numpy(pairs[k, 0, :num[k]].astype(np.int64)), torch.from_numpy(inv[pairs[k, 1, :num[k]]]))
          for k in range(num.shape[0])]
    return (idx if c["subm"] else outids), pl, list(oshape)


def raw_train_forward(convs, feats, coors, batch_size, sparse_shape, weights, bn_params, bn_buffers, masks,
                      eps, momentum, out_batch_stride=0):
    """A training forward of the raw conv chain `convs` (the conv(...) dicts of the C-ABI tests: c_in, c_out, subm,
    res, relu, ks, stride, pad) in float64 on the CPU, one BatchNorm per conv:
        z_i = conv_i(y_{i-1}),  y_i = mask_i * (bn_train_rows(z_i) [+ y_res])     (mask_i only when relu)
    feats [n, c_in] are the valid rows, coors their (b, x, y, z); weights[i] [K, c_in, c_out]; bn_params[i] =
    (gamma, beta); bn_buffers[i] = [running_mean, running_var, num_batches_tracked] (updated in place, the count
    only when the statistics moved); masks[i] bool [rows, c_out] from the run under test.  Returns (dense output
    [B, C*Z, X, Y] -- or, with out_batch_stride > 0, a [B, out_batch_stride] canvas holding it in the first
    C*Z*X*Y floats of every sample, zero elsewhere -- and the rows per level)."""
    idx, shape = np.ascontiguousarray(coors), list(sparse_shape)
    rows, outs, f = [int(idx.shape[0])], [], feats
    for i, c in enumerate(convs):
        oidx, pl, oshape = raw_rulebook(idx, batch_size, shape, c)
        w = weights[i].reshape(-1, c["cin"], c["cout"])
        z = f.new_zeros(oidx.shape[0], c["cout"])
        for k, (a, o) in enumerate(pl):
            if a.numel():
                z = z.index_add(0, o, f[a] @ w[k])
        rm, rv, nbt = bn_buffers[i]
        y, moved = bn_train_rows(z, bn_params[i][0], bn_params[i][1], rm, rv, eps, momentum)
        if moved:
            bn_buffers[i][2] = nbt + 1
        if c["res"] >= 0:
            y = y + outs[c["res"]]
        if c["relu"]:
            y = y * masks[i][:y.shape[0]]
        outs.append(y)
        f = y
        if not c["subm"]:
            rows.append(int(oidx.shape[0]))
        idx, shape = oidx, oshape
    li = torch.from_numpy(np.ascontiguousarray(idx)).long()
    dense = f.new_zeros(batch_size, *shape, f.shape[1]).index_put((li[:, 0], li[:, 1], li[:, 2], li[:, 3]), f)
    dense = dense.permute(0, 4, 3, 1, 2)                                   # [B, C, Z, X, Y]
    N, C, D, H, W = dense.shape
    dense = dense.reshape(N, C * D, H, W)
    if out_batch_stride:
        per = C * D * H * W
        dense = torch.cat([dense.reshape(N, per), dense.new_zeros(N, out_batch_stride - per)], 1)
    return dense, rows


def rel(got, want):
    """(relative L2, max-abs / max) of got against the float64 want."""
    d = (got.double() - want.double()).flatten()
    want = want.double()
    return float(d.norm() / want.norm().clamp_min(1e-300)), float(d.abs().max() / want.abs().max().clamp_min(1e-300))
