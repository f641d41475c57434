"""Float64 oracle of the SparseEncoder's fp16 precision (BEVB200_PREC_FP16) and its error bounds, in the style of
half_oracle: a device result passes when

    |got - ref| <= ulp16(ref) + c * absref

with ref the float64 value of the same formula on the same fp16 inputs, ulp16 the fp16 spacing at |ref| (one
rounding to nearest is half of it; the other half covers a result that crosses into the next binade) and absref the
same formula on absolute values.  The constants, with u = 2^-24 the unit roundoff of fp32:

  * C_ACC(n) = n * u, the conv before its one fp16 rounding.  Both operands are fp16, so every product
    (11 + 11 significant bits) is exact in fp32; what is left is the fp32 accumulation of n = kvol * c_in_eff terms,
    at most n * u * sum |terms| = n * u * absref to first order, whatever the order of the sums.
  * C_BN = 16 * u, the training apply y16 = fp16(relu(gamma (z16 - mean) invstd + beta [+ res16])).  The kernel
    forms it in fp32 as z16 * scale + shift [+ res16] from scale = gamma invstd and shift = beta - mean scale, each
    rounded once from double, then one multiply and two adds: at most 5 u of absref = |scale z16| + |shift| +
    |res16| (not of |y|: where a level's rows sit close to their mean, or a level has one row, scale z16 and shift
    nearly cancel); 16 u leaves room to spare.
  * C_EVAL(depth) = depth * 2^-10 for the eval forward of a whole chain against a twin that rounds at the same
    points: the twin's intermediate fp16 values may differ from the device's by one rounding where the device's
    fp32 sum lands on the other side of a tie, which a later conv carries forward as at most one fp16 ulp
    (2^-10 relative, 2^-11 each side) of each input; each conv adds at most one such term of its absref.
  * Backward, as a relative L2 norm per gradient tensor (the form of the BF16x3 training tests): the twin runs
    through exactly the saved z16 / y16 values with the run's ReLU masks, so the device differs from it only by its
    one fp16 rounding of dz per conv (<= 2^-11 relative per element) and fp32 sums.  A rounding at conv i reaches
    every gradient upstream of it, each relative error at most 2^-11 of the element it perturbs, so a gradient of
    conv j (dW, dgamma, dbeta) carries at most the n_convs - j roundings downstream of it: the bound is
    C_DZ * n_convs with C_DZ = 2^-11.  The features' gradient is returned as fp16, one rounding more:
    C_DZ * (n_convs + 1).  A per-element ulp + c * absref form is not used here: dgamma, dbeta and the rows of dz are
    sums whose BN-backward terms (g - mean(g) - x^ mean(g x^)) cancel by construction, so an absolute-value twin
    bounds nothing useful.
"""
import numpy as np
import torch

from encoder_train_oracle import raw_rulebook
from half_oracle import FP16_INF_FROM, check, ulp

U32 = 2.0 ** -24
C_BN = 16 * U32
C_DZ = 2.0 ** -11


def c_acc(n_terms):
    return n_terms * U32


def c_eval(depth):
    return depth * 2.0 ** -10


def fp16_round(x):
    """float64 -> the nearest fp16 value (ties to even), as float64: subnormals down to 2^-24, |x| >= 65520 -> inf
    with the sign of x, NaN kept.  Written without torch.half so the CPU tests can check it against torch.half."""
    x = x.double()
    sp = ulp(x, torch.float16)
    r = torch.round(x / sp) * sp                      # torch.round rounds half to even
    r = torch.where(x.abs() >= FP16_INF_FROM, torch.copysign(torch.full_like(x, float("inf")), x), r)
    return torch.where(torch.isnan(x), x, r)


def bwd_bounds(n_convs):
    """(bound of the conv and BN gradients, bound of the features' gradient), relative L2"""
    return C_DZ * n_convs, C_DZ * (n_convs + 1)


def check_train_forward(convs, x16, weights, bns, saved, before, after, rbs, what):
    """The training forward conv by conv from the saved state (see the module docstring).  x16: the fp16 features
    (float64, valid rows); weights[i] [K, c_in, c_out] (the fp32 values the call packed); bns[i] = (gamma, beta, eps,
    momentum); saved[i] = (z16, y16) float64 over the level's valid rows; before / after[i] = (running_mean,
    running_var) around the call.  A level with fewer than 2 rows normalises with what it has and leaves the
    running statistics alone.  Returns the worst ratio of each check."""
    worst = {"z16": 0.0, "y16": 0.0, "running": 0.0}
    x = x16
    for i, (c, (oidx, pl, _)) in enumerate(zip(convs, rbs)):
        z16, y16 = saved[i]
        assert z16.shape[0] == oidx.shape[0], (what, i, z16.shape, oidx.shape)
        w = fp16_round(weights[i].detach().double().cpu().reshape(-1, c["cin"], c["cout"]))
        ref, absref = conv64(x, w, pl, oidx.shape[0])
        kvol = c["ks"][0] * c["ks"][1] * c["ks"][2]
        cin_eff = max(16, 1 << (c["cin"] - 1).bit_length())
        worst["z16"] = max(worst["z16"], check(z16.half(), ref, absref, "%s: z16 of conv %d" % (what, i),
                                               c_acc(kvol * cin_eff)))
        gamma, beta, eps, mo = bns[i]
        n = z16.shape[0]
        mean, var = z16.mean(0), z16.var(0, unbiased=False)
        if n >= 2:
            for got, old, stat, unb in ((after[i][0], before[i][0], mean, 1.0),
                                        (after[i][1], before[i][1], var, n / (n - 1.0))):
                old = old.double().cpu()
                r = (1 - mo) * old + mo * stat * unb
                worst["running"] = max(worst["running"], check(
                    got.cpu(), r, (1 - mo) * old.abs() + mo * (stat * unb).abs(),
                    "%s: running statistics of conv %d" % (what, i), 8 * U32))
        else:
            assert torch.equal(after[i][0], before[i][0]) and torch.equal(after[i][1], before[i][1]), (what, i)
        # the kernel's form: z16 * scale + shift with scale = gamma invstd, shift = beta - mean scale; absref is that
        # form on absolute values (where the rows are close to their mean, |scale z16| and |shift| both far exceed
        # |y| and carry the fp32 rounding)
        scale = gamma.detach().double().cpu() / torch.sqrt(var + eps)
        shift = beta.detach().double().cpu() - mean * scale
        yr, ya = z16 * scale + shift, (z16 * scale).abs() + shift.abs()
        if c["res"] >= 0:
            yr, ya = yr + saved[c["res"]][1], ya + saved[c["res"]][1].abs()
        if c["relu"]:
            yr = yr.clamp_min(0)
        worst["y16"] = max(worst["y16"], check(y16.half(), yr, ya, "%s: y16 of conv %d" % (what, i), C_BN))
        x = y16
    return worst


def twin_backward(convs, rbs, x16, weights, bns, saved, R, B):
    """float64 gradients of sum(dense * R) -> (features, [dW], [dgamma], [dbeta]) through the saved z16 / y16
    values (each value the saved one, each derivative the float64 formula's: straight through) with the run's ReLU
    masks (y16 > 0 of the convs with a ReLU) and fp16(W)."""
    x0 = x16.detach().clone().requires_grad_(True)
    ws, gs, bs = [], [], []
    cur, outs = x0, []
    for i, (c, (oidx, pl, _)) in enumerate(zip(convs, rbs)):
        w = fp16_round(weights[i].detach().double().cpu().reshape(-1, c["cin"], c["cout"])).requires_grad_(True)
        gamma, beta, eps, _ = bns[i]
        gam = gamma.detach().double().cpu().requires_grad_(True)
        bet = beta.detach().double().cpu().requires_grad_(True)
        ws.append(w); gs.append(gam); bs.append(bet)
        z = cur.new_zeros(oidx.shape[0], c["cout"])
        for k, (a, o) in enumerate(pl):
            if a.numel():
                z = z.index_add(0, o, cur[a] @ w[k])
        z = saved[i][0] + (z - z.detach())
        mean = z.mean(0)
        var = ((z - mean) ** 2).mean(0)
        y = gam * (z - mean) / torch.sqrt(var + eps) + bet
        if c["res"] >= 0:
            y = y + outs[c["res"]]
        if c["relu"]:
            y = y * (saved[i][1] > 0)
        y = saved[i][1] + (y - y.detach())
        outs.append(y)
        cur = y
    (dense64(cur, rbs[-1][0], B, rbs[-1][2]) * R).sum().backward()
    return x0.grad, [w.grad for w in ws], [g.grad for g in gs], [b.grad for b in bs]


def module_convs(plan):
    """the C-ABI conv dicts of an EncoderPlan's chain (encoder_train_oracle.raw_rulebook's input)"""
    out = []
    for conv, _, relu, res in plan.chain:
        out.append(dict(cin=conv.in_channels, cout=conv.out_channels, subm=bool(conv.subm), res=res, relu=relu,
                        ks=list(conv.kernel_size),
                        stride=[1, 1, 1] if conv.subm else list(conv.stride),
                        pad=[k // 2 for k in conv.kernel_size] if conv.subm else list(conv.padding)))
    return out


def rulebooks(convs, coors, batch_size, shape):
    """[(output coordinates, pairs per offset, output shape)] of every conv, from the CPU oracle"""
    idx, shape, out = np.ascontiguousarray(coors), list(shape), []
    for c in convs:
        oidx, pl, oshape = raw_rulebook(idx, batch_size, shape, c)
        out.append((oidx, pl, oshape))
        idx, shape = oidx, oshape
    return out


def conv64(x, w, pl, n_out):
    """(sum_k x[in] @ w[k] scattered to the output rows, the same on |x|, |w|) in float64"""
    z = x.new_zeros(n_out, w.shape[-1])
    a = x.new_zeros(n_out, w.shape[-1])
    for k, (i, o) in enumerate(pl):
        if i.numel():
            z = z.index_add(0, o, x[i] @ w[k])
            a = a.index_add(0, o, x[i].abs() @ w[k].abs())
    return z, a


def dense64(rows, idx, batch_size, shape):
    """dense() + the encoder's z-major view of rows [n, C] at coordinates idx (numpy (b, x, y, z))"""
    li = torch.from_numpy(np.ascontiguousarray(idx)).long()
    d = rows.new_zeros(batch_size, *shape, rows.shape[1]).index_put((li[:, 0], li[:, 1], li[:, 2], li[:, 3]), rows)
    d = d.permute(0, 4, 3, 1, 2)
    N, C, D, H, W = d.shape
    return d.reshape(N, C * D, H, W)


def eval_twin(plan, feats, coors, batch_size, shape):
    """(dense output, absref) of the eval forward in float64, rounded to fp16 where the plan rounds: the features
    once, the weights once, and every conv's y = relu(acc * scale + shift [+ res]) once.  BN is folded as the plan
    folds it (bevfusion_b200.sparse_block.bn_scale_shift)."""
    from bevfusion_b200.sparse_block import bn_scale_shift
    convs = module_convs(plan)
    rbs = rulebooks(convs, coors, batch_size, shape)
    x = fp16_round(feats.double().cpu())
    xa = x.abs()
    outs, absouts = [], []
    for (conv, bn, relu, res), c, (oidx, pl, oshape) in zip(plan.chain, convs, rbs):
        w = fp16_round(conv.weight.detach().double().cpu().reshape(-1, c["cin"], c["cout"]))
        z, _ = conv64(x, w, pl, oidx.shape[0])
        za, _ = conv64(xa, w.abs(), pl, oidx.shape[0])
        s, t = bn_scale_shift(bn)
        s, t = s.double().cpu(), t.double().cpu()
        y, ya = z * s + t, za * s.abs() + t.abs()
        if res >= 0:
            y, ya = y + outs[res], ya + absouts[res]
        if relu:
            y = y.clamp_min(0)
        outs.append(fp16_round(y))
        absouts.append(ya)
        x, xa = outs[-1], ya
    return dense64(outs[-1], rbs[-1][0], batch_size, rbs[-1][2]), dense64(absouts[-1], rbs[-1][0], batch_size,
                                                                            rbs[-1][2])
