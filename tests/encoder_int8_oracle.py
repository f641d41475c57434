"""numpy restatement of the INT8 encoder plan's numerical contract (include/bevfusion_b200.h, DESIGN.md 4.25).

Every fp32 op of the contract is one numpy float32 op here (numpy rounds each to nearest and never contracts), the
integer products are summed exactly in int64 over the rulebooks of rulebook_oracle, so the chain is reproduced bit
for bit wherever conv 0's fp32 sums are exact:

    s_w[c] = fl(max |W[.., .., c]| / 127) (1 if 0),  q_w = clamp(rint(fl(W / s_w)), -127, 127)
    conv 0:  acc = sum fp16(x) fp16(w) (fp32), a = bn_scale
    conv i:  acc = sum u8 q_w (int32),         a = fl(fl(s_{i-1} s_w) bn_scale)
    v = fl(fl(float(acc) a) + shift) [ v = fl(v + fl(float(res_u8) s_res)) ],  v = max(v, 0)
    u8 = clamp(rint(fl(v r_i)), 0, 255) (NaN -> 0),  last conv: half(v)

Conv 0's fp32 sum is computed in float64.  It equals the device's fp32 sum when the terms are exact in fp32 on a
common grid (the exact-chain tests).  Otherwise the device sum lies within ERR of the float64 one, and a row is
TAINTED when some channel's output differs between the two ends of that interval (every step is monotone in acc, so
the ends decide); taint follows the rulebooks and the residuals to dense().

run_chain(..., stats=[]) appends one dict per conv of what its contract's edges saw (STAT_KEYS), so an edge case can
show that it reaches its edge; the results do not depend on it."""
import numpy as np
import torch

from encoder_fp16_oracle import dense64, rulebooks

F32 = np.float32
U32 = 2.0 ** -24
HALF_MAX = 65504.0

# per conv: cells with fl(v r) > 255 (+inf included), of them +inf from a finite v, NaN cells zeroed (v before the
# ReLU and fl(v r)), fl(v r) in [0, 255] with fraction .5, fl(W / s_w) with fraction .5, all-zero weight columns,
# max |acc|, accumulators past 2^24 and those float32(acc) != acc, the last conv's finite v that half() rounds to
# 65504 and to inf, cells the conv writes as fp16, max v after the ReLU, output rows, and the output scale used
STAT_KEYS = ("sat", "overflow", "nan", "ties", "w_ties", "w_zero_cols", "acc_max", "acc_past_2_24", "acc_inexact",
             "half_max", "half_inf", "f16_out", "vmax", "rows", "s_act")


def quant_weight(w):
    """(s_w [c_out] float32, q_w [K, c_in, c_out] int64) of the fp32 weight w [K, c_in, c_out]"""
    w = np.asarray(w, np.float32)
    m = np.abs(w).reshape(-1, w.shape[-1]).max(0)
    s = np.where(m > 0, m / F32(127), F32(1)).astype(np.float32)
    q = np.clip(np.rint((w / s).astype(np.float32)), -127, 127).astype(np.int64)
    return s, q


def relu(v):
    """max(v, 0) with NaN -> 0, as fmaxf"""
    return np.where(v > 0, v, F32(0)).astype(np.float32)


def quant_u8(v, r):
    """clamp(rint(fl(v r)), 0, 255): +inf -> 255, NaN -> 0"""
    t = (np.asarray(v, np.float32) * F32(r)).astype(np.float32)
    t = np.where(np.isnan(t), F32(0), t)
    return np.rint(np.clip(t, 0, 255)).astype(np.int64)


def _gather_sum(x, q, pl, n_out):
    """sum_k x[in] @ q[k] scattered to the output rows, in float64.  u8 x s8 sums are integers below 27 * 128 *
    255 * 127 < 2^27, so every partial sum is exact and the order does not matter."""
    x, q = np.asarray(x, np.float64), np.asarray(q, np.float64)
    acc = np.zeros((n_out, q.shape[-1]), np.float64)
    for k, (i, o) in enumerate(pl):
        if i.numel():
            np.add.at(acc, o.numpy(), x[i.numpy()] @ q[k])
    return acc


def _taint_rows(taint_in, pl, n_out):
    t = np.zeros(n_out, bool)
    for i, o in pl:
        if i.numel():
            t[o.numpy()[taint_in[i.numpy()]]] = True
    return t


def _frac_half(t):
    return int((np.isfinite(t) & (t - np.floor(t) == 0.5)).sum())


def _conv_stats(v_pre, t, acc, w_stats, last, n_out, c_out):
    """one conv's STAT_KEYS entry (t = fl(v r) of an u8 image, None for the last conv)"""
    st = dict(w_stats, nan=int(np.isnan(v_pre).sum()), rows=n_out, f16_out=n_out * c_out if last else 0,
              vmax=float(np.nanmax(np.where(v_pre > 0, v_pre, 0))) if v_pre.size else 0.0)
    a = np.abs(np.asarray(acc, np.float64))
    finite = a[np.isfinite(a)]
    st["acc_max"] = float(finite.max()) if finite.size else 0.0
    st["acc_past_2_24"] = int((a > 2.0 ** 24).sum())
    st["acc_inexact"] = int((np.isfinite(a) & (a.astype(np.float32).astype(np.float64) != a)).sum())
    v = np.where(v_pre > 0, v_pre, F32(0)).astype(np.float32)
    if last:
        h = v.astype(np.float16)
        st.update(sat=0, overflow=0, ties=0, half_max=int((h == HALF_MAX).sum()),
                  half_inf=int((np.isfinite(v) & np.isinf(h)).sum()))
    else:
        st.update(sat=int((t > 255).sum()), overflow=int((np.isfinite(v) & np.isposinf(t)).sum()),
                  ties=_frac_half(np.where((t >= 0) & (t <= 255), t, F32(0))), half_max=0, half_inf=0)
        st["nan"] += int(np.isnan(t).sum())
    return st


def run_chain(*args, **kw):
    with np.errstate(over="ignore", invalid="ignore"):       # inf and NaN are part of the contract
        return _run_chain(*args, **kw)


def _run_chain(convs, feats16, coors, batch_size, shape, weights, scales, shifts, s_act, exact=False, stats=None):
    """The INT8 chain of the conv dicts `convs` (cin, cout, subm, res, relu, ks, stride, pad) on fp16 features
    feats16 [n, cin] (numpy float16) at coors (numpy (b, x, y, z)).  weights[i] fp32 [K, cin, cout]; scales[i] /
    shifts[i] float32 [cout] or None; s_act[i] the output scale of conv i.  Returns (dense [B, C*Z, X, Y] float64
    tensor of the last conv's half(v), tainted-cell mask of the same shape (all False when exact), tainted fraction
    of the last level's rows).  An s_act[i] of None is chosen here as chain_scales would, from this chain's own v:
    fl(max v_i / 255), 1 when that is 0 (no fp16 rounding of the max).  stats: a list that gets one dict per conv
    (STAT_KEYS), including the s_act used."""
    rbs = rulebooks(convs, coors, batch_size, shape)
    s_act = list(s_act)
    x0 = feats16.astype(np.float64)
    outs, taints = [], []
    x_u8, x_taint = None, np.zeros(x0.shape[0], bool)
    last = len(convs) - 1
    for i, (c, (oidx, pl, oshape)) in enumerate(zip(convs, rbs)):
        n_out = oidx.shape[0]
        sc = np.ones(c["cout"], np.float32) if scales[i] is None else np.asarray(scales[i], np.float32)
        sh = np.zeros(c["cout"], np.float32) if shifts[i] is None else np.asarray(shifts[i], np.float32)
        if i == 0:
            w16 = np.asarray(weights[0], np.float32).astype(np.float16).astype(np.float64)
            z = _gather_sum(x0, w16.reshape(-1, c["cin"], c["cout"]), pl, n_out)
            za = _gather_sum(np.abs(x0), np.abs(w16).reshape(-1, c["cin"], c["cout"]), pl, n_out)
            a = sc
            exact_sum = z
            if exact:
                accs = [z.astype(np.float32)]
            else:
                # fp32 sum of n terms, any order: |error| <= n u32 sum |x w| (gamma_n), doubled for safety
                n_terms = int(np.prod(c["ks"])) * c["cin"]
                err = 2 * n_terms * U32 * za
                accs = [z.astype(np.float32), (z - err).astype(np.float32), (z + err).astype(np.float32)]
            taint = np.zeros(n_out, bool)
            w_stats = dict(w_ties=0, w_zero_cols=0)
        else:
            w32 = np.asarray(weights[i], np.float32).reshape(-1, c["cin"], c["cout"])
            s_w, q = quant_weight(w32)
            w_stats = dict(w_ties=_frac_half(np.abs((w32 / s_w).astype(np.float32))),
                           w_zero_cols=int((np.abs(w32).reshape(-1, c["cout"]).max(0) == 0).sum()))
            a = ((F32(s_act[i - 1]) * s_w).astype(np.float32) * sc).astype(np.float32)
            exact_sum = _gather_sum(x_u8, q, pl, n_out)
            accs = [exact_sum.astype(np.float32)]
            taint = _taint_rows(x_taint, pl, n_out)
        ys = []
        for j, acc in enumerate(accs):
            v = ((acc * a).astype(np.float32) + sh).astype(np.float32)
            if c["res"] >= 0:
                r_u8, r_taint, s_res = outs[c["res"]][0], taints[c["res"]], F32(s_act[c["res"]])
                v = (v + (r_u8.astype(np.float32) * s_res).astype(np.float32)).astype(np.float32)
            assert c["relu"], "the INT8 plan needs a ReLU after every conv"
            v_pre, v = v, relu(v)
            if j == 0 and s_act[i] is None:
                m = F32(v.max()) if v.size else F32(0)
                s_act[i] = float(m / F32(255)) if m > 0 else 1.0
            r = F32(1) / F32(s_act[i])
            ys.append(v.astype(np.float16) if i == last else quant_u8(v, r))
            if j == 0 and stats is not None:
                t = None if i == last else (v * r).astype(np.float32)
                st = _conv_stats(v_pre, t, exact_sum, w_stats, i == last, n_out, c["cout"])
                stats.append(dict(st, s_act=s_act[i]))
        if len(ys) == 3:
            taint |= (ys[1] != ys[2]).any(1)
        if c["res"] >= 0:
            taint |= taints[c["res"]]
        outs.append((ys[0], None))
        taints.append(taint)
        x_u8, x_taint = ys[0], taint
    oidx, _, oshape = rbs[-1]
    dense = dense64(torch.from_numpy(outs[-1][0].astype(np.float64)), oidx, batch_size, oshape)
    tmask = dense64(torch.from_numpy(np.repeat(taints[-1][:, None], convs[-1]["cout"], 1).astype(np.float64)), oidx,
                    batch_size, oshape) != 0
    return dense, tmask, float(taints[-1].mean()) if taints[-1].size else 0.0


def chain_scales(convs, feats16, coors, batch_size, shape, weights, scales, shifts):
    """Per-conv output scales consistent with the oracle's own chain: s_i = fl(max v_i / 255) of the float32 v the
    oracle computes with the scales chosen so far (1 when that max is 0).  Any positive scales give an exact chain;
    these keep the u8 images in range."""
    s_act = []
    for i in range(len(convs)):
        sub = convs[:i + 1]
        last = dict(sub[-1])
        probe = [dict(c) for c in sub[:-1]] + [last]
        # the v of conv i is the half(v) the oracle writes for its last conv; its max is rounded to fp16, which only
        # moves the scale, not the exactness
        d, _, _ = run_chain(probe, feats16, coors, batch_size, shape, weights[:i + 1], scales[:i + 1],
                            shifts[:i + 1], s_act + [1.0], exact=True)
        m = F32(float(d.max()))
        s_act.append(float(m / F32(255)) if m > 0 else 1.0)
    return s_act
