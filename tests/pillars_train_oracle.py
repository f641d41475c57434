"""Float64 numpy restatement of one PointPillars training step (mmdet3d/models/backbones/pillar_encoder.py:43-258
with BatchNorm1d in train mode): the forward with batch statistics over all M * P slots and an explicit backward,
written from the formulas of DESIGN 4.22 (no autograd).

Padded slots collapse to two row kinds: slot n (kind A) and the P - n - 1 rows after it (kind B, one row of
weight P - n - 1).  Every sum over slots is a weighted sum over the kept rows; maxes take the lowest slot that
attains them (torch's rule), so a max gradient on padding lands on kind A.  Pillars are processed in blocks,
pass by pass like the kernels, so a full-size batch needs no [M, P, 64] array."""
import numpy as np

BLOCK = 4096


def _decorate(x, n, c, geom):
    vx, vy, xo, yo = geom
    p = x.shape[1]
    mean = x[:, :, :3].sum(axis=1, keepdims=True) / n.reshape(-1, 1, 1)
    h = np.concatenate([x, x[:, :, :3] - mean, (x[:, :, 0] - (c[:, 1:2] * vx + xo))[..., None],
                        (x[:, :, 1] - (c[:, 2:3] * vy + yo))[..., None]], axis=2)
    return h * (np.arange(p)[None, :] < n[:, None])[..., None]


def _weights(n, p):
    """row weights [M, P]: 1 for real rows and kind A, P - n - 1 for kind B (slot n + 1), 0 for the rest"""
    cnt = np.minimum(n, p)[:, None]
    s = np.arange(p)[None, :]
    return np.where(s <= cnt, 1.0, 0.0) + np.where(s == cnt + 1, p - cnt - 1.0, 0.0)


def _first_argmax(v):
    return v.argmax(axis=1)  # numpy returns the first index attaining the max


def inside_canvas(coors, canvas_shape):
    """[M] bool: the pillar's (b, x, y) lies on the canvas.  Pillars off it count in both BNs but write nothing
    and take no gradient."""
    c = np.asarray(coors, np.int64)
    B, _, nx, ny = canvas_shape
    return (c[:, 0] >= 0) & (c[:, 0] < B) & (c[:, 1] >= 0) & (c[:, 1] < nx) & (c[:, 2] >= 0) & (c[:, 2] < ny)


def train_step(features, num_voxels, coors, params, geom, canvas_shape, grad_canvas, eps=1e-3, momentum=0.01):
    """features [M, P, F], num_voxels [M], coors [M, 4] (b, x, y, z); params: W1 [32, F+5], W2 [64, 64], g1, b1,
    g2, b2, rm1, rv1, rm2, rv2 (running statistics); geom (vx, vy, x_offset, y_offset); grad_canvas [B, 64, nx, ny].
    Returns a dict: canvas, dW1, dW2, dg1, db1, dg2, db2, rm1, rv1, rm2, rv2 (updated), and the batch statistics
    mu1, var1, mu2, var2."""
    x = np.asarray(features, np.float64)
    num = np.asarray(num_voxels, np.int64)
    c = np.asarray(coors, np.int64)
    m, p, _ = x.shape
    W1, W2 = (np.asarray(params[k], np.float64) for k in ("W1", "W2"))
    g1, b1, g2, b2 = (np.asarray(params[k], np.float64) for k in ("g1", "b1", "g2", "b2"))
    W2a, W2b = W2[:, :32], W2[:, 32:]
    gc = np.asarray(grad_canvas, np.float64)
    ins = inside_canvas(c, canvas_shape)
    N = float(m * p)
    blocks = [(i, min(i + BLOCK, m)) for i in range(0, m, BLOCK)]

    def rows(i0, i1):
        h = _decorate(x[i0:i1], num[i0:i1].astype(np.float64), c[i0:i1].astype(np.float64), geom)
        return h, _weights(num[i0:i1], p)[..., None]

    def stats(s, ss):
        mu = s / N
        var = ss / N - mu * mu
        return mu, var, 1.0 / np.sqrt(var + eps)

    # P1: layer-1 statistics
    s = np.zeros(32); ss = np.zeros(32)
    for i0, i1 in blocks:
        h, w = rows(i0, i1)
        z1 = h @ W1.T
        s += (w * z1).sum(axis=(0, 1)); ss += (w * z1 * z1).sum(axis=(0, 1))
    mu1, var1, inv1 = stats(s, ss)

    def layer1(h):
        z1 = h @ W1.T
        pre1 = (z1 - mu1) * inv1 * g1 + b1
        y1 = np.maximum(pre1, 0.0)
        return z1, pre1, y1, y1.max(axis=1), _first_argmax(y1)

    def layer2(y1, m1):
        return y1 @ W2a.T + (m1 @ W2b.T)[:, None, :]

    # P2: layer-2 statistics
    s = np.zeros(64); ss = np.zeros(64)
    for i0, i1 in blocks:
        h, w = rows(i0, i1)
        _, _, y1, m1, _ = layer1(h)
        z2 = layer2(y1, m1)
        s += (w * z2).sum(axis=(0, 1)); ss += (w * z2 * z2).sum(axis=(0, 1))
    mu2, var2, inv2 = stats(s, ss)

    def layer2_full(h):
        z1, pre1, y1, m1, am1 = layer1(h)
        z2 = layer2(y1, m1)
        pre2 = (z2 - mu2) * inv2 * g2 + b2
        y2 = np.maximum(pre2, 0.0)
        return z1, pre1, y1, m1, am1, z2, pre2, y2, _first_argmax(y2)

    def take(a, idx):  # a[v, idx[v, ch], ch]
        return np.take_along_axis(a, idx[:, None, :], axis=1)[:, 0, :]

    def g2_of(i0, i1, pre2, am2):
        cc, k = c[i0:i1], ins[i0:i1]
        G = np.zeros((i1 - i0, gc.shape[1]))
        G[k] = gc[cc[k, 0], :, cc[k, 1], cc[k, 2]]
        g2 = np.zeros_like(pre2)
        np.put_along_axis(g2, am2[:, None, :], G[:, None, :], axis=1)
        return g2 * (pre2 > 0)

    # P3: the canvas; B1: BN-2 backward sums
    canvas = np.zeros(canvas_shape)
    sg2 = np.zeros(64); sgx2 = np.zeros(64)
    for i0, i1 in blocks:
        h, w = rows(i0, i1)
        *_, z2, pre2, y2, am2 = layer2_full(h)
        cc, k = c[i0:i1], ins[i0:i1]
        canvas[cc[k, 0], :, cc[k, 1], cc[k, 2]] = y2.max(axis=1)[k]
        gg2 = g2_of(i0, i1, pre2, am2)
        xh2 = (z2 - mu2) * inv2
        sg2 += (w * gg2).sum(axis=(0, 1)); sgx2 += (w * gg2 * xh2).sum(axis=(0, 1))

    def back1(i0, i1):
        h, w = rows(i0, i1)
        z1, pre1, y1, m1, am1, z2, pre2, y2, am2 = layer2_full(h)
        xh2 = (z2 - mu2) * inv2
        dz2 = g2 * inv2 * (g2_of(i0, i1, pre2, am2) - sg2 / N - xh2 * sgx2 / N)
        D = (w * dz2).sum(axis=1)
        dy1 = dz2 @ W2a
        dm1 = D @ W2b
        np.put_along_axis(dy1, am1[:, None, :], take(dy1, am1)[:, None, :] + dm1[:, None, :], axis=1)
        g1_ = dy1 * (pre1 > 0)
        xh1 = (z1 - mu1) * inv1
        return h, w, y1, m1, dz2, D, g1_, xh1

    # B2: dW2, BN-1 backward sums
    dW2 = np.zeros((64, 64))
    sg1 = np.zeros(32); sgx1 = np.zeros(32)
    for i0, i1 in blocks:
        h, w, y1, m1, dz2, D, gg1, xh1 = back1(i0, i1)
        dW2[:, :32] += np.einsum("vso,vsk->ok", w * dz2, y1)
        dW2[:, 32:] += np.einsum("vo,vk->ok", D, m1)
        sg1 += (w * gg1).sum(axis=(0, 1)); sgx1 += (w * gg1 * xh1).sum(axis=(0, 1))

    # B3: dW1 (padded rows have a zero input row)
    dW1 = np.zeros_like(W1)
    for i0, i1 in blocks:
        h, w, _, _, _, _, gg1, xh1 = back1(i0, i1)
        dz1 = g1 * inv1 * (gg1 - sg1 / N - xh1 * sgx1 / N)
        dW1 += np.einsum("vsc,vsj->cj", dz1, h)

    out = dict(canvas=canvas, dW1=dW1, dW2=dW2, dg1=sgx1, db1=sg1, dg2=sgx2, db2=sg2, mu1=mu1, var1=var1, mu2=mu2,
               var2=var2)
    for k, mu, var in (("1", mu1, var1), ("2", mu2, var2)):
        out["rm" + k] = (1 - momentum) * np.asarray(params["rm" + k], np.float64) + momentum * mu
        out["rv" + k] = (1 - momentum) * np.asarray(params["rv" + k], np.float64) + momentum * var * N / (N - 1)
    return out


def params_from_state_dict(sd, prefix=""):
    """oracle params from a PillarFeatureNet state_dict (numpy values)"""
    k = prefix + "pfn_layers.%d."
    return dict(W1=sd[k % 0 + "linear.weight"], W2=sd[k % 1 + "linear.weight"],
                g1=sd[k % 0 + "norm.weight"], b1=sd[k % 0 + "norm.bias"],
                g2=sd[k % 1 + "norm.weight"], b2=sd[k % 1 + "norm.bias"],
                rm1=sd[k % 0 + "norm.running_mean"], rv1=sd[k % 0 + "norm.running_var"],
                rm2=sd[k % 1 + "norm.running_mean"], rv2=sd[k % 1 + "norm.running_var"])


def slot_values(features, num_voxels, coors, params, geom, out, eps=1e-3):
    """Per-slot values of a step whose batch statistics train_step returned in `out`: decorated rows h [M, P, F+5]
    (zero past n), BN-normalised pre-activations pre1 [M, P, 32] and pre2 [M, P, 64], y1 and the layer-1 max m1."""
    x = np.asarray(features, np.float64)
    num = np.asarray(num_voxels, np.int64)
    h = _decorate(x, num.astype(np.float64), np.asarray(coors, np.float64), geom)
    W1, W2 = (np.asarray(params[k], np.float64) for k in ("W1", "W2"))
    g1, b1, g2, b2 = (np.asarray(params[k], np.float64) for k in ("g1", "b1", "g2", "b2"))
    pre1 = (h @ W1.T - out["mu1"]) / np.sqrt(out["var1"] + eps) * g1 + b1
    y1 = np.maximum(pre1, 0.0)
    m1 = y1.max(axis=1)
    z2 = y1 @ W2[:, :32].T + (m1 @ W2[:, 32:].T)[:, None, :]
    pre2 = (z2 - out["mu2"]) / np.sqrt(out["var2"] + eps) * g2 + b2
    return h, pre1, y1, m1, pre2
