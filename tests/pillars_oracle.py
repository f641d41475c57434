"""Float64 numpy restatement of the PointPillars pillar encoder (mmdet3d/models/backbones/
pillar_encoder.py:20-258): the checker for bevfusion_b200.pillar_encoder."""
import numpy as np


def pillar_feature_net(features, num_voxels, coors, layers, vx, vy, x_offset, y_offset, with_distance=False,
                       train=False, eps=1e-3):
    """features [M, P, F], num_voxels [M], coors [M, 4] (b, x, y, z).  layers: one dict per PFN layer
    with W [units, in], gamma, beta, mean, var (running statistics) and last (bool).  train=True
    normalises with the batch statistics over all M * P slots (padded ones included).
    Returns (out [M, C], [(batch_mean, batch_var_unbiased) per layer])."""
    x = np.asarray(features, np.float64)
    m, p, _ = x.shape
    n = np.asarray(num_voxels, np.float64)
    c = np.asarray(coors, np.float64)
    mean = x[:, :, :3].sum(axis=1, keepdims=True) / n.reshape(-1, 1, 1)
    cols = [x, x[:, :, :3] - mean,
            (x[:, :, 0] - (c[:, 1:2] * vx + x_offset))[..., None],
            (x[:, :, 1] - (c[:, 2:3] * vy + y_offset))[..., None]]
    if with_distance:
        cols.append(np.linalg.norm(x[:, :, :3], axis=2, keepdims=True))
    h = np.concatenate(cols, axis=2)
    h = h * (np.arange(p)[None, :] < np.asarray(num_voxels)[:, None])[..., None]
    stats = []
    for L in layers:
        y = h @ np.asarray(L["W"], np.float64).T
        if train:
            mu = y.reshape(-1, y.shape[2]).mean(axis=0)
            var = y.reshape(-1, y.shape[2]).var(axis=0)
            stats.append((mu, y.reshape(-1, y.shape[2]).var(axis=0, ddof=1)))
        else:
            mu, var = np.asarray(L["mean"], np.float64), np.asarray(L["var"], np.float64)
        y = (y - mu) / np.sqrt(var + eps) * np.asarray(L["gamma"], np.float64) + np.asarray(L["beta"], np.float64)
        y = np.maximum(y, 0.0)
        ymax = y.max(axis=1, keepdims=True)
        h = ymax if L["last"] else np.concatenate([y, np.repeat(ymax, p, axis=1)], axis=2)
    return h[:, 0, :], stats


def pillars_scatter(feats, coors, batch_size, nx, ny):
    """canvas [B, C, nx, ny]: canvas[b, :, x, y] = feats[v] (pillar_encoder.py:203-237)."""
    feats = np.asarray(feats, np.float64)
    out = np.zeros((batch_size, feats.shape[1], nx, ny))
    c = np.asarray(coors)
    out[c[:, 0], :, c[:, 1], c[:, 2]] = feats
    return out


def layers_from_state_dict(sd, prefix, n_layers):
    """oracle layer dicts from a PillarFeatureNet state_dict (numpy values)"""
    out = []
    for i in range(n_layers):
        k = "%spfn_layers.%d." % (prefix, i)
        out.append(dict(W=sd[k + "linear.weight"], gamma=sd[k + "norm.weight"], beta=sd[k + "norm.bias"],
                        mean=sd[k + "norm.running_mean"], var=sd[k + "norm.running_var"], last=i == n_layers - 1))
    return out
