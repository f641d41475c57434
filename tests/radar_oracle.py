"""Float64 numpy restatement of the radar encoder (mmdet3d/models/backbones/radar_encoder.py:24-220):
the checker for bevfusion_b200.radar_encoder."""
import numpy as np


def radar_feature_net(features, num_voxels, coors, layers, vx, vy, x_offset, y_offset, pc_range, train=False,
                      eps=1e-3):
    """features [M, P, F], num_voxels [M], coors [M, 4] (b, x, y, z).  layers: one dict per RFN layer
    with W [units, in], gamma, beta, mean, var (running statistics).  train=True normalises with the
    batch statistics over all M * P slots (padded ones included).  The input is not modified.
    Returns (out [M, C], [(batch_mean, batch_var_unbiased) per layer])."""
    x = np.array(features, np.float64)
    m, p, _ = x.shape
    c = np.asarray(coors, np.float64)
    r = [float(v) for v in pc_range]
    f_center = np.stack([x[:, :, 0] - (c[:, 1:2] * vx + x_offset), x[:, :, 1] - (c[:, 2:3] * vy + y_offset)], 2)
    for k in range(3):
        x[:, :, k] = (x[:, :, k] - r[k]) / (r[k + 3] - r[k])
    h = np.concatenate([x, f_center], axis=2)
    mask = (np.arange(p)[None, :] < np.asarray(num_voxels)[:, None])[..., None]
    with np.errstate(invalid="ignore"):
        h = h * mask
    h = np.nan_to_num(h, nan=0.0, posinf=np.finfo(np.float32).max, neginf=-np.finfo(np.float32).max)
    stats = []
    for L in layers:
        y = h @ np.asarray(L["W"], np.float64).T
        flat = y.reshape(-1, y.shape[2])
        if train:
            mu, var = flat.mean(axis=0), flat.var(axis=0)
            stats.append((mu, flat.var(axis=0, ddof=1)))
        else:
            mu, var = np.asarray(L["mean"], np.float64), np.asarray(L["var"], np.float64)
        y = (y - mu) / np.sqrt(var + eps) * np.asarray(L["gamma"], np.float64) + np.asarray(L["beta"], np.float64)
        h = np.maximum(y, 0.0)
    return h.max(axis=1), stats


def radar_scatter(feats, coors, batch_size, nx, ny):
    """canvas [B, C, nx, ny]: canvas[b, :, x, y] = feats[v] (PointPillarsScatter)."""
    feats = np.asarray(feats, np.float64)
    out = np.zeros((batch_size, feats.shape[1], nx, ny))
    c = np.asarray(coors)
    out[c[:, 0], :, c[:, 1], c[:, 2]] = feats
    return out


def layers_from_state_dict(sd, prefix, n_layers):
    """oracle layer dicts from a RadarFeatureNet state_dict (numpy values)"""
    out = []
    for i in range(n_layers):
        k = "%srfn_layers.%d." % (prefix, i)
        out.append(dict(W=sd[k + "linear.weight"], gamma=sd[k + "norm.weight"], beta=sd[k + "norm.bias"],
                        mean=sd[k + "norm.running_mean"], var=sd[k + "norm.running_var"]))
    return out
