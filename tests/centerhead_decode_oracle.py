"""Restatements of the CenterHead box decode (core/bbox/coders/centerpoint_bbox_coders.py:62-225 and
models/heads/bbox/centerpoint.py:637-757) for the tests and the benchmark.

    decode(maps, cfg)                     numpy, from the activated maps (numpy's exp is not CUDA's, so the caller
                                          supplies the sigmoid and the sizes): the padded rows and the mask
    torch_decode(maps, cfg, stable=True)  the coder's lines on torch tensors of any device, its two top-k stages as
                                          stable descending sorts (stable=False: torch.topk, as the reference)
    torch_get_bboxes(preds_dicts, cfg, test_cfg, num_classes, norm_bbox, nms)
                                          get_bboxes: activation, torch_decode, the NMS step `nms` (centerhead_nms)
                                          and the merge

maps: dict(heatmap [B, cat, H, W] scores, height, dim (sizes), rot [B, 2, H, W], optionally reg and vel); cfg: the
coder's fields.  decode and torch_decode return dict(boxes [B, K, code], scores [B, K], labels [B, K] float32,
index [B, K], mask [B, K] bool): all K selected rows in descending score (NaN first, ties by ascending flat index)
and which of them survive the masks.  compact() turns that into the device layout (survivors first, zeros after).
"""
import numpy as np
import torch


def _f32(v):
    return np.float32(v)


def decode(maps, cfg):
    heat = maps["heatmap"]
    B, cat, H, W = heat.shape
    K = int(cfg["max_num"])
    flat = heat.reshape(B, -1)
    idx = np.arange(flat.shape[1])
    top = np.empty((B, K), np.int64)
    for b in range(B):
        v = flat[b].astype(np.float64)
        nan = np.isnan(v)
        top[b] = np.lexsort((idx, -np.where(nan, 0.0, v), ~nan))[:K]   # NaN first, value descending, index ascending
    labels, ind = top // (H * W), top % (H * W)
    scores = np.take_along_axis(flat, top, 1)

    def at(m):                                                         # [B, C, H, W] -> [B, K, C] at ind
        return np.take_along_axis(m.reshape(B, m.shape[1], H * W), ind[:, None, :], 2).transpose(0, 2, 1)

    xs, ys = (ind // W).astype(np.float32), (ind % W).astype(np.float32)   # the reference's xs is the row
    if maps.get("reg") is not None:
        reg = at(maps["reg"])
        xs, ys = xs + reg[..., 0], ys + reg[..., 1]
    else:
        xs, ys = xs + _f32(0.5), ys + _f32(0.5)
    osf, vs, pc = _f32(cfg["out_size_factor"]), cfg["voxel_size"], cfg["pc_range"]
    with np.errstate(all="ignore"):
        xs = xs * osf * _f32(vs[0]) + _f32(pc[0])
        ys = ys * osf * _f32(vs[1]) + _f32(pc[1])
        rot = at(maps["rot"])
        cols = [xs[..., None], ys[..., None], at(maps["height"]), at(maps["dim"]),
                np.arctan2(rot[..., 0:1], rot[..., 1:2])]
        if maps.get("vel") is not None:
            cols.append(at(maps["vel"]))
        boxes = np.concatenate(cols, 2).astype(np.float32)
        rng = np.asarray(cfg["post_center_range"], np.float32)
        mask = (boxes[..., :3] >= rng[:3]).all(2) & (boxes[..., :3] <= rng[3:]).all(2)
        if cfg.get("score_threshold"):
            mask &= scores > _f32(cfg["score_threshold"])
    return dict(boxes=boxes, scores=scores, labels=labels.astype(np.float32), index=ind, mask=mask)


def _gather(feat, ind):
    """[B, C, H, W] at cells ind [B, K] -> [B, K, C] (the coder's _transpose_and_gather_feat)."""
    B, C = feat.shape[:2]
    return feat.reshape(B, C, -1).gather(2, ind[:, None, :].expand(-1, C, -1)).permute(0, 2, 1)


def torch_decode(maps, cfg, stable=True):
    heat = maps["heatmap"]
    B, cat, H, W = heat.shape
    K = int(cfg["max_num"])

    def topk(x):
        if not stable:
            return torch.topk(x, K)
        v, i = x.sort(dim=-1, descending=True, stable=True)
        return v[..., :K], i[..., :K]

    # The reference divides by torch.tensor(width) and torch.tensor(K), CPU scalars.  On CUDA torch turns a division
    # by a CPU scalar into a multiplication by its fp32 reciprocal, and trunc(n * fl(1 / d)) is n // d - 1 for some
    # multiples n of d (d = 83: n = 83, 166, 332, ...; none for d = 500 or the shipped widths), which moves the best
    # cell of a class to the class before it.  The divisors live on the tensors' device here, so the quotient is the
    # IEEE one on every device, as on the CPU: trunc of it is n // d for n < 2^24.
    Wf, Kf = (torch.tensor(v, dtype=torch.float, device=heat.device) for v in (W, K))
    s1, i1 = topk(heat.view(B, cat, -1))                               # per class; i1 is the cell
    xs1 = (i1.float() / Wf).int().float()
    ys1 = (i1 % W).int().float()
    scores, i2 = topk(s1.reshape(B, -1))
    clses = (i2 / Kf).int()
    ind = i1.reshape(B, -1).gather(1, i2)
    xs, ys = xs1.reshape(B, -1).gather(1, i2)[..., None], ys1.reshape(B, -1).gather(1, i2)[..., None]
    if maps.get("reg") is not None:
        reg = _gather(maps["reg"], ind)
        xs, ys = xs + reg[:, :, 0:1], ys + reg[:, :, 1:2]
    else:
        xs, ys = xs + 0.5, ys + 0.5
    rot = _gather(maps["rot"], ind)
    rot = torch.atan2(rot[..., 0:1], rot[..., 1:2])
    xs = xs * cfg["out_size_factor"] * cfg["voxel_size"][0] + cfg["pc_range"][0]
    ys = ys * cfg["out_size_factor"] * cfg["voxel_size"][1] + cfg["pc_range"][1]
    cols = [xs, ys, _gather(maps["height"], ind), _gather(maps["dim"], ind), rot]
    if maps.get("vel") is not None:
        cols.append(_gather(maps["vel"], ind))
    boxes = torch.cat(cols, dim=2)
    rng = torch.tensor(cfg["post_center_range"], device=heat.device)
    mask = (boxes[..., :3] >= rng[:3]).all(2) & (boxes[..., :3] <= rng[3:]).all(2)
    if cfg.get("score_threshold"):
        mask = mask & (scores > cfg["score_threshold"])
    return dict(boxes=boxes, scores=scores, labels=clses.float(), index=ind, mask=mask)


def compact(d):
    """The device layout of a decode: (boxes, scores, labels, index, counts), survivors first, zeros after."""
    xp_torch = isinstance(d["mask"], torch.Tensor)
    m = d["mask"] if xp_torch else torch.from_numpy(d["mask"])
    slot = torch.argsort((~m).to(torch.int8), dim=1, stable=True)
    counts = m.sum(1)
    pad = torch.arange(m.shape[1], device=m.device)[None, :] >= counts[:, None]
    out = []
    for k in ("boxes", "scores", "labels", "index"):
        v = d[k] if xp_torch else torch.from_numpy(d[k])
        s = slot[..., None].expand(-1, -1, v.shape[2]) if v.dim() == 3 else slot
        v = v.gather(1, s).masked_fill(pad[..., None] if v.dim() == 3 else pad, 0)
        out.append(v if xp_torch else v.numpy())
    return out + [counts.int() if xp_torch else counts.int().numpy()]


def decode_lists(d):
    """The coder's return: per sample dict(bboxes, scores, labels) of the surviving rows."""
    return [dict(bboxes=d["boxes"][i][d["mask"][i]], scores=d["scores"][i][d["mask"][i]],
                 labels=d["labels"][i][d["mask"][i]]) for i in range(d["mask"].shape[0])]


def torch_get_bboxes(preds_dicts, cfg, test_cfg, num_classes, norm_bbox, nms):
    """get_bboxes (centerpoint.py:637-757) with `nms(decoded, task_id, nms_type, test_cfg, nms_scale, num_classes)`
    as its NMS step: per sample [bboxes, scores, labels int32]."""
    T = len(preds_dicts)
    types = test_cfg["nms_type"] if isinstance(test_cfg["nms_type"], list) else [test_cfg["nms_type"]] * T
    if "nms_scale" in test_cfg:
        scales = test_cfg["nms_scale"]
        if not isinstance(scales, list):
            scales = [[scales] * num_classes[t] for t in range(T)]
    else:
        scales = [[1.0] * num_classes[t] for t in range(T)]
    rets = []
    for t, preds in enumerate(preds_dicts):
        p = preds[0]
        maps = dict(heatmap=p["heatmap"].sigmoid(), reg=p.get("reg"), height=p["height"],
                    dim=torch.exp(p["dim"]) if norm_bbox else p["dim"], rot=p["rot"], vel=p.get("vel"))
        rets.append(nms(decode_lists(torch_decode(maps, cfg)), t, types[t], test_cfg, scales[t], num_classes[t]))
    out = []
    for i in range(len(rets[0])):
        bboxes = torch.cat([r[i]["bboxes"] for r in rets])
        bboxes[:, 2] = bboxes[:, 2] - bboxes[:, 5] * 0.5
        flag, labels = 0, []
        for t in range(T):
            labels.append((rets[t][i]["labels"] + flag).int())
            flag += num_classes[t]
        out.append([bboxes, torch.cat([r[i]["scores"] for r in rets]), torch.cat(labels)])
    return out
