"""numpy restatement of ImageAug3D's pixel path followed by ImageNormalize (transforms_3d.py:98-192, 992-1006):

    TF.normalize(TF.to_tensor(img.resize(dims).crop(box)[.transpose(FLIP_LEFT_RIGHT)].rotate(deg)), mean, std)

written out the way Pillow computes it, so that it equals Pillow + torchvision bit for bit:

- resize: Pillow's BICUBIC resample (a = -0.5, support 2 scaled by the reduction factor).  Coefficients in double
  in Pillow's order, normalised to 22-bit fixed point; a horizontal pass over the source rows the vertical filter
  reads, then a vertical pass, each rounding (+ 2^21, >> 22) and clipping to uint8.
- crop: pixels of the box outside the resized image are 0.
- rotate: Image.rotate(deg) with NEAREST, fill 0, no expand.  deg % 360 == 0 is a copy, 180 a 180-degree transpose,
  90 / 270 on a square image a transpose; otherwise the inverse matrix exactly as Image.rotate builds it (including
  round(cos, 15)), then Pillow's NEAREST affine: a[1] == a[3] == 0 takes the scaling path (per-axis double
  coordinates), everything else the 16.16 fixed-point path (every coordinate of a frame up to 16384 pixels is far
  inside its +-32768 range), whose integer sums equal the closed form a2 + y * a1 + x * a0 exactly.
- normalise: u8 / 255 in fp32, then (x - mean) / std in fp32.

Pure numpy and Python floats: no Pillow, so the GPU tests can use it on a machine without Pillow."""
import math

import numpy as np

PRECISION_BITS = 22


def bicubic(x):
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def coeffs(in_size, out_size):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for the full box (0, in_size): (bounds [out, 2] int,
    fixed-point coefficients [out, ksize] int64, ksize)."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int64)
    kk = np.zeros((out_size, ksize), np.int64)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [bicubic(((x + xmin) - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        for x, v in enumerate(w):
            k = v / ww if ww != 0.0 else v
            kk[xx, x] = int(-0.5 + k * (1 << PRECISION_BITS)) if k < 0 else int(0.5 + k * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return bounds, kk, ksize


def _clip8(ss):
    return np.clip(ss >> PRECISION_BITS, 0, 255).astype(np.uint8)


def _taps(bounds, kk, first, limit):
    """Per output index and tap: (source index - first, clipped to the array, and coefficient, 0 past the count)."""
    ksize = kk.shape[1]
    idx = np.minimum(bounds[:, :1] - first + np.arange(ksize)[None, :], limit - 1)
    return idx, np.where(np.arange(ksize)[None, :] < bounds[:, 1:], kk, 0)


def resample_rows(src, bounds, kk):
    """Horizontal pass of every row of src [R, W, 3] for the output columns of bounds / kk: uint8 [R, out, 3]."""
    idx, k = _taps(bounds, kk, 0, src.shape[1])
    ss = np.full((src.shape[0], bounds.shape[0], 3), 1 << (PRECISION_BITS - 1), np.int64)
    for t in range(kk.shape[1]):
        ss += src[:, idx[:, t], :].astype(np.int64) * k[None, :, t, None]
    return _clip8(ss)


def resample_cols(tmp, bounds, kk, first):
    """Vertical pass over tmp [R, w, 3] whose row 0 is source row `first`: uint8 [out, w, 3]."""
    idx, k = _taps(bounds, kk, first, tmp.shape[0])
    ss = np.full((bounds.shape[0], tmp.shape[1], 3), 1 << (PRECISION_BITS - 1), np.int64)
    for t in range(kk.shape[1]):
        ss += tmp[idx[:, t]].astype(np.int64) * k[:, t, None, None]
    return _clip8(ss)


def resize(img, dims, window=None):
    """Image.resize(dims) with the default BICUBIC on an RGB uint8 [H, W, 3] array -> [h, w, 3].  With window =
    (x0, y0, x1, y1) only those columns and rows of the result are computed (each output pixel depends on its own
    row and column alone, so they equal the full resize's)."""
    H, W, _ = img.shape
    w, h = dims
    x0, y0, x1, y1 = window if window is not None else (0, 0, w, h)
    if (w, h) == (W, H):
        return img[y0:y1, x0:x1].copy()
    hb, hk, _ = coeffs(W, w)
    vb, vk, _ = coeffs(H, h)
    hb, hk, vb, vk = hb[x0:x1], hk[x0:x1], vb[y0:y1], vk[y0:y1]
    first, last = int(vb[:, 0].min()), int((vb[:, 0] + vb[:, 1]).max())
    return resample_cols(resample_rows(img[first:last], hb, hk), vb, vk, first)


def crop(img, x0, y0, w, h):
    """Image.crop((x0, y0, x0 + w, y0 + h)): outside the image is 0."""
    out = np.zeros((h, w, 3), np.uint8)
    H, W, _ = img.shape
    ys, ye = max(y0, 0), min(y0 + h, H)
    xs, xe = max(x0, 0), min(x0 + w, W)
    if ys < ye and xs < xe:
        out[ys - y0:ye - y0, xs - x0:xe - x0] = img[ys:ye, xs:xe]
    return out


def rotate_rule(angle, w, h):
    """What Image.rotate(angle) of a w x h image does: ("copy" | "rot180" | "rot90" | "rot270", None) or
    ("scale" | "affine", the six inverse-matrix coefficients as Image.rotate computes them)."""
    angle = float(angle) % 360.0
    if angle == 0:
        return "copy", None
    if angle == 180:
        return "rot180", None
    if angle in (90, 270) and w == h:
        return ("rot90" if angle == 90 else "rot270"), None
    cx, cy = w / 2, h / 2
    t = -math.radians(angle)
    m = [round(math.cos(t), 15), round(math.sin(t), 15), 0.0, round(-math.sin(t), 15), round(math.cos(t), 15), 0.0]
    a, b, c, d, e, f = m
    m[2], m[5] = a * -cx + b * -cy + c, d * -cx + e * -cy + f
    m[2] += cx
    m[5] += cy
    return ("scale" if m[1] == 0 and m[3] == 0 else "affine"), m


def _coord(v):
    return np.where(v < 0.0, -1, np.trunc(np.maximum(v, 0.0))).astype(np.int64)


def _fix(v):
    return math.floor(v * 65536.0 + 0.5)


def rotate(img, angle):
    """Image.rotate(angle) (NEAREST, fill 0, no expand) of uint8 [h, w, 3]."""
    h, w, _ = img.shape
    kind, m = rotate_rule(angle, w, h)
    if kind == "copy":
        return img.copy()
    if kind == "rot180":
        return img[::-1, ::-1].copy()
    if kind == "rot90":
        return np.ascontiguousarray(img.transpose(1, 0, 2)[::-1])
    if kind == "rot270":
        return np.ascontiguousarray(img.transpose(1, 0, 2)[:, ::-1])
    y, x = np.mgrid[0:h, 0:w]
    if kind == "scale":
        # ImagingScaleAffine: xo = a2 + a0 / 2 advanced by a0 per column, yo = a5 + a4 / 2 by a4 per row; with
        # a1 == a3 == 0 the coefficients a0, a4 are +-1, so the running sums are exact and equal the closed form
        xo = m[2] + m[0] * 0.5
        yo = m[5] + m[4] * 0.5
        assert abs(m[0]) == 1.0 and abs(m[4]) == 1.0
        xin, yin = _coord(xo + x * m[0]), _coord(yo + y * m[4])
    else:
        a0, a1, a3, a4 = _fix(m[0]), _fix(m[1]), _fix(m[3]), _fix(m[4])
        a2 = _fix(m[2] + m[0] * 0.5 + m[1] * 0.5)
        a5 = _fix(m[5] + m[3] * 0.5 + m[4] * 0.5)
        xin = (a2 + y * a1 + x * a0) >> 16
        yin = (a5 + y * a4 + x * a3) >> 16
    ok = (xin >= 0) & (xin < w) & (yin >= 0) & (yin < h)
    out = np.zeros_like(img)
    out[ok] = img[yin[ok], xin[ok]]
    return out


def normalize(img, mean, std):
    """TF.normalize(TF.to_tensor(img), mean, std): uint8 [h, w, 3] -> fp32 [3, h, w]."""
    x = img.transpose(2, 0, 1).astype(np.float32) / np.float32(255)
    m = np.asarray(mean, np.float32)[:, None, None]
    s = np.asarray(std, np.float32)[:, None, None]
    return (x - m) / s


def augment_u8(img, resize_dims, crop_xy, final_dim, flip, rotate_deg):
    """resize, crop, flip and rotate of one uint8 [H, W, 3] image -> uint8 [fH, fW, 3]."""
    fH, fW = final_dim
    w, h = (int(v) for v in resize_dims)
    x0, y0 = int(crop_xy[0]), int(crop_xy[1])
    wx0, wy0 = min(max(x0, 0), w), min(max(y0, 0), h)
    wx1, wy1 = max(min(x0 + fW, w), wx0), max(min(y0 + fH, h), wy0)
    out = np.zeros((fH, fW, 3), np.uint8)
    if wx1 > wx0 and wy1 > wy0:
        out[wy0 - y0:wy1 - y0, wx0 - x0:wx1 - x0] = resize(img, (w, h), (wx0, wy0, wx1, wy1))
    if flip:
        out = out[:, ::-1].copy()
    return rotate(out, rotate_deg)


def augment(img, resize_dims, crop_xy, final_dim, flip, rotate_deg, mean, std):
    """The whole pixel path of one image: fp32 [3, fH, fW]."""
    return normalize(augment_u8(img, resize_dims, crop_xy, final_dim, flip, rotate_deg), mean, std)
