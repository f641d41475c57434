"""Pairs of rotated boxes in the geometric families where polygon clipping goes wrong, with their BEV overlap
and IoU in closed form (numpy only, no GPU):

    families(rng, n) -> {name: (A [n, 5], B [n, 5], overlap [n], iou [n])}   float64 [x1, y1, x2, y2, ry] boxes
    NAMES                                                                     the family names, in that order
    SIZES                                                                     the (x extent, y extent) drawn from

Every pair is built in box a's own frame and placed with the boxes' turning convention (nms_oracle.py): the point
p of a's frame lies at a's centre plus (px cos ra + py sin ra, -px sin ra + py cos ra), so a box b whose axes are
turned by phi (counter-clockwise) within a's frame has yaw ra - phi.  Yaws are fp32 values: most in [-pi, pi],
some beyond +-pi, some exactly fp32(+-pi / 2).  Centres lie within +-61 m.  The families:

    slide            same size and yaw (or yaw + pi), slid by t along a's x or y axis: IoU (s - t) / (s + t)
    touch_end        touching end to end along a's long axis, any sizes, offset across it: overlap 0
    touch_side       touching side by side along a's short axis: overlap 0
    touch_corner     touching corner to corner: overlap 0
    corner_on_edge   a corner of b on an edge of a, b outside a (overlap 0) or inside it (overlap sb)
    nested           b inside a, same yaw or yaw + pi, flush with one or two of a's edges: overlap sb
    yaw_pi           the same box turned by pi, slid along an axis (a quarter not slid)
    square_half_pi   a square and the same square turned by +-pi / 2, slid along an axis (a quarter not slid)
    yaw_ulp          the same box with its fp32 yaw one ulp up or down: the octagon of a rectangle turned about
                     its centre by the small angle
    zero_width       a box of zero width or length (sometimes both boxes) near or across another: overlap 0

Edges of the two boxes are collinear in all but the zero-width family, at yaws that are mostly not multiples of
pi / 2.  Sizes are the car-to-pedestrian SIZES, either way round, and 0.05 x 12 m slivers."""
import numpy as np

SIZES = [(0.3, 0.3), (0.6, 0.8), (0.8, 2.1), (1.95, 4.6), (2.5, 6.9), (2.9, 12.0), (0.05, 12.0)]
SPAN = 61.0
HALF_PI32 = float(np.float32(np.pi / 2))


def yaws(rng, n):
    r = rng.uniform(-np.pi, np.pi, n)
    k = rng.uniform(size=n)
    far = k < 0.15
    r[far] = rng.choice([-1.0, 1.0], far.sum()) * rng.uniform(np.pi, 3 * np.pi, far.sum())
    right = (k >= 0.15) & (k < 0.3)
    r[right] = rng.choice([-HALF_PI32, HALF_PI32], right.sum())
    return r.astype(np.float32).astype(np.float64)


def sizes(rng, n):
    s = np.array(SIZES, np.float64)[rng.integers(len(SIZES), size=n)]
    swap = rng.uniform(size=n) < 0.5
    s[swap] = s[swap, ::-1]
    return s[:, 0], s[:, 1]


def centres(rng, n):
    return rng.uniform(-SPAN, SPAN, n), rng.uniform(-SPAN, SPAN, n)


def xyxyr(cx, cy, w, l, r):
    return np.stack([cx - w / 2, cy - l / 2, cx + w / 2, cy + l / 2, r], 1)


def place(cx, cy, ra, px, py, phi, w, l):
    """Box b of extents (w, l) centred at (px, py) of a's frame, its axes turned by phi there."""
    c, s = np.cos(ra), np.sin(ra)
    return xyxyr(cx + px * c + py * s, cy - px * s + py * c, w, l, ra - phi)


def _rot(x, y, ang):
    c, s = np.cos(ang), np.sin(ang)
    return x * c - y * s, x * s + y * c


def _base(rng, n):
    cx, cy = centres(rng, n)
    w, l = sizes(rng, n)
    return cx, cy, w, l, yaws(rng, n)


def slide_offset(rng, n, w, l):
    """Offset (px, py) of t along x or y (a quarter of them 0) and the side s it slides along."""
    along_x = rng.uniform(size=n) < 0.5
    side = np.where(along_x, w, l)
    t = rng.uniform(0, 1, n) * side
    t[rng.uniform(size=n) < 0.25] = 0.0
    t *= rng.choice([-1.0, 1.0], n)
    return np.where(along_x, t, 0.0), np.where(along_x, 0.0, t), side, np.abs(t)


def _result(A, B, ov):
    sa = (A[:, 2] - A[:, 0]) * (A[:, 3] - A[:, 1])
    sb = (B[:, 2] - B[:, 0]) * (B[:, 3] - B[:, 1])
    return A, B, ov, ov / np.maximum(sa + sb - ov, 1e-8)


def slide(rng, n, phi_choices):
    cx, cy, w, l, ra = _base(rng, n)
    px, py, side, t = slide_offset(rng, n, w, l)
    phi = rng.choice(phi_choices, n)
    return _result(xyxyr(cx, cy, w, l, ra), place(cx, cy, ra, px, py, phi, w, l), (side - t) * (w * l / side))


def touch(rng, n, how):
    cx, cy, w, l, ra = _base(rng, n)
    wb, lb = sizes(rng, n)
    sx, sy = rng.choice([-1.0, 1.0], n), rng.choice([-1.0, 1.0], n)
    gx, gy = (w + wb) / 2, (l + lb) / 2                          # centre distances at which the boxes touch
    slide_x, slide_y = rng.uniform(-1, 1, n) * gx, rng.uniform(-1, 1, n) * gy
    long_x = w >= l
    if how == "end":
        px, py = np.where(long_x, sx * gx, slide_x), np.where(long_x, slide_y, sy * gy)
    elif how == "side":
        px, py = np.where(long_x, slide_x, sx * gx), np.where(long_x, sy * gy, slide_y)
    else:
        px, py = sx * gx, sy * gy
    phi = rng.choice([0.0, np.pi], n)
    return _result(xyxyr(cx, cy, w, l, ra), place(cx, cy, ra, px, py, phi, wb, lb), np.zeros(n))


def corner_on_edge(rng, n):
    """A corner of b on one of a's edges.  In the edge's frame the edge is y = off, |x| <= half, a below it;
    b's edges leave the corner along (cos f, sin f) and (-sin f, cos f): f in [0, pi / 2] keeps b above the edge
    (outside a), f in [pi, 3 pi / 2] below it (inside a, when it fits)."""
    out = []
    while sum(len(o[0]) for o in out) < n:
        m = 2 * n
        cx, cy, w, l, ra = _base(rng, m)
        edge = rng.integers(4, size=m)                           # top, left, bottom, right of a
        psi = edge * (np.pi / 2)
        half, off = np.where(edge % 2 == 0, w / 2, l / 2), np.where(edge % 2 == 0, l / 2, w / 2)
        inside = rng.uniform(size=m) < 0.5
        f = rng.uniform(0, np.pi / 2, m) + np.where(inside, np.pi, 0.0)
        small = np.minimum(w, l)
        wb_out, lb_out = sizes(rng, m)
        wb = np.where(inside, rng.uniform(0.1, 0.6, m) * small, wb_out)
        lb = np.where(inside, rng.uniform(0.1, 0.6, m) * small, lb_out)
        s = rng.uniform(-1, 1, m) * half
        d1, d2 = (np.cos(f), np.sin(f)), (-np.sin(f), np.cos(f))
        ex = s + (wb * d1[0] + lb * d2[0]) / 2                   # b's centre in the edge's frame
        ey = off + (wb * d1[1] + lb * d2[1]) / 2
        px, py = _rot(ex, ey, psi)
        # the inside case must fit: every corner of b within a (the touching corner on its edge)
        fits = np.ones(m, bool)
        for u, v in ((0, 0), (1, 0), (1, 1), (0, 1)):
            qx, qy = _rot(s + u * wb * d1[0] + v * lb * d2[0], off + u * wb * d1[1] + v * lb * d2[1], psi)
            fits &= (np.abs(qx) <= w / 2 * (1 + 1e-12)) & (np.abs(qy) <= l / 2 * (1 + 1e-12))
        keep = ~inside | fits
        A = xyxyr(cx, cy, w, l, ra)[keep]
        B = place(cx, cy, ra, px, py, f + psi, wb, lb)[keep]
        out.append(_result(A, B, np.where(inside, wb * lb, 0.0)[keep]))
    return tuple(np.concatenate([o[k] for o in out])[:n] for k in range(4))


def nested(rng, n):
    cx, cy, w, l, ra = _base(rng, n)
    fw, fl = rng.uniform(0.2, 0.95, n), rng.uniform(0.2, 0.95, n)
    fw[rng.uniform(size=n) < 0.15] = 1.0                         # as wide as a: flush on both sides
    wb, lb = fw * w, fl * l
    flush = rng.integers(3, size=n)                              # 0: x flush, 1: y flush, 2: both (a corner)
    px = np.where(flush != 1, rng.choice([-1.0, 1.0], n) * (w - wb) / 2, rng.uniform(-1, 1, n) * (w - wb) / 2)
    py = np.where(flush != 0, rng.choice([-1.0, 1.0], n) * (l - lb) / 2, rng.uniform(-1, 1, n) * (l - lb) / 2)
    phi = rng.choice([0.0, np.pi], n)
    return _result(xyxyr(cx, cy, w, l, ra), place(cx, cy, ra, px, py, phi, wb, lb), wb * lb)


def square_half_pi(rng, n):
    cx, cy, _, _, ra = _base(rng, n)
    sides = np.array(sorted({v for s in SIZES for v in s}))
    q = sides[rng.integers(len(sides), size=n)]
    px, py, side, t = slide_offset(rng, n, q, q)
    phi = rng.choice([-np.pi / 2, np.pi / 2], n)
    return _result(xyxyr(cx, cy, q, q, ra), place(cx, cy, ra, px, py, phi, q, q), (side - t) * q)


def turned_overlap(w, l, theta):
    """Overlap of a w x l rectangle with itself turned about its centre by a small theta (bigger sides x theta
    well below the smaller side): the rectangle less two pairs of corner triangles."""
    a, b, th = w / 2, l / 2, np.abs(theta)
    c, s, h = np.cos(th), np.sin(th), np.tan(th / 2)
    t1 = 0.5 * (a - b * h) * (b - (b - a * s) / c)
    t2 = 0.5 * (b - a * h) * (a - (a - b * s) / c)
    return 4 * a * b - 2 * (t1 + t2)


def yaw_ulp(rng, n):
    cx, cy, w, l, ra = _base(rng, n)
    r32 = ra.astype(np.float32)
    rb = np.nextafter(r32, np.where(rng.uniform(size=n) < 0.5, np.float32(np.inf), np.float32(-np.inf)))
    rb = rb.astype(np.float64)
    A, B = xyxyr(cx, cy, w, l, ra), xyxyr(cx, cy, w, l, rb)
    return _result(A, B, turned_overlap(w, l, rb - ra))


def zero_width(rng, n):
    cx, cy, w, l, ra = _base(rng, n)
    wb, lb = sizes(rng, n)
    k = rng.integers(3, size=n)                                   # a without width, without length, or both
    w = np.where(k != 1, 0.0, w)
    l = np.where(k == 1, 0.0, l)
    wb = np.where(rng.uniform(size=n) < 0.2, 0.0, wb)             # b without width too
    px, py = rng.uniform(-0.6, 0.6, n) * (w + wb + 1), rng.uniform(-0.6, 0.6, n) * (l + lb + 1)
    phi = rng.uniform(-np.pi, np.pi, n)
    return _result(xyxyr(cx, cy, w, l, ra), place(cx, cy, ra, px, py, phi, wb, lb), np.zeros(n))


BUILDERS = {
    "slide": lambda rng, n: slide(rng, n, (0.0,)),
    "touch_end": lambda rng, n: touch(rng, n, "end"),
    "touch_side": lambda rng, n: touch(rng, n, "side"),
    "touch_corner": lambda rng, n: touch(rng, n, "corner"),
    "corner_on_edge": corner_on_edge,
    "nested": nested,
    "yaw_pi": lambda rng, n: slide(rng, n, (np.pi, -np.pi)),
    "square_half_pi": square_half_pi,
    "yaw_ulp": yaw_ulp,
    "zero_width": zero_width,
}
NAMES = list(BUILDERS)


def families(rng, n):
    return {name: build(rng, n) for name, build in BUILDERS.items()}
