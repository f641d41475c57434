"""Generates tests/golden/nms_tiny.npz from the REFERENCE's own code, on the CPU:

  - rotated IoU: the device functions of mmdet3d/ops/iou3d/src/iou3d_kernel.cu (everything before the first
    __global__) compiled as host C++ with `g++ -ffp-contract=off` (`#define __device__`, std::min / max), and
    evaluated pair by pair;
  - greedy NMS: that fp32 IoU compared with the fp32 threshold, and the host loop of iou3d.cpp:132-145
    (restated here) over the score-sorted boxes;
  - circle_nms: the function of mmdet3d/core/post_processing/box3d_nms.py executed under numba.

Cases: IoU pairs (identical boxes, a shared edge, containment, half-shifted boxes, a zero-width box, yaw at
multiples of pi/2 and outside [-pi, pi], random overlapping pairs); NMS lists of N 1, 63, 64, 65 and 500 at
thresholds 0.2 and 0.5, and of N 65 at -0.1, 0 and 1; a degenerate list whose IoUs are exactly 0, 1/3 or 1;
circle lists at several radii.  Every random list is drawn clear of its threshold: a candidate box is
rejected when its float64 IoU (tests/nms_oracle.py) with an earlier box lies within 1e-3 of the threshold,
or, for circles, when a squared centre distance lies within 1e-6 * thresh of thresh.  Scores are distinct.

Run:  python tests/golden/make_nms_golden.py      (needs the reference tree, g++ and numba)
"""
import ctypes
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import nms_oracle as O  # noqa: E402

REF = os.environ.get("BEVFUSION_REFERENCE", "/root/reference")
SIZES = [(0.5, 0.5), (0.6, 0.8), (0.9, 1.8), (1.9, 4.6), (2.1, 5.3), (2.5, 6.9), (2.9, 11.5), (2.9, 12.0)]


def reference_iou():
    src = open(REF + "/mmdet3d/ops/iou3d/src/iou3d_kernel.cu").read()
    head = src[:src.index("__global__")]
    code = ("#include <cmath>\n#include <algorithm>\nusing std::min; using std::max; using std::fabs;\n"
            "#define __device__\n" + head +
            '\nextern "C" void ref_iou_pairs(const float *a, const float *b, int n, float *out) {\n'
            "  for (int i = 0; i < n; ++i) out[i] = iou_bev(a + 5 * i, b + 5 * i);\n}\n"
            'extern "C" void ref_iou_matrix(const float *a, int n, float *out) {\n'
            "  for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) out[i * n + j] = iou_bev(a + 5 * i, a + 5 * j);\n}\n")
    tmp = tempfile.mkdtemp()
    cpp, so = os.path.join(tmp, "iou_ref.cpp"), os.path.join(tmp, "iou_ref.so")
    open(cpp, "w").write(code)
    subprocess.check_call(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC", "-w", cpp, "-o", so])
    lib = ctypes.CDLL(so)
    P = ctypes.c_void_p

    def pairs(a, b):
        a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
        out = np.zeros(len(a), np.float32)
        lib.ref_iou_pairs(P(a.ctypes.data), P(b.ctypes.data), ctypes.c_int(len(a)), P(out.ctypes.data))
        return out

    def matrix(a):
        a = np.ascontiguousarray(a, np.float32)
        out = np.zeros((len(a), len(a)), np.float32)
        lib.ref_iou_matrix(P(a.ctypes.data), ctypes.c_int(len(a)), P(out.ctypes.data))
        return out
    return pairs, matrix


def reference_circle_nms():
    import numba
    src = open(REF + "/mmdet3d/core/post_processing/box3d_nms.py").read()
    m = re.search(r"@numba\.jit\(nopython=True\)\ndef circle_nms\(.*?(?=\n\S|\Z)", src, re.S)
    ns = {"numba": numba, "np": np}
    exec(m.group(0), ns)
    return ns["circle_nms"]


def host_loop(iou_sorted, thresh):
    """iou3d.cpp:132-145 over the fp32 IoU of the sorted boxes, `iou > thresh` in fp32 (iou3d_kernel.cu:300)."""
    n = iou_sorted.shape[0]
    removed = np.zeros(n, bool)
    keep = []
    for i in range(n):
        if not removed[i]:
            keep.append(i)
            removed[i + 1:] |= iou_sorted[i, i + 1:] > np.float32(thresh)
    return np.array(keep, np.int64)


def xyxyr(x, y, w, l, r):
    return np.array([x - w / 2, y - l / 2, x + w / 2, y + l / 2, r], np.float32)


def random_box(rng, span, centre=None, jitter=None):
    w, l = SIZES[rng.integers(len(SIZES))]
    if centre is None:
        x, y = rng.uniform(-span, span, 2)
        r = rng.uniform(-np.pi, np.pi)
    else:
        x, y = centre[0] + rng.normal(0, jitter * w), centre[1] + rng.normal(0, jitter * l)
        r = centre[2] + rng.normal(0, 0.3)
        w, l = centre[3] * rng.uniform(0.85, 1.15), centre[4] * rng.uniform(0.85, 1.15)
    return xyxyr(x, y, w, l, r), (x, y, r, w, l)


def clear_of(box, boxes, thresh):
    if not boxes:
        return True
    B = np.array(boxes, np.float64)
    for j, v in enumerate(O.iou_matrix(np.asarray(box, np.float64)[None], B)[0]):
        if abs(v - thresh) < 1e-3:
            if v == 0.0 and O._apart(B[j] + np.array([-5e-3, -5e-3, 5e-3, 5e-3, 0]), np.asarray(box, np.float64)):
                continue                       # clearly apart: exactly 0 in any arithmetic
            return False
    return True


def clustered_list(rng, n, thresh, span):
    boxes, objs = [], []
    while len(boxes) < n:
        if not objs or rng.uniform() < 0.2:
            b, o = random_box(rng, span)
            objs.append(o)
        else:
            b, _ = random_box(rng, span, objs[rng.integers(len(objs))], 0.25)
        if clear_of(b, boxes, thresh):
            boxes.append(b)
    return np.array(boxes, np.float32).reshape(-1, 5)


def main():
    iou_pairs, iou_matrix = reference_iou()
    circle = reference_circle_nms()
    rng = np.random.default_rng(20261016)
    out = {}

    # ---- IoU pairs -----------------------------------------------------------------------------------------
    a, b = [], []
    named = [
        ([0, 0, 2, 2, 0], [0, 0, 2, 2, 0]),                          # identical: 1
        ([0, 0, 2, 2, 0], [1, 0, 3, 2, 0]),                          # half-shifted: 1/3
        ([0, 0, 1, 1, 0], [0, 0, 1, 1, np.pi / 4]),                  # square against itself turned by pi/4
        ([0, 0, 1, 1, 0], [5, 5, 6, 6, 0]),                          # disjoint: 0
        ([0, 0, 2, 2, 0], [2, 0, 4, 2, 0]),                          # shared edge: 0
        ([0, 0, 4, 4, 0], [1, 1, 2, 2, 0]),                          # containment: 1/16
        ([0, 0, 4, 4, 0.3], [1.5, 1.5, 2.5, 2.5, 0.3]),              # turned containment: 1/16
        ([0, 0, 0, 2, 0], [-1, -1, 1, 1, 0]),                        # zero-width box: 0
        ([10, 20, 12, 25, 0.7], [10, 20, 12, 25, 0.7]),              # identical, turned, off-origin
    ]
    for p, q in named:
        a.append(p)
        b.append(q)
    for k in range(-4, 5):                                           # yaw at multiples of pi/2
        a.append([3, -2, 5, 2.5, 0.2])
        b.append([3.5, -1, 6, 1, 0.2 + k * np.pi / 2])
    for _ in range(600):                                             # random overlapping pairs
        p, o = random_box(rng, 61)
        q, _ = random_box(rng, 61, o, 0.3)
        if rng.uniform() < 0.2:
            q[4] += rng.choice([-2, 2]) * np.pi                      # outside [-pi, pi]
        a.append(p)
        b.append(q)
    out["iou_a"] = np.array(a, np.float32)
    out["iou_b"] = np.array(b, np.float32)
    out["iou_ref"] = iou_pairs(out["iou_a"], out["iou_b"])
    out["iou_named"] = np.int64(len(named))

    # ---- NMS lists -----------------------------------------------------------------------------------------
    cases = [(1, 0.2), (63, 0.2), (64, 0.2), (65, 0.2), (63, 0.5), (64, 0.5), (65, 0.5), (500, 0.2),
             (65, -0.1), (65, 0.0), (65, 1.0)]
    for k, (n, thresh) in enumerate(cases):
        boxes = clustered_list(rng, n, thresh, 20 if n <= 65 else 61)
        scores = rng.permutation(n).astype(np.float32) / n + rng.uniform(0, 0.5 / n, n).astype(np.float32)
        out["nms%d_boxes" % k], out["nms%d_scores" % k], out["nms%d_thresh" % k] = boxes, scores, np.float64(thresh)
    # degenerate list: IoUs exactly 0, 1/3 or 1 (identical, half-shifted, disjoint, shared edge, zero width)
    deg = np.array([[0, 0, 2, 2, 0], [0, 0, 2, 2, 0], [1, 0, 3, 2, 0], [5, 5, 6, 6, 0], [2, 0, 4, 2, 0],
                    [8, 8, 8, 9, 0], [-3, -3, -1, -1, np.pi / 2]], np.float32)
    for thresh in (0.2, 0.5):
        k = len([x for x in out if x.endswith("_thresh")])
        out["nms%d_boxes" % k], out["nms%d_thresh" % k] = deg, np.float64(thresh)
        out["nms%d_scores" % k] = np.array([0.9, 0.8, 0.7, 0.6, 0.5, 0.4, 0.3], np.float32)
    ncase = len([x for x in out if x.endswith("_thresh")])
    for k in range(ncase):
        boxes, scores, thresh = out["nms%d_boxes" % k], out["nms%d_scores" % k], float(out["nms%d_thresh" % k])
        order = np.argsort(-scores.astype(np.float64), kind="stable")
        out["nms%d_keep" % k] = order[host_loop(iou_matrix(boxes[order]), thresh)]
    out["nms_cases"] = np.int64(ncase)

    # ---- circle lists --------------------------------------------------------------------------------------
    circ = [(63, 4.0, 83), (64, 0.175, 83), (65, 1.0, 20), (500, 12.0, 83), (500, 0.85, 83), (1, 4.0, 83)]
    for k, (n, thresh, post) in enumerate(circ):
        span = 4 if thresh < 2 else 30
        pts = []
        while len(pts) < n:
            p = rng.uniform(-span, span, 2).astype(np.float32)
            if pts:
                d2 = ((np.array(pts, np.float64) - p.astype(np.float64)) ** 2).sum(1)
                if (np.abs(d2 - thresh) < 1e-6 * thresh).any():
                    continue
            pts.append(p)
        scores = (rng.permutation(n) + 1).astype(np.float32) / (n + 1)
        dets = np.concatenate([np.array(pts, np.float32), scores[:, None]], 1)
        out["circle%d_dets" % k], out["circle%d_thresh" % k], out["circle%d_post" % k] = dets, np.float64(thresh), np.int64(post)
        out["circle%d_keep" % k] = np.array(circle(dets, thresh, post_max_size=post), np.int64)
    out["circle_cases"] = np.int64(len(circ))

    path = os.path.join(HERE, "nms_tiny.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "%d IoU pairs, %d NMS lists, %d circle lists" % (len(a), ncase, len(circ)))


if __name__ == "__main__":
    main()
