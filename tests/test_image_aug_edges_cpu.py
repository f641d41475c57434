"""CPU: the camera augmentation's boundary cases (tests/data_pipeline_cases.py) -- the numpy restatement against the
installed Pillow + torchvision at the shapes no other test holds there (the tallest input, frames kMaxFrame wide and
tall on every rotate path, 1 x 1 resizes of 1600 x 900, large upscales, crops at the draw check's bound), the fixed
16.16 rotate range at kMaxFrame, and that each case builder lands on the boundary it names."""
import math

import numpy as np
import pytest

import data_pipeline_cases as C
import image_aug_oracle as O

PIL = pytest.importorskip("PIL.Image")
TF = pytest.importorskip("torchvision.transforms.functional")

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


def pillow(img, dims, xy, fH, fW, flip, rotate):
    im = PIL.fromarray(img).resize(dims).crop((xy[0], xy[1], xy[0] + fW, xy[1] + fH))
    if flip:
        im = im.transpose(PIL.FLIP_LEFT_RIGHT)
    return TF.normalize(TF.to_tensor(im.rotate(rotate)), MEAN, STD).numpy()


def bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.int32),
                                                 np.ascontiguousarray(b).view(np.int32))


@pytest.mark.parametrize("name", C.PILLOW_CALLS)
def test_oracle_equals_pillow(name):
    call = C.image_calls()[name]
    imgs = C.call_images(name, call)
    for n, ((_, dims, xy, flip, rot), st) in enumerate(zip(call["draws"], call["expect"])):
        if st:
            continue
        want = pillow(imgs[n], dims, xy, call["fH"], call["fW"], flip, rot)
        got = O.augment(imgs[n], dims, xy, (call["fH"], call["fW"]), flip, rot, MEAN, STD)
        assert bits_equal(got, want), (name, n)


def _check_fixed(m, x, y):
    # Pillow's ImagingTransformAffine takes affine_fixed only when the corners map inside +-32768
    return abs(x * m[0] + y * m[1] + m[2]) < 32768.0 and abs(x * m[3] + y * m[4] + m[5]) < 32768.0


@pytest.mark.parametrize("w,h", [(C.MAX_FRAME, C.MAX_FRAME), (C.MAX_FRAME, 1), (1, C.MAX_FRAME),
                                 (C.MAX_FRAME, C.MAX_FRAME - 1)])
def test_rotate_stays_in_the_fixed_point_range_at_the_largest_frame(w, h):
    """every angle in 0.25-degree steps (and 45 + 1e-9): Pillow's fixed-point test passes at the four corners, and
    the kernel's closed-form 16.16 sums a2 + y a1 + x a0 stay inside int32 over the whole frame"""
    fix = lambda v: math.floor(v * 65536.0 + 0.5)
    for angle in list(np.arange(0.0, 360.0, 0.25)) + [45.0 + 1e-9, 135.0 - 1e-9]:
        kind, m = O.rotate_rule(float(angle), w, h)
        if kind != "affine":
            continue
        assert all(_check_fixed(m, x, y) for x in (0, w) for y in (0, h)), (angle, w, h)
        a0, a1, a3, a4 = fix(m[0]), fix(m[1]), fix(m[3]), fix(m[4])
        a2, a5 = fix(m[2] + m[0] * 0.5 + m[1] * 0.5), fix(m[5] + m[3] * 0.5 + m[4] * 0.5)
        for x in (0, w - 1):
            for y in (0, h - 1):
                assert abs(a2 + y * a1 + x * a0) < 2 ** 31 and abs(a5 + y * a4 + x * a3) < 2 ** 31, (angle, x, y)


def test_derived_case_lists():
    """the tiling and limit edges follow the kernel's constants"""
    cols, rows = C.HPASS_COLS, C.HPASS_ROWS
    assert C.frame_width_edges() == sorted({1} | {k * c + d for c in (cols, C.VPASS_COLS) for k in (1, 2)
                                                  for d in (-1, 0, 1)})
    assert C.band_row_edges() == sorted({1} | {k * rows + d for k in (1, 2, 3) for d in (-1, 0, 1)})
    calls = C.image_calls()
    assert sorted(n for n in calls if n.startswith("fW=") and n != "fW=max") == \
        sorted("fW=%d" % v for v in C.frame_width_edges())
    assert C.CROP_LIMIT == 1 << 30                  # the header's |crop| <= 2^30


def test_band_cases_make_their_band():
    """every band edge from an upscale cropped at the top edge; every edge a downscale reaches from one cropped inside
    the image (its band starts past row 0)"""
    calls = C.image_calls()
    for n in C.band_row_edges():
        kinds = [k for k, _, _ in C.BAND_KINDS if "band=%d/%s" % (n, k) in calls]
        assert "top" in kinds, n
        if n >= 2 * C.HPASS_ROWS - 1:
            assert "inside" in kinds, n
        for kind in kinds:
            call = calls["band=%d/%s" % (n, kind)]
            for _, (w, h), (x0, y0), _, _ in call["draws"]:
                assert C.band_rows(call["H"], h, y0, call["fH"]) == n, (n, kind)
                if kind == "inside":
                    assert call["H"] > h and y0 > 0 and C.bounds(call["H"], h, y0)[0] > 0, n
                else:
                    assert call["H"] <= h and y0 == 0, n


def test_frame_width_cases_span_the_blocks():
    """each fW case has a crop that runs off the resized image on one side or the other"""
    for fW in C.frame_width_edges():
        call = C.image_calls()["fW=%d" % fW]
        assert call["fW"] == fW
        (_, (w, _), (x0, _), _, _), (_, _, (x1, _), _, _) = call["draws"]
        assert x0 < 0 and x1 + fW > w


def test_capacity_cases_sit_on_the_table_width():
    call = C.image_calls()["kcap"]
    mw, mh = call["min_resize"]
    kw, kh = C.ksize(call["W"], mw), C.ksize(call["H"], mh)
    got = [(C.ksize(call["W"], w), C.ksize(call["H"], h)) for _, (w, h), _, _, _ in call["draws"]]
    widths = [d[1][0] for d in call["draws"]]
    heights = [d[1][1] for d in call["draws"]]
    assert got[0] == (kw, kh)
    assert got[1] == (kw, kh) and widths[1] < mw and got[2][0] == kw + 2 and widths[2] == widths[1] - 1
    assert got[3] == (kw, kh) and heights[3] < mh and got[4][1] == kh + 2 and heights[4] == heights[3] - 1
    assert got[5][0] < kw // 2 and got[5][1] < kh // 2
    over = [C.OVER_CAPACITY if g[0] > kw or g[1] > kh else 0 for g in got]
    assert over == call["expect"]
    ext = C.image_calls()["to-1x1"]
    assert C.ksize(ext["W"], 1) == 2 * 2 * ext["W"] + 1 and C.ksize(ext["H"], 1) == 2 * 2 * ext["H"] + 1


def test_limit_cases_reach_the_limits():
    calls = C.image_calls()
    tall = calls["tall"]
    assert tall["H"] == C.MAX_SOURCE - 1 and C.MAX_GRID == 65535             # CUDA's grid.y limit
    assert -(-tall["H"] // C.HPASS_ROWS) > C.MAX_GRID                         # more row blocks than grid.y holds
    (_, (w, h), (x0, y0), _, _), = tall["draws"]
    assert C.band_rows(tall["H"], h, y0, tall["fH"]) > C.MAX_GRID * C.HPASS_ROWS   # rows past the grid are banded
    # and the expected output depends on them: a pass that skipped them would be caught
    assert C.tall_tail_matters(tall, C.call_images("tall", tall)[0]) > 0
    assert calls["fW=max"]["fW"] == C.MAX_FRAME and calls["fH=max"]["fH"] == C.MAX_FRAME
    for name, (w, h) in (("fW=max", (C.MAX_FRAME, 16)), ("fH=max", (16, C.MAX_FRAME))):
        kinds = [O.rotate_rule(d[4], w, h)[0] for d in calls[name]["draws"]]
        assert sorted(set(kinds)) == ["affine", "rot180", "scale"], kinds
    crops = [d[2] for d in calls["crop=limit"]["draws"]]
    L = C.CROP_LIMIT
    bad = [max(abs(x), abs(y)) > L for x, y in crops]
    assert [C.BAD_DRAW if b else 0 for b in bad] == calls["crop=limit"]["expect"]
    assert {abs(v) for xy in crops for v in xy} >= {L, L + 1}
    one = calls["frame=1x1"]
    assert (one["fH"], one["fW"]) == (1, 1)
    assert {O.rotate_rule(d[4], 1, 1)[0] for d in one["draws"]} == {"copy", "rot90", "rot180", "affine", "scale"}


def test_many_camera_draws_take_every_rotate_path():
    draws = C.many_camera_draws()
    assert len(draws) == C.CAM_DRAWS and math.gcd(C.CAM_DRAWS, C.CAM_IMAGES) == 1
    assert {O.rotate_rule(d[4], 2, 2)[0] for d in draws} == {"copy", "rot90", "rot270", "rot180", "affine", "scale"}


def test_workspace_query_refuses_past_the_camera_limit():
    from bevfusion_b200 import _C
    q = _C.lib().bevb200_image_aug_workspace_bytes
    assert q(C.MAX_GRID, 3, 3, 2, 2, 1, 1) > 0
    assert q(C.MAX_GRID + 1, 3, 3, 2, 2, 1, 1) == 0
    assert q(1, C.MAX_SOURCE - 1, 1, 8, 3, 3, 8) > 0 and q(1, C.MAX_SOURCE, 1, 8, 3, 3, 8) == 0
    assert q(1, 8, 8, C.MAX_FRAME, C.MAX_FRAME, 1, 1) > 0 and q(1, 8, 8, C.MAX_FRAME + 1, 4, 1, 1) == 0
