"""Pins oracle/detect_pre.py -- the checker of tb200_graph_upload_detect_images and tb200_detections_to_source -- against the YOLO
examples' quantised preprocessing as OpenCV computes it: (a) the committed fixture tests/golden/detect_pre_example.npz, made with the cv2
binding's cv::resize / cv::copyMakeBorder and a line-by-line transcription of the examples (generator:
tests/golden/make_golden_detect_pre.py), everywhere; (b) cv2.resize itself, live, on a seeded sweep of sizes, where cv2 is importable.
Each fixture case is asserted to exercise the quirk it is there for.  Also checks the two new structs against abi.py and the library's
tb200_detections_to_source against the restatement (no GPU needed)."""
import ctypes
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import detect_pre as dp  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "detect_pre_example.npz")
f32 = np.float32


def _case(d, k):
    mode, H, W, focus, u8, zp = (int(v) for v in d[f"cfg_{k}"])
    return d[f"pix_{k}"], mode, H, W, d[f"mean_{k}"], d[f"scale_{k}"], f32(d[f"sin_{k}"]), zp, bool(u8), bool(focus)


def _restated(d, k):
    img, mode, H, W, mean, scale, s_in, zp, u8, focus = _case(d, k)
    return dp.preprocess(img, mode, H, W, mean, scale, s_in, zp, u8, focus)


def _geo(d, k):
    img, mode, H, W = _case(d, k)[:4]
    return dp.geometry(mode, img.shape[1], img.shape[0], W, H)


def test_restatement_equals_the_fixture():
    d = np.load(FIXTURE)
    names = list(d["names"])
    assert len(names) >= 15 and str(d["cv2_version"])
    for k, name in enumerate(names):
        got, want = _restated(d, k), d[f"out_{k}"]
        assert got.dtype == want.dtype and got.shape == want.shape, name
        assert np.array_equal(got, want), (name, int((got != want).sum()))
        mode = int(d[f"cfg_{k}"][0])
        mapped = np.array([dp.to_source(mode, _geo(d, k), b) for b in d[f"boxes_{k}"]], np.float32)
        assert np.array_equal(mapped, d[f"mapped_{k}"]), name
    cfg = np.array([d[f"cfg_{k}"] for k in range(len(names))])
    assert set(cfg[:, 0]) == {dp.STRETCH, dp.LETTERBOX} and set(cfg[:, 3]) == {0, 1}
    assert {d[f"out_{k}"].dtype for k in range(len(names))} == {np.dtype(np.int8), np.dtype(np.uint8)}
    assert {int(c[5]) for c in cfg if c[4]} >= {0, 128}
    assert {int(d[f"pix_{k}"].shape[2]) for k in range(len(names))} == {3, 4}
    assert any(np.array_equal(d[f"scale_{k}"], np.float32(dp.DEFAULT_SCALE)) and not d[f"mean_{k}"].any() for k in range(len(names)))
    sizes = [d[f"pix_{k}"].shape[:2] for k in range(len(names))]
    assert min(h for h, _ in sizes) == 2 and min(w for _, w in sizes) == 2
    assert any(h > w for h, w in sizes) and any(w > h for h, w in sizes)


def _vertical_clamped(img, W, H):
    """cv_resize with the vertical axis clamped like the horizontal one: the rule that OpenCV does NOT follow."""
    h = img.shape[0]
    sy, cy0, cy1 = dp.linear_coef(H, h, True)
    sx, cx0, cx1 = dp.linear_coef(W, img.shape[1], True)
    src = img.astype(np.int64)
    hr = src[:, sx] * cx0[None, :, None] + src[:, np.minimum(sx + 1, img.shape[1] - 1)] * cx1[None, :, None]
    S0, S1 = hr[sy], hr[np.minimum(sy + 1, h - 1)]
    v = (((cy0[:, None, None] * (S0 >> 4)) >> 16) + ((cy1[:, None, None] * (S1 >> 4)) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8)


def test_the_fixture_reaches_the_quirks_it_is_there_for():
    d = np.load(FIXTURE)
    names = list(d["names"])
    ix = names.index
    # upscale: the unclamped vertical position changes the first / last rows; clamping it would miss the fixture
    for name in ("letterbox_up_focus_int8", "stretch_up_uint8_zp0", "stretch_w2_up_uint8_zp0"):
        img = d[f"pix_{ix(name)}"][:, :, :3]
        _, _, rw, rh, _, _, _ = _geo(d, ix(name))
        assert rh > img.shape[0] and rw > img.shape[1], name
        assert not np.array_equal(_vertical_clamped(img, rw, rh), dp.cv_resize(img, rw, rh)), name
    # exact 2x on both axes (OpenCV's INTER_AREA route): the linear formula gives the 2x2 mean (a + b + c + d + 2) >> 2
    for name in ("letterbox_exact2x_focus_uint8_zp0", "stretch_exact2x_focus_int8"):
        img = d[f"pix_{ix(name)}"][:, :, :3].astype(np.int64)
        _, _, rw, rh, _, _, _ = _geo(d, ix(name))
        assert (2 * rw, 2 * rh) == (img.shape[1], img.shape[0]), name
        area = (img[0::2, 0::2] + img[0::2, 1::2] + img[1::2, 0::2] + img[1::2, 1::2] + 2) >> 2
        assert np.array_equal(dp.cv_resize(d[f"pix_{ix(name)}"][:, :, :3], rw, rh), area.astype(np.uint8)), name
    # int(scale * cols) truncates: one column short of the input, so the border is 0 columns left, 1 right
    g = _geo(d, ix("letterbox_truncated_width_focus_uint8_zp128"))
    assert (g[2], g[4]) == (63, 0) and round(float(g[6]) * g[0]) == 64
    # the border is byte 0 before normalisation, not the grey 0.5 / scale + mean of the discarded img_new
    k = ix("letterbox_down_nofocus_uint8_zp128")
    img, mode, H, W, mean, scale, s_in, zp, u8, _ = _case(d, k)
    _, _, rw, rh, left, top, _ = _geo(d, k)
    assert top > 0 and rh < H
    zero = dp.quantise(np.zeros((3, 1), np.uint8), mean, scale, s_in, zp, u8)[:, 0]
    grey = dp.quantise(np.full((3, 1), 0.0, np.float32) + (f32(0.5) / scale + mean)[:, None], mean, scale, s_in, zp, u8)[:, 0]
    assert np.array_equal(d[f"out_{k}"][:, 0, 0], zero) and not np.array_equal(zero, grey)
    # Focus: group i * 2 + g holds column offset i, row offset g; the transposed reading differs
    for name in ("letterbox_up_focus_int8", "letterbox_not_square_focus_int8"):
        img, mode, H, W, mean, scale, s_in, zp, u8, _ = _case(d, ix(name))
        q = dp.preprocess(img, mode, H, W, mean, scale, s_in, zp, u8, False)
        swapped = np.concatenate([q[:, i:H:2, g:W:2] for i in range(2) for g in range(2)], axis=0)
        assert np.array_equal(d[f"out_{ix(name)}"], dp.focus(q)) and not np.array_equal(d[f"out_{ix(name)}"], swapped), name
    # ties: halfway-away rounding is what the examples do; half to even would differ
    for name in ("letterbox_ties_int8", "stretch_ties_uint8_zp3"):
        img, mode, H, W, mean, scale, s_in, zp, u8, focus = _case(d, ix(name))
        lay = dp.laid_out(img, mode, W, H).transpose(2, 0, 1)
        q = (lay.astype(np.float32) / s_in + np.float32(zp)).astype(np.float32)
        assert (np.abs(q - np.trunc(q)) == 0.5).mean() > 0.3, name
        even = np.rint(q.astype(np.float64))
        even = np.clip(even, 0, 255).astype(np.uint8) if u8 else np.clip(even, -127, 127).astype(np.int8)
        assert not np.array_equal(even, d[f"out_{ix(name)}"]), name
    # back-mapping: the letterbox's swapped ratios matter for a non-square source, and the clamps act
    k = ix("letterbox_down_nofocus_uint8_zp128")
    geo = _geo(d, k)
    src_w, src_h, rw, rh = geo[:4]
    assert f32(f32(src_h) / f32(rh)) != f32(f32(src_w) / f32(rw))
    mapped = np.concatenate([d[f"mapped_{j}"] for j in range(len(names))])
    assert (mapped[:, 0] == 0).any() and (mapped[:, 1] == 0).any()
    assert any((d[f"mapped_{j}"][:, 0] + d[f"mapped_{j}"][:, 2] == d[f"pix_{j}"].shape[1] - 1).any() for j in range(len(names)))


def test_resize_equals_cv2_on_a_seeded_sweep():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(1234)
    up = down = 0
    for trial in range(200):
        # log-uniform sizes in 2..1500: both directions and every scale in between are common
        h, w, H, W = (int(v) for v in np.exp(rng.uniform(np.log(2), np.log(1500), 4)).round())
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        got, want = dp.cv_resize(img, W, H), cv2.resize(img, (W, H))
        assert np.array_equal(got, want), (trial, (w, h), (W, H), int((got != want).sum()))
        up += H > h and W > w
        down += H < h and W < w
    assert up > 30 and down > 30, (up, down)
    for (w, h) in ((1280, 1280), (832, 832), (640, 480)):  # exact 2x: OpenCV takes INTER_AREA
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        assert np.array_equal(dp.cv_resize(img, w // 2, h // 2), cv2.resize(img, (w // 2, h // 2)))


def test_new_structs_match_the_header():
    from tengine_b200 import abi

    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "tengine_b200.h"\nint main(){printf("%zu %zu %zu %zu\\n", sizeof(tb200_detect_pre), '
           'offsetof(tb200_detect_pre, scale), sizeof(tb200_detect_geometry), offsetof(tb200_detect_geometry, scale));return 0;}')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        out = subprocess.check_output([os.path.join(d, "t")]).split()
    assert [int(x) for x in out] == [ctypes.sizeof(abi.DetectPre), abi.DetectPre.scale.offset, ctypes.sizeof(abi.DetectGeometry),
                                     abi.DetectGeometry.scale.offset]


def _geometry_array(geos):
    from tengine_b200 import abi

    return (abi.DetectGeometry * len(geos))(*[(int(a), int(b), int(c), int(e), int(f), int(g), float(s)) for a, b, c, e, f, g, s in geos])


def test_library_back_mapping_equals_the_restatement():
    from tengine_b200 import runtime as rt

    d = np.load(FIXTURE)
    names = list(d["names"])
    for mode in (dp.STRETCH, dp.LETTERBOX):
        ks = [k for k in range(len(names)) if int(d[f"cfg_{k}"][0]) == mode]
        geos = [_geo(d, k) for k in ks]
        boxes = [[(*b, 0.5, 3) for b in d[f"boxes_{k}"].tolist()] for k in ks]
        got = rt.detections_to_source(_geometry_array(geos), boxes, letterbox=mode == dp.LETTERBOX)
        for k, g in zip(ks, got):
            assert np.array_equal(np.array([b[:4] for b in g], np.float32), d[f"mapped_{k}"]), names[k]
            assert all(b[4] == np.float32(0.5) and b[5] == 3 for b in g)


def test_library_back_mapping_checks_and_overflow():
    from tengine_b200 import abi
    from tengine_b200 import runtime as rt

    L = rt.lib()
    geo = _geometry_array([(100, 50, 64, 32, 0, 16, 0.64), (30, 40, 48, 64, 8, 0, 1.6)])
    dets = (abi.Detection * 4)()
    for i in range(4):
        dets[i].x, dets[i].y, dets[i].w, dets[i].h = 10.0 + i, 20.0, 5.0, 6.0
    before = [(d.x, d.y, d.w, d.h) for d in dets]
    counts = (ctypes.c_int32 * 2)(-3, 1)  # image 0 overflowed: left as it is
    assert L.tb200_detections_to_source(abi.PRE_LETTERBOX, geo, 2, dets, 2, counts) == 0
    assert [(d.x, d.y, d.w, d.h) for d in dets[:2]] == before[:2] and (dets[3].x, dets[3].y) == before[3][:2]
    want = dp.to_source(dp.LETTERBOX, (30, 40, 48, 64, 8, 0, f32(1.6)), before[2])
    assert (dets[2].x, dets[2].y, dets[2].w, dets[2].h) == tuple(float(v) for v in want)
    ok = (ctypes.c_int32 * 2)(0, 1)
    for args in ((2, geo, 2, dets, 2, ok), (abi.PRE_STRETCH, None, 2, dets, 2, ok), (abi.PRE_STRETCH, geo, 2, None, 2, ok),
                 (abi.PRE_STRETCH, geo, 2, dets, 2, None), (abi.PRE_STRETCH, geo, -1, dets, 2, ok), (abi.PRE_STRETCH, geo, 2, dets, 0, ok),
                 (abi.PRE_STRETCH, geo, 2, dets, 2, (ctypes.c_int32 * 2)(0, 3)),
                 (abi.PRE_STRETCH, _geometry_array([(100, 50, 0, 32, 0, 0, 0.0), (30, 40, 48, 64, 8, 0, 1.6)]), 2, dets, 2, ok)):
        assert L.tb200_detections_to_source(*args) == abi.ERR_INVALID, args
    assert L.tb200_detections_to_source(abi.PRE_STRETCH, None, 0, None, 1, None) == 0
