"""Pins oracle/image_pre.py -- the checker of tb200_graph_upload_images -- against the input preprocessing of the UNMODIFIED
examples/tm_classification_int8.c and tm_classification_uint8.c: (a) the committed fixture tests/golden/image_pre_example.npz,
produced by the examples' own get_input_int8_data / get_input_uint8_data from image files (generator:
tests/golden/make_golden_image_pre.py), everywhere; (b) the compiled examples themselves, live, on freshly seeded images, where
oracle/_ref/libimage_example.so exists.  Byte for byte.  Also checks that abi.Image has the size of tb200_image."""
import ctypes
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from oracle import image_pre  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "image_pre_example.npz")


def _case(d, k):
    H, W = (int(v) for v in d[f"hw_{k}"])
    s_in, zp, u8 = d[f"quant_{k}"]
    return d[f"pix_{k}"], H, W, d[f"mean_{k}"], d[f"scale_{k}"], np.float32(s_in), int(zp), bool(u8)


def _restated(d, k):
    img, H, W, mean, scale, s_in, zp, u8 = _case(d, k)
    return image_pre.preprocess(img, H, W, mean, scale, s_in, zp, u8)


def test_restatement_equals_the_committed_output_of_the_unmodified_examples():
    d = np.load(FIXTURE)
    names = list(d["names"])
    assert len(names) >= 12
    for k, name in enumerate(names):
        got, want = _restated(d, k), d[f"out_{k}"]
        assert got.dtype == want.dtype and got.shape == want.shape, name
        assert np.array_equal(got, want), (name, int((got != want).sum()))
    dtypes = {d[f"out_{k}"].dtype for k in range(len(names))}
    assert dtypes == {np.dtype(np.int8), np.dtype(np.uint8)}
    assert {int(d[f"pix_{k}"].shape[2]) for k in range(len(names))} == {3, 4}
    assert {int(d[f"quant_{k}"][1]) for k in range(len(names)) if d[f"quant_{k}"][2]} >= {0, 3, 128}


def test_the_fixture_reaches_the_quirks_it_is_there_for():
    d = np.load(FIXTURE)
    names = list(d["names"])
    # the upsample's first columns extrapolate: resized values leave 0..255
    img, H, W = _case(d, names.index("upsample_int8"))[:3]
    v = image_pre.resize_bgr(img, H, W)
    assert v.min() < 0 and v.max() > 255
    # same size: the last column and row repeat source pixel w - 2 / h - 2 instead of copying w - 1 / h - 1
    img, H, W = _case(d, names.index("same_size_int8"))[:3]
    v = image_pre.resize_bgr(img, H, W)
    bgr = img[:, :, 2::-1].transpose(2, 0, 1).astype(np.int32)
    assert np.array_equal(v[:, :-1, :-1], bgr[:, :-1, :-1])
    assert np.array_equal(v[:, :-1, -1], bgr[:, :-1, -2]) and np.array_equal(v[:, -1, :-1], bgr[:, -2, :-1])
    assert not np.array_equal(v[:, :, -1], bgr[:, :, -1])
    # ties: every odd value / 2 is an exact .5; halfway-away rounding is what the examples do, half-to-even would differ
    for name in ("ties_int8", "ties_uint8_zp3"):
        img, H, W, mean, scale, s_in, zp, u8 = _case(d, names.index(name))
        q = (image_pre.resize_bgr(img, H, W).astype(np.float32) / s_in + np.float32(zp)).astype(np.float32)
        ties = np.abs(q - np.trunc(q)) == 0.5
        assert ties.mean() > 0.3, name
        even = np.rint(q.astype(np.float64))
        even = np.clip(even, 0, 255).astype(np.uint8) if u8 else np.clip(even, -127, 127).astype(np.int8)
        assert not np.array_equal(even, d[f"out_{names.index(name)}"]), name
    # saturation at both ends
    for name, lo, hi in (("saturating_int8", -127, 127), ("saturating_uint8_zp128", 0, 255)):
        out = d[f"out_{names.index(name)}"].astype(np.int32)
        assert (out == lo).any() and (out == hi).any(), name
    # a quotient beyond int's range converts to INT_MIN, so even positive values land on the lower bound
    for name, lo in (("tiny_scale_int8", -127), ("tiny_scale_uint8_zp128", 0)):
        img, H, W, mean, scale = _case(d, names.index(name))[:5]
        f = (image_pre.resize_bgr(img, H, W).astype(np.float32) - np.asarray(mean, np.float32).reshape(3, 1, 1)) * np.asarray(scale, np.float32).reshape(3, 1, 1)
        assert (f > 0).any() and (f < 0).any(), name
        assert (d[f"out_{names.index(name)}"].astype(np.int32) == lo).all(), name


def test_restatement_equals_the_compiled_examples_live():
    import make_golden_image_pre as gen

    if not os.path.exists(gen.LIB):
        pytest.skip("oracle/_ref/libimage_example.so absent (built by oracle/build_image_example.py where the reference tree exists)")
    L = gen.example_lib()
    rng = np.random.default_rng(2024)
    with tempfile.TemporaryDirectory() as tmp:
        for trial in range(12):
            c = 4 if trial % 4 == 3 else 3
            h, w = (int(v) for v in rng.integers(2, 90, 2))
            H, W = (int(v) for v in rng.integers(2, 70, 2))
            img = gen.random_image(rng, h, w, c)
            mean = rng.uniform(0, 255, 3).astype(np.float32)
            scale = rng.uniform(0.005, 0.05, 3).astype(np.float32)
            u8 = bool(trial % 2)
            s_in = np.float32(rng.uniform(0.005, 0.05))
            zp = int(rng.integers(0, 256)) if u8 else 0
            want = gen.run_example(L, img, H, W, mean, scale, s_in, zp, u8, tmp)
            got = image_pre.preprocess(img, H, W, mean, scale, s_in, zp, u8)
            assert np.array_equal(got, want), (trial, (h, w, c), (H, W), int((got != want).sum()))


def test_image_struct_size_matches_header():
    from tengine_b200 import abi

    src = '#include <stdio.h>\n#include <stddef.h>\n#include "tengine_b200.h"\nint main(){printf("%zu %zu\\n", sizeof(tb200_image), offsetof(tb200_image, c));return 0;}'
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        out = subprocess.check_output([os.path.join(d, "t")]).split()
    assert [int(x) for x in out] == [ctypes.sizeof(abi.Image), abi.Image.c.offset]
