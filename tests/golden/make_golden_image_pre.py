#!/usr/bin/env python3
"""Golden vectors for oracle/image_pre.py: the input preprocessing of the UNMODIFIED examples/tm_classification_int8.c and
tm_classification_uint8.c (get_input_int8_data / get_input_uint8_data, compiled by oracle/build_image_example.py into
oracle/_ref/libimage_example.so through oracle/image_example_shim.c), run on image files: RGB images are written as binary PPM, RGBA
images as PNG through the reference's own stbi_write_png, and the examples read them back with their own stbi_load.  Needs the
reference tree at build time; the .npz it writes is committed so that the pin holds anywhere.
usage: make_golden_image_pre.py [out.npz]"""
import ctypes as C
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(ROOT, "oracle", "_ref", "libimage_example.so")
REF_JPG = "/root/reference/doc/docs_en/images/clip_image004.jpg"  # 269 x 383 RGB, decoded by the example's stbi_load
DEFAULT_MEAN = (104.007, 116.669, 122.679)
DEFAULT_SCALE = (0.017, 0.017, 0.017)


def example_lib():
    L = C.CDLL(LIB)
    L.stbi_load.restype = C.c_void_p
    L.stbi_load.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    L.stbi_image_free.argtypes = [C.c_void_p]
    L.stbi_write_png.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]
    L.get_input_int8_data.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_float]
    L.get_input_uint8_data.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_int]
    return L


def stbi_load(L, path):
    """HxWxC uint8 as the examples' load_image_stb reads the file (stbi_load with desired_channels 0)."""
    w, h, c = C.c_int(), C.c_int(), C.c_int()
    p = L.stbi_load(path.encode(), C.byref(w), C.byref(h), C.byref(c), 0)
    assert p, path
    a = np.ctypeslib.as_array((C.c_uint8 * (w.value * h.value * c.value)).from_address(p)).reshape(h.value, w.value, c.value).copy()
    L.stbi_image_free(p)
    return a


def write_image(L, path_base, img):
    """RGB -> binary PPM, RGBA -> PNG (stbi_write_png); returns the path, after checking that stbi_load reads the same bytes back."""
    h, w, c = img.shape
    img = np.ascontiguousarray(img)
    if c == 3:
        path = path_base + ".ppm"
        with open(path, "wb") as f:
            f.write(b"P6\n%d %d\n255\n" % (w, h) + img.tobytes())
    else:
        path = path_base + ".png"
        assert L.stbi_write_png(path.encode(), w, h, c, img.ctypes.data, w * c)
    assert np.array_equal(stbi_load(L, path), img), path
    return path


def run_example(L, img, H, W, mean, scale, input_scale, zero_point, uint8, tmpdir):
    """The example's get_input_*_data on `img` written to a file: the [3, H, W] bytes it fills the input tensor with."""
    path = write_image(L, os.path.join(tmpdir, "img"), img)
    out = np.zeros((3, H, W), np.uint8 if uint8 else np.int8)
    m, s = (C.c_float * 3)(*mean), (C.c_float * 3)(*scale)
    if uint8:
        L.get_input_uint8_data(path.encode(), out.ctypes.data, H, W, m, s, input_scale, zero_point)
    else:
        L.get_input_int8_data(path.encode(), out.ctypes.data, H, W, m, s, input_scale)
    return out


def random_image(rng, h, w, c=3):
    return rng.integers(0, 256, (h, w, c), dtype=np.uint8)


# name, (h, w, c) of the source or "jpg", (H, W), mean, scale, input scale, zero point, uint8
CASES = [
    ("upsample_int8", (17, 31, 3), (48, 64), DEFAULT_MEAN, DEFAULT_SCALE, 0.0215, 0, False),
    ("downsample_uint8_zp128", (75, 100, 3), (30, 40), DEFAULT_MEAN, DEFAULT_SCALE, 0.0195, 128, True),
    ("same_size_int8", (30, 40, 3), (30, 40), (120.0, 110.5, 100.25), (0.02, 0.018, 0.021), 0.0215, 0, False),
    ("w2_uint8_zp3", (9, 2, 3), (12, 8), DEFAULT_MEAN, DEFAULT_SCALE, 0.019, 3, True),
    ("h2_int8", (2, 13, 3), (16, 5), DEFAULT_MEAN, DEFAULT_SCALE, 0.0215, 0, False),
    ("rgba_uint8_zp0", (23, 37, 4), (32, 24), (10.0, 20.0, 30.0), (0.01, 0.012, 0.014), 0.0125, 0, True),
    ("rgba_int8", (40, 29, 4), (21, 33), DEFAULT_MEAN, DEFAULT_SCALE, 0.0215, 0, False),
    ("jpg_224_int8", "jpg", (224, 224), DEFAULT_MEAN, DEFAULT_SCALE, 0.0215, 0, False),
    ("ties_int8", (20, 27, 3), (36, 50), (0.0, 0.0, 0.0), (1.0, 1.0, 1.0), 2.0, 0, False),
    ("ties_uint8_zp3", (27, 20, 3), (50, 36), (0.0, 0.0, 0.0), (1.0, 1.0, 1.0), 2.0, 3, True),
    ("saturating_int8", (33, 45, 3), (32, 32), DEFAULT_MEAN, (0.05, 0.05, 0.05), 0.01, 0, False),
    ("saturating_uint8_zp128", (45, 33, 3), (32, 32), DEFAULT_MEAN, (0.05, 0.05, 0.05), 0.01, 128, True),
    ("tiny_scale_int8", (16, 16, 3), (24, 20), DEFAULT_MEAN, DEFAULT_SCALE, 1e-12, 0, False),
    ("tiny_scale_uint8_zp128", (16, 16, 3), (20, 24), DEFAULT_MEAN, DEFAULT_SCALE, 1e-12, 128, True),
]


def case_image(L, k, src):
    if src == "jpg":
        return stbi_load(L, REF_JPG)
    return random_image(np.random.default_rng(100 + k), *src)


if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "image_pre_example.npz")
    L = example_lib()
    d = {"names": np.array([c[0] for c in CASES])}
    with tempfile.TemporaryDirectory() as tmp:
        for k, (name, src, (H, W), mean, scale, s_in, zp, u8) in enumerate(CASES):
            img = case_image(L, k, src)
            d[f"pix_{k}"] = img
            d[f"hw_{k}"] = np.array([H, W], np.int32)
            d[f"mean_{k}"] = np.array(mean, np.float32)
            d[f"scale_{k}"] = np.array(scale, np.float32)
            d[f"quant_{k}"] = np.array([np.float32(s_in), zp, int(u8)], np.float64)  # tensor scale (a float32 value), zero point, uint8
            d[f"out_{k}"] = run_example(L, img, H, W, mean, scale, np.float32(s_in), zp, u8, tmp)
    np.savez_compressed(out, **d)
    print("wrote", out, os.path.getsize(out), "bytes")
