"""CPU restatement of the input preprocessing of examples/tm_classification_int8.c / _uint8.c (TEST INFRASTRUCTURE; checker of
tb200_graph_upload_images): get_input_int8_data / get_input_uint8_data (:43-62) and what they call in
examples/common/tengine_operations.c -- load_image_stb (:51-82, RGBA loses its alpha byte), rgb2bgr_permute (:651-673),
tengine_resize_f32 (:870-979, the non-NEON branch), imread2caffe (:101-115).  Float steps in float32, the resize in int32 with
arithmetic shifts, round() (halfway cases away from zero) in float64 on the float32 quotient, and the x86-64 double -> int conversion
that turns anything outside int's range, or NaN, into INT_MIN before the clamp.

PINNED: tests/test_image_pre_pinned.py compares this file, byte for byte, with the examples' own functions compiled from the
unmodified sources (oracle/image_example_shim.c, built into oracle/_ref/libimage_example.so) and with a committed fixture of their
output (tests/golden/image_pre_example.npz).
"""
import numpy as np

f32 = np.float32
INT_MIN = -(2 ** 31)
DEFAULT_MEAN = (104.007, 116.669, 122.679)  # tm_classification_int8.c:37-39, B, G, R
DEFAULT_SCALE = (0.017, 0.017, 0.017)      # :34-36


def resize_coef(out_n, in_n):
    """Source position and the two 11-bit weights of every output coordinate along one axis (tengine_resize_f32 :872-920)."""
    scale = f32(f32(in_n) / f32(out_n))
    f = ((np.arange(out_n, dtype=f32) + f32(0.5)) * scale - f32(0.5)).astype(f32)
    s = np.trunc(f).astype(np.int32)  # (int)fx: toward zero, so the first outputs of an upsample keep s = 0 and a negative fx
    f = (f - s.astype(f32)).astype(f32)
    low, high = s < 0, s >= in_n - 1
    s[low], f[low] = 0, f32(0)
    s[high], f[high] = in_n - 2, f32(0)
    c1 = (f * f32(2048)).astype(np.int32).astype(np.int16).astype(np.int32)  # int16_t xCoef = fx * 2048 (truncation)
    c0 = ((f32(1) - f) * f32(2048)).astype(np.int32).astype(np.int16).astype(np.int32)
    return s, c0, c1


def round_to_int_x86(x):
    """(int)round((double)x) as the examples compile on x86-64: halfway cases away from zero; out of int's range or NaN -> INT_MIN."""
    d = np.asarray(x, np.float64)
    with np.errstate(invalid="ignore"):
        r = np.where(d >= 0, np.floor(d + 0.5), np.ceil(d - 0.5))
        ok = (r >= -2.0 ** 31) & (r < 2.0 ** 31)
    return np.where(ok, np.nan_to_num(r), INT_MIN).astype(np.int64)


def resize_bgr(img, H, W):
    """HxWxC (C = 3 or 4) uint8 RGB(A) -> [3, H, W] int32 BGR planes of the fixed-point resize (tengine_resize_f32 :937-972)."""
    h, w, _ = img.shape
    sx, cx0, cx1 = resize_coef(W, w)
    sy, cy0, cy1 = resize_coef(H, h)
    out = np.empty((3, H, W), np.int32)
    for k in range(3):
        p = img[:, :, 2 - k].astype(np.int32)
        r0, r1 = p[sy], p[sy + 1]
        u = (r0[:, sx] * cx0 >> 11) + (r0[:, sx + 1] * cx1 >> 11)
        d = (r1[:, sx] * cx0 >> 11) + (r1[:, sx + 1] * cx1 >> 11)
        out[k] = (u * cy0[:, None] + d * cy1[:, None]) >> 11
    return out


def preprocess(img, H, W, mean, scale, input_scale, zero_point=0, uint8=False):
    """One image to the [3, H, W] int8 (or uint8) bytes get_input_int8_data (get_input_uint8_data) would write."""
    v = resize_bgr(img, H, W)
    m = np.array(mean, f32).reshape(3, 1, 1)
    s = np.array(scale, f32).reshape(3, 1, 1)
    with np.errstate(all="ignore"):
        f = ((v.astype(f32) - m) * s).astype(f32)
        q = (f / f32(input_scale)).astype(f32)
        if uint8:
            q = (q + f32(zero_point)).astype(f32)
    i = round_to_int_x86(q)
    return np.clip(i, 0, 255).astype(np.uint8) if uint8 else np.clip(i, -127, 127).astype(np.int8)


def preprocess_batch(images, H, W, mean, scale, input_scale, zero_point=0, uint8=False):
    return np.stack([preprocess(a, H, W, mean, scale, input_scale, zero_point, uint8) for a in images])
