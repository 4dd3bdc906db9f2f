"""CPU restatement of the quantised detection preprocessing of the YOLO examples and of their box back-mapping (TEST INFRASTRUCTURE;
checker of tb200_graph_upload_detect_images and tb200_detections_to_source).

Two families, both after cv::imread(file, 1) + cv::cvtColor(BGR2RGB), so the planes are R, G, B:
- stretch: examples/tm_yolov3_tiny_uint8.cpp:136-170 (tm_yolov4_tiny_uint8.cpp:137-170 is the same): cv::resize to the input's W x H,
  convertTo(CV_32FC3), (v - mean[c]) * scale[c], then round(x / s_in + (float)zp) clamped to 0..255 (:164-168).
- letterbox: examples/tm_yolov5s.cpp:263-337 (get_input_data_focus) and :339-392 (get_input_data_nofocus): a float scale chosen by a
  double comparison (:277-284), int(scale * cols) (:285-286, a float product truncated), cv::resize, borders top = (rows - rh) / 2,
  bot = (rows - rh + 1) / 2 (:292-295), cv::copyMakeBorder with Scalar(0, 0, 0) (:297).  copyMakeBorder creates its destination with
  the source's type (8UC3), so the grey CV_32FC3 img_new of :291 is discarded and the border is byte 0 before normalisation.  Focus
  (:317-337): output group i * 2 + g takes column offset i and row offset g.  The example itself is fp32; its input is quantised as
  every quantised example does it: round(x / s_in + (float)zp) clamped to +-127 (tm_yolox_int8.cpp:336-341) or 0..255.

cv::resize (INTER_LINEAR, 8-bit) is restated from OpenCV's resize.cpp as the cv2 binding computes it: per axis the double position
(dx + 0.5) * (1. / ((double)dst / src)) - 0.5 rounded to float, cvFloor, 11-bit weights saturate_cast<short>(w * 2048) (round half to
even).  Horizontally a position before the first pixel or at / after the last is clamped to it with weight 1; VERTICALLY IT IS NOT: the
row index is clipped instead, so the first and last rows of an upscale blend a row with itself under weights (1 - fy, fy).  The
vertical pass is the SIMD one, ((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2, whose two truncations make those rows
differ from the row by 1 LSB.  OpenCV sends an exact 2x downscale on both axes to INTER_AREA, whose (a + b + c + d + 2) >> 2 the
formula above also gives there (weights 1024 / 1024), so one formula covers it.  Same size is a copy, which the formula reproduces.

The back-mapping is inline in the examples' main() and is restated line by line: stretch tm_yolov3_tiny_uint8.cpp:501-532, letterbox
tm_yolov5s.cpp:580-625 (ratio_x = img.rows / resize_rows is applied to x: the example's swap, kept).

PINNED: tests/test_detect_pre_pinned.py compares this file with a fixture made with the cv2 binding (tests/golden/detect_pre_example.npz)
and, where cv2 is importable, with cv2.resize live on a seeded sweep of sizes.
"""
import numpy as np

from oracle.image_pre import round_to_int_x86

f32 = np.float32
STRETCH, LETTERBOX = 0, 1  # TB200_PRE_STRETCH, TB200_PRE_LETTERBOX
DEFAULT_MEAN = (0.0, 0.0, 0.0)                  # tm_yolov5s.cpp:399, tm_yolov3_tiny_uint8.cpp:313
DEFAULT_SCALE = (0.003921, 0.003921, 0.003921)  # :400, :314


def linear_coef(dst, src, clamp):
    """Source index and 11-bit weights of every output coordinate along one axis (cv::resize INTER_LINEAR, fixed point)."""
    scale = 1.0 / (float(dst) / float(src))
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(f32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(f32)).astype(f32)
    if clamp:
        low, high = s < 0, s >= src - 1
        s[low], f[low] = 0, f32(0)
        s[high], f[high] = src - 1, f32(0)
    c0 = np.rint(((f32(1) - f).astype(f32) * f32(2048)).astype(f32)).astype(np.int64)
    c1 = np.rint((f * f32(2048)).astype(f32)).astype(np.int64)
    return s, c0, c1


def cv_resize(img, W, H):
    """cv2.resize(img, (W, H)) of an HxWxC uint8 image (INTER_LINEAR)."""
    h, w, c = img.shape
    src = img.astype(np.int64)
    sx, cx0, cx1 = linear_coef(W, w, True)
    sy, cy0, cy1 = linear_coef(H, h, False)
    right = np.minimum(sx + 1, w - 1)
    hr = src[:, sx, :] * cx0[None, :, None] + src[:, right, :] * cx1[None, :, None]
    S0 = hr[np.clip(sy, 0, h - 1)]
    S1 = hr[np.clip(sy + 1, 0, h - 1)]
    v = (((cy0[:, None, None] * (S0 >> 4)) >> 16) + ((cy1[:, None, None] * (S1 >> 4)) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8)


def geometry(mode, src_w, src_h, W, H):
    """(src_w, src_h, resize_w, resize_h, left, top, scale) of tb200_detect_geometry, with the examples' arithmetic."""
    if mode == STRETCH:
        return (src_w, src_h, W, H, 0, 0, f32(0))
    # tm_yolov5s.cpp:277-286: compare in double, keep a float, multiply in float, truncate
    if (H * 1.0 / src_h) < (W * 1.0 / src_w):
        s = f32(H * 1.0 / src_h)
    else:
        s = f32(W * 1.0 / src_w)
    rw, rh = int(f32(s * f32(src_w))), int(f32(s * f32(src_h)))
    return (src_w, src_h, rw, rh, (W - rw) // 2, (H - rh) // 2, s)


def laid_out(img, mode, W, H):
    """The H x W x 3 bytes the example normalises: the resized RGB image, inside a byte-0 border for the letterbox."""
    rgb = img[:, :, :3]
    _, _, rw, rh, left, top, _ = geometry(mode, img.shape[1], img.shape[0], W, H)
    out = np.zeros((H, W, 3), np.uint8)
    out[top:top + rh, left:left + rw] = cv_resize(np.ascontiguousarray(rgb), rw, rh)
    return out


def quantise(v, mean, scale, input_scale, zero_point, uint8):
    """[3, ...] bytes -> (v - mean[c]) * scale[c], round(x / s_in + (float)zp), clamped to 0..255 or +-127."""
    m = np.array(mean, f32).reshape(3, *([1] * (v.ndim - 1)))
    s = np.array(scale, f32).reshape(3, *([1] * (v.ndim - 1)))
    with np.errstate(all="ignore"):
        f = ((v.astype(f32) - m) * s).astype(f32)
        q = ((f / f32(input_scale)).astype(f32) + f32(zero_point)).astype(f32)
    i = round_to_int_x86(q)
    return np.clip(i, 0, 255).astype(np.uint8) if uint8 else np.clip(i, -127, 127).astype(np.int8)


def focus(x):
    """[3, H, W] -> [12, H/2, W/2]: group i * 2 + g holds column offset i, row offset g (tm_yolov5s.cpp:318-336)."""
    _, H, W = x.shape
    return np.concatenate([x[:, g:2 * (H // 2):2, i:2 * (W // 2):2] for i in range(2) for g in range(2)], axis=0)


def preprocess(img, mode, H, W, mean, scale, input_scale, zero_point=0, uint8=False, use_focus=False):
    """One HxWxC (C = 3 or 4, RGB(A)) image to the graph input bytes: [3, H, W], or [12, H/2, W/2] with Focus."""
    q = quantise(laid_out(img, mode, W, H).transpose(2, 0, 1), mean, scale, input_scale, zero_point, uint8)
    return focus(q) if use_focus else q


def preprocess_batch(images, mode, H, W, mean, scale, input_scale, zero_point=0, uint8=False, use_focus=False):
    return np.stack([preprocess(a, mode, H, W, mean, scale, input_scale, zero_point, uint8, use_focus) for a in images])


def _min(a, b):  # std::min(a, b): (b < a) ? b : a
    return b if b < a else a


def _max(a, b):  # std::max(a, b): (a < b) ? b : a
    return b if a < b else a


def to_source(mode, geo, box):
    """One (x, y, w, h) box in network-input pixels -> source pixels, as the example's main() maps and clamps it."""
    src_w, src_h, rw, rh, left, top, _ = geo
    x0, y0 = f32(box[0]), f32(box[1])
    x1, y1 = f32(x0 + f32(box[2])), f32(y0 + f32(box[3]))
    if mode == STRETCH:
        # tm_yolov3_tiny_uint8.cpp:504-527: raw size over the network size
        ratio_x, ratio_y = f32(f32(src_w) / f32(rw)), f32(f32(src_h) / f32(rh))
        x0, y0, x1, y1 = f32(x0 * ratio_x), f32(y0 * ratio_y), f32(x1 * ratio_x), f32(y1 * ratio_y)
    else:
        # tm_yolov5s.cpp:594-615: tmp_w / tmp_h are the left / top borders; ratio_x = rows / resize_rows scales x (sic)
        ratio_x, ratio_y = f32(f32(src_h) / f32(rh)), f32(f32(src_w) / f32(rw))
        x0, y0 = f32(f32(x0 - f32(left)) * ratio_x), f32(f32(y0 - f32(top)) * ratio_y)
        x1, y1 = f32(f32(x1 - f32(left)) * ratio_x), f32(f32(y1 - f32(top)) * ratio_y)
    cx, cy = f32(src_w - 1), f32(src_h - 1)
    x0, y0 = _max(_min(x0, cx), f32(0)), _max(_min(y0, cy), f32(0))
    x1, y1 = _max(_min(x1, cx), f32(0)), _max(_min(y1, cy), f32(0))
    return (x0, y0, f32(x1 - x0), f32(y1 - y0))


def detections_to_source(mode, geos, boxes):
    """Per image a list of (x, y, w, h, prob, label) -> the same list with the boxes in source pixels."""
    return [[(*to_source(mode, g, b[:4]), b[4], b[5]) for b in img] for g, img in zip(geos, boxes)]
