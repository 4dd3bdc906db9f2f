#!/usr/bin/env python3
"""Golden vectors for oracle/detect_pre.py: the quantised detection preprocessing of the YOLO examples with OpenCV's own cv::resize and
cv::copyMakeBorder (the cv2 binding), and their box back-mapping.

The application code around OpenCV is transcribed here on its own, index formula for index formula, independent of
oracle/detect_pre.py: examples/tm_yolov3_tiny_uint8.cpp:136-170 (stretch), examples/tm_yolov5s.cpp:263-337 / :339-392 (letterbox, with
and without Focus) quantised as tm_yolox_int8.cpp:336-341 / tm_yolov3_tiny_uint8.cpp:164-168, and the back-mapping of
tm_yolov3_tiny_uint8.cpp:501-532 / tm_yolov5s.cpp:580-625.  The caller's RGB(A) image stands for the example's imread + BGR2RGB
result (an RGBA file read with flag 1 loses its alpha).  Needs cv2 when it is run; the .npz it writes is committed so that the pin
holds anywhere.  usage: make_golden_detect_pre.py [out.npz]"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "detect_pre_example.npz")
f32 = np.float32
STRETCH, LETTERBOX = 0, 1
EX_MEAN, EX_SCALE = (0.0, 0.0, 0.0), (0.003921, 0.003921, 0.003921)  # tm_yolov5s.cpp:399-400

# name, source (w, h, c), mode, (H, W) of the laid-out image, focus, uint8, zero point, input scale, mean, scale (None: random)
CASES = [
    ("letterbox_up_focus_int8", (47, 33, 3), LETTERBOX, (64, 64), True, False, 0, 0.0079, None, None),
    ("letterbox_down_nofocus_uint8_zp128", (190, 110, 3), LETTERBOX, (96, 96), False, True, 128, 0.0075, None, None),
    ("letterbox_exact2x_focus_uint8_zp0", (128, 96, 3), LETTERBOX, (64, 64), True, True, 0, 0.0041, EX_MEAN, EX_SCALE),
    ("letterbox_portrait_focus_int8", (90, 200, 3), LETTERBOX, (64, 64), True, False, 0, 0.0081, None, None),
    ("letterbox_landscape_nofocus_int8", (200, 90, 4), LETTERBOX, (64, 64), False, False, 0, 0.0081, EX_MEAN, EX_SCALE),
    ("letterbox_truncated_width_focus_uint8_zp128", (82, 60, 3), LETTERBOX, (64, 64), True, True, 128, 0.0078, None, None),
    ("letterbox_not_square_focus_int8", (120, 100, 3), LETTERBOX, (48, 80), True, False, 0, 0.0079, None, None),
    ("letterbox_w2_nofocus_uint8_zp0", (2, 30, 3), LETTERBOX, (32, 32), False, True, 0, 0.0040, EX_MEAN, EX_SCALE),
    ("letterbox_ties_int8", (40, 25, 3), LETTERBOX, (48, 48), False, False, 0, 2.0, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0)),
    ("stretch_up_uint8_zp0", (47, 33, 3), STRETCH, (64, 80), False, True, 0, 0.0040, EX_MEAN, EX_SCALE),
    ("stretch_down_uint8_zp128", (150, 90, 4), STRETCH, (64, 64), False, True, 128, 0.0080, None, None),
    ("stretch_h2_int8", (50, 2, 3), STRETCH, (32, 48), False, False, 0, 0.0079, EX_MEAN, EX_SCALE),
    ("stretch_w2_up_uint8_zp0", (2, 2, 3), STRETCH, (7, 9), False, True, 0, 0.0040, EX_MEAN, EX_SCALE),
    ("stretch_exact2x_focus_int8", (96, 64, 3), STRETCH, (32, 48), True, False, 0, 0.0079, None, None),
    ("stretch_ties_uint8_zp3", (33, 20, 3), STRETCH, (40, 24), False, True, 3, 2.0, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0)),
]


def _round_int(q):
    """(int)round(q) of the x86-64 build: halfway cases away from zero; out of int's range or NaN -> INT_MIN."""
    d = q.astype(np.float64)
    with np.errstate(invalid="ignore"):
        r = np.where(d >= 0, np.floor(d + 0.5), np.ceil(d - 0.5))
        ok = (r >= -2.0 ** 31) & (r < 2.0 ** 31)
    return np.where(ok, np.nan_to_num(r), -2 ** 31).astype(np.int64)


def letterbox_geometry(rows, cols, img_rows, img_cols):
    """tm_yolov5s.cpp:274-295."""
    if (rows * 1.0 / img_rows) < (cols * 1.0 / img_cols):
        scale_letterbox = f32(rows * 1.0 / img_rows)
    else:
        scale_letterbox = f32(cols * 1.0 / img_cols)
    resize_cols = int(f32(scale_letterbox * f32(img_cols)))
    resize_rows = int(f32(scale_letterbox * f32(img_rows)))
    top, bot = (rows - resize_rows) // 2, (rows - resize_rows + 1) // 2
    left, right = (cols - resize_cols) // 2, (cols - resize_cols + 1) // 2
    return scale_letterbox, resize_cols, resize_rows, top, bot, left, right


def example_input(cv2, img, mode, rows, cols, mean, scale, s_in, zp, u8, focus):
    """The bytes the example would put in the input tensor for image `img` (RGB(A), what imread + cvtColor(BGR2RGB) give)."""
    rgb = np.ascontiguousarray(img[:, :, :3])
    mean, scale = np.asarray(mean, f32), np.asarray(scale, f32)
    if mode == STRETCH:
        lay = cv2.resize(rgb, (cols, rows))  # cv::resize(img, img, cv::Size(img_w, img_h)), INTER_LINEAR
    else:
        _, rw, rh, top, bot, left, right = letterbox_geometry(rows, cols, img.shape[0], img.shape[1])
        r = cv2.resize(rgb, (rw, rh))
        # img_new is a grey CV_32FC3 Mat (:291); copyMakeBorder creates its destination with the source's type, so it is replaced
        grey = np.empty((cols, rows, 3), np.float32)
        grey[:] = [0.5 / scale[c] + mean[c] for c in range(3)]
        lay = cv2.copyMakeBorder(r, top, bot, left, right, cv2.BORDER_CONSTANT, dst=grey, value=(0, 0, 0))
        assert lay.dtype == np.uint8 and lay.shape == (rows, cols, 3), (lay.dtype, lay.shape)
    img_data = lay.astype(np.float32).reshape(-1)  # convertTo(CV_32FC3)
    h, w, c = np.meshgrid(np.arange(rows), np.arange(cols), np.arange(3), indexing="ij")
    temp = np.empty(3 * rows * cols, np.float32)
    temp[(c * rows * cols + h * cols + w).ravel()] = ((img_data[(h * cols * 3 + w * 3 + c).ravel()] - mean[c.ravel()]) * scale[c.ravel()]).astype(f32)
    if focus:  # tm_yolov5s.cpp:318-336
        data = np.empty(3 * rows * cols, np.float32)
        i, g, c, h, w = np.meshgrid(np.arange(2), np.arange(2), np.arange(3), np.arange(rows // 2), np.arange(cols // 2), indexing="ij")
        hw = (cols // 2) * (rows // 2)
        in_index = i + g * cols + c * cols * rows + h * 2 * cols + w * 2
        out_index = i * 2 * 3 * hw + g * 3 * hw + c * hw + h * (cols // 2) + w
        data[out_index.ravel()] = temp[in_index.ravel()]
        shape = (12, rows // 2, cols // 2)
    else:
        data, shape = temp, (3, rows, cols)
    with np.errstate(all="ignore"):
        q = _round_int((data / f32(s_in)).astype(f32) + f32(zp))
    q = np.clip(q, 0, 255).astype(np.uint8) if u8 else np.clip(q, -127, 127).astype(np.int8)
    return q.reshape(shape)


def map_boxes(mode, img_w, img_h, rows, cols, boxes):
    """Back-mapping of (x, y, w, h) float32 boxes, the examples' main() line by line."""
    out = []
    for bx, by, bw, bh in boxes:
        x0, y0 = f32(bx), f32(by)
        x1, y1 = f32(f32(bx) + f32(bw)), f32(f32(by) + f32(bh))
        if mode == STRETCH:  # tm_yolov3_tiny_uint8.cpp:501-522
            ratio_x, ratio_y = f32(f32(img_w) / f32(cols)), f32(f32(img_h) / f32(rows))
            x0, y0, x1, y1 = x0 * ratio_x, y0 * ratio_y, x1 * ratio_x, y1 * ratio_y
        else:  # tm_yolov5s.cpp:580-615
            _, resize_cols, resize_rows, _, _, _, _ = letterbox_geometry(rows, cols, img_h, img_w)
            tmp_h, tmp_w = (rows - resize_rows) // 2, (cols - resize_cols) // 2
            ratio_x, ratio_y = f32(f32(img_h) / f32(resize_rows)), f32(f32(img_w) / f32(resize_cols))
            x0, y0 = f32(x0 - f32(tmp_w)) * ratio_x, f32(y0 - f32(tmp_h)) * ratio_y
            x1, y1 = f32(x1 - f32(tmp_w)) * ratio_x, f32(y1 - f32(tmp_h)) * ratio_y
        cw, ch = f32(img_w - 1), f32(img_h - 1)
        x0, y0 = max(min(f32(x0), cw), f32(0)), max(min(f32(y0), ch), f32(0))
        x1, y1 = max(min(f32(x1), cw), f32(0)), max(min(f32(y1), ch), f32(0))
        out.append((x0, y0, f32(x1 - x0), f32(y1 - y0)))
    return np.array(out, np.float32)


def random_boxes(rng, rows, cols, n=12):
    """Boxes in network-input pixels, some reaching into the border and past the edges (so the clamps act)."""
    x = rng.uniform(-0.2 * cols, 1.1 * cols, n).astype(f32)
    y = rng.uniform(-0.2 * rows, 1.1 * rows, n).astype(f32)
    return np.stack([x, y, rng.uniform(1, 0.6 * cols, n).astype(f32), rng.uniform(1, 0.6 * rows, n).astype(f32)], 1).astype(f32)


def make(out=OUT):
    import cv2

    rng = np.random.default_rng(20261016)
    data = {"names": np.array([c[0] for c in CASES]), "cv2_version": np.array(cv2.__version__)}
    for k, (name, (w, h, c), mode, (H, W), focus, u8, zp, s_in, mean, scale) in enumerate(CASES):
        if "ties" in name:  # every odd byte / 2 is an exact .5
            img = rng.integers(0, 128 if not u8 else 256, (h, w, c), dtype=np.uint8)
        else:
            img = rng.integers(0, 256, (h, w, c), dtype=np.uint8)
        mean = np.asarray(mean if mean is not None else rng.uniform(0, 80, 3), np.float32)
        scale = np.asarray(scale if scale is not None else rng.uniform(0.003, 0.006, 3), np.float32)
        data[f"pix_{k}"] = img
        data[f"cfg_{k}"] = np.array([mode, H, W, int(focus), int(u8), zp], np.int64)
        data[f"sin_{k}"] = np.float32(s_in)
        data[f"mean_{k}"], data[f"scale_{k}"] = mean, scale
        data[f"out_{k}"] = example_input(cv2, img, mode, H, W, mean, scale, np.float32(s_in), zp, u8, focus)
        boxes = random_boxes(rng, H, W)
        data[f"boxes_{k}"], data[f"mapped_{k}"] = boxes, map_boxes(mode, w, h, H, W, boxes)
    np.savez_compressed(out, **data)
    return out


if __name__ == "__main__":
    print(make(sys.argv[1] if len(sys.argv) > 1 else OUT))
