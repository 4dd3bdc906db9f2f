#!/usr/bin/env python3
"""Golden vectors for oracle/yolov5_post.py: the detection post-processing of the UNMODIFIED examples/tm_yolov5s.cpp (compiled by
oracle/build_yolov5_example.py into oracle/_ref/libyolov5_example.so through oracle/yolov5_example_shim.cpp), run on seeded
quantised head tensors.  Needs the reference tree at build time; the .npz it writes is committed so that the pin holds anywhere.
usage: make_golden_yolov5_post.py [out.npz]"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(ROOT, "oracle", "_ref", "libyolov5_example.so")
RES = 192           # network input: heads of 6x6, 12x12 and 24x24 cells
PROB, NMS = 0.25, 0.45  # the example's thresholds (main():558-559)
STRIDES = (8, 16, 32)   # graph output order: head 0 has stride 8


def example_lib():
    L = C.CDLL(LIB)
    L.yolov5_example_postprocess.restype = C.c_int
    L.yolov5_example_postprocess.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_int]
    L.yolov5_example_sigmoid.restype = C.c_float
    L.yolov5_example_sigmoid.argtypes = [C.c_float]
    return L


def random_heads(seed, int8=False, res=RES):
    """Quantised head tensors [1, 255, res/s, res/s] for s = 8, 16, 32, with per-head scales and zero points (int8: zero point 0).
    Objectness is shifted low, so that a few hundred proposals pass the example's 0.25 with plenty of overlaps for the NMS and
    equal scores for the sort's tie order.  Returns (heads, scales, zeros)."""
    rng = np.random.default_rng(seed)
    heads, scales, zeros = [], [], []
    for s in STRIDES:
        sc = np.float32(rng.uniform(0.05, 0.2))
        z = 0 if int8 else int(rng.integers(100, 180))
        lo, hi = (-128, 128) if int8 else (0, 256)
        q = rng.integers(lo, hi, (1, 255, res // s, res // s))
        for a in range(3):
            q[0, a * 85 + 4] = np.clip(rng.normal(z - 40, 25, q[0, a * 85 + 4].shape), lo, hi - 1)
        heads.append(q.astype(np.int8 if int8 else np.uint8))
        scales.append(sc)
        zeros.append(z)
    return heads, scales, zeros


def run_example(L, heads, scales, zeros, prob=PROB, nms=NMS):
    """The example's feat[a][h][w][k] (tm_yolov5s.cpp:167) is channel a * 85 + k of the raw head at (h, w)."""
    feats = []
    for q, s, z in zip(heads, scales, zeros):
        _, c, h, w = q.shape
        x = ((q[0].astype(np.float32) - np.float32(z)) * np.float32(s)).astype(np.float32)
        feats.append(np.ascontiguousarray(x.reshape(3, c // 3, h, w).transpose(0, 2, 3, 1)))
    rows, cols = heads[0].shape[2] * STRIDES[0], heads[0].shape[3] * STRIDES[0]
    out = np.zeros((16384, 6), np.float32)
    n = L.yolov5_example_postprocess(feats[0].ctypes.data, feats[1].ctypes.data, feats[2].ctypes.data, rows, cols, prob, nms, out.ctypes.data, len(out))
    assert 0 <= n <= len(out)
    return out[:n].copy()


CASES = ((21, False), (22, False), (23, True))  # (seed, int8)

if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "yolov5_example_post.npz")
    L = example_lib()
    d = {}
    for k, (seed, int8) in enumerate(CASES):
        heads, scales, zeros = random_heads(seed, int8)
        for s, q in zip(STRIDES, heads):
            d[f"q{s}_{k}"] = q
        d[f"qp_{k}"] = np.array(scales + zeros, np.float64)  # three scales, then three zero points, in STRIDES order
        d[f"boxes_{k}"] = run_example(L, heads, scales, zeros)
    xs = ((np.arange(256) - 128.0) * 0.137).astype(np.float32)
    d["sigmoid_x"] = xs
    d["sigmoid_y"] = np.array([L.yolov5_example_sigmoid(float(x)) for x in xs], np.float32)
    np.savez_compressed(out, **d)
    print("wrote", out, {k: v.shape for k, v in d.items() if k.startswith("boxes")})
