#!/usr/bin/env python3
"""Golden vectors for oracle/topk.py: the ranking step of the UNMODIFIED classification examples -- print_topk's array after its own
sort_cls_score (examples/common/tengine_operations.c, compiled by oracle/build_topk_example.py into oracle/_ref/libtopk_example.so
through oracle/topk_example_shim.c) -- on quantised outputs dequantised as examples/tm_classification_int8.c / _uint8.c do.  Needs the
reference tree at build time; the .npz it writes is committed so that the pin holds anywhere.
usage: make_golden_topk.py [out.npz]"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
LIB = os.path.join(ROOT, "oracle", "_ref", "libtopk_example.so")


def example_lib():
    L = C.CDLL(LIB)
    L.topk_example_sorted.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return L


def run_example(L, scores):
    """(scores [E] float32, ids [E] int32): the whole array print_topk holds after the example's sort of `scores`."""
    data = np.ascontiguousarray(scores, np.float32)
    ids, out = np.empty(data.size, np.int32), np.empty(data.size, np.float32)
    assert L.topk_example_sorted(data.ctypes.data, data.size, ids.ctypes.data, out.ctypes.data) == 0
    return out, ids


def _softmax_like(rng, e, background, peaks):
    """Mostly `background`, `peaks` = [(byte, how many classes share it)] at seeded positions."""
    q = np.full(e, background, np.int64)
    pos = rng.permutation(e)[:sum(n for _, n in peaks)]
    at = 0
    for v, n in peaks:
        q[pos[at:at + n]] = v
        at += n
    return q


def cases():
    """[(name, class bytes [E] int8 / uint8, scale, zero point, uint8)]"""
    rng = np.random.default_rng(20241016)
    i8 = lambda a: np.asarray(a).astype(np.int8)
    u8 = lambda a: np.asarray(a).astype(np.uint8)
    out = [
        ("all_equal_int8", i8(np.full(1000, -7)), 0.00390625, 0, False),
        ("all_equal_uint8_zp3", u8(np.full(1000, 3)), 0.00390625, 3, True),
        ("two_values_int8", i8(rng.integers(0, 2, 1000) * 50 - 20), 0.02, 0, False),
        ("two_values_uint8_zp128", u8(rng.integers(0, 2, 1001) * 7 + 125), 0.05, 128, True),
        ("ascending_int8", i8(np.arange(-127, 128)), 0.1, 0, False),
        ("descending_int8", i8(np.arange(127, -128, -1)), 0.1, 0, False),
        ("ascending_uint8_zp0", u8(np.arange(256)), 0.00390625, 0, True),
        ("descending_uint8_zp128", u8(np.arange(255, -1, -1)), 0.03, 128, True),
        # a Softmax node's output: 1 / 256 per step, nearly every class at probability 0
        ("softmax_like_int8", i8(_softmax_like(rng, 1000, 0, [(90, 1), (14, 3), (3, 2), (1, 9)])), 0.0078125, 0, False),
        ("softmax_like_uint8_zp0", u8(_softmax_like(rng, 1000, 0, [(120, 2), (5, 4), (1, 12)])), 0.00390625, 0, True),
        ("softmax_like_flat_int8", i8(_softmax_like(rng, 1000, 0, [(1, 40)])), 0.0078125, 0, False),
        ("random_int8", i8(rng.integers(-127, 128, 1000)), 0.0471, 0, False),
        ("random_int8_1001", i8(rng.integers(-128, 128, 1001)), 0.0471, 0, False),
        ("random_uint8_zp0", u8(rng.integers(0, 256, 1000)), 0.0213, 0, True),
        ("random_uint8_zp3", u8(rng.integers(0, 256, 1000)), 0.0213, 3, True),
        ("random_uint8_zp128", u8(rng.integers(0, 256, 1001)), 0.0213, 128, True),
        ("narrow_random_int8", i8(rng.integers(-3, 4, 1000)), 0.11, 0, False),
        ("e1_int8", i8([-5]), 0.5, 0, False),
        ("e2_int8", i8([-5, 9]), 0.5, 0, False),
        ("e2_equal_uint8", u8([9, 9]), 0.5, 4, True),
        ("e5_uint8_zp3", u8([3, 200, 3, 7, 200]), 0.25, 3, True),
        ("e33_int8", i8(rng.integers(-4, 5, 33)), 0.3, 0, False),
        # 1e-46 is below the smallest float: the tensor's scale is 0 and every score +0 or -0, all equal
        ("underflowing_scale_int8", i8(rng.integers(-127, 128, 1000)), 1e-46, 0, False),
        # (float)q - 2^25 keeps multiples of 4 only: distinct bytes, equal floats
        ("coarse_zero_point_uint8", u8(rng.integers(0, 256, 1000)), 0.001, 1 << 25, True),
        ("overflowing_scale_int8", i8(rng.integers(-3, 4, 200)), 3e38, 0, False),
        ("negative_scale_int8", i8(rng.integers(-127, 128, 1000)), -0.0471, 0, False),
        ("negative_scale_uint8_zp128", u8(rng.integers(0, 256, 1000)), -0.0213, 128, True),
    ]
    return out


if __name__ == "__main__":
    from oracle import topk

    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "topk_example.npz")
    L = example_lib()
    cs = cases()
    d = {"names": np.array([c[0] for c in cs])}
    for k, (name, q, scale, zp, u8) in enumerate(cs):
        d[f"q_{k}"] = q
        d[f"quant_{k}"] = np.array([np.float32(scale), zp, int(u8)], np.float64)  # tensor scale (a float32 value), zero point, uint8
        d[f"scores_{k}"], d[f"ids_{k}"] = run_example(L, topk.dequantise(q, np.float32(scale), zp, u8))
    np.savez_compressed(out, **d)
    print("wrote", out, os.path.getsize(out), "bytes")
