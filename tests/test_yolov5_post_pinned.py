"""Pins oracle/yolov5_post.py -- the checker of tb200_graph_yolov5_detect (SURVEY.md 8(f)-4) -- against the detection
post-processing of the UNMODIFIED examples/tm_yolov5s.cpp: (a) the committed fixture tests/golden/yolov5_example_post.npz, produced
by the example's own functions (generator: tests/golden/make_golden_yolov5_post.py), everywhere; (b) the compiled example itself,
live, where oracle/_ref/libyolov5_example.so exists.  Box for box, bit for bit: coordinates, scores, labels, the quicksort's tie
order, NMS."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from oracle import yolo_post, yolov5_post  # noqa: E402

# graph outputs in stride order 8, 16, 32; the example proposes from stride 32 first (main():567-572)
HEADS = [(2, 32, yolov5_post.HEADS_BY_STRIDE[32]), (1, 16, yolov5_post.HEADS_BY_STRIDE[16]), (0, 8, yolov5_post.HEADS_BY_STRIDE[8])]


def _restatement(heads, scales, zeros):
    got = yolov5_post.detect(heads, [np.float32(s) for s in scales], [int(z) for z in zeros], HEADS, 80, 0.25, 0.45)[0]
    return np.array(got, np.float32).reshape(-1, 6)


def test_restatement_equals_the_committed_output_of_the_unmodified_example():
    import make_golden_yolov5_post as gen

    d = np.load(os.path.join(ROOT, "tests", "golden", "yolov5_example_post.npz"))
    dtypes = set()
    for k in range(len(gen.CASES)):
        heads = [d[f"q{s}_{k}"] for s in gen.STRIDES]
        qp = d[f"qp_{k}"]
        want = d[f"boxes_{k}"]
        got = _restatement(heads, qp[:3], qp[3:])
        assert len(want) > 100 and got.shape == want.shape, (k, got.shape, want.shape)
        assert np.array_equal(got, want), k
        dtypes.add(heads[0].dtype)
    assert dtypes == {np.dtype(np.uint8), np.dtype(np.int8)}


def test_the_examples_sigmoid_is_the_float_expf_form():
    """tm_yolov5s.cpp:50-53 resolves exp(-x) to the float overload, as the YOLOv3-tiny example does: the restatement's and the device
    table's float-expf sigmoid reproduce its output bit for bit, where a double exp would not."""
    d = np.load(os.path.join(ROOT, "tests", "golden", "yolov5_example_post.npz"))
    got = np.array([yolo_post._sigmoid(x) for x in d["sigmoid_x"]], np.float32)
    assert np.array_equal(got, d["sigmoid_y"])
    via_double = np.array([np.float32(1.0 / (1.0 + np.exp(-np.float64(x)))) for x in d["sigmoid_x"]], np.float32)
    assert not np.array_equal(via_double, d["sigmoid_y"])


def test_restatement_equals_the_compiled_example_live():
    import make_golden_yolov5_post as gen

    if not os.path.exists(gen.LIB):
        pytest.skip("oracle/_ref/libyolov5_example.so absent (built by oracle/build_yolov5_example.py where the reference tree exists)")
    L = gen.example_lib()
    for seed, int8 in ((31, False), (32, True)):
        heads, scales, zeros = gen.random_heads(seed, int8)
        want = gen.run_example(L, heads, scales, zeros)
        got = _restatement(heads, scales, zeros)
        assert len(want) > 100 and got.shape == want.shape and np.array_equal(got, want), seed
