"""Detection post-processing on the device (SURVEY.md 8(f)-4): tb200_graph_yolov5_detect and tb200_graph_yolo_detect, which share
one decode kernel and differ only in the box formula.

- Identity graphs (each graph input passes through IDENTITY to an output) give the tests full control of the head bytes: the
  committed outputs of the unmodified examples (tests/golden/yolov5_example_post.npz, yolo_example_post.npz) are reproduced box
  for box and bit for bit, and heads with other class counts (other row paddings) are checked against the CPU restatements.
- Real YOLOv5s graphs, int8 and uint8, on one and two shards: the boxes equal the restatement (oracle/yolov5_post.py,
  oracle/yolo_post.py) run on the head tensors the graph downloaded.
- Errors: candidate overflow raises, a head whose channel count does not match the class count is TB200_ERR_INVALID."""
import os
import sys

import numpy as np
import pytest

from oracle import yolo_post, yolov5_post
from tengine_b200 import abi, workloads

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
V3_ANCHORS = [10, 14, 23, 27, 37, 58, 81, 82, 135, 169, 344, 319]  # tm_yolov3_tiny_uint8.cpp:178
# graph outputs in stride order 8, 16, 32; the YOLOv5 example proposes from stride 32 first (main():567-572)
V5_HEADS = [(2, 32, yolov5_post.HEADS_BY_STRIDE[32]), (1, 16, yolov5_post.HEADS_BY_STRIDE[16]), (0, 8, yolov5_post.HEADS_BY_STRIDE[8])]


def _devices(n):
    from tengine_b200 import runtime as rt

    have = rt.device_count()
    return [i % have for i in range(n)]


def _identity_graph(heads, scales, zeros):
    """One graph input per head, [N, C, H, W] with the head's quantisation, passed through IDENTITY to a graph output."""
    from tengine_b200.graphdef import GraphDef

    g = GraphDef(abi.DT_INT8 if heads[0].dtype == np.int8 else abi.DT_UINT8)
    for q, s, z in zip(heads, scales, zeros):
        g.mark_output(g.identity(g.input(*q.shape, float(np.float32(s)), int(z))))
    return g


def _detect_on_device(ctx, heads, scales, zeros, det_heads, version, num_classes, prob, nms, **kw):
    from tengine_b200 import runtime as rt

    gr = rt.Graph(ctx, _identity_graph(heads, scales, zeros))
    try:
        outs = gr.run(heads)
        for o, q in zip(outs, heads):
            assert np.array_equal(o, q)
        return gr.yolo_detect(det_heads, num_classes=num_classes, prob_threshold=prob, nms_threshold=nms, version=version, **kw)
    finally:
        gr.close()


def _as_rows(boxes):
    return np.array(boxes, np.float32).reshape(-1, 6)


def _assert_same(got, want):
    assert len(got) == len(want)
    for i, (gd, wd) in enumerate(zip(got, want)):
        g, w = _as_rows(gd), _as_rows(wd)
        assert g.shape == w.shape, (i, g.shape, w.shape)
        assert np.array_equal(g, w), (i, np.argwhere(g != w)[:4])


@pytest.mark.parametrize("k", [0, 1, 2])
def test_yolov5_detect_equals_the_examples_committed_output(ctx, k):
    import make_golden_yolov5_post as gen

    d = np.load(os.path.join(ROOT, "tests", "golden", "yolov5_example_post.npz"))
    heads = [d[f"q{s}_{k}"] for s in gen.STRIDES]
    qp = d[f"qp_{k}"]
    got = _detect_on_device(ctx, heads, qp[:3], qp[3:], V5_HEADS, 5, 80, gen.PROB, gen.NMS, max_per_image=1024)
    want = d[f"boxes_{k}"]
    assert len(want) > 100
    assert np.array_equal(_as_rows(got[0]), want)


@pytest.mark.parametrize("k", [0, 1, 2])
def test_yolo_detect_equals_the_yolov3_examples_committed_output(ctx, k):
    d = np.load(os.path.join(ROOT, "tests", "golden", "yolo_example_post.npz"))
    s32, z32, s16, z16 = d[f"qp_{k}"]
    heads = [d[f"q32_{k}"], d[f"q16_{k}"]]
    got = _detect_on_device(ctx, heads, [s32, s16], [z32, z16], [(0, 32, V3_ANCHORS[6:12]), (1, 16, V3_ANCHORS[0:6])], 3, 80, 0.4, 0.25,
                            max_per_image=1024)
    want = d[f"boxes_{k}"]
    assert len(want) > 100
    assert np.array_equal(_as_rows(got[0]), want)


def _random_heads(rng, num_classes, int8, batch, sizes):
    per = num_classes + 5
    lo, hi = (-128, 128) if int8 else (0, 256)
    heads, scales, zeros = [], [], []
    for hw in sizes:
        z = 0 if int8 else int(rng.integers(100, 180))
        q = rng.integers(lo, hi, (batch, 3 * per, hw, hw))
        for a in range(3):
            q[:, a * per + 4] = np.clip(rng.normal(z - 40, 25, q[:, a * per + 4].shape), lo, hi - 1)
        heads.append(q.astype(np.int8 if int8 else np.uint8))
        scales.append(np.float32(rng.uniform(0.05, 0.2)))
        zeros.append(z)
    return heads, scales, zeros


@pytest.mark.parametrize("version", [3, 5])
@pytest.mark.parametrize("num_classes,int8", [(20, False), (20, True), (1, False), (300, True)])
def test_other_class_counts(ctx, version, num_classes, int8):
    """20 classes: 75 channels in rows of 80 bytes (5 lanes per cell); 1 class: 16-byte chunks span three anchors; 300 classes:
    rows of 928 bytes, more chunks than a warp has lanes."""
    rng = np.random.default_rng(num_classes * 2 + int8 + 10 * version)
    heads, scales, zeros = _random_heads(rng, num_classes, int8, 2, (7, 14, 28))
    det_heads = V5_HEADS if version == 5 else [(2, 32, V3_ANCHORS[6:12]), (1, 16, V3_ANCHORS[0:6]), (0, 8, V3_ANCHORS[0:6])]
    post = yolov5_post if version == 5 else yolo_post
    prob = 0.35 if num_classes > 1 else 0.2
    got = _detect_on_device(ctx, heads, scales, zeros, det_heads, version, num_classes, prob, 0.45, max_per_image=1024)
    want = post.detect(heads, scales, zeros, det_heads, num_classes, prob, 0.45)
    assert min(len(w) for w in want) > 20, [len(w) for w in want]
    _assert_same(got, want)


def _scores(outs, scales, zeros, num_classes):
    """Per image, every anchor's sigmoid(obj) * sigmoid(best class), through the same per-byte table as the device."""
    per, res = num_classes + 5, []
    for q, s, z in zip(outs, scales, zeros):
        b = np.arange(256)
        x = ((b.astype(np.float32) if q.dtype == np.uint8 else b.astype(np.uint8).view(np.int8).astype(np.float32)) - np.float32(z)) * np.float32(s)
        sig = np.array([yolo_post._sigmoid(v) for v in x.astype(np.float32)], np.float32)
        n, _, h, w = q.shape
        r = q.reshape(n, 3, per, h, w).view(np.uint8)
        obj = sig[r[:, :, 4]]
        cls = np.take_along_axis(r[:, :, 5:], (q.reshape(n, 3, per, h, w)[:, :, 5:]).argmax(axis=2)[:, :, None], axis=2)[:, :, 0]
        res.append((obj * sig[cls]).reshape(n, -1))
    return np.concatenate(res, axis=1)


@pytest.mark.parametrize("gpus", [1, 2])
@pytest.mark.parametrize("dtype", [abi.DT_INT8, abi.DT_UINT8], ids=["int8", "uint8"])
def test_real_yolov5s_graph_equals_the_restatement(dtype, gpus):
    from tengine_b200 import runtime as rt

    g, b = workloads.yolov5s(dtype, batch=3, res=256, width=0.25, seed=7)
    x = b.random_input(4)
    scales = [np.float32(g.tensors[t]["scale"]) for t in g.outputs]
    zeros = [int(g.tensors[t]["zero_point"]) for t in g.outputs]
    c = rt.Context(devices=_devices(gpus)) if gpus > 1 else rt.Context(0)
    try:
        gr = rt.Graph(c, g)
        try:
            assert len(gr.shards()) == gpus
            outs = gr.run([x])
            # random weights could pass almost every anchor at a fixed threshold: take one that leaves a few hundred per image
            sc = _scores(outs, scales, zeros, 80)
            prob = float(np.max(np.quantile(sc, 1.0 - 300.0 / sc.shape[1], axis=1)))
            cands = (sc >= np.float32(prob)).sum(axis=1)
            assert cands.min() >= 50 and cands.max() <= 1000, cands
            got5 = gr.yolo_detect(V5_HEADS, num_classes=80, prob_threshold=prob, nms_threshold=0.45, max_per_image=1024, version=5)
            got3 = gr.yolo_detect(V5_HEADS, num_classes=80, prob_threshold=prob, nms_threshold=0.45, max_per_image=1024, version=3)
        finally:
            gr.close()
    finally:
        c.close()
    want5 = yolov5_post.detect(outs, scales, zeros, V5_HEADS, 80, prob, 0.45)
    _assert_same(got5, want5)
    assert sum(len(w) for w in want5) < cands.sum(), "NMS removed nothing"
    _assert_same(got3, yolo_post.detect(outs, scales, zeros, V5_HEADS, 80, prob, 0.45))


@pytest.mark.parametrize("version", [3, 5])
def test_errors(ctx, version):
    from tengine_b200 import runtime as rt

    rng = np.random.default_rng(3)
    heads, scales, zeros = _random_heads(rng, 80, False, 1, (6, 12, 24))
    with pytest.raises(rt.TB200Error, match="do not fit"):  # candidates beyond max_candidates are counted and reported
        _detect_on_device(ctx, heads, scales, zeros, V5_HEADS, version, 80, 0.1, 0.45, max_candidates=8)
    with pytest.raises(rt.TB200Error) as e:
        _detect_on_device(ctx, heads, scales, zeros, V5_HEADS, version, 79, 0.1, 0.45)
    assert e.value.code == abi.ERR_INVALID and "channels" in str(e.value)
