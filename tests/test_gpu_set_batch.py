"""Partial batches: tb200_graph_set_batch runs a prepared graph on images [0, n) of the batch it was prepared for.

- Every output at n equals the first n images of the full batch and the output of a graph prepared at n, bit for bit, for
  reduced MobileNet-v1 (int8 / uint8), ResNet-50 (uint8), YOLOv3-tiny (int8 / uint8) and YOLOv5s (int8); with
  TB200_PRERUN_NO_GRAPH every layer equals the oracle.
- The pipelined tb200_graph_run at n: two chunks (even n >= 32, a quarter split from 64) and one chunk.
- Nothing stale reaches an output and nothing beyond n images of a caller buffer is written (poisoned arena, guard bytes).
- Multi-GPU groups at every n, shards left without images included; tb200_graph_shard reports the active split.
- Pre- and post-processing at n: upload_images + topk, upload_detect_images + yolo_detect / yolov5_detect + detections_to_source.
- Errors leave the active batch and the results as they were; returning to the prepared batch gives the prerun results."""
import ctypes as C

import numpy as np
import pytest

from oracle import detect_pre as dp
from oracle import yolov5_post
from tengine_b200 import abi, workloads
from tests.helpers import layer_outputs
from tests.test_gpu_yolo_detect import _scores

pytestmark = pytest.mark.gpu

SEQUENCE = (8, 1, 3, 5, 8, 3)
V3_ANCHORS = [10, 14, 23, 27, 37, 58, 81, 82, 135, 169, 344, 319]
V5_HEADS = [(2, 32, yolov5_post.HEADS_BY_STRIDE[32]), (1, 16, yolov5_post.HEADS_BY_STRIDE[16]), (0, 8, yolov5_post.HEADS_BY_STRIDE[8])]
V3_HEADS = [(1, 32, V3_ANCHORS[6:12]), (0, 16, V3_ANCHORS[0:6])]

WORKLOADS = {
    "mobilenet_int8": lambda n: workloads.mobilenet_v1(abi.DT_INT8, batch=n, res=64, width=0.25, classes=40, seed=3),
    "mobilenet_uint8": lambda n: workloads.mobilenet_v1(abi.DT_UINT8, batch=n, res=64, width=0.25, classes=40, seed=3),
    "resnet50_uint8": lambda n: workloads.resnet50(abi.DT_UINT8, batch=n, res=64, width=0.25, classes=24, seed=5),
    "yolov3_tiny_int8": lambda n: workloads.yolov3_tiny(abi.DT_INT8, batch=n, res=96, width=0.25, head=27, seed=6),
    "yolov3_tiny_uint8": lambda n: workloads.yolov3_tiny(abi.DT_UINT8, batch=n, res=96, width=0.25, head=27, seed=6),
    "yolov5s_int8": lambda n: workloads.yolov5s(abi.DT_INT8, batch=n, res=256, width=0.25, seed=7),
}


def _devices(n):
    from tengine_b200 import runtime as rt

    have = rt.device_count()
    return [i % have for i in range(n)]


def _run_prepared_at(ctx, make, n, x, flags=abi.PRERUN_DEFAULT):
    from tengine_b200 import runtime as rt

    g, _ = make(n)
    gr = rt.Graph(ctx, g, flags)
    try:
        return gr.run([x])
    finally:
        gr.close()


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_outputs_at_n_equal_the_full_batch_and_a_graph_prepared_at_n(ctx, name):
    from tengine_b200 import runtime as rt

    make = WORKLOADS[name]
    g, b = make(8)
    x = b.random_input(11)
    gr = rt.Graph(ctx, g)
    try:
        assert gr.batch == 8
        full = gr.run([x])
        kernels = gr.layer_kernels()
        for n in SEQUENCE:
            gr.set_batch(n)
            assert gr.batch == n
            outs = gr.run([x[:n]])
            assert all(o.shape[0] == n for o in outs)
            for o, f in zip(outs, full):
                assert np.array_equal(o, f[:n]), (name, n)
            if n < 8:
                for o, p in zip(outs, _run_prepared_at(ctx, make, n, x[:n])):
                    assert np.array_equal(o, p), (name, n)
            assert gr.layer_kernels() == kernels
    finally:
        gr.close()


@pytest.mark.parametrize("dtype", [abi.DT_INT8, abi.DT_UINT8], ids=["int8", "uint8"])
def test_no_graph_every_layer_at_n_vs_oracle(ctx, oracle, dtype):
    from tengine_b200 import runtime as rt

    g, b = workloads.tiny_net(dtype, batch=8, seed=5)
    x = b.random_input(8)
    gr = rt.Graph(ctx, g, abi.PRERUN_NO_GRAPH)
    try:
        for n in SEQUENCE:
            gr.set_batch(n)
            outs = gr.run([x[:n]])
            tensors = {t: gr.read_tensor(t) for t in layer_outputs(g)}
            g_n, _ = workloads.tiny_net(dtype, batch=n, seed=5)
            want = oracle.run(g_n, [x[:n]], uint8_mode=0)
            for li, L in enumerate(g.layers):
                assert tensors[L["output"]].shape[0] == n
                assert np.array_equal(tensors[L["output"]], want[L["output"]]), (n, li, abi.OP_NAMES[L["op"]])
            for o, t in zip(outs, g.outputs):
                assert np.array_equal(o, want[t]), n
    finally:
        gr.close()


def test_pipelined_run_at_n_with_pageable_buffers(ctx):
    """Prepared at 64: n = 64 and 40 run as a quarter / three quarters and as two halves, 33 and 1 in one chunk, 32 as two halves."""
    from tengine_b200 import runtime as rt

    g, b = workloads.mobilenet_v1(abi.DT_INT8, batch=64, res=64, width=0.5, classes=100, seed=2)
    x = b.random_input(4)
    gr = rt.Graph(ctx, g)
    try:
        full = gr.run([x])[0]
        for n in (64, 40, 33, 32, 1, 40):
            gr.set_batch(n)
            xn = np.array(x[:n])  # a fresh pageable buffer of n images
            y = gr.run([xn])[0]
            assert y.shape[0] == n and np.array_equal(y, full[:n]), n
    finally:
        gr.close()


def _guarded(shape, dtype, fill, guard=4096):
    """An array of `shape` at the start of one allocation followed by `guard` bytes of 0x5C."""
    nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
    raw = np.full(nbytes + guard, 0x5C, np.uint8)
    view = raw[:nbytes].view(dtype).reshape(shape)
    view[...] = fill
    return raw, view


def _guard_intact(raw, view):
    return bool(np.all(raw[view.nbytes:] == 0x5C))


def test_no_stale_data_and_no_write_beyond_n_images(ctx):
    from tengine_b200 import runtime as rt

    g, b = workloads.mobilenet_v1(abi.DT_INT8, batch=8, res=64, width=0.25, classes=40, seed=3)
    xa, xb = b.random_input(1), b.random_input(2)
    gr = rt.Graph(ctx, g, abi.PRERUN_POISON_ARENA)
    try:
        want_b = gr.run([xb])[0]
        want_s, want_i = gr.topk(0, 5)
        gr.run([xa])
        out_t = g.outputs[0]
        for n in (3, 1, 7):
            gr.set_batch(n)
            raw_in, xin = _guarded((n,) + tuple(g.dims(g.inputs[0]))[1:], np.int8, xb[:n])
            raw_out, yout = _guarded((n,) + tuple(g.dims(out_t))[1:], np.int8, 0)
            gr.run([xin], [yout])
            assert np.array_equal(yout, want_b[:n]) and _guard_intact(raw_out, yout) and _guard_intact(raw_in, xin), n
            raw_dl, ydl = _guarded(yout.shape, np.int8, 0)
            gr.upload(0, xin)
            gr.launch()
            gr.download(0, ydl)
            gr.sync()
            assert np.array_equal(ydl, want_b[:n]) and _guard_intact(raw_dl, ydl), n
            raw_k, rec = _guarded((n, 5, 2), np.int32, 0)
            assert rt.lib().tb200_graph_topk(gr.h, 0, 5, rec.ctypes.data) == 0
            assert _guard_intact(raw_k, rec), n
            assert np.array_equal(rec[..., 1], want_i[:n]) and np.array_equal(rec[..., 0].view(np.float32).view(np.uint32),
                                                                                want_s[:n].view(np.uint32)), n
            gr.set_batch(8)
            gr.run([xa])  # the arena's images n.. now hold A's bytes again
    finally:
        gr.close()

    g, b = workloads.yolov3_tiny(abi.DT_UINT8, batch=5, res=160, width=0.5, seed=8)
    xa, xb = b.random_input(3), b.random_input(4)
    gr = rt.Graph(ctx, g, abi.PRERUN_POISON_ARENA)
    try:
        gr.run([xb])
        want = gr.yolo_detect(V3_HEADS, prob_threshold=0.27, nms_threshold=0.25, max_per_image=512)
        assert sum(len(w) for w in want) > 20
        gr.run([xa])
        n, m = 2, 512
        gr.set_batch(n)
        gr.run([xb[:n]])
        p = abi.YoloParams()
        p.num_heads = len(V3_HEADS)
        for i, (oi, stride, anchors) in enumerate(V3_HEADS):
            p.heads[i].output_index, p.heads[i].stride = oi, stride
            for k in range(6):
                p.heads[i].anchors[k] = anchors[k]
        p.num_classes, p.prob_threshold, p.nms_threshold = 80, 0.27, 0.25
        rec_size = C.sizeof(abi.Detection)
        raw_d, dets = _guarded((n * m * rec_size,), np.uint8, 0)
        raw_c, counts = _guarded((n,), np.int32, 0)
        fn = rt.lib().tb200_graph_yolo_detect
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        assert fn(gr.h, C.byref(p), dets.ctypes.data, m, counts.ctypes.data) == 0
        assert _guard_intact(raw_d, dets) and _guard_intact(raw_c, counts)
        recs = (abi.Detection * (n * m)).from_buffer(dets)
        for i in range(n):
            got = [(d.x, d.y, d.w, d.h, d.prob, d.label) for d in recs[i * m:i * m + counts[i]]]
            assert got == want[i], i
    finally:
        gr.close()


@pytest.mark.parametrize("ngpu,batch", [(2, 5), (3, 7), (4, 4)])
def test_multi_gpu_every_n(ngpu, batch):
    from tengine_b200 import runtime as rt

    mctx = rt.Context(devices=_devices(ngpu))
    try:
        g, b = workloads.tiny_net(abi.DT_INT8, batch=batch, seed=5)
        x = b.random_input(8)
        gr = rt.Graph(mctx, g)
        try:
            full = gr.run([x])
            full_s, full_i = gr.topk(0, 3)
            devs = [s[0] for s in gr.shards()]
            for n in list(range(1, batch + 1)) + [1, batch]:
                gr.set_batch(n)
                assert gr.shards() == [(devs[r],) + rt.shard_range(n, ngpu, r) for r in range(ngpu)], n
                outs = gr.run([x[:n]])
                for o, f in zip(outs, full):
                    assert np.array_equal(o, f[:n]), n
                s, i = gr.topk(0, 3)
                assert np.array_equal(i, full_i[:n]) and np.array_equal(s, full_s[:n]), n
        finally:
            gr.close()
    finally:
        mctx.close()


@pytest.mark.parametrize("shards", [1, 2])
def test_upload_images_and_topk_at_n(shards):
    from tengine_b200 import runtime as rt

    g, _ = workloads.mobilenet_v1(abi.DT_UINT8, batch=4, res=64, width=0.25, classes=40, seed=3)
    rng = np.random.default_rng(17)
    imgs = [rng.integers(0, 256, hwc, dtype=np.uint8) for hwc in ((80, 100, 3), (50, 40, 4), (64, 64, 3), (33, 90, 3))]
    mean, scale = (104.007, 116.669, 122.679), (0.017, 0.017, 0.017)
    c = rt.Context(devices=_devices(shards)) if shards > 1 else rt.Context(0)
    try:
        gr = rt.Graph(c, g)
        try:
            gr.upload_images(0, imgs, mean, scale)
            gr.launch()
            full_s, full_i = gr.topk(0, 5)
            for n in (1, 3, 2):
                gr.set_batch(n)
                gr.upload_images(0, imgs[:n], mean, scale)
                gr.launch()
                s, i = gr.topk(0, 5)
                assert s.shape == (n, 5)
                assert np.array_equal(i, full_i[:n]) and np.array_equal(s.view(np.uint32), full_s[:n].view(np.uint32)), n
                with pytest.raises(ValueError):
                    gr.upload_images(0, imgs[:n + 1], mean, scale)
        finally:
            gr.close()
    finally:
        c.close()


def _threshold(gr, g):
    """A threshold that keeps about 200 candidates of the busiest image of the last launch (the rule of the detection tests)."""
    outs = [np.empty(g.dims(t), g.np_dtype) for t in g.outputs]
    for i, o in enumerate(outs):
        gr.download(i, o)
    gr.sync()
    sc = _scores(outs, [np.float32(g.tensors[t]["scale"]) for t in g.outputs], [int(g.tensors[t]["zero_point"]) for t in g.outputs], 80)
    return float(np.max(np.quantile(sc, 1.0 - 200.0 / sc.shape[1], axis=1)))


def _geo_tuples(geo):
    return [(a.src_w, a.src_h, a.resize_w, a.resize_h, a.left, a.top, a.scale) for a in geo]


@pytest.mark.parametrize("shards", [1, 2])
@pytest.mark.parametrize("model", ["yolov5s_letterbox_focus", "yolov3_tiny_stretch"])
def test_detect_images_and_yolo_detect_at_n(model, shards):
    from tengine_b200 import runtime as rt

    rng = np.random.default_rng(29)
    imgs = [rng.integers(0, 256, hwc, dtype=np.uint8) for hwc in ((375, 500, 3), (300, 140, 4), (97, 120, 3), (200, 200, 3))]
    if model == "yolov5s_letterbox_focus":
        g, _ = workloads.yolov5s(abi.DT_INT8, batch=4, res=256, width=0.25, seed=7)
        heads, version, letterbox, focus = V5_HEADS, 5, True, True
    else:
        g, _ = workloads.yolov3_tiny(abi.DT_UINT8, batch=4, res=224, width=0.25, seed=9)
        heads, version, letterbox, focus = V3_HEADS, 3, False, False
    mean, scale = dp.DEFAULT_MEAN, dp.DEFAULT_SCALE
    c = rt.Context(devices=_devices(shards)) if shards > 1 else rt.Context(0)
    try:
        gr = rt.Graph(c, g)
        try:
            geo = gr.upload_detect_images(0, imgs, mean, scale, letterbox=letterbox, focus=focus)
            gr.launch()
            prob = _threshold(gr, g)
            full = gr.yolo_detect(heads, num_classes=80, prob_threshold=prob, nms_threshold=0.45, max_per_image=1024, version=version,
                                  geometry=geo, letterbox=letterbox)
            assert sum(len(d) for d in full) > 20, "test vacuous: nothing passes the threshold"
            full_geo = _geo_tuples(geo)
            for n in (1, 3):
                gr.set_batch(n)
                geo_n = gr.upload_detect_images(0, imgs[:n], mean, scale, letterbox=letterbox, focus=focus)
                assert len(geo_n) == n and _geo_tuples(geo_n) == full_geo[:n]
                gr.launch()
                got = gr.yolo_detect(heads, num_classes=80, prob_threshold=prob, nms_threshold=0.45, max_per_image=1024, version=version,
                                     geometry=geo_n, letterbox=letterbox)
                assert len(got) == n and got == full[:n], n
        finally:
            gr.close()
    finally:
        c.close()


def _two_batch_graph():
    """Two independent chains whose tensors have dim 0 = 2 and 3: not a plain batch dimension."""
    from tengine_b200.graphdef import GraphDef

    g = GraphDef(abi.DT_INT8)
    a = g.input(2, 16, 4, 4, 0.05, 0)
    bb = g.input(3, 16, 4, 4, 0.04, 0)
    g.mark_output(g.relu(a, 0.05, 0))
    g.mark_output(g.relu(bb, 0.04, 0))
    return g


def test_errors_leave_the_active_batch_and_results(ctx):
    from tengine_b200 import runtime as rt

    L = rt.lib()
    g, b = workloads.mobilenet_v1(abi.DT_INT8, batch=8, res=64, width=0.25, classes=40, seed=3)
    x = b.random_input(6)
    gr = rt.Graph(ctx, g)
    try:
        full = gr.run([x])[0]
        for active in (8, 3):
            gr.set_batch(active)
            for n in (0, -1, 9):
                assert L.tb200_graph_set_batch(gr.h, n) == abi.ERR_INVALID, n
                assert gr.batch == active
                assert np.array_equal(gr.run([x[:active]])[0], full[:active])
        assert L.tb200_graph_set_batch(None, 1) == abi.ERR_INVALID
        assert L.tb200_graph_batch(None) == abi.ERR_INVALID
    finally:
        gr.close()

    g2 = _two_batch_graph()
    rng = np.random.default_rng(3)
    xs = [rng.integers(-127, 128, (2, 16, 4, 4)).astype(np.int8), rng.integers(-127, 128, (3, 16, 4, 4)).astype(np.int8)]
    gr = rt.Graph(ctx, g2)
    try:
        want = gr.run(xs)
        assert gr.batch == 2
        assert L.tb200_graph_set_batch(gr.h, 1) == abi.ERR_UNSUPPORTED
        assert L.tb200_graph_set_batch(gr.h, 3) == abi.ERR_INVALID
        assert gr.batch == 2
        gr.set_batch(2)  # the prepared batch is always accepted
        for o, w in zip(gr.run(xs), want):
            assert np.array_equal(o, w)
    finally:
        gr.close()


def test_return_to_the_prepared_batch_and_repeated_calls(ctx):
    from tengine_b200 import runtime as rt

    g, b = workloads.mobilenet_v1(abi.DT_INT8, batch=8, res=64, width=0.25, classes=40, seed=3)
    x = b.random_input(9)
    gr = rt.Graph(ctx, g)
    try:
        full = gr.run([x])[0]
        launches, (ops, _) = gr.num_launches(), gr.work()
        for _ in range(2):
            gr.set_batch(3)
            gr.set_batch(3)  # no-op
            assert gr.batch == 3 and gr.num_launches() == launches
            assert gr.work()[0] == pytest.approx(ops * 3 / 8, rel=1e-12)
            assert np.array_equal(gr.run([x[:3]])[0], full[:3])
            gr.set_batch(8)
            assert gr.batch == 8 and gr.num_launches() == launches and gr.work()[0] == ops
            assert np.array_equal(gr.run([x])[0], full)
    finally:
        gr.close()
