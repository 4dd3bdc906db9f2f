"""Detection preprocessing on the device: tb200_graph_upload_detect_images fills a YOLO graph input from decoded images, and
tb200_detections_to_source maps the boxes back.

- Identity graphs ([N, 3, H, W] or [N, 12, H/2, W/2] -> IDENTITY -> output) return the filled input unchanged: every case of the
  committed fixture (tests/golden/detect_pre_example.npz) is reproduced byte for byte, and so is its geometry.
- Seeded batches of mixed sizes and channel counts, lying in the pixel buffer out of order and with gaps, equal the restatement
  (oracle/detect_pre.py) on one shard and on two (the device listed twice), from pageable and from page-locked memory.
- Real YOLOv5s (int8 and uint8, letterbox + Focus) and YOLOv3-tiny (uint8, stretch) graphs: upload_detect_images -> launch ->
  yolov5_detect / yolo_detect -> detections_to_source equals the host chain restated preprocessing -> run -> oracle/yolov5_post.py /
  yolo_post.py -> restated back-mapping.
- Every invalid call returns its code before anything is copied, and the graph keeps working."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from oracle import detect_pre as dp
from oracle import yolo_post, yolov5_post
from tengine_b200 import abi, workloads
from tests.test_gpu_yolo_detect import V3_ANCHORS, V5_HEADS, _assert_same, _scores

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "detect_pre_example.npz")
_names = list(np.load(FIXTURE)["names"])


def _identity_graph(n, c, h, w, s_in, zp, u8):
    from tengine_b200.graphdef import GraphDef

    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    g.mark_output(g.identity(g.input(n, c, h, w, float(np.float32(s_in)), int(zp))))
    return g


def _input_shape(n, H, W, focus):
    return (n, 12, H // 2, W // 2) if focus else (n, 3, H, W)


def _context(shards):
    from tengine_b200 import runtime as rt

    return rt.Context(devices=[0] * shards) if shards > 1 else rt.Context(0)


def _pack(images, rng=None):
    """The images in one byte buffer: in reverse order with gaps when rng is given.  Returns (buffer, descriptors)."""
    order = list(range(len(images)))[::-1] if rng is not None else list(range(len(images)))
    offs, off = [0] * len(images), 0
    for i in order:
        off += int(rng.integers(0, 40)) if rng is not None else 0
        offs[i] = off
        off += images[i].nbytes
    buf = np.zeros(off + 5, np.uint8)
    descs = (abi.Image * len(images))()
    for i, a in enumerate(images):
        buf[offs[i]:offs[i] + a.nbytes] = a.reshape(-1)
        descs[i].offset, descs[i].h, descs[i].w, descs[i].c = offs[i], a.shape[0], a.shape[1], a.shape[2]
    return buf, descs


def _pre(mode, focus, mean, scale):
    p = abi.DetectPre()
    p.mode, p.focus = mode, focus
    for k in range(3):
        p.mean[k], p.scale[k] = float(mean[k]), float(scale[k])
    return p


def _upload_raw(gr, i, ptr, nbytes, descs, pre, geo=None):
    from tengine_b200 import runtime as rt

    return rt.lib().tb200_graph_upload_detect_images(gr.h, i, ptr, nbytes, descs, C.byref(pre) if pre is not None else None, geo)


def _download(gr):
    out = np.empty(gr.gdef.dims(gr.gdef.outputs[0]), gr.gdef.np_dtype)
    gr.download(0, out)
    gr.sync()
    return out


def _geo_tuples(geo):
    return [(g.src_w, g.src_h, g.resize_w, g.resize_h, g.left, g.top, np.float32(g.scale)) for g in geo]


@pytest.mark.parametrize("name", _names)
def test_identity_graph_reproduces_the_fixture(ctx, name):
    from tengine_b200 import runtime as rt

    d = np.load(FIXTURE)
    k = _names.index(name)
    mode, H, W, focus, u8, zp = (int(v) for v in d[f"cfg_{k}"])
    img = d[f"pix_{k}"]
    gr = rt.Graph(ctx, _identity_graph(1, *_input_shape(1, H, W, focus)[1:], np.float32(d[f"sin_{k}"]), zp, bool(u8)))
    try:
        geo = gr.upload_detect_images(0, [img], d[f"mean_{k}"], d[f"scale_{k}"], letterbox=mode == dp.LETTERBOX, focus=bool(focus))
        gr.launch()
        got = _download(gr)
    finally:
        gr.close()
    want = d[f"out_{k}"]
    assert got.dtype == want.dtype
    assert np.array_equal(got[0], want), int((got[0] != want).sum())
    assert _geo_tuples(geo) == [dp.geometry(mode, img.shape[1], img.shape[0], W, H)]


def _mixed_images(rng, n, H, W):
    """Log-uniform sizes in 2..300, redrawn where the letterbox would leave no row or column (an invalid call)."""
    imgs = []
    while len(imgs) < n:
        h, w = (int(v) for v in np.exp(rng.uniform(np.log(2), np.log(300), 2)).round())
        if min(dp.geometry(dp.LETTERBOX, w, h, W, H)[2:4]) < 1:
            continue
        imgs.append(rng.integers(0, 256, (h, w, 4 if len(imgs) % 3 == 1 else 3), dtype=np.uint8))
    return imgs


@pytest.mark.parametrize("memory", ["pageable", "host_alloc"])
@pytest.mark.parametrize("shards", [1, 2])
@pytest.mark.parametrize("u8", [False, True], ids=["int8", "uint8"])
def test_mixed_batches_equal_the_restatement(u8, shards, memory):
    from tengine_b200 import runtime as rt

    rng = np.random.default_rng(17 + 2 * shards + u8 + (memory == "pageable") * 10)
    n, H, W = 5, 48, 64
    s_in, zp = np.float32(0.0079 if not u8 else 0.0041), (128 if u8 else 0)
    mean, scale = rng.uniform(0, 40, 3).astype(np.float32), rng.uniform(0.003, 0.005, 3).astype(np.float32)
    imgs = _mixed_images(rng, n, H, W)
    buf, descs = _pack(imgs, rng)
    pinned = None
    if memory == "host_alloc":
        pinned = rt.PinnedBuffer(buf.shape, np.uint8)
        pinned.array[:] = buf
        ptr = pinned.ptr
    else:
        ptr = buf.ctypes.data
    c = _context(shards)
    try:
        for mode, focus in ((dp.LETTERBOX, 1), (dp.STRETCH, 0)):
            want = dp.preprocess_batch(imgs, mode, H, W, mean, scale, s_in, zp, u8, bool(focus))
            gr = rt.Graph(c, _identity_graph(n, *_input_shape(n, H, W, focus)[1:], s_in, zp, u8))
            try:
                assert len(gr.shards()) == shards
                pre = _pre(mode, focus, mean, scale)
                for _ in range(2):  # the second call reuses the staging buffers
                    geo = (abi.DetectGeometry * n)()
                    assert _upload_raw(gr, 0, ptr, buf.nbytes, descs, pre, geo) == 0, rt.lib().tb200_last_error()
                    gr.launch()
                    got = _download(gr)
                    assert np.array_equal(got, want), [int((got[i] != want[i]).sum()) for i in range(n)]
                    assert _geo_tuples(geo) == [dp.geometry(mode, a.shape[1], a.shape[0], W, H) for a in imgs]
                # larger images grow the staging buffer
                imgs2 = [rng.integers(0, 256, (300, 400 - 20 * i, 3), dtype=np.uint8) for i in range(n)]
                gr.upload_detect_images(0, imgs2, mean, scale, letterbox=mode == dp.LETTERBOX, focus=bool(focus))
                gr.launch()
                assert np.array_equal(_download(gr), dp.preprocess_batch(imgs2, mode, H, W, mean, scale, s_in, zp, u8, bool(focus)))
            finally:
                gr.close()
    finally:
        c.close()
        if pinned is not None:
            pinned.free()


def _detect_chain(g, imgs, mode, focus, H, W, heads, version, post, shards):
    """(device chain, host chain) boxes in source pixels for images `imgs` through the real graph `g`."""
    from tengine_b200 import runtime as rt

    t = g.tensors[g.inputs[0]]
    s_in, zp, u8 = np.float32(t["scale"]), int(t["zero_point"]), g.np_dtype == np.uint8
    mean, scale = dp.DEFAULT_MEAN, dp.DEFAULT_SCALE
    x = dp.preprocess_batch(imgs, mode, H, W, mean, scale, s_in, zp, u8, focus)
    assert len(np.unique(x)) > 100
    geos = [dp.geometry(mode, a.shape[1], a.shape[0], W, H) for a in imgs]
    scales = [np.float32(g.tensors[o]["scale"]) for o in g.outputs]
    zeros = [int(g.tensors[o]["zero_point"]) for o in g.outputs]
    c = _context(shards)
    try:
        gr = rt.Graph(c, g)
        try:
            outs = gr.run([x])
            sc = _scores(outs, scales, zeros, 80)
            prob = float(np.max(np.quantile(sc, 1.0 - 200.0 / sc.shape[1], axis=1)))
            geo = gr.upload_detect_images(0, imgs, mean, scale, letterbox=mode == dp.LETTERBOX, focus=focus)
            gr.launch()
            got = gr.yolo_detect(heads, num_classes=80, prob_threshold=prob, nms_threshold=0.45, max_per_image=1024, version=version,
                                 geometry=geo, letterbox=mode == dp.LETTERBOX)
            assert _geo_tuples(geo) == geos
        finally:
            gr.close()
    finally:
        c.close()
    want = dp.detections_to_source(mode, geos, post.detect(outs, scales, zeros, heads, 80, prob, 0.45))
    assert sum(len(w) for w in want) > 20
    return got, want


@pytest.mark.parametrize("shards", [1, 2])
@pytest.mark.parametrize("dtype", [abi.DT_INT8, abi.DT_UINT8], ids=["int8", "uint8"])
def test_real_yolov5s_from_images_equals_the_host_chain(dtype, shards):
    g, _ = workloads.yolov5s(dtype, batch=3, res=256, width=0.25, seed=7)
    rng = np.random.default_rng(31 + shards)
    imgs = [rng.integers(0, 256, hwc, dtype=np.uint8) for hwc in ((375, 500, 3), (300, 140, 4), (97, 120, 3))]
    got, want = _detect_chain(g, imgs, dp.LETTERBOX, True, 256, 256, V5_HEADS, 5, yolov5_post, shards)
    _assert_same(got, want)


@pytest.mark.parametrize("shards", [1, 2])
def test_real_yolov3_tiny_from_images_equals_the_host_chain(shards):
    g, _ = workloads.yolov3_tiny(abi.DT_UINT8, batch=2, res=224, width=0.25, seed=9)
    rng = np.random.default_rng(41 + shards)
    imgs = [rng.integers(0, 256, hwc, dtype=np.uint8) for hwc in ((375, 500, 3), (120, 90, 4))]
    heads = [(1, 32, V3_ANCHORS[6:12]), (0, 16, V3_ANCHORS[0:6])]  # outputs: stride 16, then 32
    got, want = _detect_chain(g, imgs, dp.STRETCH, False, 224, 224, heads, 3, yolo_post, shards)
    _assert_same(got, want)


def test_errors_leave_the_graph_usable(ctx):
    from tengine_b200 import runtime as rt

    rng = np.random.default_rng(5)
    s_in = np.float32(0.0079)
    gr = rt.Graph(ctx, _identity_graph(2, 12, 8, 8, s_in, 0, False))
    try:
        imgs = [rng.integers(0, 256, (20, 30, 3), dtype=np.uint8) for _ in range(2)]
        buf, descs = _pack(imgs)
        mean, scale = dp.DEFAULT_MEAN, dp.DEFAULT_SCALE
        pre = _pre(dp.LETTERBOX, 1, mean, scale)
        x = rng.integers(-127, 128, (2, 12, 8, 8)).astype(np.int8)

        def still_usable():
            assert np.array_equal(gr.run([x])[0], x)

        def with_desc(**kw):
            b, d = _pack(imgs)
            for k, v in kw.items():
                setattr(d[1], k, v)
            return _upload_raw(gr, 0, buf.ctypes.data, buf.nbytes, d, pre)

        def with_pre(**kw):
            p = _pre(dp.LETTERBOX, 1, mean, scale)
            for k, v in kw.items():
                if k in ("mean", "scale"):
                    getattr(p, k)[1] = v
                else:
                    setattr(p, k, v)
            return _upload_raw(gr, 0, buf.ctypes.data, buf.nbytes, descs, p)

        thin = rng.integers(0, 256, (1500, 2, 3), dtype=np.uint8)  # letterboxes to 0 columns in 16 x 16
        tbuf, tdescs = _pack([imgs[0], thin])
        cases = [
            ("null pixels", abi.ERR_INVALID, lambda: _upload_raw(gr, 0, None, buf.nbytes, descs, pre)),
            ("null images", abi.ERR_INVALID, lambda: _upload_raw(gr, 0, buf.ctypes.data, buf.nbytes, None, pre)),
            ("null pre", abi.ERR_INVALID, lambda: _upload_raw(gr, 0, buf.ctypes.data, buf.nbytes, descs, None)),
            ("input index", abi.ERR_INVALID, lambda: _upload_raw(gr, 1, buf.ctypes.data, buf.nbytes, descs, pre)),
            ("negative index", abi.ERR_INVALID, lambda: _upload_raw(gr, -1, buf.ctypes.data, buf.nbytes, descs, pre)),
            ("mode", abi.ERR_INVALID, lambda: with_pre(mode=2)),
            ("focus 2", abi.ERR_INVALID, lambda: with_pre(focus=2)),
            ("no focus on 12 channels", abi.ERR_INVALID, lambda: with_pre(focus=0)),
            ("w 1", abi.ERR_INVALID, lambda: with_desc(w=1)),
            ("h 40000", abi.ERR_INVALID, lambda: with_desc(h=40000)),
            ("past the end", abi.ERR_INVALID, lambda: with_desc(offset=buf.nbytes - 20 * 30 * 3 + 1)),
            ("offset wraps", abi.ERR_INVALID, lambda: with_desc(offset=2 ** 64 - 16)),
            ("nan mean", abi.ERR_INVALID, lambda: with_pre(mean=math.nan)),
            ("inf scale", abi.ERR_INVALID, lambda: with_pre(scale=math.inf)),
            ("letterbox to nothing", abi.ERR_INVALID, lambda: _upload_raw(gr, 0, tbuf.ctypes.data, tbuf.nbytes, tdescs, pre)),
            ("grey", abi.ERR_UNSUPPORTED, lambda: with_desc(c=1)),
            ("two channels", abi.ERR_UNSUPPORTED, lambda: with_desc(c=2)),
        ]
        for name, code, call in cases:
            assert call() == code, (name, rt.lib().tb200_last_error())
            still_usable()
        assert _upload_raw(gr, 0, buf.ctypes.data, buf.nbytes, descs, pre) == 0
        gr.launch()
        assert np.array_equal(_download(gr), dp.preprocess_batch(imgs, dp.LETTERBOX, 16, 16, mean, scale, s_in, 0, False, True))
    finally:
        gr.close()
    g3 = rt.Graph(ctx, _identity_graph(2, 3, 16, 16, s_in, 0, False))
    try:
        assert _upload_raw(g3, 0, buf.ctypes.data, buf.nbytes, descs, _pre(dp.LETTERBOX, 1, mean, scale)) == abi.ERR_INVALID
        assert "channels" in rt.lib().tb200_last_error().decode()
        x3 = rng.integers(-127, 128, (2, 3, 16, 16)).astype(np.int8)
        assert np.array_equal(g3.run([x3])[0], x3)
        assert _upload_raw(g3, 0, buf.ctypes.data, buf.nbytes, descs, _pre(dp.STRETCH, 0, mean, scale)) == 0
        g3.launch()
        assert np.array_equal(_download(g3), dp.preprocess_batch(imgs, dp.STRETCH, 16, 16, mean, scale, s_in, 0, False, False))
    finally:
        g3.close()
