"""Classification preprocessing on the device: tb200_graph_upload_images fills a graph input from decoded images.

- Identity graphs ([N, 3, H, W] -> IDENTITY -> output) return the filled input unchanged: every case of the committed output of the
  unmodified examples (tests/golden/image_pre_example.npz) is reproduced byte for byte.
- Seeded batches of mixed sizes and channel counts, lying in the pixel buffer out of order and with gaps, equal the restatement
  (oracle/image_pre.py) on one shard and on two (the device listed twice), from pageable and from page-locked (tb200_host_alloc) memory.
- Real MobileNet-v1 graphs, int8 and uint8: upload_images + launch + download gives what run gives on the restated input.
- Every invalid call returns its code before anything is copied, and the graph keeps working."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from oracle import image_pre
from tengine_b200 import abi, workloads

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "image_pre_example.npz")
_names = list(np.load(FIXTURE)["names"])


def _identity_graph(n, h, w, s_in, zp, u8, c=3):
    from tengine_b200.graphdef import GraphDef

    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    g.mark_output(g.identity(g.input(n, c, h, w, float(np.float32(s_in)), int(zp))))
    return g


def _context(shards):
    from tengine_b200 import runtime as rt

    return rt.Context(devices=[0] * shards) if shards > 1 else rt.Context(0)


def _pack(images, rng=None):
    """The images in one byte buffer: in reverse order with gaps when rng is given.  Returns (buffer bytes, descriptors)."""
    order = list(range(len(images)))[::-1] if rng is not None else list(range(len(images)))
    offs, off = [0] * len(images), 0
    for i in order:
        off += int(rng.integers(0, 40)) if rng is not None else 0
        offs[i] = off
        off += images[i].nbytes
    buf = np.zeros(off + 7, np.uint8)
    descs = (abi.Image * len(images))()
    for i, a in enumerate(images):
        buf[offs[i]:offs[i] + a.nbytes] = a.reshape(-1)
        descs[i].offset, descs[i].h, descs[i].w, descs[i].c = offs[i], a.shape[0], a.shape[1], a.shape[2]
    return buf, descs


def _upload_raw(gr, i, ptr, nbytes, descs, mean, scale):
    from tengine_b200 import runtime as rt

    m = (C.c_float * 3)(*[float(v) for v in mean])
    s = (C.c_float * 3)(*[float(v) for v in scale])
    return rt.lib().tb200_graph_upload_images(gr.h, i, ptr, nbytes, descs, m, s)


def _download(gr):
    out = np.empty(gr.gdef.dims(gr.gdef.outputs[0]), gr.gdef.np_dtype)
    gr.download(0, out)
    gr.sync()
    return out


@pytest.mark.parametrize("name", _names)
def test_identity_graph_reproduces_the_examples_committed_output(ctx, name):
    from tengine_b200 import runtime as rt

    d = np.load(FIXTURE)
    k = _names.index(name)
    H, W = (int(v) for v in d[f"hw_{k}"])
    s_in, zp, u8 = d[f"quant_{k}"]
    gr = rt.Graph(ctx, _identity_graph(1, H, W, np.float32(s_in), int(zp), bool(u8)))
    try:
        gr.upload_images(0, [d[f"pix_{k}"]], d[f"mean_{k}"], d[f"scale_{k}"])
        gr.launch()
        got = _download(gr)
    finally:
        gr.close()
    want = d[f"out_{k}"]
    assert got.dtype == want.dtype
    assert np.array_equal(got[0], want), int((got[0] != want).sum())


def _mixed_images(rng, n):
    imgs = []
    for i in range(n):
        h, w = (int(v) for v in rng.integers(2, 160, 2))
        imgs.append(rng.integers(0, 256, (h, w, 4 if i % 3 == 1 else 3), dtype=np.uint8))
    return imgs


@pytest.mark.parametrize("memory", ["pageable", "host_alloc"])
@pytest.mark.parametrize("shards", [1, 2])
@pytest.mark.parametrize("u8", [False, True], ids=["int8", "uint8"])
def test_mixed_batches_equal_the_restatement(u8, shards, memory):
    from tengine_b200 import runtime as rt

    rng = np.random.default_rng(7 + 2 * shards + u8 + (memory == "pageable") * 10)
    n, H, W = 5, 40, 56
    s_in, zp = np.float32(0.0215 if not u8 else 0.0195), (131 if u8 else 0)
    mean, scale = rng.uniform(90, 130, 3).astype(np.float32), rng.uniform(0.012, 0.02, 3).astype(np.float32)
    imgs = _mixed_images(rng, n)
    buf, descs = _pack(imgs, rng)
    pinned = None
    if memory == "host_alloc":
        pinned = rt.PinnedBuffer(buf.shape, np.uint8)
        pinned.array[:] = buf
        ptr = pinned.ptr
    else:
        ptr = buf.ctypes.data
    want = image_pre.preprocess_batch(imgs, H, W, mean, scale, s_in, zp, u8)
    c = _context(shards)
    try:
        gr = rt.Graph(c, _identity_graph(n, H, W, s_in, zp, u8))
        try:
            assert len(gr.shards()) == shards
            for _ in range(2):  # the second call reuses the staging buffers
                assert _upload_raw(gr, 0, ptr, buf.nbytes, descs, mean, scale) == 0, rt.lib().tb200_last_error()
                gr.launch()
                got = _download(gr)
                assert np.array_equal(got, want), [int((got[i] != want[i]).sum()) for i in range(n)]
            # a larger batch of pixels grows the staging buffer
            imgs2 = [rng.integers(0, 256, (300, 400 - 20 * i, 3), dtype=np.uint8) for i in range(n)]
            gr.upload_images(0, imgs2, mean, scale)
            gr.launch()
            assert np.array_equal(_download(gr), image_pre.preprocess_batch(imgs2, H, W, mean, scale, s_in, zp, u8))
        finally:
            gr.close()
    finally:
        c.close()
        if pinned is not None:
            pinned.free()


@pytest.mark.parametrize("shards", [1, 2])
@pytest.mark.parametrize("dtype", [abi.DT_INT8, abi.DT_UINT8], ids=["int8", "uint8"])
def test_real_mobilenet_v1_from_images_equals_run_on_the_restated_input(dtype, shards):
    from tengine_b200 import runtime as rt

    g, _ = workloads.mobilenet_v1(dtype, batch=4, res=224, width=0.25, classes=100, seed=5)
    t = g.tensors[g.inputs[0]]
    s_in, zp, u8 = np.float32(t["scale"]), int(t["zero_point"]), dtype == abi.DT_UINT8
    rng = np.random.default_rng(11 + shards)
    imgs = [rng.integers(0, 256, hwc, dtype=np.uint8) for hwc in ((375, 500, 3), (224, 224, 3), (260, 250, 4), (120, 97, 3))]
    mean, scale = image_pre.DEFAULT_MEAN, image_pre.DEFAULT_SCALE
    x = image_pre.preprocess_batch(imgs, 224, 224, mean, scale, s_in, zp, u8)
    assert len(np.unique(x)) > 100
    c = _context(shards)
    try:
        gr = rt.Graph(c, g)
        try:
            want = gr.run([x])[0]
            gr.upload_images(0, imgs, mean, scale)
            gr.launch()
            got = _download(gr)
        finally:
            gr.close()
    finally:
        c.close()
    assert np.array_equal(got, want)


def test_errors_leave_the_graph_usable(ctx):
    from tengine_b200 import runtime as rt

    rng = np.random.default_rng(3)
    s_in = np.float32(0.0215)
    gr = rt.Graph(ctx, _identity_graph(2, 16, 16, s_in, 0, False))
    try:
        imgs = [rng.integers(0, 256, (20, 30, 3), dtype=np.uint8) for _ in range(2)]
        buf, descs = _pack(imgs)
        mean, scale = image_pre.DEFAULT_MEAN, image_pre.DEFAULT_SCALE
        x = rng.integers(-127, 128, (2, 3, 16, 16)).astype(np.int8)

        def still_usable():
            assert np.array_equal(gr.run([x])[0], x)

        def with_desc(**kw):
            b, d = _pack(imgs)
            for k, v in kw.items():
                setattr(d[1], k, v)
            return _upload_raw(gr, 0, buf.ctypes.data, buf.nbytes, d, mean, scale)

        cases = [
            ("null pixels", abi.ERR_INVALID, lambda: _upload_raw(gr, 0, None, buf.nbytes, descs, mean, scale)),
            ("null images", abi.ERR_INVALID, lambda: _upload_raw(gr, 0, buf.ctypes.data, buf.nbytes, None, mean, scale)),
            ("input index", abi.ERR_INVALID, lambda: _upload_raw(gr, 1, buf.ctypes.data, buf.nbytes, descs, mean, scale)),
            ("negative index", abi.ERR_INVALID, lambda: _upload_raw(gr, -1, buf.ctypes.data, buf.nbytes, descs, mean, scale)),
            ("w 1", abi.ERR_INVALID, lambda: with_desc(w=1)),
            ("h 1", abi.ERR_INVALID, lambda: with_desc(h=1)),
            ("w 32768", abi.ERR_INVALID, lambda: with_desc(w=32768)),
            ("h 40000", abi.ERR_INVALID, lambda: with_desc(h=40000)),
            ("past the end", abi.ERR_INVALID, lambda: with_desc(offset=buf.nbytes - 20 * 30 * 3 + 1)),
            ("offset wraps", abi.ERR_INVALID, lambda: with_desc(offset=2 ** 64 - 16)),
            ("nan mean", abi.ERR_INVALID, lambda: _upload_raw(gr, 0, buf.ctypes.data, buf.nbytes, descs, (1.0, math.nan, 2.0), scale)),
            ("inf scale", abi.ERR_INVALID, lambda: _upload_raw(gr, 0, buf.ctypes.data, buf.nbytes, descs, mean, (0.017, 0.017, math.inf))),
            ("grey", abi.ERR_UNSUPPORTED, lambda: with_desc(c=1)),
            ("two channels", abi.ERR_UNSUPPORTED, lambda: with_desc(c=2)),
        ]
        for name, code, call in cases:
            assert call() == code, (name, rt.lib().tb200_last_error())
            still_usable()
        assert _upload_raw(gr, 0, buf.ctypes.data, buf.nbytes, descs, mean, scale) == 0
        gr.launch()
        assert np.array_equal(_download(gr), image_pre.preprocess_batch(imgs, 16, 16, mean, scale, s_in, 0, False))
    finally:
        gr.close()
    g4 = rt.Graph(ctx, _identity_graph(2, 16, 16, s_in, 0, False, c=4))
    try:
        assert _upload_raw(g4, 0, buf.ctypes.data, buf.nbytes, descs, mean, scale) == abi.ERR_INVALID
        assert "channels" in rt.lib().tb200_last_error().decode()
        x4 = rng.integers(-127, 128, (2, 4, 16, 16)).astype(np.int8)
        assert np.array_equal(g4.run([x4])[0], x4)
    finally:
        g4.close()
